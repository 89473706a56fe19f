// Finding carriers in I/Q (DESIGN.md §10, "Finding carriers"): the averaged power spectrum on the device (k_spectrum),
// the host search over it (noise floor, band power, peaks, suppression, centroid) and the APT test of a candidate.
#pragma once

#include <cstdint>
#include <vector>

#include "aptb200.h"
#include "launch.hpp"

namespace aptb200 {

struct SpecPlan {
    u32 nfft = 0, log2n = 0;
    uint64_t S = 0, K = 0;        // whole segments, segments used
    std::vector<float> win;       // w[t] = 0.5 - 0.5 cos(2 pi t / nfft), in double, rounded once
    std::vector<float> tw;        // 2 * nfft interleaved exp(-2 pi i t / nfft), in double, rounded once
    // first sample of segment k < K: floor(k S / K) * nfft
    uint64_t start(uint64_t k) const {
        return static_cast<uint64_t>(static_cast<unsigned __int128>(k) * S / K) * nfft;
    }
};

// Validation (APT_ERR_BAD_ARG: nfft not a power of two in [256, 16384], fewer than nfft samples) and the tables.
// max_segments 0 means 2048.
int make_spectrum(uint64_t n, uint32_t nfft, uint32_t max_segments, SpecPlan &p);

// apt_carrier_search with its defaults filled in, checked against a recording at iq_rate (APT_ERR_BAD_ARG: inverted
// window).
struct SearchParams {
    int32_t lo = 0, hi = 0;       // both 0: the whole usable band
    uint32_t nfft = 0, max_segments = 0;
    double min_snr_db = 6.0;
};
int make_search(const apt_carrier_search *cs, uint32_t iq_rate, SearchParams &sp);

// The host search on an fftshifted spectrum of nfft bins at iq_rate: candidates sorted by descending snr_db, with
// apt_score 0 and is_apt 0 (the APT test needs the recording).
int search_carriers(const float *psd, uint32_t nfft, uint32_t iq_rate, float cutout, const SearchParams &sp,
                    std::vector<apt_carrier> &out);

// frees the per-device workspaces of apt_iq_spectrum / apt_iq_find_carriers (apt_cache_clear)
void spectrum_cache_clear();

}  // namespace aptb200
