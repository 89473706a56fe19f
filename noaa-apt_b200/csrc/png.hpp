// The PNG encoder (DESIGN.md §11): filter, match candidates, greedy parse, package-merge Huffman codes, bit emission,
// Adler-32, CRC-32 and the PNG framing, all on the device.  This module alone reads apt_png_settings: it validates them,
// sizes the workspaces, launches the kernel sequence and leaves the file's bytes and length on the device.
#pragma once

#include <cstdint>

#include "aptb200.h"
#include "launch.hpp"

namespace aptb200 {

// Device control block of one encode; `total` is the file length the host reads back before copying the bytes.
struct PngCtl {
    u64 deflate_bits;   // bits of the deflate stream (all blocks)
    u64 total;          // bytes of the PNG file
    u32 crc_raw;        // XOR of the chunk contributions to the IDAT CRC (zero initial register, no final XOR)
    u32 adler;          // Adler-32 of the filtered stream
    u32 pad[2];
};

struct PngPlan {
    apt_png_settings s{};
    u32 width = 0, height = 0;
    int in_ch = 0, ch = 0;        // input channels; channels written (3 for rgb_from_rgba)
    u64 row = 0;                  // filtered bytes per row: 1 + width * ch
    u64 n = 0;                    // filtered stream length: height * row
    u32 nblocks = 0;
    u64 bound = 0;                // apt_png_bound
    unsigned char ihdr[25];       // the IHDR chunk, CRC included
};

// Argument rules (host only, APT_ERR_BAD_ARG) and the plan.  Alpha is not looked at here.
int make_png(uint32_t width, uint32_t height, int channels, const apt_png_settings *ps, PngPlan &plan);

// Device workspaces of the encoder; they grow to the largest image seen and are kept.
struct PngWork {
    unsigned char *f = nullptr;      // filtered stream (+16 bytes of padding)
    unsigned char *lcode = nullptr;  // per position: 0, or match length - 3
    uint16_t *dist = nullptr;        // per position: match distance - 1
    unsigned char *flag = nullptr;   // per position: 1 where the greedy parse emits a token
    u32 *hist = nullptr;             // per block: 286 literal/length + 30 distance counts
    u32 *codes = nullptr;            // per block: 286 + 30 packed codes (bit-reversed code | length << 16)
    u32 *hdr = nullptr;              // per block: the header bits (kPngHdrWords words)
    u32 *hdr_bits = nullptr;         // per block
    u64 *bits = nullptr;             // per block: header + tokens + end of block
    u64 *off = nullptr;              // per block: exclusive scan of bits
    u64 *sums = nullptr;             // per block: Adler partial sums (sum F, sum (block end - i) F[i])
    unsigned char *out = nullptr;    // the PNG file (bound bytes, rounded up to words)
    PngCtl *ctl = nullptr;
    u64 cap_n = 0, cap_n_pos = 0, cap_blocks = 0, cap_out = 0;   // bytes of f; positions of lcode / dist / flag; ...
    PngWork() = default;
    PngWork(const PngWork &) = delete;
    ~PngWork() { release(); }
    int reserve(const PngPlan &p);
    void release();
    size_t device_bytes() const;
};

// Enqueues the whole encode of `pixels` (device, height * width * in_ch bytes) on c.stream.  The file is at w.out, its
// length in w.ctl->total.
int png_encode_device(const LaunchCtx &c, const PngPlan &p, PngWork &w, const unsigned char *pixels, KernelHook *hook);

// Frees the per-device workspaces apt_png_encode keeps between calls (apt_cache_clear).
void png_stage_cache_clear();

// 1 if every alpha byte of an RGBA host image is 255 (the rgb_from_rgba rule for host pixels).
bool png_alpha_opaque(const uint8_t *pixels, uint64_t npx);

}  // namespace aptb200
