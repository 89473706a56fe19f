/*
 * aptb200.h -- C ABI of the H100-native APT decode path.
 *
 * Drop-in boundary for the signal-to-image hot path of martinber/noaa-apt
 * v1.4.1 (src/{dsp,filters,decode,resample}.rs).  The reference has no FFI
 * boundary today (it is a single Rust binary crate), so every entry point
 * below names the Rust function whose body it replaces; the Rust-side shim
 * that binds them is in rust/ and INTEGRATION.md.  All signatures are plain
 * C: pointers, sizes, PODs -- no CUDA, torch or C++ types.
 *
 * Conventions
 *   - "host" entry points take ordinary host pointers, are synchronous and
 *     re-entrant (no hidden global state; each call picks its CUDA device).
 *   - `apt_decoder` is the explicit-state variant: it owns a device, a stream,
 *     device workspaces and pinned staging, and offers submit/wait so that a
 *     batch of independent recordings can be kept in flight one per stream.
 *   - Every function returns an `apt_status`.  A short human-readable message
 *     for the last failure on the calling thread is in apt_last_error().
 *   - There is NO CPU fallback: without a usable CUDA device the compute entry
 *     points fail with APT_ERR_CUDA.
 *   - Arithmetic is f32 like the reference; results match the reference's
 *     scalar CPU path to <= 1e-5 of the stage's max |value| (FMA contraction
 *     is the only difference), and sync positions match exactly.
 */
#ifndef APTB200_H
#define APTB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define APTB200_ABI_VERSION 1

/* ---------------------------------------------------------------- status */

/* Maps onto err::Error (err.rs:9-44).  1-4 are the four Error::Internal
 * conditions reachable on this path, 5 is Error::RateOverflow. */
typedef enum apt_status {
    APT_OK = 0,
    APT_ERR_RESAMPLE_TO_ZERO = 1, /* Internal("Can't resample to 0Hz")              dsp.rs:69-71     */
    APT_ERR_TOO_SHORT = 2,        /* Internal("Got less than 10 rows of samples..") decode.rs:79-83  */
    APT_ERR_FEW_SYNC_FRAMES = 3,  /* Internal("Found less than 5 sync frames...")   decode.rs:112-118*/
    APT_ERR_WORK_RATE = 4,        /* Internal("work_rate is not multiple of ...")   decode.rs:172-176*/
    APT_ERR_RATE_OVERFLOW = 5,    /* RateOverflow(...)                               dsp.rs:82-91     */
    APT_ERR_CUDA = 6,             /* CUDA runtime/driver failure, or no device (no CPU fallback)      */
    APT_ERR_BAD_ARG = 7,          /* inputs on which the reference panics (empty signal dsp.rs:367,
                                     even Kaiser window filters.rs:68-70, rate 0) or NULL pointers    */
    APT_ERR_NOMEM = 8,            /* host or device allocation failed                                 */
    APT_ERR_CAPACITY = 9,         /* caller's output buffer is too small (required size returned)     */
    APT_ERR_EMPTY_RESULT = 10,    /* Internal("Got zero samples after resampling...") resample.rs:46-52 */
    APT_ERR_IO = 11               /* Io / WavOpen (err.rs:11-17): a WAV file cannot be opened, parsed or written       */
} apt_status;

const char *apt_strerror(int status);
/* Message of the last failure on this thread ("" if none); valid until the next call on this thread. */
const char *apt_last_error(void);
int apt_abi_version(void);
/* Number of usable CUDA devices (0 if none / no driver).  Never fails. */
int apt_device_count(void);

/* -------------------------------------------------------------- settings */

/* The DSP fields of config::Settings (config.rs:85-98) -- the only part of the
 * settings that crosses the boundary (read at decode.rs:55-75,98). */
typedef struct apt_settings {
    uint32_t work_rate;           /* Hz */
    float resample_atten;         /* dB, positive */
    float resample_delta_freq;    /* Hz */
    float resample_cutout;        /* Hz */
    float demodulation_atten;     /* dB, positive */
} apt_settings;

/* "standard" profile, default_settings.toml:108-116. */
void apt_default_settings(apt_settings *s);
/* profile: "standard" | "fast" | "slow" (default_settings.toml:108-140). */
int apt_profile_settings(const char *profile, apt_settings *s);

/* --------------------------------------------------------------- filters */

/* filters.rs:18-46.  Frequencies are Freq values in fractions of pi rad/sample
 * (Freq::get_pi_rad, frequency.rs:80-82). */
typedef enum apt_filter_kind {
    APT_FILTER_NONE = 0,          /* filters::NoFilter          */
    APT_FILTER_LOWPASS = 1,       /* filters::Lowpass           */
    APT_FILTER_LOWPASS_DC = 2     /* filters::LowpassDcRemoval  */
} apt_filter_kind;

typedef struct apt_filter {
    int kind;                     /* apt_filter_kind */
    float cutout_pi;              /* cutout.get_pi_rad()  */
    float atten;                  /* dB, positive         */
    float delta_w_pi;             /* delta_w.get_pi_rad() */
} apt_filter;

/* Freq::hz(f, rate).get_pi_rad() -- frequency.rs:68-72. */
float apt_freq_hz(float f_hz, uint32_t rate_hz);
/* misc::bessel_i0 -- misc.rs:47-57. */
float apt_bessel_i0(float x);
/* Filter::resample(input_rate, output_rate) -- filters.rs:90-94,134-138 (no-op for NoFilter). */
void apt_filter_resample(apt_filter *f, uint32_t input_rate, uint32_t output_rate);
/* Filter::design() -- filters.rs:49-51,57-88,98-132 (+ kaiser :144-183).  Host code, no GPU.
 * Writes min(*n, cap) taps to out (out may be NULL when cap == 0) and the tap count to *n. */
int apt_filter_design(const apt_filter *f, float *out, size_t cap, size_t *n);

/* -------------------------------------------- stage entry points (host) */

/* Output length of dsp::resample_with_filter for `n` input samples (exact). */
int apt_resample_len(uint64_t n, uint32_t input_rate, uint32_t output_rate, const apt_filter *f,
                     uint64_t *nout);

/* dsp::resample_with_filter -- dsp.rs:62-126 (polyphase fast_resampling :186-289 when L > 1,
 * filter + decimate :105-123 when L == 1). */
int apt_resample_with_filter(const float *signal, uint64_t n, uint32_t input_rate, uint32_t output_rate,
                             const apt_filter *f, float *out, uint64_t cap, uint64_t *nout);

/* dsp::resample -- dsp.rs:132-162 (Lowpass with cutout = min(in,out)/2); the WAV->WAV tool path. */
int apt_resample(const float *signal, uint64_t n, uint32_t input_rate, uint32_t output_rate,
                 float atten, float delta_w_pi, float *out, uint64_t cap, uint64_t *nout);

/* dsp::demodulate -- dsp.rs:350-383.  carrier_pi = carrier_freq.get_pi_rad(). */
int apt_demodulate(const float *signal, uint64_t n, float carrier_pi, float *out);

/* dsp::filter -- dsp.rs:386-410 (causal, strict i > j). */
int apt_filter_signal(const float *signal, uint64_t n, const apt_filter *f, float *out);
/* Same with explicit coefficients. */
int apt_filter_taps(const float *signal, uint64_t n, const float *coeff, size_t ncoeff, float *out);

/* decode::generate_sync_frame -- decode.rs:171-199. */
int apt_generate_sync_frame(uint32_t work_rate, int8_t *out, size_t cap, size_t *n);

/* decode::find_sync -- decode.rs:204-263.  If corr != NULL it receives the n - guard_len
 * cross-correlation values (the Context::export_steps branch, decode.rs:235-237). */
int apt_find_sync(const float *signal, uint64_t n, uint32_t work_rate,
                  uint64_t *positions, size_t cap, size_t *npositions, float *corr);

/* ------------------------------------------------------- decode (host) */

/* Context::status(progress, description) -- context.rs:127-129.  Fired on the calling thread
 * at the reference's five points (decode.rs:63,87,93,107/136,154). */
typedef void (*apt_status_cb)(float progress, const char *description, void *user);

/* Upper bound, in floats, of decode()'s output for n input samples (rows * 2080). */
int apt_decode_len_bound(uint64_t n, uint32_t input_rate, const apt_settings *s, uint64_t *bound);

/* noaa_apt::decode == decode::decode -- decode.rs:43-162.
 * out receives rows*2080 f32 pixels; *nout the count.  cap in floats. */
int apt_decode(const float *signal, uint64_t n, uint32_t input_rate, const apt_settings *s, int sync,
               float *out, uint64_t cap, uint64_t *nout, apt_status_cb cb, void *user);

/* apt_decode / apt_decode_pcm16 keep the decoder they used (plan, device workspaces, pinned staging) parked per
 * (device, rate, settings) for the next call; this frees the parked ones, and the workspaces apt_png_encode keeps per
 * device.  Thread-safe. */
void apt_cache_clear(void);

/* Same, taking the PCM16 samples of the WAV directly: half the host->device bytes; the `as f32` cast of
 * wav::load_wav (wav.rs:31-40) happens on the device -- inside the resampler's load for the phase-major and generic
 * kernels (11025, 22050, 44100 Hz ...), as one conversion kernel in front of the uniform-tap / tiled kernels (48000,
 * 96000 Hz: +43 MB of HBM writes and reads per 15 minutes, which the PCIe saving outweighs 20 times). */
int apt_decode_pcm16(const int16_t *pcm, uint64_t n, uint32_t input_rate, const apt_settings *s, int sync,
                     float *out, uint64_t cap, uint64_t *nout, apt_status_cb cb, void *user);

/* ------------------------------------------------------ WAV files and the resample tool */

/* wav::load_wav -- wav.rs:11-56 (the `hound` reader restated for what this path needs): integer PCM of 8/16/24/32 bits or
 * 32-bit float, any number of channels; channel 0 is kept and integer samples are cast with `as f32` (raw values). */
typedef struct apt_wav_info {
    uint32_t sample_rate, channels, bits_per_sample, is_float;
    uint64_t frames;
} apt_wav_info;
int apt_wav_info_read(const char *path, apt_wav_info *info);
int apt_wav_load(const char *path, float *out, uint64_t cap, uint64_t *n, uint32_t *sample_rate);
/* The 16-bit samples as they are (for apt_decode_pcm16 / APT_PCM16: half the PCIe bytes, cast on the device). */
int apt_wav_load_pcm16(const char *path, int16_t *out, uint64_t cap, uint64_t *n, uint32_t *sample_rate);
/* 16-bit mono PCM file, what resample.rs:53-66 writes. */
int apt_wav_write_i16(const char *path, const int16_t *samples, uint64_t n, uint32_t sample_rate);
/* wav::write_wav's conversion for 16-bit files -- wav.rs:71-85: (sample / max * 32767.0) as i16 with max = dsp::get_max,
 * on the device; bit-identical to the reference given the same signal.  max is sample 0 if that is NaN, else the first
 * non-NaN sample equal to the largest value (-0.0 == +0.0: the first zero wins).  n < 2^32. */
int apt_quantize_i16(const float *signal, uint64_t n, int16_t *out);
/* resample::resample -- resample.rs:17-71: load WAV, dsp::resample (Lowpass, atten dB, delta_w in pi rad/sample) on the
 * GPU, normalise + quantise on the GPU, write a 16-bit WAV.  (The modification-time copy of resample.rs:30,68 is file
 * plumbing and stays with the caller.)  *nout receives the number of samples written. */
int apt_resample_wav(const char *input_path, const char *output_path, uint32_t output_rate, float atten, float delta_w_pi,
                     uint64_t *nout);

/* ------------------------------------------ image stage (after decode, on the device) */

/* The front of noaa_apt::process (noaa_apt.rs:132-190): contrast bounds, then map_signal_u8 (noaa_apt.rs:249-259).  The
 * rows stay on the device until they are u8 (4x fewer bytes leave the GPU).  Given the same f32 rows the results are
 * bit-identical to the reference's (every f32 operation rounded on its own, the reference's summation order). */
typedef enum apt_contrast {
    APT_CONTRAST_MINMAX = 0,      /* Contrast::MinMax: dsp::get_min / get_max             noaa_apt.rs:157-163, dsp.rs:20-54  */
    APT_CONTRAST_PERCENT = 1,     /* Contrast::Percent(p): misc::percent, 1000 buckets    misc.rs:119-175                    */
    APT_CONTRAST_TELEMETRY = 2,   /* Contrast::Telemetry: wedges 9 / 8 of the best frame  noaa_apt.rs:141-149, telemetry.rs  */
    APT_CONTRAST_HISTOGRAM = 3    /* Contrast::Histogram: MinMax bounds, then grey histogram equalisation per channel half
                                     (processing.rs:87-103, imageext.rs:23-46,95-119).  Only apt_process,
                                     apt_decode_image and apt_decoder_set_process_mode accept it. */
} apt_contrast;

typedef struct apt_image_info {
    float low, high;              /* contrast bounds: `low` maps to 0, `high` to 255 */
    uint64_t rows;                /* image height (width is 2080) */
    uint64_t telemetry_row;       /* telemetry: row where the best frame starts (telemetry.rs:192-221) */
    float wedges_a[16], wedges_b[16];   /* telemetry: Telemetry::values_a / values_b (telemetry.rs:30-66) */
} apt_image_info;

/* decode() + contrast + map_signal_u8 in one call: out receives rows*2080 u8 pixels (cap in bytes >= apt_decode_len_bound).
 * format: apt_sample_format of `signal` (f32 Signal or the WAV's PCM16).  Errors of the image stage: the reference's
 * Internal("Recording too short for telemetry decoding") and its panics (empty image, frame running off the image) come
 * back as APT_ERR_TOO_SHORT / APT_ERR_BAD_ARG. */
int apt_decode_image_u8(const void *signal, int format, uint64_t n, uint32_t input_rate, const apt_settings *s, int sync,
                        int contrast, float percent, uint8_t *out, uint64_t cap, uint64_t *nout, apt_image_info *info,
                        apt_status_cb cb, void *user);

/* Stage entry points on host buffers (rows = decode()'s output, n = rows*2080 values). */
/* noaa_apt::map_signal_u8 -- noaa_apt.rs:249-259. */
int apt_map_signal_u8(const float *signal, uint64_t n, float low, float high, uint8_t *out);
/* Contrast bounds of an image: MinMax / misc::percent / telemetry (info receives bounds, wedges, frame row).  Min and max
 * (MinMax, and Percent's range) are dsp::get_min / get_max's: pixel 0 for both if it is NaN; otherwise the first non-NaN
 * pixel equal to the smallest (largest) value, with its own bits (-0.0 == +0.0: the first zero wins).  NaN pixels map
 * to 0.  Fewer than 2^32 pixels. */
int apt_contrast_bounds(const float *signal, uint64_t n, int contrast, float percent, apt_image_info *info);
/* telemetry.rs:147-170: per-row means of the two telemetry bands and their pooled variance (n / 2080 values each). */
int apt_telemetry_rows(const float *signal, uint64_t n, float *mean_a, float *mean_b, float *variance);

/* The rest of noaa_apt::process (noaa_apt.rs:140-240) apart from the map overlay, on the device: contrast bounds ->
 * map_signal_u8 -> into_rgba8 -> false colour (processing.rs:108-157) -> grey histogram equalisation (processing.rs:87-103)
 * -> Rotate::Yes (processing.rs:21-37: both 909-px image rectangles turned by 180 degrees, sync / space / telemetry columns
 * kept).  Given the same f32 rows the image is bit-identical to the reference's.
 *   contrast  apt_contrast (APT_CONTRAST_HISTOGRAM included); percent is read for APT_CONTRAST_PERCENT only, in [0, 1]
 *   palette   NULL, or 256*256*3 bytes: the palette image after into_rgb8, row = channel B value, column = channel A value
 *   tune      ColorSettings::{ch_a_tune_start, ch_a_tune_end, ch_b_tune_start, ch_b_tune_end}
 *   rgba      0: grey output, 1 B/px (no palette allowed); 1: RGBA output, 4 B/px (alpha 255)
 * Colour + APT_CONTRAST_HISTOGRAM (the Lab branch, imageext.rs:50-63) is not available: APT_ERR_BAD_ARG.  The argument
 * rules are checked before any device is touched. */
typedef struct apt_process_settings {
    int contrast;
    float percent;
    int rotate;                   /* 0: Rotate::No, else Rotate::Yes */
    const uint8_t *palette;       /* 256*256*3 RGB or NULL */
    float tune[4];                /* ch_a start, ch_a end, ch_b start, ch_b end */
    int rgba;
} apt_process_settings;

/* process() on host rows (rows = decode()'s output, n = rows*2080 values): out receives rows*2080*(rgba ? 4 : 1) bytes,
 * *nout that count; cap in bytes. */
int apt_process(const float *rows, uint64_t n, const apt_process_settings *ps, uint8_t *out, uint64_t cap, uint64_t *nout,
                apt_image_info *info);
/* decode() + process() in one call; only the finished pixels leave the GPU.  cap in bytes >= apt_decode_len_bound * (rgba ? 4 : 1);
 * *nout receives the byte count.  Errors as apt_decode_image_u8. */
int apt_decode_image(const void *signal, int format, uint64_t n, uint32_t input_rate, const apt_settings *s, int sync,
                     const apt_process_settings *ps, uint8_t *out, uint64_t cap, uint64_t *nout, apt_image_info *info,
                     apt_status_cb cb, void *user);

/* ----------------------------------------------- decoder object (streams) */

typedef struct apt_decoder apt_decoder;

/* APT_F32 / APT_PCM16: audio samples.  APT_CU8 / APT_CF32 / APT_CS16: complex I/Q samples, interleaved I, Q (only the I/Q
 * entry points below take them; every other entry point that takes a format rejects them like an unknown format). */
typedef enum apt_sample_format {
    APT_F32 = 0,
    APT_PCM16 = 1,
    APT_CU8 = 2,                  /* unsigned 8-bit I/Q: rtl_sdr / librtlsdr */
    APT_CF32 = 3,                 /* complex float: GQRX I/Q recordings, the GNU Radio file sink */
    APT_CS16 = 4                  /* signed 16-bit I/Q: baseband WAVs of SDR# and SDR++ */
} apt_sample_format;

/* Creates a decoder bound to CUDA device `device` for recordings of `input_rate` Hz of up to
 * `max_samples` samples.  Designs both filters, uploads the taps and allocates every workspace
 * (nothing is allocated afterwards). */
int apt_decoder_create(int device, uint32_t input_rate, const apt_settings *s, uint64_t max_samples,
                       apt_decoder **dec);
void apt_decoder_destroy(apt_decoder *dec);

/* Enqueue one decode on the decoder's stream and return immediately.
 *   *_device: `signal` and `out` are device pointers on the decoder's device (inputs resident in HBM).
 *   *_host:   host pointers; the H2D of the samples and the D2H of the rows are part of the job
 *             (asynchronous when the buffers are pinned, e.g. from apt_host_alloc).
 * `cap` is the capacity of `out` in floats (>= apt_decode_len_bound).  One job in flight per decoder. */
int apt_decoder_submit_device(apt_decoder *dec, const void *signal, int format, uint64_t n, int sync,
                              float *out, uint64_t cap);
int apt_decoder_submit_host(apt_decoder *dec, const void *signal, int format, uint64_t n, int sync,
                            float *out, uint64_t cap);
/* Image mode of a decoder: contrast >= 0 (apt_contrast) makes every following submit produce the u8 image instead of the
 * f32 rows -- `out` is then a uint8_t buffer and `cap` / *nout count bytes; contrast < 0 switches back to f32 rows. */
int apt_decoder_set_image_mode(apt_decoder *dec, int contrast, float percent);
/* Process mode of a decoder: every following submit produces the image apt_process describes -- `out` is a uint8_t buffer,
 * `cap` and *nout count bytes (rows*2080*(rgba ? 4 : 1)).  The palette is copied to the device here, once.  NULL switches
 * back to f32 rows; apt_decoder_set_image_mode also leaves process mode. */
int apt_decoder_set_process_mode(apt_decoder *dec, const apt_process_settings *ps);
/* Sync mode of a decoder (DESIGN.md "Tracked sync").  Applies to every later submit with sync != 0, in every output
 * mode (rows, image, process, PNG); the default is APT_SYNC_PEAKS.
 *   APT_SYNC_PEAKS  the reference's picker (decode.rs:204-263), what `sync` means everywhere else.
 *   APT_SYNC_TRACK  tracked sync: the row period P = work_rate / 2 followed through the whole pass.  On the reference's
 *                   correlation c[0 .. ncorr), ncorr = N_w - template length:
 *     1. block k = [kP, min((k+1)P, ncorr)); m_k and the population deviation s_k of c over the block in double, each
 *        rounded once to float; z[i] = (c[i] - m_k) / s_k in float (z = 0 when s_k is 0 or not finite);
 *     2. S[i] = z[i] for i < P + delta, else S[i] = z[i] + max over d = -delta..delta of (S[i-P-d] - float(lambda d^2)),
 *        ties to the smaller |d|, then the negative d; before block k >= 2 the maximum S of block k-1 is subtracted from
 *        every S of blocks k-1 and k-2 (constant across every comparison, so no choice changes in exact arithmetic);
 *     3. from the argmax of S over [max(0, ncorr - P), ncorr) (first index on ties) walk back i <- i - P - d(i) while
 *        i >= P + delta; these indices, ascending, are the sync positions (apt_decoder_last_sync);
 *     4. rows as decode.rs:120-132 (every position but the last with p + row < N_w), at most floor(N_w / row) of them;
 *        fewer than 5 positions is APT_ERR_FEW_SYNC_FRAMES.
 *   Streams, watchers, batches and the one-shot entry points always use APT_SYNC_PEAKS. */
typedef enum apt_sync_mode { APT_SYNC_PEAKS = 0, APT_SYNC_TRACK = 1 } apt_sync_mode;
typedef struct apt_track_settings {
    uint32_t delta;   /* largest change of the row period between two rows, in work-rate samples: 1..8 */
    float lambda;     /* penalty per squared sample of change: finite, >= 0 */
} apt_track_settings;
/* delta 2, lambda 0.25. */
void apt_default_track_settings(apt_track_settings *ts);
/* ts == NULL takes the defaults.  Bad settings, an unknown mode, a job in flight or a decoder that cannot sync are
 * APT_ERR_BAD_ARG before any device is touched.  APT_SYNC_TRACK allocates the correlation, the per-index choices and room
 * for the positions once; APT_SYNC_PEAKS keeps them for a later switch back. */
int apt_decoder_set_sync_mode(apt_decoder *dec, int mode, const apt_track_settings *ts);
/* Contrast bounds / telemetry of the last image job (after apt_decoder_wait). */
int apt_decoder_image_info(apt_decoder *dec, apt_image_info *info);
/* 1 if the decoder's job has finished (apt_decoder_wait will not block) or none is in flight, else 0. */
int apt_decoder_poll(apt_decoder *dec);
/* Block until the job is finished; returns its status (APT_ERR_FEW_SYNC_FRAMES etc.) and *nout. */
int apt_decoder_wait(apt_decoder *dec, uint64_t *nout);

/* Introspection after a wait(): sync positions found (decode.rs:110), N_w, rows. */
int apt_decoder_last_sync(apt_decoder *dec, uint64_t *positions, size_t cap, size_t *npositions);
int apt_decoder_last_counts(apt_decoder *dec, uint64_t *n_work, uint64_t *n_rows, uint64_t *n_peaks);
/* Number of "roots" of the sync correlation the peak picker worked on in the last job (diagnostic). */
int apt_decoder_last_root_count(apt_decoder *dec, uint64_t *n_roots);
/* The roots themselves, ascending (a root is a correlation index p with no larger value in (p, p + min_distance]: the
 * only places a sync position can land -- DESIGN.md "Peak picker").  Diagnostic; valid after a wait() of a sync job. */
int apt_decoder_last_roots(apt_decoder *dec, uint64_t *roots, size_t cap, size_t *nroots);
/* What the sync record kernel wrote for the last job, tile by tile (DESIGN.md "Peak picker"): a tile is W consecutive
 * correlation positions (W = 1920, 1888, 1856 for pixel widths 3, 4, 5); its weak suffix records (no later position of the
 * tile is larger) and its strict prefix records (larger than every earlier position of the tile) are (position, value)
 * pairs, ascending.  tiles[t] receives the counts and the maximum of tile t; `records` the records of every tile in tile
 * order, each tile's suffix list then its prefix list.  At most tiles_cap / records_cap entries are written, *ntiles and
 * *nrecords are the totals (NULL buffers with cap 0 ask for the sizes).  Diagnostic; valid after a wait() of a sync job
 * that ran the record kernel and did not overflow its pool, else APT_ERR_BAD_ARG. */
typedef struct apt_tile_records {
    uint32_t n_suffix, n_prefix;  /* record counts of the tile */
    float max;                    /* maximum of the correlation over the tile */
} apt_tile_records;
typedef struct apt_record {
    uint32_t pos;                 /* correlation index */
    float val;                    /* correlation value */
} apt_record;
int apt_decoder_last_records(apt_decoder *dec, apt_tile_records *tiles, size_t tiles_cap, size_t *ntiles,
                             apt_record *records, size_t records_cap, size_t *nrecords);
/* Copy an intermediate signal of the last job back to the host (what Context::step would dump):
 * which = 0 "demodulation_result" input i.e. resample+envelope output, 1 "filter_result",
 * 2 "sync_correlation". */
int apt_decoder_read_stage(apt_decoder *dec, int which, float *out, uint64_t cap, uint64_t *n);

/* Per-kernel device time of the LAST job in milliseconds (CUDA events on the decoder's stream);
 * enable before submitting.  Names via apt_decoder_kernel_name(i).  Profiling adds event records
 * to the stream, so use it for roofline accounting, not inside a throughput measurement. */
int apt_decoder_set_profiling(apt_decoder *dec, int enabled);
int apt_decoder_kernel_count(apt_decoder *dec);
const char *apt_decoder_kernel_name(apt_decoder *dec, int i);
int apt_decoder_kernel_ms(apt_decoder *dec, float *ms, int cap, int *count);
/* The decoder's cudaStream_t, as an opaque pointer (for event timing by the caller). */
void *apt_decoder_stream(apt_decoder *dec);
/* Kernel launches issued by this decoder since creation. */
uint64_t apt_decoder_launch_count(apt_decoder *dec);

/* Binds the calling thread to the CPUs of the NUMA node CUDA device `device` hangs off (sysfs local_cpulist), so that
 * pinned buffers it allocates afterwards and its copy loops are local to the GPU's PCIe root.  1 if bound, 0 if the
 * topology is unknown / APTB200_NO_AFFINITY is set.  The library binds its own feeder and copy threads this way. */
int apt_bind_thread_to_device(int device);

/* Pinned host memory for asynchronous submit_host (cudaHostAlloc / cudaFreeHost). */
int apt_host_alloc(void **ptr, size_t bytes);
void apt_host_free(void *ptr);
/* Device memory on `device` (cudaMalloc / cudaFree) for submit_device users without a CUDA binding. */
int apt_device_alloc(int device, void **ptr, size_t bytes);
void apt_device_free(int device, void *ptr);
int apt_memcpy_h2d(int device, void *dst, const void *src, size_t bytes);
int apt_memcpy_d2h(int device, void *dst, const void *src, size_t bytes);

/* ----------------------------------------------------------- introspection */

/* Geometry of the tiled sm_90a resampler for a ratio L/M and a tap set (DESIGN.md "Tiled polyphase
 * kernel"); host code, no GPU.  usable == 0: the shape falls back to the generic kernel.  Optional
 * outputs: tile_taps (groups*group_stride floats; per group one sub-table per slice lane, slice_stride floats
 * apart, holding per loop iteration a 32-float record: taps of half A [4 samples][4 outputs], then half B) and
 * group_xs (groups entries: first input sample of each group relative to its row). */
typedef struct apt_tile_info {
    uint32_t usable, groups, p_out, p_in, usteps, row_len, rows_per_tile, smem_bytes, slices, slice_stride,
        half_taps, shift, iters, group_stride, ctas_per_sm, pair_pitch, halves, rows_per_copy;
} apt_tile_info;
int apt_tile_plan(uint32_t l, uint32_t m, const float *taps, size_t ntaps, apt_tile_info *info,
                  float *tile_taps, size_t cap_taps, uint32_t *group_xs, size_t cap_groups);

/* Geometry and tap stream of the uniform-tap resampler (noaa-apt_b200/csrc/kernels_ut.cuh), the kernel that serves
 * fast_resampling + demodulate when L == 13 (48/96/192 kHz -> 12 480 Hz): the taps travel as a kernel parameter.
 * Host logic only.  usable == 0: (l, m, taps) does not fit and the tiled / generic kernels are used.
 * A row q is the L outputs L*q .. L*q+L-1; pair p = outputs 2p, 2p+1; a chunk is chunk_len (8) consecutive samples of the row's
 * window (sample u of row q is signal[q*M + u]); pair p is active in chunks [cs[p], ce[p]).  Two warps share a block
 * of rows_per_block rows: role 0 owns pairs [0, ceil(np/2)), role 1 the rest.  `stream` (nvec float4 = 4*nvec floats;
 * role 1 starts at float4 index stream_b) holds, in the order the kernel's loop consumes them, per (chunk, active
 * pair) the 2*chunk_len taps {T[C*c][2p], T[C*c][2p+1], T[C*c+1][2p], ... T[C*c+C-1][2p+1]}, C = chunk_len, T[u][r] = h[u*L - r*M]; the order is
 * ramp-up (pairs pb..pb+a-1 over chunks [cs[pb+a-1], cs[pb+a])), steady (all pairs over [cs[last], ce[pb])), ramp-down
 * (pairs pb+a.. over [ce[pb+a-1], ce[pb+a])). */
typedef struct apt_ut_info {
    uint32_t usable, l, m, np, q, rows_per_block, vec, back, chunks, slot_floats, slot_stride, nslot, warps, smem_bytes,
        nvec, stream_b, halo_u0, halo_n, chunk_len;
    uint32_t cs[8], ce[8];
} apt_ut_info;
int apt_ut_plan(uint32_t l, uint32_t m, const float *taps, size_t ntaps, apt_ut_info *info, float *stream,
                size_t cap_stream);

/* Geometry and phase table of the phase-major resampler (noaa-apt_b200/csrc/kernels_ph.cuh), the kernel that serves
 * fast_resampling + demodulate for large interpolation factors (11025 / 22050 / 44100 Hz -> 12 480 Hz: L = 832 / 416 / 208).
 * Host logic only.  usable == 0: the shape does not fit.  Four consecutive phases (group g = r / 4) share a window of
 * jpad samples that starts at signal[m*q + xs[g] - 4]; output k = l*q + r is
 *     sum_{i < jpad} table[(g*jpad + i)*4 + r%4] * signal[m*q + xs[g] - 4 + i]   (samples outside the signal count as zero). */
typedef struct apt_ph_info {
    uint32_t usable, l, m, j, jpad, pitch, row_len, smem_bytes;
} apt_ph_info;
int apt_ph_plan(uint32_t l, uint32_t m, const float *taps, size_t ntaps, apt_ph_info *info, float *table, size_t cap_table,
                uint16_t *xs, size_t cap_xs);

/* ------------------------------------------------------------------ batch */

/* Decode `count` independent recordings (all at `input_rate`, same settings), sharded
 * recording i -> device devices[i % ndevices]; one feeder thread per device (bound to the device's NUMA node)
 * keeps streams_per_device jobs in flight and takes them back in completion order;
 * no inter-device communication.  signals[i]/lens[i] are host buffers; outs[i] (capacity caps[i]
 * floats) receive the rows, nouts[i] the counts and statuses[i] the per-recording status.
 * Returns APT_OK if every recording decoded, else the first failing status. */
int apt_decode_batch(const void *const *signals, int format, const uint64_t *lens, int count,
                     uint32_t input_rate, const apt_settings *s, int sync,
                     float *const *outs, const uint64_t *caps, uint64_t *nouts, int *statuses,
                     const int *devices, int ndevices, int streams_per_device);

/* ------------------------------------------------------------------ streaming decoder */

/* Live decoding: push audio as it arrives, get finished image rows back.
 *
 * The rows returned by the pushes plus apt_stream_finish, concatenated, are bit-identical to apt_decode /
 * apt_decode_pcm16 on the whole recording with the same settings and `sync`, however the recording is split into pushes
 * (any sizes, f32 and PCM16 mixed).  After finish, apt_stream_sync_positions equals apt_decoder_last_sync.  finish returns
 * the status apt_decode would return (APT_ERR_TOO_SHORT, APT_ERR_FEW_SYNC_FRAMES); the rows already returned are then
 * not an image apt_decode would produce and the caller discards them.
 *
 * Emission rule: rows leave as soon as they are final, within `latency_work` work-rate samples.  With sync, after a push
 * every row k with max(p_k + row, p_{k+1} + G) + latency_work <= work_final has been returned (p_k: sync position k,
 * row: samples per row, G: template length); without sync, every row r with (r+1)*row + latency_work <= work_final.
 *
 * Device memory is allocated by apt_stream_create, where it depends only on (input_rate, settings, max_push), and by
 * apt_stream_set_process_mode / apt_stream_set_png_mode (image output, below); push and finish allocate nothing.  Pushes
 * are synchronous (the rows are in `rows` on return) and take pageable host pointers;
 * pushes larger than max_push are split into steps of max_push samples.  Supported: the standard, fast and slow
 * profiles (any settings whose demodulation low-pass has 37, 43 or 61 taps) at every input rate apt_decode accepts,
 * with a work rate that is a multiple of 4160.  sync with another work rate fails with APT_ERR_WORK_RATE, sync = 0
 * with APT_ERR_BAD_ARG. */
typedef struct apt_stream apt_stream;
typedef struct apt_stream_info {
    uint64_t samples_in;      /* input samples pushed so far */
    uint64_t work_final;      /* envelope samples that no later input can change */
    uint64_t rows_out;        /* rows returned so far */
    uint64_t peaks;           /* sync positions decided so far */
    uint64_t latency_work;    /* slack of the emission rule, in work-rate samples (constant per stream) */
    uint64_t max_push;        /* samples one internal step takes; larger pushes are split */
    uint64_t device_bytes;    /* device memory the stream owns (image output included; changes only when a mode is set) */
} apt_stream_info;

int apt_stream_create(int device, uint32_t input_rate, const apt_settings *s, int sync, uint64_t max_push, apt_stream **st);
void apt_stream_destroy(apt_stream *st);
/* rows * 2080: the floats one push of n samples can return at most (the `cap` that push needs). */
int apt_stream_push_bound(apt_stream *st, uint64_t n, uint64_t *cap_floats);
/* format: APT_F32 or APT_PCM16.  APT_ERR_CAPACITY (cap below apt_stream_push_bound) leaves the stream unchanged, so the
 * push can be retried.  A push after finish (before reset), or one that takes the work-rate index past 2^32 - 1, is
 * APT_ERR_BAD_ARG. */
int apt_stream_push(apt_stream *st, const void *samples, int format, uint64_t n, float *rows, uint64_t cap, uint64_t *nout);
/* End of the recording: the remaining rows (cap: apt_stream_push_bound(st, 0)) and the status of the whole decode. */
int apt_stream_finish(apt_stream *st, float *rows, uint64_t cap, uint64_t *nout);
/* Start a new recording with the same plan and buffers. */
int apt_stream_reset(apt_stream *st);
/* Sync positions decided so far (positions == NULL: count only; APT_ERR_CAPACITY when cap is too small). */
int apt_stream_sync_positions(apt_stream *st, uint64_t *positions, size_t cap, size_t *n);
int apt_stream_get_info(apt_stream *st, apt_stream_info *info);
/* Host only, no device: the geometry a stream of these parameters would have (latency_work, max_push, device_bytes). */
int apt_stream_geometry(uint32_t input_rate, const apt_settings *s, int sync, uint64_t max_push, apt_stream_info *info);


/* ------------------------------------------------------------------ I/Q input: FM demodulation on the device */

/* Decoding straight from SDR I/Q (DESIGN.md §10; the reference has no I/Q path, so this stage is the project's own
 * definition).  One fused kernel loads the I/Q (APT_CU8 (u - 127.5), APT_CS16, APT_CF32), mixes the channel at offset_hz
 * to 0 Hz, runs the channel Lowpass (filters::Lowpass designed at iq_rate) decimated by D = iq_rate / audio_rate, and
 * discriminates: a[0] = 0, a[m] = atan2f(Im(z[m] conj z[m-1]), Re(..)) * audio_rate / 2pi, the instantaneous frequency
 * in Hz.  Output m reads inputs <= m*D only; its arithmetic depends on m and the input values alone, never on how the
 * input is split into chunks.  n counts complex samples. */
typedef struct apt_iq_settings {
    uint32_t iq_rate;             /* complex samples per second */
    uint32_t audio_rate;          /* discriminator output rate; must divide iq_rate */
    int32_t offset_hz;            /* signal centre minus tuned centre */
    float cutout, delta_freq, atten;   /* channel Lowpass: Hz, Hz, dB */
} apt_iq_settings;

/* cutout 22 kHz, delta_freq 8 kHz, atten 40 dB; audio_rate the smallest iq_rate / D that is >= 48 kHz.  APT_ERR_BAD_ARG
 * when no D >= 1 gives that or the settings fail the checks of apt_fm_demod_len. */
int apt_iq_default_settings(uint32_t iq_rate, int32_t offset_hz, apt_iq_settings *s);
/* Audio samples of n I/Q samples: ceil(n / D).  Host only.  APT_ERR_BAD_ARG unless iq_rate % audio_rate == 0,
 * cutout > 0, delta_freq > 0, atten > 8, cutout < audio_rate / 2, |offset_hz| + cutout < iq_rate / 2 and the channel
 * filter has at most 8191 taps. */
int apt_fm_demod_len(uint64_t n, const apt_iq_settings *s, uint64_t *nout);
/* The stage alone: host I/Q in, host audio (f32, Hz) out; cap in floats.  A cf32 sample with a NaN or Inf component (or
 * one whose mixed value overflows) counts as 0 + 0j, so the audio is the same bits whatever the chunk size. */
int apt_fm_demod(const void *iq, int format, uint64_t n, const apt_iq_settings *s, float *out, uint64_t cap,
                 uint64_t *nout);
/* Several channels of one I/Q input: outs[c] (cap floats each) receives apt_fm_demod with offset_hz = offsets[c], bit for
 * bit, and *nout the audio length of every channel.  Each chunk of I/Q is uploaded once and demodulated for every channel in
 * one kernel launch.  s->offset_hz is ignored.  Argument errors (NULL pointers, count outside 1..8, an offset failing
 * |offset| + cutout < iq_rate / 2 or any other check of apt_fm_demod_len, an unknown format, and cap below the audio
 * length: APT_ERR_CAPACITY) come back before any device is touched. */
int apt_fm_demod_channels(const void *iq, int format, uint64_t n, const apt_iq_settings *s, const int32_t *offsets,
                          int count, float *const *outs, uint64_t cap, uint64_t *nout);
/* apt_decode at s->audio_rate of the audio apt_fm_demod would return, produced on the device: the I/Q is uploaded in
 * chunks and the audio never leaves the GPU.  Rows, status and sync positions equal apt_decode(apt_fm_demod(iq)).
 * cap in floats >= apt_decode_len_bound(ceil(n / D), audio_rate). */
int apt_decode_iq(const void *iq, int format, uint64_t n, const apt_iq_settings *s, const apt_settings *settings, int sync,
                  float *out, uint64_t cap, uint64_t *nout, apt_status_cb cb, void *user);
/* Live decoding from a radio: a stream (apt_stream_push / finish / reset / ... as above) whose pushes are I/Q samples of
 * APT_CU8, APT_CS16 or APT_CF32, mixed freely; audio pushes are APT_ERR_BAD_ARG, as are I/Q pushes to an audio stream.
 * max_push and apt_stream_push_bound's n count I/Q samples.  Every push is converted into a cf32 window on the device that
 * keeps the N - 1 + D samples the next audio output reads; the FM kernel writes each audio sample as soon as its input is
 * complete.  The rows, positions and status equal apt_decode_iq on the whole input.  samples_in counts I/Q samples,
 * device_bytes includes the I/Q window; work_final, latency_work and the emission rule are the audio stream's. */
int apt_stream_create_iq(int device, const apt_iq_settings *iq, const apt_settings *s, int sync, uint64_t max_push,
                         apt_stream **st);
int apt_stream_geometry_iq(const apt_iq_settings *iq, const apt_settings *s, int sync, uint64_t max_push,
                           apt_stream_info *info);
/* A 2-channel 16-bit PCM WAV (SDR# / SDR++ baseband) as interleaved APT_CS16: out receives 2 * *n int16, *n the frames
 * (complex samples), cap in int16.  Any other layout is APT_ERR_IO. */
int apt_wav_load_iq16(const char *path, int16_t *out, uint64_t cap, uint64_t *n, uint32_t *sample_rate);

/* ------------------------------------------------------------------ I/Q input: finding the carriers */

/* The averaged power spectrum of an I/Q recording (DESIGN.md §10, "Finding carriers").  With S = floor(n / nfft) whole
 * segments and K = min(S, max_segments), segment k < K starts at sample floor(k S / K) nfft.  Each is loaded like
 * apt_fm_demod loads it, multiplied by the periodic Hann window 0.5 - 0.5 cos(2 pi t / nfft) and transformed; psd[b],
 * b < nfft, is the average of |X|^2 over the K segments in fftshift order: bin b is (b - nfft/2) iq_rate / nfft Hz.
 * Only the K segments cross PCIe.  The result is the same bits on every run.  *nseg receives K.  APT_ERR_BAD_ARG (NULL
 * pointers, an unknown format, nfft not a power of two in [256, 16384], fewer than nfft samples) and APT_ERR_CAPACITY
 * (cap < nfft) come back before any device is touched. */
typedef struct apt_spectrum_settings {
    uint32_t nfft;                /* power of two, 256 ... 16384 */
    uint32_t max_segments;        /* 0: 2048 */
} apt_spectrum_settings;
int apt_iq_spectrum(const void *iq, int format, uint64_t n, uint32_t iq_rate, const apt_spectrum_settings *ss,
                    float *psd, uint64_t cap, uint32_t *nseg);

/* Where to look for carriers.  Zero fields take the defaults. */
typedef struct apt_carrier_search {
    int32_t lo_hz, hi_hz;         /* search window relative to the tuned centre; 0, 0: the whole usable band */
    uint32_t nfft;                /* 0: smallest power of two with bin width <= 200 Hz, capped at 16384 */
    uint32_t max_segments;        /* 0: 2048 */
    float min_snr_db;             /* 0: 6 dB */
} apt_carrier_search;
typedef struct apt_carrier {
    int32_t offset_hz;            /* round(centre_hz); ready for apt_iq_settings.offset_hz */
    float centre_hz, snr_db;
    float apt_score;              /* fraction of the demodulated audio's power between 300 Hz and 4.8 kHz */
    int is_apt;                   /* apt_score >= 0.5 */
} apt_carrier;
/* Carriers in an I/Q recording: the spectrum above; the noise floor, the median of psd over the window; the band power
 * E(f), the sum of psd within +-20 kHz of f; a candidate at each local maximum of E in the window (the window clipped so
 * that |f| + s->cutout < iq_rate / 2) with snr_db = 10 log10(E / (floor bins_in_band)) >= min_snr_db; candidates taken
 * by descending E, each one within 40 kHz of a kept one dropped; centre_hz the floor-subtracted, power-weighted centroid
 * of the bins within +-20 kHz of the peak.  Each returned carrier is then FM-demodulated (4 s from the middle of the
 * recording at offset_hz, s's channel filter) and the audio's spectrum gives apt_score.  out receives the carriers by
 * descending snr_db; *count the full number: more than cap is APT_ERR_CAPACITY (out may be NULL when cap is 0).
 * s->offset_hz is ignored.  Argument errors (as apt_iq_spectrum, the checks of apt_fm_demod_len on s, an inverted
 * window) come back before any device is touched. */
int apt_iq_find_carriers(const void *iq, int format, uint64_t n, const apt_iq_settings *s, const apt_carrier_search *cs,
                         apt_carrier *out, uint32_t cap, uint32_t *count);
/* The search of apt_iq_find_carriers alone, on a spectrum the caller has (nfft bins in apt_iq_spectrum's order): host
 * only, no device; apt_score and is_apt are 0.  cs->nfft and cs->max_segments are not read. */
int apt_find_carriers_psd(const float *psd, uint32_t nfft, uint32_t iq_rate, float cutout, const apt_carrier_search *cs,
                          apt_carrier *out, uint32_t cap, uint32_t *count);

/* Several channels of one recording: channel c equals apt_decode_iq with offset_hz = offsets[c], bit for bit (rows,
 * nouts[c], statuses[c]).  Each chunk of I/Q is uploaded once and demodulated once per channel, into that channel's
 * decoder; the channels' decodes then run side by side.  outs[c] / caps[c] as apt_decode_iq's out / cap; a cap below the
 * bound is APT_ERR_CAPACITY for that channel alone.  Argument errors of any channel (NULL pointers, count < 1, an offset
 * failing |offset| + cutout < iq_rate / 2, and the errors apt_decode_iq decides from lengths) come back before any device
 * is touched, with every status set to the error.  Returns APT_OK or the first failing status. */
int apt_decode_iq_channels(const void *iq, int format, uint64_t n, const apt_iq_settings *s, const int32_t *offsets,
                           int count, const apt_settings *settings, int sync,
                           float *const *outs, const uint64_t *caps, uint64_t *nouts, int *statuses);
/* apt_iq_find_carriers, then apt_decode_iq_channels on the carriers with is_apt: found receives those carriers in
 * apt_iq_find_carriers' order, at most cap_found of them, *nfound their number, and outs[i] / nouts[i] / statuses[i]
 * (cap_found entries each) belong to found[i].  No APT carrier: APT_OK with *nfound = 0.  The decode's argument errors are
 * checked before any device is touched, on offset 0. */
int apt_decode_iq_auto(const void *iq, int format, uint64_t n, const apt_iq_settings *s, const apt_carrier_search *cs,
                       const apt_settings *settings, int sync, apt_carrier *found, uint32_t cap_found, uint32_t *nfound,
                       float *const *outs, const uint64_t *caps, uint64_t *nouts, int *statuses);

/* ------------------------------------------------------------------ PNG output: encoding on the device */

/* A deterministic PNG encoder (DESIGN.md §11; the reference's `img.save` pins no encoder, so the bytes are this project's
 * definition): per-row adaptive filter (minimum sum of absolute residuals, ties to the lower type), greedy LZ77 with zlib's
 * 15-bit hash, a 32 KiB window and matches of 4..258 bytes, one dynamic-Huffman deflate block per block_bytes of the
 * filtered stream with package-merge code lengths, zlib framing, and a PNG of IHDR, one IDAT and IEND.  The output bytes
 * are a pure function of the pixels and the settings.  8-bit grey (1 channel), RGB (3) or RGBA (4); no interlace.
 *   filter         -1: adaptive per row; 0..4: that PNG filter on every row
 *   matches        0: literals only (Huffman-only deflate); else LZ77 matches
 *   block_bytes    filtered bytes per deflate block: a power of two in [4096, 65536]
 *   rgb_from_rgba  1: RGBA input is written as RGB (colour type 2); every alpha must be 255, else APT_ERR_BAD_ARG */
typedef struct apt_png_settings {
    int filter;
    int matches;
    uint32_t block_bytes;
    int rgb_from_rgba;
} apt_png_settings;

/* filter -1, matches 1, block_bytes 65536, rgb_from_rgba 0. */
void apt_png_default_settings(apt_png_settings *ps);
/* Upper bound of the PNG size in bytes (host only): 63 + ceil(sum over blocks of (9 * len + 2409) / 8). */
int apt_png_bound(uint32_t width, uint32_t height, int channels, const apt_png_settings *ps, uint64_t *bytes);
/* PNG of host pixels (height rows of width * channels bytes).  out receives the file's bytes, *nout their count; a cap
 * below that count is APT_ERR_CAPACITY with the required count in *nout (cap >= apt_png_bound always suffices).  Argument
 * errors (NULL pointers, channels not 1 / 3 / 4, width or height 0, bad settings, alpha != 255 with rgb_from_rgba, an
 * IDAT that could exceed 2^31 - 1 bytes) come back before any device is touched.  The device workspace (about 5 bytes per
 * filtered byte plus the bound) is kept per device for the next call, one encode per device at a time; apt_cache_clear
 * frees it. */
int apt_png_encode(const uint8_t *pixels, uint32_t width, uint32_t height, int channels, const apt_png_settings *ps,
                   uint8_t *out, uint64_t cap, uint64_t *nout);
/* apt_png_encode of `count` host images of one width, channel count and settings, heights[k] rows each, in one batched
 * encode (one launch sequence for the group): outs[k] receives exactly the bytes apt_png_encode gives for image k alone.
 * A file larger than caps[k] is APT_ERR_CAPACITY with the required count in nouts[k]; the others are still written.
 * Returns the first failing status.  apt_png_encode is this call with count 1 and shares its per-device workspace. */
int apt_png_encode_batch(const uint8_t *const *pixels, const uint32_t *heights, uint32_t count, uint32_t width,
                         int channels, const apt_png_settings *ps, uint8_t *const *outs, const uint64_t *caps,
                         uint64_t *nouts);
/* apt_decode_image + apt_png_encode in one call: the image is encoded on the device and only the PNG bytes cross PCIe.
 * Errors as apt_decode_image, plus the settings checks of apt_png_encode and APT_ERR_CAPACITY as there. */
int apt_decode_png(const void *signal, int format, uint64_t n, uint32_t input_rate, const apt_settings *s, int sync,
                   const apt_process_settings *ps, const apt_png_settings *png, uint8_t *out, uint64_t cap, uint64_t *nout,
                   apt_image_info *info, apt_status_cb cb, void *user);
/* PNG mode of a decoder in process or image mode: every following job ends in the PNG of its image; `out` / `cap` / *nout
 * of submit and wait then count PNG bytes (cap >= apt_png_bound of the largest image suffices; a smaller one that the
 * PNG does not fit is APT_ERR_CAPACITY at wait, *nout the required count).  NULL switches PNG mode off.  Leaving image and
 * process mode also leaves PNG mode. */
int apt_decoder_set_png_mode(apt_decoder *dec, const apt_png_settings *ps);
/* The reference CLI's main job (main.rs): load a WAV (as apt_wav_load / apt_wav_load_pcm16), decode, process and write the
 * PNG to output_path.  info may be NULL. */
int apt_decode_wav_png(const char *input_path, const char *output_path, const apt_settings *s, int sync,
                       const apt_process_settings *ps, const apt_png_settings *png, apt_image_info *info);

/* apt_decode_batch, ending each recording in the image apt_process describes (png == NULL) or its PNG file.
 * outs[i] / caps[i] / nouts[i] count bytes; infos (may be NULL) receives each recording's apt_image_info.
 * Sharding, feeders and the out-of-memory fallback are those of apt_decode_batch.  Per recording, the status, info and
 * bytes equal apt_decode_image (png == NULL) or apt_decode_png of that recording alone with the same arguments; a
 * recording that fails (decode, image stage, or a file larger than caps[i]: APT_ERR_CAPACITY with the required count in
 * nouts[i]) leaves the others unaffected.  With PNG output each device's decoders hand their images to a fixed pool and
 * the images that are ready are encoded together, one launch sequence per group, on a stream of their own.  Argument
 * errors (NULL pointers, the settings checks of apt_process and apt_png_encode, rgb_from_rgba on grey output) come back
 * before any device is touched.  Returns the first failing status; statuses are never left "ok" by default. */
int apt_decode_batch_image(const void *const *signals, int format, const uint64_t *lens, int count,
                           uint32_t input_rate, const apt_settings *s, int sync,
                           const apt_process_settings *ps, const apt_png_settings *png,
                           uint8_t *const *outs, const uint64_t *caps, uint64_t *nouts, apt_image_info *infos,
                           int *statuses, const int *devices, int ndevices, int streams_per_device);

/* The layout of one batched PNG encode (host arithmetic, no device; DESIGN.md §11, "Batched encode"): `count` images of
 * width x heights[k] pixels with `channels` channels share a filtered-stream buffer (also the per-position arrays), the
 * per-block arrays and one output buffer.  images (may be NULL, else `cap` entries) receives each image's regions. */
typedef struct apt_png_group_image {
    uint64_t stream_offset;   /* of the filtered stream and the per-position arrays */
    uint64_t stream_bytes;    /* filtered bytes (the region has 16 bytes of padding after them) */
    uint64_t out_offset;      /* of the file in the output buffer */
    uint64_t out_bytes;       /* bytes reserved for the file (apt_png_bound rounded up to words) */
    uint64_t bound;           /* apt_png_bound of the image */
    uint32_t first_row, first_span, first_block, blocks, first_chunk, pad;
} apt_png_group_image;
typedef struct apt_png_group_info {
    uint64_t stream_bytes, out_bytes;          /* sizes of the shared buffers */
    uint32_t rows, spans, blocks, chunks;      /* grid sizes: filter warps, match CTAs, block CTAs, CRC threads */
} apt_png_group_info;
int apt_png_group_plan(uint32_t width, int channels, const apt_png_settings *ps, const uint32_t *heights, uint32_t count,
                       apt_png_group_info *info, apt_png_group_image *images, size_t cap);

/* ------------------------------------------------------------------ streaming decoder: image and PNG output */

/* Image output of a stream (DESIGN.md §9): the rows of the pass are kept on the device (f32, up to max_rows rows) and
 * apt_stream_finish_image ends the pass in the image apt_process describes.  Allowed only when nothing has been pushed
 * since create / reset.  ps == NULL switches image output (and PNG output) off and frees its buffers; setting a process
 * mode also switches PNG output off.  All device memory of the image output is allocated here; push and finish still
 * allocate nothing.  apt_stream_reset keeps both modes for the next pass; plain apt_stream_finish still works and makes
 * no image.  APT_ERR_BAD_ARG before the device is touched: a push since create / reset, max_rows == 0 (or 2^32 / 2080 or
 * more), and the settings apt_process rejects. */
int apt_stream_set_process_mode(apt_stream *st, const apt_process_settings *ps, uint64_t max_rows);
/* PNG output (needs process mode): apt_stream_finish_image writes the PNG file instead of the pixels.  The encoder
 * workspace for a max_rows image is reserved here.  NULL switches PNG output off.  APT_ERR_BAD_ARG before the device is
 * touched: a push since create / reset, no process mode, the settings apt_png_encode rejects for the process mode's
 * channels (rgb_from_rgba on grey output, a bad block_bytes, ...), and an IDAT for max_rows rows that could pass
 * 2^31 - 1 bytes. */
int apt_stream_set_png_mode(apt_stream *st, const apt_png_settings *png);
/* apt_stream_finish, plus the image: `image` receives rows*2080*bpp pixel bytes, or the PNG file in PNG mode; *image_n
 * its byte count; info as apt_decode_image.  The pixels, info and status equal apt_decode_image (the PNG bytes
 * apt_decode_png) on the whole recording with the same settings, sync and modes, for any split into pushes; for an I/Q
 * stream they equal apt_process (apt_png_encode) of apt_decode_iq's rows.  The rows are those apt_stream_finish returns.
 * Status, the first that applies:
 *   1. the decode's own (APT_ERR_TOO_SHORT, APT_ERR_FEW_SYNC_FRAMES): no image;
 *   2. the pass has more than max_rows rows: APT_ERR_CAPACITY, info->rows the pass's row count (the pushes still returned
 *      every row; only the image is refused);
 *   3. the image stage's errors, as apt_decode_image returns them (e.g. telemetry on a pass too short for a frame);
 *   4. image_cap below the image's size: APT_ERR_CAPACITY, *image_n the required byte count.
 * In cases 2 to 4 the pass is finished.  A stream without image output is APT_ERR_BAD_ARG. */
int apt_stream_finish_image(apt_stream *st, float *rows, uint64_t cap, uint64_t *nout, uint8_t *image, uint64_t image_cap,
                            uint64_t *image_n, apt_image_info *info);

/* ------------------------------------------------------------------ long recordings: finding the passes */

/* A recording kept in device memory (DESIGN.md §12), for finding the satellite passes in it and decoding each one without
 * sending the samples over PCIe again.  The rule is the project's own definition:
 *   e      the first stage of apt_decode at the work rate (resample + envelope, what apt_decoder_read_stage 0 returns);
 *          the work rate must be a multiple of 4160 (else APT_ERR_WORK_RATE).  R = work_rate / 2 samples per image row.
 *   q[w]   for w < W = max(0, floor(N_w / R) - 1): the Pearson correlation of e[wR, wR + R) with e[(w+1)R, (w+1)R + R);
 *          0 when the denominator is 0 or not finite.  Near 1 during a pass, near 0 in noise.
 *   passes the windows with q >= exit, joined into one group when fewer than max_gap windows lie between two of them; a
 *          group is kept when some window in it has q >= enter and it spans at least min_length windows (first to last).
 *          Group [a, b] is input samples [floor(a input_rate / 2), min(n, ceil((b + 2) input_rate / 2))).
 * Zero fields of apt_pass_search take the defaults: enter 0.30, exit 0.15, max_gap_s 30, min_length_s 60; seconds become
 * windows as floor(2 s).  APT_ERR_BAD_ARG unless 0 < exit <= enter <= 1 and both times are finite and >= 0. */
typedef struct apt_pass_search {
    float enter, exit, max_gap_s, min_length_s;
} apt_pass_search;
typedef struct apt_pass {
    uint64_t start, end;          /* input samples [start, end) */
    uint64_t first_window, windows;
    float mean_quality, peak_quality;   /* over the pass's windows */
} apt_pass;
typedef struct apt_recording apt_recording;
typedef struct apt_recording_info {
    uint64_t samples;             /* n */
    uint64_t work_samples;        /* N_w */
    uint64_t windows;             /* W */
    uint64_t device_bytes;        /* device memory the recording holds from create to destroy */
    uint32_t input_rate, row_samples;   /* R */
} apt_recording_info;

/* Uploads n samples of `signal` (host memory, APT_F32 or APT_PCM16, kept in that format) to device `device` once, through
 * the pinned staging ring when the buffer is pageable, and reserves everything apt_recording_quality needs.  A device
 * allocation failure is APT_ERR_NOMEM with nothing left allocated.  Argument errors (NULL pointers, n == 0, an unknown
 * format, the settings checks of apt_decode, a work rate that is not a multiple of 4160) come back before any device is
 * touched. */
int apt_recording_create(int device, const void *signal, int format, uint64_t n, uint32_t input_rate, const apt_settings *s,
                         apt_recording **rec);
void apt_recording_destroy(apt_recording *rec);
int apt_recording_get_info(apt_recording *rec, apt_recording_info *info);
/* q of the recording: the first stage runs over the resident samples in bounded chunks and k_pass_quality turns each
 * chunk's envelope into q; only the W floats of q are copied back.  *nq receives W; q == NULL with cap == 0 counts only;
 * cap < W is APT_ERR_CAPACITY.  The same bits on every run and for every chunk size. */
int apt_recording_quality(apt_recording *rec, float *q, uint64_t cap, uint64_t *nq);
/* The pass rule on q (host only, no device): out receives the passes in time order, *count their number; more than cap is
 * APT_ERR_CAPACITY (out may be NULL when cap is 0).  n and input_rate are the recording's. */
int apt_find_passes_quality(const float *q, uint64_t nq, uint64_t n, uint32_t input_rate, const apt_pass_search *ps,
                            apt_pass *out, uint32_t cap, uint32_t *count);
/* Decodes ranges[i].start .. ranges[i].end of the resident samples exactly as apt_decode / apt_decode_pcm16 (ps == NULL:
 * f32 rows, caps in floats), apt_decode_image (ps, png == NULL) or apt_decode_png (ps and png) decode the host slice
 * signal[start:end) with the same arguments: outs[i], nouts[i], statuses[i] and infos[i] (infos may be NULL) bit for bit.
 * Each range is copied to a 16-byte aligned device buffer and decoded by a parked decoder; a failing range (too short, too
 * few sync frames, capacity) leaves the others unaffected.  Only start, end of each range are read.  Argument errors (NULL
 * pointers, a range empty or past n, the settings checks of apt_process and apt_png_encode, png without ps) come back
 * before any device is touched with every status set.  Returns APT_OK or the first failing status. */
int apt_recording_decode(apt_recording *rec, const apt_pass *ranges, uint32_t count, int sync,
                         const apt_process_settings *ps, const apt_png_settings *png, void *const *outs,
                         const uint64_t *caps, uint64_t *nouts, apt_image_info *infos, int *statuses);

/* ------------------------------------------------------------------ continuous feeds: watching for passes */

/* The pass rule of apt_find_passes_quality fed q window by window (host only, no device; DESIGN.md §13).
 *   APT_PASS_AOS  fires at the first window that joins the open group once the group has reached enter and spans
 *                 min_length windows: from here on the group is certain to be kept.  pass holds the group so far, end 0.
 *   APT_PASS_LOS  fires at the evaluation of window last + max_gap (no later window can join the group), or at finish
 *                 (window = the number of windows fed).  pass is exactly the entry apt_find_passes_quality returns for the
 *                 same q, mean_quality included; an LOS before finish has end = ceil((last + 2) input_rate / 2), which is
 *                 within the recording whenever window last + max_gap exists.
 * A group that is dropped (never reaches enter, or spans fewer than min_length windows) emits nothing.  apt_watch also
 * emits APT_PASS_SEGMENT (apt_watch_settings).  Feeding all of q and then finishing gives the passes of
 * apt_find_passes_quality, however q is split. */
enum { APT_PASS_AOS = 1, APT_PASS_LOS = 2, APT_PASS_SEGMENT = 3 };
typedef struct apt_pass_event {
    int kind;                 /* APT_PASS_AOS, APT_PASS_LOS or APT_PASS_SEGMENT */
    uint64_t window;          /* the window whose evaluation fired the event */
    apt_pass pass;            /* SEGMENT: start = the new segment's first absolute sample, the rest 0 */
} apt_pass_event;
typedef struct apt_pass_tracker apt_pass_tracker;
/* APT_ERR_BAD_ARG for NULL pointers, input_rate 0 and the search settings apt_find_passes_quality refuses. */
int apt_pass_tracker_create(uint32_t input_rate, const apt_pass_search *search, apt_pass_tracker **t);
/* The next nq windows.  events receives the events in order and *nev their number; cap < 2 * nq is APT_ERR_CAPACITY with
 * the tracker unchanged. */
int apt_pass_tracker_feed(apt_pass_tracker *t, const float *q, uint64_t nq, apt_pass_event *events, uint64_t cap,
                          uint64_t *nev);
/* The end of a recording of n input samples: the LOS of the open group, if it is kept (cap >= 1, else APT_ERR_CAPACITY
 * with the tracker unchanged).  The tracker then starts over at window 0. */
int apt_pass_tracker_finish(apt_pass_tracker *t, uint64_t n, apt_pass_event *events, uint64_t cap, uint64_t *nev);
void apt_pass_tracker_destroy(apt_pass_tracker *t);

/* A watcher (DESIGN.md §13): a continuous audio feed (rtl_fm, a sound card) pushed as it arrives, in fixed device memory.
 * Each step (at most max_push samples) uploads the slice once, runs the first stage over the units that became complete
 * and k_pass_quality over the windows whose two rows are final, feeds the new q to the pass rule, and feeds the open group
 * from the watcher's own input window (device to device) to a streaming decoder with image / PNG output.  The callback
 * receives the AOS of a pass and, at its LOS, the pass's decode.  For any split of the feed into pushes (F32 and PCM16 mixed),
 * per segment: the q returned by pushes and finish, concatenated, equal apt_recording_quality of the segment's samples bit
 * for bit; the LOS passes equal apt_find_passes_quality on them; each LOS's status, rows, info and data equal
 * apt_recording_decode of the pass's range with the same sync, ps and png.  Statuses beyond the decode's own: a pass with
 * more than max_rows rows is APT_ERR_CAPACITY with rows set (the watcher continues), a kept pass too short to decode is
 * APT_ERR_TOO_SHORT.
 * Segments: the first stage keeps work-rate indices below 2^32.  When no group is open and the segment holds at least T
 * work samples (2^31; APTB200_WATCH_SEGMENT=n sets T), the next step first finishes the segment as apt_watch_finish does,
 * emits APT_PASS_SEGMENT with the new segment's first absolute sample, and starts a new segment there (window indices
 * restart at 0).  A group still open at 2T is closed as at finish.  Samples in events are absolute (since create / reset). */
typedef struct apt_watch apt_watch;
typedef struct apt_watch_settings {
    int sync;
    apt_pass_search search;            /* zero fields: the defaults of apt_find_passes_quality */
    const apt_process_settings *ps;    /* NULL: each pass ends in its f32 rows */
    const apt_png_settings *png;       /* with ps: each pass ends in its PNG file; NULL: in its pixels */
    uint64_t max_rows;                 /* the longest pass that gets its image / rows; 0: 2400 */
    uint64_t max_push;                 /* samples per internal step, as apt_stream; 0: input_rate */
} apt_watch_settings;
typedef struct apt_watch_event {
    apt_pass_event ev;                 /* samples absolute since create / reset; windows those of the segment */
    uint32_t index;                    /* pass number since create / reset */
    int status;                        /* LOS: the pass decode's status */
    uint64_t rows;                     /* LOS: the pass's row count */
    apt_image_info info;               /* LOS with ps */
    const void *data;                  /* LOS: f32 rows, pixels or PNG file; valid during the callback only */
    uint64_t bytes;                    /* of data */
} apt_watch_event;
typedef struct apt_watch_info {
    uint64_t samples_in;               /* since create / reset */
    uint64_t segment_start;            /* absolute first sample of the current segment */
    uint64_t windows;                  /* windows of the segment evaluated so far */
    uint64_t passes;                   /* LOS events since create / reset */
    uint64_t open;                     /* 1 while a group is open */
    uint64_t device_bytes;             /* device memory held from create to destroy */
    uint64_t max_push;
    uint64_t latency_windows;          /* windows a push can leave unevaluated behind its last sample */
} apt_watch_info;
typedef void (*apt_watch_cb)(const apt_watch_event *ev, void *user);
/* Everything (quality path, pass stream, image / PNG output) is allocated here; push, finish and reset allocate nothing.
 * Argument errors come back before any device is touched: NULL pointers, the search settings, the settings apt_process and
 * apt_png_encode refuse, png without ps, max_rows or max_push out of range, and the settings apt_stream_create refuses. */
int apt_watch_create(int device, uint32_t input_rate, const apt_settings *s, const apt_watch_settings *ws, apt_watch_cb cb,
                     void *user, apt_watch **w);
/* The device_bytes (and max_push, latency_windows) apt_watch_create would report, on the host. */
int apt_watch_geometry(uint32_t input_rate, const apt_settings *s, const apt_watch_settings *ws, apt_watch_info *info);
/* The q floats a push of n samples can return at most. */
int apt_watch_push_bound(apt_watch *w, uint64_t n, uint64_t *cap_q);
/* n samples of the feed (APT_F32 or APT_PCM16); q receives the new windows' quality, *nq their number (cap below
 * apt_watch_push_bound: APT_ERR_CAPACITY before any work).  Events are delivered through the callback during the call.
 * A pass's decode status does not fail the push. */
int apt_watch_push(apt_watch *w, const void *samples, int format, uint64_t n, float *q, uint64_t cap, uint64_t *nq);
/* The end of the feed: the tail windows (cap: apt_watch_push_bound(w, 0)) and the LOS of a group still open (end = n).
 * Pushing again needs apt_watch_reset. */
int apt_watch_finish(apt_watch *w, float *q, uint64_t cap, uint64_t *nq);
/* A new feed with the same settings and buffers. */
int apt_watch_reset(apt_watch *w);
int apt_watch_get_info(apt_watch *w, apt_watch_info *info);
void apt_watch_destroy(apt_watch *w);
/* Every call into a watcher from its own callback is APT_ERR_BAD_ARG. */

/* An I/Q watcher (DESIGN.md §14): one SDR's continuous I/Q feed (rtl_sdr) watched on up to 8 channels at once, each
 * channel an apt_watch on its own FM audio.  iq->offset_hz is ignored: channel c is the FM audio a_c of apt_fm_demod at
 * offset_hz = offsets[c], at iq->audio_rate.  Each step (at most ws->max_push I/Q samples; 0: iq_rate) uploads the slice
 * once, converts it into one cf32 window shared by the channels, demodulates every channel in one kernel launch straight
 * into that channel's input window, and then runs each channel's apt_watch step on its new audio.  For any split of the
 * feed into pushes (APT_CU8, APT_CS16 and APT_CF32 mixed), channel c keeps apt_watch's contract on a_c: per segment its q,
 * its LOS passes and each LOS's status, rows, info and data equal apt_recording_quality, apt_find_passes_quality and
 * apt_recording_decode of a_c.  Each channel has its own pass state, pass stream, segments and image / PNG output, so
 * overlapping passes on different channels both finish.  The other fields of ws apply to every channel.
 * Samples in events are audio samples of the channel (absolute since create / reset, as apt_watch reports them on a_c):
 * multiply by D = iq_rate / audio_rate for I/Q samples.  Events come through the callback during push / finish: within one
 * internal step channel 0's first, then channel 1's, and so on, each channel's in apt_watch's order; a segment roll is an
 * internal step of its own, taken before the step that needs it.  Every call into an I/Q watcher from its own callback is
 * APT_ERR_BAD_ARG.  Everything is allocated at create; push, finish and reset allocate nothing.  Argument errors come back
 * before any device is touched: NULL pointers, count outside 1..8, the checks of apt_fm_demod_len at each offset, and what
 * apt_watch_geometry refuses at audio_rate. */
#define APT_WATCH_IQ_MAX_CHANNELS 8
typedef struct apt_watch_iq apt_watch_iq;
typedef void (*apt_watch_iq_cb)(int channel, const apt_watch_event *ev, void *user);
/* device_bytes: the shared cf32 window 2 (N + 2D) + max_push + 64 complex samples (N the channel filter's taps), one step's
 * raw samples (8 max_push bytes), the polyphase taps once and a phasor table per channel, and per channel the device_bytes
 * of apt_watch_geometry(audio_rate, ws with max_push = max_push / D + 1).  max_push in I/Q samples, latency_windows the
 * channel watcher's.  Host only. */
int apt_watch_iq_geometry(const apt_iq_settings *iq, const int32_t *offsets, int count, const apt_settings *s,
                          const apt_watch_settings *ws, apt_watch_info *info);
int apt_watch_iq_create(int device, const apt_iq_settings *iq, const int32_t *offsets, int count, const apt_settings *s,
                        const apt_watch_settings *ws, apt_watch_iq_cb cb, void *user, apt_watch_iq **w);
/* The q floats a push of n I/Q samples can return at most for any one channel. */
int apt_watch_iq_push_bound(apt_watch_iq *w, uint64_t n, uint64_t *cap_q);
/* n I/Q samples (APT_CU8, APT_CS16 or APT_CF32; audio formats are APT_ERR_BAD_ARG).  Channel c's new q go to q + c * cap,
 * and nq[c] (count entries) receives their number; cap below apt_watch_iq_push_bound is APT_ERR_CAPACITY before any work. */
int apt_watch_iq_push(apt_watch_iq *w, const void *iq, int format, uint64_t n, float *q, uint64_t cap, uint64_t *nq);
/* The end of the feed on every channel, as apt_watch_finish (cap: apt_watch_iq_push_bound(w, 0)). */
int apt_watch_iq_finish(apt_watch_iq *w, float *q, uint64_t cap, uint64_t *nq);
int apt_watch_iq_reset(apt_watch_iq *w);
/* Channel `channel`'s segment_start, windows, passes, open and latency_windows; samples_in and max_push in I/Q samples;
 * device_bytes the whole watcher's (apt_watch_iq_geometry). */
int apt_watch_iq_get_info(apt_watch_iq *w, int channel, apt_watch_info *info);
void apt_watch_iq_destroy(apt_watch_iq *w);

#ifdef __cplusplus
}
#endif
#endif /* APTB200_H */
