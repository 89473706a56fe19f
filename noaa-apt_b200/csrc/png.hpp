// The PNG encoder (DESIGN.md §11): filter, match candidates, greedy parse, package-merge Huffman codes, bit emission,
// Adler-32, CRC-32 and the PNG framing, all on the device.  This module alone reads apt_png_settings: it validates them,
// sizes the workspaces, launches the kernel sequence and leaves the file's bytes and length on the device.  It also owns
// image output (OutPlan, ImageOut): the output rules and sizes, the pixels, the encode, the length read-back and the copy-out.
#pragma once

#include <cstdint>
#include <vector>

#include "aptb200.h"
#include "launch.hpp"
#include "post.hpp"

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

// One image of an encode group (DESIGN.md §11, "Batched encode").  The images of a group share width, channels and
// settings; each has its own height and pixels.  Every offset is the image's own region of a buffer shared by the
// group, and every kernel finds its image by a binary search of the first-index fields over the table.
struct PngImage {
    const unsigned char *px = nullptr;   // device pixels: height * width * in_ch bytes
    u64 pos = 0;        // offset of the filtered stream in f and of the positions in lcode / dist / flag (a multiple of 64)
    u64 out = 0;        // byte offset of the file in out (a multiple of 8)
    u64 out_bytes = 0;  // bytes of out reserved for the file: the bound rounded up to words
    u32 height = 0;
    u32 n = 0;          // filtered stream length
    u32 row0 = 0;       // first global row (k_png_filter: one warp per row)
    u32 span0 = 0;      // first global match span (k_png_match)
    u32 blk0 = 0;       // first global deflate block (parse, huffman, emit; hist / codes / hdr / bits / off / sums)
    u32 nblocks = 0;
    u32 chunk0 = 0;     // first global CRC chunk, a multiple of 32 so that no warp of k_png_crc spans two images
    unsigned char ihdr[25] = {};   // the IHDR chunk, CRC included
};

// The layout of a group: its table and the sizes of the shared buffers.
struct PngLayout {
    PngPlan shape;                  // settings, width and channels (the first image's plan)
    std::vector<PngImage> img;
    u64 f_bytes = 0;                // f, lcode, flag (and dist in u16): the last image's region end
    u64 out_bytes = 0;
    u32 rows = 0, spans = 0, blocks = 0, chunks = 0;
};

// The layout of `g` images whose plans share width, channels and settings (APT_ERR_BAD_ARG otherwise).  Host only.
int png_layout(const PngPlan *plans, const unsigned char *const *pixels, u32 g, PngLayout &lay);

// Device workspaces of the encoder; they grow to the largest group seen and are kept.
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
    unsigned char *out = nullptr;    // the PNG files (PngImage::out, out_bytes)
    PngCtl *ctl = nullptr;           // per image
    PngImage *img = nullptr;         // the group's table (device)
    PngImage *h_img = nullptr;       // and its pinned staging
    u64 cap_n = 0, cap_n_pos = 0, cap_blocks = 0, cap_out = 0, cap_img = 0;   // bytes of f; positions of lcode / dist / flag; ...
    PngLayout lay;                   // the layout of the last encode
    PngWork() = default;
    PngWork(const PngWork &) = delete;
    ~PngWork() { release(); }
    int reserve(const PngLayout &lay);
    void release();
    size_t device_bytes() const;
    static size_t bytes_for(const PngLayout &lay);   // device_bytes() after reserve(lay) on an empty workspace (host only)
};

// Enqueues the whole encode of `g` images (plans[k] and device pixels[k], height * width * in_ch bytes, as png_layout
// takes them) on c.stream: one launch per kernel for the group.  Image k's file is at w.out + w.lay.img[k].out, its length
// in w.ctl[k].total.  Every file's bytes are those of the image encoded alone.  The caller waits for the encode before
// it starts the next one on the same workspace.
int png_encode_device(const LaunchCtx &c, const PngPlan *plans, const unsigned char *const *pixels, u32 g, PngWork &w,
                      KernelHook *hook);

// What becomes of a decoded signal (DESIGN.md §9, "Image output"): f32 rows, the image of `post`, or that image as a PNG
// file.  Host only.
struct OutPlan {
    bool image = false;           // the image of `post`; false: f32 rows
    PostPlan post;
    bool png = false;             // the image as a PNG file of png_s
    apt_png_settings png_s{};
    // PNG output of the image (the settings rules for a one-row image of post.bpp channels); png == nullptr: none.
    int set_png(const apt_png_settings *png);
    // The encoder's plan for an image of `rows` rows.
    int png_plan(uint64_t rows, PngPlan &pp) const;
    // Bytes of `px` pixels: px f32 values, or px * bpp bytes of the image.
    uint64_t px_bytes(uint64_t px) const { return px * (image ? post.bpp : sizeof(float)); }
    // Bytes of the output of `px` pixels: px_bytes, or the PNG bound of max(px / 2080, 1) rows.
    int bytes(uint64_t px, uint64_t &bytes) const;
};

// The output rules, host only: the process settings (ps == nullptr: f32 rows), then PNG settings (png == nullptr: none),
// which need process settings.
int make_out_plan(const apt_process_settings *ps, const apt_png_settings *png, OutPlan &plan);

// Where an image lives after the image stage and how it reaches the caller: the stage's buffers, the pixels, the encoder's
// workspace and the pinned copies of its control blocks.  Decoders, streams, the batch's PNG feeder and apt_png_encode_batch
// each own one; it runs on the caller's CUDA stream.
struct ImageOut {
    OutPlan plan;
    PostBuffers post;
    unsigned char *px = nullptr;  // the image (or apt_png_encode_batch's input pixels), px_cap bytes
    u64 px_cap = 0;
    PngWork work;
    PngCtl *h_ctl = nullptr;      // pinned: the control blocks of the last encode, ctl_cap of them
    uint32_t ctl_cap = 0;
    apt_image_info info{};        // the decoder's last image
    bool keep = false;            // the decoder's image stays in px: nothing is copied to the caller (the batch's PNG feeder)

    ~ImageOut() { release(); }
    int reserve_px(uint64_t bytes);      // px of at least `bytes` (grown, never shrunk)
    int reserve_ctl(uint32_t g);         // h_ctl for g encodes
    // The image stage on rows (device) into out, or px when out is nullptr (post_launch with rows of 2080 pixels).
    int launch(const LaunchCtx &c, const float *rows, const SyncResult *res, u32 fixed_rows, u32 max_rows, void *out,
               KernelHook *hook);
    // Encodes g images (as png_encode_device takes them) and reads their control blocks back, both on c.stream; length(k)
    // is valid once the caller has synchronised with that stream.
    int encode(const LaunchCtx &c, const PngPlan *plans, const unsigned char *const *pixels, u32 g, KernelHook *hook);
    // encode() of the image of `rows` rows in px.
    int encode_px(const LaunchCtx &c, uint64_t rows, KernelHook *hook);
    uint64_t length(u32 k) const { return h_ctl[k].total; }
    // Enqueues the copy of file k to dst, or returns APT_ERR_CAPACITY with its length when dst is null or cap too small.
    int copy_out(u32 k, void *dst, uint64_t cap, cudaMemcpyKind kind, cudaStream_t s) const;
    // Device bytes of post, px and work for images of up to max_rows rows of `plan` (host only).
    static uint64_t device_bytes(const OutPlan &plan, uint64_t max_rows);
    void release();
};

// APT_ERR_CAPACITY with the message every output path gives when dst is null or cap is below need.
int check_room(const void *dst, uint64_t need, uint64_t cap);

// Frees the per-device workspaces apt_png_encode keeps between calls (apt_cache_clear).
void png_stage_cache_clear();

// 1 if every alpha byte of an RGBA host image is 255 (the rgb_from_rgba rule for host pixels).
bool png_alpha_opaque(const uint8_t *pixels, uint64_t npx);

}  // namespace aptb200
