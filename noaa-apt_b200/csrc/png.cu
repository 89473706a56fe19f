// The PNG encoder (see png.hpp): settings, plan, tables, workspaces, the launch sequence and apt_png_* host entry points.
#include "png.hpp"

#include <algorithm>
#include <cstring>
#include <mutex>

#include "common.hpp"
#include "decoder.hpp"
#include "kernels_png.cuh"

namespace aptb200 {

namespace {

constexpr u64 kIdatMax = 0x7FFFFFFFull;   // PNG chunk length limit

u32 crc_table_entry(u32 k) {
    u32 c = k;
    for (int j = 0; j < 8; ++j) c = c & 1 ? (c >> 1) ^ 0xEDB88320u : c >> 1;
    return c;
}

u32 host_crc32(const unsigned char *p, size_t n) {
    u32 c = 0xFFFFFFFFu;
    for (size_t k = 0; k < n; ++k) c = crc_table_entry((c ^ p[k]) & 0xFF) ^ (c >> 8);
    return c ^ 0xFFFFFFFFu;
}

u32 host_multmodp(u32 a, u32 b) {
    u32 m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}

// The constant tables, uploaded once per device (constant memory is per device).
int ensure_tables() {
    static std::mutex mu;
    static bool ready[64] = {};
    int dev = 0;
    APT_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lk(mu);
    if (dev >= 0 && dev < 64 && ready[dev]) return APT_OK;
    static const uint16_t len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
                                          131, 163, 195, 227, 258};
    static const unsigned char len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
    static const uint16_t dist_base[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537,
                                           2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
    static const unsigned char dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
    static const unsigned char cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    unsigned char len_sym[kPngMaxMatch + 1] = {0};
    for (u32 c = 0; c < 29; ++c) {
        const u32 hi = c == 27 ? 258 : (c == 28 ? 259 : len_base[c + 1]);
        for (u32 L = len_base[c]; L < hi; ++L) len_sym[L] = static_cast<unsigned char>(c);
    }
    u32 crc[256], x2n[32];
    for (u32 k = 0; k < 256; ++k) crc[k] = crc_table_entry(k);
    u32 p = 1u << 30;   // x^1
    x2n[0] = p;
    for (int k = 1; k < 32; ++k) x2n[k] = p = host_multmodp(p, p);
    APT_CUDA(cudaMemcpyToSymbol(c_png_len_sym, len_sym, sizeof(len_sym)));
    APT_CUDA(cudaMemcpyToSymbol(c_png_len_base, len_base, sizeof(len_base)));
    APT_CUDA(cudaMemcpyToSymbol(c_png_len_extra, len_extra, sizeof(len_extra)));
    APT_CUDA(cudaMemcpyToSymbol(c_png_dist_base, dist_base, sizeof(dist_base)));
    APT_CUDA(cudaMemcpyToSymbol(c_png_dist_extra, dist_extra, sizeof(dist_extra)));
    APT_CUDA(cudaMemcpyToSymbol(c_png_cl_order, cl_order, sizeof(cl_order)));
    APT_CUDA(cudaMemcpyToSymbol(c_png_crc_table, crc, sizeof(crc)));
    APT_CUDA(cudaMemcpyToSymbol(c_png_x2n, x2n, sizeof(x2n)));
    if (dev >= 0 && dev < 64) ready[dev] = true;
    return APT_OK;
}

void put_be32(unsigned char *p, u32 v) {
    p[0] = static_cast<unsigned char>(v >> 24);
    p[1] = static_cast<unsigned char>(v >> 16);
    p[2] = static_cast<unsigned char>(v >> 8);
    p[3] = static_cast<unsigned char>(v);
}

template <typename T>
int grow(T *&p, u64 &cap, u64 need, size_t elem) {
    if (cap >= need) return APT_OK;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    APT_CUDA(cudaMalloc(reinterpret_cast<void **>(&p), std::max<u64>(need, 1) * elem));
    cap = need;
    return APT_OK;
}

}  // namespace

int make_png(uint32_t width, uint32_t height, int channels, const apt_png_settings *ps, PngPlan &p) {
    if (!ps) return fail(APT_ERR_BAD_ARG, "null PNG settings");
    if (ps->filter < -1 || ps->filter > 4) return fail(APT_ERR_BAD_ARG, "PNG filter must be -1 (adaptive) or 0..4, got %d", ps->filter);
    const uint32_t bb = ps->block_bytes;
    if (bb < 4096 || bb > 65536 || (bb & (bb - 1)))
        return fail(APT_ERR_BAD_ARG, "block_bytes must be a power of two in [4096, 65536], got %u", bb);
    if (channels != 1 && channels != 3 && channels != 4) return fail(APT_ERR_BAD_ARG, "channels must be 1, 3 or 4, got %d", channels);
    if (ps->rgb_from_rgba && channels != 4) return fail(APT_ERR_BAD_ARG, "rgb_from_rgba needs RGBA pixels");
    if (width == 0 || height == 0) return fail(APT_ERR_BAD_ARG, "empty image (%u x %u)", width, height);
    p.s = *ps;
    p.width = width;
    p.height = height;
    p.in_ch = channels;
    p.ch = ps->rgb_from_rgba ? 3 : channels;
    p.row = 1 + static_cast<u64>(width) * p.ch;
    p.n = p.row * height;
    const u64 nb = (p.n + bb - 1) / bb;
    const u64 deflate_max = (9 * p.n + nb * (9 + 2400) + 7) / 8;
    if (2 + deflate_max + 4 > kIdatMax) return fail(APT_ERR_BAD_ARG, "image too large for one IDAT chunk");
    p.nblocks = static_cast<u32>(nb);
    p.bound = 57 + 6 + deflate_max;
    unsigned char *h = p.ihdr;
    put_be32(h, 13);
    memcpy(h + 4, "IHDR", 4);
    put_be32(h + 8, width);
    put_be32(h + 12, height);
    h[16] = 8;
    h[17] = p.ch == 1 ? 0 : (p.ch == 3 ? 2 : 6);
    h[18] = h[19] = h[20] = 0;
    put_be32(h + 21, host_crc32(h + 4, 17));
    return APT_OK;
}

bool png_alpha_opaque(const uint8_t *px, uint64_t npx) {
    for (uint64_t k = 0; k < npx; ++k)
        if (px[4 * k + 3] != 255) return false;
    return true;
}

int png_layout(const PngPlan *plans, const unsigned char *const *pixels, u32 g, PngLayout &lay) {
    if (g == 0) return fail(APT_ERR_BAD_ARG, "empty PNG group");
    const PngPlan &s = plans[0];
    lay.shape = s;
    lay.img.assign(g, PngImage{});
    u64 pos = 0, out = 0;
    u64 rows = 0, spans = 0, blocks = 0, chunks = 0;
    for (u32 k = 0; k < g; ++k) {
        const PngPlan &p = plans[k];
        if (p.width != s.width || p.in_ch != s.in_ch || p.ch != s.ch || p.s.filter != s.s.filter || p.s.matches != s.s.matches ||
            p.s.block_bytes != s.s.block_bytes || p.s.rgb_from_rgba != s.s.rgb_from_rgba)
            return fail(APT_ERR_BAD_ARG, "the images of a PNG group must share width, channels and settings");
        PngImage &im = lay.img[k];
        im.px = pixels ? pixels[k] : nullptr;
        im.pos = pos;
        im.out = out;
        im.out_bytes = (p.bound + 8) & ~3ull;
        im.height = p.height;
        im.n = static_cast<u32>(p.n);
        im.row0 = static_cast<u32>(rows);
        im.span0 = static_cast<u32>(spans);
        im.blk0 = static_cast<u32>(blocks);
        im.nblocks = p.nblocks;
        im.chunk0 = static_cast<u32>(chunks);
        memcpy(im.ihdr, p.ihdr, sizeof(im.ihdr));
        pos += (p.n + 16 + 63) & ~63ull;   // the stream, 16 bytes of padding png_ld32 may read, 64-byte alignment
        out += (im.out_bytes + 7) & ~7ull;
        rows += p.height;
        spans += (p.n + kPngSpan - 1) / kPngSpan;
        blocks += p.nblocks;
        chunks += ((p.bound - 37 + kPngCrcChunk - 1) / kPngCrcChunk + 31) & ~31ull;
        if (rows > 0xFFFFFFFFull || blocks > 0xFFFFFFFFull || chunks > 0xFFFFFFFFull)
            return fail(APT_ERR_BAD_ARG, "PNG group too large");
    }
    lay.f_bytes = pos;
    lay.out_bytes = out;
    lay.rows = static_cast<u32>(rows);
    lay.spans = static_cast<u32>(spans);
    lay.blocks = static_cast<u32>(blocks);
    lay.chunks = static_cast<u32>(chunks);
    return APT_OK;
}

int PngWork::reserve(const PngLayout &l) {
    APT_TRY(grow(f, cap_n, l.f_bytes, 1));
    if (cap_n_pos < l.f_bytes) {
        for (void *q : {(void *)lcode, (void *)dist, (void *)flag})
            if (q) cudaFree(q);
        lcode = nullptr;
        dist = nullptr;
        flag = nullptr;
        cap_n_pos = 0;
        APT_CUDA(cudaMalloc(&lcode, l.f_bytes));
        APT_CUDA(cudaMalloc(&dist, l.f_bytes * sizeof(uint16_t)));
        APT_CUDA(cudaMalloc(&flag, l.f_bytes));
        cap_n_pos = l.f_bytes;
    }
    if (cap_blocks < l.blocks) {
        for (void *q : {(void *)hist, (void *)codes, (void *)hdr, (void *)hdr_bits, (void *)bits, (void *)off, (void *)sums})
            if (q) cudaFree(q);
        hist = codes = hdr = hdr_bits = nullptr;
        bits = off = sums = nullptr;
        cap_blocks = 0;
        const u64 nb = l.blocks;
        APT_CUDA(cudaMalloc(&hist, nb * (kPngLit + kPngDist) * sizeof(u32)));
        APT_CUDA(cudaMalloc(&codes, nb * (kPngLit + kPngDist) * sizeof(u32)));
        APT_CUDA(cudaMalloc(&hdr, nb * kPngHdrWords * sizeof(u32)));
        APT_CUDA(cudaMalloc(&hdr_bits, nb * sizeof(u32)));
        APT_CUDA(cudaMalloc(&bits, nb * sizeof(u64)));
        APT_CUDA(cudaMalloc(&off, nb * sizeof(u64)));
        APT_CUDA(cudaMalloc(&sums, 2 * nb * sizeof(u64)));
        cap_blocks = nb;
    }
    APT_TRY(grow(out, cap_out, l.out_bytes, 1));
    const u64 g = l.img.size();
    if (cap_img < g) {
        if (ctl) cudaFree(ctl);
        if (img) cudaFree(img);
        if (h_img) cudaFreeHost(h_img);
        ctl = nullptr;
        img = nullptr;
        h_img = nullptr;
        cap_img = 0;
        APT_CUDA(cudaMalloc(&ctl, g * sizeof(PngCtl)));
        APT_CUDA(cudaMalloc(&img, g * sizeof(PngImage)));
        APT_CUDA(cudaHostAlloc(reinterpret_cast<void **>(&h_img), g * sizeof(PngImage), cudaHostAllocDefault));
        cap_img = g;
    }
    return APT_OK;
}

void PngWork::release() {
    for (void *q : {(void *)f, (void *)lcode, (void *)dist, (void *)flag, (void *)hist, (void *)codes, (void *)hdr, (void *)hdr_bits,
                    (void *)bits, (void *)off, (void *)sums, (void *)out, (void *)ctl, (void *)img})
        if (q) cudaFree(q);
    if (h_img) cudaFreeHost(h_img);
    f = lcode = flag = out = nullptr;
    dist = nullptr;
    hist = codes = hdr = hdr_bits = nullptr;
    bits = off = sums = nullptr;
    ctl = nullptr;
    img = h_img = nullptr;
    cap_n = cap_n_pos = cap_blocks = cap_out = cap_img = 0;
}

namespace {
size_t work_bytes(u64 n, u64 n_pos, u64 blocks, u64 out, u64 img) {
    return n + n_pos * 4 + blocks * (2 * (kPngLit + kPngDist) * 4 + kPngHdrWords * 4 + 4 + 4 * 8) + out +
           img * (sizeof(PngCtl) + sizeof(PngImage));
}
}  // namespace

size_t PngWork::device_bytes() const { return work_bytes(cap_n, cap_n_pos, cap_blocks, cap_out, cap_img); }

size_t PngWork::bytes_for(const PngLayout &l) { return work_bytes(l.f_bytes, l.f_bytes, l.blocks, l.out_bytes, l.img.size()); }

int png_encode_device(const LaunchCtx &c, const PngPlan *plans, const unsigned char *const *pixels, u32 g, PngWork &w,
                      KernelHook *hook) {
    APT_TRY(ensure_tables());
    PngLayout &lay = w.lay;
    APT_TRY(png_layout(plans, pixels, g, lay));
    APT_TRY(w.reserve(lay));
    const PngPlan &p = lay.shape;
    const u32 bb = p.s.block_bytes;
    memcpy(w.h_img, lay.img.data(), g * sizeof(PngImage));   // the previous encode on w has finished (png.hpp)
    APT_CUDA(cudaMemcpyAsync(w.img, w.h_img, g * sizeof(PngImage), cudaMemcpyHostToDevice, c.stream));
#ifdef APTB200_PNG_CHECK
    const u32 zero = 0;
    APT_CUDA(cudaMemcpyToSymbolAsync(g_png_violation, &zero, sizeof(zero), 0, cudaMemcpyHostToDevice, c.stream));
#endif
    APT_CUDA(cudaMemsetAsync(w.flag, 0, lay.f_bytes, c.stream));
    APT_CUDA(cudaMemsetAsync(w.out, 0, lay.out_bytes, c.stream));
    APT_CUDA(cudaMemsetAsync(w.ctl, 0, g * sizeof(PngCtl), c.stream));
    {
        KernelSlot ks(hook, "png_filter");
        const u32 grid = (lay.rows + 7) / 8;
        if (p.in_ch == 1) k_png_filter<1, 1><<<grid, 256, 0, c.stream>>>(w.img, g, lay.rows, p.width, p.s.filter, w.f);
        else if (p.in_ch == 3) k_png_filter<3, 3><<<grid, 256, 0, c.stream>>>(w.img, g, lay.rows, p.width, p.s.filter, w.f);
        else if (p.ch == 4) k_png_filter<4, 4><<<grid, 256, 0, c.stream>>>(w.img, g, lay.rows, p.width, p.s.filter, w.f);
        else k_png_filter<4, 3><<<grid, 256, 0, c.stream>>>(w.img, g, lay.rows, p.width, p.s.filter, w.f);
        APT_CUDA(cudaGetLastError());
    }
    if (p.s.matches) {
        KernelSlot ks(hook, "png_match");
        const size_t smem = 32768 * sizeof(uint16_t);
        APT_CUDA(cudaFuncSetAttribute(k_png_match, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        k_png_match<<<lay.spans, 32, smem, c.stream>>>(w.img, g, w.f, bb, w.lcode, w.dist);
        APT_CUDA(cudaGetLastError());
    } else {
        APT_CUDA(cudaMemsetAsync(w.lcode, 0, lay.f_bytes, c.stream));   // literals only
    }
    {
        KernelSlot ks(hook, "png_parse");
        APT_CUDA(cudaFuncSetAttribute(k_png_parse, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bb)));
        k_png_parse<<<lay.blocks, 256, bb, c.stream>>>(w.img, g, w.f, w.lcode, w.dist, bb, w.flag, w.hist);
        APT_CUDA(cudaGetLastError());
    }
    {
        KernelSlot ks(hook, "png_huffman");
        k_png_huffman<<<lay.blocks, 32, 0, c.stream>>>(w.img, g, w.hist, w.codes, w.hdr, w.hdr_bits, w.bits);
        APT_CUDA(cudaGetLastError());
    }
    {
        KernelSlot ks(hook, "png_scan");
        k_png_scan<<<g, 1024, 0, c.stream>>>(w.img, w.bits, w.off, w.ctl);
        APT_CUDA(cudaGetLastError());
    }
    {
        KernelSlot ks(hook, "png_emit");
        k_png_emit<<<lay.blocks, kPngEmitThreads, 0, c.stream>>>(w.img, g, w.f, w.lcode, w.dist, w.flag, bb, w.codes, w.hdr,
                                                                   w.hdr_bits, w.off, w.out, w.sums);
        APT_CUDA(cudaGetLastError());
    }
    {
        KernelSlot ks(hook, "png_frame");
        k_png_frame<<<(g + 63) / 64, 64, 0, c.stream>>>(w.img, g, w.sums, bb, w.out, w.ctl);
        APT_CUDA(cudaGetLastError());
    }
    {
        KernelSlot ks(hook, "png_crc");
        k_png_crc<<<(lay.chunks + 255) / 256, 256, 0, c.stream>>>(w.img, g, lay.chunks, w.out, w.ctl);
        APT_CUDA(cudaGetLastError());
    }
    {
        KernelSlot ks(hook, "png_end");
        k_png_end<<<(g + 63) / 64, 64, 0, c.stream>>>(w.img, g, w.out, w.ctl);
        APT_CUDA(cudaGetLastError());
    }
#ifdef APTB200_PNG_CHECK
    u32 bad = 0;
    APT_CUDA(cudaMemcpyFromSymbolAsync(&bad, g_png_violation, sizeof(bad), 0, cudaMemcpyDeviceToHost, c.stream));
    APT_CUDA(cudaStreamSynchronize(c.stream));
    if (bad) return fail(APT_ERR_CUDA, "PNG encoder bounds check failed (violation bits 0x%x)", bad);
#endif
    return APT_OK;
}

int OutPlan::set_png(const apt_png_settings *ps) {
    if (ps) {
        PngPlan pp;
        APT_TRY(make_png(kPxPerRow, 1, post.bpp, ps, pp));
        png_s = *ps;
    }
    png = ps != nullptr;
    return APT_OK;
}

int OutPlan::png_plan(uint64_t rows, PngPlan &pp) const {
    if (rows > 0xFFFFFFFFull) return fail(APT_ERR_BAD_ARG, "recording too long");
    return make_png(kPxPerRow, static_cast<uint32_t>(rows), post.bpp, &png_s, pp);
}

int OutPlan::bytes(uint64_t px, uint64_t &b) const {
    b = px_bytes(px);
    if (!png) return APT_OK;
    PngPlan pp;
    APT_TRY(png_plan(std::max<uint64_t>(px / kPxPerRow, 1), pp));
    b = pp.bound;
    return APT_OK;
}

int make_out_plan(const apt_process_settings *ps, const apt_png_settings *png, OutPlan &plan) {
    plan = OutPlan{};
    if (ps) {
        APT_TRY(make_post(*ps, plan.post));
        plan.image = true;
    }
    if (png && !ps) return fail(APT_ERR_BAD_ARG, "PNG output needs process settings");
    return plan.set_png(png);
}

int check_room(const void *dst, uint64_t need, uint64_t cap) {
    if (!dst || cap < need) return fail(APT_ERR_CAPACITY, "output needs room for %llu bytes", (unsigned long long)need);
    return APT_OK;
}

int ImageOut::reserve_px(uint64_t bytes) { return grow(px, px_cap, bytes, 1); }

int ImageOut::reserve_ctl(uint32_t g) {
    if (ctl_cap >= g) return APT_OK;
    if (h_ctl) cudaFreeHost(h_ctl);
    h_ctl = nullptr;
    ctl_cap = 0;
    APT_CUDA(cudaHostAlloc(reinterpret_cast<void **>(&h_ctl), g * sizeof(PngCtl), cudaHostAllocDefault));
    ctl_cap = g;
    return APT_OK;
}

int ImageOut::launch(const LaunchCtx &c, const float *rows, const SyncResult *res, u32 fixed_rows, u32 max_rows, void *out,
                     KernelHook *hook) {
    return post_launch(c, plan.post, post, rows, res, fixed_rows, max_rows, kPxPerRow, nullptr, out ? out : px, hook);
}

int ImageOut::encode(const LaunchCtx &c, const PngPlan *plans, const unsigned char *const *pixels, u32 g, KernelHook *hook) {
    APT_TRY(reserve_ctl(g));
    APT_TRY(png_encode_device(c, plans, pixels, g, work, hook));
    APT_CUDA(cudaMemcpyAsync(h_ctl, work.ctl, g * sizeof(PngCtl), cudaMemcpyDeviceToHost, c.stream));
    return APT_OK;
}

int ImageOut::encode_px(const LaunchCtx &c, uint64_t rows, KernelHook *hook) {
    PngPlan pp;
    APT_TRY(plan.png_plan(rows, pp));
    const unsigned char *p = px;
    return encode(c, &pp, &p, 1, hook);
}

int ImageOut::copy_out(u32 k, void *dst, uint64_t cap, cudaMemcpyKind kind, cudaStream_t s) const {
    const uint64_t n = length(k);
    APT_TRY(check_room(dst, n, cap));
    APT_CUDA(cudaMemcpyAsync(dst, work.out + work.lay.img[k].out, n, kind, s));
    return APT_OK;
}

uint64_t ImageOut::device_bytes(const OutPlan &p, uint64_t max_rows) {
    const PostPlan &q = p.post;
    uint64_t b = sizeof(PostCtl) + 3 * max_rows * sizeof(float) + (q.hist ? sizeof(ProcCtl) : 0) +
                 (q.finish ? max_rows * kPxPerRow : 0) + (q.palette ? 256 * 256 * sizeof(u32) : 0) + max_rows * kPxPerRow * q.bpp;
    PngPlan pp;
    PngLayout lay;
    if (p.png && p.png_plan(max_rows, pp) == APT_OK && png_layout(&pp, nullptr, 1, lay) == APT_OK) b += PngWork::bytes_for(lay);
    return b;
}

void ImageOut::release() {
    post.release();
    work.release();
    if (px) cudaFree(px);
    if (h_ctl) cudaFreeHost(h_ctl);
    px = nullptr;
    h_ctl = nullptr;
    px_cap = 0;
    ctl_cap = 0;
}

}  // namespace aptb200

using namespace aptb200;

namespace {

// apt_png_encode keeps one workspace per device (input pixels, encoder buffers, the pinned control blocks, a stream) for
// the next call, as the one-shot decode keeps its decoders; apt_cache_clear frees them.
constexpr int kStageDevices = 64;
struct PngStage {
    std::mutex mu;
    ImageOut out;                    // px: the input pixels
    cudaStream_t stream = nullptr;
    void release() {
        if (stream) cudaStreamSynchronize(stream);
        out.release();
        if (stream) cudaStreamDestroy(stream);
        stream = nullptr;
    }
};
std::mutex g_stage_mu;
PngStage *g_stage[kStageDevices] = {};

}  // namespace

void aptb200::png_stage_cache_clear() {
    int cur = 0;
    const bool have = cudaGetDevice(&cur) == cudaSuccess;
    std::lock_guard<std::mutex> lk(g_stage_mu);
    for (int d = 0; d < kStageDevices; ++d) {
        if (!g_stage[d]) continue;
        std::lock_guard<std::mutex> lk2(g_stage[d]->mu);
        cudaSetDevice(d);
        g_stage[d]->release();
    }
    if (have) cudaSetDevice(cur);
}

extern "C" void apt_png_default_settings(apt_png_settings *ps) {
    if (!ps) return;
    ps->filter = -1;
    ps->matches = 1;
    ps->block_bytes = 65536;
    ps->rgb_from_rgba = 0;
}

extern "C" int apt_png_bound(uint32_t width, uint32_t height, int channels, const apt_png_settings *ps, uint64_t *bytes) {
    if (!bytes) return fail(APT_ERR_BAD_ARG, "null argument");
    *bytes = 0;
    PngPlan p;
    APT_TRY(make_png(width, height, channels, ps, p));
    *bytes = p.bound;
    return APT_OK;
}

extern "C" int apt_png_group_plan(uint32_t width, int channels, const apt_png_settings *ps, const uint32_t *heights, uint32_t count,
                                  apt_png_group_info *info, apt_png_group_image *images, size_t cap) {
    if (!heights || !info) return fail(APT_ERR_BAD_ARG, "null argument");
    memset(info, 0, sizeof(*info));
    std::vector<PngPlan> plans(count);
    for (uint32_t k = 0; k < count; ++k) APT_TRY(make_png(width, heights[k], channels, ps, plans[k]));
    PngLayout lay;
    APT_TRY(png_layout(plans.data(), nullptr, count, lay));
    *info = apt_png_group_info{lay.f_bytes, lay.out_bytes, lay.rows, lay.spans, lay.blocks, lay.chunks};
    for (uint32_t k = 0; images && k < count && k < cap; ++k) {
        const PngImage &im = lay.img[k];
        images[k] = apt_png_group_image{im.pos, im.n, im.out, im.out_bytes, plans[k].bound, im.row0, im.span0, im.blk0,
                                        im.nblocks, im.chunk0, 0};
    }
    return APT_OK;
}

extern "C" int apt_png_encode(const uint8_t *pixels, uint32_t width, uint32_t height, int channels, const apt_png_settings *ps,
                              uint8_t *out, uint64_t cap, uint64_t *nout) {
    return apt_png_encode_batch(&pixels, &height, 1, width, channels, ps, &out, &cap, nout);
}

extern "C" int apt_png_encode_batch(const uint8_t *const *pixels, const uint32_t *heights, uint32_t count, uint32_t width,
                                    int channels, const apt_png_settings *ps, uint8_t *const *outs, const uint64_t *caps,
                                    uint64_t *nouts) {
    if (!pixels || !heights || !outs || !caps || !nouts) return fail(APT_ERR_BAD_ARG, "null argument");
    std::vector<PngPlan> plans(count);
    std::vector<u64> in_off(count + 1, 0);
    for (uint32_t k = 0; k < count; ++k) {
        if (!pixels[k] || !outs[k]) return fail(APT_ERR_BAD_ARG, "null argument");
        nouts[k] = 0;
        APT_TRY(make_png(width, heights[k], channels, ps, plans[k]));
        const u64 npx = static_cast<u64>(width) * heights[k];
        if (ps->rgb_from_rgba && !png_alpha_opaque(pixels[k], npx))
            return fail(APT_ERR_BAD_ARG, "rgb_from_rgba needs every alpha to be 255");
        in_off[k + 1] = in_off[k] + ((npx * channels + 15) & ~15ull);
    }
    if (count == 0) return APT_OK;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev <= 0) {
        cudaGetLastError();
        return fail(APT_ERR_CUDA, "no usable CUDA device (%s); this library has no CPU fallback",
                    e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    }
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (dev < 0 || dev >= kStageDevices) return fail(APT_ERR_CUDA, "device %d out of range", dev);
    PngStage *&slot = g_stage[dev];
    {
        std::lock_guard<std::mutex> lk(g_stage_mu);
        if (!slot) slot = new PngStage();
    }
    PngStage &sg = *slot;
    std::lock_guard<std::mutex> lk(sg.mu);   // one encode per device at a time: they share the workspace
    auto run = [&]() -> int {
        if (!sg.stream) APT_CUDA(cudaStreamCreateWithFlags(&sg.stream, cudaStreamNonBlocking));
        APT_TRY(sg.out.reserve_px(in_off[count]));
        std::vector<const unsigned char *> px(count);
        for (uint32_t k = 0; k < count; ++k) {
            px[k] = sg.out.px + in_off[k];
            APT_CUDA(cudaMemcpyAsync(sg.out.px + in_off[k], pixels[k], static_cast<u64>(width) * heights[k] * channels,
                                     cudaMemcpyHostToDevice, sg.stream));
        }
        APT_TRY(sg.out.encode(LaunchCtx{sg.stream, std::max(sms, 1)}, plans.data(), px.data(), count, nullptr));
        APT_CUDA(cudaStreamSynchronize(sg.stream));
        int first = APT_OK;
        for (uint32_t k = 0; k < count; ++k) {
            nouts[k] = sg.out.length(k);
            const int st = sg.out.copy_out(k, outs[k], caps[k], cudaMemcpyDeviceToHost, sg.stream);
            if (st == APT_ERR_CAPACITY && first == APT_OK) first = st;
            else if (st != APT_OK && st != APT_ERR_CAPACITY) return st;
        }
        APT_CUDA(cudaStreamSynchronize(sg.stream));
        return first;
    };
    const int st = run();
    if (st != APT_OK && sg.stream) cudaStreamSynchronize(sg.stream);
    return st;
}
