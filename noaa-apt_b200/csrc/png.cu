// The PNG encoder (see png.hpp): settings, plan, tables, workspaces, the launch sequence and apt_png_* host entry points.
#include "png.hpp"

#include <algorithm>
#include <cstring>
#include <mutex>

#include "common.hpp"
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

int PngWork::reserve(const PngPlan &p) {
    APT_TRY(grow(f, cap_n, p.n + 16, 1));
    if (cap_n_pos < p.n) {
        for (void *q : {(void *)lcode, (void *)dist, (void *)flag})
            if (q) cudaFree(q);
        lcode = nullptr;
        dist = nullptr;
        flag = nullptr;
        cap_n_pos = 0;
        APT_CUDA(cudaMalloc(&lcode, p.n));
        APT_CUDA(cudaMalloc(&dist, p.n * sizeof(uint16_t)));
        APT_CUDA(cudaMalloc(&flag, p.n));
        cap_n_pos = p.n;
    }
    if (cap_blocks < p.nblocks) {
        for (void *q : {(void *)hist, (void *)codes, (void *)hdr, (void *)hdr_bits, (void *)bits, (void *)off, (void *)sums})
            if (q) cudaFree(q);
        hist = codes = hdr = hdr_bits = nullptr;
        bits = off = sums = nullptr;
        cap_blocks = 0;
        const u64 nb = p.nblocks;
        APT_CUDA(cudaMalloc(&hist, nb * (kPngLit + kPngDist) * sizeof(u32)));
        APT_CUDA(cudaMalloc(&codes, nb * (kPngLit + kPngDist) * sizeof(u32)));
        APT_CUDA(cudaMalloc(&hdr, nb * kPngHdrWords * sizeof(u32)));
        APT_CUDA(cudaMalloc(&hdr_bits, nb * sizeof(u32)));
        APT_CUDA(cudaMalloc(&bits, nb * sizeof(u64)));
        APT_CUDA(cudaMalloc(&off, nb * sizeof(u64)));
        APT_CUDA(cudaMalloc(&sums, 2 * nb * sizeof(u64)));
        cap_blocks = nb;
    }
    APT_TRY(grow(out, cap_out, (p.bound + 8) & ~3ull, 1));
    if (!ctl) APT_CUDA(cudaMalloc(&ctl, sizeof(PngCtl)));
    return APT_OK;
}

void PngWork::release() {
    for (void *q : {(void *)f, (void *)lcode, (void *)dist, (void *)flag, (void *)hist, (void *)codes, (void *)hdr, (void *)hdr_bits,
                    (void *)bits, (void *)off, (void *)sums, (void *)out, (void *)ctl})
        if (q) cudaFree(q);
    f = lcode = flag = out = nullptr;
    dist = nullptr;
    hist = codes = hdr = hdr_bits = nullptr;
    bits = off = sums = nullptr;
    ctl = nullptr;
    cap_n = cap_n_pos = cap_blocks = cap_out = 0;
}

size_t PngWork::device_bytes() const {
    return cap_n + cap_n_pos * 4 + cap_blocks * (2 * (kPngLit + kPngDist) * 4 + kPngHdrWords * 4 + 4 + 4 * 8) + cap_out +
           (ctl ? sizeof(PngCtl) : 0);
}

int png_encode_device(const LaunchCtx &c, const PngPlan &p, PngWork &w, const unsigned char *pixels, KernelHook *hook) {
    APT_TRY(ensure_tables());
    APT_TRY(w.reserve(p));
    const u32 n = static_cast<u32>(p.n);
    const u32 bb = p.s.block_bytes;
#ifdef APTB200_PNG_CHECK
    const PngLimits lim{p.n + 16, p.n, static_cast<u64>(p.width) * p.height * p.in_ch, (p.bound + 8) & ~3ull, p.nblocks};
    const u32 zero = 0;
    APT_CUDA(cudaMemcpyToSymbolAsync(c_png_lim, &lim, sizeof(lim), 0, cudaMemcpyHostToDevice, c.stream));
    APT_CUDA(cudaMemcpyToSymbolAsync(g_png_violation, &zero, sizeof(zero), 0, cudaMemcpyHostToDevice, c.stream));
#endif
    APT_CUDA(cudaMemsetAsync(w.f + p.n, 0, 16, c.stream));   // the padding png_ld32 may read past the last position
    APT_CUDA(cudaMemsetAsync(w.flag, 0, p.n, c.stream));
    APT_CUDA(cudaMemsetAsync(w.out, 0, (p.bound + 8) & ~3ull, c.stream));
    APT_CUDA(cudaMemsetAsync(w.ctl, 0, sizeof(PngCtl), c.stream));
    {
        KernelSlot ks(hook, "png_filter");
        const u32 grid = (p.height + 7) / 8;
        if (p.in_ch == 1) k_png_filter<1, 1><<<grid, 256, 0, c.stream>>>(pixels, p.width, p.height, p.s.filter, w.f);
        else if (p.in_ch == 3) k_png_filter<3, 3><<<grid, 256, 0, c.stream>>>(pixels, p.width, p.height, p.s.filter, w.f);
        else if (p.ch == 4) k_png_filter<4, 4><<<grid, 256, 0, c.stream>>>(pixels, p.width, p.height, p.s.filter, w.f);
        else k_png_filter<4, 3><<<grid, 256, 0, c.stream>>>(pixels, p.width, p.height, p.s.filter, w.f);
        APT_CUDA(cudaGetLastError());
    }
    if (p.s.matches) {
        KernelSlot ks(hook, "png_match");
        const size_t smem = 32768 * sizeof(uint16_t);
        APT_CUDA(cudaFuncSetAttribute(k_png_match, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
        k_png_match<<<(n + kPngSpan - 1) / kPngSpan, 32, smem, c.stream>>>(w.f, n, bb, w.lcode, w.dist);
        APT_CUDA(cudaGetLastError());
    } else {
        APT_CUDA(cudaMemsetAsync(w.lcode, 0, p.n, c.stream));   // literals only
    }
    {
        KernelSlot ks(hook, "png_parse");
        APT_CUDA(cudaFuncSetAttribute(k_png_parse, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bb)));
        k_png_parse<<<p.nblocks, 256, bb, c.stream>>>(w.f, w.lcode, w.dist, n, bb, w.flag, w.hist);
        APT_CUDA(cudaGetLastError());
    }
    {
        KernelSlot ks(hook, "png_huffman");
        k_png_huffman<<<p.nblocks, 32, 0, c.stream>>>(w.hist, p.nblocks, w.codes, w.hdr, w.hdr_bits, w.bits);
        APT_CUDA(cudaGetLastError());
    }
    {
        KernelSlot ks(hook, "png_scan");
        k_png_scan<<<1, 1024, 0, c.stream>>>(w.bits, p.nblocks, w.off, w.ctl);
        APT_CUDA(cudaGetLastError());
    }
    {
        KernelSlot ks(hook, "png_emit");
        k_png_emit<<<p.nblocks, kPngEmitThreads, 0, c.stream>>>(w.f, w.lcode, w.dist, w.flag, n, bb, w.codes, w.hdr, w.hdr_bits,
                                                                  w.off, reinterpret_cast<u32 *>(w.out), w.sums);
        APT_CUDA(cudaGetLastError());
    }
    {
        KernelSlot ks(hook, "png_frame");
        PngIhdr ih;
        memcpy(ih.b, p.ihdr, sizeof(ih.b));
        k_png_frame<<<1, 1, 0, c.stream>>>(w.sums, p.nblocks, n, bb, ih, w.out, w.ctl);
        APT_CUDA(cudaGetLastError());
    }
    {
        KernelSlot ks(hook, "png_crc");
        const u64 chunks = (p.bound - 37 + kPngCrcChunk - 1) / kPngCrcChunk;
        k_png_crc<<<static_cast<u32>((chunks + 255) / 256), 256, 0, c.stream>>>(w.out, w.ctl);
        APT_CUDA(cudaGetLastError());
    }
    {
        KernelSlot ks(hook, "png_end");
        k_png_end<<<1, 1, 0, c.stream>>>(w.out, w.ctl);
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

}  // namespace aptb200

using namespace aptb200;

namespace {

// apt_png_encode keeps one workspace per device (input pixels, encoder buffers, a stream, the pinned control block) for
// the next call, as the one-shot decode keeps its decoders; apt_cache_clear frees them.
constexpr int kStageDevices = 64;
struct PngStage {
    std::mutex mu;
    PngWork w;
    unsigned char *px = nullptr;
    u64 px_cap = 0;
    cudaStream_t stream = nullptr;
    PngCtl *h_ctl = nullptr;
    void release() {
        if (stream) cudaStreamSynchronize(stream);
        w.release();
        if (px) cudaFree(px);
        px = nullptr;
        px_cap = 0;
        if (h_ctl) cudaFreeHost(h_ctl);
        h_ctl = nullptr;
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

extern "C" int apt_png_encode(const uint8_t *pixels, uint32_t width, uint32_t height, int channels, const apt_png_settings *ps,
                              uint8_t *out, uint64_t cap, uint64_t *nout) {
    if (!pixels || !out || !nout) return fail(APT_ERR_BAD_ARG, "null argument");
    *nout = 0;
    PngPlan p;
    APT_TRY(make_png(width, height, channels, ps, p));
    const u64 npx = static_cast<u64>(width) * height;
    if (ps->rgb_from_rgba && !png_alpha_opaque(pixels, npx))
        return fail(APT_ERR_BAD_ARG, "rgb_from_rgba needs every alpha to be 255");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0) {
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
    const u64 in_bytes = npx * channels;
    auto run = [&]() -> int {
        if (!sg.stream) APT_CUDA(cudaStreamCreateWithFlags(&sg.stream, cudaStreamNonBlocking));
        if (!sg.h_ctl) APT_CUDA(cudaHostAlloc(reinterpret_cast<void **>(&sg.h_ctl), sizeof(PngCtl), cudaHostAllocDefault));
        APT_TRY(grow(sg.px, sg.px_cap, in_bytes, 1));
        APT_CUDA(cudaMemcpyAsync(sg.px, pixels, in_bytes, cudaMemcpyHostToDevice, sg.stream));
        APT_TRY(png_encode_device(LaunchCtx{sg.stream, std::max(sms, 1)}, p, sg.w, sg.px, nullptr));
        APT_CUDA(cudaMemcpyAsync(sg.h_ctl, sg.w.ctl, sizeof(PngCtl), cudaMemcpyDeviceToHost, sg.stream));
        APT_CUDA(cudaStreamSynchronize(sg.stream));
        const u64 total = sg.h_ctl->total;
        *nout = total;
        if (total > cap) return fail(APT_ERR_CAPACITY, "output needs room for %llu bytes", (unsigned long long)total);
        APT_CUDA(cudaMemcpyAsync(out, sg.w.out, total, cudaMemcpyDeviceToHost, sg.stream));
        APT_CUDA(cudaStreamSynchronize(sg.stream));
        return APT_OK;
    };
    const int st = run();
    if (st != APT_OK && sg.stream) cudaStreamSynchronize(sg.stream);
    return st;
}
