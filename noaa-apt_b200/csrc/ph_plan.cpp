// Geometry and phase table of the phase-major resampler (kernels_ph.cuh): host logic only.
#include <algorithm>

#include "launch.hpp"

namespace aptb200 {

bool make_ph_plan(u32 l, u32 m, const std::vector<float> &taps, PhPlan &pp, std::vector<float> &table,
                  std::vector<unsigned short> &xs) {
    pp = PhPlan{};
    if (l < 32 || m == 0 || m > 4096 || taps.empty()) return false;       // small L: the uniform-tap / tiled kernels
    const u64 n = taps.size();
    const u64 off2 = 2 * ((n - 1) / 2);                                   // highest tap index fast_resampling touches
    // taps per output: indices i0 + l*j <= off2 with i0 = xs*l - r*m in [0, l)
    u32 jmax = 0;
    xs.assign(l, 0);
    for (u32 r = 0; r < l; ++r) {
        const u64 x = (static_cast<u64>(r) * m + l - 1) / l;              // ceil(r*m / l)
        if (x > 65535) return false;
        xs[r] = static_cast<unsigned short>(x);
        const u64 i0 = x * l - static_cast<u64>(r) * m;
        if (i0 <= off2) jmax = std::max<u32>(jmax, static_cast<u32>((off2 - i0) / l + 1));
    }
    if (jmax == 0 || l % 4 != 0) return false;
    // groups of 4 consecutive phases share a window that starts at the 16-byte aligned row index xa[g] = (xs[4g] + 4) & ~3
    // (row[0] is X[M*q - 4]); the window must reach the last tap of the group's last phase
    const u32 ngroups = l / 4;
    u32 need = 0;
    std::vector<unsigned short> xa(ngroups);
    for (u32 gi = 0; gi < ngroups; ++gi) {
        const u32 a = (xs[4 * gi] + 4u) & ~3u;
        xa[gi] = static_cast<unsigned short>(a);
        need = std::max<u32>(need, xs[4 * gi + 3] + 4u - a + jmax);
    }
    const u32 win = need <= 24 ? 24 : need <= 44 ? 44 : need <= 84 ? 84 : 0;   // the kernel's instantiations
    if (win == 0) return false;
    const u32 row_len = (m + win + 8 + 3) / 4 * 4;
    u32 pitch = row_len;
    while (pitch % 32 != 4) pitch += 4;                                   // conflict-free LDS.128 across the 32 rows
    const size_t smem = (static_cast<size_t>(ngroups) * win * 4 + 33ull * pitch + 8ull * 32 * 33) * sizeof(float) +
                        ngroups * sizeof(unsigned short) + 16;
    if (smem > 227 * 1024) return false;
    // table[g][i][p] = tap of phase 4g+p that meets window element i, i.e. h[i0(r) + l*(i - (xs[r] + 4 - xa[g]))]
    table.assign(static_cast<size_t>(ngroups) * win * 4, 0.f);
    for (u32 r = 0; r < l; ++r) {
        const u32 gi = r / 4, ph = r % 4;
        const u64 i0 = static_cast<u64>(xs[r]) * l - static_cast<u64>(r) * m;
        const u32 shift = xs[r] + 4u - xa[gi];
        for (u32 j = 0; j < jmax; ++j) {
            const u64 idx = i0 + static_cast<u64>(l) * j;
            if (idx <= off2 && idx < n && shift + j < win)
                table[(static_cast<size_t>(gi) * win + shift + j) * 4 + ph] = taps[idx];
        }
    }
    xs = xa;                                                              // what the kernel needs: one window start per group
    pp.l = l;
    pp.m = m;
    pp.j = jmax;
    pp.jpad = win;
    pp.pitch = pitch;
    pp.row_len = row_len;
    pp.smem_bytes = static_cast<u32>(smem);
    return true;
}

}  // namespace aptb200
