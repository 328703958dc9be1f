// K22: simulated Byzantine clients (model poisoning) over a [C, M, P] upload arena.
//
// Row r = c·M + m of rows [C·M, P] is the upload of client c for slot m; θ_m = theta + m·t_stride (a padded ModelBank row
// stride is fine).  An attacker pair is one with attackers[c] != 0 and n[r] > 0; only the entries whose mask byte is
// nonzero (all when mask is null) change.  Two shapes of pass (ops/reference.py attack_slots_ is the definition):
//   * sign_flip / gaussian: one elementwise pass over the attacker rows, 4 consecutive entries per thread, read and
//     written with 128-bit accesses when the rows, θ and the mask are 16/16/4-byte aligned (scalar otherwise).
//   * alie / ipm: a grid over (column tile, slot).  A thread owns one column of its slot and walks the participants in
//     client order: the honest mean μ, for ALIE then the population deviation σ, and writes the crafted value into every
//     attacker row of the slot.  __fadd_rn / __fmul_rn / __fdiv_rn / __fsqrt_rn keep every rounding of the oracle, and
//     there are no atomics, so the result is bit-identical to the CPU at any C and from launch to launch.
#include "common.cuh"
#include "kernels.h"

namespace fdb {

namespace {

inline int attack_grid_x(long long groups, int R) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long need = (groups + 255) / 256, cap = (long long)sms * 8;
    return (int)max(1LL, min(need, cap) / max(1, min(R, 16)));
}

template <bool kVec>
__global__ void __launch_bounds__(256) attack_rows_kernel(float* __restrict__ rows, const float* __restrict__ theta, long long t_stride,
                                                          int M, const float* __restrict__ n, const unsigned char* __restrict__ attackers,
                                                          const unsigned char* __restrict__ mask, long long P, int kind, float s,
                                                          uint32_t seed) {
    const int r = blockIdx.y;
    if (!attackers[r / M] || !(n[r] > 0.f)) return;
    float* x = rows + (size_t)r * P;
    const float* th = theta + (size_t)(r % M) * t_stride;
    const long long groups = (P + 3) / 4;
    for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < groups; g += (long long)gridDim.x * blockDim.x) {
        const long long i0 = g * 4;
        if (kVec) {
            float4 a = *reinterpret_cast<const float4*>(x + i0);
            const float4 t = *reinterpret_cast<const float4*>(th + i0);
            uchar4 mk = make_uchar4(1, 1, 1, 1);
            if (mask) mk = *reinterpret_cast<const uchar4*>(mask + i0);
            if (mk.x) a.x = attack_entry(kind, a.x, t.x, s, seed, (uint32_t)r, (unsigned long long)i0);
            if (mk.y) a.y = attack_entry(kind, a.y, t.y, s, seed, (uint32_t)r, (unsigned long long)i0 + 1);
            if (mk.z) a.z = attack_entry(kind, a.z, t.z, s, seed, (uint32_t)r, (unsigned long long)i0 + 2);
            if (mk.w) a.w = attack_entry(kind, a.w, t.w, s, seed, (uint32_t)r, (unsigned long long)i0 + 3);
            *reinterpret_cast<float4*>(x + i0) = a;
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const long long i = i0 + j;
                if (i < P && (!mask || mask[i])) x[i] = attack_entry(kind, x[i], th[i], s, seed, (uint32_t)r, (unsigned long long)i);
            }
        }
    }
}

__global__ void __launch_bounds__(256) attack_columns_kernel(float* __restrict__ rows, const float* __restrict__ theta, long long t_stride,
                                                             int C, int M, const float* __restrict__ n,
                                                             const unsigned char* __restrict__ attackers,
                                                             const unsigned char* __restrict__ mask, long long P, int kind, float s) {
    const int m = blockIdx.y;
    const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (e >= P || (mask && !mask[e])) return;
    const size_t rs = (size_t)M * P;
    const float* col = rows + (size_t)m * P + e;
    float acc = 0.f;
    int h = 0;
    for (int c = 0; c < C; ++c)
        if (!attackers[c] && n[c * M + m] > 0.f) { acc = __fadd_rn(acc, col[c * rs]); ++h; }
    if (h == 0) return;
    const float hf = (float)h, mu = __fdiv_rn(acc, hf);
    float v;
    if (kind == kAttackAlie) {
        float ss = 0.f;
        for (int c = 0; c < C; ++c)
            if (!attackers[c] && n[c * M + m] > 0.f) {
                const float d = __fsub_rn(col[c * rs], mu);
                ss = __fadd_rn(ss, __fmul_rn(d, d));
            }
        v = __fsub_rn(mu, __fmul_rn(s, __fsqrt_rn(__fdiv_rn(ss, hf))));
    } else {
        const float th = theta[(size_t)m * t_stride + e];
        v = __fsub_rn(th, __fmul_rn(s, __fsub_rn(mu, th)));
    }
    for (int c = 0; c < C; ++c)
        if (attackers[c] && n[c * M + m] > 0.f) rows[c * rs + (size_t)m * P + e] = v;
}

}  // namespace

int attack_slots_launch(float* rows, const float* theta, long long t_stride, int C, int M, long long P, const float* n,
                        const unsigned char* attackers, int kind, float scale, const unsigned char* mask, unsigned seed,
                        cudaStream_t stream) {
    if (C <= 0 || M <= 0 || P <= 0 || kind == kAttackNone) return 0;
    if (kind < kAttackSignFlip || kind > kAttackIpm || !(scale > 0.f) || !isfinite(scale)) return -5;
    if (kind == kAttackSignFlip || kind == kAttackGaussian) {
        const int R = C * M;
        if (R > 65535) return -5;
        const bool vec = (P % 4 == 0) && (t_stride % 4 == 0) && ((reinterpret_cast<uintptr_t>(rows) & 15) == 0) &&
                         ((reinterpret_cast<uintptr_t>(theta) & 15) == 0) && ((reinterpret_cast<uintptr_t>(mask) & 3) == 0);
        const dim3 grid(attack_grid_x((P + 3) / 4, R), R);
        if (vec)
            attack_rows_kernel<true><<<grid, 256, 0, stream>>>(rows, theta, t_stride, M, n, attackers, mask, P, kind, scale, seed);
        else
            attack_rows_kernel<false><<<grid, 256, 0, stream>>>(rows, theta, t_stride, M, n, attackers, mask, P, kind, scale, seed);
    } else {
        if (M > 65535) return -5;
        const dim3 grid((unsigned)((P + 255) / 256), M);
        attack_columns_kernel<<<grid, 256, 0, stream>>>(rows, theta, t_stride, C, M, n, attackers, mask, P, kind, scale);
    }
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

}  // namespace fdb
