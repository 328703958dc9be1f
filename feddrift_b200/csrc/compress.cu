// K17: unbiased stochastic quantization (QSGD) of the client uploads of a [C, M, P] arena against their slots' models.
//
// Row r of rows [R, P] (R = C·M, row r = (c, m) with m = r % M) is quantized against θ_m = theta + m·t_stride (a padded
// ModelBank row stride is fine).  Two memory-bound passes per row, both skipping rows whose weight n[r] is not > 0:
//   1. bucket maxima σ_k = max |x_e − θ_e| over the trainable entries of the flat range [k·b, (k+1)·b) into smax [R, nb].
//      The values are non-negative floats, so their bit patterns order like unsigned ints and atomicMax on the bits is a
//      max that does not depend on the order of the updates: the result is bit-deterministic.  A warp folds the entries
//      it holds per bucket with a segmented shuffle scan first, so a bucket of b ≥ 128 costs one atomic per warp.
//   2. every trainable entry of a bucket with σ_k > 0 becomes qsgd_entry(x, θ, σ_k, s, uniform_hash(seed, r, e)).
// Each thread owns groups of 4 consecutive entries, read and written with 128-bit accesses when the row, anchor and mask
// are 16/16/4-byte aligned.  In-row indices are 32-bit (the binding caps P below 2³¹).
#include <climits>

#include "common.cuh"
#include "kernels.h"

namespace fdb {

namespace {

inline int qsgd_grid_x(long long groups, int R) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long need = (groups + 255) / 256, cap = (long long)sms * 8;
    return (int)max(1LL, min(need, cap) / max(1, min(R, 16)));
}

// the 4 entries of group g: |x − θ| of the trainable ones (0 otherwise) or the values themselves
template <bool kVec>
FDB_DEVICE void load4(const float* __restrict__ x, const float* __restrict__ th, const unsigned char* __restrict__ mask,
                      unsigned i0, unsigned P, float xv[4], float tv[4], bool on[4]) {
    if (kVec) {
        const float4 a = *reinterpret_cast<const float4*>(x + i0), t = *reinterpret_cast<const float4*>(th + i0);
        xv[0] = a.x; xv[1] = a.y; xv[2] = a.z; xv[3] = a.w;
        tv[0] = t.x; tv[1] = t.y; tv[2] = t.z; tv[3] = t.w;
        if (mask) {
            const uchar4 mk = *reinterpret_cast<const uchar4*>(mask + i0);
            on[0] = mk.x; on[1] = mk.y; on[2] = mk.z; on[3] = mk.w;
        } else {
            on[0] = on[1] = on[2] = on[3] = true;
        }
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const unsigned i = i0 + j;
            on[j] = i < P && (!mask || mask[i]);
            xv[j] = i < P ? x[i] : 0.f;
            tv[j] = i < P ? th[i] : 0.f;
        }
    }
}

template <bool kVec>
__global__ void __launch_bounds__(256) qsgd_bucket_max_kernel(const float* __restrict__ rows, const float* __restrict__ theta,
                                                              long long t_stride, int M, const float* __restrict__ n,
                                                              const unsigned char* __restrict__ mask, unsigned P, unsigned b,
                                                              unsigned nb, unsigned* __restrict__ smax) {
    const int r = blockIdx.y;
    if (n && !(n[r] > 0.f)) return;
    const float* x = rows + (size_t)r * P;
    const float* th = theta + (size_t)(r % M) * t_stride;
    unsigned* sm = smax + (size_t)r * nb;
    const unsigned lane = threadIdx.x & 31u, groups = (P + 3u) / 4u;
    const unsigned stride = gridDim.x * blockDim.x;
    // the loop runs per warp (every lane takes part in the shuffles); lanes past the end carry an out-of-range key
    for (unsigned base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < groups; base += stride) {
        const unsigned g = base + lane, i0 = g * 4u;
        float xv[4], tv[4];
        bool on[4];
        unsigned key = UINT_MAX;
        float acc = 0.f;
        if (g < groups) {
            load4<kVec>(x, th, mask, i0, P, xv, tv, on);
            key = i0 / b;
            unsigned kj = key, rj = i0 - key * b;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (j > 0 && ++rj == b) { rj = 0; ++kj; }
                const float v = on[j] ? fabsf(xv[j] - tv[j]) : 0.f;
                if (kj == key) acc = fmaxf(acc, v);
                else if (v > 0.f) atomicMax(sm + kj, __float_as_uint(v));   // a lane that straddles a bucket edge
            }
        }
        // segmented inclusive max over lanes with equal keys (keys are non-decreasing in the lane index)
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float ov = __shfl_up_sync(0xffffffffu, acc, o);
            const unsigned ok = __shfl_up_sync(0xffffffffu, key, o);
            if ((int)lane >= o && ok == key) acc = fmaxf(acc, ov);
        }
        const unsigned next = __shfl_down_sync(0xffffffffu, key, 1);
        if (g < groups && (lane == 31u || next != key) && acc > 0.f) atomicMax(sm + key, __float_as_uint(acc));
    }
}

template <bool kVec>
__global__ void __launch_bounds__(256) qsgd_apply_kernel(float* __restrict__ rows, const float* __restrict__ theta, long long t_stride,
                                                         int M, const float* __restrict__ n, const unsigned char* __restrict__ mask,
                                                         unsigned P, unsigned b, unsigned nb, const unsigned* __restrict__ smax,
                                                         float s, uint32_t seed) {
    const int r = blockIdx.y;
    if (n && !(n[r] > 0.f)) return;
    float* x = rows + (size_t)r * P;
    const float* th = theta + (size_t)(r % M) * t_stride;
    const unsigned* sm = smax + (size_t)r * nb;
    const unsigned groups = (P + 3u) / 4u;
    for (unsigned g = blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += gridDim.x * blockDim.x) {
        const unsigned i0 = g * 4u;
        float xv[4], tv[4];
        bool on[4];
        load4<kVec>(x, th, mask, i0, P, xv, tv, on);
        unsigned kj = i0 / b, rj = i0 - kj * b;
        bool any = false;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (j > 0 && ++rj == b) { rj = 0; ++kj; }
            if (!on[j]) continue;
            const float sg = __uint_as_float(sm[kj]);
            if (sg > 0.f) {
                xv[j] = qsgd_entry(xv[j], tv[j], sg, s, uniform_hash(seed, (uint32_t)r, (unsigned long long)(i0 + j)));
                any = true;
            }
        }
        if (!any) continue;
        if (kVec) {
            *reinterpret_cast<float4*>(x + i0) = make_float4(xv[0], xv[1], xv[2], xv[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (on[j]) x[i0 + j] = xv[j];
        }
    }
}

}  // namespace

int qsgd_slots_launch(float* rows, const float* theta, long long t_stride, int M, const float* n, const unsigned char* mask, int R,
                      long long P, int level, long long bucket, unsigned* scratch_smax, unsigned seed, cudaStream_t stream) {
    if (R <= 0 || P <= 0) return 0;
    if (P >= (1LL << 31) || level < 1 || level > 65535 || bucket < 1) return -5;
    const unsigned Pu = (unsigned)P, b = (unsigned)min(bucket, P), nb = (Pu + b - 1) / b;
    const bool vec = (P % 4 == 0) && (t_stride % 4 == 0) && ((reinterpret_cast<uintptr_t>(rows) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(theta) & 15) == 0) && ((reinterpret_cast<uintptr_t>(mask) & 3) == 0);
    cudaMemsetAsync(scratch_smax, 0, (size_t)R * nb * sizeof(unsigned), stream);
    const dim3 grid(qsgd_grid_x((P + 3) / 4, R), R);
    if (vec) {
        qsgd_bucket_max_kernel<true><<<grid, 256, 0, stream>>>(rows, theta, t_stride, M, n, mask, Pu, b, nb, scratch_smax);
        qsgd_apply_kernel<true><<<grid, 256, 0, stream>>>(rows, theta, t_stride, M, n, mask, Pu, b, nb, scratch_smax, (float)level, seed);
    } else {
        qsgd_bucket_max_kernel<false><<<grid, 256, 0, stream>>>(rows, theta, t_stride, M, n, mask, Pu, b, nb, scratch_smax);
        qsgd_apply_kernel<false><<<grid, 256, 0, stream>>>(rows, theta, t_stride, M, n, mask, Pu, b, nb, scratch_smax, (float)level, seed);
    }
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

}  // namespace fdb
