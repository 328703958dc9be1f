// K19: coordinate-wise robust aggregation (median / trimmed mean) of a [C, M, P] upload arena into the cluster models.
//
// ops/reference.py robust_aggregate_slots_ is the definition.  For slot m the participants are the rows c with
// n[c, m] > 0, each counted once.  Per entry, upload i has rank #{j : a_j < a_i} + #{j < i : a_j == a_i}; the values of
// rank b … n−1−b are summed in ascending rank order starting from the smallest kept one and divided once by (n − 2b).  A
// column holding a NaN yields NaN.  Every add and the division are rounded on their own, so the result matches the CPU
// oracle bit for bit and does not depend on the order of the clients.
//
// The values of one column are M·P floats apart, so a CTA stages a tile of T columns of all n participant rows in shared
// memory (128-bit streaming loads when aligned, row pitch T + 1 so that a warp reading one column down the rows hits 32
// banks), then each warp ranks one column at a time: lane i compares its values against the column (broadcast reads)
// and scatters them to their rank in a per-warp buffer; lane 0 sums the kept ranks.  The grid is persistent over the tiles
// of each slot, so the participant list is compacted once per CTA.  The ranking is O(n²) per column on chip.
//
// With a server optimizer (so.kind != 0) the statistic is avg_m and θ_m takes the common.cuh server_opt_update step on
// θ_m − avg_m in the store phase (entries with mask 0 take avg_m); the launcher's caller advances the step counters of the
// slots with a participant after the launch, as K1 does.
#include "common.cuh"
#include "kernels.h"

namespace fdb {

namespace {

constexpr int kThreads = 256, kWarps = kThreads / 32;
constexpr int kSmemBudget = 200 * 1024;

struct RobustOpt {
    int kind;  // 0 none, 1 sgd, 2 adam, 3 adagrad, 4 yogi
    float lr, momentum, b1, b2, eps;
    float *s0, *s1;
    const int* steps;
    const unsigned char* mask;
};

// floats of dynamic shared memory for tiles of T columns and up to C participants
inline size_t smem_floats_for(int C, int T) {
    return (size_t)C * (T + 1) + (size_t)kWarps * C + (size_t)C /* participant list */ + T /* results */ + 4;
}

__global__ void __launch_bounds__(kThreads) robust_aggregate_kernel(float* __restrict__ theta, long long t_stride,
                                                                   const float* __restrict__ cp, const float* __restrict__ n,
                                                                   int C, int M, long long P, int T, int median, float beta,
                                                                   RobustOpt so) {
    extern __shared__ __align__(16) float sm[];
    float* tile = sm;                                         // [nrows][T + 1]
    float* sorted = tile + (size_t)C * (T + 1);               // [kWarps][C]
    int* rows = reinterpret_cast<int*>(sorted + (size_t)kWarps * C);   // participant c, ascending
    float* res = reinterpret_cast<float*>(rows + C);          // [T] statistics of the tile
    __shared__ int cnt_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int m = blockIdx.y;

    if (warp == 0) {   // ordered compaction of the participants of slot m
        int base = 0;
        for (int c0 = 0; c0 < C; c0 += 32) {
            const int c = c0 + lane;
            const bool on = c < C && n[(size_t)c * M + m] > 0.f;
            const unsigned bal = __ballot_sync(0xffffffffu, on);
            if (on) rows[base + __popc(bal & ((1u << lane) - 1u))] = c;
            base += __popc(bal);
        }
        if (lane == 0) cnt_s = base;
    }
    __syncthreads();
    const int cnt = cnt_s;
    if (cnt == 0) return;
    const int b = median ? (cnt - 1) / 2 : (int)floorf(__fmul_rn(beta, (float)cnt));
    const float div = (float)(cnt - 2 * b);
    float bc1 = 1.f, bc2 = 1.f;
    if (so.kind != 0) {
        const float ts = (float)(so.steps[m] + 1);
        bc1 = 1.f - powf(so.b1, ts); bc2 = 1.f - powf(so.b2, ts);
    }
    const size_t rstride = (size_t)M * P;
    const int pitch = T + 1, T4 = T >> 2;
    const bool vec = ((P & 3) == 0) && ((((uintptr_t)cp) & 15) == 0);
    float* out = theta + (size_t)m * t_stride;
    float* mine = sorted + (size_t)warp * C;
    const long long ntiles = (P + T - 1) / T;

    for (long long tile_i = blockIdx.x; tile_i < ntiles; tile_i += gridDim.x) {
        const long long col0 = tile_i * T;
        const int tw = (int)min((long long)T, P - col0);
        // ---- stage the tile: participant r's columns [col0, col0 + tw)
        if (vec && tw == T) {
            for (int i = tid; i < cnt * T4; i += kThreads) {
                const int r = i / T4, q = i - r * T4;
                const float4 v = __ldcs(reinterpret_cast<const float4*>(cp + (size_t)rows[r] * rstride + (size_t)m * P + col0) + q);
                float* d = tile + (size_t)r * pitch + 4 * q;
                d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
            }
        } else {
            for (int i = tid; i < cnt * T; i += kThreads) {
                const int r = i / T, j = i - r * T;
                if (j < tw) tile[(size_t)r * pitch + j] = __ldcs(cp + (size_t)rows[r] * rstride + (size_t)m * P + col0 + j);
            }
        }
        __syncthreads();
        // ---- rank each column (warp per column), sum the kept ranks
        for (int j = warp; j < tw; j += kWarps) {
            bool nan = false;
            for (int i = lane; i < cnt; i += 32) {
                const float a = tile[(size_t)i * pitch + j];
                nan |= isnan(a);
                int rk = 0;
                for (int q = 0; q < cnt; ++q) {
                    const float x = tile[(size_t)q * pitch + j];
                    rk += (x < a || (x == a && q < i)) ? 1 : 0;
                }
                if (!isnan(a)) mine[rk] = a;   // ranks form a permutation unless the column holds a NaN
            }
            nan = __any_sync(0xffffffffu, nan);
            __syncwarp();
            if (lane == 0) {
                float v;
                if (nan) {
                    v = __int_as_float(0x7FC00000);
                } else {
                    float s = mine[b];
                    for (int q = b + 1; q < cnt - b; ++q) s = __fadd_rn(s, mine[q]);
                    v = __fdiv_rn(s, div);
                }
                res[j] = v;
            }
            __syncwarp();
        }
        __syncthreads();
        // ---- store (and step) the tile's entries of θ_m
        for (int j = tid; j < tw; j += kThreads) {
            const long long e = col0 + j;
            float v = res[j];
            if (so.kind != 0 && !(so.mask && !so.mask[e]))
                v = server_opt_update(so.kind, out[e], v, so.s0, so.s1, (size_t)m * P + e, so.lr, so.momentum, so.b1, so.b2, so.eps,
                                      bc1, bc2);
            out[e] = v;
        }
        __syncthreads();   // the next tile overwrites tile / res
    }
}

}  // namespace

int robust_aggregate_launch(float* theta, long long t_stride, const float* cp, const float* n, int C, int M, long long P,
                            int median, float beta, int opt_kind, float lr, float momentum, float b1, float b2, float eps,
                            float* s0, float* s1, const int* steps, const unsigned char* mask, cudaStream_t stream) {
    if (C <= 0 || M <= 0 || P <= 0) return 0;
    if (M > 65535) return -5;
    // widest tile (a multiple of 4 columns for the 128-bit loads) whose staging fits the budget for C participants
    int T = 128;
    while (T > 4 && smem_floats_for(C, T) * sizeof(float) > (size_t)kSmemBudget) T >>= 1;
    const size_t smem = smem_floats_for(C, T) * sizeof(float);
    if (smem > 227 * 1024) return -2;
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(robust_aggregate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return -3;
    }
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long ntiles = (P + T - 1) / T;
    const long long want = max(1LL, (long long)sms * 8 / M);
    dim3 grid((unsigned)min(ntiles, want), (unsigned)M);
    RobustOpt so{opt_kind, lr, momentum, b1, b2, eps, s0, s1, steps, mask};
    robust_aggregate_kernel<<<grid, kThreads, smem, stream>>>(theta, t_stride, cp, n, C, M, P, T, median, beta, so);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

}  // namespace fdb
