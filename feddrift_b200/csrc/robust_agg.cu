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
//
// K20: geometric median (RFA's smoothed Weiszfeld iteration; ops/reference.py geomed_aggregate_slots_ is the definition) of
// the same participants, as R + 2 passes over their rows that share K19's compaction, tile staging and store phase:
//   pass 0        K19 (median) into the [M, P] iterate v;
//   pass 1 … R    per tile, v^(t−1) (v⁰ read back; later the weighted sum Σ fl32(w_i·x_i) / W of the tile's rows, written
//                 to v so that a slot whose W becomes 0 keeps it), then each row's fp64 partial distance over the tile's
//                 trainable columns, warp per row, accumulated per CTA in tile order and stored to [M, gridX, C];
//                 geomed_finish_kernel sums them in CTA order into d_i², w_i = fl32(1 / max(ν, d_i)) and W (fp32, client
//                 order), and marks the slot kept (n ≤ 2 or W = 0) or NaN (a NaN distance);
//   pass R + 1    v^R into θ_m through the store phase (server step included).
// No float atomics and a grid that depends only on the device and the shape, so every launch gives the same bits.
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

// widest tile (a multiple of 4 columns for the 128-bit loads) whose staging (floats_for(C, T) floats) fits the budget
template <class F>
inline int tile_width(int C, F floats_for) {
    int T = 128;
    while (T > 4 && floats_for(C, T) * sizeof(float) > (size_t)kSmemBudget) T >>= 1;
    return T;
}

inline int persistent_grid_x(long long ntiles, int M) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return (int)min(ntiles, max(1LL, (long long)sms * 8 / M));
}

// warp 0 lists the participants of slot m (n[c, m] > 0) in ascending c into rows; every thread gets their count
__device__ __forceinline__ int compact_participants(const float* __restrict__ n, int C, int M, int m, int* rows, int* cnt_s) {
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        int base = 0;
        for (int c0 = 0; c0 < C; c0 += 32) {
            const int c = c0 + lane;
            const bool on = c < C && n[(size_t)c * M + m] > 0.f;
            const unsigned bal = __ballot_sync(0xffffffffu, on);
            if (on) rows[base + __popc(bal & ((1u << lane) - 1u))] = c;
            base += __popc(bal);
        }
        if (lane == 0) *cnt_s = base;
    }
    __syncthreads();
    return *cnt_s;
}

// stage columns [col0, col0 + tw) of the cnt participant rows of slot m into tile (row pitch T + 1); vec: 128-bit loads
__device__ __forceinline__ void stage_tile(float* tile, const float* __restrict__ cp, const int* rows, int cnt, size_t rstride,
                                           int m, long long P, long long col0, int T, int tw, bool vec) {
    const int pitch = T + 1, T4 = T >> 2;
    if (vec && tw == T) {
        for (int i = threadIdx.x; i < cnt * T4; i += kThreads) {
            const int r = i / T4, q = i - r * T4;
            const float4 v = __ldcs(reinterpret_cast<const float4*>(cp + (size_t)rows[r] * rstride + (size_t)m * P + col0) + q);
            float* d = tile + (size_t)r * pitch + 4 * q;
            d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
        }
    } else {
        for (int i = threadIdx.x; i < cnt * T; i += kThreads) {
            const int r = i / T, j = i - r * T;
            if (j < tw) tile[(size_t)r * pitch + j] = __ldcs(cp + (size_t)rows[r] * rstride + (size_t)m * P + col0 + j);
        }
    }
}

// the store phase: θ_m[e] = v, or the server optimizer's step on θ_m[e] − v (entries with mask 0 take v)
__device__ __forceinline__ void store_entry(float* out, long long e, float v, const RobustOpt& so, size_t m, long long P,
                                            float bc1, float bc2) {
    if (so.kind != 0 && !(so.mask && !so.mask[e]))
        v = server_opt_update(so.kind, out[e], v, so.s0, so.s1, m * P + e, so.lr, so.momentum, so.b1, so.b2, so.eps, bc1, bc2);
    out[e] = v;
}

__device__ __forceinline__ void server_bias_corrections(const RobustOpt& so, int m, float* bc1, float* bc2) {
    *bc1 = 1.f; *bc2 = 1.f;
    if (so.kind != 0) {
        const float ts = (float)(so.steps[m] + 1);
        *bc1 = 1.f - powf(so.b1, ts); *bc2 = 1.f - powf(so.b2, ts);
    }
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

    const int cnt = compact_participants(n, C, M, m, rows, &cnt_s);
    if (cnt == 0) return;
    const int b = median ? (cnt - 1) / 2 : (int)floorf(__fmul_rn(beta, (float)cnt));
    const float div = (float)(cnt - 2 * b);
    float bc1, bc2;
    server_bias_corrections(so, m, &bc1, &bc2);
    const size_t rstride = (size_t)M * P;
    const int pitch = T + 1;
    const bool vec = ((P & 3) == 0) && ((((uintptr_t)cp) & 15) == 0);
    float* out = theta + (size_t)m * t_stride;
    float* mine = sorted + (size_t)warp * C;
    const long long ntiles = (P + T - 1) / T;

    for (long long tile_i = blockIdx.x; tile_i < ntiles; tile_i += gridDim.x) {
        const long long col0 = tile_i * T;
        const int tw = (int)min((long long)T, P - col0);
        // ---- stage the tile: participant r's columns [col0, col0 + tw)
        stage_tile(tile, cp, rows, cnt, rstride, m, P, col0, T, tw, vec);
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
        for (int j = tid; j < tw; j += kThreads) store_entry(out, col0 + j, res[j], so, (size_t)m, P, bc1, bc2);
        __syncthreads();   // the next tile overwrites tile / res
    }
}

// ---------------------------------------------------------------------------------------------------------------- K20
struct GeomedState {
    float* v;       // [M, P] iterate
    double* part;   // [M, gridX, C] per-CTA partial squared distances of the participants (compacted order)
    float* w;       // [M, C] Weiszfeld weights
    float* wsum;    // [M] W
    int* mode;      // [M] 0 iterate, 1 keep v (n <= 2 or W = 0), 2 NaN
};
constexpr int kGmIterate = 0, kGmKeep = 1, kGmNaN = 2;

// bytes of dynamic shared memory of geomed_pass_kernel: distance accumulators [C] (double), tile [C][T + 1], participant
// list [C], weights [C], the tile's v [T]
inline size_t geomed_smem_bytes(int C, int T) {
    return (size_t)C * sizeof(double) + ((size_t)C * (T + 1) + 2 * (size_t)C + T) * sizeof(float) + 16;
}

// One pass of K20 over the column tiles of each slot (grid (gridX, M), persistent like K19).  pass 1 starts from v⁰;
// later passes form v from the weights of the previous finish step; the last pass stores v into θ_m.
__global__ void __launch_bounds__(kThreads) geomed_pass_kernel(float* __restrict__ theta, long long t_stride,
                                                              const float* __restrict__ cp, const float* __restrict__ n, int C,
                                                              int M, long long P, int T, bool first, bool last,
                                                              const unsigned char* __restrict__ dmask, RobustOpt so,
                                                              GeomedState gs) {
    extern __shared__ __align__(16) float sm[];
    double* dacc = reinterpret_cast<double*>(sm);             // [C] this CTA's partial distances
    float* tile = reinterpret_cast<float*>(dacc + C);         // [nrows][T + 1]
    int* rows = reinterpret_cast<int*>(tile + (size_t)C * (T + 1));
    float* wts = reinterpret_cast<float*>(rows + C);           // [C]
    float* res = wts + C;                                      // [T] the tile's entries of v
    __shared__ int cnt_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int m = blockIdx.y;
    const int cnt = compact_participants(n, C, M, m, rows, &cnt_s);
    if (cnt == 0) return;
    const int mode = (cnt <= 2) ? kGmKeep : gs.mode[m];
    if (!last && mode != kGmIterate) return;   // nothing left to refine: the last pass stores v (or NaN)
    float bc1, bc2;
    server_bias_corrections(so, m, &bc1, &bc2);
    float* out = theta + (size_t)m * t_stride;
    float* vm = gs.v + (size_t)m * P;
    const long long ntiles = (P + T - 1) / T;
    if (mode != kGmIterate) {   // last pass of a kept / NaN slot: no rows to read
        for (long long tile_i = blockIdx.x; tile_i < ntiles; tile_i += gridDim.x)
            for (int j = tid; j < T && tile_i * T + j < P; j += kThreads) {
                const long long e = tile_i * T + j;
                store_entry(out, e, mode == kGmNaN ? __int_as_float(0x7FC00000) : vm[e], so, (size_t)m, P, bc1, bc2);
            }
        return;
    }
    for (int i = tid; i < cnt; i += kThreads) {
        dacc[i] = 0.0;
        if (!first) wts[i] = gs.w[(size_t)m * C + i];
    }
    const float W = first ? 1.f : gs.wsum[m];
    const size_t rstride = (size_t)M * P;
    const int pitch = T + 1;
    const bool vec = ((P & 3) == 0) && ((((uintptr_t)cp) & 15) == 0);
    __syncthreads();

    for (long long tile_i = blockIdx.x; tile_i < ntiles; tile_i += gridDim.x) {
        const long long col0 = tile_i * T;
        const int tw = (int)min((long long)T, P - col0);
        stage_tile(tile, cp, rows, cnt, rstride, m, P, col0, T, tw, vec);
        __syncthreads();
        // ---- v of the tile: v⁰, or fl32(Σ_i fl32(w_i·x_i)) / W in client order over the rows with w_i != 0
        for (int j = tid; j < tw; j += kThreads) {
            float v;
            if (first) {
                v = vm[col0 + j];
            } else {
                float acc = 0.f;
                for (int i = 0; i < cnt; ++i) {
                    const float wi = wts[i];
                    if (wi != 0.f) acc = __fadd_rn(acc, __fmul_rn(wi, tile[(size_t)i * pitch + j]));
                }
                v = __fdiv_rn(acc, W);
            }
            res[j] = v;
            if (last) store_entry(out, col0 + j, v, so, (size_t)m, P, bc1, bc2);
            else if (!first) vm[col0 + j] = v;   // a slot whose W becomes 0 keeps this iterate
        }
        if (!last) {
            __syncthreads();
            // ---- squared distances to v over the tile's trainable columns, warp per row, added in tile order
            for (int i = warp; i < cnt; i += kWarps) {
                double s = 0.0;
                for (int j = lane; j < tw; j += 32)
                    if (!dmask || dmask[col0 + j]) {
                        const double d = (double)__fsub_rn(tile[(size_t)i * pitch + j], res[j]);
                        s = fma(d, d, s);
                    }
                s = warp_sum(s);
                if (lane == 0) dacc[i] += s;
            }
        }
        __syncthreads();   // the next tile overwrites tile / res
    }
    if (!last)
        for (int i = tid; i < cnt; i += kThreads) gs.part[((size_t)m * gridDim.x + blockIdx.x) * C + i] = dacc[i];
}

// After pass t: d_i² = the CTA partials summed in CTA order, w_i = fl32(1 / max(ν, d_i)) (float64), W = their fp32 sum in
// client order; a NaN distance marks the slot NaN, W = 0 (or n <= 2) keeps v.  One CTA per slot.
__global__ void __launch_bounds__(kThreads) geomed_finish_kernel(const float* __restrict__ n, int C, int M, int gx, double nu,
                                                                GeomedState gs) {
    extern __shared__ __align__(16) float sm[];
    int* rows = reinterpret_cast<int*>(sm);
    float* w = reinterpret_cast<float*>(rows + C);
    __shared__ int cnt_s, nan_s;
    const int m = blockIdx.x;
    if (threadIdx.x == 0) nan_s = 0;
    const int cnt = compact_participants(n, C, M, m, rows, &cnt_s);
    if (cnt <= 2 || gs.mode[m] != kGmIterate) {
        if (threadIdx.x == 0 && cnt > 0 && cnt <= 2) gs.mode[m] = kGmKeep;
        return;
    }
    for (int i = threadIdx.x; i < cnt; i += kThreads) {
        double d = 0.0;
        for (int b = 0; b < gx; ++b) d += gs.part[((size_t)m * gx + b) * C + i];
        if (isnan(d)) nan_s = 1;
        const float wi = isnan(d) ? 0.f : (float)(1.0 / fmax(nu, sqrt(d)));
        w[i] = wi;
        gs.w[(size_t)m * C + i] = wi;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float W = 0.f;
        for (int i = 0; i < cnt; ++i) W = __fadd_rn(W, w[i]);
        gs.wsum[m] = W;
        gs.mode[m] = nan_s ? kGmNaN : (W == 0.f ? kGmKeep : kGmIterate);
    }
}

}  // namespace

int robust_aggregate_launch(float* theta, long long t_stride, const float* cp, const float* n, int C, int M, long long P,
                            int median, float beta, int opt_kind, float lr, float momentum, float b1, float b2, float eps,
                            float* s0, float* s1, const int* steps, const unsigned char* mask, cudaStream_t stream) {
    if (C <= 0 || M <= 0 || P <= 0) return 0;
    if (M > 65535) return -5;
    const int T = tile_width(C, smem_floats_for);
    const size_t smem = smem_floats_for(C, T) * sizeof(float);
    if (smem > 227 * 1024) return -2;
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(robust_aggregate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return -3;
    }
    dim3 grid((unsigned)persistent_grid_x((P + T - 1) / T, M), (unsigned)M);
    RobustOpt so{opt_kind, lr, momentum, b1, b2, eps, s0, s1, steps, mask};
    robust_aggregate_kernel<<<grid, kThreads, smem, stream>>>(theta, t_stride, cp, n, C, M, P, T, median, beta, so);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

namespace {
inline int geomed_tile(int C) {
    return tile_width(C, [](int c, int t) { return (geomed_smem_bytes(c, t) + 3) / 4; });
}
}  // namespace

long long geomed_scratch_bytes(int C, int M, long long P) {
    if (C <= 0 || M <= 0 || P <= 0) return 0;
    const int T = geomed_tile(C);
    const long long gx = persistent_grid_x((P + T - 1) / T, M);
    return (long long)M * gx * C * 8 + (long long)M * P * 4 + (long long)M * C * 4 + (long long)M * 8;
}

int geomed_aggregate_launch(float* theta, long long t_stride, const float* cp, const float* n, int C, int M, long long P, int iters,
                            double nu, const unsigned char* dmask, int opt_kind, float lr, float momentum, float b1, float b2,
                            float eps, float* s0, float* s1, const int* steps, const unsigned char* mask, void* scratch,
                            cudaStream_t stream) {
    if (C <= 0 || M <= 0 || P <= 0) return 0;
    if (M > 65535) return -5;
    const int T = geomed_tile(C);
    const size_t smem = geomed_smem_bytes(C, T);
    if (smem > 227 * 1024) return -2;
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(geomed_pass_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return -3;
    }
    const size_t fsmem = (size_t)C * 8;
    if (fsmem > 227 * 1024) return -2;
    if (fsmem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(geomed_finish_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem);
        if (e != cudaSuccess) return -3;
    }
    const int gx = persistent_grid_x((P + T - 1) / T, M);
    char* sp = static_cast<char*>(scratch);
    GeomedState gs;
    gs.part = reinterpret_cast<double*>(sp);              sp += (size_t)M * gx * C * 8;
    gs.v = reinterpret_cast<float*>(sp);                  sp += (size_t)M * P * 4;
    gs.w = reinterpret_cast<float*>(sp);                  sp += (size_t)M * C * 4;
    gs.wsum = reinterpret_cast<float*>(sp);               sp += (size_t)M * 4;
    gs.mode = reinterpret_cast<int*>(sp);
    // pass 0: v⁰ = the coordinate-wise median (K19, no server step)
    int rc = robust_aggregate_launch(gs.v, P, cp, n, C, M, P, 1, 0.f, 0, 0.f, 0.f, b1, b2, eps, nullptr, nullptr, nullptr, nullptr,
                                     stream);
    if (rc != 0) return rc;
    if (cudaMemsetAsync(gs.mode, 0, (size_t)M * sizeof(int), stream) != cudaSuccess) return -4;
    const RobustOpt none{0, 0.f, 0.f, b1, b2, eps, nullptr, nullptr, nullptr, nullptr};
    const RobustOpt so{opt_kind, lr, momentum, b1, b2, eps, s0, s1, steps, mask};
    const dim3 grid((unsigned)gx, (unsigned)M);
    for (int t = 1; t <= iters + 1; ++t) {
        const bool last = t == iters + 1;
        geomed_pass_kernel<<<grid, kThreads, smem, stream>>>(theta, t_stride, cp, n, C, M, P, T, t == 1, last, dmask,
                                                             last ? so : none, gs);
        if (!last) geomed_finish_kernel<<<M, kThreads, fsmem, stream>>>(n, C, M, gx, nu, gs);
        if (cudaGetLastError() != cudaSuccess) return -4;
    }
    return 0;
}

}  // namespace fdb
