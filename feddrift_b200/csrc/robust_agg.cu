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
//
// K21: Multi-Krum (ops/reference.py krum_aggregate_slots_ is the definition) of the same participants, in three launches:
//   distance pass  K19's compaction and tile staging; thread per pair (i < j), the fp64 partial Σ fl32(x_i − x_j)² over
//                  the tile's trainable columns, added in tile order into the pair's accumulator (shared memory when the
//                  n(n − 1)/2 pairs fit beside a tile of ≥ 32 columns, else the CTA's own row in global memory, so any C
//                  the staging takes works); stored per CTA to [M, gridX, npairs];
//   select step    one CTA per slot sums the partials in CTA order, warp per row ranks its distances and sums the k
//                  smallest in order into the score, ranks the scores and writes the m_eff selected rows (client order);
//   store pass     the fp32 sum of the selected rows in client order, one division by m_eff, into θ_m through the store
//                  phase (server step included).
// The participants' rows are read once (the store pass reads the m_eff selected ones again).  No float atomics and a grid
// fixed by the device and the shape, so every launch gives the same bits.
//
// K23: centered clipping (ops/reference.py cclip_aggregate_slots_ is the definition) of the same participants around the
// slot's state h_m (center [M, P]), as L + 1 passes that share K19's compaction, tile staging and store phase:
//   pass 1 … L    per tile, v^(l−1) (pass 1: h read back; later v^(l−2) + fl32(Σ_i fl32(s_i·u_i) / n) from the clip factors
//                 of the previous finish step, written over h in place so that the next pass reads it), then each row's
//                 fp64 partial Σ fl32(fl32(x − θ) − v)² over the tile's trainable columns, warp per row, accumulated per
//                 CTA in tile order and stored to [M, gridX, C]; cclip_finish_kernel sums them in CTA order into r_i²,
//                 s_i = fl32(min(1, τ / r_i)) (float64) and marks the slot NaN on a NaN distance;
//   pass L + 1    v^L, θ_m + v^L into θ_m through the store phase (server step included) and v^L into h_m.
// The participants' rows are read L + 1 times.  No float atomics and a grid that depends only on the device and the shape,
// so every launch gives the same bits.
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

// ---------------------------------------------------------------------------------------------------------------- K21
constexpr long long kKrumPartBudget = 1LL << 23;   // doubles of [M, gridX, npairs] partials (64 MB) the grid may use

__host__ __device__ inline long long krum_npairs(int C) { return C >= 2 ? (long long)C * (C - 1) / 2 : 1; }

// bytes of dynamic shared memory of krum_dist_kernel: the pair accumulators [npairs(C)] (double; only when they stay on
// chip), tile [C][T + 1], participant list [C], the tile's distance mask [T] (bytes)
inline size_t krum_dist_smem_bytes(int C, int T, bool acc_on_chip) {
    return (acc_on_chip ? (size_t)krum_npairs(C) * sizeof(double) : 0) + (size_t)C * (T + 2) * sizeof(float) + T + 16;
}

// bytes of dynamic shared memory of krum_select_kernel: scores [C] and two distance rows [C] per warp (double), the
// participant list and the selection flags [C] (int)
inline size_t krum_select_smem_bytes(int C) { return (size_t)C * (1 + 2 * kWarps) * sizeof(double) + (size_t)C * 8 + 16; }

// pair p of the lower triangle, p = j(j − 1)/2 + i with 0 ≤ i < j (consecutive p: consecutive rows i of one j)
__device__ __forceinline__ void krum_pair(int p, int* i, int* j) {
    int r = (int)((1.0 + sqrt(1.0 + 8.0 * (double)p)) * 0.5);
    while ((long long)r * (r - 1) / 2 > p) --r;
    while ((long long)(r + 1) * r / 2 <= p) ++r;
    *j = r;
    *i = p - (int)((long long)r * (r - 1) / 2);
}

// Distance pass (grid (gridX, M), persistent over the column tiles of each slot like K19): the fp64 partials
// Σ fl32(x_i − x_j)² over this CTA's trainable columns of every pair of participants, thread per pair, each tile's sum
// added in tile order into the pair's accumulator (on chip when they fit, else the CTA's own row of part), stored to
// part [M, gridX, npairs(C)].  The participants' rows are read once.
__global__ void __launch_bounds__(kThreads) krum_dist_kernel(const float* __restrict__ cp, const float* __restrict__ n, int C,
                                                            int M, long long P, int T, bool acc_on_chip,
                                                            const unsigned char* __restrict__ dmask, double* __restrict__ part) {
    extern __shared__ __align__(16) float sm[];
    const long long npmax = krum_npairs(C);
    double* dacc = reinterpret_cast<double*>(sm);
    float* tile = reinterpret_cast<float*>(dacc + (acc_on_chip ? npmax : 0));   // [nrows][T + 1]
    int* rows = reinterpret_cast<int*>(tile + (size_t)C * (T + 1));
    unsigned char* mk = reinterpret_cast<unsigned char*>(rows + C);          // [T]
    __shared__ int cnt_s;
    const int tid = threadIdx.x;
    const int m = blockIdx.y;
    const int cnt = compact_participants(n, C, M, m, rows, &cnt_s);
    if (cnt < 2) return;
    const int np = cnt * (cnt - 1) / 2;
    double* mine = part + ((size_t)m * gridDim.x + blockIdx.x) * npmax;
    double* acc = acc_on_chip ? dacc : mine;
    for (int p = tid; p < np; p += kThreads) acc[p] = 0.0;
    const size_t rstride = (size_t)M * P;
    const int pitch = T + 1;
    const bool vec = ((P & 3) == 0) && ((((uintptr_t)cp) & 15) == 0);
    const long long ntiles = (P + T - 1) / T;
    for (long long tile_i = blockIdx.x; tile_i < ntiles; tile_i += gridDim.x) {
        const long long col0 = tile_i * T;
        const int tw = (int)min((long long)T, P - col0);
        stage_tile(tile, cp, rows, cnt, rstride, m, P, col0, T, tw, vec);
        for (int j = tid; j < tw; j += kThreads) mk[j] = dmask ? dmask[col0 + j] : 1;
        __syncthreads();
        for (int p = tid; p < np; p += kThreads) {
            int i, j;
            krum_pair(p, &i, &j);
            const float* a = tile + (size_t)i * pitch;
            const float* b = tile + (size_t)j * pitch;
            double s = 0.0;
            for (int c = 0; c < tw; ++c)
                if (mk[c]) {
                    const double d = (double)__fsub_rn(a[c], b[c]);
                    s = fma(d, d, s);
                }
            acc[p] += s;
        }
        __syncthreads();   // the next tile overwrites tile / mk
    }
    if (acc_on_chip)
        for (int p = tid; p < np; p += kThreads) mine[p] = dacc[p];
}

// Select step, one CTA per slot: D_ij = the CTA partials summed in CTA order (NaN → +∞, written over the first CTA's
// partial), score_i = Σ of the k = clamp(n − f − 2, 1, n − 1) smallest D_ij (j ≠ i) in ascending order, ties by j (warp
// per row: rank, scatter, lane 0 sums), then the m_eff = min(mkeep, n) best scores (ties to the lower row) as client
// indices in client order into sel [M, C] and m_eff into selcnt [M] (n = 1: that row; n = 0: 0).
__global__ void __launch_bounds__(kThreads) krum_select_kernel(const float* __restrict__ n, int C, int M, int gx, int f, int mkeep,
                                                              double* __restrict__ part, int* __restrict__ sel,
                                                              int* __restrict__ selcnt) {
    extern __shared__ __align__(16) float sm[];
    double* score = reinterpret_cast<double*>(sm);            // [C]
    double* dbuf = score + C;                                 // [kWarps][C] distances of the warp's row
    double* sbuf = dbuf + (size_t)kWarps * C;                 // [kWarps][C] the same, sorted
    int* rows = reinterpret_cast<int*>(sbuf + (size_t)kWarps * C);
    int* chosen = rows + C;
    __shared__ int cnt_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int m = blockIdx.x;
    const int cnt = compact_participants(n, C, M, m, rows, &cnt_s);
    if (cnt < 2) {
        if (tid == 0) {
            if (cnt == 1) sel[(size_t)m * C] = rows[0];
            selcnt[m] = cnt;
        }
        return;
    }
    const long long npmax = krum_npairs(C);
    const int np = cnt * (cnt - 1) / 2;
    double* D = part + (size_t)m * gx * npmax;
    for (int p = tid; p < np; p += kThreads) {
        double d = 0.0;
        for (int b = 0; b < gx; ++b) d += D[(size_t)b * npmax + p];
        D[p] = isnan(d) ? (double)INFINITY : d;
    }
    __syncthreads();
    const int k = min(max(cnt - f - 2, 1), cnt - 1);
    double* dv = dbuf + (size_t)warp * C;
    double* sv = sbuf + (size_t)warp * C;
    for (int i = warp; i < cnt; i += kWarps) {
        for (int j = lane; j < cnt; j += 32)
            if (j != i) dv[j] = D[j > i ? j * (j - 1) / 2 + i : i * (i - 1) / 2 + j];
        __syncwarp();
        for (int j = lane; j < cnt; j += 32) {
            if (j == i) continue;
            const double a = dv[j];
            int rk = 0;
            for (int l = 0; l < cnt; ++l) {
                if (l == i) continue;
                const double x = dv[l];
                rk += (x < a || (x == a && l < j)) ? 1 : 0;
            }
            if (rk < k) sv[rk] = a;
        }
        __syncwarp();
        if (lane == 0) {
            double s = 0.0;
            for (int r = 0; r < k; ++r) s += sv[r];
            score[i] = s;
        }
        __syncwarp();
    }
    __syncthreads();
    const int meff = min(mkeep, cnt);
    for (int i = tid; i < cnt; i += kThreads) {
        const double a = score[i];
        int rk = 0;
        for (int l = 0; l < cnt; ++l) rk += (score[l] < a || (score[l] == a && l < i)) ? 1 : 0;
        chosen[i] = rk < meff;
    }
    __syncthreads();
    if (tid == 0) {
        int q = 0;
        for (int i = 0; i < cnt; ++i)
            if (chosen[i]) sel[(size_t)m * C + q++] = rows[i];
        selcnt[m] = q;
    }
}

// Store pass (grid (gridX, M)): v_e = the fp32 sum of the selected rows in client order from the first one, one division
// by m_eff when m_eff > 1, into θ_m through K19's store phase (server step included).  Reads only the selected rows.
__global__ void __launch_bounds__(kThreads) krum_store_kernel(float* __restrict__ theta, long long t_stride,
                                                             const float* __restrict__ cp, int C, int M, long long P,
                                                             const int* __restrict__ sel, const int* __restrict__ selcnt,
                                                             RobustOpt so) {
    extern __shared__ __align__(16) float sm[];
    int* rows = reinterpret_cast<int*>(sm);
    const int m = blockIdx.y;
    const int q = selcnt[m];
    if (q == 0) return;
    for (int i = threadIdx.x; i < q; i += kThreads) rows[i] = sel[(size_t)m * C + i];
    __syncthreads();
    float bc1, bc2;
    server_bias_corrections(so, m, &bc1, &bc2);
    const size_t rstride = (size_t)M * P;
    const float* base = cp + (size_t)m * P;
    float* out = theta + (size_t)m * t_stride;
    for (long long e = (long long)blockIdx.x * kThreads + threadIdx.x; e < P; e += (long long)gridDim.x * kThreads) {
        float v = __ldcs(base + (size_t)rows[0] * rstride + e);
        for (int i = 1; i < q; ++i) v = __fadd_rn(v, __ldcs(base + (size_t)rows[i] * rstride + e));
        if (q > 1) v = __fdiv_rn(v, (float)q);
        store_entry(out, e, v, so, (size_t)m, P, bc1, bc2);
    }
}

// ---------------------------------------------------------------------------------------------------------------- K23
struct CclipState {
    float* h;       // [M, P] the slots' centers; holds the iterate v between passes
    double* part;   // [M, gridX, C] per-CTA partial squared distances of the participants (compacted order)
    float* s;       // [M, C] clip factors of the last finish step
    int* nan;       // [M] 1: a NaN distance, the slot becomes NaN
};

// bytes of dynamic shared memory of cclip_pass_kernel: distance accumulators [C] (double), tile [C][T + 1], participant
// list [C], clip factors [C], the tile's θ and v [2T]
inline size_t cclip_smem_bytes(int C, int T) {
    return (size_t)C * sizeof(double) + ((size_t)C * (T + 1) + 2 * (size_t)C + 2 * (size_t)T) * sizeof(float) + 16;
}

// One pass of K23 over the column tiles of each slot (grid (gridX, M), persistent like K19).  The first pass starts from
// v⁰ = h; later passes form v from the clip factors of the previous finish step; the last pass stores θ + v into θ_m and
// v into h_m.
__global__ void __launch_bounds__(kThreads) cclip_pass_kernel(float* __restrict__ theta, long long t_stride,
                                                             const float* __restrict__ cp, const float* __restrict__ n, int C,
                                                             int M, long long P, int T, bool first, bool last,
                                                             const unsigned char* __restrict__ dmask, RobustOpt so,
                                                             CclipState cs) {
    extern __shared__ __align__(16) float sm[];
    double* dacc = reinterpret_cast<double*>(sm);             // [C] this CTA's partial distances
    float* tile = reinterpret_cast<float*>(dacc + C);         // [nrows][T + 1]
    int* rows = reinterpret_cast<int*>(tile + (size_t)C * (T + 1));
    float* sf = reinterpret_cast<float*>(rows + C);            // [C] clip factors
    float* thv = sf + C;                                       // [T] the tile's θ
    float* res = thv + T;                                      // [T] the tile's v
    __shared__ int cnt_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int m = blockIdx.y;
    const int cnt = compact_participants(n, C, M, m, rows, &cnt_s);
    if (cnt == 0) return;
    const bool nan = !first && cs.nan[m] != 0;
    if (nan && !last) return;   // nothing left to iterate: the last pass writes NaN
    float bc1, bc2;
    server_bias_corrections(so, m, &bc1, &bc2);
    float* out = theta + (size_t)m * t_stride;
    float* hm = cs.h + (size_t)m * P;
    const long long ntiles = (P + T - 1) / T;
    if (nan) {   // last pass of a NaN slot: no rows to read
        const float q = __int_as_float(0x7FC00000);
        for (long long tile_i = blockIdx.x; tile_i < ntiles; tile_i += gridDim.x)
            for (int j = tid; j < T && tile_i * T + j < P; j += kThreads) {
                const long long e = tile_i * T + j;
                store_entry(out, e, q, so, (size_t)m, P, bc1, bc2);
                hm[e] = q;
            }
        return;
    }
    for (int i = tid; i < cnt; i += kThreads) {
        dacc[i] = 0.0;
        if (!first) sf[i] = cs.s[(size_t)m * C + i];
    }
    const float nf = (float)cnt;
    const size_t rstride = (size_t)M * P;
    const int pitch = T + 1;
    const bool vec = ((P & 3) == 0) && ((((uintptr_t)cp) & 15) == 0);
    __syncthreads();

    for (long long tile_i = blockIdx.x; tile_i < ntiles; tile_i += gridDim.x) {
        const long long col0 = tile_i * T;
        const int tw = (int)min((long long)T, P - col0);
        stage_tile(tile, cp, rows, cnt, rstride, m, P, col0, T, tw, vec);
        __syncthreads();
        // ---- v of the tile: h, or v + fl32(fl32(Σ_i fl32(s_i·u_i)) / n) in client order over the rows with s_i != 0
        for (int j = tid; j < tw; j += kThreads) {
            const long long e = col0 + j;
            const float th = out[e];
            float v = hm[e];
            if (!first) {
                float acc = 0.f;
                for (int i = 0; i < cnt; ++i) {
                    const float si = sf[i];
                    if (si != 0.f) acc = __fadd_rn(acc, __fmul_rn(si, __fsub_rn(__fsub_rn(tile[(size_t)i * pitch + j], th), v)));
                }
                v = __fadd_rn(v, __fdiv_rn(acc, nf));
            }
            thv[j] = th;
            res[j] = v;
            if (last) {
                store_entry(out, e, __fadd_rn(th, v), so, (size_t)m, P, bc1, bc2);
                hm[e] = v;
            } else if (!first) {
                hm[e] = v;   // the next pass starts from this iterate
            }
        }
        if (!last) {
            __syncthreads();
            // ---- squared distances of u = fl32(fl32(x − θ) − v) over the tile's trainable columns, warp per row
            for (int i = warp; i < cnt; i += kWarps) {
                double s = 0.0;
                for (int j = lane; j < tw; j += 32)
                    if (!dmask || dmask[col0 + j]) {
                        const double d = (double)__fsub_rn(__fsub_rn(tile[(size_t)i * pitch + j], thv[j]), res[j]);
                        s = fma(d, d, s);
                    }
                s = warp_sum(s);
                if (lane == 0) dacc[i] += s;
            }
        }
        __syncthreads();   // the next tile overwrites tile / thv / res
    }
    if (!last)
        for (int i = tid; i < cnt; i += kThreads) cs.part[((size_t)m * gridDim.x + blockIdx.x) * C + i] = dacc[i];
}

// After a distance pass: r_i² = the CTA partials summed in CTA order, s_i = fl32(min(1, τ / r_i)) (float64; r = 0 gives 1,
// r = +∞ gives 0); a NaN distance marks the slot NaN.  One CTA per slot.
__global__ void __launch_bounds__(kThreads) cclip_finish_kernel(const float* __restrict__ n, int C, int M, int gx, double tau,
                                                               CclipState cs) {
    extern __shared__ __align__(16) float sm[];
    int* rows = reinterpret_cast<int*>(sm);
    __shared__ int cnt_s, nan_s;
    const int m = blockIdx.x;
    if (threadIdx.x == 0) nan_s = 0;
    const int cnt = compact_participants(n, C, M, m, rows, &cnt_s);
    if (cnt == 0 || cs.nan[m] != 0) return;
    for (int i = threadIdx.x; i < cnt; i += kThreads) {
        double r2 = 0.0;
        for (int b = 0; b < gx; ++b) r2 += cs.part[((size_t)m * gx + b) * C + i];
        if (isnan(r2)) nan_s = 1;
        cs.s[(size_t)m * C + i] = isnan(r2) ? 0.f : (float)fmin(1.0, tau / sqrt(r2));
    }
    __syncthreads();
    if (threadIdx.x == 0 && nan_s) cs.nan[m] = 1;
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

namespace {
// K21's distance tile: the widest tile of at least 32 columns with the pair accumulators on chip, else the widest tile
// with them in the CTA's row of the partials
struct KrumPlan {
    int T;
    bool acc_on_chip;
};
inline KrumPlan krum_plan(int C) {
    for (int T = 128; T >= 32; T >>= 1)
        if (krum_dist_smem_bytes(C, T, true) <= (size_t)kSmemBudget) return {T, true};
    return {tile_width(C, [](int c, int t) { return (krum_dist_smem_bytes(c, t, false) + 3) / 4; }), false};
}

inline int krum_grid_x(int C, int M, long long P) {
    const KrumPlan kp = krum_plan(C);
    const long long cap = max(1LL, kKrumPartBudget / ((long long)M * krum_npairs(C)));
    return (int)min((long long)persistent_grid_x((P + kp.T - 1) / kp.T, M), cap);
}
}  // namespace

long long krum_scratch_bytes(int C, int M, long long P) {
    if (C <= 0 || M <= 0 || P <= 0) return 0;
    return (long long)M * krum_grid_x(C, M, P) * krum_npairs(C) * 8 + (long long)M * C * 4 + (long long)M * 4;
}

int krum_aggregate_launch(float* theta, long long t_stride, const float* cp, const float* n, int C, int M, long long P, int f,
                          int mkeep, const unsigned char* dmask, int opt_kind, float lr, float momentum, float b1, float b2,
                          float eps, float* s0, float* s1, const int* steps, const unsigned char* mask, void* scratch,
                          cudaStream_t stream) {
    if (C <= 0 || M <= 0 || P <= 0) return 0;
    if (M > 65535) return -5;
    const KrumPlan kp = krum_plan(C);
    const size_t dsmem = krum_dist_smem_bytes(C, kp.T, kp.acc_on_chip), ssmem = krum_select_smem_bytes(C);
    if (dsmem > 227 * 1024 || ssmem > 227 * 1024) return -2;
    if (dsmem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(krum_dist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dsmem);
        if (e != cudaSuccess) return -3;
    }
    if (ssmem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(krum_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssmem);
        if (e != cudaSuccess) return -3;
    }
    const int gx = krum_grid_x(C, M, P);
    char* sp = static_cast<char*>(scratch);
    double* part = reinterpret_cast<double*>(sp);         sp += (size_t)M * gx * krum_npairs(C) * 8;
    int* sel = reinterpret_cast<int*>(sp);                sp += (size_t)M * C * 4;
    int* selcnt = reinterpret_cast<int*>(sp);
    krum_dist_kernel<<<dim3((unsigned)gx, (unsigned)M), kThreads, dsmem, stream>>>(cp, n, C, M, P, kp.T, kp.acc_on_chip, dmask,
                                                                                    part);
    krum_select_kernel<<<M, kThreads, ssmem, stream>>>(n, C, M, gx, f, mkeep, part, sel, selcnt);
    const RobustOpt so{opt_kind, lr, momentum, b1, b2, eps, s0, s1, steps, mask};
    const dim3 sgrid((unsigned)persistent_grid_x((P + kThreads - 1) / kThreads, M), (unsigned)M);
    krum_store_kernel<<<sgrid, kThreads, (size_t)C * sizeof(int), stream>>>(theta, t_stride, cp, C, M, P, sel, selcnt, so);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

namespace {
inline int cclip_tile(int C) {
    return tile_width(C, [](int c, int t) { return (cclip_smem_bytes(c, t) + 3) / 4; });
}
}  // namespace

long long cclip_scratch_bytes(int C, int M, long long P) {
    if (C <= 0 || M <= 0 || P <= 0) return 0;
    const int T = cclip_tile(C);
    const long long gx = persistent_grid_x((P + T - 1) / T, M);
    return (long long)M * gx * C * 8 + (long long)M * C * 4 + (long long)M * 4;
}

int cclip_aggregate_launch(float* theta, long long t_stride, const float* cp, const float* n, float* center, int C, int M,
                           long long P, int iters, double tau, const unsigned char* dmask, int opt_kind, float lr, float momentum,
                           float b1, float b2, float eps, float* s0, float* s1, const int* steps, const unsigned char* mask,
                           void* scratch, cudaStream_t stream) {
    if (C <= 0 || M <= 0 || P <= 0) return 0;
    if (M > 65535) return -5;
    const int T = cclip_tile(C);
    const size_t smem = cclip_smem_bytes(C, T);
    if (smem > 227 * 1024) return -2;
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(cclip_pass_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return -3;
    }
    const size_t fsmem = (size_t)C * sizeof(int);
    if (fsmem > 227 * 1024) return -2;
    if (fsmem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(cclip_finish_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem);
        if (e != cudaSuccess) return -3;
    }
    const int gx = persistent_grid_x((P + T - 1) / T, M);
    char* sp = static_cast<char*>(scratch);
    CclipState cs;
    cs.h = center;
    cs.part = reinterpret_cast<double*>(sp);              sp += (size_t)M * gx * C * 8;
    cs.s = reinterpret_cast<float*>(sp);                  sp += (size_t)M * C * 4;
    cs.nan = reinterpret_cast<int*>(sp);
    if (cudaMemsetAsync(cs.nan, 0, (size_t)M * sizeof(int), stream) != cudaSuccess) return -4;
    const RobustOpt none{0, 0.f, 0.f, b1, b2, eps, nullptr, nullptr, nullptr, nullptr};
    const RobustOpt so{opt_kind, lr, momentum, b1, b2, eps, s0, s1, steps, mask};
    const dim3 grid((unsigned)gx, (unsigned)M);
    for (int t = 1; t <= iters + 1; ++t) {
        const bool last = t == iters + 1;
        cclip_pass_kernel<<<grid, kThreads, smem, stream>>>(theta, t_stride, cp, n, C, M, P, T, t == 1, last, dmask,
                                                            last ? so : none, cs);
        if (!last) cclip_finish_kernel<<<M, kThreads, fsmem, stream>>>(n, C, M, gx, tau, cs);
        if (cudaGetLastError() != cudaSuccess) return -4;
    }
    return 0;
}

}  // namespace fdb
