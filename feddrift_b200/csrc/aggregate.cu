// Arena-streaming kernels: K1 (per-cluster weighted FedAvg reduce+apply), K5 merge, K8 Ada statistics,
// K10 robust clipping, K11 FedOpt server step (fused into the K1 epilogue), K12 gossip mixing.
//
// All are HBM-bandwidth bound: every client row is read exactly once with 128-bit loads, 8 independent
// rows in flight per thread (MLP ≥ 8 hides the ~600-cycle DRAM latency), weights are staged in shared
// memory once per CTA, the result row is written once.  Grids are persistent (132 SMs × resident CTAs).
//
// reference loops replaced: FedAvgEnsAggregatorSoftCluster.py:174-185 (python `for k: for i:` over CPU
// state_dicts), FedAVGAggregator.py:72-85, robust_aggregation.py:38-55, fedopt_trainer.py (pseudo-gradient),
// client_dsgd.py:88-102.
#include "common.cuh"
#include "kernels.h"

namespace fdb {

static inline int persistent_grid(long long work_items, int threads) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    long long need = (work_items + threads - 1) / threads;
    long long cap = (long long)sms * 8;
    return (int)max(1LL, min(need, cap));
}

// Dynamic shared memory for an n-float weight table, padded by one 16-byte vector: the compiler unrolls the weight loops
// with LDS.64/96/128 whose tail lanes may read (never use) up to 3 floats past the table — compute-sanitizer memcheck
// flags that as an out-of-bounds shared read when the allocation is exactly n floats.
static inline size_t smem_floats(int n) { return ((size_t)n + 4) * sizeof(float); }

// ------------------------------------------------------------------------------------------------ K1
// theta[m, :] = Σ_c (n[c,m]/tot[m]) · cp[c, m, :]   for every m with tot[m] > 0.
// server_opt != 0 fuses the FedOpt step: g = theta_old - avg, then sgd(+momentum)/adam/adagrad/yogi on theta.
// steps != nullptr: per-slot step counts [M] (steps already applied; the kernel only reads them, the launcher's caller
// advances the slots that aggregated), Adam's bias corrections then use t = steps[m] + 1 instead of the launch-wide bc1 / bc2.
// mask != nullptr: [P] entries with mask[i] == 0 (BatchNorm statistics) take the plain average and keep their state.
struct ServerOpt {
    int kind;  // 0 none (plain overwrite), 1 sgd, 2 adam, 3 adagrad, 4 yogi
    float lr, momentum, b1, b2, eps, bc1, bc2;
    float *s0, *s1;  // optimizer state rows [M, P] (momentum / m , v)
    const int* steps;
    const unsigned char* mask;
};

__global__ void __launch_bounds__(256) cluster_aggregate_kernel(float* __restrict__ theta, int theta_stride,
                                                                const float* __restrict__ cp, const float* __restrict__ n,
                                                                int C, int M, int P, float* __restrict__ tot_out, ServerOpt so) {
    extern __shared__ float wsm[];  // [C] normalised weights of the current model
    __shared__ float red[32];
    const int P4 = P >> 2;
    for (int m = blockIdx.y; m < M; m += gridDim.y) {
        float part = 0.f;
        for (int c = threadIdx.x; c < C; c += blockDim.x) part += n[c * M + m];
        const float tot = block_sum(part, red);
        if (blockIdx.x == 0 && threadIdx.x == 0 && tot_out) tot_out[m] = tot;
        if (!(tot > 0.f)) { __syncthreads(); continue; }
        for (int c = threadIdx.x; c < C; c += blockDim.x) wsm[c] = n[c * M + m] / tot;
        __syncthreads();
        float* out = theta + (size_t)m * theta_stride;
        float bc1 = so.bc1, bc2 = so.bc2;
        if (so.kind != 0 && so.steps) {
            const float ts = (float)(so.steps[m] + 1);
            bc1 = 1.f - powf(so.b1, ts); bc2 = 1.f - powf(so.b2, ts);
        }
        const size_t cstride = (size_t)M * P;
        const float* base = cp + (size_t)m * P;
        const bool vec_ok = ((P & 3) == 0) && ((((uintptr_t)base) & 15) == 0) && ((((uintptr_t)out) & 15) == 0) && ((cstride & 3) == 0);
        if (vec_ok) {
            for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P4; i += gridDim.x * blockDim.x) {
                float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
                int c = 0;
                for (; c + 8 <= C; c += 8) {
                    float4 v[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) v[u] = __ldcs(reinterpret_cast<const float4*>(base + (size_t)(c + u) * cstride) + i);
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        const float w = wsm[c + u];
                        acc.x = fmaf(v[u].x, w, acc.x); acc.y = fmaf(v[u].y, w, acc.y);
                        acc.z = fmaf(v[u].z, w, acc.z); acc.w = fmaf(v[u].w, w, acc.w);
                    }
                }
                for (; c < C; ++c) {
                    const float4 v = __ldcs(reinterpret_cast<const float4*>(base + (size_t)c * cstride) + i);
                    const float w = wsm[c];
                    acc.x = fmaf(v.x, w, acc.x); acc.y = fmaf(v.y, w, acc.y); acc.z = fmaf(v.z, w, acc.z); acc.w = fmaf(v.w, w, acc.w);
                }
                float r[4] = {acc.x, acc.y, acc.z, acc.w};
                if (so.kind != 0) {
                    const float4 old = reinterpret_cast<const float4*>(out)[i];
                    const float o4[4] = {old.x, old.y, old.z, old.w};
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const size_t i1 = (size_t)i * 4 + u;
                        if (so.mask && !so.mask[i1]) continue;
                        r[u] = server_opt_update(so.kind, o4[u], r[u], so.s0, so.s1, (size_t)m * P + i1, so.lr, so.momentum, so.b1,
                                                 so.b2, so.eps, bc1, bc2);
                    }
                }
                reinterpret_cast<float4*>(out)[i] = make_float4(r[0], r[1], r[2], r[3]);
            }
        } else {  // unaligned / tiny rows: scalar path
            for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
                float acc = 0.f;
                for (int c = 0; c < C; ++c) acc = fmaf(base[(size_t)c * cstride + i], wsm[c], acc);
                if (so.kind == 0 || (so.mask && !so.mask[i])) out[i] = acc;
                else out[i] = server_opt_update(so.kind, out[i], acc, so.s0, so.s1, (size_t)m * P + i, so.lr, so.momentum, so.b1, so.b2,
                                                so.eps, bc1, bc2);
            }
        }
        __syncthreads();
    }
}

int cluster_aggregate_launch(float* theta, int theta_stride, const float* cp, const float* n, int C, int M, int P, float* tot_out,
                             int opt_kind, float lr, float momentum, float b1, float b2, float eps, int step, float* s0, float* s1,
                             const int* steps, const unsigned char* mask, cudaStream_t stream) {
    ServerOpt so{};
    so.kind = opt_kind; so.lr = lr; so.momentum = momentum; so.b1 = b1; so.b2 = b2; so.eps = eps;
    so.bc1 = 1.f - powf(b1, (float)max(step, 1)); so.bc2 = 1.f - powf(b2, (float)max(step, 1));
    so.s0 = s0; so.s1 = s1; so.steps = steps; so.mask = mask;
    const int threads = 256;
    const int gx = persistent_grid((P + 3) / 4, threads);
    dim3 grid(max(1, gx / max(1, min(M, 8))), min(M, 65535));
    if (M * (long long)gx <= 132 * 8) grid.x = gx;
    cluster_aggregate_kernel<<<grid, threads, smem_floats(C), stream>>>(theta, theta_stride, cp, n, C, M, P, tot_out, so);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

// ------------------------------------------------------------------------------------------------ plain weighted average
__global__ void __launch_bounds__(256) weighted_average_kernel(const float* __restrict__ rows, const float* __restrict__ w, int n,
                                                               long long P, float* __restrict__ out) {
    extern __shared__ float wsm[];
    __shared__ float red[32];
    float part = 0.f;
    for (int c = threadIdx.x; c < n; c += blockDim.x) part += w[c];
    const float tot = block_sum(part, red);
    for (int c = threadIdx.x; c < n; c += blockDim.x) wsm[c] = w[c] / tot;
    __syncthreads();
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x) {
        float acc = 0.f;
        int c = 0;
        for (; c + 8 <= n; c += 8) {
            float v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) v[u] = __ldcs(rows + (size_t)(c + u) * P + i);
#pragma unroll
            for (int u = 0; u < 8; ++u) acc = fmaf(v[u], wsm[c + u], acc);
        }
        for (; c < n; ++c) acc = fmaf(__ldcs(rows + (size_t)c * P + i), wsm[c], acc);
        out[i] = acc;
    }
}

int weighted_average_launch(const float* rows, const float* w, int n, long long P, float* out, cudaStream_t stream) {
    const int threads = 256;
    weighted_average_kernel<<<persistent_grid(P, threads), threads, smem_floats(n), stream>>>(rows, w, n, P, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

// ------------------------------------------------------------------------------------------------ K5 merge / K8 / K12
__global__ void axpby_rows_kernel(float* __restrict__ a, const float* __restrict__ b, float wa, float wb, long long P) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x)
        a[i] = a[i] * wa + b[i] * wb;
}
int merge_axpby_launch(float* base_row, const float* second_row, float w1, float w2, long long P, cudaStream_t stream) {
    axpby_rows_kernel<<<persistent_grid(P, 256), 256, 0, stream>>>(base_row, second_row, w1, w2, P);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

__global__ void __launch_bounds__(256) sq_diff_sum_kernel(const float* __restrict__ a, const float* __restrict__ b, long long P,
                                                          double* __restrict__ out) {
    __shared__ double red[32];
    double acc = 0.0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x) {
        const float d = a[i] - b[i];
        acc += (double)d * (double)d;
    }
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) atomicAdd(out, acc);
}
int sq_diff_sum_launch(const float* a, const float* b, long long P, double* out, cudaStream_t stream) {
    cudaMemsetAsync(out, 0, sizeof(double), stream);
    sq_diff_sum_kernel<<<persistent_grid(P, 256), 256, 0, stream>>>(a, b, P, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

// x'_i = Σ_j Wmix[i,j] · x_j   (neighbour sets are tiny: each output row reads only rows with W_ij != 0)
__global__ void __launch_bounds__(256) gossip_mix_kernel(const float* __restrict__ X, const float* __restrict__ Wm, int n, long long P,
                                                         float* __restrict__ out) {
    extern __shared__ float wrow[];  // [n]
    const int i = blockIdx.y;
    for (int j = threadIdx.x; j < n; j += blockDim.x) wrow[j] = Wm[(size_t)i * n + j];
    __syncthreads();
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < P; e += (long long)gridDim.x * blockDim.x) {
        float acc = 0.f;
        for (int j = 0; j < n; ++j) {
            const float w = wrow[j];
            if (w != 0.f) acc = fmaf(w, X[(size_t)j * P + e], acc);
        }
        out[(size_t)i * P + e] = acc;
    }
}
int gossip_mix_launch(const float* X, const float* Wm, int n, long long P, float* out, cudaStream_t stream) {
    dim3 grid(max(1, persistent_grid(P, 256) / max(1, min(n, 16))), n);
    gossip_mix_kernel<<<grid, 256, smem_floats(n), stream>>>(X, Wm, n, P, out);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

// ------------------------------------------------------------------------------------------------ K10
// rows[r] <- g_r + (rows[r]-g_r) / max(1, ||mask·(rows[r]-g_r)|| / bound); one CTA-group per row, two passes (norm, apply);
// the second pass re-reads the row from L2 (a 46.8 MB ResNet-18 row fits the 126 MB L2).  Row r's anchor is
// g_r = g + (r % M)·g_stride (the slot's model for a [C, M, P] upload arena; M = 1, g_stride = 0: one shared anchor), and
// rows whose weight n[r] is 0 are left alone (n == nullptr: every row is clipped).
__global__ void __launch_bounds__(256) row_diff_norm_kernel(const float* __restrict__ rows, const float* __restrict__ g, long long g_stride,
                                                            int M, const float* __restrict__ n, const unsigned char* __restrict__ mask,
                                                            long long P, float* __restrict__ nrm2) {
    __shared__ float red[32];
    const int r = blockIdx.y;
    if (n && n[r] == 0.f) return;
    const float* gr = g + (size_t)(r % M) * g_stride;
    float acc = 0.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x) {
        if (mask && !mask[i]) continue;
        const float d = rows[(size_t)r * P + i] - gr[i];
        acc = fmaf(d, d, acc);
    }
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) atomicAdd(nrm2 + r, acc);
}
__global__ void __launch_bounds__(256) row_clip_apply_kernel(float* __restrict__ rows, const float* __restrict__ g_base, long long g_stride,
                                                             int M, const float* __restrict__ n, const unsigned char* __restrict__ mask,
                                                             long long P, const float* __restrict__ nrm2, float bound,
                                                             float* __restrict__ nrm_out, float stddev, uint32_t seed) {
    const int r = blockIdx.y;
    if (n && n[r] == 0.f) return;
    const float* g = g_base + (size_t)(r % M) * g_stride;
    const float nrm = sqrtf(nrm2[r]);
    if (blockIdx.x == 0 && threadIdx.x == 0 && nrm_out) nrm_out[r] = nrm;
    const float scale = 1.f / fmaxf(1.f, nrm / bound);
    if (scale == 1.f && stddev == 0.f) return;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x) {
        if (mask && !mask[i]) continue;
        const float gi = g[i];
        float v = gi + (rows[(size_t)r * P + i] - gi) * scale;
        if (stddev != 0.f) v = fmaf(stddev, gauss_hash(seed, (uint32_t)r, (unsigned long long)i), v);   // weak-DP noise, same pass
        rows[(size_t)r * P + i] = v;
    }
}
int robust_clip_launch(float* rows, const float* g, long long g_stride, int M, const float* n, const unsigned char* mask, int R,
                       long long P, float bound, float* scratch_nrm2, float* nrm_out, float stddev, unsigned seed, cudaStream_t stream) {
    cudaMemsetAsync(scratch_nrm2, 0, R * sizeof(float), stream);
    dim3 grid(max(1, persistent_grid(P, 256) / max(1, min(R, 16))), R);
    row_diff_norm_kernel<<<grid, 256, 0, stream>>>(rows, g, g_stride, M, n, mask, P, scratch_nrm2);
    row_clip_apply_kernel<<<grid, 256, 0, stream>>>(rows, g, g_stride, M, n, mask, P, scratch_nrm2, bound, nrm_out, stddev, seed);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

}  // namespace fdb
