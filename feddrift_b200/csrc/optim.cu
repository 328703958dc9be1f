// Fused arena optimizers for the big-model client path: ONE launch updates every (client, model) row of the
// ClientArena (reference: torch.optim.Adam(amsgrad=True, weight_decay=wd) per client per model —
// FedAvgEnsTrainer.py:25-33 — ~10 eager launches per parameter tensor per step).
#include "common.cuh"
#include "kernels.h"

namespace fdb {

// FedProx: g + mu·(w − a) on masked entries (the gradient of mu/2‖mask⊙(w − a)‖²), g elsewhere
__device__ __forceinline__ float prox_grad(const ProxAnchor& px, const float* arow, long long e, float w, float g) {
    return (px.mask == nullptr || px.mask[e]) ? fmaf(px.mu, w - arow[e], g) : g;
}

// FedProx pre-pass of the Adam rows: g ← g + mu·mask⊙(p − anchor row) in place, so that the Adam kernel below runs the same
// code (and rounding) with and without the proximal term
__global__ void __launch_bounds__(256) prox_grad_rows_kernel(float* __restrict__ g, const float* __restrict__ p,
                                                             const unsigned char* __restrict__ row_mask, long long P, const ProxAnchor px) {
    const int r = blockIdx.y;
    if (row_mask && !row_mask[r]) return;
    const float* arow = px.anchor + (size_t)px.rows[r] * px.astride;
    const size_t base = (size_t)r * P;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x)
        g[base + i] = prox_grad(px, arow, i, p[base + i], g[base + i]);
}

__global__ void __launch_bounds__(256) adam_amsgrad_rows_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                                float* __restrict__ v, float* __restrict__ vmax, const int* __restrict__ steps,
                                                                const unsigned char* __restrict__ row_mask, long long P, float lr, float wd,
                                                                float b1, float b2, float eps) {
    const int r = blockIdx.y;
    if (row_mask && !row_mask[r]) return;
    const int step = steps[r] + 1;
    const double bc1 = 1.0 - pow((double)b1, (double)step);
    const float bc2s = (float)sqrt(1.0 - pow((double)b2, (double)step));
    const float step_size = (float)((double)lr / bc1);
    const size_t base = (size_t)r * P;
    const bool vec = ((P & 3) == 0);
    if (vec) {
        const long long P4 = P >> 2;
        float4* p4 = reinterpret_cast<float4*>(p + base);
        const float4* g4 = reinterpret_cast<const float4*>(g + base);
        float4* m4 = reinterpret_cast<float4*>(m + base);
        float4* v4 = reinterpret_cast<float4*>(v + base);
        float4* x4 = reinterpret_cast<float4*>(vmax + base);
        for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < P4; i += (long long)gridDim.x * blockDim.x) {
            float4 pp = p4[i], gg = __ldcs(g4 + i), mm = m4[i], vv = v4[i], xx = x4[i];
            float* pa = &pp.x; float* ga = &gg.x; float* ma = &mm.x; float* va = &vv.x; float* xa = &xx.x;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float gr = fmaf(wd, pa[u], ga[u]);
                ma[u] = fmaf(gr - ma[u], 1.f - b1, ma[u]);
                va[u] = fmaf((1.f - b2) * gr, gr, va[u] * b2);
                xa[u] = fmaxf(xa[u], va[u]);
                pa[u] -= step_size * (ma[u] / (sqrtf(xa[u]) / bc2s + eps));
            }
            p4[i] = pp; m4[i] = mm; v4[i] = vv; x4[i] = xx;
        }
    } else {
        for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x) {
            const float w = p[base + i];
            const float gr = fmaf(wd, w, g[base + i]);
            const float mm = fmaf(gr - m[base + i], 1.f - b1, m[base + i]);
            const float vv = fmaf((1.f - b2) * gr, gr, v[base + i] * b2);
            const float xx = fmaxf(vmax[base + i], vv);
            m[base + i] = mm; v[base + i] = vv; vmax[base + i] = xx;
            p[base + i] = w - step_size * (mm / (sqrtf(xx) / bc2s + eps));
        }
    }
}
__global__ void bump_steps_kernel(int* steps, const unsigned char* row_mask, int R) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < R && (!row_mask || row_mask[r])) steps[r] += 1;
}

int adam_amsgrad_rows_launch(float* p, float* g, float* m, float* v, float* vmax, int* steps, const unsigned char* row_mask, int R,
                             long long P, float lr, float wd, float b1, float b2, float eps, const ProxAnchor& prox, cudaStream_t stream) {
    int sms = 132;
    long long per_row = ((P + 3) / 4 + 255) / 256;
    dim3 grid((unsigned)max(1LL, min(per_row, (long long)max(1, sms * 8 / max(R, 1)))), R);
    if (prox.anchor) prox_grad_rows_kernel<<<grid, 256, 0, stream>>>(g, p, row_mask, P, prox);
    adam_amsgrad_rows_kernel<<<grid, 256, 0, stream>>>(p, g, m, v, vmax, steps, row_mask, P, lr, wd, b1, b2, eps);
    bump_steps_kernel<<<(R + 127) / 128, 128, 0, stream>>>(steps, row_mask, R);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

__global__ void __launch_bounds__(256) sgd_rows_kernel(float* __restrict__ p, const float* __restrict__ g, long long n, float lr, float wd) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float w = p[i];
        p[i] = w - lr * fmaf(wd, w, __ldcs(g + i));
    }
}
int sgd_rows_launch(float* p, const float* g, long long n, float lr, float wd, cudaStream_t stream) {
    const long long blocks = max(1LL, min((n + 255) / 256, 132LL * 8));
    sgd_rows_kernel<<<(unsigned)blocks, 256, 0, stream>>>(p, g, n, lr, wd);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

// row-structured SGD: skips rows with row_mask[r] == 0 and, with kProx, adds the FedProx term; the update is written as in
// sgd_rows_kernel, so both compile to the same rounding
template <bool kProx>
__global__ void __launch_bounds__(256) sgd_rows_masked_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                              const unsigned char* __restrict__ row_mask, long long P, float lr, float wd,
                                                              const ProxAnchor px) {
    const int r = blockIdx.y;
    if (row_mask && !row_mask[r]) return;
    const float* arow = kProx ? px.anchor + (size_t)px.rows[r] * px.astride : nullptr;
    const size_t base = (size_t)r * P;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < P; i += (long long)gridDim.x * blockDim.x) {
        const float w = p[base + i];
        float gi = __ldcs(g + base + i);
        if constexpr (kProx) gi = prox_grad(px, arow, i, w, gi);
        p[base + i] = w - lr * fmaf(wd, w, gi);
    }
}
int sgd_rows_masked_launch(float* p, const float* g, const unsigned char* row_mask, int R, long long P, float lr, float wd,
                           const ProxAnchor& prox, cudaStream_t stream) {
    const long long per_row = (P + 255) / 256;
    dim3 grid((unsigned)max(1LL, min(per_row, (long long)max(1, 132 * 8 / max(R, 1)))), R);
    if (prox.anchor)
        sgd_rows_masked_kernel<true><<<grid, 256, 0, stream>>>(p, g, row_mask, P, lr, wd, prox);
    else
        sgd_rows_masked_kernel<false><<<grid, 256, 0, stream>>>(p, g, row_mask, P, lr, wd, prox);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

}  // namespace fdb
