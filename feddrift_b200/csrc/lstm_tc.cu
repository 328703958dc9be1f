// lstm_tc — persistent, cluster-resident 2-layer LSTM (hidden 256) forward + BPTT for RNN_OriginalFedAvg
// (reference: fedml_api/model/nlp/rnn.py:18-33 — Embedding(90,8) → 2×LSTM(256, batch_first) → Linear on the last step;
// the reference runs it through cuDNN's per-timestep kernels: ~10 launches per timestep per layer per direction).
//
// ONE launch runs the whole sequence for MANY (client, model) pairs: grid = npairs × 8 CTAs, one thread-block CLUSTER of 8
// CTAs per pair (and per 16-row batch chunk).  CTA j of a cluster owns hidden units [32j, 32j+32) of BOTH layers, i.e. 128
// gate rows (i, f, g, o × 32 units) per layer.
//
// Forward (lstm2_fwd_kernel):
//   * every timestep is one tensor-core GEMM per layer, run "swapped" so that the 128 gate rows are the M side even at batch 16:
//     gatesᵀ = W_slice · [h_{t-1} | x_t]ᵀ with warp-level mma.sync m16n8k16 (bf16 operands, fp32 accumulation).  Warp w of a
//     layer group owns gate w of the CTA's 32 units (two m16 tiles × the 16 batch columns); its weight fragments are read
//     from the fp32 parameter rows (L2-resident: the CTA's slice is 400 KB, more than shared memory can hold next to the
//     exchange buffers) and rounded to bf16, the activations come from shared memory in the K-major core-matrix layout;
//   * layers are WAVEFRONT-pipelined: phase p computes layer 1 at time p and layer 2 at time p-1 (both only need h1_{p-1}),
//     so there is one cluster exchange per timestep instead of two;
//   * the epilogue (bias → σ/tanh → cell update, c kept in registers) produces the CTA's 32 new hidden units for 16 batch rows,
//     stages them as bf16 in the operand layout and BROADCASTS the 1-KB slice into all 8 CTAs' next-step operand buffers with
//     cp.async.bulk shared::cta → shared::cluster (DSMEM); arrival is tracked by an mbarrier transaction count in each
//     destination — no cluster barrier in the time loop;
//   * gate activations, cell states and hidden states are written to a history workspace for BPTT.
//
// Backward (lstm2_bwd_kernel): same ownership, reversed wavefront.  Per phase: sum the 8 partial dh blocks that arrived in the
// inbox (fixed order → deterministic), elementwise LSTM backward for the own units (dc carried in registers), dG (bf16) →
// smem operand + global history, partial dhᵀ[256 × 16] = W_sliceᵀ · dGᵀ on mma.sync (W_hh2ᵀ, W_ih2ᵀ, W_hh1ᵀ fragments from
// the fp32 rows) and a DSMEM bulk REDUCE-SCATTER of the 2-KB blocks to the owners of those hidden units.  Weight gradients are
// GEMMs over the saved histories (dW = dGᵀ · H with the MN-major wgmma GEMM of gemm_tc.cu), outside this file.
//
// All waits are bounded (trap after 4 s).  bf16 operands, fp32 accumulation, fp32 cell state / gates / gradients.
#include <cooperative_groups.h>

#include "kernels.h"
#include "hopper.cuh"

namespace cg = cooperative_groups;

namespace fdb {

namespace lstm {
constexpr int H = 256, CL = 8, U = 32, NB = 16, KX = 16;
constexpr int kFwdThreads = 288;   // 2 layer groups of 4 warps + 1 warp that arms the inbound-exchange barriers
}  // namespace lstm

// element offset of (batch row b, reduction index k) in a no-swizzle K-major operand tile of 16 rows
FDB_DEVICE int op_off(int b, int k) { return (((k >> 3) * (lstm::NB / 8) + (b >> 3)) << 6) + ((b & 7) << 3) + (k & 7); }

FDB_DEVICE uint32_t mapa_u32(uint32_t smem_addr, uint32_t cta_rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(cta_rank));
    return r;
}
// DSMEM bulk copy: this CTA's shared memory → a cluster peer's shared memory; completion = tx bytes on the PEER's mbarrier
FDB_DEVICE void bulk_copy_s2c(uint32_t dst_cluster_addr, uint32_t src_cta_addr, uint32_t bytes, uint32_t mbar_cluster_addr) {
    asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst_cluster_addr), "r"(src_cta_addr), "r"(bytes), "r"(mbar_cluster_addr) : "memory");
}
FDB_DEVICE void mbar_wait_long(uint64_t* bar, uint32_t parity) {
    SpinGuard g;
    while (!mbar_try_wait(bar, parity)) {
        if (g.expired(4000000000LL)) __trap();
    }
}
FDB_DEVICE uint32_t pack_bf16(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);   // .x (low half) = lo
    return *reinterpret_cast<uint32_t*>(&v);
}
// MUFU.TANH: one instruction, |abs err| ≲ 5e-4 — far below the bf16 rounding of the operands these activations feed; the
// forward saves the activations it used, so BPTT differentiates exactly the function that was evaluated
FDB_DEVICE float tanh_fast(float x) { float y; asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
FDB_DEVICE float sigmoid_fast(float x) { return fmaf(0.5f, tanh_fast(0.5f * x), 0.5f); }

// acc[t][n] += W[rows row0 + 16t …][k] · actᵀ over k < 16·ksteps: the warp's 32 weight rows (two m16 tiles, row stride ldw,
// columns ≥ kvalid read as 0) against the 16 batch rows of an op_off-layout operand (two n8 tiles)
FDB_DEVICE void rows_mma(float (&acc)[2][2][4], const float* __restrict__ W, int ldw, int kvalid, int row0, const __nv_bfloat16* act,
                         int ksteps, int l) {
    const int g = l >> 2, c = l & 3;
    const uint32_t* act32 = reinterpret_cast<const uint32_t*>(act);
    // float2 loads need 8-byte aligned rows (even row offset and ldw); otherwise the scalar path below
    const bool vec = kvalid >= 16 * ksteps && (reinterpret_cast<uintptr_t>(W) & 7) == 0 && (ldw & 1) == 0;
#pragma unroll 4
    for (int ks = 0; ks < ksteps; ++ks) {
        const int k = 16 * ks + 2 * c;
        uint32_t b[2][2];
#pragma unroll
        for (int n = 0; n < 2; ++n) { b[n][0] = act32[op_off(8 * n + g, k) >> 1]; b[n][1] = act32[op_off(8 * n + g, k + 8) >> 1]; }
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const float* ra = W + (size_t)(row0 + 16 * t + g) * ldw;
            const float* rb = ra + (size_t)8 * ldw;
            uint32_t a[4];
            if (vec) {
                const float2 x0 = __ldg(reinterpret_cast<const float2*>(ra + k)), x1 = __ldg(reinterpret_cast<const float2*>(rb + k));
                const float2 x2 = __ldg(reinterpret_cast<const float2*>(ra + k + 8)), x3 = __ldg(reinterpret_cast<const float2*>(rb + k + 8));
                a[0] = pack_bf16(x0.x, x0.y); a[1] = pack_bf16(x1.x, x1.y); a[2] = pack_bf16(x2.x, x2.y); a[3] = pack_bf16(x3.x, x3.y);
            } else {
                auto ld = [&](const float* r, int kk) { return kk < kvalid ? __ldg(r + kk) : 0.f; };
                a[0] = pack_bf16(ld(ra, k), ld(ra, k + 1)); a[1] = pack_bf16(ld(rb, k), ld(rb, k + 1));
                a[2] = pack_bf16(ld(ra, k + 8), ld(ra, k + 9)); a[3] = pack_bf16(ld(rb, k + 8), ld(rb, k + 9));
            }
#pragma unroll
            for (int n = 0; n < 2; ++n) mma_bf16_16816(acc[t][n], a, b[n][0], b[n][1]);
        }
    }
}

// ======================================================================================================= forward
// Warp roles (288 threads): warps 0-3 = layer-1 group, warps 4-7 = layer-2 group (warp w computes gate w of the CTA's 32
// units), warp 8 arms the inbound barriers.  Each group runs GEMM → activations → cell update → staging → DSMEM broadcast on
// its own named barrier, so the two layers overlap.  The layer-2 GEMM of phase p reads h1_{p-1} from the buffer the peers
// fill with h1_{p+1}; they can only do so after this CTA has broadcast h1_p, so that broadcast waits for the layer-2 group's
// reads (l2bar).
__global__ void __cluster_dims__(lstm::CL, 1, 1) __launch_bounds__(lstm::kFwdThreads, 1)
lstm2_fwd_kernel(const __grid_constant__ LstmArgs a) {
    using namespace lstm;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    cg::cluster_group cluster = cg::this_cluster();
    const int crank = (int)cluster.block_rank();
    const int pair = blockIdx.x / CL;
    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), l = tid & 31;   // uniform warp index
    const int T = a.T, E = a.E;

    // ---- shared memory carve-up
    __nv_bfloat16* H1s = reinterpret_cast<__nv_bfloat16*>(smem_raw);            // [2][NB*256]
    __nv_bfloat16* H2s = H1s + 2 * NB * H;                                       // [2][NB*256]
    __nv_bfloat16* Xs = H2s + 2 * NB * H;                                        // [2][NB*16]
    __nv_bfloat16* stage = Xs + 2 * NB * KX;                                     // [2 parities][2 layers][NB*32]
    float* act_s = reinterpret_cast<float*>(stage + 2 * 2 * NB * U);             // [2 layers][4 gates][NB][32]
    uint64_t* hbar = reinterpret_cast<uint64_t*>(act_s + 2 * 4 * NB * U);        // [2]
    uint64_t* l2bar = hbar + 2;                                                  // layer-2 group done reading this phase's operands

    const float* prow = a.params + a.row_off[pair];
    const float* w_ih1 = prow + a.off_wih1;
    const float* w_hh1 = prow + a.off_whh1;
    const float* w_ih2 = prow + a.off_wih2;
    const float* w_hh2 = prow + a.off_whh2;
    const float* emb = prow + a.off_emb;
    const int* tok = a.tokens + (size_t)pair * NB * T;

    if (tid == 0) {
        mbar_init(hbar + 0, 1); mbar_init(hbar + 1, 1); mbar_init(l2bar, 4);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // zero the operand buffers (h_{-1} = 0, padded x columns = 0)
    for (int i = tid; i < (2 * NB * H * 2 + 2 * NB * KX) / 2; i += kFwdThreads) reinterpret_cast<uint32_t*>(H1s)[i] = 0u;
    __syncthreads();

    const int grp = warp >> 2;                      // 0: layer-1 group, 1: layer-2 group, 2: barrier warp
    const int w = warp & 3, gt = tid & 127;         // gate index / thread index inside the group
    const int row0 = w * H + crank * U;             // first row of the PyTorch [4H, K] weight matrices owned by this warp
    float bias[2][2] = {{0.f, 0.f}, {0.f, 0.f}};    // units 16t + l/4 + 8hh
    if (grp < 2) {
        const float* bi = prow + (grp == 0 ? a.off_bih1 : a.off_bih2);
        const float* bh = prow + (grp == 0 ? a.off_bhh1 : a.off_bhh2);
#pragma unroll
        for (int t = 0; t < 2; ++t)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int R = row0 + 16 * t + (l >> 2) + 8 * hh;
                bias[t][hh] = __ldg(bi + R) + __ldg(bh + R);
            }
    }
    if (grp == 0) {
        for (int i = gt; i < NB * KX; i += 128) {    // x_0 → Xs[0]
            const int b = i / KX, k = i % KX;
            const float xv = (k < E) ? __ldg(emb + (size_t)tok[b * T + 0] * E + k) : 0.f;
            Xs[op_off(b, k)] = __float2bfloat16(xv);
        }
    }
    fence_proxy_async_smem();
    cluster.sync();            // every CTA's barriers / buffers are initialised before any peer writes into them

    // history layout is LAYER-outermost: [2][npairs][T (+1)][16][...]
    const int NP = (int)gridDim.x / CL;
    const bool keep = a.gates != nullptr;            // training: save gates / cell states for BPTT
    const bool keep_h = a.hhist != nullptr;
    const int unit = crank * U + l;
    const uint32_t bytes_each = NB * U * 2;

    if (grp == 2) {
        // =================================================== barrier warp: arm phase p's inbound barrier (the slices of phase p
        // land in hbar[p&1]) only after its previous phase completed
        for (int p = 0; p <= T; ++p) {
            const bool doL1 = p < T, doL2 = p >= 1;
            if (p < T && elect_one()) mbar_expect_tx(hbar + (p & 1), CL * bytes_each * ((doL1 ? 1u : 0u) + (doL2 ? 1u : 0u)));
            if (p >= 1) mbar_wait_long(hbar + ((p - 1) & 1), ((p - 1) >> 1) & 1);   // h1_{p-1} (and h2_{p-2}) from all 8 CTAs
        }
    } else {
        // =================================================== layer groups (layer = grp)
        const int layer = grp;
        float* gates_l = a.gates + (size_t)(layer * NP + pair) * T * NB * 4 * H;
        float* cst_l = a.cst + (size_t)(layer * NP + pair) * T * NB * H;
        __nv_bfloat16* hh_l = reinterpret_cast<__nv_bfloat16*>(a.hhist) + (size_t)(layer * NP + pair) * (T + 1) * NB * H;
        float* act = act_s + layer * 4 * NB * U;
        float creg[4] = {0.f, 0.f, 0.f, 0.f};
        // layer 1 runs in phases 0 … T-1 (time p), layer 2 in phases 1 … T (time p-1)
        const int p_lo = layer == 0 ? 0 : 1, p_hi = layer == 0 ? T - 1 : T;
        for (int p = p_lo; p <= p_hi; ++p) {
            const int t = p - layer;
            // prefetch next step's token / embedding values early (layer-1 group only): 2 values per thread
            float xv[2] = {0.f, 0.f};
            if (layer == 0 && p + 1 < T) {
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int i = gt + 128 * q, b = i / KX, k = i % KX;
                    if (k < E) xv[q] = __ldg(emb + (size_t)__ldg(tok + b * T + p + 1) * E + k);
                }
            }
            if (p >= 1) mbar_wait_long(hbar + ((p - 1) & 1), ((p - 1) >> 1) & 1);   // h1_{p-1} (and h2_{p-2}) from all 8 CTAs
            // ---- GEMM: this warp's 32 gate rows × 16 batch columns
            {
                float acc[2][2][4];
#pragma unroll
                for (int i = 0; i < 16; ++i) (&acc[0][0][0])[i] = 0.f;
                const __nv_bfloat16* h1prev = H1s + ((p + 1) & 1) * NB * H;     // h1_{p-1}
                if (layer == 0) {
                    rows_mma(acc, w_hh1, H, H, row0, h1prev, H / 16, l);
                    rows_mma(acc, w_ih1, E, E, row0, Xs + (p & 1) * NB * KX, 1, l);
                } else {
                    rows_mma(acc, w_ih2, H, H, row0, h1prev, H / 16, l);
                    rows_mma(acc, w_hh2, H, H, row0, H2s + (p & 1) * NB * H, H / 16, l);   // h2_{p-2}
                    __syncwarp();
                    if (l == 0) mbar_arrive(l2bar);
                }
#pragma unroll
                for (int tt = 0; tt < 2; ++tt)
#pragma unroll
                    for (int n = 0; n < 2; ++n)
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int u = 16 * tt + (l >> 2) + 8 * (e >> 1), b = 8 * n + 2 * (l & 3) + (e & 1);
                            const float x = acc[tt][n][e] + bias[tt][e >> 1];
                            act[(w * NB + b) * U + u] = (w == 2) ? tanh_fast(x) : sigmoid_fast(x);
                        }
            }
            named_bar_sync(1 + layer, 128);
            // ---- cell update for the own 32 units (unit l) × rows b = w + 4 i; stage the bf16 slice in operand layout
            __nv_bfloat16* st = stage + ((p & 1) * 2 + layer) * NB * U;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int b = w + 4 * i;
                const float gi = act[(0 * NB + b) * U + l], gf = act[(1 * NB + b) * U + l];
                const float gg = act[(2 * NB + b) * U + l], go = act[(3 * NB + b) * U + l];
                creg[i] = gf * creg[i] + gi * gg;
                const float h = go * tanh_fast(creg[i]);
                const size_t row = (size_t)t * NB + b;
                if (keep) {
                    float* g = gates_l + row * 4 * H + unit;
                    g[0] = gi; g[H] = gf; g[2 * H] = gg; g[3 * H] = go;
                    cst_l[row * H + unit] = creg[i];
                }
                const __nv_bfloat16 hb = __float2bfloat16(h);
                if (keep_h) hh_l[((size_t)(t + 1) * NB + b) * H + unit] = hb;
                st[op_off(b, l)] = hb;     // k_core = l/8 local to the slice
                if (layer == 1 && t == T - 1) a.hlast[((size_t)pair * NB + b) * H + unit] = h;
            }
            if (layer == 0 && p + 1 < T) {   // x_{p+1} → Xs[(p+1)&1]
                __nv_bfloat16* xd = Xs + ((p + 1) & 1) * NB * KX;
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int i = gt + 128 * q;
                    xd[op_off(i / KX, i % KX)] = __float2bfloat16(xv[q]);
                }
            }
            fence_proxy_async_smem();   // generic-proxy writes (stage) → visible to the async proxy (bulk copy)
            named_bar_sync(1 + layer, 128);
            // ---- all-gather: my 1-KB slice → every CTA's next-step operand buffer (incl. my own); lane d serves CTA d.
            //      (the last phase's h2_{T-1} is only needed as hlast, no exchange)
            if (p < T && gt < CL) {
                if (layer == 0 && p >= 1) mbar_wait_long(l2bar, (p - 1) & 1);   // this CTA's layer-2 GEMM of phase p has read h1_{p-1}
                const uint32_t bar = smem_u32(hbar + (p & 1));
                const uint32_t dst = (layer == 0 ? smem_u32(H1s + (p & 1) * NB * H) : smem_u32(H2s + ((p + 1) & 1) * NB * H)) + crank * bytes_each;
                bulk_copy_s2c(mapa_u32(dst, gt), smem_u32(st), bytes_each, mapa_u32(bar, gt));
            }
        }
    }
    // ---- teardown: nobody may exit while peers still copy into its shared memory
    cluster.sync();
}

// ======================================================================================================= backward
// acc[h][t][n] = Σ_j W[R(j)][k] · dG[b][j] for the warp's hidden rows k = 128h + 32w + 16t + … (transposed slice: K = the CTA's
// own 128 gate rows j, R(j) = (j/32)·H + crank·U + j%32)
FDB_DEVICE void cols_mma(float (&acc)[2][2][2][4], const float* __restrict__ W, int crank, int w, const __nv_bfloat16* dg, int l) {
    using namespace lstm;
    const int g = l >> 2, c = l & 3;
    const uint32_t* dg32 = reinterpret_cast<const uint32_t*>(dg);
#pragma unroll
    for (int i = 0; i < 32; ++i) (&acc[0][0][0][0])[i] = 0.f;
#pragma unroll 2
    for (int ks = 0; ks < 8; ++ks) {
        const int j = 16 * ks + 2 * c;
        uint32_t b[2][2];
#pragma unroll
        for (int n = 0; n < 2; ++n) { b[n][0] = dg32[op_off(8 * n + g, j) >> 1]; b[n][1] = dg32[op_off(8 * n + g, j + 8) >> 1]; }
        // rows R(j), R(j+1), R(j+8), R(j+9) of W (j even: j and j+1 are in the same 32-row gate block)
        const float* r0 = W + (size_t)((j >> 5) * H + crank * U + (j & 31)) * H;
        const float* r8 = W + (size_t)(((j + 8) >> 5) * H + crank * U + ((j + 8) & 31)) * H;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int t = 0; t < 2; ++t) {
                const int k = 128 * h + 32 * w + 16 * t + g;
                uint32_t a[4];
                a[0] = pack_bf16(__ldg(r0 + k), __ldg(r0 + H + k));
                a[1] = pack_bf16(__ldg(r0 + k + 8), __ldg(r0 + H + k + 8));
                a[2] = pack_bf16(__ldg(r8 + k), __ldg(r8 + H + k));
                a[3] = pack_bf16(__ldg(r8 + k + 8), __ldg(r8 + H + k + 8));
#pragma unroll
                for (int n = 0; n < 2; ++n) mma_bf16_16816(acc[h][t][n], a, b[n][0], b[n][1]);
            }
    }
}

// Warp roles (288 threads): warps 0-3 = layer-2 group (time p), warps 4-7 = layer-1 group (time p+1), warp 8 arms the inbox
// barriers.  Per phase each group: prefetch its history rows → wait for the inbox → Σ partial dh → LSTM cell backward → dG
// (bf16) to the smem operand + global history → partial dhᵀ GEMMs → staging → DSMEM bulk reduce-scatter (one lane per copy).
__global__ void __cluster_dims__(lstm::CL, 1, 1) __launch_bounds__(lstm::kFwdThreads, 1)
lstm2_bwd_kernel(const __grid_constant__ LstmArgs a) {
    using namespace lstm;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    cg::cluster_group cluster = cg::this_cluster();
    const int crank = (int)cluster.block_rank();
    const int pair = blockIdx.x / CL;
    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), l = tid & 31;   // uniform warp index
    const int T = a.T;

    // ---- shared memory: inbox [2 bufs][8 src][3 kinds][NB][32] fp32, out staging [2 bufs][3 kinds][8 dst][NB][32] fp32,
    //      dG operands [2 layers][NB × 128] bf16
    constexpr int BLK = NB * U;   // 512 floats = 2 KB
    float* inbox = reinterpret_cast<float*>(smem_raw);                  // 2*8*3*BLK
    float* outst = inbox + 2 * CL * 3 * BLK;                            // 2*3*8*BLK
    __nv_bfloat16* dGs = reinterpret_cast<__nv_bfloat16*>(outst + 2 * 3 * CL * BLK);   // [2][NB*128]: [0] layer 1, [1] layer 2
    uint64_t* ibar = reinterpret_cast<uint64_t*>(dGs + 2 * NB * 128);  // [2] inbox arrival (tx bytes)

    const float* prow = a.params + a.row_off[pair];
    const float* w_hh1 = prow + a.off_whh1;
    const float* w_ih2 = prow + a.off_wih2;
    const float* w_hh2 = prow + a.off_whh2;

    if (tid == 0) {
        for (int i = 0; i < 2; ++i) mbar_init(ibar + i, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int grp = warp >> 2;                 // 0: layer 2, 1: layer 1, 2: barrier warp
    const int w = warp & 3, gt = tid & 127;
    cluster.sync();

    const int unit = crank * U + l;
    const int NP = (int)gridDim.x / CL;

    if (grp == 2) {
        // =================================================== arm each phase's inbox barrier once its previous use completed
        for (int p = T - 1, it = 0; p >= 0; --p, ++it) {
            const bool doL1 = p + 1 <= T - 1;
            if (it >= 2) mbar_wait_long(ibar + (it & 1), ((it - 2) >> 1) & 1);
            if (elect_one()) mbar_expect_tx(ibar + (it & 1), (uint32_t)(CL * (doL1 ? 3 : 2) * BLK * 4));   // this phase's inbound partial blocks
        }
    } else {
        // =================================================== layer groups
        const int layer = 1 - grp;                 // group 0 ↔ layer index 1 (second layer), group 1 ↔ layer index 0
        const float* gates_l = a.gates + (size_t)(layer * NP + pair) * T * NB * 4 * H;
        const float* cst_l = a.cst + (size_t)(layer * NP + pair) * T * NB * H;
        __nv_bfloat16* dG_l = reinterpret_cast<__nv_bfloat16*>(a.dgates) + (size_t)(layer * NP + pair) * T * NB * 4 * H;
        __nv_bfloat16* dg_s = dGs + layer * NB * 128;
        float dcar[4] = {0.f, 0.f, 0.f, 0.f};
        // group 0 (layer 2) runs in phases it = 0 … T-1 at time t = T-1-it; group 1 (layer 1) in phases it = 1 … T at time t = T-it
        const int it_lo = grp, it_hi = T - 1 + grp;
        for (int it = it_lo; it <= it_hi; ++it) {
            const int t = T - 1 - it + grp;
            const int p = T - 1 - it;                                  // the phase's layer-2 time (−1 in the last phase)
            // ---- prefetch this step's history rows (independent of the inbox) before waiting
            float hg[4][4], hc[4], hcp[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int b = w + 4 * i;
                const size_t row = (size_t)t * NB + b;
                const float* g = gates_l + row * 4 * H + unit;
                hg[i][0] = g[0]; hg[i][1] = g[H]; hg[i][2] = g[2 * H]; hg[i][3] = g[3 * H];
                hc[i] = cst_l[row * H + unit];
                hcp[i] = (t > 0) ? cst_l[((size_t)(t - 1) * NB + b) * H + unit] : 0.f;
            }
            const bool have_in = it > 0;
            const int ibuf = (it + 1) & 1;                             // inbox buffer written during phase it-1
            if (have_in) mbar_wait_long(ibar + ibuf, ((it - 1) >> 1) & 1);
            const float* in = inbox + (size_t)ibuf * CL * 3 * BLK;
            const bool prev_had_L1 = have_in && (p + 2 <= T - 1);      // phase it-1 also ran layer 1 (at time p+2)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int b = w + 4 * i;
                float dh = 0.f;
                if (grp == 0) {
                    if (a.dh2_all) dh = a.dh2_all[(((size_t)pair * T + t) * NB + b) * H + unit];
                    else if (t == T - 1) dh = a.dh2_last[((size_t)pair * NB + b) * H + unit];
                    if (have_in) {
#pragma unroll
                        for (int sidx = 0; sidx < CL; ++sidx) dh += in[(sidx * 3 + 0) * BLK + b * U + l];
                    }
                } else {
#pragma unroll
                    for (int sidx = 0; sidx < CL; ++sidx) dh += in[(sidx * 3 + 1) * BLK + b * U + l];
                    if (prev_had_L1) {
#pragma unroll
                        for (int sidx = 0; sidx < CL; ++sidx) dh += in[(sidx * 3 + 2) * BLK + b * U + l];
                    }
                }
                const float gi = hg[i][0], gf = hg[i][1], gg = hg[i][2], go = hg[i][3];
                const float tc = tanh_fast(hc[i]);
                const float dcv = dcar[i] + dh * go * (1.f - tc * tc);
                const float dzi = dcv * gg * gi * (1.f - gi), dzf = dcv * hcp[i] * gf * (1.f - gf);
                const float dzg = dcv * gi * (1.f - gg * gg), dzo = dh * tc * go * (1.f - go);
                dcar[i] = dcv * gf;
                __nv_bfloat16* o = dG_l + ((size_t)t * NB + b) * 4 * H + unit;
                const __nv_bfloat16 bi = __float2bfloat16(dzi), bf = __float2bfloat16(dzf), bg = __float2bfloat16(dzg), bo = __float2bfloat16(dzo);
                o[0] = bi; o[H] = bf; o[2 * H] = bg; o[3 * H] = bo;
                dg_s[op_off(b, 0 * 32 + l)] = bi; dg_s[op_off(b, 1 * 32 + l)] = bf; dg_s[op_off(b, 2 * 32 + l)] = bg; dg_s[op_off(b, 3 * 32 + l)] = bo;
            }
            if (p < 0) break;                                          // layer 1 at time 0: its dh_{-1} has no consumer
            named_bar_sync(1 + grp, 128);                              // the group's dG operand is complete
            // ---- partial dhᵀ of this warp's 64 hidden rows per kind → staging blocks [b][unit-in-owner] (owner 4h + w)
            float* ob = outst + (size_t)(it & 1) * 3 * CL * BLK;
            const int k_lo = grp == 0 ? 0 : 2, k_hi = grp == 0 ? 1 : 2;
            for (int kind = k_lo; kind <= k_hi; ++kind) {
                float acc[2][2][2][4];
                cols_mma(acc, kind == 0 ? w_hh2 : (kind == 1 ? w_ih2 : w_hh1), crank, w, dg_s, l);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float* dst = ob + (size_t)(kind * CL + (4 * h + w)) * BLK;
#pragma unroll
                    for (int tt = 0; tt < 2; ++tt)
#pragma unroll
                        for (int n = 0; n < 2; ++n)
#pragma unroll
                            for (int e = 0; e < 4; ++e)
                                dst[(8 * n + 2 * (l & 3) + (e & 1)) * U + 16 * tt + (l >> 2) + 8 * (e >> 1)] = acc[h][tt][n][e];
                }
            }
            fence_proxy_async_smem();
            named_bar_sync(1 + grp, 128);
            // ---- reduce-scatter: block (kind, owner d) → owner d's inbox slot [src = me][kind]; one lane per copy
            {
                const int obuf = it & 1, ncopy = (k_hi - k_lo + 1) * CL;
                if (gt < ncopy) {
                    const int kind = k_lo + gt / CL, d = gt % CL;
                    const uint32_t dst = smem_u32(inbox + ((size_t)obuf * CL + crank) * 3 * BLK + kind * BLK);
                    bulk_copy_s2c(mapa_u32(dst, d), smem_u32(ob + (size_t)(kind * CL + d) * BLK), BLK * 4, mapa_u32(smem_u32(ibar + obuf), d));
                }
            }
        }
    }
    cluster.sync();
}

// ======================================================================================================= classifier head
// Linear(256 → V) on the last hidden state + softmax cross-entropy + every gradient of the head, one CTA per 16-row chunk:
// logits, CE (mean over the pair's real rows via `scale`), dlogits, dW_fc, db_fc and dh2_{T-1} (the BPTT kernel's input).
// Replaces fc GEMM + log_softmax + nll + three backward GEMMs + bias reduction (~9 launches) per pair and step.
__global__ void __launch_bounds__(256) lstm_head_kernel(const __grid_constant__ LstmHeadArgs a) {
    constexpr int H = lstm::H, NB = lstm::NB, VP = 96;
    __shared__ float h_s[NB][H];
    __shared__ float dl_s[NB][VP];
    __shared__ float red_s[8];
    const int ch = blockIdx.x, tid = threadIdx.x, w = tid >> 5, l = tid & 31, V = a.V;
    const float* prow = a.params + a.row_off[ch];
    const float* Wfc = prow + a.off_fcw;
    const float* bfc = prow + a.off_fcb;
    const float* hl = a.hlast + (size_t)ch * NB * H;
    for (int i = tid; i < NB * H; i += 256) h_s[i / H][i % H] = hl[i];
    __syncthreads();
    // logits[b][v] = h[b]·W[v] + bias[v]: one warp per output neuron, lanes split K, 16 rows at once
    for (int v = w; v < V; v += 8) {
        float wv[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) wv[j] = __ldg(Wfc + (size_t)v * H + l + 32 * j);
        const float bv = __ldg(bfc + v);
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            float acc = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) acc = fmaf(wv[j], h_s[b][l + 32 * j], acc);
            acc = warp_sum(acc);
            if (l == 0) dl_s[b][v] = acc + bv;
        }
    }
    __syncthreads();
    // softmax-CE per row; dlogits = (p − onehot)·scale   (scale = 1 / #real rows of the pair; padding rows: label < 0 → 0)
    const float scale = a.scale[ch];
    float lsum = 0.f;
    for (int b = w; b < NB; b += 8) {
        const int y = a.labels[ch * NB + b];
        float mx = -INFINITY;
        for (int v = l; v < V; v += 32) mx = fmaxf(mx, dl_s[b][v]);
        mx = warp_max(mx);
        float se = 0.f;
        for (int v = l; v < V; v += 32) se += __expf(dl_s[b][v] - mx);
        se = warp_sum(se);
        const float inv = 1.f / se;
        for (int v = l; v < V; v += 32) {
            const float z = dl_s[b][v];
            const float pr = __expf(z - mx) * inv;
            if (y >= 0 && v == y) lsum += (mx + __logf(se) - z) * scale;
            dl_s[b][v] = (y >= 0) ? (pr - (v == y ? 1.f : 0.f)) * scale : 0.f;
        }
    }
    lsum = warp_sum(lsum);
    if (l == 0) red_s[w] = lsum;
    __syncthreads();
    if (tid == 0 && a.loss) { float t = 0.f; for (int i = 0; i < 8; ++i) t += red_s[i]; a.loss[ch] = t; }
    // thread k: dW[v][k] = Σ_b dl[b][v] h[b][k],  dh[b][k] = Σ_v dl[b][v] W[v][k]
    {
        const int k = tid;
        float hr[NB], dh[NB];
#pragma unroll
        for (int b = 0; b < NB; ++b) { hr[b] = h_s[b][k]; dh[b] = 0.f; }
        float* dW = a.dW + (size_t)ch * V * H;
        for (int v = 0; v < V; ++v) {
            const float wv = __ldg(Wfc + (size_t)v * H + k);
            float acc = 0.f;
#pragma unroll
            for (int b = 0; b < NB; ++b) { const float d = dl_s[b][v]; acc = fmaf(d, hr[b], acc); dh[b] = fmaf(d, wv, dh[b]); }
            dW[(size_t)v * H + k] = acc;
        }
        float* dho = a.dh + (size_t)ch * NB * H;
#pragma unroll
        for (int b = 0; b < NB; ++b) dho[b * H + k] = dh[b];
    }
    if (tid < V) {
        float acc = 0.f;
#pragma unroll
        for (int b = 0; b < NB; ++b) acc += dl_s[b][tid];
        a.db[(size_t)ch * V + tid] = acc;
    }
}

int lstm_head_launch(const LstmHeadArgs& a, int nchunks, cudaStream_t stream) {
    if (a.V > 96 || a.V < 1) return -5;
    lstm_head_kernel<<<nchunks, 256, 0, stream>>>(a);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

// ======================================================================================================= small gradients
// Bias, W_ih1 and embedding gradients of every chunk in one pass over the bf16 gate-gradient histories.  Because the layer-1
// input is x_r = emb[tok_r], all three follow from the token-segmented column sums S[v][col] = Σ_{r: tok_r = v} dG1[r][col]:
//   db1[col] = Σ_v S[v][col],   dW_ih1[col][e] = Σ_v S[v][col]·emb[v][e],   d emb[v][e] = Σ_col S[v][col]·W_ih1[col][e]
// (emb / W_ih1 rounded to bf16 exactly as the forward kernel fed them to the tensor core); db2 is a plain column sum of dG2.
// grid = (chunks, 8 column slices of 128); one thread per gate column; S lives in shared memory (no atomics: a thread owns
// its column).  Replaces ~12 eager kernels that converted both histories to fp32 (≈1.3 GB of traffic per local step).
__global__ void __launch_bounds__(128) lstm_small_grads_kernel(const __grid_constant__ LstmSmallArgs a) {
    constexpr int H4 = 4 * lstm::H, NB = lstm::NB, VP = 96, EP = 16;
    extern __shared__ float sg[];
    float* S = sg;                       // [VP][129]
    float* embq = S + VP * 129;          // [VP][EP]
    float* wq = embq + VP * EP;          // [128][EP]
    int* tokr = reinterpret_cast<int*>(wq + 128 * EP);   // [T*NB] token of history row r = t*16 + b
    const int ch = blockIdx.x, slice = blockIdx.y, tid = threadIdx.x, col = slice * 128 + tid;
    const int T = a.T, E = a.E, V = a.V, TB = T * NB, NP = (int)gridDim.x;
    const float* prow = a.params + a.row_off[ch];
    for (int i = tid; i < VP * 129; i += 128) S[i] = 0.f;
    for (int i = tid; i < VP * EP; i += 128) {
        const int v = i / EP, e = i % EP;
        embq[i] = (v < V && e < E) ? __bfloat162float(__float2bfloat16(__ldg(prow + a.off_emb + (size_t)v * E + e))) : 0.f;
    }
    for (int i = tid; i < 128 * EP; i += 128) {
        const int c = i / EP, e = i % EP;
        wq[i] = (e < E) ? __bfloat162float(__float2bfloat16(__ldg(prow + a.off_wih1 + (size_t)(slice * 128 + c) * E + e))) : 0.f;
    }
    const int* tk = a.tokens + (size_t)ch * NB * T;
    for (int r = tid; r < TB; r += 128) tokr[r] = tk[(r % NB) * T + r / NB];
    __syncthreads();
    const __nv_bfloat16* g1 = reinterpret_cast<const __nv_bfloat16*>(a.dgates) + ((size_t)(0 * NP + ch) * TB) * H4 + col;
    const __nv_bfloat16* g2 = reinterpret_cast<const __nv_bfloat16*>(a.dgates) + ((size_t)(1 * NP + ch) * TB) * H4 + col;
    float b2 = 0.f;
    int r = 0;
    for (; r + 4 <= TB; r += 4) {          // 8 independent loads in flight per thread
        float x1[4], x2[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) { x1[q] = __bfloat162float(g1[(size_t)(r + q) * H4]); x2[q] = __bfloat162float(g2[(size_t)(r + q) * H4]); }
#pragma unroll
        for (int q = 0; q < 4; ++q) { S[tokr[r + q] * 129 + tid] += x1[q]; b2 += x2[q]; }
    }
    for (; r < TB; ++r) { S[tokr[r] * 129 + tid] += __bfloat162float(g1[(size_t)r * H4]); b2 += __bfloat162float(g2[(size_t)r * H4]); }
    // per-column results (this thread's column only: no sync needed yet)
    float b1 = 0.f, dw[EP];
#pragma unroll
    for (int e = 0; e < EP; ++e) dw[e] = 0.f;
    for (int v = 0; v < V; ++v) {
        const float sv = S[v * 129 + tid];
        b1 += sv;
#pragma unroll
        for (int e = 0; e < EP; ++e) dw[e] = fmaf(sv, embq[v * EP + e], dw[e]);
    }
    a.db1[(size_t)ch * H4 + col] = b1;
    a.db2[(size_t)ch * H4 + col] = b2;
    for (int e = 0; e < E; ++e) a.dwih1[((size_t)ch * H4 + col) * E + e] = dw[e];
    __syncthreads();
    // embedding partial of this column slice: demb_part[ch][slice][v][e] = Σ_c S[v][c]·W_ih1[c][e]
    for (int i = tid; i < V * E; i += 128) {
        const int v = i / E, e = i % E;
        float acc = 0.f;
        for (int c = 0; c < 128; ++c) acc = fmaf(S[v * 129 + c], wq[c * EP + e], acc);
        a.demb_part[(((size_t)ch * 8 + slice) * V + v) * E + e] = acc;
    }
}

int lstm_small_grads_launch(const LstmSmallArgs& a, int nchunks, cudaStream_t stream) {
    if (a.V > 96 || a.E > 16) return -5;
    const size_t smem = (size_t)(96 * 129 + 96 * 16 + 128 * 16) * 4 + (size_t)a.T * lstm::NB * 4;
    cudaError_t e = cudaFuncSetAttribute(lstm_small_grads_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return -3;
    lstm_small_grads_kernel<<<dim3(nchunks, 8), 128, smem, stream>>>(a);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

// ======================================================================================================= launchers
static size_t fwd_smem_bytes() {
    using namespace lstm;
    const size_t b = (size_t)(2 * NB * H + 2 * NB * H + 2 * NB * KX + 2 * 2 * NB * U) * 2 + (size_t)2 * 4 * NB * U * 4 + 128;
    return b;
}
static size_t bwd_smem_bytes() {
    using namespace lstm;
    return (size_t)(2 * CL * 3 + 2 * 3 * CL) * NB * U * 4 + (size_t)2 * NB * 128 * 2 + 128;
}

int lstm2_fwd_launch(const LstmArgs& a, int npairs, cudaStream_t stream) {
    const size_t smem = fwd_smem_bytes();
    cudaError_t e = cudaFuncSetAttribute(lstm2_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return -3;
    lstm2_fwd_kernel<<<npairs * lstm::CL, lstm::kFwdThreads, smem, stream>>>(a);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

int lstm2_bwd_launch(const LstmArgs& a, int npairs, cudaStream_t stream) {
    const size_t smem = bwd_smem_bytes();
    cudaError_t e = cudaFuncSetAttribute(lstm2_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return -3;
    lstm2_bwd_kernel<<<npairs * lstm::CL, lstm::kFwdThreads, smem, stream>>>(a);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

}  // namespace fdb
