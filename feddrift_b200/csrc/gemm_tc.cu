// gemm_tn: D[M,N] = act(A[M,K] · B[N,K]ᵀ + bias[N])   bf16 operands, fp32 accumulation in registers (wgmma).
//
// Hand-written Hopper GEMM used by TcLinear (fnn-MNIST 784→1568→10, CNN fc 9216→128, LSTM/classifier heads):
//   * PERSISTENT, warp-specialised: grid = min(#tiles, #SMs); every CTA walks tiles tile = blockIdx.x + i·gridDim.x
//     (M-fastest rasterisation so concurrently running CTAs share the same B panel in L2);
//   * warp 0 = TMA producer (cp.async.bulk.tensor.2d, 128B-swizzled 128×64 / BN×64 bf16 boxes) into a 4 / 6 / 8-stage (BN 256 / 128 / 64) smem ring
//     with full/empty mbarriers; warpgroups 1 and 2 = consumers: each issues wgmma m64×BN×16 for its 64 rows of the 128-row
//     tile (accumulator in registers, one k-block of MMAs kept in flight) and runs the epilogue of those rows (bias + ReLU +
//     cast in registers → 128B-swizzled staging → TMA tile stores) while the producer already fills the next tile's stages;
//   * split-K (grid.z) for skinny outputs (e.g. 512×128×9216): partial tiles are accumulated with fp32 atomics into a
//     zeroed output and bias/activation are applied by a small second kernel.
//   * operand layouts: each of A and B may be K-major ([rows, K], the "TN" form) or MN-major ([K, rows], rows
//     contiguous).  MN-major tiles are fetched as 64×64 TMA boxes (128-byte rows along M/N, 8-row swizzle atoms along
//     K) and described to the tensor core with the MN-major canonical layout (LBO = 8 KB between 64-wide M/N groups,
//     SBO = 1 KB between 8-row K groups, transpose operands of wgmma), so the backward GEMMs
//     dX = dY·W and dW = dYᵀ·X run directly on the row-major tensors autograd hands us — no transpose kernels.
//   * IMPLICIT-GEMM CONVOLUTION on the same mainloop (struct ConvIm below, ops/conv.py): the producer thread issues TMA *im2col*
//     loads (cp.async.bulk.tensor.4d…im2col) from the bf16 NHWC activation tensor — the TMA unit walks the output pixels with the
//     conv stride, applies the filter-tap offset and zero-fills the halo — for the forward, the data gradient (the forward
//     weight pack read MN-major, taps flipped; strided layers on zero-dilated dY) and the weight gradient (reduction over
//     pixels, im2col boxes as the MN-major B operand, cp.reduce.async.bulk adds into the channels_last gradient), optionally
//     GROUPED with one group per stacked (client, model) pair (sim/stacked.py).
// All waits are bounded (trap after 2 s) so a protocol bug faults the context instead of hanging the GPU.
// The reference's equivalent is eager `nn.Linear` + separate bias/ReLU kernels in fp32 on cuBLAS
// (fedml_api/model/fnn/fnn.py:11-15, cv/cnn.py:128-136).
#include <cuda.h>

#include <algorithm>
#include <cstring>
#include <cuda_bf16.h>

#include "common.cuh"
#include "kernels.h"
#include "hopper.cuh"

namespace fdb {

constexpr int BM = 128, BK = 64, MMA_K = 16;
constexpr int kGemmThreads = 384;  // warpgroup 0: warp 0 = TMA producer; warpgroups 1, 2 = wgmma consumers + epilogue (64 rows each)
constexpr uint32_t kStageBytesA = BM * BK * 2;
struct GemmBatch { int batch, a_k0, a_kstride, b_k0, b_kstride; };
// Implicit-GEMM convolution modes: one operand is fetched with TMA *im2col* loads straight from the bf16 NHWC tensor.
//   mode 1 (forward / stride-1 data gradient): A[pixel, (tap, c)] — K-major 128-pixel × 64-channel boxes, one per k-block
//           (k-block kb = tap·cchunks + c-chunk); B = packed weights [Cout, R·S·C], K-major for the forward; the data gradient
//           reads THE SAME pack as an MN-major operand (b_mn: 64(cin) × 64(cout) boxes at column tap'·Cin, taps flipped), so
//           no transposed copy of the weights is ever made;
//   GROUPED convolution (one group per stacked (client, model) pair, sim/stacked.py): gb.batch = groups, M / N are per-group
//   sizes; group g reads channel chunk g·Cg + c of the NHWC tensor, weight rows g·N + n, and writes output columns g·N + n
//   (mode 1) or slice g of the 3-D gradient map [groups][Cout][R·S·C] (mode 2, which therefore clips rows ≥ Cout);
//   mode 2 (weight gradient): reduction over output pixels; A = dY [pixels, Cout] (MN-major tiled loads), B[(tap, c), pixel] —
//           MN-major 64-pixel × 64-channel im2col boxes, one per 64-wide column group of the N tile.
struct ConvIm { int mode, S, cchunks, ntaps, Q, PQ, stride, pad_h, pad_w, flip, bcols; };

template <int BN> struct GemmCfg {
    static constexpr uint32_t kStageBytesB = BN * BK * 2;
    static constexpr uint32_t kStagingBytes = 2 /*consumer warpgroups*/ * 2 /*double buffer*/ * 8192;   // 64 rows × 128 B per buffer
    // 192 KB of operand ring in every configuration: 4 × 48 KB (BN 256), 6 × 32 KB (BN 128), 8 × 24 KB (BN 64) — the narrow tiles
    // of the convolution modes have short K loops, a deeper ring keeps their TMA (im2col) loads far enough ahead
    static constexpr int kStages = BN == 256 ? 4 : (BN == 128 ? 6 : 8);
    static constexpr uint32_t kSmemBytes = kStages * (kStageBytesA + kStageBytesB) + kStagingBytes + 1024 /*align slack*/ + 256 /*barriers*/;
};

template <int BN, int TA, int TB>
FDB_DEVICE void gemm_kblock(float (&d)[BN / 2], uint64_t da0, uint64_t db0, bool first) {
    // per MMA_K step the start address moves by 32 B (K-major: 16 elements along the row) or 2048 B (MN-major: 16 K-rows =
    // two 1024-B atoms)
    constexpr uint32_t a_kstep = TA ? (2048u >> 4) : ((MMA_K * 2u) >> 4), b_kstep = TB ? (2048u >> 4) : ((MMA_K * 2u) >> 4);
#pragma unroll
    for (int k = 0; k < BK / MMA_K; ++k)
        Wgmma<BN, TA, TB>::mma(d, da0 + (uint64_t)(k * a_kstep), db0 + (uint64_t)(k * b_kstep), (first && k == 0) ? 0u : 1u);
}

template <int BN>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tn_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
               const __grid_constant__ CUtensorMap map_d, void* __restrict__ D, const float* __restrict__ bias, int M, int N, int K,
               int relu, int out_fp32, int splits, int tma_out, int a_mn, int b_mn, GemmBatch gb, ConvIm ci) {
    using Cfg = GemmCfg<BN>;
    constexpr int STAGES = Cfg::kStages;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem + STAGES * kStageBytesA;
    uint8_t* staging = smem + STAGES * (kStageBytesA + Cfg::kStageBytesB);   // 1024-aligned: [2 warpgroups][2][64 rows × 128 B]
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + Cfg::kStagingBytes);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;   // warp index in a uniform register
    const int m_tiles = (M + BM - 1) / BM, n_tiles = (N + BN - 1) / BN;
    // batched mode (gb.batch > 1; both operands MN-major, M % 128 == 0, K % 64 == 0): batch bt multiplies the reduction rows
    // [a_k0 + bt·a_kstride, +K) of A' with [b_k0 + bt·b_kstride, +K) of B' into rows [bt·M, bt·M + M) of D — one launch for
    // the weight gradients dW_p = dG_pᵀ·H_p of every (client, model) pair
    const int tiles_per_batch = m_tiles * n_tiles;
    const int num_tiles = tiles_per_batch * gb.batch;
    const int kb_total = (K + BK - 1) / BK;
    const int kb_per = (kb_total + splits - 1) / splits;
    const int kb_lo = blockIdx.z * kb_per, kb_hi = min(kb_total, kb_lo + kb_per);
    const int nkb = max(kb_hi - kb_lo, 0);

    if (warp == 0 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b) : "memory");
        if (tma_out) asm volatile("prefetch.tensormap [%0];" ::"l"(&map_d) : "memory");
    }
    if (warp == 1 && lane == 0) {
        // a stage is released by lane 0 of each of the 8 consumer warps once its wgmma reads are complete
        for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar + s, 1); mbar_init(empty_bar + s, 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 0) {
        if (nkb > 0) {  // ===== TMA producer: the whole warp walks the loop (uniform control flow), one elected lane issues
            uint32_t it = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int bt = tile / tiles_per_batch, rem = tile - bt * tiles_per_batch;
                const int m_blk = rem % m_tiles, n_blk = rem / m_tiles;
                const int ak = gb.a_k0 + bt * gb.a_kstride, bk = gb.b_k0 + bt * gb.b_kstride;   // 0 unless batched
                int cw = 0, chh = 0, cn = 0;          // im2col anchor of the tile's first pixel (mode 1)
                if (ci.mode == 1) {
                    const int m0 = m_blk * BM;
                    cn = m0 / ci.PQ;
                    const int rem2 = m0 - cn * ci.PQ, p = rem2 / ci.Q, q = rem2 - p * ci.Q;
                    cw = q * ci.stride - ci.pad_w;
                    chh = p * ci.stride - ci.pad_h;
                }
                int nvalid = BN / 64;                  // mode 2: 64-wide (tap, c-chunk) column groups of this N tile that exist
                if (ci.mode == 2) nvalid = max(0, min(BN / 64, ci.ntaps * ci.cchunks - n_blk * (BN / 64)));
                for (int kb = kb_lo; kb < kb_hi; ++kb, ++it) {
                    const int s = it % STAGES;
                    const uint32_t ph = (it / STAGES) & 1;
                    mbar_wait(empty_bar + s, ph ^ 1);
                    uint8_t* sa = smem_a + s * kStageBytesA;
                    uint8_t* sb = smem_b + s * Cfg::kStageBytesB;
                    if (!elect_one()) continue;
                    if (ci.mode == 1) {
                        mbar_expect_tx(full_bar + s, kStageBytesA + Cfg::kStageBytesB);
                        const int tap = kb / ci.cchunks, cc = kb - tap * ci.cchunks;
                        const int r = tap / ci.S, sx = tap - r * ci.S;
                        const int cg = bt * ci.cchunks * 64;        // first channel of this group in the NHWC tensor / first K row
                        tma_load_im2col_4d(&map_a, full_bar + s, sa, cg + cc * 64, cw, chh, cn, (uint16_t)sx, (uint16_t)r);
                        const int wtap = ci.flip ? ci.ntaps - 1 - tap : tap;
                        if (b_mn) {
#pragma unroll
                            for (int h = 0; h < BN / 64; ++h)
                                tma_load_2d(&map_b, full_bar + s, sb + h * 8192, wtap * ci.bcols + n_blk * BN + h * 64, cg + cc * BK);
                        } else {
                            tma_load_2d(&map_b, full_bar + s, sb, (wtap * ci.cchunks + cc) * BK, bt * N + n_blk * BN);
                        }
                        continue;
                    }
                    if (ci.mode == 2) {
                        mbar_expect_tx(full_bar + s, kStageBytesA + (uint32_t)nvalid * 8192u);
#pragma unroll
                        for (int h = 0; h < BM / 64; ++h) tma_load_2d(&map_a, full_bar + s, sa + h * 8192, bt * M + m_blk * BM + h * 64, kb * BK);
                        const int p0 = kb * BK, pn = p0 / ci.PQ, prem = p0 - pn * ci.PQ, pp = prem / ci.Q, pq = prem - pp * ci.Q;
                        for (int h = 0; h < nvalid; ++h) {
                            const int j = n_blk * (BN / 64) + h, tap = j / ci.cchunks, cc = j - tap * ci.cchunks;
                            const int r = tap / ci.S, sx = tap - r * ci.S;
                            tma_load_im2col_4d(&map_b, full_bar + s, sb + h * 8192, bt * ci.cchunks * 64 + cc * 64, pq * ci.stride - ci.pad_w,
                                               pp * ci.stride - ci.pad_h, pn, (uint16_t)sx, (uint16_t)r);
                        }
                        continue;
                    }
                    mbar_expect_tx(full_bar + s, kStageBytesA + Cfg::kStageBytesB);
                    if (a_mn) {   // [K, M] tensor: two 64(M)×64(K) boxes
#pragma unroll
                        for (int h = 0; h < BM / 64; ++h) tma_load_2d(&map_a, full_bar + s, sa + h * 8192, m_blk * BM + h * 64, ak + kb * BK);
                    } else {
                        tma_load_2d(&map_a, full_bar + s, sa, kb * BK, m_blk * BM);
                    }
                    if (b_mn) {
#pragma unroll
                        for (int h = 0; h < BN / 64; ++h) tma_load_2d(&map_b, full_bar + s, sb + h * 8192, n_blk * BN + h * 64, bk + kb * BK);
                    } else {
                        tma_load_2d(&map_b, full_bar + s, sb, kb * BK, n_blk * BN);
                    }
                }
            }
        }
    } else if (warp >= 4 && nkb > 0) {
        // ===== consumer warpgroup wg: rows [64·wg, 64·wg + 64) of every tile; warp w of the group holds rows 16w + lane/4 (+8)
        const int wg = (warp >> 2) - 1, w = warp & 3, tg = threadIdx.x & 127;
        const int g8 = lane >> 2, c4 = lane & 3;
        uint32_t it = 0, chunk_it = 0;
        // the 64-row half of an A stage: K-major rows 64·wg… (64 × 128 B) or MN-major M group wg (64 K-rows × 128 B): 8 KB in both
        const uint64_t desc_a0 = (a_mn ? make_smem_desc_mn(smem_u32(smem_a)) : make_smem_desc(smem_u32(smem_a))) + (uint64_t)((wg * 8192) >> 4);
        const uint64_t desc_b0 = b_mn ? make_smem_desc_mn(smem_u32(smem_b)) : make_smem_desc(smem_u32(smem_b));
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            const int bt = tile / tiles_per_batch, rem = tile - bt * tiles_per_batch;
            const int m_blk = rem % m_tiles, n_blk = rem / m_tiles;
            float d[BN / 2];   // no initialisation: the first k-block's MMAs run with scale-d = 0
            int s_prev = -1;
            for (int kb = 0; kb < nkb; ++kb, ++it) {
                const int s = it % STAGES;
                const uint32_t ph = (it / STAGES) & 1;
                mbar_wait(full_bar + s, ph);
                const uint64_t da0 = desc_a0 + (uint64_t)((s * kStageBytesA) >> 4);
                const uint64_t db0 = desc_b0 + (uint64_t)((s * Cfg::kStageBytesB) >> 4);
                wgmma_fence();
                if (a_mn) {
                    if (b_mn) gemm_kblock<BN, 1, 1>(d, da0, db0, kb == 0); else gemm_kblock<BN, 1, 0>(d, da0, db0, kb == 0);
                } else {
                    if (b_mn) gemm_kblock<BN, 0, 1>(d, da0, db0, kb == 0); else gemm_kblock<BN, 0, 0>(d, da0, db0, kb == 0);
                }
                wgmma_commit();
                wgmma_wait<1>();   // the previous k-block's MMAs are complete: its stage may be refilled
                if (s_prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(empty_bar + s_prev); }
                s_prev = s;
            }
            wgmma_wait<0>();
            fence_acc(d);
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar + s_prev);

            const int rbase = m_blk * BM + 64 * wg + 16 * w + g8;   // row of d[i] with (i/2)%2 == 0; +8 for the other half
            if (tma_out) {
                // Coalesced path: registers (bias/ReLU/cast) → 128B-swizzled smem staging → TMA tile stores (or fp32 reduce-add
                // for split-K) of two 32-row boxes per 128-byte column chunk.  Staging is double-buffered per warpgroup; TMA clips
                // the M/N edges.  Batched GEMM outputs are stacked along the rows of D; grouped convolutions write column block g·N
                // (mode 1) or slice g of the 3-D gradient map (mode 2).
                constexpr int CPC = 32;                      // fp32 columns per chunk (bf16: 64, see below)
                const int row0 = (ci.mode ? 0 : bt * M) + m_blk * BM + 64 * wg;
                const int colg = ci.mode == 1 ? bt * N : 0;
                uint8_t* const bufs = staging + wg * 2 * 8192;
                const int rb = 16 * (w & 1) + g8;             // row inside this warp's 32-row box (box = w / 2); +8 for the other half
#pragma unroll
                for (int c0 = 0; c0 < BN; c0 += CPC) {   // constant stride: the accumulator stays in registers
                    if (n_blk * BN + c0 >= N) break;   // uniform
                    if (!out_fp32 && (c0 & CPC)) continue;
                    const int col0 = colg + n_blk * BN + c0;
                    uint8_t* buf = bufs + (chunk_it & 1) * 8192;
                    if (chunk_it >= 2 && tg == 0) tma_store_wait_read<1>();   // the store that last read this buffer is done
                    named_bar_sync(1 + wg, 128);
                    const uint32_t sbox = smem_u32(buf) + (uint32_t)(w >> 1) * 4096u;
                    if (out_fp32) {
#pragma unroll
                        for (int jj = 0; jj < 4; ++jj) {
                            const int ib = ((c0 >> 3) + jj) * 4;
                            if (ib >= BN / 2) break;
                            const int lc = 8 * jj + 2 * c4;
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                float x0 = d[ib + 2 * h], x1 = d[ib + 2 * h + 1];
                                if (splits == 1) {
                                    if (bias) {
                                        x0 += (col0 - colg + lc < N) ? __ldg(bias + col0 + lc) : 0.f;
                                        x1 += (col0 - colg + lc + 1 < N) ? __ldg(bias + col0 + lc + 1) : 0.f;
                                    }
                                    if (relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
                                }
                                const int r = rb + 8 * h, chunk = 2 * jj + (c4 >> 1);
                                const uint32_t addr = sbox + r * 128 + ((chunk ^ (r & 7)) << 4) + (c4 & 1) * 8;
                                asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(__float_as_uint(x0)), "r"(__float_as_uint(x1)) : "memory");
                            }
                        }
                    } else {
#pragma unroll
                        for (int jj = 0; jj < 8; ++jj) {
                            const int ib = ((c0 >> 3) + jj) * 4;
                            if (ib >= BN / 2) break;
                            const int lc = 8 * jj + 2 * c4;
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                float x0 = d[ib + 2 * h], x1 = d[ib + 2 * h + 1];
                                if (bias) {
                                    x0 += (col0 + lc < N) ? __ldg(bias + col0 + lc) : 0.f;
                                    x1 += (col0 + lc + 1 < N) ? __ldg(bias + col0 + lc + 1) : 0.f;
                                }
                                if (relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
                                __nv_bfloat162 pk = __floats2bfloat162_rn(x0, x1);
                                const int r = rb + 8 * h;
                                const uint32_t addr = sbox + r * 128 + ((jj ^ (r & 7)) << 4) + c4 * 4;
                                asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(*reinterpret_cast<uint32_t*>(&pk)) : "memory");
                            }
                        }
                    }
                    fence_proxy_async_smem();
                    named_bar_sync(1 + wg, 128);
                    if (tg == 0) {
#pragma unroll
                        for (int bx = 0; bx < 2; ++bx) {
                            const uint8_t* src = buf + bx * 4096;
                            if (ci.mode == 2) tma_reduce_add_3d(&map_d, src, col0, row0 + 32 * bx, bt);   // wgrad always accumulates into slice g
                            else if (splits > 1) tma_reduce_add_2d(&map_d, src, col0, row0 + 32 * bx);
                            else tma_store_2d(&map_d, src, col0, row0 + 32 * bx);
                        }
                        tma_store_commit();
                    }
                    ++chunk_it;
                }
            } else {
#pragma unroll
                for (int i = 0; i < BN / 2; i += 2) {
                    const int row = rbase + 8 * ((i >> 1) & 1);
                    const int col = n_blk * BN + 8 * (i >> 2) + 2 * c4;
                    if (row >= M) continue;
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        if (col + e >= N) continue;
                        float x = d[i + e];
                        if (splits > 1) { atomicAdd(reinterpret_cast<float*>(D) + (size_t)row * N + col + e, x); continue; }
                        if (bias) x += __ldg(bias + col + e);
                        if (relu) x = fmaxf(x, 0.f);
                        if (out_fp32) reinterpret_cast<float*>(D)[(size_t)row * N + col + e] = x;
                        else reinterpret_cast<__nv_bfloat16*>(D)[(size_t)row * N + col + e] = __float2bfloat16(x);
                    }
                }
            }
        }
        if (tma_out && tg == 0) tma_store_wait_all();   // smem must outlive the in-flight bulk stores
    }
    __syncthreads();
}

// bias + activation (+ cast) pass for split-K outputs
__global__ void bias_act_kernel(const float* __restrict__ acc, void* __restrict__ D, const float* __restrict__ bias, long long MN, int N,
                                int relu, int out_fp32) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < MN; i += (long long)gridDim.x * blockDim.x) {
        float x = acc[i];
        if (bias) x += bias[i % N];
        if (relu) x = fmaxf(x, 0.f);
        if (out_fp32) reinterpret_cast<float*>(D)[i] = x;
        else reinterpret_cast<__nv_bfloat16*>(D)[i] = __float2bfloat16(x);
    }
}

// ---------------------------------------------------------------- host side: tensor maps via the driver entry point
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    return fn;
}

static int make_map(CUtensorMap* map, const void* base, int rows, int cols /*K*/, int box_rows) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return -1;
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -2;
}

// exported for conv_igemm.cu: K-major 128B-swizzled map of a bf16 [rows, cols] matrix with (64 × box_rows) boxes
int make_kmajor_sw128_map(void* map_out, const void* base, int rows, int cols, int box_rows) {
    return make_map(reinterpret_cast<CUtensorMap*>(map_out), base, rows, cols, box_rows);
}

// output map: 32-row × 128-byte boxes (32 fp32 or 64 bf16 columns), 128B swizzle — what one epilogue warp stages per chunk.
// Returns 0 and sets *ok = 1 when D qualifies for TMA stores (16-byte aligned base and row pitch).
static int make_out_map(CUtensorMap* map, void* D, int M, int N, int out_fp32, int* ok) {
    *ok = 0;
    memset(map, 0, sizeof(*map));
    const size_t es = out_fp32 ? 4 : 2;
    if ((reinterpret_cast<uintptr_t>(D) & 15) || ((size_t)N * es) % 16 != 0) return 0;
    EncodeTiledFn enc = get_encode();
    if (!enc) return -1;
    cuuint64_t dims[2] = {(cuuint64_t)N, (cuuint64_t)M};
    cuuint64_t strides[1] = {(cuuint64_t)N * es};
    cuuint32_t box[2] = {(cuuint32_t)(out_fp32 ? 32 : 64), 32u};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, out_fp32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, D, dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return -2;
    *ok = 1;
    return 0;
}

// MN-major operand X'[K, rows] (rows contiguous): 64×64 boxes, 128-byte rows
static int make_map_mn(CUtensorMap* map, const void* base, int rows, int K) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return -1;
    cuuint64_t dims[2] = {(cuuint64_t)rows, (cuuint64_t)K};
    cuuint64_t strides[1] = {(cuuint64_t)rows * 2};
    cuuint32_t box[2] = {64u, (cuuint32_t)BK};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -2;
}

// im2col map over a bf16 NHWC tensor [N, H, W, C]: boxes of `pixels` anchor pixels × 64 channels, 128B swizzle; the bounding
// box of anchors is the set of output positions of an R×S filter with symmetric padding, walked with the conv stride
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const int*,
                                   const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeIm2colFn get_encode_im2col() {
    static EncodeIm2colFn fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeIm2colFn>(ptr);
    }
    return fn;
}
static int make_im2col_map(CUtensorMap* map, const void* base, int N, int H, int W, int C, int R, int S, int pad_h, int pad_w, int stride,
                           int pixels) {
    EncodeIm2colFn enc = get_encode_im2col();
    if (!enc) return -1;
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
    int lower[2] = {-pad_w, -pad_h};
    int upper[2] = {pad_w - (S - 1), pad_h - (R - 1)};
    cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, lower, upper, 64u, (cuuint32_t)pixels,
                     estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -2;
}

template <int BN>
static int launch_gemm(const CUtensorMap& ma, const CUtensorMap& mb, void* D, const float* bias, int M, int N, int K, int relu,
                       int out_fp32, int splits, int sms, int a_mn, int b_mn, cudaStream_t stream, GemmBatch gb = GemmBatch{1, 0, 0, 0, 0},
                       ConvIm ci = ConvIm{0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0}, const CUtensorMap* md_conv = nullptr) {
    CUtensorMap md;
    int tma_out = 0;
    if (md_conv) { md = *md_conv; tma_out = 1; }     // convolution modes bring their own output map (grouped columns / 3-D gradient)
    else if (make_out_map(&md, D, M * gb.batch, N, out_fp32, &tma_out) != 0) return -7;
    if (gb.batch > 1 && !tma_out) return -9;
    using Cfg = GemmCfg<BN>;
    static bool attr_set = false;
    if (!attr_set) {
        if (cudaFuncSetAttribute(gemm_tn_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::kSmemBytes) != cudaSuccess) return -3;
        attr_set = true;
    }
    const int tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN) * gb.batch;
    dim3 grid(min(tiles, max(1, sms / splits)), 1, splits);
    gemm_tn_kernel<BN><<<grid, kGemmThreads, Cfg::kSmemBytes, stream>>>(ma, mb, md, D, bias, M, N, K, relu, out_fp32, splits, tma_out, a_mn, b_mn, gb, ci);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

// number of K-splits gemm_launch will use for this problem (callers that want a bf16 output pre-allocate the fp32
// accumulation workspace with their own allocator when this is > 1)
int gemm_split_count(int M, int N, int K) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int bn = (N > 128) ? 256 : 128;
    const int tiles = ((M + BM - 1) / BM) * ((N + bn - 1) / bn);
    const int kb_total = (K + BK - 1) / BK;
    int splits = 1;
    if (tiles * 4 <= sms && kb_total >= 16) {   // too few output tiles to fill the machine and a long K
        splits = min(min(sms / tiles, kb_total / 4), 32);
        if (splits < 2) splits = 1;
    }
    return splits;
}

int gemm_launch(const void* A, const void* B, void* D, const float* bias, int M, int N, int K, int a_mn, int b_mn, int relu, int out_fp32,
                cudaStream_t stream, float* splitk_ws) {
    // TMA global strides must be multiples of 16 B: the contiguous extent of each operand must be a multiple of 8 bf16
    if (M <= 0 || N <= 0 || K <= 0) return -5;
    if ((a_mn ? M : K) % 8 != 0 || (b_mn ? N : K) % 8 != 0) return -5;
    if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15)) return -6;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int bn = (N > 128) ? 256 : 128;
    CUtensorMap ma, mb;
    if ((a_mn ? make_map_mn(&ma, A, M, K) : make_map(&ma, A, M, K, BM)) != 0) return -7;
    if ((b_mn ? make_map_mn(&mb, B, N, K) : make_map(&mb, B, N, K, bn)) != 0) return -7;
    const int tiles = ((M + BM - 1) / BM) * ((N + bn - 1) / bn);
    const int kb_total = (K + BK - 1) / BK;
    (void)tiles; (void)kb_total;
    const int splits = gemm_split_count(M, N, K);
    if (splits > 1) {
        float* acc = nullptr;
        const size_t bytes = (size_t)M * N * sizeof(float);
        bool own = false;
        if (out_fp32) acc = reinterpret_cast<float*>(D);
        else if (splitk_ws) acc = splitk_ws;     // caller's allocator (torch caching allocator: no driver call on the hot path)
        else { if (cudaMallocAsync(&acc, bytes, stream) != cudaSuccess) return -8; own = true; }
        cudaMemsetAsync(acc, 0, bytes, stream);
        int rc = (bn == 256) ? launch_gemm<256>(ma, mb, acc, nullptr, M, N, K, 0, 1, splits, sms, a_mn, b_mn, stream)
                             : launch_gemm<128>(ma, mb, acc, nullptr, M, N, K, 0, 1, splits, sms, a_mn, b_mn, stream);
        if (rc != 0) return rc;
        if (bias || relu || !out_fp32) {
            const long long MN = (long long)M * N;
            bias_act_kernel<<<(int)min((MN + 255) / 256, 132LL * 8), 256, 0, stream>>>(acc, D, bias, MN, N, relu, out_fp32);
        }
        if (own) cudaFreeAsync(acc, stream);
        return cudaGetLastError() == cudaSuccess ? 0 : -4;
    }
    return (bn == 256) ? launch_gemm<256>(ma, mb, D, bias, M, N, K, relu, out_fp32, 1, sms, a_mn, b_mn, stream)
                       : launch_gemm<128>(ma, mb, D, bias, M, N, K, relu, out_fp32, 1, sms, a_mn, b_mn, stream);
}

// Batched dW-style GEMM: D[bt·M + m, n] = Σ_k A'[a_k0 + bt·a_kstride + k, m] · B'[b_k0 + bt·b_kstride + k, n]   (k < K), fp32 out.
// A' is [a_rows_total, M] and B' is [b_rows_total, N] (bf16, row-major = MN-major operands).
int gemm_batched_mn_launch(const void* A, const void* B, float* D, int M, int N, int K, int batch, int a_rows_total, int b_rows_total,
                           int a_k0, int a_kstride, int b_k0, int b_kstride, cudaStream_t stream) {
    if (M <= 0 || N <= 0 || K <= 0 || batch <= 0) return -5;
    if (M % BM != 0 || K % BK != 0 || M % 8 != 0 || N % 8 != 0) return -5;
    if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15)) return -6;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int bn = (N > 128) ? 256 : 128;
    CUtensorMap ma, mb;
    if (make_map_mn(&ma, A, M, a_rows_total) != 0) return -7;
    if (make_map_mn(&mb, B, N, b_rows_total) != 0) return -7;
    GemmBatch gb{batch, a_k0, a_kstride, b_k0, b_kstride};
    return (bn == 256) ? launch_gemm<256>(ma, mb, D, nullptr, M, N, K, 0, 1, 1, sms, 1, 1, stream, gb)
                       : launch_gemm<128>(ma, mb, D, nullptr, M, N, K, 0, 1, 1, sms, 1, 1, stream, gb);
}

static int launch_bn(int bn, const CUtensorMap& ma, const CUtensorMap& mb, void* D, const float* bias, int M, int N, int K, int relu,
                     int out_fp32, int splits, int sms, int a_mn, int b_mn, cudaStream_t stream, const ConvIm& ci, int groups,
                     const CUtensorMap& md) {
    const GemmBatch gb{groups, 0, 0, 0, 0};
    if (bn == 256) return launch_gemm<256>(ma, mb, D, bias, M, N, K, relu, out_fp32, splits, sms, a_mn, b_mn, stream, gb, ci, &md);
    if (bn == 128) return launch_gemm<128>(ma, mb, D, bias, M, N, K, relu, out_fp32, splits, sms, a_mn, b_mn, stream, gb, ci, &md);
    return launch_gemm<64>(ma, mb, D, bias, M, N, K, relu, out_fp32, splits, sms, a_mn, b_mn, stream, gb, ci, &md);
}

// 3-D fp32 output map of the weight-gradient GEMM: [groups][Cout][R·S·C] with `gstride` floats between the groups' gradients
// (the flat gradient rows of the stacked pairs); 32-row × 32-column × 1 boxes, rows ≥ Cout are clipped
static int make_wgrad_map(CUtensorMap* map, float* base, int groups, int cout, int rsc, long long gstride) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return -1;
    cuuint64_t dims[3] = {(cuuint64_t)rsc, (cuuint64_t)cout, (cuuint64_t)groups};
    cuuint64_t strides[2] = {(cuuint64_t)rsc * 4, (cuuint64_t)(groups > 1 ? gstride : (long long)rsc * cout) * 4};
    cuuint32_t box[3] = {32u, 32u, 1u};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -2;
}

// Implicit-GEMM convolution on the GEMM mainloop (TMA im2col producer), optionally GROUPED (groups > 1: one group per stacked
// (client, model) pair; C and Cout are PER-GROUP channel counts, the tensors hold groups·C / groups·Cout channels).
// xb: bf16 NHWC [N, H, W, groups·C] (C % 64 == 0), wq: bf16 weights [groups·Cout, R·S·C] (the channels_last storage of the
// parameters, cast), y: fp32 NHWC [N, P, Q, groups·Cout].  Square filters, symmetric padding.
//   dgrad = 0: forward, y = act(conv(x, w) + bias).
//   dgrad = 1: stride-1 data gradient: xb = dY [N, P, Q, groups·Cout_fwd] (C = Cout_fwd), wq = the SAME forward pack
//              [groups·Cout_fwd, R·S·Cin_fwd], `Cout` = Cin_fwd, pad = R-1-pad_fwd; the pack is read MN-major with flipped taps.
int conv_tma_fwd_launch(const void* xb, const void* wq, float* y, const float* bias, int N, int H, int W, int C, int Cout, int R, int S, int P,
                        int Q, int pad, int stride, int dgrad, int relu, int groups, cudaStream_t stream) {
    if (C % 64 != 0 || Cout % 8 != 0 || R != S || N <= 0 || groups < 1) return -5;
    if (groups > 1 && Cout % 32 != 0) return -5;       // a 32-column output chunk must not straddle two groups
    if ((reinterpret_cast<uintptr_t>(xb) & 15) || (reinterpret_cast<uintptr_t>(wq) & 15) || (reinterpret_cast<uintptr_t>(y) & 15)) return -6;
    const long long Mll = (long long)N * P * Q;
    if (Mll >= (1LL << 31) - 256 || (long long)groups * C >= (1LL << 31)) return -5;
    const int M = (int)Mll, K = R * S * C;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int m_tiles = (M + BM - 1) / BM;
    // widest N tile that still gives every SM a tile; otherwise the narrowest and split K over the taps
    int bn = Cout <= 64 ? 64 : 128;
    if (Cout >= 256 && (long long)m_tiles * ((Cout + 255) / 256) * groups >= sms) bn = 256;
    const long long tiles = (long long)m_tiles * ((Cout + bn - 1) / bn) * groups;
    const int kb_total = K / BK;
    int splits = 1;
    if (tiles * 2 <= sms && kb_total >= 8) splits = std::max(1, std::min(std::min(sms / (int)tiles, kb_total / 4), 16));
    CUtensorMap ma, mb, md;
    int ok = 0;
    if (make_im2col_map(&ma, xb, N, H, W, groups * C, R, S, pad, pad, stride, BM) != 0) return -7;
    if (dgrad) { if (make_map_mn(&mb, wq, R * S * Cout, groups * C) != 0) return -7; }   // [groups·Cout_fwd rows (K), R·S·Cin_fwd contiguous]
    else if (make_map(&mb, wq, groups * Cout, K, bn) != 0) return -7;
    if (make_out_map(&md, y, M, groups * Cout, 1, &ok) != 0 || !ok) return -7;
    const ConvIm ci{1, S, C / 64, R * S, Q, P * Q, stride, pad, pad, dgrad, Cout};
    if (splits > 1) {
        cudaMemsetAsync(y, 0, (size_t)M * groups * Cout * sizeof(float), stream);
        int rc = launch_bn(bn, ma, mb, y, nullptr, M, Cout, K, 0, 1, splits, sms, 0, dgrad, stream, ci, groups, md);
        if (rc != 0) return rc;
        if (bias || relu) {
            const long long MN = (long long)M * groups * Cout;
            bias_act_kernel<<<(int)std::min<long long>((MN + 255) / 256, 132LL * 8), 256, 0, stream>>>(y, y, bias, MN, groups * Cout, relu, 1);
        }
        return cudaGetLastError() == cudaSuccess ? 0 : -4;
    }
    return launch_bn(bn, ma, mb, y, bias, M, Cout, K, relu, 1, 1, sms, 0, dgrad, stream, ci, groups, md);
}

// Weight gradient: dw[g][Cout, (r, s, c)] (fp32) += Σ_pixels dY[pixel, g·Cout + k] · X[gather(pixel, r, s), g·C + c] — the tiles are
// REDUCE-ADDED (cp.reduce.async.bulk) into the buffer, which is the channels_last storage of the parameters' gradients: the
// flat gradient rows of the federated executors (`gstride` floats between the groups' segments), or a zeroed tensor.
// xb: bf16 NHWC activations [N, H, W, groups·C], dyb: bf16 [N·P·Q, groups·Cout].
int conv_tma_wgrad_launch(const void* xb, const void* dyb, float* dw_ohwi, int N, int H, int W, int C, int Cout, int R, int S, int P, int Q,
                          int pad, int stride, int groups, long long gstride, cudaStream_t stream) {
    if (C % 64 != 0 || Cout % 8 != 0 || R != S || N <= 0 || groups < 1) return -5;
    if ((reinterpret_cast<uintptr_t>(xb) & 15) || (reinterpret_cast<uintptr_t>(dyb) & 15) || (reinterpret_cast<uintptr_t>(dw_ohwi) & 15)) return -6;
    if (groups > 1 && (gstride % 4 != 0 || gstride < (long long)Cout * R * S * C)) return -6;
    const long long Kll = (long long)N * P * Q;
    if (Kll >= (1LL << 31) - 256) return -5;
    const int Kpix = (int)Kll, RSC = R * S * C;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int bn = 128;
    const long long tiles = (long long)((Cout + BM - 1) / BM) * ((RSC + bn - 1) / bn) * groups;
    const int kb_total = (Kpix + BK - 1) / BK;
    int splits = tiles >= sms ? 1 : std::max(1, std::min(std::min(sms / (int)tiles, kb_total / 2), 64));
    CUtensorMap ma, mb, md;
    if (make_map_mn(&ma, dyb, groups * Cout, Kpix) != 0) return -7;
    if (make_im2col_map(&mb, xb, N, H, W, groups * C, R, S, pad, pad, stride, BK) != 0) return -7;
    if (make_wgrad_map(&md, dw_ohwi, groups, Cout, RSC, gstride) != 0) return -7;
    const ConvIm ci{2, S, C / 64, R * S, Q, P * Q, stride, pad, pad, 0, 0};
    return launch_bn(bn, ma, mb, dw_ohwi, nullptr, Cout, RSC, Kpix, 0, 1, splits, sms, 1, 1, stream, ci, groups, md);
}

int gemm_tn_launch(const void* A, const void* B, void* D, const float* bias, int M, int N, int K, int relu, int out_fp32,
                   cudaStream_t stream) {
    return gemm_launch(A, B, D, bias, M, N, K, 0, 0, relu, out_fp32, stream, nullptr);
}

}  // namespace fdb
