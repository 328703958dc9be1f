// Host-callable launchers of the feddrift_b200 sm_90a kernels (raw pointers; bindings.cpp wraps them).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <cstdint>

namespace fdb {
// aggregate.cu
int cluster_aggregate_launch(float* theta, int theta_stride, const float* cp, const float* n, int C, int M, int P, float* tot_out,
                             int opt_kind, float lr, float momentum, float b1, float b2, float eps, int step, float* s0, float* s1,
                             const int* steps, const unsigned char* mask, cudaStream_t stream);
int weighted_average_launch(const float* rows, const float* w, int n, long long P, float* out, cudaStream_t stream);
int merge_axpby_launch(float* base_row, const float* second_row, float w1, float w2, long long P, cudaStream_t stream);
int sq_diff_sum_launch(const float* a, const float* b, long long P, double* out, cudaStream_t stream);
int gossip_mix_launch(const float* X, const float* Wm, int n, long long P, float* out, cudaStream_t stream);
int gossip_mix_peer_launch(const long long* x_ptrs, const long long* flag_ptrs, const float* w, int P, int world, int rank,
                           unsigned* grid_sync, unsigned grid_base, unsigned epoch, int grid, long long timeout_ms, int* error_flag,
                           cudaStream_t stream);
// K10: row r of rows [R, P] is clipped around g + (r % M)·g_stride; rows with n[r] == 0 are skipped (n may be nullptr)
int robust_clip_launch(float* rows, const float* g, long long g_stride, int M, const float* n, const unsigned char* mask, int R,
                       long long P, float bound, float* scratch_nrm2, float* nrm_out, float stddev, unsigned seed, cudaStream_t stream);
// compress.cu (K17): QSGD of row r of rows [R, P] against theta + (r % M)·t_stride with level s and bucket b; rows with
// n[r] <= 0 are skipped (n may be nullptr), entries with mask 0 pass through; scratch_smax holds R·⌈P / min(b, P)⌉ words
int qsgd_slots_launch(float* rows, const float* theta, long long t_stride, int M, const float* n, const unsigned char* mask, int R,
                      long long P, int level, long long bucket, unsigned* scratch_smax, unsigned seed, cudaStream_t stream);
// sparsify.cu (K18): top-k with error feedback of row r of rows [R, P] and its residual row res[r] against
// theta + (r % M)·t_stride, keeping k trainable entries; rows with n[r] <= 0 are skipped (n may be nullptr), entries with
// mask 0 pass through; scratch holds eftopk_scratch_words(R, P) words
long long eftopk_scratch_words(int R, long long P);
int eftopk_slots_launch(float* rows, const float* theta, long long t_stride, int M, float* res, const float* n,
                        const unsigned char* mask, int R, long long P, long long k, unsigned* scratch, cudaStream_t stream);
// robust_agg.cu (K19): coordinate-wise median (median = 1) or trimmed mean (trim ratio beta) of the rows with n[c·M + m] > 0
// of cp [C, M, P] into theta + m·t_stride for every slot with a participant; opt_kind != 0 steps each such slot with the
// server optimizer (bias corrections from steps[m] + 1; the caller advances steps).  -2: C too large for the staging tile
int robust_aggregate_launch(float* theta, long long t_stride, const float* cp, const float* n, int C, int M, long long P,
                            int median, float beta, int opt_kind, float lr, float momentum, float b1, float b2, float eps,
                            float* s0, float* s1, const int* steps, const unsigned char* mask, cudaStream_t stream);
// robust_agg.cu (K20): geometric median (smoothed Weiszfeld, iters passes from the K19 median, smoothing nu; dmask [P]
// uint8 or null: the entries in the distances) of the same participants into theta, server step as K19.  scratch holds
// geomed_scratch_bytes(C, M, P) bytes (8-byte aligned).  -2: C too large for the staging tile
long long geomed_scratch_bytes(int C, int M, long long P);
int geomed_aggregate_launch(float* theta, long long t_stride, const float* cp, const float* n, int C, int M, long long P, int iters,
                            double nu, const unsigned char* dmask, int opt_kind, float lr, float momentum, float b1, float b2,
                            float eps, float* s0, float* s1, const int* steps, const unsigned char* mask, void* scratch,
                            cudaStream_t stream);
// robust_agg.cu (K21): Multi-Krum (f assumed Byzantine uploads per slot, the mkeep best-scored uploads averaged; dmask [P]
// uint8 or null: the entries in the distances) of the same participants into theta, server step as K19.  scratch holds
// krum_scratch_bytes(C, M, P) bytes (8-byte aligned).  -2: C too large for the shared-memory staging
long long krum_scratch_bytes(int C, int M, long long P);
int krum_aggregate_launch(float* theta, long long t_stride, const float* cp, const float* n, int C, int M, long long P, int f,
                          int mkeep, const unsigned char* dmask, int opt_kind, float lr, float momentum, float b1, float b2,
                          float eps, float* s0, float* s1, const int* steps, const unsigned char* mask, void* scratch,
                          cudaStream_t stream);
// robust_agg.cu (K23): centered clipping (iters clipping steps around center [M, P], the slots' previous outputs, radius
// tau = fl32(τ) widened; dmask [P] uint8 or null: the entries in the distances) of the same participants into theta (θ + v)
// and center (v), server step as K19.  scratch holds cclip_scratch_bytes(C, M, P) bytes (8-byte aligned).  -2: C too large
// for the staging tile
long long cclip_scratch_bytes(int C, int M, long long P);
int cclip_aggregate_launch(float* theta, long long t_stride, const float* cp, const float* n, float* center, int C, int M,
                           long long P, int iters, double tau, const unsigned char* dmask, int opt_kind, float lr, float momentum,
                           float b1, float b2, float eps, float* s0, float* s1, const int* steps, const unsigned char* mask,
                           void* scratch, cudaStream_t stream);
// attack.cu (K22): simulated Byzantine clients of rows [C, M, P] against theta + m·t_stride: every attacker pair
// (attackers[c] != 0, n[c·M + m] > 0) uploads the kind's poisoned value (1 sign_flip, 2 gaussian with gauss_hash(seed,
// c·M + m, e), 3 alie, 4 ipm; scale s > 0) on the entries with mask != 0 (mask may be nullptr).  -5: bad kind or scale
int attack_slots_launch(float* rows, const float* theta, long long t_stride, int C, int M, long long P, const float* n,
                        const unsigned char* attackers, int kind, float scale, const unsigned char* mask, unsigned seed,
                        cudaStream_t stream);
// aggregate_peer.cu : multi-GPU reduce-scatter + apply + all-gather over NVLink peer memory (cooperative launch)
int fedavg_reduce_apply_peer_launch(const float* cp, const int* cidx, const float* n, int C, int M, int P, int theta_stride, int world, int rank,
                                    const long long* part_ptrs, const long long* theta_ptrs, const long long* tot_ptrs,
                                    const long long* flag_ptrs, long long mc_part, long long mc_theta, unsigned* grid_sync, unsigned* chunk_done,
                                    int max_chunks, unsigned launch_idx, unsigned epoch, unsigned grid_base, int grid, long long timeout_ms,
                                    int* error_flag, cudaStream_t stream);
// eval.cu
int eval_logits_launch(const float* logits, const int* target, int B, int K, float* acc3, cudaStream_t stream);
int aue_sqerr_launch(const float* logits, const int* target, int B, int K, float* out1, cudaStream_t stream);
int ensemble_vote_launch(const int* preds, const float* w, int Kmodels, int B, int classes, int* out, cudaStream_t stream);
int confusion_matrix_launch(const int* pred, const int* target, int B, int classes, int* out, cudaStream_t stream);
// optim.cu
// FedProx anchor of the row optimizers (anchor == nullptr: off): row r's gradient becomes g + mu·mask⊙(w − anchor row
// rows[r]); anchor is [A, astride ≥ P] with unit column stride, mask a [P] uint8 entry mask or nullptr (every entry)
struct ProxAnchor {
    float mu;
    const float* anchor;
    long long astride;
    const int* rows;
    const unsigned char* mask;
};
// with a prox anchor, g is overwritten by the effective gradient
int adam_amsgrad_rows_launch(float* p, float* g, float* m, float* v, float* vmax, int* steps, const unsigned char* row_mask, int R,
                             long long P, float lr, float wd, float b1, float b2, float eps, const ProxAnchor& prox, cudaStream_t stream);
int sgd_rows_launch(float* p, const float* g, long long n, float lr, float wd, cudaStream_t stream);
// rows [R, P]: rows with row_mask[r] == 0 are skipped
int sgd_rows_masked_launch(float* p, const float* g, const unsigned char* row_mask, int R, long long P, float lr, float wd,
                           const ProxAnchor& prox, cudaStream_t stream);
// cluster_ops.cu
long long gram_workspace_doubles();
int gram_launch(const float* U, int n, long long P, double eps, double* S, double* nrm, double* part, cudaStream_t stream);
// mpc.cu
int modp_matmul_launch(const long long* A, const long long* B, long long* C, int M, int K, int N, long long p, cudaStream_t stream);
// misc.cu
int kd_kl_launch(const float* s, const float* t, int B, int K, float T, float* loss1, float* grad_s, cudaStream_t stream);
int vfl_bce_launch(const float* parts, const float* y, int K, int B, float* loss1, float* grad, cudaStream_t stream);
int group_norm_fwd_launch(const float* x, float* y, const float* w, const float* b, int N, int C, int HW, int G, float eps,
                          cudaStream_t stream, float* mean_out = nullptr, float* rstd_out = nullptr);
int bn_nhwc_fwd_launch(const float* x, const float* w, const float* b, float* y, float* mean, float* rstd, float* run_mean, float* run_var,
                       float* sums, long long rows, int C, float eps, float momentum, cudaStream_t stream);
int bn_nhwc_bwd_launch(const float* x, const float* dy, const float* w, const float* mean, const float* rstd, float* dx, float* dw, float* db,
                       float* sums, long long rows, int C, cudaStream_t stream);
int group_norm_bwd_launch(const float* x, const float* dy, const float* w, const float* mean, const float* rstd, float* dx, float* dg_part,
                          float* db_part, int N, int C, int HW, int G, cudaStream_t stream);
// gemm_tc.cu : D[M,N] (fp32 or bf16) = act(A[M,K] · B[N,K]^T + bias[N]); A,B bf16 row-major (K contiguous)
int gemm_split_count(int M, int N, int K);
int gemm_launch(const void* A, const void* B, void* D, const float* bias, int M, int N, int K, int a_mn, int b_mn, int relu, int out_fp32,
                cudaStream_t stream, float* splitk_ws = nullptr);
int gemm_batched_mn_launch(const void* A, const void* B, float* D, int M, int N, int K, int batch, int a_rows_total, int b_rows_total,
                           int a_k0, int a_kstride, int b_k0, int b_kstride, cudaStream_t stream);
int gemm_tn_launch(const void* A, const void* B, void* D, const float* bias, int M, int N, int K, int relu, int out_fp32,
                   cudaStream_t stream);
// conv_igemm.cu : implicit-GEMM convolution on wgmma (forward / dgrad / wgrad), NHWC fp32 activations
struct ConvArgs {
    const float* x;        // NHWC input of the gather: [N, H, W, C]   (forward: activations; dgrad: dY; wgrad: activations)
    const __nv_bfloat16* wq;   // packed bf16 weights [Kout][R][S][C] (forward / dgrad)
    const float* bias;     // [Kout] or nullptr (forward)
    float* y;              // [N, P, Q, Kout] output of forward / dgrad
    const float* dy;       // wgrad: [N·P·Q, Kout]
    float* dw;             // wgrad: fp32 gradient to add into — OIHW [Kout][C][R][S] (mode 0) or [Kout][R][S][C] (mode 1)
    int N, H, W, C, Kout, R, S, P, Q, pad_h, pad_w, stride, mode, relu;
};
int make_kmajor_sw128_map(void* map_out /* CUtensorMap* */, const void* base, int rows, int cols, int box_rows);   // gemm_tc.cu
int conv_igemm_launch(const ConvArgs& a, cudaStream_t stream);
int conv_wgrad_launch(const ConvArgs& a, cudaStream_t stream);
int conv_cast_bf16_launch(const float* x, const float* gate, void* out, long long n, cudaStream_t stream);
int conv_pack_t_launch(const void* wq, void* out, int K, int C, int RS, cudaStream_t stream);
// gemm_tc.cu: implicit-GEMM convolution on the GEMM mainloop with a TMA-im2col producer (bf16 NHWC operands)
int conv_tma_fwd_launch(const void* xb, const void* wq, float* y, const float* bias, int N, int H, int W, int C, int Cout, int R, int S, int P,
                        int Q, int pad, int stride, int dgrad, int relu, int groups, cudaStream_t stream);
int conv_tma_wgrad_launch(const void* xb, const void* dyb, float* dw_ohwi, int N, int H, int W, int C, int Cout, int R, int S, int P, int Q,
                          int pad, int stride, int groups, long long gstride, cudaStream_t stream);
int conv_cast_rows_bf16_launch(const float* x, long long row_stride, void* out, int rows, long long n, cudaStream_t stream);
// lstm_tc.cu : persistent cluster-resident 2-layer LSTM(256) forward / BPTT over many (client, model) pairs per launch
struct LstmArgs {
    const float* params;          // parameter arena base
    const long long* row_off;     // [npairs] element offset of each pair's flat parameter row
    long long off_emb, off_wih1, off_whh1, off_bih1, off_bhh1, off_wih2, off_whh2, off_bih2, off_bhh2;   // offsets inside a row
    const int* tokens;            // [npairs, 16, T] int32 token ids (rows beyond the real batch are padding)
    float* gates;                 // [2, npairs, T, 16, 4, 256] activated gates (i, f, g, o); nullptr = inference (no history)
    float* cst;                   // [2, npairs, T, 16, 256]    cell states
    void* hhist;                  // [2, npairs, T+1, 16, 256]  bf16 hidden states, index 0 = h_{-1} = 0; nullptr = not kept
    float* hlast;                 // [npairs, 16, 256]          fp32 h2_{T-1}
    // backward only
    const float* dh2_last;        // [npairs, 16, 256] gradient wrt h2_{T-1}            (used when dh2_all == nullptr)
    const float* dh2_all;         // [npairs, T, 16, 256] gradient wrt every h2_t, or nullptr
    void* dgates;                 // [2, npairs, T, 16, 1024] bf16 pre-activation gate gradients (PyTorch row order)
    int T, E;
};
struct LstmHeadArgs {
    const float* params;          // parameter arena base
    const long long* row_off;     // [nchunks] element offset of each chunk's parameter row
    long long off_fcw, off_fcb;   // fc.weight [V, 256] / fc.bias [V] offsets inside a row
    const float* hlast;           // [nchunks, 16, 256]
    const int* labels;            // [nchunks, 16]  (-1 = padding row)
    const float* scale;           // [nchunks] 1 / (#real rows of the chunk's pair)
    float* dh;                    // [nchunks, 16, 256]  d loss / d h2_{T-1}
    float* dW;                    // [nchunks, V, 256]
    float* db;                    // [nchunks, V]
    float* loss;                  // [nchunks] or nullptr
    int V;
};
int lstm_head_launch(const LstmHeadArgs& a, int nchunks, cudaStream_t stream);
struct LstmSmallArgs {
    const float* params;          // parameter arena base
    const long long* row_off;     // [nchunks]
    long long off_emb, off_wih1;
    const int* tokens;            // [nchunks, 16, T]
    const void* dgates;           // [2, nchunks, T, 16, 1024] bf16
    float* db1;                   // [nchunks, 1024]
    float* db2;                   // [nchunks, 1024]
    float* dwih1;                 // [nchunks, 1024, E]
    float* demb_part;             // [nchunks, 8, V, E]  (summed over the 8 column slices by the caller)
    int T, E, V;
};
int lstm_small_grads_launch(const LstmSmallArgs& a, int nchunks, cudaStream_t stream);
int lstm2_fwd_launch(const LstmArgs& a, int npairs, cudaStream_t stream);
int lstm2_bwd_launch(const LstmArgs& a, int npairs, cudaStream_t stream);
}  // namespace fdb
