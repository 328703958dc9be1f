// Argument block of the fused persistent FL-round kernel (fed_round_small.cu).
#pragma once
#include <cuda_runtime.h>

namespace fdb {

constexpr int kMaxPeers = 8;

struct RoundParams {
    // data (device-resident for the whole experiment)
    const float* X;      // [T1, C, S, IN]
    const int* Y;        // [T1, C, S]
    const int* nsamp;    // [T1, C]
    // plan
    float* W;                  // [t_cur+1, M, C]   (rewritten in place by IFCA re-clustering)
    const int* train_index;    // [M, C, Lmax] flat (t'*S + s) sample ids   (sample_mode == 2)
    const int* train_count;    // [M, C]
    const float* feat_mask;    // [M, IN] or nullptr (training inputs only)
    const int* eval_train_model;  // [C] or nullptr (-1 → argmax_m W[t, m, c])
    const int* eval_test_model;   // [C] or nullptr
    const float* ens_w;        // [C, M] or nullptr
    const unsigned char* part; // [part_rows, C] client participation (row = round % part_rows) or nullptr: everyone trains
    int part_rows;
    // model / optimizer state
    float* theta;        // [M, theta_stride]
    float* opt_m;        // [C, M, P]
    float* opt_v;
    float* opt_vmax;
    int* opt_step;       // [C, M]
    // server optimizer on the cluster models (FedOpt per slot, sopt_kind 0 = plain FedAvg): after the weighted average
    // avg_m of a slot with total weight > 0, θ_m takes one step on g = θ_m − avg_m (common.cuh server_opt_update)
    int sopt_kind;       // 0 none, 1 sgd(+momentum), 2 adam, 3 adagrad, 4 yogi
    float sopt_lr, sopt_momentum, sopt_eps;
    float* sopt_s0;      // [M, P] momentum / Adagrad sum / first moment, or nullptr (sgd without momentum)
    float* sopt_s1;      // [M, P] second moment (adam / yogi) or nullptr
    int* sopt_step;      // [M] steps applied per slot (Adam bias correction), advanced by every round the slot aggregates
    // robust aggregation (def_bound 0 = off): each pair's upload x enters its slot's average as θ_m + s·(x − θ_m),
    // s = 1 / max(1, ‖x − θ_m‖ / def_bound), plus def_stddev·gauss_hash(defense_seed(seed, round), c·M + m, e) (weak DP)
    float def_bound, def_stddev;
    // FedProx (0 = off): every local step of pair (c, m) adds prox_mu·(w − θ_m) to the gradient, θ_m the round-start model
    float prox_mu;
    // QSGD upload compression (q_level 0 = off): each pair's local model is quantized against θ_m with level q_level and
    // bucket q_bucket (common.cuh qsgd_entry, draws uniform_hash(compress_seed(seed, round), c·M + m, e)) before client_out,
    // the defense and the average see it
    int q_level, q_bucket;
    // top-k with error feedback (topk_k 0 = off): each pair keeps its topk_k largest entries of v = (x − θ_m) + e, e its row
    // of ef_res [C, M, P] (common.cuh eftopk_value / eftopk_key, ties to the lower index), uploads θ elsewhere and carries
    // the rest in ef_res, before client_out, the defense and the average see it
    float* ef_res;
    int topk_k;
    // cluster aggregation rule (0 = weighted mean): 1 coordinate-wise median, 2 trimmed mean dropping
    // ⌊fl32(trim_ratio · n)⌋ values at each end, over the n uploads of a slot as published (after compression and the
    // defense), each counted once (ops/reference.py robust_aggregate_slots_); the server optimizer then steps on θ − it
    int agg_rule;
    float trim_ratio;
    // agg_rule 3: geometric median (ops/reference.py geomed_aggregate_slots_): gm_iters smoothed Weiszfeld steps from the
    // coordinate-wise median, weights 1 / max(gm_nu, distance)
    int gm_iters;
    double gm_nu;
    // agg_rule 4: Multi-Krum (ops/reference.py krum_aggregate_slots_): the average of the min(krum_m, n) uploads whose
    // summed squared distances to their clamp(n − krum_f − 2, 1, n − 1) nearest neighbours are smallest
    int krum_f, krum_m;
    // agg_rule 5: centered clipping (ops/reference.py cclip_aggregate_slots_): cc_iters clipping steps of radius cc_tau
    // (fl32(τ) widened) around the slot's center cc_center [M, P], its previous output, which the slot's owner CTA rewrites
    int cc_iters;
    double cc_tau;
    float* cc_center;
    // simulated Byzantine clients (attack_kind 0 = off, 1 sign_flip, 2 gaussian; ops/reference.py attack_slots_): after
    // compression, every pair of a client with attack_mask[c] != 0 uploads θ_m − s·(x − θ_m) or θ_m + s·gauss_hash(
    // attack_seed(seed, round), c·M + m, e) instead of x, s = attack_scale, before client_out, the defense and the rule
    int attack_kind;
    float attack_scale;
    const unsigned char* attack_mask;   // [C]
    float* client_out; // optional [C, M, P] export of the local models of the LAST round (nullptr = off)
    const float* lr_ptr; // optional device scalar overriding lr
    // outputs
    float* metrics;      // [rounds, C, 4]
    long long* timers;   // optional [rounds, 4] globaltimer ns stamps of CTA 0 (train end, agg end, eval end, -)
    int* counters;       // optional device counters {round_in_step, global_epoch}: read at start, advanced at exit
    // scalars
    float lr, wd, beta1, beta2, eps;
    int T1, C, S, M, Lmax, theta_stride;
    int batch_size, epochs, t_cur, rounds, round0;
    unsigned seed;
    int use_adam;       // 1 = Adam(amsgrad, L2 wd), 0 = SGD
    int sample_mode;    // 0 pool, 1 time-weighted, 2 explicit index lists
    int n_mode;         // 0 Σ W·nb, 1 Σ W·nsamp       (pool mode only)
    int recluster_hard; // IFCA: argmax re-clustering after every aggregation
    int ens_mode;       // 0 none, 1 weighted hard vote, 2 weighted soft vote (test metric)
    int skip_aggregate; // 1 = train + export only (CFL inspects raw updates)
    int warps_per_pair; // 1, 2 or 4 warps cooperate on one (client, model) pair
    // multi-GPU (clients sharded c % world == rank); world == 1 → everything local
    int world, rank;
    float* inbox[kMaxPeers];     // inbox[g]: this rank's view of peer g's symmetric inbox: LL words {value, epoch} [2, world, M*P] x 8 B
    float* metrics_peer[kMaxPeers];  // every rank's (symmetric) metrics STAGING area: LL words {corr, epoch, loss, epoch} [rounds, C, 2] x 16 B
    unsigned flag_base;          // monotonically increasing epoch base (per launch)
    long long spin_timeout_ns;   // bail out instead of hanging the GPU if a peer never arrives
    int* error_flag;             // set to nonzero on timeout
    // fused host I/O (single-GPU end-to-end round): the kernel itself performs the host→device copy of the round's inputs
    // from PINNED host memory (UVA pointers; 16-byte system-scope loads over PCIe) into the X / Y arenas before round 0,
    // and mirrors every metric row into a pinned host buffer — the whole round is ONE graph node, no memcpy nodes.
    const float* host_x;         // pinned [host_steps, C, S, IN] or nullptr
    const int* host_y;           // pinned [host_steps, C, S]
    float* host_metrics;         // pinned [rounds, C, 4] or nullptr
    int host_t0, host_steps;     // destination time steps [host_t0, host_t0 + host_steps)
};

struct SmallLaunchInfo {
    int threads, cluster, smem_bytes;
};

// returns 0 on success, -1 if (kind,in,hid,out) is not an instantiated shape
int fed_round_small_launch(int kind, int din, int hid, int dout, const RoundParams& p, int cluster, cudaStream_t stream,
                           SmallLaunchInfo* info);
int fed_round_small_supported(int kind, int din, int hid, int dout);
int fed_round_small_fits(int kind, int din, int hid, int dout, int C, int M, int t_cur, bool server_opt, int agg_rule,
                         int attack_kind);
int mlp_eval_matrix_launch(int kind, int din, int hid, int dout, const float* theta, int theta_stride, int M, const float* X,
                           const int* Y, const int* nsamp, int C, int S, float* correct, float* loss, float* sqerr,
                           cudaStream_t stream);

}  // namespace fdb
