// Shared device helpers for the feddrift_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#define FDB_HOST_DEVICE __host__ __device__ __forceinline__
#define FDB_DEVICE __device__ __forceinline__

namespace fdb {

// ---------------------------------------------------------------- counter-based RNG (same as ops/reference.py)
FDB_HOST_DEVICE uint32_t mix32(uint32_t x) {
    x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
    return x;
}
FDB_HOST_DEVICE uint32_t batch_hash(uint32_t seed, uint32_t rnd, uint32_t client, uint32_t model, uint32_t step) {
    uint32_t h = mix32(seed + 0x9E3779B9u * (rnd + 1u));
    h = mix32(h ^ (client * 0x85EBCA6Bu + 0x165667B1u));
    h = mix32(h ^ (model * 0xC2B2AE35u + 0x27D4EB2Fu));
    h = mix32(h ^ (step * 0x2545F491u + 1u));
    return h;
}
FDB_DEVICE uint32_t hash_choice(uint32_t h, uint32_t n) { return __umulhi(h, n); }
// counter-based N(0,1): Box–Muller on two lowbias32 hashes of (seed, row, element) — same function in ops/reference.py
FDB_DEVICE float gauss_hash(uint32_t seed, uint32_t r, unsigned long long i) {
    const uint32_t base = mix32(seed ^ mix32(r * 0x9E3779B9u + 0x7F4A7C15u)) ^ (uint32_t)(i >> 32) * 0x85EBCA6Bu;
    const uint32_t h1 = mix32(base ^ ((uint32_t)i * 2u + 1u));
    const uint32_t h2 = mix32(base ^ ((uint32_t)i * 2u + 2u) ^ 0x68E31DA4u);
    const float u1 = ((float)(h1 >> 8) + 1.0f) * (1.0f / 16777216.0f);   // (0, 1]
    const float u2 = (float)(h2 >> 8) * (1.0f / 16777216.0f);            // [0, 1)
    return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}
// gauss_hash seed of the weak-DP noise of round `rnd` of a time step whose engine seed is `seed` (ops/reference.py
// defense_seed); the noise of (client c, slot m) is gauss_hash(defense_seed(seed, rnd), c·M + m, element)
FDB_HOST_DEVICE uint32_t defense_seed(uint32_t seed, uint32_t rnd) { return mix32(seed ^ mix32(rnd * 0xC2B2AE35u + 0x2545F491u)); }
// counter-based U[0, 1): (h >> 8)·2⁻²⁴ with h the first lowbias32 hash of gauss_hash for (seed, row, element) — same
// function as uniform_hash in ops/reference.py
FDB_HOST_DEVICE float uniform_hash(uint32_t seed, uint32_t r, unsigned long long i) {
    const uint32_t base = mix32(seed ^ mix32(r * 0x9E3779B9u + 0x7F4A7C15u)) ^ (uint32_t)(i >> 32) * 0x85EBCA6Bu;
    return (float)(mix32(base ^ ((uint32_t)i * 2u + 1u)) >> 8) * (1.0f / 16777216.0f);
}
// uniform_hash seed of the QSGD draws of round `rnd` of a time step whose engine seed is `seed` (ops/reference.py
// compress_seed); its constants differ from defense_seed's so that quantization draws and weak-DP noise are independent
FDB_HOST_DEVICE uint32_t compress_seed(uint32_t seed, uint32_t rnd) { return mix32(seed ^ mix32(rnd * 0x27D4EB2Fu + 0x165667B1u)); }
// gauss_hash seed of the gaussian model-poisoning attack of round `rnd` (ops/reference.py attack_seed); constants distinct
// from defense_seed's and compress_seed's
FDB_HOST_DEVICE uint32_t attack_seed(uint32_t seed, uint32_t rnd) { return mix32(seed ^ mix32(rnd * 0x85EBCA77u + 0x3C6EF372u)); }
// attack kinds (ops/reference.py ATTACK_ID) and the upload an elementwise attacker sends for one trainable entry x with
// round-start model th (sign_flip: th − s·(x − th); gaussian: th + s·xi), every operation rounded on its own
constexpr int kAttackNone = 0, kAttackSignFlip = 1, kAttackGaussian = 2, kAttackAlie = 3, kAttackIpm = 4;
FDB_DEVICE float attack_entry(int kind, float x, float th, float s, uint32_t seed, uint32_t r, unsigned long long e) {
    return kind == kAttackSignFlip ? __fsub_rn(th, __fmul_rn(s, __fsub_rn(x, th)))
                                   : __fadd_rn(th, __fmul_rn(s, gauss_hash(seed, r, e)));
}
// QSGD of one trainable entry x with anchor th, bucket scale sigma > 0, level s and uniform draw u (ops/reference.py
// qsgd_slots_): a = (|d| / σ)·s, q = floor(a) + (u < frac(a)), x' = th + copysign(σ·(q / s), d) with d = x − th.  Every
// operation is rounded on its own (no FMA contraction), so the result matches the CPU oracle bit for bit.
FDB_DEVICE float qsgd_entry(float x, float th, float sigma, float s, float u) {
    const float d = __fsub_rn(x, th);
    const float a = __fmul_rn(__fdiv_rn(fabsf(d), sigma), s);
    const float l = floorf(a);
    const float q = (u < __fsub_rn(a, l)) ? __fadd_rn(l, 1.f) : l;
    return __fadd_rn(th, copysignf(__fmul_rn(sigma, __fdiv_rn(q, s)), d));
}
// top-k with error feedback (ops/reference.py eftopk_slots_): the error-corrected update v = (x − th) + e of one trainable
// entry, each operation rounded on its own, and its selection key, the bit pattern of |v| (a total order with the index)
FDB_DEVICE float eftopk_value(float x, float th, float e) { return __fadd_rn(__fsub_rn(x, th), e); }
FDB_DEVICE unsigned eftopk_key(float v) { return __float_as_uint(v) & 0x7FFFFFFFu; }

// ---------------------------------------------------------------- warp reductions
FDB_DEVICE float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
FDB_DEVICE double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
FDB_DEVICE float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// block-wide sum (blockDim.x multiple of 32, <= 1024); result valid in every thread
template <typename T>
FDB_DEVICE T block_sum(T v, T* smem /* >= 32 entries */) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) smem[warp] = v;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    T r = (lane < nw) ? smem[lane] : T(0);
    r = warp_sum(r);
    return r;
}

// ---------------------------------------------------------------- cross-GPU flag helpers (system scope)
FDB_DEVICE void st_release_sys(unsigned* p, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
FDB_DEVICE unsigned ld_acquire_sys(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
FDB_DEVICE void st_relaxed_sys_f32(float* p, float v) {
    asm volatile("st.relaxed.sys.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
FDB_DEVICE float ld_relaxed_sys_f32(const float* p) {
    float v;
    asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
    return v;
}
// LL ("low latency") words: payload and epoch tag travel in ONE 8- or 16-byte store, so the receiver needs neither a
// fence nor a separate flag — it polls the word until the tag matches.  (8-byte stores are single-copy atomic; the 16-byte
// variant carries the tag twice and the reader checks both halves, as NCCL's LL lines do.)
FDB_DEVICE void st_ll(uint2* p, float v, unsigned tag) {
    asm volatile("st.relaxed.sys.global.v2.b32 [%0], {%1, %2};" ::"l"(p), "r"(__float_as_uint(v)), "r"(tag) : "memory");
}
FDB_DEVICE uint2 ld_ll(const uint2* p) {
    uint2 w;
    asm volatile("ld.relaxed.sys.global.v2.b32 {%0, %1}, [%2];" : "=r"(w.x), "=r"(w.y) : "l"(p) : "memory");
    return w;
}
FDB_DEVICE void st_ll2(uint4* p, float a, float b, unsigned tag) {
    asm volatile("st.relaxed.sys.global.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(__float_as_uint(a)), "r"(tag),
                 "r"(__float_as_uint(b)), "r"(tag) : "memory");
}
FDB_DEVICE uint4 ld_ll2(const uint4* p) {
    uint4 w;
    asm volatile("ld.relaxed.sys.global.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(w.x), "=r"(w.y), "=r"(w.z), "=r"(w.w) : "l"(p) : "memory");
    return w;
}
FDB_DEVICE long long globaltimer_ns() {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// Bounded spinning without a timer read on the fast path: %globaltimer is a slow, chip-level register — reading it before and
// inside every wait put hundreds of cycles on each hop of the mbarrier / flag handshake chains of the pipelined kernels).  The guard looks at the timer only every 256 failed polls; the first look
// starts the clock.
struct SpinGuard {
    long long t0 = 0;
    unsigned n = 0;
    FDB_DEVICE bool expired(long long timeout_ns) {
        if ((++n & 255u) != 0) return false;
        const long long now = globaltimer_ns();
        if (t0 == 0) { t0 = now; return false; }
        return now - t0 > timeout_ns;
    }
};

// ---------------------------------------------------------------- FedOpt server step (K11), one entry
// g = th - avg is the pseudo-gradient; returns the stepped entry.  kind 1 sgd (+momentum), 2 adam, 3 adagrad, 4 yogi;
// s0[idx] / s1[idx] are the entry's state (sgd: momentum buffer, adagrad: sum of squares, adam / yogi: first / second
// moment) and are only touched by the kinds that own them; bc1 = 1 - β1^t, bc2 = 1 - β2^t are Adam's bias corrections.
// Same update law as ops.reference.server_opt_step_.
FDB_DEVICE float server_opt_update(int kind, float th, float avg, float* s0, float* s1, size_t idx, float lr, float momentum,
                                   float b1, float b2, float eps, float bc1, float bc2) {
    const float g = th - avg;
    if (kind == 1) {
        float gg = g;
        if (momentum != 0.f) { gg = s0[idx] * momentum + g; s0[idx] = gg; }
        th -= lr * gg;
    } else if (kind == 2) {
        const float mm = s0[idx] * b1 + (1.f - b1) * g;
        const float vv = s1[idx] * b2 + (1.f - b2) * g * g;
        s0[idx] = mm; s1[idx] = vv;
        th -= (lr / bc1) * mm / (sqrtf(vv) / sqrtf(bc2) + eps);
    } else if (kind == 3) {
        const float ss = s0[idx] + g * g;
        s0[idx] = ss;
        th -= lr * g / (sqrtf(ss) + eps);
    } else {
        const float mm = s0[idx] * b1 + (1.f - b1) * g;
        const float g2 = g * g, vo = s1[idx];
        const float sg = (vo - g2 > 0.f) ? 1.f : ((vo - g2 < 0.f) ? -1.f : 0.f);
        const float vv = vo - (1.f - b2) * sg * g2;
        s0[idx] = mm; s1[idx] = vv;
        th -= lr * mm / (sqrtf(vv) + eps);
    }
    return th;
}

}  // namespace fdb
