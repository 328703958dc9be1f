// K18: top-k sparsification with error feedback of the client uploads of a [C, M, P] arena against their slots' models.
//
// Row r of rows [R, P] (R = C·M, row r = (c, m) with m = r % M) and its residual row res[r] are updated in place against
// θ_m = theta + m·t_stride (a padded ModelBank row stride is fine); rows whose weight n[r] is not > 0 are skipped.  Over
// the trainable entries (mask byte != 0) v = (x − θ) + e and key = bits(|v|) as uint32; the k entries with the largest keys
// are kept (ties to the lower flat index), see ops/reference.py eftopk_slots_.  The selection is a radix select:
//   1. three histogram passes over the 11 / 11 / 10-bit digits of the key, each restricted to the entries that match the
//      digits fixed so far.  A CTA counts into a shared-memory histogram, then adds its non-zero bins into [3, R, 2048]
//      with integer atomics: the sums do not depend on the order of the updates, so the result is deterministic.  After
//      each pass a one-CTA-per-row kernel walks the bins from the top and fixes the digit and the count still to take.
//      The threshold T is then the full key and `rem` the number of entries with key == T to keep.
//   2. when fewer than all entries with key == T are kept, a tie pass counts them per chunk of kChunk entries and one CTA
//      per row turns the counts into exclusive prefixes (the index-order rank of each chunk's first tie).
//   3. the apply pass keeps key > T plus the first `rem` entries with key == T (block scan inside the chunk), writes
//      x + e (x when e == 0) and e = 0 for the kept entries, θ and e = v for the others.
// Every pass recomputes v from (x, θ, e); each thread owns groups of 4 consecutive entries, read and written with 128-bit
// accesses when the rows, residual, anchor and mask are 16/16/16/4-byte aligned.  When k is at least the trainable count
// every entry is kept and the selection passes are skipped.  In-row indices are 32-bit (the binding caps P below 2³¹).
#include "common.cuh"
#include "kernels.h"

namespace fdb {

namespace {

constexpr int kThreads = 256;
constexpr unsigned kChunk = 4u * kThreads;   // entries per chunk of the tie and apply passes
constexpr int kBins = 2048;
constexpr int kScanThreads = 1024;
// per-row state words: threshold prefix, count still to take among the entries matching it, tie flag, keep-all flag
enum { kPrefix = 0, kRem = 1, kTie = 2, kAll = 3, kStateWords = 4 };

inline int eftopk_grid_x(long long groups, int R) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long need = (groups + kThreads - 1) / kThreads, cap = (long long)sms * 8;
    return (int)max(1LL, min(need, cap) / max(1, min(R, 16)));
}

FDB_DEVICE int digit_shift(int pass) { return pass == 0 ? 21 : (pass == 1 ? 10 : 0); }
FDB_DEVICE unsigned digit_bins(int pass) { return pass == 2 ? 1024u : 2048u; }

// the 4 entries of group g: row value, anchor, residual and whether the entry is trainable (and inside the row)
template <bool kVec>
FDB_DEVICE void load4(const float* __restrict__ x, const float* __restrict__ th, const float* __restrict__ e,
                      const unsigned char* __restrict__ mask, unsigned i0, unsigned P, float xv[4], float tv[4], float ev[4],
                      bool on[4]) {
    if (kVec) {
        const float4 a = *reinterpret_cast<const float4*>(x + i0), t = *reinterpret_cast<const float4*>(th + i0),
                     r = *reinterpret_cast<const float4*>(e + i0);
        xv[0] = a.x; xv[1] = a.y; xv[2] = a.z; xv[3] = a.w;
        tv[0] = t.x; tv[1] = t.y; tv[2] = t.z; tv[3] = t.w;
        ev[0] = r.x; ev[1] = r.y; ev[2] = r.z; ev[3] = r.w;
        if (mask) {
            const uchar4 mk = *reinterpret_cast<const uchar4*>(mask + i0);
            on[0] = mk.x; on[1] = mk.y; on[2] = mk.z; on[3] = mk.w;
        } else {
            on[0] = on[1] = on[2] = on[3] = true;
        }
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const unsigned i = i0 + j;
            on[j] = i < P && (!mask || mask[i]);
            xv[j] = i < P ? x[i] : 0.f;
            tv[j] = i < P ? th[i] : 0.f;
            ev[j] = i < P ? e[i] : 0.f;
        }
    }
}

template <bool kVec>
__global__ void __launch_bounds__(kThreads) eftopk_hist_kernel(const float* __restrict__ rows, const float* __restrict__ theta,
                                                               long long t_stride, int M, const float* __restrict__ res,
                                                               const float* __restrict__ n, const unsigned char* __restrict__ mask,
                                                               unsigned P, int R, int pass, const unsigned* __restrict__ state,
                                                               unsigned* __restrict__ hist) {
    __shared__ unsigned sh[kBins];
    const int r = blockIdx.y;
    if (n && !(n[r] > 0.f)) return;
    const unsigned* s = state + (size_t)r * kStateWords;
    if (pass > 0 && s[kAll]) return;
    const int shift = digit_shift(pass);
    const unsigned nbins = digit_bins(pass);
    const int hs = shift + (pass == 2 ? 10 : 11);   // the digits above this one must equal the prefix fixed so far
    const unsigned prefix = pass == 0 ? 0u : s[kPrefix];
    for (unsigned b = threadIdx.x; b < nbins; b += blockDim.x) sh[b] = 0u;
    __syncthreads();
    const float* x = rows + (size_t)r * P;
    const float* e = res + (size_t)r * P;
    const float* th = theta + (size_t)(r % M) * t_stride;
    const unsigned groups = (P + 3u) / 4u;
    for (unsigned g = blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += gridDim.x * blockDim.x) {
        float xv[4], tv[4], ev[4];
        bool on[4];
        load4<kVec>(x, th, e, mask, g * 4u, P, xv, tv, ev, on);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (!on[j]) continue;
            const unsigned key = eftopk_key(eftopk_value(xv[j], tv[j], ev[j]));
            if (pass == 0 || (key >> hs) == (prefix >> hs)) atomicAdd(&sh[(key >> shift) & (nbins - 1u)], 1u);
        }
    }
    __syncthreads();
    unsigned* h = hist + ((size_t)pass * R + r) * kBins;
    for (unsigned b = threadIdx.x; b < nbins; b += blockDim.x)
        if (sh[b]) atomicAdd(h + b, sh[b]);
}

// one CTA per row: fix this pass's digit.  Thread t owns the bins [nbins − (t+1)·per, nbins − t·per), walked from the top.
__global__ void __launch_bounds__(kThreads) eftopk_select_kernel(const float* __restrict__ n, int R, int pass, unsigned k,
                                                                 const unsigned* __restrict__ hist, unsigned* __restrict__ state) {
    __shared__ unsigned sc[kThreads];
    const int r = blockIdx.x, tid = threadIdx.x;
    if (n && !(n[r] > 0.f)) return;
    unsigned* s = state + (size_t)r * kStateWords;
    if (pass > 0 && s[kAll]) return;
    const unsigned* h = hist + ((size_t)pass * R + r) * kBins;
    const unsigned nbins = digit_bins(pass), per = nbins / kThreads, hi = nbins - tid * per;
    const unsigned want = pass == 0 ? k : s[kRem];   // read before the scan's barriers: one thread rewrites it below
    unsigned tot = 0;
    for (unsigned q = 1; q <= per; ++q) tot += h[hi - q];
    sc[tid] = tot;
    __syncthreads();
    for (int o = 1; o < kThreads; o <<= 1) {   // inclusive scan over the threads, highest bins first
        const unsigned v = tid >= o ? sc[tid - o] : 0u;
        __syncthreads();
        sc[tid] += v;
        __syncthreads();
    }
    const unsigned incl = sc[tid], excl = incl - tot;
    if (pass == 0 && k >= sc[kThreads - 1]) {   // k covers every trainable entry: keep them all
        if (tid == 0) s[kAll] = 1u;
        return;
    }
    if (!(excl < want && want <= incl)) return;
    unsigned cum = excl;
    for (unsigned q = 1; q <= per; ++q) {
        const unsigned b = hi - q, c = h[b];
        if (cum + c >= want) {
            const int shift = digit_shift(pass);
            s[kPrefix] = (pass == 0 ? 0u : s[kPrefix]) | (b << shift);
            s[kRem] = want - cum;
            if (pass == 2) s[kTie] = (want - cum) < c ? 1u : 0u;
            return;
        }
        cum += c;
    }
}

template <bool kVec>
__global__ void __launch_bounds__(kThreads) eftopk_tie_count_kernel(const float* __restrict__ rows, const float* __restrict__ theta,
                                                                    long long t_stride, int M, const float* __restrict__ res,
                                                                    const float* __restrict__ n, const unsigned char* __restrict__ mask,
                                                                    unsigned P, unsigned nch, const unsigned* __restrict__ state,
                                                                    unsigned* __restrict__ cnt) {
    __shared__ unsigned wsum[kThreads / 32];
    const int r = blockIdx.y, tid = threadIdx.x;
    if (n && !(n[r] > 0.f)) return;
    const unsigned* s = state + (size_t)r * kStateWords;
    if (s[kAll] || !s[kTie]) return;
    const unsigned T = s[kPrefix];
    const float* x = rows + (size_t)r * P;
    const float* e = res + (size_t)r * P;
    const float* th = theta + (size_t)(r % M) * t_stride;
    for (unsigned ch = blockIdx.x; ch < nch; ch += gridDim.x) {
        const unsigned i0 = ch * kChunk + tid * 4u;
        unsigned c = 0;
        if (i0 < P) {
            float xv[4], tv[4], ev[4];
            bool on[4];
            load4<kVec>(x, th, e, mask, i0, P, xv, tv, ev, on);
#pragma unroll
            for (int j = 0; j < 4; ++j) c += (on[j] && eftopk_key(eftopk_value(xv[j], tv[j], ev[j])) == T) ? 1u : 0u;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if ((tid & 31) == 0) wsum[tid >> 5] = c;
        __syncthreads();
        if (tid == 0) {
            unsigned t = 0;
            for (int w = 0; w < kThreads / 32; ++w) t += wsum[w];
            cnt[(size_t)r * nch + ch] = t;
        }
        __syncthreads();
    }
}

// one CTA per row: chunk tie counts → exclusive prefixes, in place
__global__ void __launch_bounds__(kScanThreads) eftopk_tie_scan_kernel(const float* __restrict__ n, const unsigned* __restrict__ state,
                                                                       unsigned nch, unsigned* __restrict__ cnt) {
    __shared__ unsigned sc[kScanThreads];
    const int r = blockIdx.x, tid = threadIdx.x;
    if (n && !(n[r] > 0.f)) return;
    const unsigned* s = state + (size_t)r * kStateWords;
    if (s[kAll] || !s[kTie]) return;
    unsigned* c = cnt + (size_t)r * nch;
    const unsigned per = (nch + kScanThreads - 1) / kScanThreads, lo = min(nch, tid * per), hi = min(nch, lo + per);
    unsigned sum = 0;
    for (unsigned i = lo; i < hi; ++i) sum += c[i];
    sc[tid] = sum;
    __syncthreads();
    for (int o = 1; o < kScanThreads; o <<= 1) {
        const unsigned v = tid >= o ? sc[tid - o] : 0u;
        __syncthreads();
        sc[tid] += v;
        __syncthreads();
    }
    unsigned run = sc[tid] - sum;
    for (unsigned i = lo; i < hi; ++i) {
        const unsigned v = c[i];
        c[i] = run;
        run += v;
    }
}

template <bool kVec>
__global__ void __launch_bounds__(kThreads) eftopk_apply_kernel(float* __restrict__ rows, const float* __restrict__ theta,
                                                                long long t_stride, int M, float* __restrict__ res,
                                                                const float* __restrict__ n, const unsigned char* __restrict__ mask,
                                                                unsigned P, unsigned nch, int keep_all, const unsigned* __restrict__ state,
                                                                const unsigned* __restrict__ cnt) {
    __shared__ unsigned wsum[kThreads / 32];
    const int r = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (n && !(n[r] > 0.f)) return;
    const unsigned* s = state + (size_t)r * kStateWords;
    const bool all = keep_all || s[kAll];
    const bool tie = !all && s[kTie];
    const unsigned T = s[kPrefix], rem = s[kRem];
    float* x = rows + (size_t)r * P;
    float* e = res + (size_t)r * P;
    const float* th = theta + (size_t)(r % M) * t_stride;
    for (unsigned ch = blockIdx.x; ch < nch; ch += gridDim.x) {
        const unsigned i0 = ch * kChunk + tid * 4u;
        const bool in = i0 < P;
        float xv[4], tv[4], ev[4], v[4];
        unsigned key[4];
        bool on[4] = {false, false, false, false};
        unsigned eq = 0;
        if (in) {
            load4<kVec>(x, th, e, mask, i0, P, xv, tv, ev, on);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                v[j] = eftopk_value(xv[j], tv[j], ev[j]);
                key[j] = eftopk_key(v[j]);
                eq += (on[j] && key[j] == T) ? 1u : 0u;
            }
        }
        unsigned rank = 0;   // index-order rank among the row's ties of this thread's first tie
        if (tie) {
            unsigned inc = eq;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned u = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += u;
            }
            if (lane == 31) wsum[warp] = inc;
            __syncthreads();
            unsigned wbase = 0;
            for (int w = 0; w < warp; ++w) wbase += wsum[w];
            rank = cnt[(size_t)r * nch + ch] + wbase + inc - eq;
            __syncthreads();   // wsum is rewritten by the next chunk
        }
        if (!in) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (!on[j]) continue;
            const bool keep = all || key[j] > T || (key[j] == T && (!tie || rank++ < rem));
            if (keep) {
                if (ev[j] != 0.f) xv[j] = __fadd_rn(xv[j], ev[j]);
                ev[j] = 0.f;
            } else {
                xv[j] = tv[j];
                ev[j] = v[j];
            }
        }
        if (kVec) {
            *reinterpret_cast<float4*>(x + i0) = make_float4(xv[0], xv[1], xv[2], xv[3]);
            *reinterpret_cast<float4*>(e + i0) = make_float4(ev[0], ev[1], ev[2], ev[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (on[j]) { x[i0 + j] = xv[j]; e[i0 + j] = ev[j]; }
        }
    }
}

template <bool kVec>
void eftopk_run(float* rows, const float* theta, long long t_stride, int M, float* res, const float* n, const unsigned char* mask,
                int R, unsigned P, unsigned k, bool keep_all, unsigned* hist, unsigned* state, unsigned* cnt, cudaStream_t stream) {
    const unsigned groups = (P + 3u) / 4u, nch = (P + kChunk - 1) / kChunk;
    const dim3 grid(eftopk_grid_x(groups, R), R);
    if (!keep_all) {
        for (int pass = 0; pass < 3; ++pass) {
            eftopk_hist_kernel<kVec><<<grid, kThreads, 0, stream>>>(rows, theta, t_stride, M, res, n, mask, P, R, pass, state, hist);
            eftopk_select_kernel<<<R, kThreads, 0, stream>>>(n, R, pass, k, hist, state);
        }
        eftopk_tie_count_kernel<kVec><<<grid, kThreads, 0, stream>>>(rows, theta, t_stride, M, res, n, mask, P, nch, state, cnt);
        eftopk_tie_scan_kernel<<<R, kScanThreads, 0, stream>>>(n, state, nch, cnt);
    }
    eftopk_apply_kernel<kVec><<<grid, kThreads, 0, stream>>>(rows, theta, t_stride, M, res, n, mask, P, nch, keep_all ? 1 : 0,
                                                             state, cnt);
}

}  // namespace

long long eftopk_scratch_words(int R, long long P) {
    return (long long)R * (3 * kBins + kStateWords) + (long long)R * ((P + kChunk - 1) / kChunk);
}

int eftopk_slots_launch(float* rows, const float* theta, long long t_stride, int M, float* res, const float* n,
                        const unsigned char* mask, int R, long long P, long long k, unsigned* scratch, cudaStream_t stream) {
    if (R <= 0 || P <= 0) return 0;
    if (P >= (1LL << 31) || k < 1 || M < 1) return -5;
    const unsigned Pu = (unsigned)P, ku = (unsigned)min(k, P);
    unsigned* hist = scratch;
    unsigned* state = hist + (size_t)R * 3 * kBins;
    unsigned* cnt = state + (size_t)R * kStateWords;
    const bool keep_all = mask == nullptr && k >= P;   // every entry is trainable and kept: no selection
    if (!keep_all) cudaMemsetAsync(scratch, 0, (size_t)R * (3 * kBins + kStateWords) * sizeof(unsigned), stream);
    const bool vec = (P % 4 == 0) && (t_stride % 4 == 0) && ((reinterpret_cast<uintptr_t>(rows) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(res) & 15) == 0) && ((reinterpret_cast<uintptr_t>(theta) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(mask) & 3) == 0);
    if (vec) eftopk_run<true>(rows, theta, t_stride, M, res, n, mask, R, Pu, ku, keep_all, hist, state, cnt, stream);
    else eftopk_run<false>(rows, theta, t_stride, M, res, n, mask, R, Pu, ku, keep_all, hist, state, cnt, stream);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

}  // namespace fdb
