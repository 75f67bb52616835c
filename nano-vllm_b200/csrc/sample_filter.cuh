// Top-k / top-p / min-p thresholds of the filtered sampler (sample_filter.cu: stages 0-3; sampler.cu: the masked race).
//
// The kept set of a row is {j : x_j >= tau} for one bf16 threshold tau = max(tau_min_p, tau_k, tau_p).  A bf16 logit has
// an order-preserving 16-bit key (key16 below), so tau is found exactly by a two-level radix select: a 256-bin histogram
// of the key's high byte, then a 256-bin histogram of the low byte inside one selected high-byte bin.  Counts are integers
// and probability masses exp((x - max) / t) are fixed point (round(mass * 2^32), uint64), so every sum is associative:
// it depends neither on CTA order nor on the split count, and a vocab-sharded run whose workspaces are all-reduced with
// SUM (MAX for the row maximum) reaches exactly the unsharded tau.  A token whose mass is below 2^-33 of the row
// maximum contributes 0; with at most 2^18 tokens per row the error of any partial mass is below 2^-15 of the maximum's
// mass, and the sums stay below 2^50.
//
// Workspace: FW_ROW_WORDS int64 words per row, row r at r * FW_ROW_WORDS (the layout is the same for every row count):
//   FW_MAX           stage 0, reduced with MAX: key16 of the row maximum
//   FW_TAU           written by the masked race: key16 of tau (0 = nothing filtered); never needs resetting
//   FW_S1 .. +512    stage 1, SUM: counts[256] then masses[256] of the high byte, over tokens >= tau_min_p
//   FW_S2 .. +512    stage 2, SUM: the same for the low byte inside the stage-2 bin
//   FW_S3 .. +512    stage 3, SUM: the same inside the stage-3 bin
// Every word but FW_TAU is zero when stage 0 starts; the race's last CTA of a row zeroes them again.
#pragma once
#include "sample_common.cuh"

namespace b200sample {

constexpr int FILTER_THREADS = 256;
constexpr int FW_MAX = 0, FW_TAU = 1, FW_S1 = 2, FW_S2 = FW_S1 + 512, FW_S3 = FW_S2 + 512;
constexpr int FW_ROW_WORDS = FW_S3 + 512;
constexpr int FILTER_MAX_VOCAB = 1 << 18;

// order-preserving key of a bf16 (given as the fp32 it widens to); -0 is folded onto +0 so equal values share a key
__device__ __forceinline__ uint32_t key16(float x) {
    uint32_t b = __float_as_uint(x) >> 16;
    if (b == 0x8000u) b = 0;
    return b ^ ((b & 0x8000u) ? 0xffffu : 0x8000u);
}
__device__ __forceinline__ float key16_value(uint32_t key) {
    const uint32_t b = key ^ ((key & 0x8000u) ? 0x8000u : 0xffffu);
    return __uint_as_float(b << 16);
}

// The filter parameters of one row; a row is active when it samples (t > 0) and some filter is on.
struct FilterRow {
    float t, inv_t, p, min_p;
    int k;
    bool k_on, p_on, mp_on, active;
    __device__ __forceinline__ FilterRow(const float* temperatures, const int32_t* top_k, const float* top_p,
                                         const float* min_p_arr, int row) {
        t = temperatures ? temperatures[row] : 0.f;
        inv_t = t > 0.f ? 1.f / t : 1.f;
        k = top_k ? top_k[row] : 0;
        p = top_p ? top_p[row] : 1.f;
        min_p = min_p_arr ? min_p_arr[row] : 0.f;
        k_on = k > 0;
        p_on = p < 1.f;
        mp_on = min_p > 0.f;
        active = (t > 0.f) && (k_on || p_on || mp_on);
    }
};

// mass exp((x - m) / t) of one token in fixed point (2^32 = the row maximum's mass)
__device__ __forceinline__ unsigned long long fixed_mass(float x, float m, float inv_t) {
    return __float2ull_rn(expf((x - m) * inv_t) * 4294967296.0f);
}

// smallest key whose value x satisfies x - m >= t * ln(min_p) in float64 (prob_x >= min_p * prob_max), never above the
// row maximum's key
__device__ __forceinline__ uint32_t min_p_key(uint32_t m_key, const FilterRow& f) {
    if (!f.mp_on) return 0;
    const double lnt = log((double)f.min_p) * (double)f.t, m = (double)key16_value(m_key);
    uint32_t lo = 0, hi = m_key;                                          // answer in [lo, hi]
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if ((double)key16_value(mid) - m >= lnt) hi = mid; else lo = mid + 1;
    }
    return lo;
}

// Suffix sums over one 256-bin (count, mass) histogram, plus a base: cnt[b] = base_c + sum_{b' >= b} counts[b'];
// cnt[256] = base_c (same for mass).  Block-uniform; FILTER_THREADS == 256, one bin per thread.
struct SuffixSums {
    unsigned long long cnt[257], mass[257];
};
struct ScanScratch {
    unsigned long long wc[FILTER_THREADS / 32], wm[FILTER_THREADS / 32];
};
__device__ __forceinline__ void suffix_scan256(const int64_t* hist, unsigned long long base_c, unsigned long long base_m,
                                               SuffixSums& s, ScanScratch& tmp) {
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int b = 255 - t;                                                // ascending t = descending bin
    unsigned long long c = (unsigned long long)__ldcg(hist + b), m = (unsigned long long)__ldcg(hist + 256 + b);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long oc = __shfl_up_sync(0xffffffffu, c, o), om = __shfl_up_sync(0xffffffffu, m, o);
        if (lane >= o) { c += oc; m += om; }
    }
    if (lane == 31) { tmp.wc[warp] = c; tmp.wm[warp] = m; }
    __syncthreads();
    for (int w = 0; w < warp; ++w) { c += tmp.wc[w]; m += tmp.wm[w]; }
    s.cnt[b] = c + base_c;
    s.mass[b] = m + base_m;
    if (t == 0) { s.cnt[256] = base_c; s.mass[256] = base_m; }
    __syncthreads();
}
// largest bin whose suffix count reaches k (the bin of the k-th largest key); -1 if none
__device__ __forceinline__ int bin_of_count(const SuffixSums& s, unsigned long long k) {
    return __syncthreads_count(s.cnt[threadIdx.x] >= k) - 1;
}
// largest bin whose (non-zero) suffix mass reaches target: where the top-p cumulative mass crosses p * Z
__device__ __forceinline__ int bin_of_mass(const SuffixSums& s, double target) {
    const unsigned long long v = s.mass[threadIdx.x];
    return __syncthreads_count(v > 0 && (double)v >= target) - 1;
}

// What one row's threshold search knows after `have` stages (1..4) have completed and been reduced: the bins stages 2 and
// 3 must histogram (-1 = none) and, once it is final, tau.  Every CTA of a row derives it from the workspace alone.
struct Plan {
    uint32_t m_key, tmp_key, tau;
    int bin2, bin3;
};
struct PlanSmem {
    SuffixSums coarse, fine;
    ScanScratch tmp;
};
__device__ __forceinline__ int clamp_bin(int b) { return b < 0 ? 0 : b; }

__device__ __forceinline__ Plan plan_row(const int64_t* w, const FilterRow& f, int have, PlanSmem& sm) {
    Plan P;
    P.m_key = (uint32_t)__ldcg(w + FW_MAX);
    P.tmp_key = min_p_key(P.m_key, f);
    P.tau = P.tmp_key;
    P.bin2 = P.bin3 = -1;
    if (have < 2) return P;
    suffix_scan256(w + FW_S1, 0, 0, sm.coarse, sm.tmp);
    // top-k is off when the candidates (tokens >= tau_min_p, over the whole reduced vocabulary) are not more than k
    const bool kk = f.k_on && sm.coarse.cnt[0] > (unsigned long long)f.k;
    unsigned long long cnt_above = 0, mass_above = 0;
    int bk = -1, bp = -1;
    double target = 0.0;
    if (kk) {
        bk = clamp_bin(bin_of_count(sm.coarse, (unsigned long long)f.k));
        cnt_above = sm.coarse.cnt[bk + 1];
        mass_above = sm.coarse.mass[bk + 1];
        P.bin2 = bk;
    } else if (f.p_on) {
        target = (double)f.p * (double)sm.coarse.mass[0];
        bp = clamp_bin(bin_of_mass(sm.coarse, target));
        mass_above = sm.coarse.mass[bp + 1];
        P.bin2 = bp;
    } else {
        return P;                                                     // min-p only: tau = tau_min_p
    }
    if (have < 3) return P;
    suffix_scan256(w + FW_S2, cnt_above, mass_above, sm.fine, sm.tmp);
    if (!kk) {                                                        // top-p crossed inside bin bp
        P.tau = ((uint32_t)bp << 8) | (uint32_t)clamp_bin(bin_of_mass(sm.fine, target));
        return P;
    }
    const int lk = clamp_bin(bin_of_count(sm.fine, (unsigned long long)f.k));
    P.tau = ((uint32_t)bk << 8) | (uint32_t)lk;                      // tau_k (>= tau_min_p by construction)
    if (!f.p_on) return P;
    target = (double)f.p * (double)sm.fine.mass[lk];                  // p * Z, Z = mass of the tokens >= tau_k
    bp = bin_of_mass(sm.coarse, target);                              // exact for bins above bk
    if (bp <= bk) {                                                   // crossed inside bk: stage 2 already has it
        P.tau = ((uint32_t)bk << 8) | (uint32_t)clamp_bin(bin_of_mass(sm.fine, target));
        return P;
    }
    P.bin3 = bp;
    if (have < 4) return P;
    suffix_scan256(w + FW_S3, 0, sm.coarse.mass[bp + 1], sm.fine, sm.tmp);
    P.tau = ((uint32_t)bp << 8) | (uint32_t)clamp_bin(bin_of_mass(sm.fine, target));
    return P;
}

// Vocabulary slice [lo, hi) of split `split` (8-aligned, as in sample_kernel) and the visit of its bf16 logits.
__device__ __forceinline__ void filter_slice(int vocab, int splits, int split, int& lo, int& hi) {
    const int per = (((vocab + splits - 1) / splits) + 7) & ~7;
    lo = split * per;
    hi = lo + per;
    hi = hi > vocab ? vocab : hi;
}
template <typename F>
__device__ __forceinline__ void for_each_logit(const __nv_bfloat16* rowp, int lo, int hi, F&& f) {
    const int v_lo = lo >> 3, v_hi = hi >> 3;
    const uint4* r4 = reinterpret_cast<const uint4*>(rowp);
    for (int vi = v_lo + threadIdx.x; vi < v_hi; vi += FILTER_THREADS) {
        float x[8];
        unpack8(r4[vi], x);
#pragma unroll
        for (int e = 0; e < 8; ++e) f(x[e], vi * 8 + e);
    }
    for (int i = (v_hi << 3) + threadIdx.x; i < hi; i += FILTER_THREADS)
        if (i >= lo) f(__bfloat162float(rowp[i]), i);
}

// Vocabulary splits per row, b200_sample's grid: about eight CTAs per SM, slices of at least 2048 tokens, up to 16
// splits for batches of at most 1024 rows (one CTA per row above that).
constexpr int FILTER_MAX_SPLITS = 16;
constexpr int FILTER_MAX_ROWS_SPLIT = 1024;
static inline int filter_splits(int rows, int vocab) {
    int splits = 1;
    if (rows <= FILTER_MAX_ROWS_SPLIT) {
        splits = (b200_current_sm_count() * 8) / rows;
        splits = splits < 1 ? 1 : (splits > FILTER_MAX_SPLITS ? FILTER_MAX_SPLITS : splits);
        while (splits > 1 && vocab / splits < 2048) --splits;
    }
    return splits;
}

}  // namespace b200sample
