// Per-token logprobs of the raw logits (DESIGN.md 3.3.2): log_softmax over the full vocabulary of the bf16 LM-head output,
// read before the penalties, temperature and the filters.  Per row with k >= 0 (k = -1: off), the sampled token's logprob
// and rank #{j : x_j >= x_sampled}, and the k largest logits (value descending, then id ascending) with their logprobs.
//
// A step runs, in stream order:
//   b200_logprob_topk      before the penalties: the exact top max(k, 1) of every row as packed (value, global id) keys,
//                          and the row maximum m.  Every CTA of b200_sample's split grid keeps one sorted list per warp
//                          in registers, merges them, and the last CTA of a row (self-resetting counter) merges the slices.
//   b200_logprob_save      before the penalties: the raw bf16 of every position b200_penalty_apply rewrites in place.
//   ... penalties, filter stages, race ...
//   b200_logprob_restore   writes the saved values back (the logits are raw again) and reads x_sampled.
//   b200_logprob_rank      S = sum_j round(exp(x_j - m) * 2^40) (uint64) and #{j : x_j >= x_sampled}.
//   b200_logprob_finish    merges the top-k keys of every vocab shard and writes ids, logprobs and rank; each value is
//                          (x - m) - ln(S * 2^-40) in float64, rounded once to fp32.  Returns the workspace to zero.
// Every sum is an integer, so the result depends neither on the split count nor on how the vocabulary is sharded.
#include "sample_filter.cuh"

namespace {

using namespace b200sample;

constexpr int LP_THREADS = FILTER_THREADS;                  // for_each_logit strides by FILTER_THREADS
constexpr int LP_WARPS = LP_THREADS / 32;
constexpr int LP_MAX_K = 20;
constexpr int LP_MAX_ROWS = FILTER_MAX_ROWS_SPLIT;
constexpr int LP_MAX_SOURCES = 64;
// workspace words of one row (include/b200_paged_attn.h)
constexpr int LW_MAX = 0, LW_XS = 1, LW_MASS = 2, LW_CNT = 3, LW_NSAVE = 4, LW_ROW_WORDS = 8;
constexpr float FIXED_ONE = 1099511627776.0f;               // 2^40: the row maximum's mass
constexpr unsigned FULL = 0xffffffffu;

__device__ unsigned long long g_lp_slice_keys[LP_MAX_ROWS * FILTER_MAX_SPLITS * LP_MAX_K];
__device__ unsigned int g_lp_row_done[LP_MAX_ROWS];

__device__ __forceinline__ int row_k(const int32_t* k, int row) {
    const int v = k[row];
    return v > LP_MAX_K ? LP_MAX_K : v;
}
// inverse of pack_key: the fp32 value and the vocabulary id of a key
__device__ __forceinline__ float key_value(unsigned long long key) {
    const uint32_t b = (uint32_t)(key >> 32);
    return __uint_as_float((b & 0x80000000u) ? (b ^ 0x80000000u) : ~b);
}
__device__ __forceinline__ int key_id(unsigned long long key) { return (int)(0xffffffffu - (uint32_t)key); }
// pack_key with -0 folded onto +0 (as key16 does), so that equal logits order by token id alone
__device__ __forceinline__ unsigned long long logit_key(float x, uint32_t id) { return pack_key(x == 0.f ? 0.f : x, id); }

// The K largest distinct keys offered to one warp, sorted: lane i holds the i-th largest (0 = empty).  Every call is
// warp-wide with a warp-uniform K.
struct WarpTopK {
    unsigned long long v = 0, thr = 0;                       // thr: the K-th largest so far (0 while fewer than K)
    int K;
    __device__ __forceinline__ explicit WarpTopK(int k) : K(k) {}
    __device__ __forceinline__ void insert(unsigned long long c) {
        const int lane = threadIdx.x & 31;
        const int pos = __popc(__ballot_sync(FULL, v > c));
        if (pos >= K) return;
        const unsigned long long up = __shfl_up_sync(FULL, v, 1);
        if (lane == pos) v = c;
        else if (lane > pos && lane < K) v = up;
        thr = __shfl_sync(FULL, v, K - 1);
    }
    // each lane offers one key (0: none)
    __device__ __forceinline__ void offer(unsigned long long c) {
        unsigned m = __ballot_sync(FULL, c > thr);
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            insert(__shfl_sync(FULL, c, src));
        }
    }
};

__global__ void __launch_bounds__(LP_THREADS) logprob_topk_kernel(const __nv_bfloat16* __restrict__ logits, int64_t stride,
                                                                  const int32_t* __restrict__ ks, int vocab,
                                                                  int64_t index_offset, int64_t* __restrict__ ws,
                                                                  long long* __restrict__ topk_keys, int splits) {
    B200_PDL_SYNC();
    const int row = blockIdx.x, split = blockIdx.y;
    const int k = row_k(ks, row);
    if (k < 0) return;
    const int K = k > 0 ? k : 1;                             // the maximum is needed even when k = 0
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int lo, hi;
    filter_slice(vocab, splits, split, lo, hi);
    const __nv_bfloat16* rowp = logits + (int64_t)row * stride;
    const uint32_t off = (uint32_t)index_offset;
    WarpTopK t(K);
    const int v_lo = lo >> 3, v_hi = hi >> 3;
    const uint4* r4 = reinterpret_cast<const uint4*>(rowp);
    for (int vb = v_lo + warp * 32; vb < v_hi; vb += LP_THREADS) {  // warp-uniform trip count
        const int vi = vb + lane;
        float x[8];
        const bool ok = vi < v_hi;
        if (ok) unpack8(r4[vi], x);
#pragma unroll
        for (int e = 0; e < 8; ++e) t.offer(ok ? logit_key(x[e], off + (uint32_t)(vi * 8 + e)) : 0ull);
    }
    if (warp == 0) {                                         // the < 8 tokens past the last whole vector
        const int i = max(v_hi << 3, lo) + lane;
        t.offer(i < hi ? logit_key(__bfloat162float(rowp[i]), off + (uint32_t)i) : 0ull);
    }
    __shared__ unsigned long long s_keys[LP_WARPS * 32];
    s_keys[threadIdx.x] = t.v;
    __syncthreads();
    if (warp != 0) return;
    WarpTopK m(K);
    for (int w = 0; w < LP_WARPS; ++w) m.offer(s_keys[w * 32 + lane]);
    if (splits > 1) {
        unsigned long long* slot = g_lp_slice_keys + ((int64_t)row * FILTER_MAX_SPLITS + split) * LP_MAX_K;
        if (lane < LP_MAX_K) slot[lane] = m.v;
        __threadfence();
        __syncwarp();
        unsigned int done = 0;
        if (lane == 0) done = atomicAdd(&g_lp_row_done[row], 1u);
        done = __shfl_sync(FULL, done, 0);
        if (done != (unsigned int)splits - 1) return;
        __threadfence();
        WarpTopK r(K);
        for (int s = 0; s < splits; ++s) {
            const unsigned long long* sk = g_lp_slice_keys + ((int64_t)row * FILTER_MAX_SPLITS + s) * LP_MAX_K;
            r.offer(lane < K ? __ldcg(sk + lane) : 0ull);
        }
        m = r;
        if (lane == 0) g_lp_row_done[row] = 0;               // ready for the next launch
    }
    if (lane < LP_MAX_K) topk_keys[(int64_t)row * LP_MAX_K + lane] = (long long)m.v;
    const unsigned long long top = __shfl_sync(FULL, m.v, 0);
    if (lane == 0) ws[(int64_t)row * LW_ROW_WORDS + LW_MAX] = (int64_t)key16(key_value(top));
}

// history entry = token << 32 | in_prompt << 31 | count (penalty.cu); a saved pair = column << 16 | raw bf16 bits, -1 = none
__global__ void __launch_bounds__(LP_THREADS) logprob_save_kernel(const __nv_bfloat16* __restrict__ logits, int64_t stride,
                                                                  const int32_t* __restrict__ ks, int vocab,
                                                                  int64_t index_offset,
                                                                  const long long* __restrict__ history,
                                                                  const int32_t* __restrict__ lengths, int num_slots,
                                                                  int capacity, const int32_t* __restrict__ slots,
                                                                  const int64_t* __restrict__ pending,
                                                                  int64_t* __restrict__ ws, long long* __restrict__ saved) {
    B200_PDL_SYNC();
    const int row = blockIdx.x;
    if (row_k(ks, row) < 0) return;
    const int slot = slots[row];
    if (slot < 0 || slot >= num_slots) return;              // the rows b200_penalty_apply leaves alone
    const long long* h = history + (int64_t)slot * capacity;
    const unsigned short* x = reinterpret_cast<const unsigned short*>(logits + (int64_t)row * stride);
    long long* out = saved + (int64_t)row * (capacity + 1);
    int n = lengths[slot];
    n = n < 0 ? 0 : (n > capacity ? capacity : n);
    auto pair = [&](long long tok) -> long long {
        const long long col = tok - index_offset;
        return (tok >= 0 && col >= 0 && col < vocab) ? (col << 16) | x[col] : -1ll;
    };
    for (int i = threadIdx.x; i < n; i += LP_THREADS) out[i] = pair(h[i] >> 32);
    if (threadIdx.x == 0) {
        out[n] = pair(pending ? pending[row] : -1);           // absorbed (and penalised) by the apply if still absent
        ws[(int64_t)row * LW_ROW_WORDS + LW_NSAVE] = n + 1;
    }
}

__global__ void __launch_bounds__(LP_THREADS) logprob_restore_kernel(__nv_bfloat16* __restrict__ logits, int64_t stride,
                                                                     const int32_t* __restrict__ ks, int vocab,
                                                                     int64_t index_offset,
                                                                     const int64_t* __restrict__ tokens,
                                                                     int64_t* __restrict__ ws,
                                                                     const long long* __restrict__ saved, int capacity) {
    B200_PDL_SYNC();
    const int row = blockIdx.x;
    if (row_k(ks, row) < 0) return;
    int64_t* w = ws + (int64_t)row * LW_ROW_WORDS;
    unsigned short* x = reinterpret_cast<unsigned short*>(logits + (int64_t)row * stride);
    if (saved) {
        const long long* in = saved + (int64_t)row * (capacity + 1);
        const int n = (int)w[LW_NSAVE];
        for (int i = threadIdx.x; i < n; i += LP_THREADS) {
            const long long e = in[i];
            if (e >= 0) x[e >> 16] = (unsigned short)(e & 0xffff);   // a repeated column gets the same value
        }
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    w[LW_NSAVE] = 0;
    const int64_t col = tokens[row] - index_offset;
    if (col >= 0 && col < vocab) w[LW_XS] = (int64_t)key16(__uint_as_float((uint32_t)x[col] << 16));
}

__global__ void __launch_bounds__(LP_THREADS) logprob_rank_kernel(const __nv_bfloat16* __restrict__ logits, int64_t stride,
                                                                  const int32_t* __restrict__ ks, int vocab,
                                                                  int64_t* __restrict__ ws, int splits) {
    B200_PDL_SYNC();
    const int row = blockIdx.x;
    if (row_k(ks, row) < 0) return;
    int64_t* w = ws + (int64_t)row * LW_ROW_WORDS;
    const float m = key16_value((uint32_t)__ldcg(w + LW_MAX));
    const float xs = key16_value((uint32_t)__ldcg(w + LW_XS));
    int lo, hi;
    filter_slice(vocab, splits, blockIdx.y, lo, hi);
    unsigned long long mass = 0, cnt = 0;
    for_each_logit(logits + (int64_t)row * stride, lo, hi, [&](float x, int) {
        mass += __float2ull_rn(expf(x - m) * FIXED_ONE);
        cnt += x >= xs;
    });
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mass += __shfl_xor_sync(FULL, mass, o);
        cnt += __shfl_xor_sync(FULL, cnt, o);
    }
    __shared__ unsigned long long s_mass[LP_WARPS], s_cnt[LP_WARPS];
    if ((threadIdx.x & 31) == 0) { s_mass[threadIdx.x >> 5] = mass; s_cnt[threadIdx.x >> 5] = cnt; }
    __syncthreads();
    if (threadIdx.x != 0) return;
    for (int i = 1; i < LP_WARPS; ++i) { mass += s_mass[i]; cnt += s_cnt[i]; }
    if (mass) atomicAdd(reinterpret_cast<unsigned long long*>(w + LW_MASS), mass);
    if (cnt) atomicAdd(reinterpret_cast<unsigned long long*>(w + LW_CNT), cnt);
}

// one warp per row
__global__ void __launch_bounds__(32) logprob_finish_kernel(const int32_t* __restrict__ ks, int rows,
                                                            const int64_t* __restrict__ tokens,
                                                            const long long* __restrict__ topk_keys, int sources,
                                                            int64_t* __restrict__ ws, int32_t* __restrict__ out_ids,
                                                            float* __restrict__ out_logprobs, int32_t* __restrict__ out_rank,
                                                            int64_t out_stride) {
    B200_PDL_SYNC();
    const int row = blockIdx.x, lane = threadIdx.x;
    const int k = row_k(ks, row);
    if (k < 0) return;
    int64_t* w = ws + (int64_t)row * LW_ROW_WORDS;
    WarpTopK t(k > 0 ? k : 1);
    if (k > 0)
        for (int s = 0; s < sources; ++s)
            t.offer(lane < k ? (unsigned long long)topk_keys[((int64_t)s * rows + row) * LP_MAX_K + lane] : 0ull);
    const double m = (double)key16_value((uint32_t)w[LW_MAX]);
    const double lse = log((double)(unsigned long long)w[LW_MASS] * 0x1p-40);
    auto lp = [&](float x) { return (float)(((double)x - m) - lse); };
    int32_t* ids = out_ids + (int64_t)row * out_stride;
    float* lps = out_logprobs + (int64_t)row * out_stride;
    if (lane < k) {
        ids[1 + lane] = key_id(t.v);
        lps[1 + lane] = lp(key_value(t.v));
    }
    if (lane == 0) {
        ids[0] = (int32_t)tokens[row];
        lps[0] = lp(key16_value((uint32_t)w[LW_XS]));
        out_rank[(int64_t)row * out_stride] = (int32_t)w[LW_CNT];
    }
    __syncwarp();
    if (lane < LW_ROW_WORDS) w[lane] = 0;
}

int check_logits(const void* logits, int64_t stride, const int32_t* k, int rows, int vocab, const int64_t* ws) {
    if (!logits || !k || !ws || rows <= 0 || rows > LP_MAX_ROWS || vocab <= 0) return B200_EINVAL;
    if (((uintptr_t)logits & 15) || (stride % 8) || (rows > 1 && stride < vocab)) return B200_EINVAL;
    if (vocab > FILTER_MAX_VOCAB) return B200_EUNSUPPORTED;
    return B200_OK;
}

}  // namespace

extern "C" int64_t b200_logprob_workspace_words(int rows) {
    return rows <= 0 || rows > LP_MAX_ROWS ? 0 : (int64_t)rows * LW_ROW_WORDS;
}

extern "C" int b200_logprob_topk(const void* logits, int64_t logits_stride0, const int32_t* k, int rows, int vocab,
                                 int64_t index_offset, int64_t* workspace, int64_t* topk_keys, void* stream) {
    int rc = check_logits(logits, logits_stride0, k, rows, vocab, workspace);
    if (rc) return rc;
    if (!topk_keys || index_offset < 0) return B200_EINVAL;
    if (index_offset + vocab > FILTER_MAX_VOCAB) return B200_EUNSUPPORTED;
    const int splits = filter_splits(rows, vocab);
    B200_LAUNCH((logprob_topk_kernel), dim3(rows, splits), LP_THREADS, 0, static_cast<cudaStream_t>(stream),
                static_cast<const __nv_bfloat16*>(logits), logits_stride0, k, vocab, index_offset, workspace,
                reinterpret_cast<long long*>(topk_keys), splits);
    return b200_launch_status(nullptr);
}

extern "C" int b200_logprob_save(const void* logits, int64_t logits_stride0, const int32_t* k, int rows, int vocab,
                                 int64_t index_offset, const int64_t* history, const int32_t* lengths, int num_slots,
                                 int capacity, const int32_t* slots, const int64_t* pending, int64_t* workspace,
                                 int64_t* saved, void* stream) {
    int rc = check_logits(logits, logits_stride0, k, rows, vocab, workspace);
    if (rc) return rc;
    if (!history || !lengths || !slots || !saved || num_slots <= 0 || capacity <= 0 || index_offset < 0) return B200_EINVAL;
    B200_LAUNCH((logprob_save_kernel), rows, LP_THREADS, 0, static_cast<cudaStream_t>(stream),
                static_cast<const __nv_bfloat16*>(logits), logits_stride0, k, vocab, index_offset,
                reinterpret_cast<const long long*>(history), lengths, num_slots, capacity, slots, pending, workspace,
                reinterpret_cast<long long*>(saved));
    return b200_launch_status(nullptr);
}

extern "C" int b200_logprob_restore(void* logits, int64_t logits_stride0, const int32_t* k, int rows, int vocab,
                                    int64_t index_offset, const int64_t* tokens, int64_t* workspace, const int64_t* saved,
                                    int capacity, void* stream) {
    int rc = check_logits(logits, logits_stride0, k, rows, vocab, workspace);
    if (rc) return rc;
    if (!tokens || index_offset < 0 || (saved && capacity <= 0)) return B200_EINVAL;
    B200_LAUNCH((logprob_restore_kernel), rows, LP_THREADS, 0, static_cast<cudaStream_t>(stream),
                static_cast<__nv_bfloat16*>(logits), logits_stride0, k, vocab, index_offset, tokens, workspace,
                reinterpret_cast<const long long*>(saved), capacity);
    return b200_launch_status(nullptr);
}

extern "C" int b200_logprob_rank(const void* logits, int64_t logits_stride0, const int32_t* k, int rows, int vocab,
                                 int64_t* workspace, void* stream) {
    int rc = check_logits(logits, logits_stride0, k, rows, vocab, workspace);
    if (rc) return rc;
    const int splits = filter_splits(rows, vocab);
    B200_LAUNCH((logprob_rank_kernel), dim3(rows, splits), LP_THREADS, 0, static_cast<cudaStream_t>(stream),
                static_cast<const __nv_bfloat16*>(logits), logits_stride0, k, vocab, workspace, splits);
    return b200_launch_status(nullptr);
}

extern "C" int b200_logprob_finish(const int32_t* k, int rows, const int64_t* tokens, const int64_t* topk_keys, int sources,
                                   int64_t* workspace, int32_t* out_ids, float* out_logprobs, int32_t* out_rank,
                                   int64_t out_stride, void* stream) {
    if (!k || !tokens || !topk_keys || !workspace || !out_ids || !out_logprobs || !out_rank) return B200_EINVAL;
    if (rows <= 0 || rows > LP_MAX_ROWS || sources <= 0 || sources > LP_MAX_SOURCES || out_stride < LP_MAX_K + 1)
        return B200_EINVAL;
    B200_LAUNCH((logprob_finish_kernel), rows, 32, 0, static_cast<cudaStream_t>(stream), k, rows, tokens,
                reinterpret_cast<const long long*>(topk_keys), sources, workspace, out_ids, out_logprobs, out_rank,
                out_stride);
    return b200_launch_status(nullptr);
}
