// Token sampling for sm_90a: replaces Sampler.forward (nanovllm/layers/sampler.py:7-12, an
// Inductor-compiled softmax + exponential race) and adds the greedy branch (temperature == 0)
// the north-star requires.  The logits are streamed once with 128-bit loads and only a running
// (value, index) maximum is kept: nothing of size [rows, vocab] is materialised.
//
// Each row is cut into `splits` vocabulary slices (one CTA each, so a single-sequence decode step still
// fills many SMs); slices leave packed (score, index) keys in a static scratch array and the last CTA
// to finish a row (self-resetting counter) folds them.  Ties go to the lowest index at every level, so
// the result does not depend on the split count.
//
// sample_masked_kernel is the same race restricted to {x >= tau}, tau being the top-k / top-p / min-p threshold that the
// stages of sample_filter.cu leave in their workspace (see sample_filter.cuh).
#include "sample_common.cuh"
#include "sample_filter.cuh"

namespace {

using namespace b200sample;

constexpr int SAMPLE_THREADS = 256;
constexpr int MAX_SPLITS = 16;
constexpr int MAX_ROWS_SPLIT = 1024;

__device__ unsigned long long g_slice_keys[MAX_ROWS_SPLIT * MAX_SPLITS];
__device__ unsigned int g_row_done[MAX_ROWS_SPLIT];

template <bool FP32>
__global__ void __launch_bounds__(SAMPLE_THREADS) sample_kernel(const void* __restrict__ logits, int64_t stride,
                                                                const float* __restrict__ temperatures, int vocab,
                                                                int64_t index_offset, uint64_t seed, uint64_t step,
                                                                const int64_t* __restrict__ step_dev,
                                                                int64_t* out, int64_t* out_keys, int splits) {
    B200_PDL_SYNC();
    const int row = blockIdx.x;
    const int split = blockIdx.y;
    const float t = temperatures ? temperatures[row] : 0.f;
    const bool greedy = !(t > 0.f);
    const float inv_t = greedy ? 1.f : 1.f / t;
    if (step_dev) step += (uint64_t)*step_dev;
    const uint64_t key64 = mix64(seed ^ mix64(step * 0x9e3779b97f4a7c15ull + (uint64_t)row));
    const uint32_t k0 = (uint32_t)key64, k1 = (uint32_t)(key64 >> 32);
    Best best{-INFINITY, 0x7fffffff};

    // Exponential race (sampler.py:10-11): argmax softmax(x/t)_j / E_j == argmax x_j/t - log E_j, E_j = -log u_j.
    auto score = [&](float x, int idx) -> float {
        if (greedy) return x;
        const uint32_t r = mix32(((uint32_t)(index_offset + idx) ^ k0) * 0x9e3779b1u + k1);
        const float u = ((float)(r >> 8) + 0.5f) * (1.0f / 16777216.0f);       // (0, 1)
        const float e = fmaxf(-__logf(u), 1e-10f);                             // clamp as in sampler.py:11
        return fmaf(x, inv_t, -__logf(e));
    };

    // slice [lo, hi) of the vocabulary, 8-aligned so the vector loads stay aligned
    const int per = (((vocab + splits - 1) / splits) + 7) & ~7;
    const int lo = split * per;
    int hi = lo + per;
    hi = hi > vocab ? vocab : hi;

    if (FP32) {
        const float* rowp = static_cast<const float*>(logits) + (int64_t)row * stride;
        for (int i = lo + threadIdx.x; i < hi; i += SAMPLE_THREADS) take(best, score(rowp[i], i), i);
    } else {
        const __nv_bfloat16* rowp = static_cast<const __nv_bfloat16*>(logits) + (int64_t)row * stride;
        const int v_lo = lo >> 3, v_hi = hi >> 3;                              // whole 8-element vectors
        const uint4* r4 = reinterpret_cast<const uint4*>(rowp);
        for (int vi = v_lo + threadIdx.x; vi < v_hi; vi += SAMPLE_THREADS) {
            float f[8];
            unpack8(r4[vi], f);
#pragma unroll
            for (int e = 0; e < 8; ++e) take(best, score(f[e], vi * 8 + e), vi * 8 + e);
        }
        for (int i = (v_hi << 3) + threadIdx.x; i < hi; i += SAMPLE_THREADS)
            if (i >= lo) take(best, score(__bfloat162float(rowp[i]), i), i);
    }

#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best.v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, best.i, o);
        take(best, ov, oi);
    }
    __shared__ float sv[SAMPLE_THREADS / 32];
    __shared__ int si[SAMPLE_THREADS / 32];
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best.v; si[threadIdx.x >> 5] = best.i; }
    __syncthreads();
    if (threadIdx.x != 0) return;
    Best b{sv[0], si[0]};
    for (int w = 1; w < SAMPLE_THREADS / 32; ++w) take(b, sv[w], si[w]);
    unsigned long long key = b.i == 0x7fffffff ? 0ull : pack_key(b.v, (uint32_t)(index_offset + b.i));
    if (splits > 1) {
        g_slice_keys[row * MAX_SPLITS + split] = key;
        __threadfence();
        const unsigned int done = atomicAdd(&g_row_done[row], 1u);
        if (done != (unsigned int)splits - 1) return;
        __threadfence();
        key = 0ull;
        for (int s = 0; s < splits; ++s) {
            const unsigned long long k = __ldcg(&g_slice_keys[row * MAX_SPLITS + s]);
            key = k > key ? k : key;
        }
        g_row_done[row] = 0;                                   // ready for the next launch
    }
    const int64_t tok = key ? (int64_t)(0xffffffffu - (uint32_t)(key & 0xffffffffull)) : index_offset;
    if (out) out[row] = tok;
    if (out_keys) out_keys[row] = (int64_t)(key ^ 0x8000000000000000ull);   // signed order == unsigned order
}

__device__ unsigned long long g_masked_slice_keys[MAX_ROWS_SPLIT * MAX_SPLITS];
__device__ unsigned int g_masked_row_done[MAX_ROWS_SPLIT];

// The exponential race of sample_kernel<false> over the kept set {x : key16(x) >= tau} of each row: the same
// RowSampler::score of the same (seed, step, row, vocabulary id), so it is an exact draw from the softmax renormalised
// over the kept set.  A row with every filter off (or a greedy row) has tau = 0, keeps everything and gets the token
// b200_sample gives it.  The last CTA of a row writes tau to FW_TAU and returns the row's other workspace words to zero.
__global__ void __launch_bounds__(SAMPLE_THREADS) sample_masked_kernel(const __nv_bfloat16* __restrict__ logits, int64_t stride,
                                                                       const float* __restrict__ temperatures,
                                                                       const int32_t* __restrict__ top_k,
                                                                       const float* __restrict__ top_p,
                                                                       const float* __restrict__ min_p, int vocab,
                                                                       int64_t index_offset, uint64_t seed, uint64_t step,
                                                                       const int64_t* __restrict__ step_dev, int64_t* ws,
                                                                       int64_t* out, int64_t* out_keys, int splits) {
    B200_PDL_SYNC();
    const int row = blockIdx.x;
    const int split = blockIdx.y;
    const FilterRow f(temperatures, top_k, top_p, min_p, row);
    int64_t* w = ws + (int64_t)row * FW_ROW_WORDS;
    __shared__ PlanSmem sm;
    uint32_t tau = 0;
    if (f.active) tau = plan_row(w, f, 4, sm).tau;                    // block-uniform
    if (step_dev) step += (uint64_t)*step_dev;
    const RowSampler rs(f.t, seed, step, row);
    Best best{-INFINITY, 0x7fffffff};
    int lo, hi;
    filter_slice(vocab, splits, split, lo, hi);
    for_each_logit(logits + (int64_t)row * stride, lo, hi, [&](float x, int i) {
        if (key16(x) >= tau) take(best, rs.score(x, index_offset + i), i);
    });

#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best.v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, best.i, o);
        take(best, ov, oi);
    }
    __shared__ float sv[SAMPLE_THREADS / 32];
    __shared__ int si[SAMPLE_THREADS / 32];
    __shared__ int s_last;
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best.v; si[threadIdx.x >> 5] = best.i; }
    __syncthreads();
    if (threadIdx.x == 0) {
        Best b{sv[0], si[0]};
        for (int wi = 1; wi < SAMPLE_THREADS / 32; ++wi) take(b, sv[wi], si[wi]);
        unsigned long long key = b.i == 0x7fffffff ? 0ull : pack_key(b.v, (uint32_t)(index_offset + b.i));
        int last = 1;
        if (splits > 1) {
            g_masked_slice_keys[row * MAX_SPLITS + split] = key;
            __threadfence();
            const unsigned int done = atomicAdd(&g_masked_row_done[row], 1u);
            last = done == (unsigned int)splits - 1;
            if (last) {
                __threadfence();
                key = 0ull;
                for (int s = 0; s < splits; ++s) {
                    const unsigned long long k = __ldcg(&g_masked_slice_keys[row * MAX_SPLITS + s]);
                    key = k > key ? k : key;
                }
                g_masked_row_done[row] = 0;                           // ready for the next launch
            }
        }
        if (last) {
            const int64_t tok = key ? (int64_t)(0xffffffffu - (uint32_t)(key & 0xffffffffull)) : index_offset;
            if (out) out[row] = tok;
            if (out_keys) out_keys[row] = (int64_t)(key ^ 0x8000000000000000ull);
            w[FW_TAU] = (int64_t)tau;
        }
        s_last = last;
    }
    __syncthreads();
    // every CTA of the row has finished its prologue (it counted itself done after it): reset the row for the next launch
    if (!s_last || !f.active) return;
    if (threadIdx.x == 0) w[FW_MAX] = 0;
    for (int i = FW_S1 + threadIdx.x; i < FW_ROW_WORDS; i += SAMPLE_THREADS) w[i] = 0;
}

}  // namespace

extern "C" int b200_sample(const void* logits, int logits_is_fp32, int64_t logits_stride0,
                           const float* temperatures, int rows, int vocab, int64_t index_offset,
                           uint64_t seed, uint64_t step, const int64_t* step_dev, int64_t* out,
                           int64_t* out_keys, void* stream) {
    if (!logits || (!out && !out_keys) || rows < 0 || vocab <= 0 || index_offset < 0) return B200_EINVAL;
    if (index_offset + vocab > 0xffffffffll) return B200_EUNSUPPORTED;
    if (rows == 0) return B200_OK;
    int splits = 1;
    if (rows <= MAX_ROWS_SPLIT) {
        splits = (b200_current_sm_count() * 8) / rows;          // about eight CTAs per SM
        splits = splits < 1 ? 1 : (splits > MAX_SPLITS ? MAX_SPLITS : splits);
        while (splits > 1 && vocab / splits < 2048) --splits;      // keep slices worth a CTA
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    dim3 grid(rows, splits);
    if (logits_is_fp32) {
        B200_LAUNCH((sample_kernel<true>), grid, SAMPLE_THREADS, 0, st, logits, logits_stride0, temperatures, vocab, index_offset, seed, step, step_dev, out, out_keys, splits);
    } else {
        if (((uintptr_t)logits & 15) || (logits_stride0 % 8)) return B200_EINVAL;
        B200_LAUNCH((sample_kernel<false>), grid, SAMPLE_THREADS, 0, st, logits, logits_stride0, temperatures, vocab, index_offset, seed, step, step_dev, out, out_keys, splits);
    }
    return b200_launch_status(nullptr);
}

extern "C" int b200_sample_filtered(const void* logits, int64_t logits_stride0, const float* temperatures,
                                    const int32_t* top_k, const float* top_p, const float* min_p, int rows, int vocab,
                                    int64_t index_offset, uint64_t seed, uint64_t step, const int64_t* step_dev,
                                    int64_t* workspace, int64_t* out, int64_t* out_keys, void* stream) {
    if (!logits || !temperatures || !workspace || (!out && !out_keys) || rows <= 0 || vocab <= 0 || index_offset < 0)
        return B200_EINVAL;
    if (((uintptr_t)logits & 15) || (logits_stride0 % 8) || (rows > 1 && logits_stride0 < vocab)) return B200_EINVAL;
    if (vocab > FILTER_MAX_VOCAB || index_offset + vocab > 0xffffffffll) return B200_EUNSUPPORTED;
    const int splits = filter_splits(rows, vocab);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    B200_LAUNCH((sample_masked_kernel), dim3(rows, splits), SAMPLE_THREADS, 0, st, static_cast<const __nv_bfloat16*>(logits),
                logits_stride0, temperatures, top_k, top_p, min_p, vocab, index_offset, seed, step, step_dev, workspace, out,
                out_keys, splits);
    return b200_launch_status(nullptr);
}
