// Stages 0-3 of the filtered sampler (top-k / top-p / min-p): the exact bf16 threshold tau of every row, by the two-level
// radix select described in sample_filter.cuh.  The race that draws a token from {x >= tau} is sample_masked_kernel in
// sampler.cu.  Every stage runs on b200_sample's split-vocab grid, so one decode row still fills the GPU; each CTA builds
// its histogram in shared memory and adds it to the row's workspace with one integer atomic per non-empty bin.  A stage's
// prologue reads the reduced results of the stages before it and repeats the 256-bin scans that pick its bin in every
// CTA of the row; rows the stage has nothing to do for (every filter off, greedy, or top-p already settled) return at once.
#include "sample_filter.cuh"

namespace {

using namespace b200sample;

// Histogram copies per CTA: lane l adds to copy l % 8, so the few hot high-byte bins of a logit row (a bin spans a factor
// of four in magnitude) see at most 4-way same-address conflicts.  A copy receives an eighth of the slice, at most 2^15
// tokens, so (count << 48) | mass fits one 64-bit shared atomic: count < 2^16, mass < 2^15 * 2^32.
constexpr int HIST_COPIES = 8;
constexpr unsigned long long MASS_MASK = (1ull << 48) - 1;

__global__ void __launch_bounds__(FILTER_THREADS) filter_max_kernel(const __nv_bfloat16* __restrict__ logits, int64_t stride,
                                                                    const float* __restrict__ temperatures,
                                                                    const int32_t* __restrict__ top_k,
                                                                    const float* __restrict__ top_p,
                                                                    const float* __restrict__ min_p, int vocab,
                                                                    int64_t* ws, int splits) {
    B200_PDL_SYNC();
    const int row = blockIdx.x;
    const FilterRow f(temperatures, top_k, top_p, min_p, row);
    if (!f.active) return;
    int lo, hi;
    filter_slice(vocab, splits, blockIdx.y, lo, hi);
    uint32_t best = 0;
    for_each_logit(logits + (int64_t)row * stride, lo, hi, [&](float x, int) {
        const uint32_t k = key16(x);
        best = k > best ? k : best;
    });
    best = __reduce_max_sync(0xffffffffu, best);
    __shared__ uint32_t sw[FILTER_THREADS / 32];
    if ((threadIdx.x & 31) == 0) sw[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x != 0) return;
    for (int w = 1; w < FILTER_THREADS / 32; ++w) best = sw[w] > best ? sw[w] : best;
    if (best) atomicMax(reinterpret_cast<unsigned long long*>(ws + (int64_t)row * FW_ROW_WORDS + FW_MAX), (unsigned long long)best);
}

// stage 1: high-byte histogram of the tokens >= tau_min_p; stages 2 / 3: low-byte histogram inside the plan's bin
__global__ void __launch_bounds__(FILTER_THREADS) filter_hist_kernel(const __nv_bfloat16* __restrict__ logits, int64_t stride,
                                                                     const float* __restrict__ temperatures,
                                                                     const int32_t* __restrict__ top_k,
                                                                     const float* __restrict__ top_p,
                                                                     const float* __restrict__ min_p, int vocab, int stage,
                                                                     int64_t* ws, int splits) {
    B200_PDL_SYNC();
    const int row = blockIdx.x;
    const FilterRow f(temperatures, top_k, top_p, min_p, row);
    if (!f.active) return;
    int64_t* w = ws + (int64_t)row * FW_ROW_WORDS;
    __shared__ PlanSmem sm;
    const Plan P = plan_row(w, f, stage, sm);
    const int sel = stage == 1 ? -1 : (stage == 2 ? P.bin2 : P.bin3);
    if (stage > 1 && sel < 0) return;                                  // block-uniform

    __shared__ unsigned long long hist[256 * HIST_COPIES];
    for (int i = threadIdx.x; i < 256 * HIST_COPIES; i += FILTER_THREADS) hist[i] = 0ull;
    __syncthreads();
    int lo, hi;
    filter_slice(vocab, splits, blockIdx.y, lo, hi);
    const float m = key16_value(P.m_key);
    const uint32_t tmp_key = P.tmp_key;
    unsigned long long* mine = hist + (threadIdx.x & (HIST_COPIES - 1));
    for_each_logit(logits + (int64_t)row * stride, lo, hi, [&](float x, int) {
        const uint32_t key = key16(x);
        if (key < tmp_key) return;
        if (sel >= 0 && (int)(key >> 8) != sel) return;
        const uint32_t bin = sel < 0 ? key >> 8 : key & 255u;
        atomicAdd(mine + bin * HIST_COPIES, (1ull << 48) | fixed_mass(x, m, f.inv_t));
    });
    __syncthreads();
    const int region = stage == 1 ? FW_S1 : (stage == 2 ? FW_S2 : FW_S3);
    const int b = threadIdx.x;
    unsigned long long c = 0, mass = 0;
#pragma unroll
    for (int r = 0; r < HIST_COPIES; ++r) {
        const unsigned long long v = hist[b * HIST_COPIES + r];
        c += v >> 48;
        mass += v & MASS_MASK;
    }
    if (c) {
        atomicAdd(reinterpret_cast<unsigned long long*>(w + region + b), c);
        if (mass) atomicAdd(reinterpret_cast<unsigned long long*>(w + region + 256 + b), mass);
    }
}

}  // namespace

extern "C" int64_t b200_sample_filter_workspace_words(int rows) {
    return rows <= 0 ? 0 : (int64_t)rows * FW_ROW_WORDS;
}

extern "C" int b200_sample_filter_stage(const void* logits, int64_t logits_stride0, const float* temperatures,
                                        const int32_t* top_k, const float* top_p, const float* min_p, int rows, int vocab,
                                        int stage, int64_t* workspace, void* stream) {
    if (!logits || !temperatures || !workspace || rows <= 0 || vocab <= 0 || stage < 0 || stage > 3) return B200_EINVAL;
    if (((uintptr_t)logits & 15) || (logits_stride0 % 8) || (rows > 1 && logits_stride0 < vocab)) return B200_EINVAL;
    if (vocab > FILTER_MAX_VOCAB) return B200_EUNSUPPORTED;
    const int splits = filter_splits(rows, vocab);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const dim3 grid(rows, splits);
    const __nv_bfloat16* x = static_cast<const __nv_bfloat16*>(logits);
    if (stage == 0) {
        B200_LAUNCH((filter_max_kernel), grid, FILTER_THREADS, 0, st, x, logits_stride0, temperatures, top_k, top_p, min_p,
                    vocab, workspace, splits);
    } else {
        B200_LAUNCH((filter_hist_kernel), grid, FILTER_THREADS, 0, st, x, logits_stride0, temperatures, top_k, top_p, min_p,
                    vocab, stage, workspace, splits);
    }
    return b200_launch_status(nullptr);
}
