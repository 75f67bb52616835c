// Mixture-of-experts layer of Qwen3 MoE checkpoints (Qwen3MoeSparseMoeBlock), around the grouped wgmma GEMM of
// linear_tc.cu (b200_moe_linear).  One MoE MLP is
//
//   router logits (library GEMM, bf16 [T, E]) -> b200_moe_route -> b200_moe_align -> b200_moe_gather
//   -> b200_moe_linear (gate_up + SiluAndMul) -> b200_moe_linear (down) -> b200_moe_combine
//
// Every launch has a grid that depends on T only, never on the routing, so a decode step that contains them can be captured
// once and replayed with any routing.  Nothing is summed with atomics: the only atomics hand out row slots inside an
// expert's segment, and no value depends on which slot a row gets (a GEMM row is a function of its own x row).
#include "common.cuh"

namespace {

constexpr int MOE_MAX_EXPERTS = 256;
constexpr int MOE_MAX_TOPK = 16;
constexpr int MOE_TILE_ROWS = 128;          // rows of one grouped-GEMM tile (linear_tc.cu's LM)
constexpr int ALIGN_THREADS = 1024;

// Softmax over the E router logits in fp32 (expf), the top k by (probability descending, expert id ascending), and, with
// norm, the k weights divided by their fp32 sum in rank order.  One warp per token; lane l holds experts l, l + 32, ...
__global__ void __launch_bounds__(256) moe_route_kernel(const __nv_bfloat16* __restrict__ logits, int64_t stride, int tokens, int E,
                                                        int k, int norm, int32_t* __restrict__ ids, float* __restrict__ weights) {
    B200_PDL_SYNC();
    const int t = (int)(((int64_t)blockIdx.x * 256 + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (t >= tokens) return;
    constexpr int PER = MOE_MAX_EXPERTS / 32;
    float v[PER];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
        const int e = lane + 32 * i;
        v[i] = e < E ? __bfloat162float(logits[(int64_t)t * stride + e]) : -INFINITY;
        mx = fmaxf(mx, v[i]);
    }
    mx = warp_max(mx);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
        v[i] = lane + 32 * i < E ? expf(v[i] - mx) : 0.f;
        s += v[i];
    }
    s = warp_sum(s);
    // keys: probability bits (non-negative floats order as integers) above the complemented expert id; 0 = taken / absent
    unsigned long long key[PER];
#pragma unroll
    for (int i = 0; i < PER; ++i) {
        const int e = lane + 32 * i;
        key[i] = e < E ? ((unsigned long long)__float_as_uint(__fdiv_rn(v[i], s)) << 32) | (0xffffffffu - (uint32_t)e) : 0ull;
    }
    float w_mine = 0.f;                     // lane j keeps the weight of rank j
    int id_mine = 0;
    float total = 0.f;
    for (int j = 0; j < k; ++j) {
        unsigned long long best = 0ull;
#pragma unroll
        for (int i = 0; i < PER; ++i) best = key[i] > best ? key[i] : best;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
            best = other > best ? other : best;
        }
        const int e = (int)(0xffffffffu - (uint32_t)(best & 0xffffffffull));
        const float p = __uint_as_float((uint32_t)(best >> 32));
#pragma unroll
        for (int i = 0; i < PER; ++i)
            if (lane + 32 * i == e) key[i] = 0ull;
        total += p;
        if (lane == j) { w_mine = p; id_mine = e; }
    }
    if (lane < k) {
        ids[(int64_t)t * k + lane] = id_mine;
        weights[(int64_t)t * k + lane] = norm ? __fdiv_rn(w_mine, total) : w_mine;
    }
}

// One CTA: per-expert row counts, the segment of each expert in the permuted buffer (experts in id order, no padding),
// the tile table of b200_moe_linear and the permuted row of every (token, rank) entry.
__global__ void __launch_bounds__(ALIGN_THREADS) moe_align_kernel(const int32_t* __restrict__ ids, int entries, int E,
                                                                   int32_t* __restrict__ perm, int4* __restrict__ tiles) {
    __shared__ int cnt[MOE_MAX_EXPERTS], off[MOE_MAX_EXPERTS], toff[MOE_MAX_EXPERTS], cur[MOE_MAX_EXPERTS];
    B200_PDL_SYNC();
    const int tid = threadIdx.x;
    for (int e = tid; e < E; e += ALIGN_THREADS) cnt[e] = 0, cur[e] = 0;
    __syncthreads();
    for (int i = tid; i < entries; i += ALIGN_THREADS) atomicAdd(&cnt[ids[i]], 1);
    __syncthreads();
    if (tid == 0) {
        int rows = 0, nt = 0;
        for (int e = 0; e < E; ++e) {
            off[e] = rows;
            toff[e] = nt;
            rows += cnt[e];
            nt += (cnt[e] + MOE_TILE_ROWS - 1) / MOE_TILE_ROWS;
        }
        tiles[0] = make_int4(nt, rows, 0, 0);
    }
    __syncthreads();
    for (int e = tid; e < E; e += ALIGN_THREADS) {
        const int c = cnt[e], o = off[e];
        for (int r = 0, i = toff[e]; r < c; r += MOE_TILE_ROWS, ++i) tiles[1 + i] = make_int4(e, o + r, o + min(r + MOE_TILE_ROWS, c), 0);
    }
    for (int i = tid; i < entries; i += ALIGN_THREADS) {
        const int e = ids[i];
        perm[i] = off[e] + atomicAdd(&cur[e], 1);
    }
}

// x_perm[perm[t k + j]] = x[t]: one warp per (token, rank) entry, 16-byte vectors
__global__ void __launch_bounds__(256) moe_gather_kernel(const __nv_bfloat16* __restrict__ x, int64_t x_stride, int entries, int k,
                                                         int vecs, const int32_t* __restrict__ perm, __nv_bfloat16* __restrict__ xp) {
    B200_PDL_SYNC();
    const int i = (int)(((int64_t)blockIdx.x * 256 + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= entries) return;
    const uint4* src = reinterpret_cast<const uint4*>(x + (int64_t)(i / k) * x_stride);
    uint4* dst = reinterpret_cast<uint4*>(xp + (int64_t)perm[i] * vecs * 8);
    for (int c = lane; c < vecs; c += 32) dst[c] = src[c];
}

// out[t] = bf16(sum_j w[t, j] * y[perm[t k + j]]), an fp32 fma chain in rank order j
__global__ void __launch_bounds__(256) moe_combine_kernel(const __nv_bfloat16* __restrict__ y, const int32_t* __restrict__ perm,
                                                          const float* __restrict__ weights, int k, int vecs,
                                                          __nv_bfloat16* __restrict__ out, int64_t out_stride) {
    B200_PDL_SYNC();
    const int t = blockIdx.x;
    __shared__ int rows[MOE_MAX_TOPK];
    __shared__ float ws[MOE_MAX_TOPK];
    if (threadIdx.x < k) {
        rows[threadIdx.x] = perm[(int64_t)t * k + threadIdx.x];
        ws[threadIdx.x] = weights[(int64_t)t * k + threadIdx.x];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < vecs; c += blockDim.x) {
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int j = 0; j < k; ++j) {
            float v[8];
            unpack8(reinterpret_cast<const uint4*>(y + (int64_t)rows[j] * vecs * 8)[c], v);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] = fmaf(ws[j], v[e], acc[e]);
        }
        reinterpret_cast<uint4*>(out + (int64_t)t * out_stride)[c] = pack8(acc);
    }
}

}  // namespace

extern "C" int b200_moe_max_tiles(int entries, int num_experts) {
    if (entries < 0 || num_experts <= 0) return -1;
    return (entries + MOE_TILE_ROWS - 1) / MOE_TILE_ROWS + (entries < num_experts ? entries : num_experts);
}

extern "C" int b200_moe_route(const void* logits, int64_t logits_stride0, int tokens, int num_experts, int top_k, int norm_topk,
                              int32_t* topk_ids, float* topk_weights, void* stream) {
    if (!logits || !topk_ids || !topk_weights || tokens < 0 || num_experts <= 0 || top_k <= 0) return B200_EINVAL;
    if (((uintptr_t)logits & 1) || ((uintptr_t)topk_ids & 3) || ((uintptr_t)topk_weights & 3) || logits_stride0 < num_experts)
        return B200_EINVAL;
    if (num_experts > MOE_MAX_EXPERTS || top_k > MOE_MAX_TOPK || top_k > num_experts) return B200_EUNSUPPORTED;
    if (tokens == 0) return B200_OK;
    const int64_t blocks = ((int64_t)tokens + 7) / 8;
    if (blocks > 0x7fffffff) return B200_EUNSUPPORTED;
    B200_LAUNCH((moe_route_kernel), (unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream),
                static_cast<const __nv_bfloat16*>(logits), logits_stride0, tokens, num_experts, top_k, norm_topk ? 1 : 0, topk_ids,
                topk_weights);
    return b200_launch_status(nullptr);
}

extern "C" int b200_moe_align(const int32_t* topk_ids, int entries, int num_experts, int32_t* perm, int32_t* tiles, int max_tiles,
                              void* stream) {
    if (!topk_ids || !perm || !tiles || entries < 0 || num_experts <= 0) return B200_EINVAL;
    if (((uintptr_t)topk_ids & 3) || ((uintptr_t)perm & 3) || ((uintptr_t)tiles & 15)) return B200_EINVAL;
    if (num_experts > MOE_MAX_EXPERTS) return B200_EUNSUPPORTED;
    if (max_tiles < b200_moe_max_tiles(entries, num_experts)) return B200_EWORKSPACE;
    B200_LAUNCH((moe_align_kernel), 1, ALIGN_THREADS, 0, static_cast<cudaStream_t>(stream), topk_ids, entries, num_experts, perm,
                reinterpret_cast<int4*>(tiles));
    return b200_launch_status(nullptr);
}

extern "C" int b200_moe_gather(const void* x, int64_t x_stride0, int tokens, int hidden, int top_k, const int32_t* perm,
                               void* x_perm, void* stream) {
    if (!x || !perm || !x_perm || tokens < 0 || hidden <= 0 || top_k <= 0) return B200_EINVAL;
    if (((uintptr_t)x & 15) || ((uintptr_t)x_perm & 15) || ((uintptr_t)perm & 3) || (x_stride0 % 8) || x_stride0 < hidden)
        return B200_EINVAL;
    if (hidden % 8) return B200_EUNSUPPORTED;
    const int64_t entries = (int64_t)tokens * top_k;
    if (entries == 0) return B200_OK;
    if (entries > 0x7fffffff / 32) return B200_EUNSUPPORTED;
    B200_LAUNCH((moe_gather_kernel), (unsigned)((entries + 7) / 8), 256, 0, static_cast<cudaStream_t>(stream),
                static_cast<const __nv_bfloat16*>(x), x_stride0, (int)entries, top_k, hidden / 8, perm,
                static_cast<__nv_bfloat16*>(x_perm));
    return b200_launch_status(nullptr);
}

extern "C" int b200_moe_combine(const void* y, const int32_t* perm, const float* topk_weights, int tokens, int hidden, int top_k,
                                void* out, int64_t out_stride0, void* stream) {
    if (!y || !perm || !topk_weights || !out || tokens < 0 || hidden <= 0 || top_k <= 0) return B200_EINVAL;
    if (((uintptr_t)y & 15) || ((uintptr_t)out & 15) || ((uintptr_t)perm & 3) || ((uintptr_t)topk_weights & 3) || (out_stride0 % 8) ||
        out_stride0 < hidden)
        return B200_EINVAL;
    if (hidden % 8 || top_k > MOE_MAX_TOPK) return B200_EUNSUPPORTED;
    if (tokens == 0) return B200_OK;
    B200_LAUNCH((moe_combine_kernel), (unsigned)tokens, 256, 0, static_cast<cudaStream_t>(stream), static_cast<const __nv_bfloat16*>(y),
                perm, topk_weights, top_k, hidden / 8, static_cast<__nv_bfloat16*>(out), out_stride0);
    return b200_launch_status(nullptr);
}
