// The small bandwidth-bound ops around the attention operator, hand-written for sm_90a.
// They replace the reference's Triton KV scatter and its five @torch.compile sites (SURVEY.md 2b,
// K1 and K5-K8): fp32 math, one rounding at every stored output (what Inductor generates on a
// GPU), 128-bit coalesced global accesses, warp-shuffle reductions.
#include <cstdlib>

#include "common.cuh"

namespace {

constexpr int NORM_THREADS = 128;
constexpr int NORM_MAXV = 8;   // uint4 per thread -> cols <= 128 * 8 * 8 = 8192

__device__ __forceinline__ float block_sum_128(float v, float* red) {
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = red[0] + red[1] + red[2] + red[3];
    __syncthreads();
    return t;
}

// RMSNorm.rms_forward (layers/layernorm.py:16-26) when HAS_RES == false,
// RMSNorm.add_rms_forward (layers/layernorm.py:28-40) when true.
template <bool HAS_RES>
__global__ void __launch_bounds__(NORM_THREADS) rmsnorm_kernel(const __nv_bfloat16* __restrict__ x, int64_t x_stride,
                                                               __nv_bfloat16* residual,
                                                               const __nv_bfloat16* __restrict__ w,
                                                               __nv_bfloat16* out, int64_t out_stride, int cols,
                                                               float eps) {
    B200_PDL_SYNC();
    __shared__ float red[4];
    const int row = blockIdx.x;
    const int nvec = cols >> 3;
    const uint4* x4 = reinterpret_cast<const uint4*>(x + (int64_t)row * x_stride);
    uint4* r4 = HAS_RES ? reinterpret_cast<uint4*>(residual + (int64_t)row * cols) : nullptr;
    const uint4* w4 = reinterpret_cast<const uint4*>(w);
    uint4* o4 = reinterpret_cast<uint4*>(out + (int64_t)row * out_stride);

    float v[NORM_MAXV][8];
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < NORM_MAXV; ++k) {
        const int idx = threadIdx.x + k * NORM_THREADS;
        if (idx < nvec) {
            unpack8(x4[idx], v[k]);
            if (HAS_RES) {
                float r[8];
                unpack8(r4[idx], r);
#pragma unroll
                for (int e = 0; e < 8; ++e) v[k][e] += r[e];
                r4[idx] = pack8(v[k]);            // residual <- bf16(x + residual)
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) ss = fmaf(v[k][e], v[k][e], ss);
        }
    }
    const float tot = block_sum_128(ss, red);
    const float rstd = 1.0f / sqrtf(tot / (float)cols + eps);
#pragma unroll
    for (int k = 0; k < NORM_MAXV; ++k) {
        const int idx = threadIdx.x + k * NORM_THREADS;
        if (idx < nvec) {
            float wf[8], y[8];
            unpack8(w4[idx], wf);
#pragma unroll
            for (int e = 0; e < 8; ++e) y[e] = __fmul_rn(__fmul_rn(v[k][e], rstd), wf[e]);
            o4[idx] = pack8(y);
        }
    }
}

// Same two ops, one WARP per row (no block barrier) for rows of at most 2048 elements: a decode step has only a few
// hundred rows, so the kernel is pure latency and the shorter dependency chain wins.
template <bool HAS_RES, int NV>   // NV = uint4 per lane, cols = NV * 256
__global__ void __launch_bounds__(128) rmsnorm_warp_kernel(const __nv_bfloat16* __restrict__ x, int64_t x_stride,
                                                           __nv_bfloat16* residual, const __nv_bfloat16* __restrict__ w,
                                                           __nv_bfloat16* out, int64_t out_stride, int rows, float eps) {
    B200_PDL_SYNC();
    constexpr int cols = NV * 256;
    const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const uint4* x4 = reinterpret_cast<const uint4*>(x + (int64_t)row * x_stride);
    uint4* r4 = HAS_RES ? reinterpret_cast<uint4*>(residual + (int64_t)row * cols) : nullptr;
    const uint4* w4 = reinterpret_cast<const uint4*>(w);
    uint4* o4 = reinterpret_cast<uint4*>(out + (int64_t)row * out_stride);
    uint4 xin[NV], rin[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        xin[k] = x4[lane + k * 32];
        if (HAS_RES) rin[k] = r4[lane + k * 32];
    }
    float v[NV][8];
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        unpack8(xin[k], v[k]);
        if (HAS_RES) {
            float r[8];
            unpack8(rin[k], r);
#pragma unroll
            for (int e = 0; e < 8; ++e) v[k][e] += r[e];
            r4[lane + k * 32] = pack8(v[k]);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) ss = fmaf(v[k][e], v[k][e], ss);
    }
    ss = warp_sum(ss);
    const float rstd = 1.0f / sqrtf(ss / (float)cols + eps);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        float wf[8], y[8];
        unpack8(w4[lane + k * 32], wf);
#pragma unroll
        for (int e = 0; e < 8; ++e) y[e] = __fmul_rn(__fmul_rn(v[k][e], rstd), wf[e]);
        o4[lane + k * 32] = pack8(y);
    }
}

template <bool HAS_RES>
bool launch_rmsnorm_warp(const __nv_bfloat16* x, int64_t xs, __nv_bfloat16* res, const __nv_bfloat16* w, __nv_bfloat16* out,
                         int64_t os, int rows, int cols, float eps, cudaStream_t st) {
    static const int max_rows = [] { const char* e = getenv("B200_NORM_WARP_MAX_ROWS"); return e ? atoi(e) : 4096; }();
    if (cols % 256 || cols > 2048 || rows > max_rows) return false;   // beyond that the block-per-row kernel (tuning knob)
    const unsigned grid = (rows + 3) / 4;
    switch (cols / 256) {
        case 1: B200_LAUNCH((rmsnorm_warp_kernel<HAS_RES, 1>), grid, 128, 0, st, x, xs, res, w, out, os, rows, eps); return true;
        case 2: B200_LAUNCH((rmsnorm_warp_kernel<HAS_RES, 2>), grid, 128, 0, st, x, xs, res, w, out, os, rows, eps); return true;
        case 4: B200_LAUNCH((rmsnorm_warp_kernel<HAS_RES, 4>), grid, 128, 0, st, x, xs, res, w, out, os, rows, eps); return true;
        case 8: B200_LAUNCH((rmsnorm_warp_kernel<HAS_RES, 8>), grid, 128, 0, st, x, xs, res, w, out, os, rows, eps); return true;
        default: return false;
    }
}

// q_norm / k_norm (models/qwen3.py:82-84) + rotary_emb (layers/rotary_embedding.py:37-48) +
// store_kvcache (layers/attention.py:10-40) over the fused qkv GEMM output.  One HALF-warp per (token, head):
// lane j owns elements 8j..8j+7 (one 16-byte access), its rotation partner (element +-64) is lane j^8.
__global__ void __launch_bounds__(128) qknorm_rope_store_kernel(
    __nv_bfloat16* qkv, int64_t stride, int hq, int hkv, const int64_t* __restrict__ positions,
    const __nv_bfloat16* __restrict__ qw, const __nv_bfloat16* __restrict__ kw,
    const float* __restrict__ cos_sin, float eps, const int32_t* __restrict__ slot_mapping,
    __nv_bfloat16* k_cache, __nv_bfloat16* v_cache, int block_shift, int n) {
    B200_PDL_SYNC();
    const int heads = hq + 2 * hkv;
    const int64_t unit = ((int64_t)blockIdx.x * 128 + threadIdx.x) >> 4;        // (token, head) index
    const int j = threadIdx.x & 15;
    const int64_t total = (int64_t)n * heads;
    // the shuffles below involve whole warps: a warp whose second half-warp is past the end still runs them
    const bool live = unit < total;
    const int64_t u = live ? unit : total - 1;
    const int tok = (int)(u / heads);
    const int head = (int)(u - (int64_t)tok * heads);
    __nv_bfloat16* src = qkv + (int64_t)tok * stride + head * B200_HEAD_DIM + j * 8;

    int slot = -1;
    if (slot_mapping != nullptr && k_cache != nullptr) slot = slot_mapping[tok];
    const int64_t crow = slot < 0 ? 0
        : ((((int64_t)(slot >> block_shift)) * hkv) << block_shift) + (slot & ((1 << block_shift) - 1));   // + kvh << shift below

    const uint4 raw = *reinterpret_cast<const uint4*>(src);
    const bool is_v = head >= hq + hkv;
    const bool is_q = head < hq;
    float x[8];
    unpack8(raw, x);
    float ss = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) ss = fmaf(x[e], x[e], ss);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float rstd = 1.0f / sqrtf(ss / (float)B200_HEAD_DIM + eps);
    float wf[8];
    unpack8(*reinterpret_cast<const uint4*>((is_q ? qw : kw) + j * 8), wf);
    const float* cs = cos_sin + positions[tok] * B200_HEAD_DIM + (j & 7) * 8;
    const float4 c0 = *reinterpret_cast<const float4*>(cs), c1 = *reinterpret_cast<const float4*>(cs + 4);
    const float4 s0 = *reinterpret_cast<const float4*>(cs + 64), s1 = *reinterpret_cast<const float4*>(cs + 68);
    const float cosv[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    const float sinv[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    float y[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        // the reference's norm is its own kernel: its output is a stored bf16 tensor
        const float nv = round_bf16(__fmul_rn(__fmul_rn(x[e], rstd), wf[e]));
        const float other = __shfl_xor_sync(0xffffffffu, nv, 8);
        y[e] = (j < 8) ? __fsub_rn(__fmul_rn(nv, cosv[e]), __fmul_rn(other, sinv[e]))
                       : __fadd_rn(__fmul_rn(nv, cosv[e]), __fmul_rn(other, sinv[e]));
    }
    if (!live) return;
    if (is_v) {                                    // a value head: scatter only
        if (slot >= 0) {
            const int kvh = head - hq - hkv;
            *reinterpret_cast<uint4*>(v_cache + (crow + ((int64_t)kvh << block_shift)) * B200_HEAD_DIM + j * 8) = raw;
        }
        return;
    }
    const uint4 outv = pack8(y);
    *reinterpret_cast<uint4*>(src) = outv;
    if (!is_q && slot >= 0) {
        const int kvh = head - hq;
        *reinterpret_cast<uint4*>(k_cache + (crow + ((int64_t)kvh << block_shift)) * B200_HEAD_DIM + j * 8) = outv;
    }
}

// The same op for prefill-size batches: one HALF-warp per TOKEN walking over its heads.  Lane j owns the same 8 dims of
// every head, so positions / cos / sin / norm weights / the cache row are fetched once per token instead of once per
// (token, head), there is no 64-bit division, and U independent 16-byte loads per lane are in flight.
template <int U>
__global__ void __launch_bounds__(128) qknorm_rope_store_tok_kernel(
    __nv_bfloat16* qkv, int64_t stride, int hq, int hkv, const int64_t* __restrict__ positions,
    const __nv_bfloat16* __restrict__ qw, const __nv_bfloat16* __restrict__ kw,
    const float* __restrict__ cos_sin, float eps, const int32_t* __restrict__ slot_mapping,
    __nv_bfloat16* k_cache, __nv_bfloat16* v_cache, int block_shift, int n) {
    B200_PDL_SYNC();
    const int heads = hq + 2 * hkv;
    const int t_raw = blockIdx.x * 8 + (threadIdx.x >> 4);
    const bool live = t_raw < n;                       // a dead half-warp still takes part in the full-warp shuffles
    const int tok = live ? t_raw : n - 1;
    const int j = threadIdx.x & 15;
    __nv_bfloat16* row = qkv + (int64_t)tok * stride + j * 8;

    int slot = -1;
    if (slot_mapping != nullptr && k_cache != nullptr) slot = slot_mapping[tok];
    const int64_t crow = slot < 0 ? 0
        : ((((int64_t)(slot >> block_shift)) * hkv) << block_shift) + (slot & ((1 << block_shift) - 1));
    float qwf[8], kwf[8];
    unpack8(*reinterpret_cast<const uint4*>(qw + j * 8), qwf);
    unpack8(*reinterpret_cast<const uint4*>(kw + j * 8), kwf);
    const float* cs = cos_sin + positions[tok] * B200_HEAD_DIM + (j & 7) * 8;
    const float4 c0 = *reinterpret_cast<const float4*>(cs), c1 = *reinterpret_cast<const float4*>(cs + 4);
    const float4 s0 = *reinterpret_cast<const float4*>(cs + 64), s1 = *reinterpret_cast<const float4*>(cs + 68);
    const float cosv[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    const float sinv[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};

    for (int h0 = 0; h0 < heads; h0 += U) {
        uint4 raw[U];
#pragma unroll
        for (int u = 0; u < U; ++u)
            if (h0 + u < heads) raw[u] = *reinterpret_cast<const uint4*>(row + (h0 + u) * B200_HEAD_DIM);
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int head = h0 + u;
            if (head >= heads) break;                  // uniform across the warp
            if (head >= hq + hkv) {                    // a value head: scatter only
                if (live && slot >= 0)
                    *reinterpret_cast<uint4*>(v_cache + (crow + ((int64_t)(head - hq - hkv) << block_shift)) * B200_HEAD_DIM + j * 8) = raw[u];
                continue;
            }
            const bool is_q = head < hq;
            float x[8];
            unpack8(raw[u], x);
            float ss = 0.f;
#pragma unroll
            for (int e = 0; e < 8; ++e) ss = fmaf(x[e], x[e], ss);
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
            const float rstd = 1.0f / sqrtf(ss / (float)B200_HEAD_DIM + eps);
            float y[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float nv = round_bf16(__fmul_rn(__fmul_rn(x[e], rstd), is_q ? qwf[e] : kwf[e]));
                const float other = __shfl_xor_sync(0xffffffffu, nv, 8);
                y[e] = (j < 8) ? __fsub_rn(__fmul_rn(nv, cosv[e]), __fmul_rn(other, sinv[e]))
                               : __fadd_rn(__fmul_rn(nv, cosv[e]), __fmul_rn(other, sinv[e]));
            }
            if (live) {
                const uint4 outv = pack8(y);
                *reinterpret_cast<uint4*>(row + head * B200_HEAD_DIM) = outv;
                if (!is_q && slot >= 0)
                    *reinterpret_cast<uint4*>(k_cache + (crow + ((int64_t)(head - hq) << block_shift)) * B200_HEAD_DIM + j * 8) = outv;
            }
        }
    }
}

// store_kvcache_kernel (layers/attention.py:10-30): one warp per (token, kv head).
__global__ void __launch_bounds__(128) store_kv_kernel(const __nv_bfloat16* __restrict__ k, int64_t k_stride,
                                                       const __nv_bfloat16* __restrict__ v, int64_t v_stride,
                                                       const int32_t* __restrict__ slot_mapping,
                                                       __nv_bfloat16* k_cache, __nv_bfloat16* v_cache, int hkv,
                                                       int block_shift, int n) {
    B200_PDL_SYNC();
    const int64_t gwarp = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (gwarp >= (int64_t)n * hkv) return;
    const int tok = (int)(gwarp / hkv);
    const int kvh = (int)(gwarp - (int64_t)tok * hkv);
    const int lane = threadIdx.x & 31;
    const int slot = slot_mapping[tok];
    if (slot < 0) return;
    const int64_t row = ((((int64_t)(slot >> block_shift)) * hkv + kvh) << block_shift) + (slot & ((1 << block_shift) - 1));
    reinterpret_cast<uint2*>(k_cache + row * B200_HEAD_DIM)[lane] =
        reinterpret_cast<const uint2*>(k + (int64_t)tok * k_stride + kvh * B200_HEAD_DIM)[lane];
    reinterpret_cast<uint2*>(v_cache + row * B200_HEAD_DIM)[lane] =
        reinterpret_cast<const uint2*>(v + (int64_t)tok * v_stride + kvh * B200_HEAD_DIM)[lane];
}

// SiluAndMul.forward (layers/activation.py:8-11)
__global__ void __launch_bounds__(256) silu_mul_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* out,
                                                       int64_t total_vec, int inter_vec) {
    B200_PDL_SYNC();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total_vec; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = i / inter_vec;
        const int col = (int)(i - row * inter_vec);
        const uint4* xr = reinterpret_cast<const uint4*>(x) + row * 2 * inter_vec;
        float g[8], u[8], y[8];
        unpack8(xr[col], g);
        unpack8(xr[inter_vec + col], u);
#pragma unroll
        for (int e = 0; e < 8; ++e) y[e] = __fmul_rn(g[e] / (1.0f + expf(-g[e])), u[e]);
        reinterpret_cast<uint4*>(out)[i] = pack8(y);
    }
}

// F.embedding (layers/embed_head.py:38)
__global__ void __launch_bounds__(128) embedding_kernel(const int64_t* __restrict__ ids,
                                                        const __nv_bfloat16* __restrict__ table,
                                                        __nv_bfloat16* out, int hidden_vec, int64_t vocab) {
    B200_PDL_SYNC();
    const int tok = blockIdx.x;
    const int64_t id = ids[tok];
    uint4* dst = reinterpret_cast<uint4*>(out) + (int64_t)tok * hidden_vec;
    if (id < 0 || id >= vocab) {          // never read outside the table: an id that is not a token embeds to zeros
        for (int i = threadIdx.x; i < hidden_vec; i += 128) dst[i] = make_uint4(0, 0, 0, 0);
        return;
    }
    const uint4* src = reinterpret_cast<const uint4*>(table) + id * hidden_vec;
    for (int i = threadIdx.x; i < hidden_vec; i += 128) dst[i] = src[i];
}

__global__ void gather_tokens_kernel(int64_t* ids, const int32_t* __restrict__ src, const int64_t* __restrict__ prev, int n) {
    B200_PDL_SYNC();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const int s = src[i];
        if (s >= 0) ids[i] = prev[s];
    }
}

inline bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

extern "C" int b200_rmsnorm(const void* x, int64_t x_stride0, const void* weight, void* out,
                            int64_t out_stride0, int rows, int cols, float eps, void* stream) {
    if (!x || !weight || !out || rows < 0) return B200_EINVAL;
    if (cols <= 0 || cols % 8 || cols > NORM_THREADS * NORM_MAXV * 8) return B200_EUNSUPPORTED;
    if (x_stride0 % 8 || out_stride0 % 8 || !aligned16(x) || !aligned16(out) || !aligned16(weight)) return B200_EINVAL;
    if (rows == 0) return B200_OK;
    if (launch_rmsnorm_warp<false>(static_cast<const __nv_bfloat16*>(x), x_stride0, nullptr, static_cast<const __nv_bfloat16*>(weight),
                                   static_cast<__nv_bfloat16*>(out), out_stride0, rows, cols, eps, static_cast<cudaStream_t>(stream)))
        return b200_launch_status(nullptr);
    B200_LAUNCH((rmsnorm_kernel<false>), rows, NORM_THREADS, 0, static_cast<cudaStream_t>(stream), 
        static_cast<const __nv_bfloat16*>(x), x_stride0, nullptr, static_cast<const __nv_bfloat16*>(weight),
        static_cast<__nv_bfloat16*>(out), out_stride0, cols, eps);
    return b200_launch_status(nullptr);
}

extern "C" int b200_add_rmsnorm(const void* x, void* residual, const void* weight, void* out,
                                int rows, int cols, float eps, void* stream) {
    if (!x || !residual || !weight || !out || rows < 0) return B200_EINVAL;
    if (cols <= 0 || cols % 8 || cols > NORM_THREADS * NORM_MAXV * 8) return B200_EUNSUPPORTED;
    if (!aligned16(x) || !aligned16(out) || !aligned16(weight) || !aligned16(residual)) return B200_EINVAL;
    if (rows == 0) return B200_OK;
    if (launch_rmsnorm_warp<true>(static_cast<const __nv_bfloat16*>(x), cols, static_cast<__nv_bfloat16*>(residual),
                                  static_cast<const __nv_bfloat16*>(weight), static_cast<__nv_bfloat16*>(out), cols, rows, cols, eps,
                                  static_cast<cudaStream_t>(stream)))
        return b200_launch_status(nullptr);
    B200_LAUNCH((rmsnorm_kernel<true>), rows, NORM_THREADS, 0, static_cast<cudaStream_t>(stream), 
        static_cast<const __nv_bfloat16*>(x), cols, static_cast<__nv_bfloat16*>(residual),
        static_cast<const __nv_bfloat16*>(weight), static_cast<__nv_bfloat16*>(out), cols, cols, eps);
    return b200_launch_status(nullptr);
}

extern "C" int b200_qknorm_rope_store(b200_ctx* ctx, int layer, void* qkv, int64_t qkv_stride0,
                                      int num_q_heads, int num_kv_heads, const int64_t* positions,
                                      const void* q_norm_weight, const void* k_norm_weight,
                                      const float* cos_sin, float eps, const int32_t* slot_mapping,
                                      int n, void* stream) {
    if (!ctx || !qkv || !positions || !q_norm_weight || !k_norm_weight || !cos_sin || n < 0) return B200_EINVAL;
    if (qkv_stride0 % 8 || !aligned16(qkv)) return B200_EINVAL;
    if (n == 0) return B200_OK;
    __nv_bfloat16 *kc = nullptr, *vc = nullptr;
    int shift = 0;
    if (slot_mapping != nullptr && ctx->k_base != nullptr) {
        if (layer < 0 || layer >= ctx->layers || num_kv_heads != ctx->num_kv_heads) return B200_EINVAL;
        kc = ctx->k_layer(layer);
        vc = ctx->v_layer(layer);
        shift = ctx->block_shift;
    }
    static const int tok_min = [] { const char* e = getenv("B200_QKNORM_TOK_MIN"); return e ? atoi(e) : 2048; }();
    if (n >= tok_min) {             // prefill-size batch: one half-warp per token (see the kernel)
        B200_LAUNCH((qknorm_rope_store_tok_kernel<8>), (unsigned)((n + 7) / 8), 128, 0, static_cast<cudaStream_t>(stream),
            static_cast<__nv_bfloat16*>(qkv), qkv_stride0, num_q_heads, num_kv_heads, positions,
            static_cast<const __nv_bfloat16*>(q_norm_weight), static_cast<const __nv_bfloat16*>(k_norm_weight),
            cos_sin, eps, slot_mapping, kc, vc, shift, n);
        return b200_launch_status(ctx);
    }
    const int64_t units = (int64_t)n * (num_q_heads + 2 * num_kv_heads);       // one half-warp each, 8 per block
    const unsigned blocks = (unsigned)((units + 7) / 8);
    B200_LAUNCH((qknorm_rope_store_kernel), blocks, 128, 0, static_cast<cudaStream_t>(stream), 
        static_cast<__nv_bfloat16*>(qkv), qkv_stride0, num_q_heads, num_kv_heads, positions,
        static_cast<const __nv_bfloat16*>(q_norm_weight), static_cast<const __nv_bfloat16*>(k_norm_weight),
        cos_sin, eps, slot_mapping, kc, vc, shift, n);
    return b200_launch_status(ctx);
}

extern "C" int b200_store_kv(b200_ctx* ctx, int layer, const void* k, int64_t k_stride0,
                             const void* v, int64_t v_stride0, const int32_t* slot_mapping, int n,
                             void* stream) {
    if (!ctx || !k || !v || !slot_mapping || n < 0) return B200_EINVAL;
    if (!ctx->k_base) return B200_ENOTBOUND;
    if (layer < 0 || layer >= ctx->layers) return B200_EINVAL;
    if (k_stride0 % 4 || v_stride0 % 4 || ((uintptr_t)k & 7) || ((uintptr_t)v & 7)) return B200_EINVAL;
    if (n == 0) return B200_OK;
    const int64_t warps = (int64_t)n * ctx->num_kv_heads;
    B200_LAUNCH((store_kv_kernel), (unsigned)((warps + 3) / 4), 128, 0, static_cast<cudaStream_t>(stream), 
        static_cast<const __nv_bfloat16*>(k), k_stride0, static_cast<const __nv_bfloat16*>(v), v_stride0,
        slot_mapping, ctx->k_layer(layer), ctx->v_layer(layer), ctx->num_kv_heads, ctx->block_shift, n);
    return b200_launch_status(ctx);
}

extern "C" int b200_silu_mul(const void* x, void* out, int rows, int inter, void* stream) {
    if (!x || !out || rows < 0) return B200_EINVAL;
    if (inter <= 0 || inter % 8 || !aligned16(x) || !aligned16(out)) return B200_EINVAL;
    if (rows == 0) return B200_OK;
    const int64_t total = (int64_t)rows * (inter / 8);
    int64_t blocks = (total + 255) / 256;
    const int64_t cap = (int64_t)b200_current_sm_count() * 16;         // grid-stride beyond 16 CTAs per SM
    if (blocks > cap) blocks = cap;
    B200_LAUNCH((silu_mul_kernel), (unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream), 
        static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(out), total, inter / 8);
    return b200_launch_status(nullptr);
}

extern "C" int b200_embedding(const int64_t* ids, const void* table, void* out, int n, int hidden, int64_t vocab,
                              void* stream) {
    if (!ids || !table || !out || n < 0 || vocab <= 0) return B200_EINVAL;
    if (hidden <= 0 || hidden % 8 || !aligned16(table) || !aligned16(out)) return B200_EINVAL;
    if (n == 0) return B200_OK;
    B200_LAUNCH((embedding_kernel), n, 128, 0, static_cast<cudaStream_t>(stream), 
        ids, static_cast<const __nv_bfloat16*>(table), static_cast<__nv_bfloat16*>(out), hidden / 8, vocab);
    return b200_launch_status(nullptr);
}

extern "C" int b200_gather_tokens(int64_t* ids, const int32_t* src, const int64_t* prev_tokens, int n, void* stream) {
    if (!ids || !src || !prev_tokens || n < 0) return B200_EINVAL;
    if (n == 0) return B200_OK;
    B200_LAUNCH((gather_tokens_kernel), (n + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream), ids, src, prev_tokens, n);
    return b200_launch_status(nullptr);
}
