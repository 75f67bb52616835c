// Shared between the two decode kernels (decode_attn.cu: fp32-FMA formulation, decode_mma.cu: warp-level
// tensor-core formulation): launch parameters, the chunk cursor of the stream-K partition, constants.
#pragma once
#include "common.cuh"

namespace b200dec {

constexpr int CHUNK = 16;                          // tokens per pipeline stage
constexpr int ROW_BYTES = B200_HEAD_DIM * 2;       // one token of one kv head
constexpr int CHUNK_BYTES = CHUNK * ROW_BYTES;     // 4096
constexpr int MAX_BATCH = 1024;                    // sequences per launch (prefix table in smem)
constexpr int MIN_CHUNKS = 8;                      // smallest range handed to one warp (128 tokens)

struct DecodeParams {
    const __nv_bfloat16* q;
    int64_t q_stride;
    __nv_bfloat16* out;
    int64_t out_stride;
    const __nv_bfloat16* k_layer;
    const __nv_bfloat16* v_layer;
    const int32_t* block_tables;
    int bt_stride;
    const int32_t* context_lens;
    int batch;
    int hkv;
    int block_shift;
    float scale_log2;
    float* part_o;    // [slots][G][128]
    float* part_ml;   // [slots][G][2]
    int* counters;    // [batch * hkv], zero on entry, zero on exit
    // fused mode (b200_paged_decode_fused): q points at the raw qkv GEMM output; the kernel itself applies
    // q/k RMSNorm + RoPE and appends the step's K/V row to the cache
    const __nv_bfloat16* q_norm_w;
    const __nv_bfloat16* k_norm_w;
    const float* cos_sin;
    __nv_bfloat16* k_layer_w;   // writable aliases of k_layer / v_layer
    __nv_bfloat16* v_layer_w;
    float eps;
    int l2_hint;                // 1: K/V bulk copies carry an L2 evict_first policy (tuning knob)
    // fp8 binding (decode_mma.cu's fp8 kernel): the layer's e4m3 K / V bytes; the K scale is already in scale_log2
    const uint8_t* k8;
    const uint8_t* v8;
    float v_scale;
};

// Walks chunks in (sequence, kv head, chunk) order.  Warp-uniform.
struct ChunkCursor {
    int b, h, ck, n, ctx;
    __device__ __forceinline__ void seek(const int* cum, const int* ctxs, int batch, int hkv, long long c) {
        int key = (int)(c / hkv);
        int lo = 0, hi = batch;            // largest b with cum[b] <= key
        while (hi - lo > 1) {
            int mid = (lo + hi) >> 1;
            if (cum[mid] <= key) lo = mid; else hi = mid;
        }
        b = lo;
        n = cum[b + 1] - cum[b];
        ctx = ctxs[b];
        int rem = (int)(c - (long long)hkv * cum[b]);
        h = rem / n;
        ck = rem - h * n;
    }
    __device__ __forceinline__ void advance(const int* cum, const int* ctxs, int batch, int hkv) {
        if (++ck < n) return;
        ck = 0;
        if (++h < hkv) return;
        h = 0;
        do { ++b; } while (b < batch && cum[b + 1] == cum[b]);
        if (b < batch) { n = cum[b + 1] - cum[b]; ctx = ctxs[b]; }
    }
};


}  // namespace b200dec
