// C-ABI entry of the prefill branch of the reference's Attention.forward (nanovllm/layers/attention.py:64-70,
// flash_attn_varlen_func with an optional block_table).  The kernels themselves are the wgmma / TMA
// flash-attentions in prefill_tc.cu (default) and prefill_ws.cu; this file validates arguments and forwards.
#include <cstdlib>

#include "common.cuh"

int b200_prefill_tc_launch(b200_ctx* ctx, int layer, const void* q, int64_t q_stride0, const void* k, int64_t k_stride0,
                           const void* v, int64_t v_stride0, const int32_t* cu_q, const int32_t* cu_k,
                           const int32_t* block_tables, int bt_stride, void* out, int64_t out_stride0, int total_q,
                           int num_seqs, int max_seqlen_q, int num_q_heads, int num_kv_heads, float scale,
                           cudaStream_t stream);

int b200_prefill_ws_launch(b200_ctx* ctx, int layer, const void* q, int64_t q_stride0, const void* k, int64_t k_stride0,
                           const void* v, int64_t v_stride0, const int32_t* cu_q, const int32_t* cu_k,
                           const int32_t* block_tables, int bt_stride, void* out, int64_t out_stride0, int total_q,
                           int num_seqs, int max_seqlen_q, int num_q_heads, int num_kv_heads, float scale,
                           cudaStream_t stream);

// B200_PREFILL=ws selects the warp-specialised kernel (prefill_ws.cu: two q-heads of a GQA group per CTA, one consumer
// warpgroup per head and a TMA producer warp), B200_PREFILL=tc (or unset) the first-generation kernel (prefill_tc.cu).
// Read once.
static bool use_ws_kernel() {
    static const bool ws = [] {
        const char* e = getenv("B200_PREFILL");
        return e ? (e[0] == 'w') : false;
    }();
    return ws;
}

extern "C" int b200_paged_prefill(b200_ctx* ctx, int layer, const void* q, int64_t q_stride0,
                                  const void* k, int64_t k_stride0, const void* v,
                                  int64_t v_stride0, const int32_t* cu_seqlens_q,
                                  const int32_t* cu_seqlens_k, const int32_t* block_tables,
                                  int bt_stride, void* out, int64_t out_stride0, int total_q,
                                  int num_seqs, int max_seqlen_q, int max_seqlen_k,
                                  int num_q_heads, int num_kv_heads, float scale, void* stream) {
    (void)max_seqlen_k;
    if (!ctx || !q || !out || !cu_seqlens_q || !cu_seqlens_k || num_seqs < 0 || total_q < 0) return B200_EINVAL;
    if (num_kv_heads <= 0 || num_q_heads % num_kv_heads) return B200_EINVAL;
    if (total_q == 0 || num_seqs == 0 || max_seqlen_q <= 0) return B200_OK;
    if ((q_stride0 % 8) || (out_stride0 % 8) || ((uintptr_t)q & 15) || ((uintptr_t)out & 15)) return B200_EINVAL;
    if (block_tables) {
        if (!ctx->k_base) return B200_ENOTBOUND;
        if (layer < 0 || layer >= ctx->layers || num_kv_heads != ctx->num_kv_heads) return B200_EINVAL;
    } else {
        if (!k || !v || (k_stride0 % 8) || (v_stride0 % 8) || ((uintptr_t)k & 15) || ((uintptr_t)v & 15)) return B200_EINVAL;
    }
    if (use_ws_kernel())
        return b200_prefill_ws_launch(ctx, layer, q, q_stride0, k, k_stride0, v, v_stride0, cu_seqlens_q, cu_seqlens_k,
                                      block_tables, bt_stride, out, out_stride0, total_q, num_seqs, max_seqlen_q,
                                      num_q_heads, num_kv_heads, scale, static_cast<cudaStream_t>(stream));
    return b200_prefill_tc_launch(ctx, layer, q, q_stride0, k, k_stride0, v, v_stride0, cu_seqlens_q, cu_seqlens_k,
                                  block_tables, bt_stride, out, out_stride0, total_q, num_seqs, max_seqlen_q,
                                  num_q_heads, num_kv_heads, scale, static_cast<cudaStream_t>(stream));
}
