/*
 * b200_paged_attn.h -- C ABI of libb200attn.so, the H100 (sm_90a) paged-attention path that
 * drops in behind nano-vLLM's attention operator and the small fused ops around it.
 *
 * Every entry point cites the reference interface (GeeeekExplorer/nano-vllm @ bb823b3e) it
 * replaces.  The reference has no FFI layer of its own: its seams are Python-level
 * (SURVEY.md section 8b), so this header is the binding a maintainer would load with ctypes
 * (see INTEGRATION.md).
 *
 * Conventions
 *   - returns 0 on success, a negative B200_E* code otherwise (b200_strerror names it);
 *   - the caller owns every buffer (device pointers from the PyTorch allocator);
 *     the library allocates nothing after b200_init / b200_kv_bind;
 *   - nothing synchronises the host; every launch goes to the stream passed in, so a whole
 *     decode step is CUDA-graph capturable; per-step variation flows only through
 *     device-resident metadata (block_tables, context_lens, slot_mapping, cu_seqlens);
 *   - no C++ or torch types cross the boundary; `stream` is a cudaStream_t passed as void*;
 *   - one b200_ctx per process/GPU, not thread-safe (one engine thread per rank, like the
 *     reference's ModelRunner, engine/model_runner.py:17-48).
 *
 * Dtypes match the tensors the reference builds (engine/model_runner.py:129-188):
 *   activations / caches  bf16;   input_ids, positions  int64;
 *   slot_mapping, context_lens, block_tables, cu_seqlens  int32.
 *
 * KV-cache layout in HBM (ours; only block ids and slot numbers are contract):
 *   k_base, v_base : [layers][num_blocks][num_kv_heads][block_size][head_dim] bf16
 *   slot s  ->  block = s / block_size, row = s % block_size   (model_runner.py:151-161,181)
 *   so one (block, kv head) page is block_size*head_dim*2 contiguous bytes.
 */
#ifndef B200_PAGED_ATTN_H
#define B200_PAGED_ATTN_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200_ctx b200_ctx;

enum {
    B200_OK = 0,
    B200_EINVAL = -1,       /* bad argument (null pointer, unsupported shape) */
    B200_EUNSUPPORTED = -2, /* head_dim != 128, group size not in {1,2,4,8}, block_size not a power of two in [16,256] */
    B200_ECUDA = -3,        /* a CUDA runtime call failed; b200_last_cuda_error() has the text */
    B200_ENOTBOUND = -4,    /* KV cache not bound (b200_kv_bind) */
    B200_EWORKSPACE = -5,   /* workspace too small */
    B200_EARCH = -6         /* device is not compute capability 9.0 */
};

/* ---- lifetime ------------------------------------------------------------------------- */

/* Replaces the device setup in ModelRunner.__init__ (engine/model_runner.py:26-30): selects
 * `device`, checks it is sm_90, records the SM count.  */
int b200_init(int device, b200_ctx** out);
void b200_destroy(b200_ctx* ctx);
const char* b200_strerror(int code);
const char* b200_last_cuda_error(b200_ctx* ctx);
int b200_sm_count(const b200_ctx* ctx);
/* Per calling host thread: enabled == 0 makes every following launch of this library a plain stream-ordered launch
 * (no programmatic-dependent-launch attribute) until it is enabled again; returns the previous setting.  No reference
 * counterpart (the reference has no native launches): used around the kernels that follow a cross-stream event wait in
 * the two-stream decode step.  A no-op in the library flavour built without PDL. */
int b200_set_pdl(int enabled);
/* ABI version of this header; bumped on any signature change. */
int b200_abi_version(void);

/* Replaces the per-module k_cache / v_cache binding of ModelRunner.allocate_kv_cache
 * (engine/model_runner.py:103-121).  The caller allocates 2 * layers * num_blocks * num_kv_heads *
 * block_size * head_dim bf16 elements (layout above) and hands over the two base pointers. */
int b200_kv_bind(b200_ctx* ctx, void* k_base, void* v_base, int layers, int64_t num_blocks,
                 int block_size, int num_kv_heads, int head_dim);

/* The same binding over an fp8 (e4m3, OCP "fn" flavour) cache: same layout with 1-byte elements, so the caller allocates
 * 2 * layers * num_blocks * num_kv_heads * block_size * head_dim bytes.  vLLM's kv_cache_dtype="fp8" (no reference
 * counterpart).  Every cache write stores e4m3_satfinite_rn(x / scale) of the bf16 value the bf16 binding would store
 * (k_scale for keys, v_scale for values; out-of-range values saturate to +-448); every read uses float(e4m3) * scale.
 * Scales must be finite and > 0 (B200_EINVAL otherwise).  On such a binding:
 *   b200_store_kv, b200_qknorm_rope_store   quantize;
 *   b200_paged_decode                       runs the tensor-core kernel's fp8 variant for every head group;
 *   b200_paged_decode_fused                 returns B200_EUNSUPPORTED (use b200_qknorm_rope_store + b200_paged_decode);
 *   b200_paged_prefill with block_tables    returns B200_EUNSUPPORTED: dequantize with b200_kv_gather and run
 *                                           b200_prefill_packed_kv on the packed bf16 rows. */
int b200_kv_bind_fp8(b200_ctx* ctx, void* k_base, void* v_base, int layers, int64_t num_blocks, int block_size,
                     int num_kv_heads, int head_dim, float k_scale, float v_scale);

/* Dequantizes keys and values 0..len_k(s)-1 of each of num_seqs sequences of an fp8 binding (b200_kv_bind_fp8) into
 * packed bf16 rows: row r of sequence s goes to k_out / v_out row cu_seqlens_k[s] + r ([total_k, num_kv_heads, head_dim],
 * row strides in elements), value bf16(float(e4m3) * scale).  len_k(s) = cu_seqlens_k[s+1] - cu_seqlens_k[s]; pages
 * through block_tables[s] (row stride bt_stride) as b200_paged_prefill reads them.  total_k = cu_seqlens_k[num_seqs].
 * B200_EUNSUPPORTED on a bf16 binding. */
int b200_kv_gather(b200_ctx* ctx, int layer, const int32_t* block_tables, int bt_stride, const int32_t* cu_seqlens_k,
                   int num_seqs, void* k_out, int64_t k_stride0, void* v_out, int64_t v_stride0, int total_k,
                   void* stream);

/* Bytes of scratch b200_paged_decode needs for batches up to max_batch with num_q_heads query
 * heads.  The caller zero-fills it once (and again after a b200_kv_bind that changes num_kv_heads: the
 * layout depends on it); every launch leaves its counters zeroed. */
size_t b200_decode_workspace_bytes(const b200_ctx* ctx, int max_batch, int num_q_heads);

/* ---- the attention operator (layers/attention.py) -------------------------------------- */

/* store_kvcache (layers/attention.py:10-40): for i < n with slot_mapping[i] != -1 copy
 * k[i] (num_kv_heads*head_dim bf16, row stride k_stride0 elements) and v[i] into slot
 * slot_mapping[i] of layer `layer`. */
int b200_store_kv(b200_ctx* ctx, int layer, const void* k, int64_t k_stride0, const void* v,
                  int64_t v_stride0, const int32_t* slot_mapping, int n, void* stream);

/* Decode branch of Attention.forward (layers/attention.py:71-74), i.e.
 * flash_attn_with_kvcache(q.unsqueeze(1), k_cache, v_cache, cache_seqlens=context_lens,
 * block_table=block_tables, softmax_scale=scale, causal=True):
 *   out[b,h,:] = softmax(scale * q[b,h,:] K_b^T) V_b over keys 0..context_lens[b]-1 reached
 *   through block_tables[b, j / block_size].  Rows with context_lens[b] == 0 (graph padding,
 *   model_runner.py:207) write zeros.
 * q, out: [batch, num_q_heads, head_dim] bf16 with row strides in elements. */
int b200_paged_decode(b200_ctx* ctx, int layer, const void* q, int64_t q_stride0,
                      const int32_t* block_tables, int bt_stride, const int32_t* context_lens,
                      void* out, int64_t out_stride0, int batch, int num_q_heads, float scale,
                      void* workspace, size_t workspace_bytes, void* stream);

/* One-launch decode layer front end: what Qwen3Attention.forward does between the qkv GEMM and o_proj for a decode
 * step (models/qwen3.py:77-86 + layers/attention.py:62-63,71-74): q_norm / k_norm (RMSNorm over head_dim, rounded
 * to bf16), NeoX RoPE at position context_lens[b]-1 (cos_sin: fp32 [max_pos, head_dim] = cat(cos, sin)), the step's
 * K/V row appended to slot block_tables[b, (ctx-1)/block_size]*block_size + (ctx-1)%block_size of `layer` -- the slot
 * ModelRunner.prepare_decode computes (model_runner.py:181) -- and attention over keys 0..ctx-1.
 * qkv: the raw fused projection output [batch, (num_q_heads + 2*num_kv_heads) * head_dim] bf16 (not modified).
 * Same result as b200_qknorm_rope_store followed by b200_paged_decode, one kernel instead of two.
 * Only for num_q_heads / num_kv_heads <= 2 (B200_EUNSUPPORTED otherwise). */
int b200_paged_decode_fused(b200_ctx* ctx, int layer, const void* qkv, int64_t qkv_stride0,
                            const void* q_norm_weight, const void* k_norm_weight, const float* cos_sin,
                            float eps, const int32_t* block_tables, int bt_stride,
                            const int32_t* context_lens, void* out, int64_t out_stride0, int batch,
                            int num_q_heads, float scale, void* workspace, size_t workspace_bytes,
                            void* stream);

/* Prefill branch of Attention.forward (layers/attention.py:64-70), i.e.
 * flash_attn_varlen_func(q, k, v, cu_seqlens_q/k, max_seqlen_q/k, softmax_scale=scale,
 * causal=True, block_table=block_tables): bottom-right aligned causal mask, query i of a
 * sequence sees keys j <= i + len_k - len_q.
 *   block_tables == NULL : k, v are the packed [total_k, num_kv_heads, head_dim] rows
 *                          (row strides in elements), cu_seqlens_k indexes them.
 *   block_tables != NULL : prefix-cache hit / chunked prefill (attention.py:65-66): keys and
 *                          values are read from the bound cache of `layer`; k, v ignored. */
int b200_paged_prefill(b200_ctx* ctx, int layer, const void* q, int64_t q_stride0, const void* k,
                       int64_t k_stride0, const void* v, int64_t v_stride0,
                       const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k,
                       const int32_t* block_tables, int bt_stride, void* out, int64_t out_stride0,
                       int total_q, int num_seqs, int max_seqlen_q, int max_seqlen_k,
                       int num_q_heads, int num_kv_heads, float scale, void* stream);

/* The packed form of b200_paged_prefill (block_tables == NULL) when keys outnumber queries: sequence s attends
 * len_k(s) = cu_seqlens_k[s+1] - cu_seqlens_k[s] >= len_q(s) keys at rows cu_seqlens_k[s].. of k, v
 * ([total_k, num_kv_heads, head_dim], total_k = cu_seqlens_k[num_seqs]), same bottom-right aligned causal mask.  This is
 * the prefix-hit / chunked prefill over an fp8 cache once b200_kv_gather has dequantized its keys and values (in
 * b200_paged_prefill's packed mode the keys are the step's own rows, so total_k = total_q there). */
int b200_prefill_packed_kv(b200_ctx* ctx, const void* q, int64_t q_stride0, const void* k, int64_t k_stride0,
                           const void* v, int64_t v_stride0, const int32_t* cu_seqlens_q, const int32_t* cu_seqlens_k,
                           void* out, int64_t out_stride0, int total_q, int total_k, int num_seqs, int max_seqlen_q,
                           int num_q_heads, int num_kv_heads, float scale, void* stream);

/* ---- the fused ops around it (the reference's five @torch.compile sites) ---------------- */

/* RMSNorm.rms_forward (layers/layernorm.py:16-26): out = x * rsqrt(mean(x^2)+eps) * w, fp32
 * math, one rounding.  x/out: [rows, cols] bf16 with row strides. */
int b200_rmsnorm(const void* x, int64_t x_stride0, const void* weight, void* out,
                 int64_t out_stride0, int rows, int cols, float eps, void* stream);

/* RMSNorm.add_rms_forward (layers/layernorm.py:28-40): residual <- bf16(x + residual);
 * out = norm(x + residual) * w with the variance taken on the un-rounded fp32 sum. */
int b200_add_rmsnorm(const void* x, void* residual, const void* weight, void* out, int rows,
                     int cols, float eps, void* stream);

/* q_norm + k_norm + rotary_emb + store_kvcache of Qwen3Attention.forward (models/qwen3.py:82-86,
 * layers/rotary_embedding.py:37-48, layers/attention.py:62-63) in one pass over the fused qkv
 * GEMM output: per token, per head RMSNorm over head_dim (rounded to bf16 as the reference's
 * separate kernel does), NeoX rotation with cos_sin[positions[i]] (fp32 [max_pos, head_dim] =
 * cat(cos, sin)), q and k rewritten in place, k and v scattered to slot_mapping[i] of `layer`
 * when slot_mapping != NULL and a cache is bound.
 * qkv: [n, (num_q_heads + 2*num_kv_heads) * head_dim] bf16, row stride qkv_stride0. */
int b200_qknorm_rope_store(b200_ctx* ctx, int layer, void* qkv, int64_t qkv_stride0,
                           int num_q_heads, int num_kv_heads, const int64_t* positions,
                           const void* q_norm_weight, const void* k_norm_weight,
                           const float* cos_sin, float eps, const int32_t* slot_mapping, int n,
                           void* stream);

/* Tensor-parallel exchange fused with the op that follows it: dist.all_reduce after o_proj / down_proj
 * (RowParallelLinear.forward, layers/linear.py:152-156) + RMSNorm.add_rms_forward (layers/layernorm.py:28-40) in one
 * kernel over NVLink peer memory.  Every rank has written its partial GEMM output [rows, cols] bf16 at byte offset
 * data_offset of its slice of a symmetric (peer-mapped) allocation; peer_bases_dev is a DEVICE array of `world`
 * pointers to the slices' bases (e.g. torch symmetric memory's buffer_ptrs_dev); int32 flags[world] live at
 * flag_offset of every slice (zeroed once); epoch / done are two private zero-initialised device words; *err_flag
 * (device int, may be NULL) is set to 1 if a peer did not announce itself within ~18 s (the launch then completes with
 * undefined output instead of spinning forever).  Computes, on every rank, bit-identically:
 *   s = (((residual + partial_0) + partial_1) + ... + partial_{world-1}),  every addition in fp32, in that order;
 *   residual <- bf16(s), the one rounding;  out = bf16(s * rsqrt(mean(s^2) + eps) * weight).
 * The residual comes first and the partials follow in rank order whichever rank computes: that fixed order is what
 * makes the ranks agree bit for bit.  Callers alternate two data offsets between consecutive calls (see
 * csrc/tp_allreduce.cu for the protocol). */
int b200_allreduce_add_rmsnorm(const void* peer_bases_dev, uint64_t data_offset, uint64_t flag_offset,
                               int* epoch, unsigned int* done, int* err_flag, int rank, int world,
                               void* residual, const void* weight, void* out, int rows, int cols, float eps,
                               void* stream);

/* The same exchange with the sum taken inside the NVSwitch (NVLS; the engine's default from 4 ranks): partials are read
 * through `multicast_base`, the multicast mapping of the same symmetric allocation, with multimem.ld_reduce (fp32
 * accumulation in the switch, ONE rounding to bf16 -- the rounding point of the reference's bf16 all_reduce), so a
 * rank moves `rows x cols x 2` bytes instead of world times that.  Handshake, arguments and outputs as above, except
 * that residual <- bf16(residual + bf16(sum_p partial_p)). */
int b200_allreduce_add_rmsnorm_nvls(const void* peer_bases_dev, const void* multicast_base, uint64_t data_offset,
                                    uint64_t flag_offset, int* epoch, unsigned int* done, int* err_flag, int rank,
                                    int world, void* residual, const void* weight, void* out, int rows, int cols,
                                    float eps, void* stream);

/* SiluAndMul.forward (layers/activation.py:8-11): out[r, c] = silu(x[r, c]) * x[r, inter + c]. */
int b200_silu_mul(const void* x, void* out, int rows, int inter, void* stream);

/* F.embedding of VocabParallelEmbedding.forward (layers/embed_head.py:34-42), single shard.  `vocab` = rows of
 * `table`; an id outside [0, vocab) never reads outside the table: its output row is zeros (the reference's
 * F.embedding device-asserts there; callers validate ids on the host). */
int b200_embedding(const int64_t* ids, const void* table, void* out, int n, int hidden, int64_t vocab,
                   void* stream);

/* Feeds a decode step's input_ids straight from the previous step's sampled tokens, on the device:
 *   ids[i] = prev_tokens[src[i]]  where src[i] >= 0,  unchanged otherwise.
 * Replaces the host round trip of ModelRunner.prepare_decode (engine/model_runner.py:177, seq.last_token of a
 * token that was sampled one step earlier), so step N+1 can be enqueued before step N's tokens reach the host. */
int b200_gather_tokens(int64_t* ids, const int32_t* src, const int64_t* prev_tokens, int n, void* stream);

/* Sampler.forward (layers/sampler.py:7-12) plus the greedy branch the north-star adds:
 *   temperature[r] == 0 : out[r] = argmax_j logits[r, j]  (lowest index on ties)
 *   temperature[r]  > 0 : exponential race  argmax_j softmax(logits/t)_j / E_j,  E_j ~ Exp(1)
 *                         computed as argmax_j (logits[r,j]/t - log E_j), counter-based RNG
 *                         keyed by (seed, step, r, index_offset + j); when step_dev != NULL the
 *                         device value *step_dev is added to step at run time, so a captured
 *                         CUDA graph draws fresh noise on every replay.
 * logits: [rows, vocab] bf16 (logits_is_fp32 == 0) or fp32, row stride in elements.
 * out: [rows] int64 token ids = index_offset + winning column (the dtype Sampler returns).
 * Vocab-parallel use (replaces the dist.gather of ParallelLMHead.forward, layers/embed_head.py:62-65):
 * each rank passes its shard with index_offset = first vocab id of the shard and a non-NULL
 * out_keys; out_keys[r] is an int64 whose signed order is (winning score, then lower token id),
 * so one all-reduce(MAX) over ranks picks the global winner:
 *   token = 0xffffffff - (key & 0xffffffff).   out may be NULL when out_keys is given. */
int b200_sample(const void* logits, int logits_is_fp32, int64_t logits_stride0,
                const float* temperatures, int rows, int vocab, int64_t index_offset,
                uint64_t seed, uint64_t step, const int64_t* step_dev, int64_t* out,
                int64_t* out_keys, void* stream);

/* Top-k / top-p / min-p sampling (vLLM v1 semantics; the reference samples the full softmax only), bf16 logits only.
 * Per row r, with t = temperatures[r] and probabilities those of logits / t:
 *   top_k[r]  <= 0 or >= vocab: off;  else keep x_j >= the k-th largest logit (ties at the boundary kept)
 *   top_p[r]  >= 1: off;  else keep x_j iff the mass of the tokens with a strictly larger logit is < top_p[r] times
 *             the mass that survives top-k and min-p (ties at the boundary kept)
 *   min_p[r]  <= 0: off;  else keep x_j iff prob_j >= min_p[r] * prob_max
 * top_k / top_p / min_p may each be NULL (off for every row).  The kept set is {j : x_j >= tau} for one bf16 tau per
 * row, and the token is b200_sample's exponential race (same RNG, same keys) restricted to it.  Rows with t == 0
 * (greedy) or every filter off get exactly b200_sample's token.
 *
 * Call b200_sample_filter_stage with stage = 0, 1, 2, 3, then b200_sample_filtered, all on the same rows, logits and
 * workspace.  workspace: b200_sample_filter_workspace_words(rows) int64 words, zero before its first use; the last call
 * leaves it zero again except for the tau words.  Row r owns words [r * 1538, (r + 1) * 1538):
 *   word 0             written by stage 0, reduce with MAX: order-preserving key of the row maximum
 *   word 1             written by b200_sample_filtered: key of tau (bf16 bits b -> b ^ (b & 0x8000 ? 0xffff : 0x8000),
 *                      -0 as +0); every x with key(x) >= tau is kept.  Not part of any stage.
 *   words 2..513       written by stage 1, reduce with SUM (256 counts, then 256 fixed-point masses)
 *   words 514..1025    written by stage 2, reduce with SUM (same form)
 *   words 1026..1537   written by stage 3, reduce with SUM (same form)
 * Vocab-parallel use: each rank runs every stage on its shard and all-reduces that stage's words over the ranks before
 * the next call (every rank launches every stage, whatever its rows need); b200_sample_filtered then takes index_offset
 * and out_keys as b200_sample does, and one all-reduce(MAX) of out_keys picks the token.  The result is bit-identical
 * to the unsharded call.  The (global) vocabulary is at most 2^18 tokens (B200_EUNSUPPORTED above that).
 * B200_EINVAL: NULL logits / temperatures / workspace (or both out and out_keys), rows or vocab <= 0, stage outside
 * 0..3, logits not 16-byte aligned or a row stride not a multiple of 8. */
int64_t b200_sample_filter_workspace_words(int rows);
int b200_sample_filter_stage(const void* logits, int64_t logits_stride0, const float* temperatures, const int32_t* top_k,
                             const float* top_p, const float* min_p, int rows, int vocab, int stage, int64_t* workspace,
                             void* stream);
int b200_sample_filtered(const void* logits, int64_t logits_stride0, const float* temperatures, const int32_t* top_k,
                         const float* top_p, const float* min_p, int rows, int vocab, int64_t index_offset, uint64_t seed,
                         uint64_t step, const int64_t* step_dev, int64_t* workspace, int64_t* out, int64_t* out_keys,
                         void* stream);

/* Presence / frequency / repetition penalties (vLLM v1 semantics; the reference has none: they run on the logits before
 * Sampler.forward, layers/sampler.py:8-12, and before the filters above).  bf16 logits only, in place.
 *
 * History: num_slots slots of `capacity` int64 entries, plus lengths[num_slots] (int32).  An entry is one distinct token
 * of a sequence: token << 32 | in_prompt << 31 | c, where c counts the token's occurrences after the prompt.  A slot's
 * entries are distinct, so capacity = min(max_model_len, vocab) always suffices.
 *
 * b200_penalty_load: for every row with 0 <= slots[r] < num_slots, copies entries[offsets[r] .. offsets[r + 1]) into the
 *   slot and sets its length (clamped to capacity).  Rows with slot -1 do nothing.
 * b200_penalty_apply: for every row with 0 <= slots[r] < num_slots, in one pass over the slot's entries:
 *   1. absorbs the pending token pending[r] (skipped when pending is NULL or pending[r] < 0): the matching entry's count
 *      goes up by one, or, if no entry matches and the slot is not full, (pending[r] << 32) | 1 is appended;
 *   2. rewrites the logit of each entry's token j with index_offset <= j < index_offset + vocab, using the updated c_j:
 *        y = (in_prompt or c_j > 0) ? (x > 0 ? x / r : x * r) : x      (IEEE division, round to nearest)
 *        y = y - f * c_j                                               (rounded multiply, then rounded subtract)
 *        y = y - (c_j > 0 ? p : 0)
 *      in fp32, then bf16 round-to-nearest-even; r, f, p = repetition[r], frequency[r], presence[r].
 *   Every other logit keeps its bits.  Rows with slot -1 return at once.  Vocab-parallel use: every rank holds and
 *   absorbs the whole history and passes its shard with index_offset = its first vocab id.
 * B200_EINVAL: a NULL pointer (other than pending), rows <= 0 or > 1024, vocab / num_slots / capacity <= 0,
 *   index_offset < 0, misaligned logits, or a row stride < vocab with rows > 1. */
int b200_penalty_load(int64_t* history, int32_t* lengths, int num_slots, int capacity, const int64_t* entries,
                      const int32_t* offsets, const int32_t* slots, int rows, void* stream);
int b200_penalty_apply(void* logits, int64_t logits_stride0, int rows, int vocab, int64_t index_offset, int64_t* history,
                       int32_t* lengths, int num_slots, int capacity, const int32_t* slots, const int64_t* pending,
                       const float* repetition, const float* frequency, const float* presence, void* stream);

/* Per-token logprobs of the raw logits (vLLM v1's raw_logprobs; the reference has none).  bf16 logits only.
 * Per row r with k[r] >= 0 (k[r] = -1: off, every call returns at once for the row; k above 20 is taken as 20), over the
 * logits as the LM head wrote them (before penalties, temperature and filters):
 *   logprob(x) = (x - m) - ln(S * 2^-40), m = the row maximum, S = sum_j round(exp(x_j - m) * 2^40) (uint64, expf),
 *   computed in float64 and rounded once to fp32;
 *   rank = #{j : x_j >= x_t} for the sampled token t (at least 1; ties raise it);
 *   the top k: the k largest x_j, value descending then token id ascending.
 * Call order: b200_logprob_topk and (for penalised rows) b200_logprob_save before b200_penalty_apply; after the token is
 * known, b200_logprob_restore, b200_logprob_rank, b200_logprob_finish.  All on the same rows, k, logits and workspace.
 *
 * workspace: b200_logprob_workspace_words(rows) int64 words (0 for rows <= 0 or > 1024), zero before the first use; the
 * finish leaves every word of a logprob row zero again.  Row r owns words [r * 8, r * 8 + 8):
 *   word 0   written by b200_logprob_topk, reduce with MAX: order-preserving key of m (as word 1 of the filter workspace)
 *   word 1   written by b200_logprob_restore, reduce with MAX: key of x_t (0 on a shard that does not hold t)
 *   word 2   written by b200_logprob_rank, reduce with SUM: S
 *   word 3   written by b200_logprob_rank, reduce with SUM: the rank
 *   word 4   number of saved pairs (b200_logprob_save -> b200_logprob_restore), local to the rank
 * topk_keys: int64 [rows, 20]; row r's first max(k[r], 1) words are its shard's largest logits as b200_sample keys
 *   (value << 32 | 0xffffffff - global id, order-preserving, -0 as +0), not accumulated: nothing to zero.
 * saved: int64 [rows, capacity + 1], the raw bf16 of every logit b200_penalty_apply will rewrite for the row (its slot's
 *   entries and the pending token, read as the apply reads them), as column << 16 | bits, -1 = none.
 * b200_logprob_restore writes them back (saved may be NULL when no row was penalised) and reads x_t from tokens[r].
 * b200_logprob_finish merges `sources` top-k lists, topk_keys being [sources, rows, 20], and writes per row:
 *   out_ids[r * out_stride + 0] = t, out_logprobs[... + 0] = logprob(x_t), out_rank[r * out_stride] = rank,
 *   out_ids / out_logprobs[r * out_stride + 1 + i], i < k[r]: the i-th largest token and its logprob.
 * Vocab-parallel use: each rank passes its shard with index_offset = its first vocab id, all-reduces word 0 (MAX) after
 * b200_logprob_topk, word 1 (MAX) after b200_logprob_restore, words 2-3 (SUM) after b200_logprob_rank, gathers topk_keys
 * over the ranks and passes sources = world.  The result is bit-identical to the unsharded call.
 * B200_EINVAL: a NULL pointer (other than pending and restore's saved), rows <= 0 or > 1024, vocab <= 0, index_offset
 *   < 0, logits not 16-byte aligned, a row stride not a multiple of 8 or < vocab with rows > 1, num_slots / capacity <= 0
 *   (save), sources outside 1..64 or out_stride < 21 (finish).  B200_EUNSUPPORTED: a global vocabulary above 2^18. */
int64_t b200_logprob_workspace_words(int rows);
int b200_logprob_topk(const void* logits, int64_t logits_stride0, const int32_t* k, int rows, int vocab, int64_t index_offset,
                      int64_t* workspace, int64_t* topk_keys, void* stream);
int b200_logprob_save(const void* logits, int64_t logits_stride0, const int32_t* k, int rows, int vocab, int64_t index_offset,
                      const int64_t* history, const int32_t* lengths, int num_slots, int capacity, const int32_t* slots,
                      const int64_t* pending, int64_t* workspace, int64_t* saved, void* stream);
int b200_logprob_restore(void* logits, int64_t logits_stride0, const int32_t* k, int rows, int vocab, int64_t index_offset,
                         const int64_t* tokens, int64_t* workspace, const int64_t* saved, int capacity, void* stream);
int b200_logprob_rank(const void* logits, int64_t logits_stride0, const int32_t* k, int rows, int vocab, int64_t* workspace,
                      void* stream);
int b200_logprob_finish(const int32_t* k, int rows, const int64_t* tokens, const int64_t* topk_keys, int sources,
                        int64_t* workspace, int32_t* out_ids, float* out_logprobs, int32_t* out_rank, int64_t out_stride,
                        void* stream);

/* ---- decode-size projections on the tensor cores (wgmma; tests/test_gpu_linear.py) ---------------------------------
 *
 * F.linear of the reference's *ParallelLinear layers (layers/linear.py:51,73,153) for small batches, on wgmma,
 * with what follows fused in (csrc/linear_tc.cu):
 *   x [rows, k] bf16 (row stride x_stride0), w [n, k] bf16 contiguous, k % 64 == 0.
 *   epilogue 0: out[rows, n_out] bf16 = bf16(x w^T)                                      (k_splits must be 1)
 *   epilogue 1: w is [2 * n_out, k] (gate rows then up rows, the reference's gate_up_proj);
 *               out[rows, n_out] = SiluAndMul(bf16(x w^T))  (layers/activation.py:8-11)  (k_splits must be 1)
 *   epilogue 2: out is fp32 [k_splits, rows, n_out] (out_stride0 = n_out): per-split partial sums, to be
 *               consumed in order by b200_add_rmsnorm_partials
 * block_n: accumulator columns per CTA, one of 16 (not for epilogue 1), 32, 64, 128; n_out must be a multiple of
 * block_n (block_n / 2 for epilogue 1).  flags bit 0: launch with programmatic stream serialization (the kernel
 * prefetches its weight tiles before waiting for the previous kernel in the stream). */
int b200_linear(const void* x, int64_t x_stride0, const void* w, void* out, int64_t out_stride0, int rows,
                int n_out, int k, int epilogue, int block_n, int k_splits, int flags, void* stream);

/* ---- block-scaled FP8 projections (Qwen / DeepSeek "fp8" checkpoints with weight_block_size [128, 128]) -------------
 *
 * b200_quant_fp8: dynamic activation quantization of x [rows, k] bf16 (row stride x_stride0, k % 128 == 0): per row and
 *   128-column group g, s = max(amax_g, 1e-10) / 448 and q = e4m3_satfinite_rn(x / s) (IEEE fp32 divisions);
 *   q [rows, k] e4m3 bytes (row stride q_stride0), scales [rows, k / 128] fp32 (row stride scales_stride0).
 * b200_linear_fp8: b200_linear on e4m3 operands.  x [rows, k] e4m3 (x_stride0 % 16 == 0) with x_scale from
 *   b200_quant_fp8; w [w_rows, k] e4m3 contiguous with w_scale [w_rows / 128, k / 128] fp32 contiguous (w_rows = n_out,
 *   2 * n_out for epilogue 1); k and n_out multiples of 128.  Each 128-wide block of K is summed by the tensor cores into
 *   a fresh fp32 partial, then acc += partial * (x_scale[row, kb] * w_scale[nb, kb]).  epilogue, k_splits and flags as
 *   b200_linear (k_splits divides k / 128); block_n one of 16 (not for epilogue 1), 32, 64. */
int b200_quant_fp8(const void* x, int64_t x_stride0, void* q, int64_t q_stride0, float* scales, int64_t scales_stride0,
                   int rows, int k, void* stream);
int b200_linear_fp8(const void* x, int64_t x_stride0, const float* x_scale, int64_t x_scale_stride0, const void* w,
                    const float* w_scale, void* out, int64_t out_stride0, int rows, int n_out, int k, int epilogue,
                    int block_n, int k_splits, int flags, void* stream);

/* ---- mixture-of-experts MLP of Qwen3 MoE checkpoints (Qwen3MoeSparseMoeBlock; csrc/moe.cu, DESIGN.md 3.7) -----------
 *
 * T tokens, E experts (E <= 256), top_k experts per token (top_k <= 16, top_k <= E); an entry is a (token t, rank j)
 * pair, entry index t * top_k + j.  Launch grids depend on T only, so a captured step serves every routing.
 * b200_moe_route: logits [T, E] bf16 (row stride logits_stride0 >= E) -> per token the top_k experts by fp32 softmax
 *   probability (expf; descending, ties to the lower expert id) in topk_ids [T, top_k] int32 and their fp32 probabilities in
 *   topk_weights [T, top_k], divided by their fp32 sum in rank order when norm_topk is non-zero.
 * b200_moe_max_tiles: rows of the tile table b200_moe_align may write for `entries` entries (ceil(entries / 128) +
 *   min(E, entries)), -1 on bad arguments.
 * b200_moe_align: from topk_ids [entries] -> perm [entries] int32, the row of every entry in the permuted buffer (one
 *   contiguous segment per expert, experts in id order, rows of a segment in no particular order), and the tile table
 *   tiles [1 + max_tiles] x int4 (16-byte aligned): {n_tiles, rows, 0, 0}, then per tile {expert, first row, end row, 0}
 *   of at most 128 rows.  B200_EWORKSPACE when max_tiles < b200_moe_max_tiles(entries, E).
 * b200_moe_gather: x_perm[perm[t top_k + j]] = x[t]; x [T, hidden] bf16 (row stride x_stride0), x_perm [T top_k, hidden]
 *   contiguous; hidden % 8 == 0.
 * b200_moe_linear: the grouped wgmma GEMM of b200_linear: out[r] = x[r] w_e^T for every row r of every tile of expert e,
 *   x [rows, k] bf16 contiguous (the permuted buffer, rows = T top_k), w [num_experts, w_rows, k] bf16 contiguous,
 *   out [rows, n_out] (row stride out_stride0); epilogue 0 (w_rows = n_out) or 1 (w_rows = 2 n_out: each expert's gate
 *   rows then its up rows, out = SiluAndMul), block_n as b200_linear; max_tiles as given to b200_moe_align; flags: bit 0
 *   PDL, bits 4-7 ring depth.
 * b200_moe_combine: out[t] = bf16(sum_j topk_weights[t, j] y[perm[t top_k + j]]), an fp32 fma chain in rank order j;
 *   y [T top_k, hidden] contiguous, out [T, hidden] (row stride out_stride0). */
int b200_moe_max_tiles(int entries, int num_experts);
int b200_moe_route(const void* logits, int64_t logits_stride0, int tokens, int num_experts, int top_k, int norm_topk,
                   int32_t* topk_ids, float* topk_weights, void* stream);
int b200_moe_align(const int32_t* topk_ids, int entries, int num_experts, int32_t* perm, int32_t* tiles, int max_tiles,
                   void* stream);
int b200_moe_gather(const void* x, int64_t x_stride0, int tokens, int hidden, int top_k, const int32_t* perm, void* x_perm,
                    void* stream);
int b200_moe_linear(const void* x, const void* w, void* out, int64_t out_stride0, int rows, int num_experts, int n_out, int k,
                    const int32_t* tiles, int max_tiles, int epilogue, int block_n, int flags, void* stream);
int b200_moe_combine(const void* y, const int32_t* perm, const float* topk_weights, int tokens, int hidden, int top_k,
                     void* out, int64_t out_stride0, void* stream);

/* (opt-in) ParallelLMHead.forward + Sampler.forward in one pass (layers/embed_head.py:56-66, layers/sampler.py:7-12):
 * logits = bf16(hidden lm_head^T) are produced tile by tile in registers, scored exactly as b200_sample scores
 * them (same RNG keyed by (seed, step, row, vocabulary id); temperature 0 = greedy, lowest index on ties) and
 * reduced to one packed (score, token) key per row with atomicMax -- the [rows, vocab] logits are never written.
 *   hidden [rows, k] bf16 (last-token rows), lm_head [vocab, k] bf16 contiguous (this rank's shard), k % 64 == 0;
 *   vocab may be ragged with respect to block_n (16/32/64/128); key_workspace: rows x uint64, ZERO on entry, left
 *   zero on exit (a second tiny kernel turns keys into out / out_keys and clears them);
 *   out / out_keys / index_offset / seed / step / step_dev: as b200_sample.  flags: as b200_linear. */
int b200_lm_head_sample(const void* hidden, int64_t hidden_stride0, const void* lm_head, int rows, int vocab, int k,
                        const float* temperatures, int64_t index_offset, uint64_t seed, uint64_t step,
                        const int64_t* step_dev, void* key_workspace, int64_t* out, int64_t* out_keys, int block_n,
                        int flags, void* stream);

/* RMSNorm.add_rms_forward (layers/layernorm.py:28-40) whose input is a split-K projection:
 *   h = bf16(sum_s partials[s]) in split order (deterministic), then as b200_add_rmsnorm.  cols <= 8192. */
int b200_add_rmsnorm_partials(const float* partials, int splits, void* residual, const void* weight, void* out,
                              int rows, int cols, float eps, int flags, void* stream);

/* The tail of a decoder layer for a decode-size batch on one GPU, as ONE persistent kernel (csrc/layer_tail.cu):
 *   o_proj -> residual add + RMSNorm -> gate_up_proj + SiluAndMul -> down_proj -> residual add + RMSNorm [-> next qkv_proj]
 * i.e. RowParallelLinear o_proj + RMSNorm.add_rms_forward + Qwen3MLP + the next layer's input_layernorm and
 * QKVParallelLinear (reference models/qwen3.py:72-76,87,91-117,146-159; layers/linear.py; layers/layernorm.py:28-40;
 * layers/activation.py:8-11).  Rounding points are the reference's: every projection is rounded to bf16 where F.linear's
 * output is bf16, the norms use the un-rounded fp32 sum.
 *   attn_out [rows, q_size] bf16 (row stride attn_stride0); residual [rows, hidden] bf16, updated in place (twice);
 *   w_o [hidden, q_size], w_gate_up [2*inter, hidden] (gate rows, then up rows), w_down [hidden, inter], bf16 contiguous;
 *   ln_mid / ln_next: the two RMSNorm weights; x_next [rows, hidden] bf16: the normalised input of the next layer;
 *   w_qkv_next [qkv_n, hidden] + qkv_out [rows, qkv_n] (row stride qkv_stride0): optional (NULL: stop after x_next);
 *   splits_o / splits_down: split-K factors of the two hidden-wide projections (partials are summed in split order);
 *   workspace: b200_layer_tail_workspace_bytes(rows, hidden, inter, max(splits)) bytes, 256-byte aligned, ZERO before
 *   the first use (it holds the grid-barrier state); rows <= 1024; hidden, q_size, inter multiples of 64.
 * Launched cooperatively (one CTA per SM, all resident); graph-capturable; a barrier that cannot complete sets the error
 * word at workspace + 8 instead of hanging. */
size_t b200_layer_tail_workspace_bytes(int max_rows, int hidden, int inter, int max_splits);
int b200_layer_tail(b200_ctx* ctx, const void* attn_out, int64_t attn_stride0, void* residual, const void* w_o,
                    const void* ln_mid, const void* w_gate_up, const void* w_down, const void* ln_next, void* x_next,
                    const void* w_qkv_next, void* qkv_out, int64_t qkv_stride0, int qkv_n, void* workspace,
                    size_t workspace_bytes, int rows, int hidden, int q_size, int inter, float eps, int splits_o,
                    int splits_down, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200_PAGED_ATTN_H */
