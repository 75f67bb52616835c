"""The fp8 (e4m3) KV-cache mode of the CPU oracle: the numeric contract of b200_kv_bind_fp8 restated in torch.

* store:       element = e4m3_satfinite_rn(float(x_bf16) / scale), x the bf16 value a bf16 cache would hold (the
               post-norm, post-RoPE key; the raw value).  torch's float -> float8_e4m3fn conversion turns values past
               448 into NaN where the hardware saturates, hence the clamp.
* decode:      reads every key and value of the cache as float(e4m3) * scale (fp32, no further rounding);
* prefill with block tables (prefix hit / chunked prefill): reads every key and value of the cache, this step's own
               included, dequantized to bf16 (what the engine's gather writes into its bf16 scratch);
* packed prefill (no block tables): attends the fresh bf16 K/V, as with a bf16 cache.

``Qwen3RefFp8`` is the oracle's Qwen3 forward with that operator; caches are logical [nblk, bs, Hkv, D] uint8 tensors
holding e4m3 bytes (``alloc_logical_kv_fp8``).
"""
from __future__ import annotations

from types import SimpleNamespace
from unittest import mock

import torch

from oracle import qwen3_ref
from oracle.paged_attention_ref import paged_decode_ref, store_kvcache_ref, varlen_prefill_ref
from oracle.qwen3_ref import Qwen3Ref

E4M3_MAX = 448.0


def quantize_e4m3(x: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """e4m3_satfinite_rn(float(x) / scale) as float8_e4m3fn.  The divisor is a tensor: torch may turn a division by a
    scalar into a multiplication by its reciprocal, which rounds differently."""
    xf = x.float()
    return torch.div(xf, torch.full_like(xf, scale)).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)


def dequantize_e4m3(q: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """float(e4m3) * scale in fp32; ``q`` is float8_e4m3fn or its uint8 bytes."""
    if q.dtype == torch.uint8:
        q = q.view(torch.float8_e4m3fn)
    return q.float() * scale


def alloc_logical_kv_fp8(dims, num_blocks: int, block_size: int):
    shape = (num_blocks, block_size, dims.num_key_value_heads, dims.head_dim)
    return [(torch.zeros(shape, dtype=torch.uint8), torch.zeros(shape, dtype=torch.uint8))
            for _ in range(dims.num_hidden_layers)]


def attention_forward_fp8_ref(q, k, v, k_cache, v_cache, ctx, scale, k_scale=1.0, v_scale=1.0, p_dtype=None):
    """oracle.paged_attention_ref.attention_forward_ref over e4m3 caches (uint8 bytes)."""
    if k_cache is not None and k_cache.numel():
        store_kvcache_ref(quantize_e4m3(k, k_scale).view(torch.uint8), quantize_e4m3(v, v_scale).view(torch.uint8),
                          k_cache, v_cache, ctx.slot_mapping)
    if ctx.is_prefill:
        if ctx.block_tables is None:
            return varlen_prefill_ref(q, k, v, ctx.cu_seqlens_q, ctx.cu_seqlens_k, scale, None, None, None, p_dtype)
        kc = dequantize_e4m3(k_cache, k_scale).to(torch.bfloat16)
        vc = dequantize_e4m3(v_cache, v_scale).to(torch.bfloat16)
        return varlen_prefill_ref(q, k, v, ctx.cu_seqlens_q, ctx.cu_seqlens_k, scale, ctx.block_tables, kc, vc, p_dtype)
    return paged_decode_ref(q, dequantize_e4m3(k_cache, k_scale), dequantize_e4m3(v_cache, v_scale), ctx.context_lens,
                            ctx.block_tables, scale, p_dtype)


class Qwen3RefFp8(Qwen3Ref):
    """Qwen3Ref whose attention operator keeps an e4m3 cache (unit scales, as the engine binds it)."""
    k_scale = 1.0
    v_scale = 1.0

    def forward(self, input_ids, positions, ctx, kv_caches):
        def attention(q, k, v, kc, vc, c, scale, p_dtype=None):
            return attention_forward_fp8_ref(q, k, v, kc, vc, c, scale, self.k_scale, self.v_scale, p_dtype)
        with mock.patch.object(qwen3_ref, "attention_forward_ref", attention):
            return super().forward(input_ids, positions, ctx, kv_caches)


def oracle_fp8_step_fn(model: Qwen3RefFp8, kv):
    """model_script step function of the fp8 oracle (the counterpart of test_oracle_golden.oracle_step_fn)."""
    def step(ids, pos, c):
        ctx = SimpleNamespace(is_prefill=c["is_prefill"], cu_seqlens_q=c.get("cu_seqlens_q"), cu_seqlens_k=c.get("cu_seqlens_k"),
                              max_seqlen_q=c.get("max_seqlen_q", 0), max_seqlen_k=c.get("max_seqlen_k", 0),
                              slot_mapping=c.get("slot_mapping"), context_lens=c.get("context_lens"),
                              block_tables=c.get("block_tables"))
        return model.logits(model.forward(ids, pos, ctx, kv), ctx)
    return step
