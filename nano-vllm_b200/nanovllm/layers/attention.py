"""The attention operator seam (reference nanovllm/layers/attention.py:33-75), backed by libb200attn.

Same module contract as the reference: ``Attention(num_heads, head_dim, scale, num_kv_heads)``,
attributes ``k_cache`` / ``v_cache`` (discovered with ``hasattr`` by the runner,
engine/model_runner.py:117-121), ``forward(q, k, v) -> o`` reading the process-global Context.

What differs is what the cache tensors look like: a layer's ``k_cache`` is the physical
page array ``[num_blocks, num_kv_heads, block_size, head_dim]`` (head-major pages, DESIGN.md), bound
to the library once by the runner; block ids and slot numbers mean exactly what they mean in the
reference.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch
from torch import nn

from .. import ops
from ..utils.context import get_context


def store_kvcache(key: torch.Tensor, value: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor,
                  slot_mapping: torch.Tensor, layer_id: int = 0):
    """Scatter new K/V rows into their slots (reference layers/attention.py:33-40).

    ``k_cache`` / ``v_cache`` must be the layer views of the cache bound with ``ops.bind_kv_cache``;
    they are accepted for signature compatibility and checked, the library addresses the bound cache.
    """
    n, num_heads, head_dim = key.shape
    assert key.stride(-1) == 1 and value.stride(-1) == 1
    assert key.stride(1) == head_dim and value.stride(1) == head_dim
    assert slot_mapping.numel() == n
    assert k_cache.dim() == 4 and k_cache.shape[1] == num_heads and k_cache.shape[3] == head_dim
    ops.store_kv(layer_id, key, value, slot_mapping)


class KVGroup(NamedTuple):
    """Sequences s0..s1-1 of a paged prefill over an fp8 cache whose keys are dequantized into the scratch together."""
    s0: int
    s1: int
    q0: int                  # their query rows q0..q1-1 of the step
    q1: int
    total_k: int             # their keys, packed from scratch row 0
    max_q: int
    cu_q: torch.Tensor       # int32 [s1 - s0 + 1], rebased to 0 (device)
    cu_k: torch.Tensor


def plan_kv_groups(cu_k: np.ndarray, max_rows: int) -> list[tuple[int, int]]:
    """Cut sequences 0..S-1 into consecutive groups [s0, s1) whose keys (cu_k[s1] - cu_k[s0]) fit max_rows scratch rows;
    a group always takes at least one sequence (one sequence fits: max_rows >= max_model_len)."""
    groups, s0, n = [], 0, len(cu_k) - 1
    for s in range(n):
        if s > s0 and cu_k[s + 1] - cu_k[s0] > max_rows:
            groups.append((s0, s))
            s0 = s
    if n:
        groups.append((s0, n))
    return groups


def kv_group_arrays(cu_q: np.ndarray, cu_k: np.ndarray, groups):
    """Host side of each group: (s0, s1, q0, q1, total_k, max_q, rebased cu_q, rebased cu_k)."""
    out = []
    for s0, s1 in groups:
        gq = (cu_q[s0:s1 + 1] - cu_q[s0]).astype(np.int32)
        gk = (cu_k[s0:s1 + 1] - cu_k[s0]).astype(np.int32)
        out.append((s0, s1, int(cu_q[s0]), int(cu_q[s1]), int(gk[-1]), int(np.diff(gq).max()), gq, gk))
    return out


class Attention(nn.Module):
    def __init__(self, num_heads: int, head_dim: int, scale: float, num_kv_heads: int):
        super().__init__()
        self.num_heads = num_heads
        self.head_dim = head_dim
        self.scale = scale
        self.num_kv_heads = num_kv_heads
        self.k_cache = self.v_cache = torch.tensor([])
        self.layer_id = 0                       # set by the runner when it binds the cache
        self.kv_scratch = None                  # fp8 cache: bf16 [2, rows, Hkv, D] the paged prefill dequantizes into

    def forward(self, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, kv_stored: bool = False) -> torch.Tensor:
        """q [T, Hq, D], k/v [T, Hkv, D] (views of the qkv GEMM output are fine).

        ``kv_stored=True`` tells the operator that the fused q/k-norm+RoPE kernel already scattered
        this step's K/V (the model's fast path); the default does the scatter itself, like the reference.
        """
        ctx = get_context()
        have_cache = self.k_cache.numel() > 0 and self.v_cache.numel() > 0
        if have_cache and not kv_stored:
            store_kvcache(k, v, self.k_cache, self.v_cache, ctx.slot_mapping, self.layer_id)
        if ctx.is_prefill and ctx.block_tables is not None and self.k_cache.dtype == torch.float8_e4m3fn:
            return self._prefill_fp8_cache(q, ctx)
        if ctx.is_prefill:
            return ops.paged_prefill(self.layer_id, q, k, v, ctx.cu_seqlens_q, ctx.cu_seqlens_k,
                                     ctx.max_seqlen_q, ctx.max_seqlen_k, self.scale,
                                     block_tables=ctx.block_tables, num_kv_heads=self.num_kv_heads)
        o = ops.paged_decode(self.layer_id, q, ctx.block_tables, ctx.context_lens, self.scale)
        return o.unsqueeze(1)                   # [B, 1, Hq, D] like flash_attn_with_kvcache

    def _prefill_fp8_cache(self, q: torch.Tensor, ctx) -> torch.Tensor:
        """Prefix hit / chunked prefill over an fp8 cache: per group of sequences, dequantize every key and value the
        step reads (this step's own included, as flash-attn reads k_cache / v_cache) into the bf16 scratch, then run
        the packed prefill kernel on it."""
        if ctx.kv_groups is None or self.kv_scratch is None:
            raise RuntimeError("a paged prefill over an fp8 cache needs Context.kv_groups and the layer's kv_scratch")
        out = torch.empty(q.shape, dtype=q.dtype, device=q.device)
        ks, vs = self.kv_scratch[0], self.kv_scratch[1]
        for g in ctx.kv_groups:
            ops.kv_gather(self.layer_id, ctx.block_tables[g.s0:g.s1], g.cu_k, ks, vs, g.total_k)
            ops.prefill_packed_kv(q[g.q0:g.q1], ks[:g.total_k], vs[:g.total_k], g.cu_q, g.cu_k, g.max_q, self.scale,
                                  out=out[g.q0:g.q1])
        return out
