"""Tensor-facing wrappers over the C ABI: pass data_ptr()s, strides and the current stream.

PyTorch is plumbing here (device memory + streams); every function below is one
launch of a hand-written sm_90a kernel in libb200attn.so.
"""
from __future__ import annotations

import torch

from . import _native as nat


LAUNCHES = [0]          # kernels of libb200attn launched through this module (graph replays add their node count)


def reset_launch_count() -> None:
    LAUNCHES[0] = 0


def _stream() -> int:
    LAUNCHES[0] += 1        # every wrapper below asks for the stream exactly once per kernel launch
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: torch.Tensor | None) -> int | None:
    return None if t is None else t.data_ptr()


def _need(t: torch.Tensor, dtype, name: str):
    if not t.is_cuda:
        raise nat.B200Error(f"{name} must be a CUDA tensor (there is no CPU path)")
    if t.dtype != dtype:
        raise nat.B200Error(f"{name} must be {dtype}, got {t.dtype}")


# ---- KV cache ---------------------------------------------------------------
def kv_cache_shape(layers, num_blocks, num_kv_heads, block_size, head_dim):
    """Physical layout (DESIGN.md): [2, layers, blocks, kv_heads, block_size, head_dim]."""
    return (2, layers, num_blocks, num_kv_heads, block_size, head_dim)


def bind_kv_cache(kv_cache: torch.Tensor, k_scale: float = 1.0, v_scale: float = 1.0):
    """kv_cache: [2, L, nblk, Hkv, bs, D] bf16 or float8_e4m3fn contiguous (engine/model_runner.py:103-121 equivalent).
    An fp8 cache stores e4m3(x / scale) and reads e4m3 * scale, k_scale for keys and v_scale for values."""
    if kv_cache.dtype != torch.float8_e4m3fn:
        _need(kv_cache, torch.bfloat16, "kv_cache")
        if k_scale != 1.0 or v_scale != 1.0:
            raise nat.B200Error("k_scale / v_scale apply to an fp8 (float8_e4m3fn) cache only")
    elif not kv_cache.is_cuda:
        raise nat.B200Error("kv_cache must be a CUDA tensor (there is no CPU path)")
    assert kv_cache.is_contiguous() and kv_cache.dim() == 6 and kv_cache.shape[0] == 2
    h = nat.handle()
    _, layers, nblk, hkv, bs, d = kv_cache.shape
    if kv_cache.dtype == torch.float8_e4m3fn:
        nat.check(h.lib.b200_kv_bind_fp8(h.ptr, kv_cache[0].data_ptr(), kv_cache[1].data_ptr(), layers, nblk, bs, hkv, d,
                                         k_scale, v_scale), h.ptr)
    else:
        nat.check(h.lib.b200_kv_bind(h.ptr, kv_cache[0].data_ptr(), kv_cache[1].data_ptr(), layers, nblk, bs, hkv, d), h.ptr)
    h.kv = kv_cache
    h.workspace = None          # its layout depends on the head count: start again from zeros
    return h


def ensure_workspace(max_batch: int, num_q_heads: int) -> torch.Tensor:
    h = nat.handle()
    need = h.lib.b200_decode_workspace_bytes(h.ptr, max_batch, num_q_heads)
    if need == 0:
        raise nat.B200Error("decode workspace size query failed (cache not bound or bad head counts)")
    if h.workspace is None or h.workspace.numel() < need:
        h.workspace = torch.zeros(need, dtype=torch.uint8, device="cuda")
    return h.workspace


# ---- attention operator -------------------------------------------------------
def store_kv(layer: int, k: torch.Tensor, v: torch.Tensor, slot_mapping: torch.Tensor):
    _need(k, torch.bfloat16, "k"); _need(v, torch.bfloat16, "v"); _need(slot_mapping, torch.int32, "slot_mapping")
    n, hkv, d = k.shape
    assert k.stride(2) == 1 and k.stride(1) == d and v.stride(2) == 1 and v.stride(1) == d
    assert slot_mapping.numel() == n
    h = nat.handle()
    nat.check(h.lib.b200_store_kv(h.ptr, layer, k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
                                  slot_mapping.data_ptr(), n, _stream()), h.ptr)


def kv_gather(layer: int, block_tables: torch.Tensor, cu_seqlens_k: torch.Tensor, k_out: torch.Tensor, v_out: torch.Tensor,
              total_k: int) -> None:
    """Dequantize keys / values 0..len_k(s)-1 of every sequence of the bound fp8 cache into packed bf16 rows
    k_out / v_out [>= total_k, Hkv, D] (row cu_seqlens_k[s] + r for row r of sequence s)."""
    _need(block_tables, torch.int32, "block_tables"); _need(cu_seqlens_k, torch.int32, "cu_seqlens_k")
    _need(k_out, torch.bfloat16, "k_out"); _need(v_out, torch.bfloat16, "v_out")
    d = k_out.shape[-1]
    assert block_tables.stride(1) == 1 and k_out.stride(2) == 1 and k_out.stride(1) == d and v_out.stride(2) == 1 and v_out.stride(1) == d
    assert k_out.shape[0] >= total_k and v_out.shape[0] >= total_k
    h = nat.handle()
    nat.check(h.lib.b200_kv_gather(h.ptr, layer, block_tables.data_ptr(), block_tables.stride(0), cu_seqlens_k.data_ptr(),
                                   cu_seqlens_k.numel() - 1, k_out.data_ptr(), k_out.stride(0), v_out.data_ptr(), v_out.stride(0),
                                   int(total_k), _stream()), h.ptr)


def paged_decode(layer: int, q: torch.Tensor, block_tables: torch.Tensor, context_lens: torch.Tensor,
                 scale: float, out: torch.Tensor | None = None) -> torch.Tensor:
    """q [B, Hq, D] -> out [B, Hq, D]."""
    _need(q, torch.bfloat16, "q"); _need(block_tables, torch.int32, "block_tables"); _need(context_lens, torch.int32, "context_lens")
    b, hq, d = q.shape
    assert q.stride(2) == 1 and q.stride(1) == d and block_tables.stride(1) == 1
    if out is None:
        out = torch.empty((b, hq, d), dtype=q.dtype, device=q.device)
    ws = ensure_workspace(b, hq)
    h = nat.handle()
    nat.check(h.lib.b200_paged_decode(h.ptr, layer, q.data_ptr(), q.stride(0), block_tables.data_ptr(),
                                      block_tables.stride(0), context_lens.data_ptr(), out.data_ptr(), out.stride(0),
                                      b, hq, scale, ws.data_ptr(), ws.numel(), _stream()), h.ptr)
    return out


def paged_decode_fused(layer: int, qkv: torch.Tensor, num_q_heads: int, q_norm_weight, k_norm_weight, cos_sin: torch.Tensor,
                       eps: float, block_tables: torch.Tensor, context_lens: torch.Tensor, scale: float,
                       out: torch.Tensor | None = None) -> torch.Tensor:
    """Raw qkv GEMM output [B, (Hq+2Hkv)*D] -> attention output [B, Hq, D]; q/k-norm, RoPE and the KV append happen
    inside the decode kernel (qkv itself is left untouched)."""
    _need(qkv, torch.bfloat16, "qkv"); _need(block_tables, torch.int32, "block_tables"); _need(context_lens, torch.int32, "context_lens")
    _need(cos_sin, torch.float32, "cos_sin")
    assert qkv.dim() == 2 and qkv.stride(1) == 1 and block_tables.stride(1) == 1
    b = qkv.shape[0]
    if out is None:
        out = torch.empty((b, num_q_heads, 128), dtype=qkv.dtype, device=qkv.device)
    ws = ensure_workspace(b, num_q_heads)
    h = nat.handle()
    nat.check(h.lib.b200_paged_decode_fused(h.ptr, layer, qkv.data_ptr(), qkv.stride(0), q_norm_weight.data_ptr(),
                                            k_norm_weight.data_ptr(), cos_sin.data_ptr(), eps, block_tables.data_ptr(),
                                            block_tables.stride(0), context_lens.data_ptr(), out.data_ptr(), out.stride(0),
                                            b, num_q_heads, scale, ws.data_ptr(), ws.numel(), _stream()), h.ptr)
    return out


def paged_prefill(layer: int, q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q: int, max_seqlen_k: int,
                  scale: float, block_tables=None, num_kv_heads: int | None = None, out=None) -> torch.Tensor:
    """q [T, Hq, D]; k, v [Tk, Hkv, D] (ignored when block_tables is given)."""
    _need(q, torch.bfloat16, "q"); _need(cu_seqlens_q, torch.int32, "cu_seqlens_q"); _need(cu_seqlens_k, torch.int32, "cu_seqlens_k")
    t, hq, d = q.shape
    assert q.stride(2) == 1 and q.stride(1) == d
    if block_tables is None:
        _need(k, torch.bfloat16, "k"); _need(v, torch.bfloat16, "v")
        hkv = k.shape[1]
        assert k.stride(2) == 1 and k.stride(1) == d and v.stride(2) == 1 and v.stride(1) == d
        kp, ks, vp, vs, btp, bts = k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), None, 0
    else:
        _need(block_tables, torch.int32, "block_tables")
        hkv = num_kv_heads if num_kv_heads is not None else k.shape[1]
        kp, ks, vp, vs = None, 0, None, 0
        btp, bts = block_tables.data_ptr(), block_tables.stride(0)
    if out is None:
        out = torch.empty((t, hq, d), dtype=q.dtype, device=q.device)
    h = nat.handle()
    nat.check(h.lib.b200_paged_prefill(h.ptr, layer, q.data_ptr(), q.stride(0), kp, ks, vp, vs,
                                       cu_seqlens_q.data_ptr(), cu_seqlens_k.data_ptr(), btp, bts,
                                       out.data_ptr(), out.stride(0), t, cu_seqlens_q.numel() - 1,
                                       int(max_seqlen_q), int(max_seqlen_k), hq, hkv, scale, _stream()), h.ptr)
    return out


def prefill_packed_kv(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q: int, scale: float, out=None) -> torch.Tensor:
    """Packed causal varlen prefill where sequence s has len_k(s) >= len_q(s) keys: q [T, Hq, D], k / v [Tk, Hkv, D]
    (all Tk rows are keys: Tk = cu_seqlens_k[-1])."""
    for t, name in ((q, "q"), (k, "k"), (v, "v")):
        _need(t, torch.bfloat16, name)
    _need(cu_seqlens_q, torch.int32, "cu_seqlens_q"); _need(cu_seqlens_k, torch.int32, "cu_seqlens_k")
    t, hq, d = q.shape
    hkv = k.shape[1]
    assert q.stride(2) == 1 and q.stride(1) == d
    assert k.stride(2) == 1 and k.stride(1) == d and v.stride(2) == 1 and v.stride(1) == d and v.shape[0] == k.shape[0]
    if out is None:
        out = torch.empty((t, hq, d), dtype=q.dtype, device=q.device)
    h = nat.handle()
    nat.check(h.lib.b200_prefill_packed_kv(h.ptr, q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
                                           cu_seqlens_q.data_ptr(), cu_seqlens_k.data_ptr(), out.data_ptr(), out.stride(0), t,
                                           k.shape[0], cu_seqlens_q.numel() - 1, int(max_seqlen_q), hq, hkv, scale, _stream()), h.ptr)
    return out


# ---- fused ops around it ---------------------------------------------------------
def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float, out: torch.Tensor | None = None) -> torch.Tensor:
    """x: contiguous [..., cols], or 2-D with unit inner stride (a column slice of a wider row)."""
    _need(x, torch.bfloat16, "x")
    cols = x.shape[-1]
    if x.dim() == 2 and x.stride(1) == 1:
        rows, xs = x.shape[0], x.stride(0)
    else:
        assert x.is_contiguous(), "rmsnorm needs a contiguous tensor or a 2-D row-strided view"
        rows, xs = x.numel() // cols, cols
    if out is None:
        out = torch.empty(x.shape, dtype=x.dtype, device=x.device)
    assert out.is_contiguous()
    lib = nat.load()
    nat.check(lib.b200_rmsnorm(x.data_ptr(), xs, weight.data_ptr(), out.data_ptr(), cols, rows, cols, eps, _stream()))
    return out


def add_rmsnorm(x: torch.Tensor, residual: torch.Tensor, weight: torch.Tensor, eps: float,
                out: torch.Tensor | None = None):
    """In place on `residual` (<- bf16(x + residual)); returns (normed, residual) like layernorm.py:28-40."""
    _need(x, torch.bfloat16, "x"); _need(residual, torch.bfloat16, "residual")
    assert x.is_contiguous() and residual.is_contiguous() and x.shape == residual.shape
    cols = x.shape[-1]
    if out is None:
        out = torch.empty_like(x)
    lib = nat.load()
    nat.check(lib.b200_add_rmsnorm(x.data_ptr(), residual.data_ptr(), weight.data_ptr(), out.data_ptr(),
                                   x.numel() // cols, cols, eps, _stream()))
    return out, residual


def qknorm_rope_store(layer: int, qkv: torch.Tensor, num_q_heads: int, num_kv_heads: int, positions: torch.Tensor,
                      q_norm_weight, k_norm_weight, cos_sin: torch.Tensor, eps: float, slot_mapping=None):
    """In place on the fused qkv GEMM output [n, (Hq+2Hkv)*D]; scatters k, v into the bound cache."""
    _need(qkv, torch.bfloat16, "qkv"); _need(positions, torch.int64, "positions"); _need(cos_sin, torch.float32, "cos_sin")
    assert qkv.dim() == 2 and qkv.stride(1) == 1
    if slot_mapping is not None:
        _need(slot_mapping, torch.int32, "slot_mapping")
    h = nat.handle()
    nat.check(h.lib.b200_qknorm_rope_store(h.ptr, layer, qkv.data_ptr(), qkv.stride(0), num_q_heads, num_kv_heads,
                                           positions.data_ptr(), q_norm_weight.data_ptr(), k_norm_weight.data_ptr(),
                                           cos_sin.data_ptr(), eps, _ptr(slot_mapping), qkv.shape[0], _stream()), h.ptr)
    return qkv


def silu_mul(x: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    _need(x, torch.bfloat16, "x")
    assert x.is_contiguous()
    inter = x.shape[-1] // 2
    rows = x.numel() // (2 * inter)
    if out is None:
        out = torch.empty(x.shape[:-1] + (inter,), dtype=x.dtype, device=x.device)
    lib = nat.load()
    nat.check(lib.b200_silu_mul(x.data_ptr(), out.data_ptr(), rows, inter, _stream()))
    return out


def embedding(ids: torch.Tensor, table: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    _need(ids, torch.int64, "ids"); _need(table, torch.bfloat16, "table")
    assert table.is_contiguous() and ids.is_contiguous()
    n, hidden = ids.numel(), table.shape[1]
    if out is None:
        out = torch.empty((n, hidden), dtype=table.dtype, device=table.device)
    lib = nat.load()
    nat.check(lib.b200_embedding(ids.data_ptr(), table.data_ptr(), out.data_ptr(), n, hidden, table.shape[0], _stream()))
    return out


def gather_tokens(ids: torch.Tensor, src: torch.Tensor, prev_tokens: torch.Tensor) -> torch.Tensor:
    """ids[i] = prev_tokens[src[i]] where src[i] >= 0 (in place)."""
    _need(ids, torch.int64, "ids"); _need(src, torch.int32, "src"); _need(prev_tokens, torch.int64, "prev_tokens")
    lib = nat.load()
    nat.check(lib.b200_gather_tokens(ids.data_ptr(), src.data_ptr(), prev_tokens.data_ptr(), ids.numel(), _stream()))
    return ids


def sample(logits: torch.Tensor, temperatures: torch.Tensor | None, seed: int, step: int,
           out: torch.Tensor | None = None, index_offset: int = 0, out_keys: torch.Tensor | None = None,
           step_dev: torch.Tensor | None = None) -> torch.Tensor:
    """logits [rows, vocab] bf16 or fp32 -> int64 token ids (greedy where temperature == 0).

    With ``out_keys`` (int64 [rows]) also writes order-preserving (score, token) keys for the
    vocab-parallel all-reduce(MAX) combine; ``index_offset`` is the shard's first vocab id."""
    assert logits.dim() == 2 and logits.stride(1) == 1 and logits.is_cuda
    is32 = logits.dtype == torch.float32
    if not is32:
        _need(logits, torch.bfloat16, "logits")
    rows, vocab = logits.shape
    if out is None:
        out = torch.empty(rows, dtype=torch.int64, device=logits.device)
    lib = nat.load()
    nat.check(lib.b200_sample(logits.data_ptr(), int(is32), logits.stride(0), _ptr(temperatures), rows, vocab,
                              index_offset, seed & (2**64 - 1), step & (2**64 - 1), _ptr(step_dev), out.data_ptr(), _ptr(out_keys),
                              _stream()))
    return out


FILTER_ROW_WORDS = 1538                    # int64 words per row of the filter workspace (include/b200_paged_attn.h)
_FILTER_STAGE_WORDS = ((0, 1), (2, 514), (514, 1026), (1026, 1538))    # [lo, hi) of each stage's words within a row
FILTER_TAU_WORD = 1


def filter_workspace(rows: int, device="cuda") -> torch.Tensor:
    """Zeroed workspace of ``sample_filtered`` for up to ``rows`` rows (every call leaves it zero again)."""
    n = nat.load().b200_sample_filter_workspace_words(rows)
    if n <= 0:
        raise nat.B200Error("bad filter workspace row count")
    return torch.zeros(n, dtype=torch.int64, device=device)


def filter_stage_words(workspace: torch.Tensor, rows: int, stage: int) -> torch.Tensor:
    """The words stage ``stage`` writes for ``rows`` rows, a [rows, n] strided view (all-reduce MAX for stage 0, SUM
    for stages 1-3 under vocab parallelism)."""
    lo, hi = _FILTER_STAGE_WORDS[stage]
    return workspace[:rows * FILTER_ROW_WORDS].view(rows, FILTER_ROW_WORDS)[:, lo:hi]


def filter_tau_keys(workspace: torch.Tensor, rows: int) -> torch.Tensor:
    """Per row, the order-preserving 16-bit key of the threshold tau of the last ``sample_filtered`` call (0 = no filter)."""
    return workspace[:rows * FILTER_ROW_WORDS].view(rows, FILTER_ROW_WORDS)[:, FILTER_TAU_WORD]


def sample_filtered(logits: torch.Tensor, temps: torch.Tensor, top_k: torch.Tensor | None, top_p: torch.Tensor | None,
                    min_p: torch.Tensor | None, seed: int, step: int, workspace: torch.Tensor, out: torch.Tensor | None = None,
                    index_offset: int = 0, out_keys: torch.Tensor | None = None, step_dev: torch.Tensor | None = None,
                    reduce=None) -> torch.Tensor:
    """Top-k / top-p / min-p sampling: bf16 logits [rows, vocab] -> int64 token ids, as ``sample`` restricted per row to
    {x >= tau} (include/b200_paged_attn.h).  ``top_k`` int32 [rows] (<= 0 off), ``top_p`` / ``min_p`` fp32 [rows]
    (>= 1 / <= 0 off), each may be None; ``workspace`` from ``filter_workspace``.  Runs stages 0-3 and the race; after
    stage s it calls ``reduce(filter_stage_words(workspace, rows, s), "max" if s == 0 else "sum")`` when ``reduce`` is
    given (the vocab-parallel all-reduce of the stage's words)."""
    assert logits.dim() == 2 and logits.stride(1) == 1 and logits.is_cuda
    if logits.dtype == torch.float32:
        nat.check(-2)                               # B200_EUNSUPPORTED: the filtered sampler reads bf16 logits only
    _need(logits, torch.bfloat16, "logits"); _need(temps, torch.float32, "temps"); _need(workspace, torch.int64, "workspace")
    if top_k is not None:
        _need(top_k, torch.int32, "top_k")
    for t, name in ((top_p, "top_p"), (min_p, "min_p")):
        if t is not None:
            _need(t, torch.float32, name)
    rows, vocab = logits.shape
    assert workspace.numel() >= rows * FILTER_ROW_WORDS, "filter workspace too small"
    if out is None and out_keys is None:
        out = torch.empty(rows, dtype=torch.int64, device=logits.device)
    for stage in range(4):
        sample_filter_stage(stage, logits, temps, top_k, top_p, min_p, workspace)
        if reduce is not None:
            reduce(filter_stage_words(workspace, rows, stage), "max" if stage == 0 else "sum")
    sample_filter_race(logits, temps, top_k, top_p, min_p, seed, step, workspace, out, index_offset, out_keys, step_dev)
    return out if out is not None else out_keys


def sample_filter_race(logits, temps, top_k, top_p, min_p, seed: int, step: int, workspace: torch.Tensor, out=None,
                       index_offset: int = 0, out_keys=None, step_dev=None) -> None:
    """The last launch of ``sample_filtered``: the exponential race over {x >= tau} (workspace reduced by then)."""
    rows, vocab = logits.shape
    nat.check(nat.load().b200_sample_filtered(logits.data_ptr(), logits.stride(0), temps.data_ptr(), _ptr(top_k), _ptr(top_p),
                                              _ptr(min_p), rows, vocab, index_offset, seed & (2**64 - 1), step & (2**64 - 1),
                                              _ptr(step_dev), workspace.data_ptr(), _ptr(out), _ptr(out_keys), _stream()))


def sample_filter_stage(stage: int, logits: torch.Tensor, temps: torch.Tensor, top_k, top_p, min_p,
                        workspace: torch.Tensor) -> None:
    """One threshold stage (0-3) of ``sample_filtered`` (for callers that reduce the stages' words themselves)."""
    rows, vocab = logits.shape
    nat.check(nat.load().b200_sample_filter_stage(logits.data_ptr(), logits.stride(0), temps.data_ptr(), _ptr(top_k),
                                                  _ptr(top_p), _ptr(min_p), rows, vocab, stage, workspace.data_ptr(),
                                                  _stream()))


def tokens_from_keys(keys: torch.Tensor) -> torch.Tensor:
    """Decode the token ids out of (all-reduced) sample keys."""
    return 0xffffffff - (keys & 0xffffffff)


# ---- presence / frequency / repetition penalties (csrc/penalty.cu) ------------------------------------------------------
PENALTY_IN_PROMPT = 1 << 31                # entry = token << 32 | in_prompt << 31 | generated count


def penalty_history(slots: int, capacity: int, device="cuda") -> tuple[torch.Tensor, torch.Tensor]:
    """Zeroed history pool: int64 [slots, capacity] entries and int32 [slots] lengths."""
    return (torch.zeros(slots, capacity, dtype=torch.int64, device=device),
            torch.zeros(slots, dtype=torch.int32, device=device))


def penalty_load(history: torch.Tensor, lengths: torch.Tensor, entries: torch.Tensor, offsets: torch.Tensor,
                 slots: torch.Tensor) -> None:
    """Slot slots[r] <- entries[offsets[r]:offsets[r + 1]] for every row with slots[r] >= 0 (rows = slots.numel())."""
    _need(history, torch.int64, "history"); _need(lengths, torch.int32, "lengths"); _need(entries, torch.int64, "entries")
    _need(offsets, torch.int32, "offsets"); _need(slots, torch.int32, "slots")
    assert history.dim() == 2 and history.is_contiguous() and offsets.numel() == slots.numel() + 1
    num_slots, capacity = history.shape
    nat.check(nat.load().b200_penalty_load(history.data_ptr(), lengths.data_ptr(), num_slots, capacity, entries.data_ptr(),
                                           offsets.data_ptr(), slots.data_ptr(), slots.numel(), _stream()))


def penalty_apply(logits: torch.Tensor, history: torch.Tensor, lengths: torch.Tensor, slots: torch.Tensor,
                  repetition: torch.Tensor, frequency: torch.Tensor, presence: torch.Tensor,
                  pending: torch.Tensor | None = None, index_offset: int = 0) -> torch.Tensor:
    """Absorb pending[r] (int64, may be None) into slot slots[r] and penalise row r of the bf16 logits [rows, vocab] in
    place (include/b200_paged_attn.h); rows with slot -1 are left alone."""
    assert logits.dim() == 2 and logits.stride(1) == 1 and logits.is_cuda
    if logits.dtype == torch.float32:
        nat.check(-2)                               # B200_EUNSUPPORTED: both samplers read bf16 logits
    _need(logits, torch.bfloat16, "logits"); _need(history, torch.int64, "history"); _need(lengths, torch.int32, "lengths")
    _need(slots, torch.int32, "slots")
    for t, name in ((repetition, "repetition"), (frequency, "frequency"), (presence, "presence")):
        _need(t, torch.float32, name)
    if pending is not None:
        _need(pending, torch.int64, "pending")
    assert history.dim() == 2 and history.is_contiguous()
    rows, vocab = logits.shape
    num_slots, capacity = history.shape
    nat.check(nat.load().b200_penalty_apply(logits.data_ptr(), logits.stride(0), rows, vocab, index_offset, history.data_ptr(),
                                            lengths.data_ptr(), num_slots, capacity, slots.data_ptr(), _ptr(pending),
                                            repetition.data_ptr(), frequency.data_ptr(), presence.data_ptr(), _stream()))
    return logits


# ---- per-token logprobs of the raw logits (csrc/logprobs.cu) ------------------------------------------------------------
LOGPROB_MAX_K = 20
LOGPROB_ROW_WORDS = 8                      # int64 workspace words per row (include/b200_paged_attn.h)
# one packed output row (int32 words): ids[0..20] (sampled token, then the top k), logprobs[21..41] (fp32 bits), rank[42]
LOGPROB_OUT_WORDS = 2 * (LOGPROB_MAX_K + 1) + 1
LOGPROB_LP_COL = LOGPROB_MAX_K + 1
LOGPROB_RANK_COL = 2 * (LOGPROB_MAX_K + 1)


def logprob_workspace(rows: int, device="cuda") -> torch.Tensor:
    """Zeroed logprob workspace for up to ``rows`` rows (every ``logprobs_finish`` leaves it zero again)."""
    n = nat.load().b200_logprob_workspace_words(rows)
    if n <= 0:
        raise nat.B200Error("bad logprob workspace row count")
    return torch.zeros(n, dtype=torch.int64, device=device)


def logprob_words(workspace: torch.Tensor, rows: int, lo: int, hi: int) -> torch.Tensor:
    """Words [lo, hi) of every row of the workspace, a [rows, hi - lo] strided view."""
    return workspace[:rows * LOGPROB_ROW_WORDS].view(rows, LOGPROB_ROW_WORDS)[:, lo:hi]


def _logprob_args(logits: torch.Tensor, k: torch.Tensor, workspace: torch.Tensor):
    assert logits.dim() == 2 and logits.stride(1) == 1 and logits.is_cuda
    if logits.dtype == torch.float32:
        nat.check(-2)                               # B200_EUNSUPPORTED: the logprob kernels read bf16 logits only
    _need(logits, torch.bfloat16, "logits"); _need(k, torch.int32, "k"); _need(workspace, torch.int64, "workspace")
    rows = logits.shape[0]
    assert k.numel() >= rows and workspace.numel() >= rows * LOGPROB_ROW_WORDS, "logprob workspace too small"
    return rows, logits.shape[1]


def logprobs_topk(logits: torch.Tensor, k: torch.Tensor, workspace: torch.Tensor, topk_keys: torch.Tensor,
                  index_offset: int = 0, reduce=None) -> None:
    """Before the penalties: each row's top max(k, 1) keys into ``topk_keys`` (int64 [rows, 20]) and its maximum into the
    workspace, then ``reduce(words, "max")`` of that word when ``reduce`` is given (vocab parallelism)."""
    rows, vocab = _logprob_args(logits, k, workspace)
    _need(topk_keys, torch.int64, "topk_keys")
    assert topk_keys.is_contiguous() and topk_keys.numel() >= rows * LOGPROB_MAX_K
    nat.check(nat.load().b200_logprob_topk(logits.data_ptr(), logits.stride(0), k.data_ptr(), rows, vocab, index_offset,
                                           workspace.data_ptr(), topk_keys.data_ptr(), _stream()))
    if reduce is not None:
        reduce(logprob_words(workspace, rows, 0, 1), "max")


def logprob_saved_buffer(rows: int, capacity: int, device="cuda") -> torch.Tensor:
    """Scratch of ``logprobs_save``: int64 [rows, capacity + 1] (capacity = the penalty history's)."""
    return torch.empty(rows, capacity + 1, dtype=torch.int64, device=device)


def logprobs_save(logits: torch.Tensor, k: torch.Tensor, workspace: torch.Tensor, saved: torch.Tensor, history: torch.Tensor,
                  lengths: torch.Tensor, slots: torch.Tensor, pending: torch.Tensor | None = None,
                  index_offset: int = 0) -> None:
    """Before ``penalty_apply`` on the same arguments: keep the raw value of every logit it will rewrite."""
    rows, vocab = _logprob_args(logits, k, workspace)
    _need(saved, torch.int64, "saved"); _need(history, torch.int64, "history"); _need(lengths, torch.int32, "lengths")
    _need(slots, torch.int32, "slots")
    if pending is not None:
        _need(pending, torch.int64, "pending")
    num_slots, capacity = history.shape
    assert saved.is_contiguous() and saved.numel() >= rows * (capacity + 1)
    nat.check(nat.load().b200_logprob_save(logits.data_ptr(), logits.stride(0), k.data_ptr(), rows, vocab, index_offset,
                                           history.data_ptr(), lengths.data_ptr(), num_slots, capacity, slots.data_ptr(),
                                           _ptr(pending), workspace.data_ptr(), saved.data_ptr(), _stream()))


def logprobs_finish(logits: torch.Tensor, k: torch.Tensor, tokens: torch.Tensor, workspace: torch.Tensor,
                    topk_keys: torch.Tensor, out: torch.Tensor, index_offset: int = 0, saved: torch.Tensor | None = None,
                    capacity: int = 0, reduce=None, gather=None) -> torch.Tensor:
    """After the token ids ``tokens`` (int64 [rows]) are known: restore the saved logits (``saved`` from
    ``logprobs_save``, None when no row was penalised), count the rank, sum the softmax mass and write one packed row per
    logprob row into ``out`` (int32 [rows, LOGPROB_OUT_WORDS]).  Under vocab parallelism ``reduce(words, op)`` all-reduces
    the words each launch wrote and ``gather(topk_keys)`` returns every rank's keys as one [world, rows, 20] tensor."""
    rows, vocab = _logprob_args(logits, k, workspace)
    _need(tokens, torch.int64, "tokens"); _need(out, torch.int32, "out")
    assert out.dim() == 2 and out.stride(1) == 1 and out.shape[0] >= rows and out.shape[1] >= LOGPROB_OUT_WORDS
    lib = nat.load()
    if saved is not None:
        _need(saved, torch.int64, "saved")
        assert saved.numel() >= rows * (capacity + 1)
    nat.check(lib.b200_logprob_restore(logits.data_ptr(), logits.stride(0), k.data_ptr(), rows, vocab, index_offset,
                                       tokens.data_ptr(), workspace.data_ptr(), _ptr(saved), capacity, _stream()))
    if reduce is not None:
        reduce(logprob_words(workspace, rows, 1, 2), "max")
    nat.check(lib.b200_logprob_rank(logits.data_ptr(), logits.stride(0), k.data_ptr(), rows, vocab, workspace.data_ptr(),
                                    _stream()))
    if reduce is not None:
        reduce(logprob_words(workspace, rows, 2, 4), "sum")
    mine = topk_keys.view(-1)[:rows * LOGPROB_MAX_K]
    keys = mine if gather is None else gather(mine)
    sources = keys.numel() // (rows * LOGPROB_MAX_K)
    lps = out[:, LOGPROB_LP_COL:].view(torch.float32)
    nat.check(lib.b200_logprob_finish(k.data_ptr(), rows, tokens.data_ptr(), keys.data_ptr(), sources, workspace.data_ptr(),
                                      out.data_ptr(), lps.data_ptr(), out[:, LOGPROB_RANK_COL:].data_ptr(), out.stride(0),
                                      _stream()))
    return out


def logprobs(logits: torch.Tensor, k: torch.Tensor, tokens: torch.Tensor, workspace: torch.Tensor | None = None,
             out: torch.Tensor | None = None, index_offset: int = 0) -> torch.Tensor:
    """Logprobs of unpenalised bf16 logits [rows, vocab] for the sampled ``tokens``, unsharded: ``logprobs_topk`` then
    ``logprobs_finish``.  Returns the packed int32 [rows, LOGPROB_OUT_WORDS] rows (``unpack_logprobs`` reads them)."""
    rows = logits.shape[0]
    if workspace is None:
        workspace = logprob_workspace(rows, device=logits.device)
    if out is None:
        out = torch.zeros(rows, LOGPROB_OUT_WORDS, dtype=torch.int32, device=logits.device)
    keys = torch.empty(rows, LOGPROB_MAX_K, dtype=torch.int64, device=logits.device)
    logprobs_topk(logits, k, workspace, keys, index_offset)
    return logprobs_finish(logits, k, tokens, workspace, keys, out, index_offset)


def unpack_logprobs(rows, k: int):
    """One packed row (numpy int32 [LOGPROB_OUT_WORDS] or [n, LOGPROB_OUT_WORDS]) -> (ids [.., 1 + k], fp32 logprobs
    [.., 1 + k], rank [..]); column 0 is the sampled token, 1.. the top k."""
    return (rows[..., :1 + k], rows[..., LOGPROB_LP_COL:LOGPROB_LP_COL + 1 + k].view("float32"), rows[..., LOGPROB_RANK_COL])


# ---- decode-size projections on wgmma (csrc/linear_tc.cu) -------------------------------------------------------------
EPI_BF16, EPI_SILU, EPI_PARTIAL = 0, 1, 2


class pdl_off:
    """Context manager: launches inside carry no programmatic-dependent-launch attribute (b200_set_pdl)."""

    def __enter__(self):
        self._was = nat.load().b200_set_pdl(0)
        return self

    def __exit__(self, *exc):
        nat.load().b200_set_pdl(self._was)
        return False


def linear(x: torch.Tensor, w: torch.Tensor, epilogue: int = EPI_BF16, block_n: int = 32, k_splits: int = 1,
           pdl: bool = False, out: torch.Tensor | None = None, shallow: bool = False, cluster: int = 1,
           stages: int = 0) -> torch.Tensor:
    """x [rows, k] @ w[n, k]^T on wgmma.  EPI_SILU: w = [gate; up] rows, returns silu(gate) * up [rows, n/2];
    EPI_PARTIAL: returns fp32 [k_splits, rows, n] partial sums for ``add_rmsnorm_partials``.
    ``stages`` (0 = default): ring depth in slots of 16 KB + block_n * 128 B."""
    _need(x, torch.bfloat16, "x"); _need(w, torch.bfloat16, "w")
    assert x.dim() == 2 and w.dim() == 2 and x.stride(1) == 1 and w.is_contiguous() and x.shape[1] == w.shape[1]
    rows, k = x.shape
    n_out = w.shape[0] // 2 if epilogue == EPI_SILU else w.shape[0]
    if out is None:
        if epilogue == EPI_PARTIAL:
            out = torch.empty(k_splits, rows, n_out, dtype=torch.float32, device=x.device)
        else:
            out = torch.empty(rows, n_out, dtype=torch.bfloat16, device=x.device)
    lib = nat.load()
    nat.check(lib.b200_linear(x.data_ptr(), x.stride(0), w.data_ptr(), out.data_ptr(), out.stride(-2), rows, n_out, k,
                              epilogue, block_n, k_splits,
                              int(pdl) | (2 if shallow else 0) | ({1: 0, 2: 1, 4: 2}[cluster] << 2) | ((stages & 15) << 4),
                              _stream()))
    return out


def quant_fp8(x: torch.Tensor, out: torch.Tensor | None = None, scales: torch.Tensor | None = None):
    """Dynamic per-token, per-128-column e4m3 quantization of x [rows, k] bf16 -> (q [rows, k] e4m3, scales [rows, k/128] fp32)."""
    _need(x, torch.bfloat16, "x")
    assert x.dim() == 2 and x.stride(1) == 1
    rows, k = x.shape
    if out is None:
        out = torch.empty(rows, k, dtype=torch.float8_e4m3fn, device=x.device)
    if scales is None:
        scales = torch.empty(rows, k // 128, dtype=torch.float32, device=x.device)
    nat.check(nat.load().b200_quant_fp8(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), scales.data_ptr(),
                                        scales.stride(0), rows, k, _stream()))
    return out, scales


def linear_fp8(xq: torch.Tensor, x_scale: torch.Tensor, w: torch.Tensor, w_scale: torch.Tensor, epilogue: int = EPI_BF16,
               block_n: int = 64, k_splits: int = 1, pdl: bool = False, out: torch.Tensor | None = None,
               shallow: bool = False, cluster: int = 1, stages: int = 0) -> torch.Tensor:
    """``linear`` on block-scaled e4m3 operands: xq [rows, k] with x_scale [rows, k/128] (``quant_fp8``), w [n, k] with
    w_scale [n/128, k/128].  Same epilogues and flags as ``linear``."""
    _need(xq, torch.float8_e4m3fn, "xq"); _need(w, torch.float8_e4m3fn, "w")
    _need(x_scale, torch.float32, "x_scale"); _need(w_scale, torch.float32, "w_scale")
    assert xq.dim() == 2 and w.dim() == 2 and xq.stride(1) == 1 and w.is_contiguous() and xq.shape[1] == w.shape[1]
    rows, k = xq.shape
    assert w_scale.is_contiguous() and w_scale.shape == (w.shape[0] // 128, k // 128)
    assert x_scale.stride(1) == 1 and x_scale.shape == (rows, k // 128)
    n_out = w.shape[0] // 2 if epilogue == EPI_SILU else w.shape[0]
    if out is None:
        if epilogue == EPI_PARTIAL:
            out = torch.empty(k_splits, rows, n_out, dtype=torch.float32, device=xq.device)
        else:
            out = torch.empty(rows, n_out, dtype=torch.bfloat16, device=xq.device)
    nat.check(nat.load().b200_linear_fp8(xq.data_ptr(), xq.stride(0), x_scale.data_ptr(), x_scale.stride(0), w.data_ptr(),
                                         w_scale.data_ptr(), out.data_ptr(), out.stride(-2), rows, n_out, k, epilogue, block_n,
                                         k_splits,
                                         int(pdl) | (2 if shallow else 0) | ({1: 0, 2: 1, 4: 2}[cluster] << 2) | ((stages & 15) << 4),
                                         _stream()))
    return out


def add_rmsnorm_partials(partials: torch.Tensor, residual: torch.Tensor, weight: torch.Tensor, eps: float,
                         pdl: bool = False, out: torch.Tensor | None = None):
    """residual <- bf16(bf16(sum_s partials[s]) + residual); returns (rmsnorm(residual) * weight, residual)."""
    _need(partials, torch.float32, "partials"); _need(residual, torch.bfloat16, "residual"); _need(weight, torch.bfloat16, "weight")
    assert partials.dim() == 3 and partials.is_contiguous() and residual.is_contiguous()
    splits, rows, cols = partials.shape
    assert residual.shape == (rows, cols)
    if out is None:
        out = torch.empty_like(residual)
    lib = nat.load()
    nat.check(lib.b200_add_rmsnorm_partials(partials.data_ptr(), splits, residual.data_ptr(), weight.data_ptr(), out.data_ptr(),
                                            rows, cols, eps, int(pdl), _stream()))
    return out, residual


def lm_head_sample(hidden: torch.Tensor, lm_head: torch.Tensor, temperatures: torch.Tensor | None, seed: int, step: int,
                   key_workspace: torch.Tensor, out: torch.Tensor | None = None, index_offset: int = 0,
                   out_keys: torch.Tensor | None = None, step_dev: torch.Tensor | None = None, block_n: int = 128,
                   pdl: bool = False, shallow: bool = True, cluster: int = 1) -> torch.Tensor:
    """Fused LM head + sampling: hidden [rows, k] x lm_head [vocab, k] -> token ids, without materialising the logits.
    ``key_workspace``: int64/uint64 [>= rows], zero before the call, zero again after it."""
    _need(hidden, torch.bfloat16, "hidden"); _need(lm_head, torch.bfloat16, "lm_head")
    assert hidden.dim() == 2 and hidden.stride(1) == 1 and lm_head.is_contiguous() and hidden.shape[1] == lm_head.shape[1]
    assert key_workspace.is_cuda and key_workspace.element_size() == 8 and key_workspace.numel() >= hidden.shape[0]
    rows, k = hidden.shape
    if out is None and out_keys is None:
        out = torch.empty(rows, dtype=torch.int64, device=hidden.device)
    lib = nat.load()
    flags = int(pdl) | (2 if shallow and cluster == 1 else 0) | ({1: 0, 2: 1, 4: 2}[cluster] << 2)
    nat.check(lib.b200_lm_head_sample(hidden.data_ptr(), hidden.stride(0), lm_head.data_ptr(), rows, lm_head.shape[0], k,
                                      _ptr(temperatures), index_offset, seed & (2**64 - 1), step & (2**64 - 1), _ptr(step_dev),
                                      key_workspace.data_ptr(), _ptr(out), _ptr(out_keys), block_n, flags, _stream()))
    LAUNCHES[0] += 1                      # two kernels behind one call
    return out if out is not None else out_keys


# ---- mixture-of-experts MLP (csrc/moe.cu, grouped mode of csrc/linear_tc.cu; DESIGN.md 3.7) ------------------------------
MOE_MAX_EXPERTS, MOE_MAX_TOPK = 256, 16


def moe_route(logits: torch.Tensor, top_k: int, norm_topk: bool, ids: torch.Tensor | None = None,
              weights: torch.Tensor | None = None) -> tuple[torch.Tensor, torch.Tensor]:
    """bf16 router logits [T, E] -> (int32 expert ids [T, top_k], fp32 weights [T, top_k]), rank order."""
    _need(logits, torch.bfloat16, "logits")
    assert logits.dim() == 2 and logits.stride(1) == 1
    t, e = logits.shape
    if ids is None:
        ids = torch.empty(t, top_k, dtype=torch.int32, device=logits.device)
    if weights is None:
        weights = torch.empty(t, top_k, dtype=torch.float32, device=logits.device)
    _need(ids, torch.int32, "ids"); _need(weights, torch.float32, "weights")
    assert ids.is_contiguous() and weights.is_contiguous() and ids.shape == (t, top_k) and weights.shape == (t, top_k)
    nat.check(nat.load().b200_moe_route(logits.data_ptr(), logits.stride(0), t, e, top_k, int(norm_topk), ids.data_ptr(),
                                        weights.data_ptr(), _stream()))
    return ids, weights


def moe_max_tiles(entries: int, num_experts: int) -> int:
    n = nat.load().b200_moe_max_tiles(entries, num_experts)
    if n < 0:
        nat.check(-1)
    return n


def moe_align(ids: torch.Tensor, num_experts: int, perm: torch.Tensor | None = None,
              tiles: torch.Tensor | None = None) -> tuple[torch.Tensor, torch.Tensor]:
    """Expert ids (int32, any shape, entries in row-major order) -> (perm int32 [entries]: each entry's row in the
    permuted buffer, tiles int32 [1 + max_tiles, 4]: {n_tiles, rows, 0, 0} then {expert, first row, end row, 0})."""
    _need(ids, torch.int32, "ids")
    assert ids.is_contiguous()
    n = ids.numel()
    max_tiles = moe_max_tiles(n, num_experts)
    if perm is None:
        perm = torch.empty(n, dtype=torch.int32, device=ids.device)
    if tiles is None:
        tiles = torch.empty(1 + max_tiles, 4, dtype=torch.int32, device=ids.device)
    _need(perm, torch.int32, "perm"); _need(tiles, torch.int32, "tiles")
    assert perm.is_contiguous() and perm.numel() >= n and tiles.is_contiguous() and tiles.dim() == 2 and tiles.shape[1] == 4
    nat.check(nat.load().b200_moe_align(ids.data_ptr(), n, num_experts, perm.data_ptr(), tiles.data_ptr(), tiles.shape[0] - 1,
                                        _stream()))
    return perm, tiles


def moe_gather(x: torch.Tensor, top_k: int, perm: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """x [T, hidden] bf16 -> x_perm [T * top_k, hidden] with x_perm[perm[t * top_k + j]] = x[t]."""
    _need(x, torch.bfloat16, "x"); _need(perm, torch.int32, "perm")
    assert x.dim() == 2 and x.stride(1) == 1 and perm.is_contiguous() and perm.numel() >= x.shape[0] * top_k
    t, hidden = x.shape
    if out is None:
        out = torch.empty(t * top_k, hidden, dtype=x.dtype, device=x.device)
    _need(out, torch.bfloat16, "out")
    assert out.is_contiguous() and out.shape == (t * top_k, hidden)
    nat.check(nat.load().b200_moe_gather(x.data_ptr(), x.stride(0), t, hidden, top_k, perm.data_ptr(), out.data_ptr(), _stream()))
    return out


def moe_linear(x: torch.Tensor, w: torch.Tensor, tiles: torch.Tensor, epilogue: int = EPI_BF16, block_n: int = 64,
               pdl: bool = False, out: torch.Tensor | None = None, stages: int = 0) -> torch.Tensor:
    """Grouped GEMM over the permuted rows x [rows, k] and the stacked expert weights w [E, w_rows, k] (``moe_align``'s
    tiles say which rows belong to which expert).  EPI_SILU: w_rows = 2 n (gate rows, then up rows), returns
    SiluAndMul [rows, n]; EPI_BF16: returns [rows, w_rows]."""
    _need(x, torch.bfloat16, "x"); _need(w, torch.bfloat16, "w"); _need(tiles, torch.int32, "tiles")
    assert x.dim() == 2 and x.is_contiguous() and w.dim() == 3 and w.is_contiguous() and x.shape[1] == w.shape[2]
    assert tiles.is_contiguous() and tiles.dim() == 2 and tiles.shape[1] == 4
    if epilogue not in (EPI_BF16, EPI_SILU):
        nat.check(-1)
    rows, k = x.shape
    e = w.shape[0]
    n_out = w.shape[1] // 2 if epilogue == EPI_SILU else w.shape[1]
    if out is None:
        out = torch.empty(rows, n_out, dtype=torch.bfloat16, device=x.device)
    _need(out, torch.bfloat16, "out")
    assert out.dim() == 2 and out.stride(1) == 1 and out.shape == (rows, n_out)
    nat.check(nat.load().b200_moe_linear(x.data_ptr(), w.data_ptr(), out.data_ptr(), out.stride(0), rows, e, n_out, k,
                                         tiles.data_ptr(), tiles.shape[0] - 1, epilogue, block_n, int(pdl) | ((stages & 15) << 4),
                                         _stream()))
    return out


def moe_combine(y: torch.Tensor, perm: torch.Tensor, weights: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """y [T * top_k, hidden] (expert outputs in permuted order), weights fp32 [T, top_k] -> bf16 [T, hidden],
    out[t] = bf16(sum_j weights[t, j] * y[perm[t * top_k + j]]) in rank order."""
    _need(y, torch.bfloat16, "y"); _need(perm, torch.int32, "perm"); _need(weights, torch.float32, "weights")
    assert y.is_contiguous() and weights.is_contiguous() and weights.dim() == 2 and perm.is_contiguous()
    t, top_k = weights.shape
    hidden = y.shape[1]
    assert y.shape[0] == t * top_k and perm.numel() >= t * top_k
    if out is None:
        out = torch.empty(t, hidden, dtype=torch.bfloat16, device=y.device)
    _need(out, torch.bfloat16, "out")
    assert out.dim() == 2 and out.stride(1) == 1 and out.shape == (t, hidden)
    nat.check(nat.load().b200_moe_combine(y.data_ptr(), perm.data_ptr(), weights.data_ptr(), t, hidden, top_k, out.data_ptr(),
                                          out.stride(0), _stream()))
    return out


def moe_mlp(x: torch.Tensor, router_logits: torch.Tensor, w_gate_up: torch.Tensor, w_down: torch.Tensor, top_k: int,
            norm_topk: bool, gate_up_block_n: int = 64, down_block_n: int = 64, pdl: bool = True,
            out: torch.Tensor | None = None) -> torch.Tensor:
    """The MoE MLP of Qwen3MoeSparseMoeBlock on the normalised input x [T, hidden] and its bf16 router logits [T, E]:
    route -> align -> gather -> grouped gate_up + SiluAndMul -> grouped down -> combine (six launches)."""
    e = w_gate_up.shape[0]
    ids, weights = moe_route(router_logits, top_k, norm_topk)
    perm, tiles = moe_align(ids, e)
    xp = moe_gather(x, top_k, perm)
    act = moe_linear(xp, w_gate_up, tiles, EPI_SILU, gate_up_block_n, pdl=pdl)
    y = moe_linear(act, w_down, tiles, EPI_BF16, down_block_n, pdl=pdl)
    return moe_combine(y, perm, weights, out=out)


# ---- the tail of a decoder layer as one persistent kernel (csrc/layer_tail.cu) ---------------------------------------------
def layer_tail_workspace(max_rows: int, hidden: int, inter: int, max_splits: int, device="cuda") -> torch.Tensor:
    """Zeroed workspace (grid-barrier state, split-K partials, the two intermediate activations)."""
    lib = nat.load()
    n = lib.b200_layer_tail_workspace_bytes(max_rows, hidden, inter, max_splits)
    if n == 0:
        raise nat.B200Error("bad layer-tail workspace dimensions")
    return torch.zeros(n, dtype=torch.uint8, device=device)


def layer_tail(attn_out: torch.Tensor, residual: torch.Tensor, w_o: torch.Tensor, ln_mid: torch.Tensor, w_gate_up: torch.Tensor,
               w_down: torch.Tensor, ln_next: torch.Tensor, eps: float, workspace: torch.Tensor, w_qkv_next: torch.Tensor | None = None,
               splits_o: int = 8, splits_down: int = 8, x_next: torch.Tensor | None = None, qkv_out: torch.Tensor | None = None):
    """o_proj -> add+RMSNorm -> gate_up+SiluAndMul -> down_proj -> add+RMSNorm [-> next qkv_proj] in ONE launch.
    ``residual`` is updated in place; returns (x_next, qkv_out or None)."""
    _need(attn_out, torch.bfloat16, "attn_out"); _need(residual, torch.bfloat16, "residual")
    for t, name in ((w_o, "w_o"), (w_gate_up, "w_gate_up"), (w_down, "w_down"), (ln_mid, "ln_mid"), (ln_next, "ln_next")):
        _need(t, torch.bfloat16, name)
        assert t.is_contiguous()
    assert attn_out.dim() == 2 and attn_out.stride(1) == 1 and residual.is_contiguous()
    rows, q_size = attn_out.shape
    hidden = residual.shape[1]
    inter = w_down.shape[1]
    assert w_o.shape == (hidden, q_size) and w_gate_up.shape == (2 * inter, hidden) and w_down.shape == (hidden, inter)
    if x_next is None:
        x_next = torch.empty_like(residual)
    qkv_n = 0
    if w_qkv_next is not None:
        _need(w_qkv_next, torch.bfloat16, "w_qkv_next")
        assert w_qkv_next.is_contiguous() and w_qkv_next.shape[1] == hidden
        qkv_n = w_qkv_next.shape[0]
        if qkv_out is None:
            qkv_out = torch.empty(rows, qkv_n, dtype=torch.bfloat16, device=residual.device)
    h = nat.handle()
    nat.check(h.lib.b200_layer_tail(h.ptr, attn_out.data_ptr(), attn_out.stride(0), residual.data_ptr(), w_o.data_ptr(), ln_mid.data_ptr(),
                                    w_gate_up.data_ptr(), w_down.data_ptr(), ln_next.data_ptr(), x_next.data_ptr(), _ptr(w_qkv_next),
                                    _ptr(qkv_out), qkv_out.stride(0) if qkv_out is not None else 0, qkv_n, workspace.data_ptr(),
                                    workspace.numel(), rows, hidden, q_size, inter, eps, splits_o, splits_down, _stream()), h.ptr)
    return x_next, qkv_out


def layer_tail_error(workspace: torch.Tensor) -> bool:
    """True if a grid barrier of some launch on this workspace gave up waiting (results of that launch are undefined)."""
    return int(workspace[8:12].view(torch.int32).item()) != 0
