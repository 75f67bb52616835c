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
