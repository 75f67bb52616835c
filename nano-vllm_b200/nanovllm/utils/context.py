"""Per-step attention metadata, handed to the operator out of band.

The reference threads these tensors to ``Attention.forward`` through a process-global record instead of
function arguments (reference nanovllm/utils/context.py:5-27); the operator seam keeps that contract, so the
field names and the three accessors below are the reference's.  Here the record is one long-lived object
whose fields are overwritten in place every step (no allocation on the step path).

Field meaning (shapes as built by the runner, engine/model_runner.py:129-188 in the reference):
  is_prefill      bool    prefill (varlen) or decode (one token per sequence)
  cu_seqlens_q/k  int32   [S+1] cumulative query / key lengths of a prefill batch
  max_seqlen_q/k  int     their maxima (host ints)
  slot_mapping    int32   [T] cache slot of every new token, -1 = skip
  context_lens    int32   [B] keys visible to each decode row, 0 = CUDA-graph padding row
  block_tables    int32   [S or B, W] page ids, -1 padded; None = packed prefill without cache reads
  kv_groups       list    fp8 cache only: the paged prefill's sequences cut into groups whose keys fit the
                          dequantization scratch (layers/attention.py:KVGroup); None otherwise
"""
from __future__ import annotations

_FIELDS = ("is_prefill", "cu_seqlens_q", "cu_seqlens_k", "max_seqlen_q", "max_seqlen_k",
           "slot_mapping", "context_lens", "block_tables", "kv_groups")
_DEFAULTS = (False, None, None, 0, 0, None, None, None, None)


class Context:
    __slots__ = _FIELDS

    def __init__(self, *values, **named):
        self.assign(*values, **named)

    def assign(self, *values, **named) -> "Context":
        merged = dict(zip(_FIELDS, _DEFAULTS))
        merged.update(zip(_FIELDS, values))
        merged.update(named)
        for name in _FIELDS:
            setattr(self, name, merged[name])
        return self

    def __repr__(self) -> str:
        return "Context(" + ", ".join(f"{n}={getattr(self, n)!r}" for n in _FIELDS) + ")"


_STEP = Context()


def get_context() -> Context:
    return _STEP


def set_context(is_prefill, cu_seqlens_q=None, cu_seqlens_k=None, max_seqlen_q=0, max_seqlen_k=0,
                slot_mapping=None, context_lens=None, block_tables=None, kv_groups=None) -> None:
    _STEP.assign(is_prefill, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k,
                 slot_mapping, context_lens, block_tables, kv_groups)


def reset_context() -> None:
    _STEP.assign()
