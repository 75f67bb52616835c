"""Qwen3 dense decoder on the libb200attn kernels (reference nanovllm/models/qwen3.py:14-216).

Same architecture and the same rounding points as the reference's GPU path: GQA with per-head q/k
RMSNorm before NeoX RoPE, SwiGLU MLP, fused residual-add + RMSNorm; bf16 tensors between ops, fp32
inside them.  Per layer and per step this issues

    add_rmsnorm -> qkv GEMM -> [q/k-norm + RoPE + KV scatter] -> paged attention -> o GEMM (+all-reduce)
    -> add_rmsnorm -> gate_up GEMM -> silu*mul -> down GEMM (+all-reduce)
(for small decode batches the bracket and the attention are one kernel, b200_paged_decode_fused)

GEMMs are library calls (cuBLAS through ``F.linear``, as in the reference, linear.py:51,73,153);
everything else is one hand-written kernel from libb200attn.  Tensor parallelism shards heads and
MLP columns exactly like the reference's *ParallelLinear classes (linear.py:54-156) and all-reduces
after o_proj and down_proj only; the embedding table is replicated and the LM head stays
vocab-sharded with a (max, argmax) combine instead of a logits gather (embed_head.py:56-66).

This is a plain object, not an nn.Module tree: weights are named tensors, ``forward`` is a flat
list of launches, which is what gets captured into the decode CUDA graphs.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from types import SimpleNamespace

import torch
import torch.distributed as dist
import torch.nn.functional as F

from .. import ops
from ..layers.attention import Attention
from ..layers.rotary_embedding import build_cos_sin
from ..utils import fp8 as fp8fmt
from ..utils.context import get_context


@dataclass
class LayerWeights:
    qkv: torch.Tensor         # [(Hq + 2 Hkv) * D / tp, hidden]
    o: torch.Tensor           # [hidden, Hq * D / tp]
    gate_up: torch.Tensor     # [2 * I / tp, hidden]
    down: torch.Tensor        # [hidden, I / tp]
    ln1: torch.Tensor
    ln2: torch.Tensor
    q_norm: torch.Tensor
    k_norm: torch.Tensor
    # block-FP8 checkpoints: the four projections above are e4m3 and these are their fp32 [N / 128, K / 128] block scales
    qkv_s: torch.Tensor | None = None
    o_s: torch.Tensor | None = None
    gate_up_s: torch.Tensor | None = None
    down_s: torch.Tensor | None = None
    # mixture-of-experts layers (models/qwen3_moe.py): the router [E, hidden]; gate_up / down are then [E, 2 * I / tp, hidden]
    # and [E, hidden, I / tp]
    gate: torch.Tensor | None = None


class Qwen3ForCausalLM:
    # HF checkpoint name -> (packed parameter, shard id), as in the reference (qwen3.py:187-193)
    packed_modules_mapping = {
        "q_proj": ("qkv_proj", "q"), "k_proj": ("qkv_proj", "k"), "v_proj": ("qkv_proj", "v"),
        "gate_proj": ("gate_up_proj", 0), "up_proj": ("gate_up_proj", 1),
    }

    def __init__(self, hf_config, tp_rank: int = 0, tp_size: int = 1, device="cuda", max_position: int | None = None):
        c = hf_config
        self.cfg = c
        self.fp8 = fp8fmt.is_block_fp8(c)          # the checkpoint's quantization_config is the switch (DESIGN.md 3.6)
        self.tp_rank, self.tp_size = tp_rank, tp_size
        self.device = torch.device(device)
        self.hidden = c.hidden_size
        self.head_dim = getattr(c, "head_dim", None) or c.hidden_size // c.num_attention_heads
        assert c.num_attention_heads % tp_size == 0 and c.num_key_value_heads % tp_size == 0
        assert c.vocab_size % tp_size == 0 and self._intermediate_size(c) % tp_size == 0
        self.num_heads = c.num_attention_heads // tp_size
        self.num_kv_heads = c.num_key_value_heads // tp_size
        self.inter = self._intermediate_size(c) // tp_size
        self.vocab_shard = c.vocab_size // tp_size
        self.eps = c.rms_norm_eps
        self.q_size = self.num_heads * self.head_dim
        self.kv_size = self.num_kv_heads * self.head_dim
        if self.fp8:
            fp8fmt.check_shapes(self.q_size, self.kv_size, self.hidden, self.inter)
        self.tie = bool(getattr(c, "tie_word_embeddings", False))
        # b200_paged_decode_fused folds q/k-norm + RoPE + KV append into the decode kernel (one launch less per
        # layer).  The extra per-segment math lands on warps that are already busy, which costs more than the saved
        # launch at large batches, so it is used for decode batches up to this many rows; it exists for head groups
        # <= 2 only.
        self.fused_decode_max_batch = 128 if self.num_heads // self.num_kv_heads <= 2 else 0
        if "B200_FUSED_DECODE_MAX" in os.environ and self.fused_decode_max_batch:      # tuning knob (e.g. under TP)
            self.fused_decode_max_batch = int(os.environ["B200_FUSED_DECODE_MAX"])
        self.peer = None        # engine/peer_reduce.PeerReduce when tensor parallel over NVLink peer memory
        # Decode-size projections (profiles/step_time.py compares the policies step for step):
        #   B200_LINEAR=auto (default): the two row-parallel projections (o_proj, down_proj) of decode steps of up to 128 rows
        #       run on wgmma with split-K 8 and the add+RMSNorm that follows consumes the fp32 partials in split order
        #       (csrc/linear_tc.cu), so that all SMs stream weights; the wide projections (qkv, gate_up) stay cuBLAS, as
        #       under tensor parallelism;
        #   cublas: every projection through the library;  rows / tc: force the wgmma path for o/down / all four;
        #   gu: only gate_up + SiluAndMul on wgmma (one launch less per layer), the rest through the library.
        #   B200_LINEAR_CFG = "qkv_bn,gate_up_bn,o_bn,o_splits,down_bn,down_splits,pdl".
        mode = os.environ.get("B200_LINEAR", "auto")
        self.tc_linear = mode in ("tc", "rows") or (mode == "auto" and tp_size == 1)
        self.tc_cols = mode == "tc"               # "rows"/"auto": only the row-parallel o_proj / down_proj
        self.tc_gate_up = mode == "gu" and self.inter % 32 == 0
        self.tc_gate_up_max = int(os.environ.get("B200_LINEAR_GU_MAX_ROWS", "256"))
        self.tc_cfg = [int(v) for v in os.environ.get("B200_LINEAR_CFG", "64,64,64,8,64,8,1").split(",")]
        self.tc_max_rows = int(os.environ.get("B200_LINEAR_MAX_ROWS", "128" if mode == "auto" else "256"))
        # above 128 rows a CTA row block is added, so fewer k splits cover the SMs; B200_LINEAR_SPLITS_BIG overrides.
        self.tc_big_splits = int(os.environ.get("B200_LINEAR_SPLITS_BIG", "4"))
        fit = lambda k, s: next(d for d in range(max(1, min(s, k // 64)), 0, -1) if (k // 64) % d == 0)     # split-K factors must divide the k tiles
        tcc = self.tc_cfg
        if self.q_size % 64 or self.inter % 64 or self.hidden % tcc[2] or self.hidden % tcc[4]:
            self.tc_linear = False                # shapes the wgmma kernel does not tile: library GEMMs
        else:
            tcc[3], tcc[5] = fit(self.q_size, tcc[3]), fit(self.inter, tcc[5])
            self.tc_big = (fit(self.q_size, min(tcc[3], self.tc_big_splits)), fit(self.inter, min(tcc[5], self.tc_big_splits)))
        # B200_TAIL=mega: in decode steps of up to 256 rows on one GPU, everything between two attention kernels
        # (o_proj, add+norm, gate_up+SiluAndMul, down_proj, add+norm, the next layer's qkv_proj) is ONE persistent launch
        # (csrc/layer_tail.cu) instead of seven.  Every phase is an all-to-all dependency (a norm needs whole rows), so a grid
        # barrier and a pipeline refill per phase compete with a launch boundary under PDL: an opt-in experiment, off by default.
        self.mega_tail = os.environ.get("B200_TAIL", "") == "mega" and tp_size == 1
        self.mega_rows = 256
        want = [int(v) for v in os.environ.get("B200_TAIL_SPLITS", "8,8").split(",")]
        fit = lambda k, s: next(d for d in range(min(s, k // 64), 0, -1) if (k // 64) % d == 0)     # split-K factors must divide the k tiles
        self.mega_splits = [fit(self.q_size, want[0]), fit(self.inter, want[1])] if self.q_size % 64 == 0 and self.inter % 64 == 0 else [1, 1]
        self._tail_ws = None
        # Two-stream decode step (B200_DUAL, _forward_dual): a decode batch of >= dual_min rows is cut into two halves that
        # run on two streams, half a layer out of phase: while one half is in its HBM-bound attention kernel (fp32-FMA pipe +
        # bulk copies, ~155 KB of shared memory, one CTA per SM) the other half's latency-bound projection chain runs on
        # the SAME SMs -- wgmma + TMA, a 3-slot ring (~72 KB) and ~30k registers, which is what the attention CTA leaves
        # free.  Attention kernels never overlap each other (an event chain orders them), so HBM always has one streaming
        # kernel and the chain of the other half hides under it.  One GPU, head groups <= 2 (the FMA decode kernel).
        #   B200_DUAL_CFG = "qkv_bn,gate_up_bn,o_bn,o_splits,down_bn,down_splits,ring_slots"
        # A half batch costs more than half of a full one (attention and the projection chain are both latency bound at
        # these sizes), so this is off by default.
        dual = os.environ.get("B200_DUAL", "0")
        self.dual = dual not in ("0", "", "off") and tp_size == 1 and self.num_heads // self.num_kv_heads <= 2
        self.dual_min = int(os.environ.get("B200_DUAL_MIN", "144"))
        self.dual_cfg = [int(v) for v in os.environ.get("B200_DUAL_CFG", "64,64,64,8,64,8,3").split(",")]
        if self.q_size % 64 or self.inter % 64 or self.hidden % self.dual_cfg[2] or self.hidden % self.dual_cfg[4] \
                or (self.q_size + 2 * self.kv_size) % self.dual_cfg[0] or self.inter % (self.dual_cfg[1] // 2):
            self.dual = False
        else:
            self.dual_cfg[3], self.dual_cfg[5] = fit(self.q_size, self.dual_cfg[3]), fit(self.inter, self.dual_cfg[5])
        self._dual_state = None
        if self.fp8:            # the wgmma / layer-tail / two-stream experiments above are bf16-only
            self.tc_linear = self.tc_gate_up = self.mega_tail = self.dual = False
        if getattr(c, "attention_bias", False):
            raise NotImplementedError("qkv bias (Qwen2-style) is outside the Qwen3 hot path")
        theta = getattr(c, "rope_theta", 1000000.0)
        scaling = getattr(c, "rope_scaling", None) or getattr(c, "rope_parameters", None)
        if isinstance(scaling, dict):
            theta = scaling.get("rope_theta", theta)
        self.rope_theta = float(theta)
        self.cos_sin = build_cos_sin(self.head_dim, max_position or c.max_position_embeddings, self.rope_theta, self.device)

        dt, dev = torch.bfloat16, self.device
        e = lambda *s: torch.empty(*s, dtype=dt, device=dev)
        self.embed = e(c.vocab_size, self.hidden)                       # replicated
        self.lm_head = (self.embed[tp_rank * self.vocab_shard:(tp_rank + 1) * self.vocab_shard]
                        if self.tie else e(self.vocab_shard, self.hidden))
        self.norm = e(self.hidden)
        proj = [(self.q_size + 2 * self.kv_size, self.hidden), (self.hidden, self.q_size), *self._mlp_shapes()]
        if self.fp8:
            q8 = lambda n, k: torch.empty(n, k, dtype=torch.float8_e4m3fn, device=dev)
            sc = lambda n, k: torch.empty(n // fp8fmt.BLOCK, k // fp8fmt.BLOCK, dtype=torch.float32, device=dev)
            self.layers = [LayerWeights(*(q8(*p) for p in proj), e(self.hidden), e(self.hidden), e(self.head_dim), e(self.head_dim),
                                        *(sc(*p) for p in proj))
                           for _ in range(c.num_hidden_layers)]
        else:
            self.layers = [LayerWeights(*(e(*p) for p in proj), e(self.hidden), e(self.hidden), e(self.head_dim), e(self.head_dim))
                           for _ in range(c.num_hidden_layers)]
        scale = self.head_dim ** -0.5
        self.attn = [Attention(self.num_heads, self.head_dim, scale, self.num_kv_heads) for _ in self.layers]
        for i, a in enumerate(self.attn):
            a.layer_id = i

    @staticmethod
    def _intermediate_size(c) -> int:
        return c.intermediate_size

    def _mlp_shapes(self) -> list[tuple]:
        """Shapes of this rank's gate_up and down weights."""
        return [(2 * self.inter, self.hidden), (self.hidden, self.inter)]

    # ---- weights -------------------------------------------------------------------------------
    def load_hf_tensor(self, name: str, w: torch.Tensor) -> None:
        """Place one HF-named checkpoint tensor, slicing this rank's shard (linear.py:65-70,87-93,114-128,142-150)."""
        r, n = self.tp_rank, self.tp_size
        if name == "model.embed_tokens.weight":
            self.embed.copy_(w); return
        if name == "lm_head.weight":
            if not self.tie:
                self.lm_head.copy_(w.chunk(n, 0)[r])
            return
        if name == "model.norm.weight":
            self.norm.copy_(w); return
        parts = name.split(".")
        assert parts[0] == "model" and parts[1] == "layers", name
        L = self.layers[int(parts[2])]
        leaf = ".".join(parts[3:-1])
        if leaf in fp8fmt.PROJECTIONS:
            scale = parts[-1] == "weight_scale_inv"
            if scale and not self.fp8:
                raise NotImplementedError(f"{name}: block-FP8 scales in a checkpoint whose config.json has no fp8 quantization_config")
            if not scale and self.fp8 != (w.dtype == torch.float8_e4m3fn):
                raise NotImplementedError(f"{name} is {w.dtype}, but the checkpoint's config.json says "
                                          f"{'block-FP8 (e4m3)' if self.fp8 else 'unquantized'} projections")
            dst, dim = self._projection_slot(L, leaf, scale)
            dst.copy_(w.chunk(n, dim)[r])        # scales: column-parallel rows / row-parallel columns, whole 128-blocks
        elif leaf == "input_layernorm":
            L.ln1.copy_(w)
        elif leaf == "post_attention_layernorm":
            L.ln2.copy_(w)
        elif leaf == "self_attn.q_norm":
            L.q_norm.copy_(w)
        elif leaf == "self_attn.k_norm":
            L.k_norm.copy_(w)
        else:
            raise KeyError(f"unexpected checkpoint tensor {name}")

    def _projection_slot(self, L: LayerWeights, leaf: str, scale: bool):
        """(destination, tensor-parallel split dim) of a projection weight, or of its block scales (one row / column per
        128 weight rows / columns): q/k/v pack into qkv, gate/up into gate_up (linear.py:65-70,87-93,114-128,142-150)."""
        b = fp8fmt.BLOCK if scale else 1
        q, kv, inter = self.q_size // b, self.kv_size // b, self.inter // b
        qkv, o, gu, down = (L.qkv_s, L.o_s, L.gate_up_s, L.down_s) if scale else (L.qkv, L.o, L.gate_up, L.down)
        return {"self_attn.q_proj": (qkv[:q], 0), "self_attn.k_proj": (qkv[q:q + kv], 0), "self_attn.v_proj": (qkv[q + kv:], 0),
                "self_attn.o_proj": (o, 1), "mlp.gate_proj": (gu[:inter], 0), "mlp.up_proj": (gu[inter:], 0),
                "mlp.down_proj": (down, 1)}[leaf]

    def modules(self):
        """The attention operators, in layer order (what allocate_kv_cache walks, model_runner.py:116-121)."""
        return iter(self.attn)

    # ---- forward -------------------------------------------------------------------------------
    def _fp8_linear(self, x: torch.Tensor, w: torch.Tensor, s: torch.Tensor, epilogue: int, block_n: int, k_splits: int = 1,
                    out: torch.Tensor | None = None) -> torch.Tensor:
        """Block-FP8 projection: per-token e4m3 quantization of x, then the wgmma e4m3 GEMM (csrc/linear_tc.cu)."""
        pdl = bool(self.tc_cfg[6])
        xq, xs = ops.quant_fp8(x)
        return ops.linear_fp8(xq, xs, w, s, epilogue, block_n, k_splits, pdl=pdl, out=out)

    def _row_linear_fp8(self, x: torch.Tensor, w: torch.Tensor, s: torch.Tensor):
        """_row_linear on block-FP8 weights: split-K fp32 partials for decode-size batches on one GPU, bf16 into the
        peer-mapped buffer under tensor parallelism, a bf16 output otherwise (prefill)."""
        t, peer = x.shape[0], self.peer
        if self.tp_size == 1 and t <= 128:
            kb = x.shape[1] // fp8fmt.BLOCK
            splits = next(d for d in range(min(8, kb), 0, -1) if kb % d == 0)
            return self._fp8_linear(x, w, s, ops.EPI_PARTIAL, 64, splits), "parts"
        if peer is not None and t <= peer.rows_cap:
            out = peer.next_out(t)
            self._fp8_linear(x, w, s, ops.EPI_BF16, 32, out=out)
            return out, True
        return self._fp8_linear(x, w, s, ops.EPI_BF16, 64), False

    def _row_linear(self, x: torch.Tensor, w: torch.Tensor, tc=None):
        """Row-parallel GEMM (o_proj / down_proj).  Returns (partial, where): where is True when the partial sits in
        the peer-mapped buffer, "parts" when it is the fp32 split-K partials of the wgmma path."""
        peer = self.peer
        if tc is not None and self.tp_size == 1:
            return ops.linear(x, w, ops.EPI_PARTIAL, tc[0], tc[1], pdl=bool(self.tc_cfg[6])), "parts"
        if tc is not None:           # tensor parallel: K is already divided by the ranks; write bf16 straight into the peer buffer
            out = peer.next_out(x.shape[0])
            ops.linear(x, w, ops.EPI_BF16, min(tc[0], 32), pdl=bool(self.tc_cfg[6]), out=out)
            return out, True
        if peer is not None and x.shape[0] <= peer.rows_cap:
            out = peer.next_out(x.shape[0])
            torch.mm(x, w.t(), out=out)
            return out, True
        return F.linear(x, w), False

    def _reduce_add_norm(self, h, in_peer: bool, residual, weight):
        """all-reduce over the TP ranks + residual add + RMSNorm (linear.py:152-156 + layernorm.py:28-40)."""
        if in_peer == "parts":
            return ops.add_rmsnorm_partials(h, residual, weight, self.eps, pdl=bool(self.tc_cfg[6]))
        if in_peer:
            return self.peer.reduce_add_norm(h.shape[0], residual, weight, self.eps)
        if self.tp_size > 1:
            dist.all_reduce(h)
        return ops.add_rmsnorm(h, residual, weight, self.eps)

    def _attention(self, li: int, qkv: torch.Tensor, positions: torch.Tensor, ctx, before_attention=None, no_pdl: bool = False):
        """q/k-norm + RoPE + KV append + attention on the raw qkv projection (one or two launches) -> [t, q_size].
        ``before_attention`` runs right before the attention launch (cross-stream waits of the two-stream step);
        ``no_pdl``: that launch carries no programmatic-dependent-launch attribute.  Decode steps only when either is used."""
        import contextlib
        L, attn = self.layers[li], self.attn[li]
        hq, hkv, d, t = self.num_heads, self.num_kv_heads, self.head_dim, qkv.shape[0]
        cached = attn.k_cache.numel() > 0
        plain = ops.pdl_off() if no_pdl else contextlib.nullcontext()
        if cached and not ctx.is_prefill and t <= self.fused_decode_max_batch:
            if before_attention is not None:
                before_attention()
            with plain:
                o = ops.paged_decode_fused(li, qkv, hq, L.q_norm, L.k_norm, self.cos_sin, self.eps, ctx.block_tables,
                                           ctx.context_lens, attn.scale)
        else:
            ops.qknorm_rope_store(li, qkv, hq, hkv, positions, L.q_norm, L.k_norm, self.cos_sin, self.eps,
                                  ctx.slot_mapping if cached else None)
            q = qkv[:, :self.q_size].view(t, hq, d)
            k = qkv[:, self.q_size:self.q_size + self.kv_size].view(t, hkv, d)
            v = qkv[:, self.q_size + self.kv_size:].view(t, hkv, d)
            if before_attention is not None:
                before_attention()
                with plain:                                   # decode: the operator's decode branch, on this half's metadata
                    o = ops.paged_decode(li, q, ctx.block_tables, ctx.context_lens, attn.scale)
            else:
                o = attn(q, k, v, kv_stored=True)
        return o.reshape(t, self.q_size)

    def _forward_mega(self, input_ids: torch.Tensor, positions: torch.Tensor, ctx) -> torch.Tensor:
        """Decode step with two launches per layer: attention, then the persistent layer tail (which also produces the
        next layer's qkv projection)."""
        if self._tail_ws is None:
            self._tail_ws = ops.layer_tail_workspace(self.mega_rows, self.hidden, self.inter, max(self.mega_splits), self.device)
        residual = ops.embedding(input_ids, self.embed)
        x = ops.rmsnorm(residual, self.layers[0].ln1, self.eps)
        qkv = F.linear(x, self.layers[0].qkv)
        n = len(self.layers)
        for li, L in enumerate(self.layers):
            o = self._attention(li, qkv, positions, ctx)
            nxt = self.layers[li + 1] if li + 1 < n else None
            x, qkv = ops.layer_tail(o, residual, L.o, L.ln2, L.gate_up, L.down, nxt.ln1 if nxt is not None else self.norm, self.eps,
                                    self._tail_ws, w_qkv_next=nxt.qkv if nxt is not None else None,
                                    splits_o=self.mega_splits[0], splits_down=self.mega_splits[1])
        return x

    # ---- two-stream decode step ------------------------------------------------------------------
    def _dual_streams(self):
        """(main stream, side stream, one event per layer and half, fork/join events); CPU tensors (glue tests): no streams."""
        if self.device.type != "cuda":
            return None
        if self._dual_state is None:
            n = len(self.layers)
            self._dual_state = (torch.cuda.Stream(self.device), [[torch.cuda.Event(), torch.cuda.Event()] for _ in range(n)],
                                torch.cuda.Event(), torch.cuda.Event())
        return self._dual_state

    def _forward_dual(self, input_ids: torch.Tensor, positions: torch.Tensor, ctx) -> torch.Tensor:
        """Decode step as two half batches on two streams, half a layer out of phase (see __init__).  Per half and layer:
        add+norm(split-K partials) -> qkv (wgmma) -> attention [no PDL, after the other half's attention] -> o_proj split-K
        [no PDL] -> add+norm -> gate_up+SiluAndMul (wgmma) -> down_proj split-K.  Same rounding points as the single-stream
        wgmma path (split-K partials summed in split order by the add+norm)."""
        import contextlib
        n = input_ids.shape[0]
        h0 = (n + 1) // 2
        cfg, eps = self.dual_cfg, self.eps
        ring = cfg[6]
        st = self._dual_streams()
        hidden = ops.embedding(input_ids, self.embed)        # the residual stream of both halves, updated in place
        out = torch.empty_like(hidden)
        if st is not None:
            side, events, ev_fork, ev_join = st
            main = torch.cuda.current_stream()
            ev_fork.record(main)
            side.wait_event(ev_fork)
            streams = (main, side)
        halves = []
        for k, (a, b) in enumerate(((0, h0), (h0, n))):
            sub = SimpleNamespace(is_prefill=False, slot_mapping=ctx.slot_mapping[a:b] if ctx.slot_mapping is not None else None,
                                  context_lens=ctx.context_lens[a:b], block_tables=ctx.block_tables[a:b])
            halves.append(SimpleNamespace(a=a, b=b, residual=hidden[a:b], pos=positions[a:b], ctx=sub, parts=None))
        last_attn = None                                      # event of the most recent attention launch (either half)
        nl = len(self.layers)
        for li, L in enumerate(self.layers):
            for k, hb in enumerate(halves):
                if hb.b == hb.a:
                    continue
                scope = torch.cuda.stream(streams[k]) if st is not None else contextlib.nullcontext()
                with scope:
                    if hb.parts is None:
                        x = ops.rmsnorm(hb.residual, L.ln1, eps)
                    else:
                        x, _ = ops.add_rmsnorm_partials(hb.parts, hb.residual, L.ln1, eps, pdl=True)
                    qkv = ops.linear(x, L.qkv, ops.EPI_BF16, cfg[0], pdl=True, stages=ring)

                    def before_attention(k=k):
                        if st is not None and last_attn is not None:
                            streams[k].wait_event(last_attn)

                    o = self._attention(li, qkv, hb.pos, hb.ctx, before_attention=before_attention, no_pdl=True)
                    if st is not None:
                        last_attn = events[li][k]
                        last_attn.record(streams[k])
                    # an early-launched dependent of the attention kernel would sit on the shared memory the other half needs
                    parts = ops.linear(o, L.o, ops.EPI_PARTIAL, cfg[2], cfg[3], pdl=False, stages=ring)
                    x, _ = ops.add_rmsnorm_partials(parts, hb.residual, L.ln2, eps, pdl=True)
                    act = ops.linear(x, L.gate_up, ops.EPI_SILU, cfg[1], pdl=True, stages=ring)
                    hb.parts = ops.linear(act, L.down, ops.EPI_PARTIAL, cfg[4], cfg[5], pdl=True, stages=ring)
                    if li == nl - 1:
                        ops.add_rmsnorm_partials(hb.parts, hb.residual, self.norm, eps, pdl=True, out=out[hb.a:hb.b])
        if st is not None:
            ev_join.record(side)
            main.wait_event(ev_join)
        return out

    @torch.inference_mode()
    def forward(self, input_ids: torch.Tensor, positions: torch.Tensor) -> torch.Tensor:
        ctx = get_context()
        eps, hq, hkv, d = self.eps, self.num_heads, self.num_kv_heads, self.head_dim
        if self.dual and not ctx.is_prefill and input_ids.shape[0] >= self.dual_min and self.attn[0].k_cache.numel() > 0:
            return self._forward_dual(input_ids, positions, ctx)
        if self.mega_tail and not ctx.is_prefill and input_ids.shape[0] <= self.mega_rows and self.attn[0].k_cache.numel() > 0:
            return self._forward_mega(input_ids, positions, ctx)
        h = ops.embedding(input_ids, self.embed)
        residual, in_peer = None, False
        cfg = self.tc_cfg
        tc = self.tc_linear and h.shape[0] <= self.tc_max_rows and (
            self.tp_size == 1 or (self.peer is not None and h.shape[0] <= self.peer.rows_cap))
        for li, L in enumerate(self.layers):
            attn = self.attn[li]
            if residual is None:
                residual, x = h, ops.rmsnorm(h, L.ln1, eps)
            else:
                x, residual = self._reduce_add_norm(h, in_peer, residual, L.ln1)
            t = x.shape[0]
            if self.fp8:
                qkv = self._fp8_linear(x, L.qkv, L.qkv_s, ops.EPI_BF16, 64)
            else:
                qkv = ops.linear(x, L.qkv, ops.EPI_BF16, cfg[0], pdl=bool(cfg[6])) if (tc and self.tc_cols) else F.linear(x, L.qkv)
            cached = attn.k_cache.numel() > 0
            if cached and not ctx.is_prefill and t <= self.fused_decode_max_batch:
                # decode: q/k-norm, RoPE, KV append and attention in ONE launch on the raw projection output
                o = ops.paged_decode_fused(li, qkv, hq, L.q_norm, L.k_norm, self.cos_sin, eps, ctx.block_tables,
                                           ctx.context_lens, attn.scale)
            else:
                ops.qknorm_rope_store(li, qkv, hq, hkv, positions, L.q_norm, L.k_norm, self.cos_sin, eps,
                                      ctx.slot_mapping if cached else None)
                q = qkv[:, :self.q_size].view(t, hq, d)
                k = qkv[:, self.q_size:self.q_size + self.kv_size].view(t, hkv, d)
                v = qkv[:, self.q_size + self.kv_size:].view(t, hkv, d)
                o = attn(q, k, v, kv_stored=True)
            big = tc and t > 128
            if self.fp8:
                h, in_peer = self._row_linear_fp8(o.reshape(t, self.q_size), L.o, L.o_s)
            else:
                h, in_peer = self._row_linear(o.reshape(t, self.q_size), L.o, (cfg[2], self.tc_big[0] if big else cfg[3]) if tc else None)
            x, residual = self._reduce_add_norm(h, in_peer, residual, L.ln2)
            h, in_peer = self._mlp(L, x, ctx, tc, big)
        x, _ = self._reduce_add_norm(h, in_peer, residual, self.norm)
        return x

    def _mlp(self, L: LayerWeights, x: torch.Tensor, ctx, tc: bool, big: bool):
        """gate_up -> SiluAndMul -> down on the normalised x; returns (partial, where) as _row_linear."""
        t, cfg = x.shape[0], self.tc_cfg
        if self.fp8:
            act = self._fp8_linear(x, L.gate_up, L.gate_up_s, ops.EPI_SILU, 64)
        elif (tc and self.tc_cols) or (self.tc_gate_up and not ctx.is_prefill and t <= self.tc_gate_up_max):
            act = ops.linear(x, L.gate_up, ops.EPI_SILU, cfg[1], pdl=bool(cfg[6]))
        else:
            act = ops.silu_mul(F.linear(x, L.gate_up))
        if self.fp8:
            return self._row_linear_fp8(act, L.down, L.down_s)
        return self._row_linear(act, L.down, (cfg[4], self.tc_big[1] if big else cfg[5]) if tc else None)

    __call__ = forward

    @torch.inference_mode()
    def last_token_rows(self, hidden: torch.Tensor) -> torch.Tensor:
        """The hidden state of the last token of every sequence (embed_head.py:58-60)."""
        ctx = get_context()
        if ctx.is_prefill:
            last = (ctx.cu_seqlens_q[1:] - 1).to(torch.long)
            hidden = hidden.index_select(0, last)
        return hidden

    @torch.inference_mode()
    def compute_logits(self, hidden: torch.Tensor) -> torch.Tensor:
        """Logits of this rank's vocab shard for the last token of every sequence (embed_head.py:56-61)."""
        return F.linear(self.last_token_rows(hidden), self.lm_head)
