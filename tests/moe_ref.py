"""Reference of the Qwen3 mixture-of-experts MLP (DESIGN.md 3.7), restated in torch.

* router logits x W_gate^T, rounded to the dtype of x (bf16 in the engine's pipeline);
* routing: softmax over the E experts in fp32, the top k by probability descending then expert id ascending, divided by
  their fp32 sum when norm_topk_prob is set; the weights stay fp32;
* expert MLP down_e(SiluAndMul(gate_up_e(x))) with the dense model's rounding points (oracle.qwen3_ref, "fused");
* combine: out[t] = sum_j w[t, j] y_j[t] in rank order, rounded once.
``moe_block_ref`` runs in the dtype of its inputs: bf16 tensors give the engine's rounding points, float64 tensors the
exact block (routing still in fp32, as HF's router computes it).  ``Qwen3MoeRef`` is oracle.qwen3_ref's forward with
the MLP replaced by it; it records every layer's router logits of the last forward for the routing-gap checks.
"""
from __future__ import annotations

import math
import random
from types import SimpleNamespace

import torch
import torch.nn.functional as F

from oracle import qwen3_ref
from oracle.paged_attention_ref import attention_forward_ref


def route_ref(logits: torch.Tensor, k: int, norm: bool) -> tuple[torch.Tensor, torch.Tensor]:
    """logits [T, E] -> (expert ids int64 [T, k], fp32 weights [T, k]) in rank order."""
    p = torch.softmax(logits.float(), dim=-1)
    order = torch.sort(-p, dim=-1, stable=True).indices[:, :k]         # ties: the lower expert id first
    w = p.gather(1, order)
    if norm:
        w = w / w.sum(dim=-1, keepdim=True)
    return order, w


def routing_gap(logits: torch.Tensor, k: int) -> torch.Tensor:
    """Per token, log(p_k / p_(k+1)) of its k-th and (k+1)-th routing probabilities (= their logit gap); inf when k = E."""
    if k >= logits.shape[-1]:
        return torch.full(logits.shape[:1], math.inf, dtype=torch.float64)
    top = torch.topk(logits.double(), k + 1, dim=-1).values
    return top[:, k - 1] - top[:, k]


def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    """One bf16 ulp at |x| (float64)."""
    e = torch.floor(torch.log2(x.double().abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def expert_mlp_ref(x: torch.Tensor, gate_up: torch.Tensor, down: torch.Tensor) -> torch.Tensor:
    """One expert's SwiGLU MLP, rounding where the dense model's kernels round (exact in float64)."""
    h = F.linear(x, gate_up)
    if h.dtype == torch.float64:                          # silu_mul_ref computes in fp32
        g, u = h.chunk(2, -1)
        return F.linear(F.silu(g) * u, down)
    return F.linear(qwen3_ref.silu_mul_ref(h, "fused"), down)


def moe_block_ref(x: torch.Tensor, gate: torch.Tensor, gate_up: torch.Tensor, down: torch.Tensor, k: int, norm: bool,
                  routing: tuple | None = None) -> torch.Tensor:
    """Qwen3MoeSparseMoeBlock on x [T, hidden]: gate [E, hidden], gate_up [E, 2 I, hidden] (gate rows then up rows),
    down [E, hidden, I].  ``routing`` (ids, weights) replaces the router's choice when given."""
    ids, w = routing if routing is not None else route_ref(F.linear(x, gate), k, norm)
    y = torch.zeros(x.shape[0], k, x.shape[1], dtype=x.dtype)
    for e in torch.unique(ids).tolist():
        t, j = torch.where(ids == e)
        y[t, j] = expert_mlp_ref(x[t], gate_up[e], down[e])
    acc = torch.zeros(x.shape, dtype=torch.float64 if x.dtype == torch.float64 else torch.float32)
    for j in range(k):
        acc = acc + w[:, j:j + 1].to(acc.dtype) * y[:, j].to(acc.dtype)
    return acc.to(x.dtype)


def stack_experts(weights: dict, layer: int, num_experts: int) -> dict:
    """The router and the stacked expert tensors of one layer from the Hub's per-expert names."""
    p = f"model.layers.{layer}.mlp."
    ex = lambda e, n: weights[f"{p}experts.{e}.{n}.weight"]
    return dict(gate=weights[p + "gate.weight"],
                gate_up=torch.stack([torch.cat([ex(e, "gate_proj"), ex(e, "up_proj")], 0) for e in range(num_experts)]),
                down=torch.stack([ex(e, "down_proj") for e in range(num_experts)]))


class Qwen3MoeRef(qwen3_ref.Qwen3Ref):
    """The fp32 oracle of a Qwen3 MoE checkpoint: the dense oracle with every MLP a ``moe_block_ref``."""

    def __init__(self, dims, weights: dict, num_experts: int, top_k: int, norm_topk: bool, **kw):
        bf = dict(weights)
        for i in range(dims.num_hidden_layers):        # placeholders for the base class's dense MLP (never used)
            for n in ("gate_proj", "up_proj", "down_proj"):
                bf[f"model.layers.{i}.mlp.{n}.weight"] = torch.empty(0)
        super().__init__(dims, bf, **kw)
        self.top_k, self.norm_topk = top_k, norm_topk
        self.moe = [stack_experts(weights, i, num_experts) for i in range(dims.num_hidden_layers)]
        self.router_logits: list[torch.Tensor] = []

    @classmethod
    def from_preset(cls, dims_dict: dict, weights: dict, **kw) -> "Qwen3MoeRef":
        from nanovllm.utils.synthetic import hf_config_dict
        return cls(qwen3_ref.RefDims.from_json(hf_config_dict(dims_dict)), weights, dims_dict["num_experts"],
                   dims_dict["num_experts_per_tok"], dims_dict.get("norm_topk_prob", True), **kw)

    def mlp(self, li: int, h: torch.Tensor) -> torch.Tensor:
        W = self.moe[li]
        logits = F.linear(h, W["gate"])
        self.router_logits.append(logits)
        return moe_block_ref(h, W["gate"], W["gate_up"], W["down"], self.top_k, self.norm_topk,
                             routing=route_ref(logits, self.top_k, self.norm_topk))

    def forward(self, input_ids, positions, ctx, kv_caches):
        d = self.d
        self.router_logits = []
        h = F.embedding(input_ids, self.embed)
        residual = None
        for li, L in enumerate(self.layers):
            if residual is None:
                h, residual = self.rmsnorm(h, L.ln1), h
            else:
                h, residual = self.add_rmsnorm(h, residual, L.ln1)
            qkv = F.linear(h, L.qkv)
            qs, ks = d.num_attention_heads * d.head_dim, d.num_key_value_heads * d.head_dim
            q, k, v = qkv.split([qs, ks, ks], dim=-1)
            q = self.rope(positions, self.rmsnorm(q.reshape(-1, d.num_attention_heads, d.head_dim), L.q_norm))
            k = self.rope(positions, self.rmsnorm(k.reshape(-1, d.num_key_value_heads, d.head_dim), L.k_norm))
            v = v.reshape(-1, d.num_key_value_heads, d.head_dim)
            kc, vc = kv_caches[li] if kv_caches is not None else (None, None)
            o = attention_forward_ref(q, k, v, kc, vc, ctx, self.scale, self.p_dtype)
            h = F.linear(o.reshape(o.shape[0], -1), L.o)
            h, residual = self.add_rmsnorm(h, residual, L.ln2)
            h = self.mlp(li, h)
        h, _ = self.add_rmsnorm(h, residual, self.final_norm)
        return h

    def min_gap_over_ulp(self) -> float:
        """Over every token and layer of the last forward: the smallest logit gap between the k-th and (k+1)-th expert,
        in bf16 ulps of the token's largest |router logit|."""
        worst = math.inf
        for lg in self.router_logits:
            gap = routing_gap(lg, self.top_k)
            ulp = bf16_ulp(lg.double().abs().amax(-1))
            worst = min(worst, (gap / ulp).min().item())
        return worst


def prefill_ctx(lens: list[int]) -> SimpleNamespace:
    """Context of one packed causal prefill of sequences of these lengths, without a cache."""
    cu = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32)
    return SimpleNamespace(is_prefill=True, cu_seqlens_q=cu, cu_seqlens_k=cu, max_seqlen_q=max(lens), max_seqlen_k=max(lens),
                           slot_mapping=None, context_lens=None, block_tables=None)


def gap_safe_sequences(oracle: Qwen3MoeRef, vocab: int, lens: list[int], seed: int, gap_ulps: float) -> list[list[int]]:
    """Token sequences built one token at a time, each drawn until every layer of the oracle routes it with a logit gap of
    at least ``gap_ulps`` bf16 ulps between its k-th and (k+1)-th expert (a token's routing depends only on the tokens
    before it), so that no bf16-level difference between two pipelines can flip one of its selections."""
    rnd = random.Random(seed)
    seqs = []
    for n in lens:
        seq = []
        while len(seq) < n:
            cand = seq + [rnd.randint(2, vocab - 1)]
            oracle.forward(torch.tensor(cand), torch.arange(len(cand)), prefill_ctx([len(cand)]), None)
            if all((routing_gap(lg[-1:], oracle.top_k) / bf16_ulp(lg[-1:].abs().amax(-1))).item() >= gap_ulps
                   for lg in oracle.router_logits):
                seq = cand
        seqs.append(seq)
    return seqs


def tile_table_ref(ids: torch.Tensor, num_experts: int, tile_rows: int = 128) -> tuple[list, list]:
    """What b200_moe_align must produce, up to the order of rows inside a segment: per-expert (first row, count) of the
    permuted buffer, and the tiles (expert, first row, end row)."""
    counts = torch.bincount(ids.reshape(-1).long(), minlength=num_experts).tolist()
    segs, tiles, row = [], [], 0
    for e, c in enumerate(counts):
        segs.append((row, c))
        for r in range(0, c, tile_rows):
            tiles.append((e, row + r, row + min(r + tile_rows, c)))
        row += c
    return segs, tiles
