"""Reference of the block-FP8 projections (DESIGN.md 3.6), restated in torch.

* activation quantization: per row and 128-column group, s = max(amax, 1e-10) / 448 (fp32 division) and
  q = e4m3_satfinite_rn(x / s) (fp32 division; e4m3 as tests/kv_fp8_ref.py: clamp to +-448, then round to nearest even);
* the GEMM, in float64 on the dequantized operands: y[m, n] = sum_kb s_x[m, kb] s_w[n / 128, kb] sum_{k in kb} q_x q_w;
* the error bar of the kernel's result against that, per element:
    bf16 output rounding  2^-8 |y|   (half an ulp is 2^-9 relative; twice that for the scale product's fp32 roundings)
  + in-block accumulation 2^-11 A,   A = sum_k |x_deq[m, k] w_deq[n, k]|
  fp8 wgmma sums the 32 products of one instruction, and chains the four instructions of a block, with fewer mantissa
  bits than fp32: errors up to 1.08 x 2^-12 A were measured on the H100, hence 2^-11.  The fp32 promotion across
  blocks adds about (k / 128) 2^-24 A, which the second term also covers.
``Qwen3RefFp8W`` is oracle.qwen3_ref's forward with its four projections replaced by that quantize + GEMM.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import qwen3_ref
from oracle.paged_attention_ref import attention_forward_ref
from kv_fp8_ref import E4M3_MAX

BLOCK = 128
ACC_REL = 2.0 ** -11
OUT_REL = 2.0 ** -8


def quant_act_ref(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """x [rows, k] -> (float8_e4m3fn [rows, k], fp32 [rows, k / 128])."""
    rows, k = x.shape
    xf = x.float().reshape(rows, k // BLOCK, BLOCK)
    amax = xf.abs().amax(-1)
    s = torch.div(amax.clamp_min(1e-10), torch.full_like(amax, E4M3_MAX))
    q = torch.div(xf, s[..., None].expand_as(xf)).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q.reshape(rows, k), s


def dequant(q: torch.Tensor, s: torch.Tensor, block_rows: int) -> torch.Tensor:
    """float64 q * s, with s [rows / block_rows, k / 128]."""
    n, k = q.shape
    d = q.view(torch.float8_e4m3fn).double().reshape(n // block_rows, block_rows, k // BLOCK, BLOCK)
    return (d * s.double()[:, None, :, None]).reshape(n, k)


def gemm_ref(xq, xs, wq, ws):
    """(y, A): float64 y = x_deq w_deq^T and the absolute product sum A of the bar."""
    xd, wd = dequant(xq, xs, 1), dequant(wq, ws, BLOCK)
    return xd @ wd.t(), xd.abs() @ wd.abs().t()


def bar(y, a, rounded: bool = True):
    return (OUT_REL * y.abs() if rounded else 2.0 ** -20 * y.abs()) + ACC_REL * a


def fp8_linear_ref(x: torch.Tensor, wq: torch.Tensor, ws: torch.Tensor) -> torch.Tensor:
    """What a block-FP8 projection computes, rounded to bf16 as F.linear's output is."""
    xq, xs = quant_act_ref(x)
    y, _ = gemm_ref(xq, xs, wq, ws)
    return y.to(torch.bfloat16)


class Qwen3RefFp8W(qwen3_ref.Qwen3Ref):
    """The fp32 oracle on a block-FP8 checkpoint: projections quantize their input at the points the engine does and
    multiply the dequantized operands in float64.  ``weights`` holds e4m3 projections plus their ``*_scale_inv``."""

    def __init__(self, dims, weights: dict, **kw):
        bf = {n: w for n, w in weights.items() if w.dtype != torch.float8_e4m3fn and not n.endswith("_scale_inv")}
        for n, w in weights.items():           # placeholders of the right shape for the base class (never used)
            if w.dtype == torch.float8_e4m3fn:
                bf[n] = torch.empty(0)
        super().__init__(dims, bf, **kw)
        self.fp8 = []
        for i in range(dims.num_hidden_layers):
            p = f"model.layers.{i}."
            cat = lambda *names: (torch.cat([weights[p + n + ".weight"] for n in names], 0),
                                  torch.cat([weights[p + n + ".weight_scale_inv"].float() for n in names], 0))
            self.fp8.append(dict(qkv=cat("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj"),
                                 o=cat("self_attn.o_proj"), gate_up=cat("mlp.gate_proj", "mlp.up_proj"),
                                 down=cat("mlp.down_proj")))

    def forward(self, input_ids, positions, ctx, kv_caches):
        d = self.d
        lin = lambda h, wq: fp8_linear_ref(h, *wq)
        h = F.embedding(input_ids, self.embed)
        residual = None
        for li, L in enumerate(self.layers):
            W = self.fp8[li]
            if residual is None:
                h, residual = self.rmsnorm(h, L.ln1), h
            else:
                h, residual = self.add_rmsnorm(h, residual, L.ln1)
            qkv = lin(h, W["qkv"])
            qs, ks = d.num_attention_heads * d.head_dim, d.num_key_value_heads * d.head_dim
            q, k, v = qkv.split([qs, ks, ks], dim=-1)
            q = self.rope(positions, self.rmsnorm(q.reshape(-1, d.num_attention_heads, d.head_dim), L.q_norm))
            k = self.rope(positions, self.rmsnorm(k.reshape(-1, d.num_key_value_heads, d.head_dim), L.k_norm))
            v = v.reshape(-1, d.num_key_value_heads, d.head_dim)
            kc, vc = kv_caches[li] if kv_caches is not None else (None, None)
            o = attention_forward_ref(q, k, v, kc, vc, ctx, self.scale, self.p_dtype)
            h = lin(o.reshape(o.shape[0], -1), W["o"])
            h, residual = self.add_rmsnorm(h, residual, L.ln2)
            h = lin(self.silu_mul(lin(h, W["gate_up"])), W["down"])
        h, _ = self.add_rmsnorm(h, residual, self.final_norm)
        return h
