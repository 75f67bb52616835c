"""Block-scaled FP8 checkpoints (the "fp8" ``quantization_config`` of Qwen3-*-FP8 and DeepSeek-V3; DESIGN.md 3.6).

Projection weights (q/k/v/o/gate/up/down) are e4m3 ``[N, K]`` with one fp32 scale per 128 x 128 block,
``weight_scale_inv [N / 128, K / 128]`` (the weight is ``q * s``: despite the name the scale multiplies), and
activations are quantized on the fly per token and 128 columns.  Embedding, LM head and norms stay bf16.
"""
from __future__ import annotations

import torch

BLOCK = 128
E4M3_MAX = 448.0
# the amax floor of a block before the division, so that an all-zero block gets a finite scale (its elements stay 0)
AMAX_FLOOR = 1e-10

PROJECTIONS = ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj",
               "mlp.gate_proj", "mlp.up_proj", "mlp.down_proj")


def quantization_config_dict() -> dict:
    """The quantization_config Qwen's FP8 checkpoints carry in config.json."""
    return {"quant_method": "fp8", "fmt": "e4m3", "weight_block_size": [BLOCK, BLOCK], "activation_scheme": "dynamic"}


def is_block_fp8(hf_config) -> bool:
    """True for the block-FP8 format above, False without a quantization_config; NotImplementedError for any other
    quantization (static activation scales, other block sizes, other methods), before any weight is touched."""
    q = getattr(hf_config, "quantization_config", None)
    if q is None:
        return False
    if not isinstance(q, dict):
        q = q.to_dict() if hasattr(q, "to_dict") else vars(q)
    method = q.get("quant_method")
    if method != "fp8":
        raise NotImplementedError(f"quantization_config quant_method {method!r}: only block-scaled 'fp8' is supported")
    if list(q.get("weight_block_size") or []) != [BLOCK, BLOCK]:
        raise NotImplementedError(f"fp8 weight_block_size {q.get('weight_block_size')!r}: only [128, 128] is supported")
    if q.get("activation_scheme", "dynamic") != "dynamic":
        raise NotImplementedError(f"fp8 activation_scheme {q.get('activation_scheme')!r}: only 'dynamic' is supported")
    if q.get("fmt", "e4m3") != "e4m3":
        raise NotImplementedError(f"fp8 fmt {q.get('fmt')!r}: only 'e4m3' is supported")
    return True


def check_shapes(q_size: int, kv_size: int, hidden: int, inter: int) -> None:
    """Every projection dimension of one tensor-parallel rank must be whole 128-blocks (sharding cuts at block edges)."""
    dims = dict(q_size=q_size, kv_size=kv_size, hidden=hidden, intermediate=inter)
    bad = {k: v for k, v in dims.items() if v % BLOCK}
    if bad:
        raise NotImplementedError(f"block-FP8 weights need every per-rank projection dimension to be a multiple of {BLOCK}: {bad}")


def quantize_weight(w: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """[N, K] -> (e4m3 [N, K], fp32 scales [N / 128, K / 128]): s = max(amax, 1e-10) / 448 per block, q = e4m3_rn(w / s).
    Runs where ``w`` lives (the device for random init)."""
    n, k = w.shape
    assert n % BLOCK == 0 and k % BLOCK == 0, (n, k)
    wf = w.float().view(n // BLOCK, BLOCK, k // BLOCK, BLOCK)
    amax = wf.abs().amax(dim=(1, 3))
    s = torch.div(amax.clamp_min(AMAX_FLOOR), torch.full_like(amax, E4M3_MAX))
    q = torch.div(wf, s[:, None, :, None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q.view(n, k), s


def dequantize_weight(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """fp32 [N, K] = float(q) * s of its block."""
    n, k = q.shape
    return (q.float().view(n // BLOCK, BLOCK, k // BLOCK, BLOCK) * s.float()[:, None, :, None]).view(n, k)
