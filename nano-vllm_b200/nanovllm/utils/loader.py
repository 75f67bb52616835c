"""Checkpoint loading (reference nanovllm/utils/loader.py:12-28): every ``*.safetensors`` tensor in the
model directory is handed to the model, which slices its own tensor-parallel shard.

Unlike the reference, a directory without weights is an error unless ``allow_random`` is set, in
which case the model is filled from a seeded generator (the reference would silently run on
``torch.empty`` garbage, SURVEY.md S4).
"""
from __future__ import annotations

import os
from glob import glob

import torch


def load_model(model, path: str, allow_random: bool = False, seed: int = 0) -> int:
    files = sorted(glob(os.path.join(path, "*.safetensors")))
    if not files:
        if not allow_random:
            raise FileNotFoundError(f"no *.safetensors under {path}")
        return _random_fill(model, seed)
    from safetensors import safe_open
    n = 0
    for file in files:
        with safe_open(file, "pt", "cpu") as f:
            for name in f.keys():
                model.load_hf_tensor(name, f.get_tensor(name))
                n += 1
    return n


def _random_fill(model, seed: int, init_std: float = 0.02) -> int:
    """Seeded random weights for a directory that has none (benchmarks at 8B / 32B dimensions: no checkpoint exists
    offline).  On a CUDA model every tensor is drawn ON THE DEVICE from a generator keyed by (seed, parameter name) at
    its FULL shape and handed to ``load_hf_tensor``, which slices this rank's shard -- so all tensor-parallel ranks hold
    shards of one well-defined model without 64 GB of host memory or a broadcast.  On a CPU model the values are
    ``synthetic.random_weights`` (what the tests compare against).

    A block-FP8 model (its config's quantization_config) gets the same bf16 draws, each projection block-quantized
    (``fp8.quantize_weight``) into its e4m3 weight and ``weight_scale_inv``: the quantized version of the bf16 model of the
    same seed.  A mixture-of-experts model gets the Hub's per-expert names (synthetic.weight_shapes), so its experts are
    stacked by the same ``load_hf_tensor`` that reads a checkpoint."""
    from .synthetic import quantize_checkpoint, random_weights, weight_shapes, weight_std
    c = model.cfg
    dims = dict(hidden_size=c.hidden_size, num_hidden_layers=c.num_hidden_layers,
                num_attention_heads=c.num_attention_heads, num_key_value_heads=c.num_key_value_heads,
                head_dim=model.head_dim, intermediate_size=c.intermediate_size, vocab_size=c.vocab_size,
                tie_word_embeddings=model.tie)
    if getattr(model, "num_experts", 0):
        dims.update(num_experts=c.num_experts, num_experts_per_tok=c.num_experts_per_tok,
                    moe_intermediate_size=c.moe_intermediate_size, norm_topk_prob=model.norm_topk)
    if model.device.type != "cuda":
        ws = random_weights(dims, seed)
        if model.fp8:
            ws = quantize_checkpoint(ws)
        for name, w in ws.items():
            model.load_hf_tensor(name, w)
        return len(ws)
    import zlib
    from .fp8 import quantize_weight
    from .synthetic import is_projection
    gen = torch.Generator(device=model.device)
    shapes = weight_shapes(dims)
    for name, shape in shapes.items():
        gen.manual_seed((seed << 32) ^ zlib.crc32(name.encode()))
        w = torch.randn(shape, generator=gen, device=model.device, dtype=torch.float32)
        w = (1.0 + 0.1 * w) if len(shape) == 1 else weight_std(name, shape, init_std) * w
        w = w.to(torch.bfloat16)
        if model.fp8 and is_projection(name):
            q, s = quantize_weight(w)
            model.load_hf_tensor(name + "_scale_inv", s)
            w = q
        model.load_hf_tensor(name, w)
        del w
    return len(shapes)
