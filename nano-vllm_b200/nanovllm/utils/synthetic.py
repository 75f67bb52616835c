"""Random-init Qwen3 checkpoints for benchmarking and tests (no network, no real weights here).

Writes what ``Config`` / ``LLMEngine`` / the loader read from a model directory (the same three
things the reference reads, SURVEY.md appendix A): ``config.json``, a WordLevel ``tokenizer.json``
covering the whole vocabulary, and ``model.safetensors`` with HF parameter names.  Weights are
N(0, init_std) from a seeded CPU generator, norm weights 1 + 0.1 N(0, 1); the same file is loaded
by the product, by the CPU oracle and (when present) by the reference itself, so all three see
identical bytes.
"""
from __future__ import annotations

import json
import os

import torch

PRESETS = {
    # public HF configs (dims only)
    "qwen3-0.6b": dict(hidden_size=1024, num_hidden_layers=28, num_attention_heads=16, num_key_value_heads=8,
                       head_dim=128, intermediate_size=3072, vocab_size=151936, tie_word_embeddings=True),
    "qwen3-8b": dict(hidden_size=4096, num_hidden_layers=36, num_attention_heads=32, num_key_value_heads=8,
                     head_dim=128, intermediate_size=12288, vocab_size=151936, tie_word_embeddings=False),
    "qwen3-32b": dict(hidden_size=5120, num_hidden_layers=64, num_attention_heads=64, num_key_value_heads=8,
                      head_dim=128, intermediate_size=25600, vocab_size=151936, tie_word_embeddings=False),
    # small shapes for parity tests
    "tiny": dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
                 head_dim=128, intermediate_size=512, vocab_size=2048, tie_word_embeddings=True),
    "tiny-g4": dict(hidden_size=256, num_hidden_layers=3, num_attention_heads=8, num_key_value_heads=2,
                    head_dim=128, intermediate_size=768, vocab_size=4096, tie_word_embeddings=False),
    "tiny-g1": dict(hidden_size=192, num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=2,
                    head_dim=128, intermediate_size=320, vocab_size=1024, tie_word_embeddings=True),
    "tiny-g8": dict(hidden_size=320, num_hidden_layers=2, num_attention_heads=8, num_key_value_heads=1,
                    head_dim=128, intermediate_size=448, vocab_size=3072, tie_word_embeddings=False),
    # mixture of experts (model_type "qwen3_moe"): intermediate_size is the config's dense-MLP size, unused when every
    # layer is sparse; the experts' MLPs are moe_intermediate_size wide
    "qwen3-30b-a3b": dict(hidden_size=2048, num_hidden_layers=48, num_attention_heads=32, num_key_value_heads=4,
                          head_dim=128, intermediate_size=6144, vocab_size=151936, tie_word_embeddings=False,
                          num_experts=128, num_experts_per_tok=8, moe_intermediate_size=768, norm_topk_prob=True),
    "tiny-moe": dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
                     head_dim=128, intermediate_size=512, vocab_size=2048, tie_word_embeddings=True,
                     num_experts=16, num_experts_per_tok=4, moe_intermediate_size=128, norm_topk_prob=True),
    # head group 8 (the wide-group decode kernel 30B-A3B runs on), 8 of 32 experts, weights not renormalised
    "tiny-moe-g8": dict(hidden_size=320, num_hidden_layers=2, num_attention_heads=8, num_key_value_heads=1,
                        head_dim=128, intermediate_size=448, vocab_size=3072, tie_word_embeddings=False,
                        num_experts=32, num_experts_per_tok=8, moe_intermediate_size=192, norm_topk_prob=False),
}
# Router weights are drawn with std ROUTER_LOGIT_STD / sqrt(hidden), so that router logits have a spread of about
# ROUTER_LOGIT_STD: with the projections' 0.02 the logits of a small model would all sit within a few bf16 ulps of each
# other and the routing would be decided by rounding noise.
ROUTER_LOGIT_STD = 2.0


def is_moe(dims: dict) -> bool:
    return bool(dims.get("num_experts"))


def hf_config_dict(dims: dict) -> dict:
    cfg = dict(architectures=["Qwen3ForCausalLM"], model_type="qwen3", max_position_embeddings=40960,
               rms_norm_eps=1e-6, rope_theta=1000000, hidden_act="silu", attention_bias=False,
               torch_dtype="bfloat16", bos_token_id=0, eos_token_id=1)
    if is_moe(dims):
        cfg.update(architectures=["Qwen3MoeForCausalLM"], model_type="qwen3_moe", decoder_sparse_step=1, mlp_only_layers=[],
                   norm_topk_prob=True)
    cfg.update(dims)
    return cfg


def weight_shapes(d: dict) -> dict[str, tuple]:
    H, D = d["hidden_size"], d["head_dim"]
    hq, hkv, I, V = d["num_attention_heads"], d["num_key_value_heads"], d["intermediate_size"], d["vocab_size"]
    shapes = {"model.embed_tokens.weight": (V, H), "model.norm.weight": (H,)}
    if not d.get("tie_word_embeddings", False):
        shapes["lm_head.weight"] = (V, H)
    for i in range(d["num_hidden_layers"]):
        p = f"model.layers.{i}."
        shapes.update({
            p + "self_attn.q_proj.weight": (hq * D, H), p + "self_attn.k_proj.weight": (hkv * D, H),
            p + "self_attn.v_proj.weight": (hkv * D, H), p + "self_attn.o_proj.weight": (H, hq * D),
            p + "self_attn.q_norm.weight": (D,), p + "self_attn.k_norm.weight": (D,)})
        if is_moe(d):                   # the Hub's per-expert names (Qwen3MoeSparseMoeBlock)
            E, Ie = d["num_experts"], d["moe_intermediate_size"]
            shapes[p + "mlp.gate.weight"] = (E, H)
            for e in range(E):
                q = f"{p}mlp.experts.{e}."
                shapes.update({q + "gate_proj.weight": (Ie, H), q + "up_proj.weight": (Ie, H), q + "down_proj.weight": (H, Ie)})
        else:                           # (this order is the order of random_weights' draws)
            shapes.update({p + "mlp.gate_proj.weight": (I, H), p + "mlp.up_proj.weight": (I, H), p + "mlp.down_proj.weight": (H, I)})
        shapes.update({p + "input_layernorm.weight": (H,), p + "post_attention_layernorm.weight": (H,)})
    return shapes


def weight_std(name: str, shape: tuple, init_std: float = 0.02) -> float:
    """Standard deviation of a matrix's random draw: ROUTER_LOGIT_STD / sqrt(hidden) for a MoE router, else init_std."""
    return ROUTER_LOGIT_STD / shape[1] ** 0.5 if name.endswith(".mlp.gate.weight") else init_std


def random_weights(dims: dict, seed: int = 0, init_std: float = 0.02) -> dict[str, torch.Tensor]:
    gen = torch.Generator(device="cpu").manual_seed(seed)
    out = {}
    for name, shape in weight_shapes(dims).items():
        if len(shape) == 1:
            w = 1.0 + 0.1 * torch.randn(shape, generator=gen)
        else:
            w = weight_std(name, shape, init_std) * torch.randn(shape, generator=gen)
        out[name] = w.to(torch.bfloat16)
    return out


def is_projection(name: str) -> bool:
    """A q/k/v/o/gate/up/down weight: what a block-FP8 checkpoint stores as e4m3 with a weight_scale_inv."""
    from .fp8 import PROJECTIONS
    return name.endswith(".weight") and name.split(".")[-2] in {p.split(".")[-1] for p in PROJECTIONS}


def quantize_checkpoint(weights: dict[str, torch.Tensor], scale_dtype=torch.float32) -> dict[str, torch.Tensor]:
    """A bf16 checkpoint in Qwen's block-FP8 layout: every projection becomes e4m3 ``<name>`` plus ``<name>_scale_inv``
    (fp8.quantize_weight); everything else is kept as it is."""
    from .fp8 import quantize_weight
    out = {}
    for name, w in weights.items():
        if is_projection(name):
            q, s = quantize_weight(w)
            out[name], out[name + "_scale_inv"] = q, s.to(scale_dtype)
        else:
            out[name] = w
    return out


def write_tokenizer(path: str, vocab_size: int, eos_id: int = 1) -> None:
    vocab = {f"t{i}": i for i in range(vocab_size)}
    vocab[f"t{eos_id}"] = eos_id
    tok = {
        "version": "1.0", "truncation": None, "padding": None, "added_tokens": [], "normalizer": None,
        "pre_tokenizer": {"type": "Whitespace"}, "post_processor": None, "decoder": None,
        "model": {"type": "WordLevel", "vocab": vocab, "unk_token": "t0"},
    }
    with open(os.path.join(path, "tokenizer.json"), "w") as f:
        json.dump(tok, f)
    with open(os.path.join(path, "tokenizer_config.json"), "w") as f:
        json.dump({"tokenizer_class": "PreTrainedTokenizerFast", "eos_token": f"t{eos_id}", "unk_token": "t0"}, f)


def make_model_dir(path: str, preset: str | dict = "qwen3-0.6b", seed: int = 0, init_std: float = 0.02,
                   weights: bool = True, tokenizer: bool = True, fp8: bool = False) -> str:
    """Create (idempotently) a loadable model directory; returns ``path``.  ``fp8``: a block-FP8 checkpoint in Qwen's
    format (its quantization_config in config.json; the weights, if written, are the bf16 draws of the same seed
    block-quantized, see ``quantize_checkpoint``)."""
    dims = dict(PRESETS[preset]) if isinstance(preset, str) else dict(preset)
    os.makedirs(path, exist_ok=True)
    stamp = os.path.join(path, ".synthetic.json")
    want = dict(dims=dims, seed=seed, init_std=init_std, weights=weights, tokenizer=tokenizer, v=2)
    if fp8:
        if is_moe(dims):
            raise NotImplementedError("FP8 mixture-of-experts checkpoints are not supported")
        want["fp8"] = True
    if os.path.exists(stamp):
        with open(stamp) as f:
            if json.load(f) == want:
                return path
    cfg = hf_config_dict(dims)
    if fp8:
        from .fp8 import quantization_config_dict
        cfg["quantization_config"] = quantization_config_dict()
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(cfg, f, indent=1)
    if tokenizer:
        write_tokenizer(path, dims["vocab_size"])
    if weights:
        from safetensors.torch import save_file
        ws = random_weights(dims, seed, init_std)
        save_file(quantize_checkpoint(ws) if fp8 else ws, os.path.join(path, "model.safetensors"))
    with open(stamp, "w") as f:
        json.dump(want, f)
    return path
