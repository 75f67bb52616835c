"""Block-FP8 checkpoints without a GPU: the quantization_config switch and its refusals, the shape rule, the reference
quantizers against hand-computed values, the C entry points' argument checks, and the tensor-parallel sharding of
weights and scales (DESIGN.md 3.6)."""
import json
import os
from types import SimpleNamespace

import pytest
import torch

from nanovllm import _native as nat
from nanovllm.models.qwen3 import Qwen3ForCausalLM
from nanovllm.utils import fp8 as fp8fmt
from nanovllm.utils.loader import load_model
from nanovllm.utils.synthetic import PRESETS, hf_config_dict, make_model_dir, quantize_checkpoint, random_weights
from fp8_ref import quant_act_ref

EINVAL, EUNSUPPORTED = -1, -2


def _hf(preset="tiny", quant=None):
    cfg = hf_config_dict(PRESETS[preset])
    if quant is not None:
        cfg["quantization_config"] = quant
    return SimpleNamespace(**cfg)


def _qc(**over):
    q = fp8fmt.quantization_config_dict()
    q.update(over)
    return q


# ---- the switch -------------------------------------------------------------------------------------------------------
def test_quantization_config_accepted():
    assert fp8fmt.is_block_fp8(_hf(quant=_qc())) is True
    assert fp8fmt.is_block_fp8(_hf()) is False
    qwen_style = {"activation_scheme": "dynamic", "modules_to_not_convert": None, "fmt": "e4m3",
                  "quant_method": "fp8", "weight_block_size": [128, 128]}
    assert fp8fmt.is_block_fp8(_hf(quant=qwen_style)) is True


@pytest.mark.parametrize("over", [
    dict(activation_scheme="static"), dict(weight_block_size=[64, 64]), dict(weight_block_size=[128, 64]),
    dict(weight_block_size=None), dict(quant_method="gptq"), dict(quant_method="awq"), dict(quant_method="compressed-tensors"),
    dict(fmt="e5m2"),
])
def test_unsupported_quantization_refused_before_weights(over):
    with pytest.raises(NotImplementedError):
        fp8fmt.is_block_fp8(_hf(quant=_qc(**over)))
    with pytest.raises(NotImplementedError):
        Qwen3ForCausalLM(_hf(quant=_qc(**over)), 0, 1, device="cpu", max_position=64)


@pytest.mark.parametrize("preset", ["tiny-g1", "tiny-g8"])
def test_ragged_shapes_refused(preset):
    with pytest.raises(NotImplementedError, match="multiple of 128"):
        Qwen3ForCausalLM(_hf(preset, _qc()), 0, 1, device="cpu", max_position=64)


@pytest.mark.parametrize("preset", ["qwen3-0.6b", "qwen3-8b", "qwen3-32b", "tiny", "tiny-g4"])
def test_public_sizes_pass_the_shape_rule(preset):
    d = PRESETS[preset]
    tps = (1, 2) if preset.startswith("tiny") else (1, 2, 4, 8)
    for tp in tps:
        if d["num_key_value_heads"] % tp:
            continue
        fp8fmt.check_shapes(d["num_attention_heads"] // tp * d["head_dim"], d["num_key_value_heads"] // tp * d["head_dim"],
                            d["hidden_size"], d["intermediate_size"] // tp)


def test_tensor_parallel_shape_rule():
    with pytest.raises(NotImplementedError):           # an intermediate of 768 over 4 ranks is 192 per rank
        fp8fmt.check_shapes(4 * 128, 128, 256, 768 // 4)


# ---- reference quantizers against hand-computed values -------------------------------------------------------------------
def test_activation_quantizer_hand_values():
    x = torch.zeros(3, 256, dtype=torch.bfloat16)
    x[0, 0], x[0, 1], x[0, 2], x[0, 3] = 1.0, -1.0, 0.5, 0.30078125      # amax 1 -> s = 1/448
    x[0, 128], x[0, 129] = -2.0, 1.0                                     # second group: amax 2 -> s = 2/448
    x[2, :] = 3.0                                                        # row 1 all zero (amax 0)
    q, s = quant_act_ref(x)
    f = q.float()
    assert s.dtype == torch.float32 and s.shape == (3, 2)
    assert s[0, 0].item() == pytest.approx(1.0 / 448, rel=1e-7)
    assert (f[0, 0].item(), f[0, 1].item(), f[0, 2].item()) == (448.0, -448.0, 224.0)    # saturation at +-448 exactly
    assert f[0, 3].item() == 128.0                                       # 134.75 rounds to the e4m3 neighbour 128
    assert f[0, 128].item() == -448.0 and f[0, 129].item() == 224.0
    assert s[1].tolist() == [pytest.approx(1e-10 / 448)] * 2 and (f[1] == 0).all()      # amax = 0: floor, zeros
    assert (f[2] == 448.0).all() and s[2, 0].item() == pytest.approx(3.0 / 448, rel=1e-7)


def test_weight_quantizer_hand_values():
    w = torch.zeros(256, 128, dtype=torch.bfloat16)
    w[0, 0], w[5, 7], w[127, 127] = 0.25, -0.125, 0.0625       # block (0, 0): amax 0.25
    w[200, 3] = -4.0                                            # block (1, 0): amax 4
    q, s = fp8fmt.quantize_weight(w)
    assert q.dtype == torch.float8_e4m3fn and s.shape == (2, 1)
    assert s[0, 0].item() == pytest.approx(0.25 / 448, rel=1e-7) and s[1, 0].item() == pytest.approx(4.0 / 448, rel=1e-7)
    f = q.float()
    assert (f[0, 0].item(), f[5, 7].item(), f[127, 127].item(), f[200, 3].item()) == (448.0, -224.0, 112.0, -448.0)
    z, sz = fp8fmt.quantize_weight(torch.zeros(128, 128))
    assert (z.float() == 0).all() and torch.isfinite(sz).all()
    assert torch.allclose(fp8fmt.dequantize_weight(q, s), w.float())


def test_dequantized_checkpoint_is_close_to_bf16():
    ws = random_weights(PRESETS["tiny"], seed=5)
    qs = quantize_checkpoint(ws)
    name = "model.layers.0.mlp.down_proj.weight"
    d = fp8fmt.dequantize_weight(qs[name], qs[name + "_scale_inv"])
    rel = ((d - ws[name].float()).norm() / ws[name].float().norm()).item()
    assert rel < 0.04                                     # e4m3 keeps 3 mantissa bits: about 2^-5 relative
    assert "model.layers.0.input_layernorm.weight" in qs and qs["model.embed_tokens.weight"].dtype == torch.bfloat16


# ---- C entry points: argument checks need no GPU ------------------------------------------------------------------------
def test_quant_entry_point_refuses_bad_arguments():
    lib = nat.load()
    P = 1 << 20                                            # a well-aligned non-null address: never dereferenced here
    ok = dict(x=P, xs=256, q=P, qs=256, s=P, ss=2, rows=4, k=256)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.b200_quant_fp8(a["x"], a["xs"], a["q"], a["qs"], a["s"], a["ss"], a["rows"], a["k"], None)
    assert call(x=None) == EINVAL and call(q=None) == EINVAL and call(s=None) == EINVAL
    assert call(rows=-1) == EINVAL and call(k=0) == EINVAL
    assert call(k=192, xs=192, qs=192) == EUNSUPPORTED
    assert call(ss=1) == EINVAL and call(xs=128) == EINVAL and call(x=P + 2) == EINVAL
    assert call(rows=0) == 0


def test_linear_fp8_entry_point_refuses_bad_arguments():
    lib = nat.load()
    P = 1 << 20
    ok = dict(x=P, xs=256, xsc=P, xscs=2, w=P, wsc=P, out=P, os=256, rows=4, n=256, k=256, epi=0, bn=64, splits=1)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.b200_linear_fp8(a["x"], a["xs"], a["xsc"], a["xscs"], a["w"], a["wsc"], a["out"], a["os"], a["rows"],
                                   a["n"], a["k"], a["epi"], a["bn"], a["splits"], 0, None)
    for null in ("x", "xsc", "w", "wsc", "out"):
        assert call(**{null: None}) == EINVAL, null
    assert call(k=192, xs=192) == EUNSUPPORTED                       # k % 128
    assert call(n=192) == EUNSUPPORTED                               # whole 128-row scale blocks of W
    assert call(bn=128) == EUNSUPPORTED and call(bn=48) == EUNSUPPORTED
    assert call(epi=1, bn=16) == EUNSUPPORTED
    assert call(xscs=1) == EINVAL                                    # x scales narrower than k / 128
    assert call(splits=3, epi=2) == EUNSUPPORTED and call(splits=2, epi=0) == EINVAL
    assert call(epi=3) == EINVAL and call(xs=8) == EINVAL and call(x=P + 8) == EINVAL and call(w=P + 4) == EINVAL
    assert call(rows=0) == 0


# ---- loading and tensor-parallel sharding on CPU -----------------------------------------------------------------------
def _load(preset, rank, world, weights):
    m = Qwen3ForCausalLM(_hf(preset, _qc()), rank, world, device="cpu", max_position=64)
    for name, w in weights.items():
        m.load_hf_tensor(name, w)
    return m


@pytest.mark.parametrize("scale_dtype", [torch.float32, torch.bfloat16])
def test_sharding_matches_slices_of_the_dequantized_tensor(scale_dtype):
    preset = "tiny-g4"          # tp 2: q 512, kv 128, intermediate 384 per rank
    full = quantize_checkpoint(random_weights(PRESETS[preset], seed=11), scale_dtype)
    deq = lambda n: fp8fmt.dequantize_weight(full[n + ".weight"], full[n + ".weight_scale_inv"].float())
    p = "model.layers.1."
    for rank in range(2):
        m = _load(preset, rank, 2, full)
        L = m.layers[1]
        part = lambda n, dim: deq(p + n).chunk(2, dim)[rank]
        want_qkv = torch.cat([part("self_attn.q_proj", 0), part("self_attn.k_proj", 0), part("self_attn.v_proj", 0)])
        assert torch.equal(fp8fmt.dequantize_weight(L.qkv, L.qkv_s), want_qkv)
        assert torch.equal(fp8fmt.dequantize_weight(L.o, L.o_s), part("self_attn.o_proj", 1))
        assert torch.equal(fp8fmt.dequantize_weight(L.gate_up, L.gate_up_s), torch.cat([part("mlp.gate_proj", 0), part("mlp.up_proj", 0)]))
        assert torch.equal(fp8fmt.dequantize_weight(L.down, L.down_s), part("mlp.down_proj", 1))
        assert m.embed.dtype == torch.bfloat16 and L.ln1.dtype == torch.bfloat16


def test_mismatched_checkpoints_refused():
    bf = random_weights(PRESETS["tiny"], seed=1)
    q = quantize_checkpoint(bf)
    name = "model.layers.0.self_attn.q_proj.weight"
    with pytest.raises(NotImplementedError):              # scales in a checkpoint without the fp8 config
        Qwen3ForCausalLM(_hf("tiny"), 0, 1, device="cpu", max_position=64).load_hf_tensor(name + "_scale_inv", q[name + "_scale_inv"])
    with pytest.raises(NotImplementedError):              # e4m3 weights without the fp8 config
        Qwen3ForCausalLM(_hf("tiny"), 0, 1, device="cpu", max_position=64).load_hf_tensor(name, q[name])
    with pytest.raises(NotImplementedError):              # a bf16 projection under the fp8 config
        Qwen3ForCausalLM(_hf("tiny", _qc()), 0, 1, device="cpu", max_position=64).load_hf_tensor(name, bf[name])


def test_fp8_model_dir_and_random_init(tmp_path):
    d = make_model_dir(str(tmp_path / "fp8"), "tiny", seed=3, fp8=True, tokenizer=False)
    cfg = json.load(open(os.path.join(d, "config.json")))
    assert cfg["quantization_config"] == fp8fmt.quantization_config_dict()
    from safetensors import safe_open
    with safe_open(os.path.join(d, "model.safetensors"), "pt", "cpu") as f:
        assert f.get_tensor("model.layers.0.mlp.up_proj.weight").dtype == torch.float8_e4m3fn
        assert f.get_tensor("model.layers.0.mlp.up_proj.weight_scale_inv").shape == (512 // 128, 256 // 128)
    loaded = Qwen3ForCausalLM(_hf("tiny", _qc()), 0, 1, device="cpu", max_position=64)
    load_model(loaded, d)
    # a directory without weights: the same bf16 draws, block-quantized
    rnd = Qwen3ForCausalLM(_hf("tiny", _qc()), 0, 1, device="cpu", max_position=64)
    load_model(rnd, str(tmp_path), allow_random=True, seed=3)
    for a, b in ((loaded, rnd),):
        for La, Lb in zip(a.layers, b.layers):
            assert torch.equal(La.gate_up.view(torch.uint8), Lb.gate_up.view(torch.uint8)) and torch.equal(La.gate_up_s, Lb.gate_up_s)
            assert torch.equal(La.qkv.view(torch.uint8), Lb.qkv.view(torch.uint8)) and torch.equal(La.down_s, Lb.down_s)
    bf_dir = make_model_dir(str(tmp_path / "bf"), "tiny", seed=3, tokenizer=False)
    assert "quantization_config" not in json.load(open(os.path.join(bf_dir, "config.json")))


def test_fp8_disables_the_bf16_experiments(monkeypatch):
    monkeypatch.setenv("B200_TAIL", "mega")
    monkeypatch.setenv("B200_DUAL", "1")
    monkeypatch.setenv("B200_LINEAR", "tc")
    m = Qwen3ForCausalLM(_hf("tiny", _qc()), 0, 1, device="cpu", max_position=64)
    assert not (m.mega_tail or m.dual or m.tc_linear or m.tc_gate_up)
    b = Qwen3ForCausalLM(_hf("tiny"), 0, 1, device="cpu", max_position=64)
    assert b.mega_tail and b.tc_linear and not b.fp8
