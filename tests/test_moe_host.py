"""Qwen3 mixture-of-experts checkpoints without a GPU (DESIGN.md 3.7): the config refusals, the synthetic presets and model
directories, the loader's stacking and tensor-parallel slicing of per-expert tensors, the C entry points' argument checks,
the tile table reference, and tests/moe_ref.py's block against HF transformers' Qwen3MoeSparseMoeBlock in float64."""
import ctypes
import json
import os
from types import SimpleNamespace

import pytest
import torch

from nanovllm import _native as nat
from nanovllm.models.qwen3 import Qwen3ForCausalLM
from nanovllm.models.qwen3_moe import Qwen3MoeForCausalLM, model_class
from nanovllm.utils.loader import load_model
from nanovllm.utils.synthetic import PRESETS, hf_config_dict, make_model_dir, random_weights, weight_shapes
from moe_ref import moe_block_ref, route_ref, stack_experts, tile_table_ref

EINVAL, EUNSUPPORTED, EWORKSPACE = -1, -2, -5


def _hf(preset="tiny-moe", **over):
    cfg = hf_config_dict(PRESETS[preset])
    cfg.update(over)
    return SimpleNamespace(**cfg)


# ---- config ------------------------------------------------------------------------------------------------------------
def test_model_type_selects_the_class():
    assert model_class(_hf()) is Qwen3MoeForCausalLM
    assert model_class(_hf("tiny")) is Qwen3ForCausalLM
    assert model_class(SimpleNamespace(**{k: v for k, v in vars(_hf("tiny")).items() if k != "model_type"})) is Qwen3ForCausalLM


@pytest.mark.parametrize("over,match", [
    (dict(quantization_config={"quant_method": "fp8", "weight_block_size": [128, 128]}), "quantization_config"),
    (dict(mlp_only_layers=[1]), "mlp_only_layers"),
    (dict(decoder_sparse_step=2), "decoder_sparse_step"),
    (dict(moe_intermediate_size=96), "multiples of 64"),
    (dict(hidden_size=288), "multiples of 64"),
    (dict(num_experts=257), "at most 256 experts"),
    (dict(num_experts_per_tok=17, num_experts=64), "16 per token"),
    (dict(num_experts_per_tok=20), "16 per token"),
])
def test_unsupported_configs_refused_before_weights(over, match):
    with pytest.raises(NotImplementedError, match=match):
        Qwen3MoeForCausalLM(_hf(**over), 0, 1, device="cpu", max_position=64)


def test_tensor_parallel_shape_rule():
    Qwen3MoeForCausalLM(_hf(), 1, 2, device="cpu", max_position=64)             # 128 / 2 = 64
    with pytest.raises(NotImplementedError, match="multiples of 64"):
        Qwen3MoeForCausalLM(_hf(), 0, 4, device="cpu", max_position=64)         # 128 / 4 = 32
    with pytest.raises(NotImplementedError):
        Qwen3MoeForCausalLM(_hf(moe_intermediate_size=192), 0, 2, device="cpu", max_position=64)


def test_public_30b_a3b_dims_pass_and_size():
    d = PRESETS["qwen3-30b-a3b"]
    hf = _hf("qwen3-30b-a3b")
    from nanovllm.models.qwen3_moe import check_moe_config
    for tp in (1, 2, 4):
        check_moe_config(hf, tp)
    shapes = weight_shapes(d)
    params = sum(torch.Size(s).numel() for s in shapes.values())
    assert 30.4e9 < params < 30.6e9                       # Qwen3-30B-A3B: 30.5 B parameters
    assert len([n for n in shapes if ".experts." in n]) == 48 * 128 * 3


# ---- presets, directories and the loader ---------------------------------------------------------------------------------
@pytest.mark.parametrize("preset", ["tiny-moe", "tiny-moe-g8", "qwen3-30b-a3b"])
def test_weight_shapes_use_the_hub_names(preset):
    d = PRESETS[preset]
    s = weight_shapes(d)
    H, E, I = d["hidden_size"], d["num_experts"], d["moe_intermediate_size"]
    p = "model.layers.1.mlp."
    assert s[p + "gate.weight"] == (E, H)
    assert s[p + f"experts.{E - 1}.gate_proj.weight"] == (I, H) and s[p + "experts.0.up_proj.weight"] == (I, H)
    assert s[p + "experts.3.down_proj.weight"] == (H, I)
    assert not any(n.endswith(("mlp.gate_proj.weight", "mlp.down_proj.weight")) for n in s)
    cfg = hf_config_dict(d)
    assert cfg["model_type"] == "qwen3_moe" and cfg["architectures"] == ["Qwen3MoeForCausalLM"]
    assert cfg["decoder_sparse_step"] == 1 and cfg["mlp_only_layers"] == []


def test_router_weights_are_drawn_wide():
    w = random_weights(PRESETS["tiny-moe"], seed=5)
    g = w["model.layers.0.mlp.gate.weight"].float()
    assert abs(g.std().item() * 256 ** 0.5 - 2.0) < 0.1
    assert abs(w["model.layers.0.mlp.experts.2.up_proj.weight"].float().std().item() - 0.02) < 0.002


def test_make_model_dir_writes_a_moe_checkpoint(tmp_path):
    d = make_model_dir(str(tmp_path / "m"), "tiny-moe", seed=3, tokenizer=False)
    cfg = json.load(open(os.path.join(d, "config.json")))
    assert cfg["model_type"] == "qwen3_moe" and cfg["num_experts"] == 16 and cfg["num_experts_per_tok"] == 4
    from transformers import AutoConfig
    hf = AutoConfig.from_pretrained(d)
    assert type(hf).__name__ == "Qwen3MoeConfig" and hf.moe_intermediate_size == 128 and hf.norm_topk_prob
    from safetensors import safe_open
    with safe_open(os.path.join(d, "model.safetensors"), "pt", "cpu") as f:
        assert set(f.keys()) == set(weight_shapes(PRESETS["tiny-moe"]))
    with pytest.raises(NotImplementedError):
        make_model_dir(str(tmp_path / "q"), "tiny-moe", fp8=True, tokenizer=False)


def _load(preset, rank, world, weights):
    m = Qwen3MoeForCausalLM(_hf(preset), rank, world, device="cpu", max_position=64)
    for n, w in weights.items():
        m.load_hf_tensor(n, w)
    return m


@pytest.mark.parametrize("world", [1, 2])
def test_loader_stacks_and_slices_experts(world):
    d = PRESETS["tiny-moe"]
    full = random_weights(d, seed=11)
    I = d["moe_intermediate_size"] // world
    for rank in range(world):
        m = _load("tiny-moe", rank, world, full)
        for li in range(d["num_hidden_layers"]):
            L, ref = m.layers[li], stack_experts(full, li, d["num_experts"])
            assert torch.equal(L.gate, ref["gate"])
            assert L.gate_up.shape == (16, 2 * I, 256) and L.down.shape == (16, 256, I)
            Ifull = d["moe_intermediate_size"]
            want_gu = torch.cat([ref["gate_up"][:, rank * I:(rank + 1) * I], ref["gate_up"][:, Ifull + rank * I:Ifull + (rank + 1) * I]], 1)
            assert torch.equal(L.gate_up, want_gu)
            assert torch.equal(L.down, ref["down"][:, :, rank * I:(rank + 1) * I])
            assert torch.equal(L.qkv[:m.q_size], full[f"model.layers.{li}.self_attn.q_proj.weight"].chunk(world, 0)[rank])


def test_unexpected_moe_tensors_refused():
    m = Qwen3MoeForCausalLM(_hf(), 0, 1, device="cpu", max_position=64)
    for name in ("model.layers.0.mlp.gate_proj.weight", "model.layers.0.mlp.experts.16.up_proj.weight",
                 "model.layers.0.mlp.experts.0.wi.weight", "model.layers.0.mlp.shared_expert.up_proj.weight"):
        with pytest.raises(KeyError):
            m.load_hf_tensor(name, torch.zeros(128, 256, dtype=torch.bfloat16))


def test_random_init_matches_the_checkpoint_of_the_same_seed(tmp_path):
    d = make_model_dir(str(tmp_path / "m"), "tiny-moe", seed=3, tokenizer=False)
    a = Qwen3MoeForCausalLM(_hf(), 0, 1, device="cpu", max_position=64)
    load_model(a, d)
    b = Qwen3MoeForCausalLM(_hf(), 0, 1, device="cpu", max_position=64)
    load_model(b, str(tmp_path), allow_random=True, seed=3)
    for La, Lb in zip(a.layers, b.layers):
        assert torch.equal(La.gate, Lb.gate) and torch.equal(La.gate_up, Lb.gate_up) and torch.equal(La.down, Lb.down)


def test_dense_experiments_ignored(monkeypatch):
    monkeypatch.setenv("B200_TAIL", "mega")
    monkeypatch.setenv("B200_DUAL", "1")
    monkeypatch.setenv("B200_LINEAR", "gu")
    m = Qwen3MoeForCausalLM(_hf(), 0, 1, device="cpu", max_position=64)
    assert not (m.mega_tail or m.dual or m.tc_gate_up)
    monkeypatch.setenv("B200_LINEAR", "auto")
    assert Qwen3MoeForCausalLM(_hf(), 0, 1, device="cpu", max_position=64).tc_linear      # o_proj keeps its dense path


# ---- the C entry points ---------------------------------------------------------------------------------------------------
def _scratch():
    buf = ctypes.create_string_buffer(1 << 16)
    return buf, ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16


def test_entry_points_refuse_bad_arguments():
    lib = nat.load()
    buf, P = _scratch()
    assert lib.b200_moe_max_tiles(2048, 128) == 16 + 128 and lib.b200_moe_max_tiles(1, 128) == 2
    assert lib.b200_moe_max_tiles(0, 8) == 0 and lib.b200_moe_max_tiles(-1, 8) == -1 and lib.b200_moe_max_tiles(4, 0) == -1
    # route: logits [T, E] bf16, E <= 256, top_k <= min(16, E)
    route = lambda lg=P, st=16, t=1, e=16, k=4, ids=P, w=P: lib.b200_moe_route(lg, st, t, e, k, 1, ids, w, None)
    assert route(lg=None) == EINVAL and route(ids=None) == EINVAL and route(w=None) == EINVAL
    assert route(t=-1) == EINVAL and route(e=0) == EINVAL and route(k=0) == EINVAL and route(st=8) == EINVAL
    assert route(lg=P + 1) == EINVAL and route(ids=P + 2) == EINVAL
    assert route(e=257, st=257) == EUNSUPPORTED and route(k=17, e=32, st=32) == EUNSUPPORTED and route(k=5, e=4) == EUNSUPPORTED
    assert route(t=0) == 0
    # align: the tile table must hold b200_moe_max_tiles rows
    align = lambda ids=P, n=8, e=16, perm=P, tiles=P, mt=16: lib.b200_moe_align(ids, n, e, perm, tiles, mt, None)
    assert align(ids=None) == EINVAL and align(perm=None) == EINVAL and align(tiles=None) == EINVAL
    assert align(n=-1) == EINVAL and align(e=0) == EINVAL and align(tiles=P + 4) == EINVAL
    assert align(e=300) == EUNSUPPORTED and align(mt=8) == EWORKSPACE
    # gather / combine: 16-byte rows
    gather = lambda x=P, st=64, t=1, h=64, k=4, perm=P, out=P: lib.b200_moe_gather(x, st, t, h, k, perm, out, None)
    assert gather(x=None) == EINVAL and gather(out=P + 8) == EINVAL and gather(st=60) == EINVAL and gather(st=32) == EINVAL
    assert gather(h=60, st=64) == EUNSUPPORTED and gather(t=0) == 0
    combine = lambda y=P, perm=P, w=P, t=1, h=64, k=4, out=P, st=64: lib.b200_moe_combine(y, perm, w, t, h, k, out, st, None)
    assert combine(y=None) == EINVAL and combine(w=None) == EINVAL and combine(out=P + 2) == EINVAL and combine(st=32) == EINVAL
    assert combine(k=17) == EUNSUPPORTED and combine(h=12, st=16) == EUNSUPPORTED and combine(t=0) == 0
    # grouped GEMM: epilogue 0 / 1, k % 64, block_n from the list, n_out a multiple of the CTA's output columns
    lin = lambda x=P, w=P, out=P, st=128, rows=8, e=16, n=128, k=256, tiles=P, mt=8, epi=1, bn=64: \
        lib.b200_moe_linear(x, w, out, st, rows, e, n, k, tiles, mt, epi, bn, 0, None)
    assert lin(x=None) == EINVAL and lin(tiles=None) == EINVAL and lin(tiles=P + 4) == EINVAL and lin(epi=2) == EINVAL
    assert lin(st=64) == EINVAL and lin(rows=-1) == EINVAL and lin(mt=-1) == EINVAL
    assert lin(k=96) == EUNSUPPORTED and lin(bn=16) == EUNSUPPORTED and lin(bn=48) == EUNSUPPORTED
    assert lin(n=112) == EUNSUPPORTED and lin(mt=70000) == EUNSUPPORTED
    assert lin(rows=0) == 0 and lin(mt=0) == 0


# ---- the tile table --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["empty_experts", "one_hot_expert", "tile_edges", "one_token_per_expert"])
def test_tile_table_reference(case):
    E, BM = 8, 128
    if case == "empty_experts":
        ids = torch.tensor([[5, 2], [2, 5], [5, 7]])
    elif case == "one_hot_expert":
        ids = torch.full((300, 1), 3)
    elif case == "tile_edges":
        ids = torch.cat([torch.full((c,), e) for e, c in ((0, BM - 1), (1, BM), (2, BM + 1), (4, 2 * BM))]).reshape(-1, 1)
    else:
        ids = torch.arange(E).reshape(-1, 1)
    segs, tiles = tile_table_ref(ids, E, BM)
    counts = torch.bincount(ids.reshape(-1), minlength=E).tolist()
    n = ids.numel()
    assert len(tiles) <= nat.load().b200_moe_max_tiles(n, E)
    assert [c for _, c in segs] == counts and segs[0][0] == 0
    assert all(segs[e + 1][0] == segs[e][0] + segs[e][1] for e in range(E - 1))
    covered = []
    for e, r0, r1 in tiles:
        assert 0 < r1 - r0 <= BM and segs[e][0] <= r0 and r1 <= segs[e][0] + segs[e][1]
        covered += list(range(r0, r1))
    assert covered == list(range(n))                      # every row in exactly one tile, tiles in row order
    if case == "tile_edges":
        assert [(e, r1 - r0) for e, r0, r1 in tiles] == [(0, 127), (1, 128), (2, 128), (2, 1), (4, 128), (4, 128)]
    if case == "empty_experts":
        assert [e for e, _, _ in tiles] == [2, 5, 7]


# ---- the reference against HF transformers ---------------------------------------------------------------------------------
@pytest.mark.parametrize("norm", [True, False])
def test_moe_ref_matches_hf_sparse_moe_block_in_float64(norm):
    try:
        from transformers import Qwen3MoeConfig
        from transformers.models.qwen3_moe.modeling_qwen3_moe import Qwen3MoeSparseMoeBlock
    except ImportError:
        pytest.skip("transformers has no Qwen3MoeSparseMoeBlock")
    E, k, H, I, T = 16, 4, 64, 32, 97
    cfg = Qwen3MoeConfig(hidden_size=H, moe_intermediate_size=I, num_experts=E, num_experts_per_tok=k, norm_topk_prob=norm)
    g = torch.Generator().manual_seed(4)
    gate = torch.randn(E, H, generator=g, dtype=torch.float64) * 0.3
    gate_up = torch.randn(E, 2 * I, H, generator=g, dtype=torch.float64) * 0.1
    down = torch.randn(E, H, I, generator=g, dtype=torch.float64) * 0.1
    x = torch.randn(T, H, generator=g, dtype=torch.float64)
    block = Qwen3MoeSparseMoeBlock(cfg).double()
    sd = block.state_dict()
    names = {n: p.shape for n, p in sd.items()}
    if "experts.gate_up_proj" in names:                     # transformers 5.x: stacked experts
        block.load_state_dict({"gate.weight": gate, "experts.gate_up_proj": gate_up, "experts.down_proj": down})
    else:                                                   # 4.x: one module per expert
        w = {"gate.weight": gate}
        for e in range(E):
            w[f"experts.{e}.gate_proj.weight"] = gate_up[e, :I]
            w[f"experts.{e}.up_proj.weight"] = gate_up[e, I:]
            w[f"experts.{e}.down_proj.weight"] = down[e]
        block.load_state_dict(w)
    with torch.no_grad():
        out = block(x[None])
        out = out[0] if isinstance(out, tuple) else out
        want = out.reshape(T, H)
        router = block.gate(x)
        hf_ids = router[2] if isinstance(router, tuple) and len(router) == 3 else torch.topk(torch.softmax(router.float(), -1), k).indices
    ids, w = route_ref(x @ gate.t(), k, norm)
    assert torch.equal(ids, hf_ids.long())
    got = moe_block_ref(x, gate, gate_up, down, k, norm)
    assert (got - want).abs().max().item() <= 1e-12 * max(1.0, want.abs().max().item())


def test_route_ref_ties_and_order():
    lg = torch.tensor([[1.0, 3.0, 3.0, 0.5, 3.0]], dtype=torch.bfloat16)
    ids, w = route_ref(lg, 3, False)
    assert ids.tolist() == [[1, 2, 4]] and torch.equal(w[0, 0], w[0, 2])
    ids, w = route_ref(lg, 4, True)
    assert ids.tolist() == [[1, 2, 4, 0]] and abs(w.sum().item() - 1.0) < 1e-6
