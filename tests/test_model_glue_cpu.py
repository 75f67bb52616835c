"""The product's model code (nanovllm/models/qwen3.py) with every GPU op replaced by a CPU stand-in built from the
oracle's free functions: checks the PYTHON around the kernels -- which op is called when, with which views, strides,
argument order and return values -- without a GPU.  On the default path the stand-ins are the oracle's own arithmetic,
so the logits must equal the oracle's bit for bit; on the wgmma paths (B200_LINEAR=tc: wgmma projections with fused
SiluAndMul / split-K partial sums) only the summation order differs.

This does not test any kernel (tests/test_gpu_*.py do); it exists so that a typo in the glue of a path that has not
reached a GPU yet costs a CPU test failure instead of a GPU call.
"""
from types import SimpleNamespace

import pytest
import torch

from oracle.model_script import make_script, run_script
from oracle.paged_attention_ref import paged_decode_ref, store_kvcache_ref, varlen_prefill_ref
from oracle.qwen3_ref import Qwen3Ref, RefDims, add_rmsnorm_ref, alloc_logical_kv, rmsnorm_ref, rope_ref, silu_mul_ref


class CpuOps:
    """Stand-ins with the signatures of nanovllm.ops; the KV cache lives in the reference's logical layout."""
    EPI_BF16, EPI_SILU, EPI_PARTIAL = 0, 1, 2

    def __init__(self, dims: RefDims, num_blocks: int, block_size: int):
        self.d, self.bs = dims, block_size
        self.kv = alloc_logical_kv(dims, num_blocks, block_size)
        self.calls: dict[str, int] = {}

    def _count(self, name):
        self.calls[name] = self.calls.get(name, 0) + 1

    # ---- elementwise ----------------------------------------------------------------------------------------------
    def embedding(self, ids, table, out=None):
        self._count("embedding")
        return table[ids]

    def rmsnorm(self, x, weight, eps, out=None):
        self._count("rmsnorm")
        return rmsnorm_ref(x, weight, eps)

    def add_rmsnorm(self, x, residual, weight, eps, out=None):
        self._count("add_rmsnorm")
        assert x.is_contiguous() and residual.is_contiguous() and x.shape == residual.shape
        y, r = add_rmsnorm_ref(x, residual, weight, eps)
        residual.copy_(r)                                     # the kernel updates the residual in place
        return y, residual

    def silu_mul(self, x, out=None):
        self._count("silu_mul")
        return silu_mul_ref(x)

    def _qk(self, qkv, hq, hkv, positions, qn, kn, cos_sin, eps):
        D = self.d.head_dim
        n = qkv.shape[0]
        q = qkv[:, :hq * D].reshape(n, hq, D)
        k = qkv[:, hq * D:(hq + hkv) * D].reshape(n, hkv, D)
        v = qkv[:, (hq + hkv) * D:].reshape(n, hkv, D)
        q = rope_ref(cos_sin, positions, rmsnorm_ref(q, qn, eps))
        k = rope_ref(cos_sin, positions, rmsnorm_ref(k, kn, eps))
        return q, k, v

    def qknorm_rope_store(self, layer, qkv, hq, hkv, positions, qn, kn, cos_sin, eps, slot_mapping=None):
        self._count("qknorm_rope_store")
        assert qkv.dim() == 2 and qkv.stride(1) == 1 and positions.dtype == torch.int64
        D = self.d.head_dim
        q, k, v = self._qk(qkv, hq, hkv, positions, qn, kn, cos_sin, eps)
        qkv[:, :hq * D] = q.reshape(qkv.shape[0], -1)         # in place, like the kernel
        qkv[:, hq * D:(hq + hkv) * D] = k.reshape(qkv.shape[0], -1)
        if slot_mapping is not None:
            assert slot_mapping.dtype == torch.int32
            store_kvcache_ref(k, v, self.kv[layer][0], self.kv[layer][1], slot_mapping)
        return qkv

    # ---- attention ------------------------------------------------------------------------------------------------
    def paged_decode_fused(self, layer, qkv, hq, qn, kn, cos_sin, eps, block_tables, context_lens, scale, out=None):
        self._count("paged_decode_fused")
        hkv = self.d.num_key_value_heads
        pos = (context_lens.to(torch.int64) - 1).clamp(min=0)
        q, k, v = self._qk(qkv.clone(), hq, hkv, pos, qn, kn, cos_sin, eps)         # qkv itself stays untouched
        rows = torch.arange(qkv.shape[0])
        slots = (block_tables[rows, (pos // self.bs)].to(torch.int64) * self.bs + pos % self.bs).to(torch.int32)
        slots[context_lens == 0] = -1                                                  # graph padding rows
        store_kvcache_ref(k, v, self.kv[layer][0], self.kv[layer][1], slots)
        return paged_decode_ref(q, self.kv[layer][0], self.kv[layer][1], context_lens, block_tables, scale, p_dtype=torch.bfloat16)

    def paged_decode(self, layer, q, block_tables, context_lens, scale, out=None):
        self._count("paged_decode")
        assert q.stride(2) == 1 and q.stride(1) == q.shape[2]
        return paged_decode_ref(q, self.kv[layer][0], self.kv[layer][1], context_lens, block_tables, scale, p_dtype=torch.bfloat16)

    def paged_prefill(self, layer, q, k, v, cu_q, cu_k, max_q, max_k, scale, block_tables=None, num_kv_heads=None, out=None):
        self._count("paged_prefill")
        assert q.stride(2) == 1 and q.stride(1) == q.shape[2]
        return varlen_prefill_ref(q, k, v, cu_q, cu_k, scale, block_tables, self.kv[layer][0], self.kv[layer][1], p_dtype=torch.bfloat16)

    def store_kv(self, layer, k, v, slot_mapping):
        self._count("store_kv")
        store_kvcache_ref(k, v, self.kv[layer][0], self.kv[layer][1], slot_mapping)

    # ---- wgmma projections ------------------------------------------------------------------------------------------
    class pdl_off:
        depth = 0

        def __enter__(self):
            type(self).depth += 1
            return self

        def __exit__(self, *exc):
            type(self).depth -= 1
            return False

    def linear(self, x, w, epilogue=0, block_n=32, k_splits=1, pdl=False, out=None, shallow=False, cluster=1, stages=0):
        self._count(f"linear{epilogue}")
        assert 0 <= stages <= 8
        assert x.dim() == 2 and x.stride(1) == 1 and w.is_contiguous() and x.shape[1] == w.shape[1] and x.shape[1] % 64 == 0
        xf, wf = x.float(), w.float()
        if epilogue == self.EPI_PARTIAL:
            assert (x.shape[1] // 64) % k_splits == 0 and w.shape[0] % block_n == 0
            ks = x.shape[1] // k_splits
            return torch.stack([xf[:, s * ks:(s + 1) * ks] @ wf[:, s * ks:(s + 1) * ks].t() for s in range(k_splits)])
        assert k_splits == 1
        y = (xf @ wf.t()).to(torch.bfloat16)
        if epilogue == self.EPI_SILU:
            assert (w.shape[0] // 2) % (block_n // 2) == 0
            y = silu_mul_ref(y)
        else:
            assert w.shape[0] % block_n == 0
        if out is not None:
            out.copy_(y)
            return out
        return y

    def add_rmsnorm_partials(self, partials, residual, weight, eps, pdl=False, out=None):
        self._count("add_rmsnorm_partials")
        assert partials.dtype == torch.float32 and partials.dim() == 3 and partials.shape[1:] == residual.shape
        assert residual.is_contiguous() and (out is None or (out.is_contiguous() and out.shape == residual.shape))
        h = partials[0].clone()
        for s in range(1, partials.shape[0]):
            h += partials[s]
        y, r = add_rmsnorm_ref(h.to(torch.bfloat16), residual, weight, eps)
        residual.copy_(r)
        if out is not None:
            out.copy_(y)
            return out, residual
        return y, residual


    # ---- persistent layer tail (csrc/layer_tail.cu) ------------------------------------------------------------------
    def layer_tail_workspace(self, max_rows, hidden, inter, max_splits, device="cpu"):
        self._count("layer_tail_workspace")
        return torch.zeros(16, dtype=torch.uint8)

    def layer_tail(self, attn_out, residual, w_o, ln_mid, w_gate_up, w_down, ln_next, eps, workspace, w_qkv_next=None,
                   splits_o=8, splits_down=8, x_next=None, qkv_out=None):
        self._count("layer_tail")
        import torch.nn.functional as F
        assert attn_out.dim() == 2 and attn_out.stride(1) == 1 and residual.is_contiguous()
        assert (attn_out.shape[1] // 64) % splits_o == 0 and (w_down.shape[1] // 64) % splits_down == 0
        x, r = add_rmsnorm_ref(F.linear(attn_out, w_o), residual, ln_mid, eps)
        h = F.linear(silu_mul_ref(F.linear(x, w_gate_up)), w_down)
        xn, r = add_rmsnorm_ref(h, r, ln_next, eps)
        residual.copy_(r)                                     # updated in place, like the kernel
        return xn, (F.linear(xn, w_qkv_next) if w_qkv_next is not None else None)


def run_product_model(monkeypatch, preset, env, fused_decode_max=None):
    import nanovllm.layers.attention as attn_mod
    import nanovllm.models.qwen3 as model_mod
    from nanovllm.utils.context import reset_context, set_context
    from nanovllm.utils.synthetic import PRESETS, hf_config_dict, random_weights
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    dims = RefDims.from_json(hf_config_dict(PRESETS[preset]))
    weights = random_weights(PRESETS[preset], seed=1234)
    script = make_script(PRESETS[preset]["vocab_size"])
    fake = CpuOps(dims, script["num_blocks"], script["block_size"])
    monkeypatch.setattr(model_mod, "ops", fake)
    monkeypatch.setattr(attn_mod, "ops", fake)
    hf = SimpleNamespace(**hf_config_dict(PRESETS[preset]))
    model = model_mod.Qwen3ForCausalLM(hf, 0, 1, "cpu", max_position=4096)
    if fused_decode_max is not None:
        model.fused_decode_max_batch = fused_decode_max
    for name, w in weights.items():
        model.load_hf_tensor(name, w)
    for i, a in enumerate(model.modules()):                    # "cache allocated" is all the model asks of these
        a.k_cache = a.v_cache = torch.zeros(1, dims.num_key_value_heads, script["block_size"], dims.head_dim, dtype=torch.bfloat16)
        a.layer_id = i

    def step(ids, pos, c):
        set_context(c["is_prefill"], c.get("cu_seqlens_q"), c.get("cu_seqlens_k"), c.get("max_seqlen_q", 0),
                    c.get("max_seqlen_k", 0), c.get("slot_mapping"), c.get("context_lens"), c.get("block_tables"))
        out = model.compute_logits(model(ids, pos))
        reset_context()
        return out

    got = run_script(torch, script, step)
    oracle = Qwen3Ref(dims, weights, rounding="fused", max_pos=4096, p_dtype=torch.bfloat16)
    kv = alloc_logical_kv(dims, script["num_blocks"], script["block_size"])
    from test_oracle_golden import oracle_step_fn
    want = run_script(torch, script, oracle_step_fn(oracle, kv))
    return got, want, fake, model


@pytest.mark.parametrize("preset", ["tiny", "tiny-g4"])
def test_default_path_glue_is_the_oracle(preset, monkeypatch):
    got, want, fake, model = run_product_model(monkeypatch, preset, {"B200_LINEAR": "cublas"})
    for i, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g, w), f"step {i}: max diff {(g.float() - w.float()).abs().max().item()}"
    assert fake.calls.get("qknorm_rope_store", 0) > 0 and fake.calls.get("paged_prefill", 0) > 0
    if model.num_heads // model.num_kv_heads <= 2:             # the fused decode front end serves small head groups
        assert fake.calls.get("paged_decode_fused", 0) > 0 and "paged_decode" not in fake.calls
    else:
        assert fake.calls.get("paged_decode", 0) > 0 and "paged_decode_fused" not in fake.calls


def test_two_kernel_decode_path_glue(monkeypatch):
    """Batches above the fused-decode threshold take q/k-norm+RoPE+store and attention as two ops."""
    got, want, fake, _ = run_product_model(monkeypatch, "tiny", {"B200_LINEAR": "cublas"}, fused_decode_max=0)
    for g, w in zip(got, want):
        assert torch.equal(g, w)
    assert fake.calls.get("paged_decode", 0) > 0 and "paged_decode_fused" not in fake.calls


@pytest.mark.parametrize("preset", ["tiny", "tiny-g4"])
def test_mega_tail_path_glue_is_the_oracle(preset, monkeypatch):
    """B200_TAIL=mega: decode steps run attention + ONE layer-tail op per layer; the glue (which norm weight, which next
    qkv weight, residual in place, the last layer) must reproduce the oracle bit for bit when the op is exact."""
    got, want, fake, model = run_product_model(monkeypatch, preset, {"B200_LINEAR": "cublas", "B200_TAIL": "mega"})
    assert model.mega_tail
    for i, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g, w), f"step {i}: max diff {(g.float() - w.float()).abs().max().item()}"
    decode_steps = 3                                           # steps 1, 2 and 6 of the script
    assert fake.calls["layer_tail"] == decode_steps * model.cfg.num_hidden_layers


@pytest.mark.parametrize("preset", ["tiny", "tiny-g4"])
def test_tc_linear_path_glue(preset, monkeypatch):
    got, want, fake, model = run_product_model(monkeypatch, preset, {"B200_LINEAR": "tc", "B200_LINEAR_CFG": "32,32,64,4,64,4,0"})
    assert model.tc_linear
    layers = model.cfg.num_hidden_layers
    steps = len(got)
    assert fake.calls["linear0"] == layers * steps and fake.calls["linear1"] == layers * steps      # qkv, gate_up+silu
    assert fake.calls["linear2"] == 2 * layers * steps and fake.calls["add_rmsnorm_partials"] == 2 * layers * steps
    assert "silu_mul" not in fake.calls and "add_rmsnorm" not in fake.calls
    for i, (g, w) in enumerate(zip(got, want)):
        rel = ((g.float() - w.float()).norm() / w.float().norm()).item()
        assert rel < 1e-2, f"step {i}: relative L2 {rel}"


@pytest.mark.parametrize("preset,fused_max", [("tiny", None), ("tiny", 0)])
def test_two_stream_decode_path_glue(preset, fused_max, monkeypatch):
    """B200_DUAL=1: decode batches are cut into two halves (streams on the GPU; plain order here) that each run the wgmma
    chain on their own rows / block tables / context lengths; the result must be the single-stream wgmma result (only
    the split-K summation order differs from the oracle)."""
    got, want, fake, model = run_product_model(monkeypatch, preset, {"B200_DUAL": "1", "B200_DUAL_MIN": "2", "B200_LINEAR": "cublas",
                                                                    "B200_DUAL_CFG": "32,32,64,4,64,4,3"}, fused_decode_max=fused_max)
    assert model.dual and model.dual_min == 2
    layers = model.cfg.num_hidden_layers
    assert fake.calls.get("linear2", 0) >= 2 * 2 * layers           # o/down split-K partials of both halves of >= 1 decode step
    assert fake.calls.get("linear1", 0) >= 2 * layers and fake.calls.get("linear0", 0) >= 2 * layers
    assert fake.pdl_off.depth == 0
    if fused_max == 0:
        assert fake.calls.get("paged_decode", 0) > 0
    else:
        assert fake.calls.get("paged_decode_fused", 0) > 0
    for i, (g, w) in enumerate(zip(got, want)):
        rel = ((g.float() - w.float()).norm() / w.float().norm()).item()
        assert rel < 1e-2, f"step {i}: relative L2 {rel}"


def test_gate_up_only_tc_mode_glue(monkeypatch):
    """B200_LINEAR=gu: decode steps run gate_up + SiluAndMul as ONE wgmma op, every other projection stays a library call
    (the mode tensor-parallel runs use to save a launch per layer); prefill keeps the two-op path."""
    got, want, fake, model = run_product_model(monkeypatch, "tiny", {"B200_LINEAR": "gu"})
    assert model.tc_gate_up and not model.tc_linear
    layers, decode_steps = model.cfg.num_hidden_layers, 3
    assert fake.calls["linear1"] == layers * decode_steps
    assert "linear0" not in fake.calls and "linear2" not in fake.calls and fake.calls.get("silu_mul", 0) > 0
    for i, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g, w), f"step {i}"            # the stand-in rounds exactly where the two-op path rounds


def test_fused_lm_head_runner_glue(monkeypatch):
    """ModelRunner._forward_and_sample with B200_LM_HEAD=fused hands the right tensors to ops.lm_head_sample (opt-in path)."""
    import nanovllm.engine.model_runner as mr
    from nanovllm.models.qwen3 import Qwen3ForCausalLM
    from nanovllm.utils.context import reset_context, set_context
    seen = {}

    class Ops:
        @staticmethod
        def lm_head_sample(hidden, lm_head, temps, seed, step, key_ws, out=None, index_offset=0, out_keys=None, step_dev=None, **kw):
            assert hidden.dim() == 2 and hidden.shape[1] == lm_head.shape[1] and key_ws.numel() >= hidden.shape[0]
            assert out is not None and out.shape == (hidden.shape[0],) and out.dtype == torch.int64
            seen.update(rows=hidden.shape[0], seed=seed, step=step, step_dev=step_dev, offset=index_offset)
            out.copy_((hidden.float() @ lm_head.float().t()).argmax(-1))
            return out

        @staticmethod
        def sample(*a, **k):
            raise AssertionError("the two-kernel path must not run when the fused head is on")

    monkeypatch.setattr(mr, "ops", Ops)
    hidden_all = torch.randn(10, 64).to(torch.bfloat16)
    head = torch.randn(500, 64).to(torch.bfloat16)

    class Model:
        lm_head = head

        def __call__(self, ids, pos):
            return hidden_all

        def last_token_rows(self, h):
            return Qwen3ForCausalLM.last_token_rows(self, h)

    runner = SimpleNamespace(model=Model(), fused_lm_head=True, world_size=1, sample_seed=3, vocab_offset=0,
                             g_keyws=torch.zeros(16, dtype=torch.int64), g_tokens=torch.zeros(16, dtype=torch.int64),
                             g_keys=torch.zeros(16, dtype=torch.int64))
    cu = torch.tensor([0, 4, 10], dtype=torch.int32)
    set_context(True, cu, cu, 6, 6, None, None, None)                       # prefill: the last token of each of 2 sequences
    step_dev = torch.zeros(1, dtype=torch.int64)
    mr.ModelRunner._forward_and_sample(runner, torch.zeros(10, dtype=torch.int64), torch.zeros(10, dtype=torch.int64),
                                       torch.zeros(2), step_dev, 2)
    reset_context()
    assert seen == dict(rows=2, seed=3, step=0, step_dev=step_dev, offset=0)
    want = (hidden_all[[3, 9]].float() @ head.float().t()).argmax(-1)
    assert torch.equal(runner.g_tokens[:2], want)


@pytest.mark.parametrize("preset", ["tiny", "tiny-g4"])
def test_default_auto_linear_policy_glue(preset, monkeypatch):
    """The default policy (B200_LINEAR=auto): o_proj / down_proj of small batches through the split-K wgmma path with the
    fused add-norm, qkv / gate_up through the library; only the summation order differs from the oracle."""
    monkeypatch.delenv("B200_LINEAR", raising=False)
    got, want, fake, model = run_product_model(monkeypatch, preset, {})
    assert model.tc_linear and not model.tc_cols and model.tc_max_rows == 128
    assert fake.calls.get("linear2", 0) > 0 and fake.calls.get("add_rmsnorm_partials", 0) > 0
    assert "linear0" not in fake.calls and "linear1" not in fake.calls and fake.calls.get("silu_mul", 0) > 0
    for i, (g, w) in enumerate(zip(got, want)):
        rel = ((g.float() - w.float()).norm() / w.float().norm()).item()
        assert rel < 1e-2, f"step {i}: relative L2 {rel}"
