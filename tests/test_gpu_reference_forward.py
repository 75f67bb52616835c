"""North-star parity: the product forward vs the REFERENCE'S OWN GPU FORWARD on identical inputs.

Three implementations see the same weights and the same teacher-forced serving script (packed prefill, decode across a
block boundary, prefix-cache hit batched with a fresh prompt, a two-chunk prompt, mixed decode) at Qwen3-0.6B dimensions
(hidden 1024, 16/8 heads, vocab 151 936) with 256-token pages and 256...1 120-token sequences:

  ref    the unmodified reference: its nn.Modules, flash-attn, Triton store_kvcache, torch.compile'd norm/rope/activation,
         run on an H100 by oracle/make_gpu_golden.py (through tests/ref_gpu_forward.py), which stored per step its error
         against the truth, its greedy tokens and its logits at a seeded sample of columns in tests/golden/ref_gpu_forward_L*.npz;
  ours   the product model (libb200attn kernels + cuBLAS) in this process;
  truth  the oracle restatement evaluated in fp32 end to end (fp32 weights, no bf16 rounding anywhere) on the CPU.

The bar: ours is no further from the fp32 truth than the reference's own GPU path is (x1.25 + 1e-3 slack), and every row
whose fp32 argmax wins by more than 8 bf16 roundings is decoded identically by ours and the truth.  The numbers are recorded with gpu_helpers.record.
"""
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import pytest
import torch

from gpu_helpers import ROOT, record
from oracle.model_script import make_script, run_script
from oracle.qwen3_ref import Qwen3Ref, RefDims, alloc_logical_kv

pytestmark = pytest.mark.gpu

REF = os.path.join(ROOT, "oracle", "_ref", "nanovllm")


def _dims(layers: int) -> dict:
    from nanovllm.utils.synthetic import PRESETS
    d = dict(PRESETS["qwen3-0.6b"])
    d["num_hidden_layers"] = layers
    return d


def _run_reference(model_dir: str, script: dict, tmp: str, compiled: bool, dropin: bool = False):
    import numpy as np
    sp, op = os.path.join(tmp, "script.json"), os.path.join(tmp, f"ref_{int(compiled)}_{int(dropin)}.npz")
    with open(sp, "w") as f:
        json.dump(script, f)
    env = dict(os.environ)
    env.pop("TORCH_COMPILE_DISABLE", None)
    if not compiled:
        env["TORCH_COMPILE_DISABLE"] = "1"
    env["REF_FORWARD_PORT"] = str(29731 + (os.getpid() % 200))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "ref_gpu_forward.py"), model_dir, sp, op] + (["--dropin"] if dropin else []),
                       env=env, capture_output=True, text=True, timeout=900)
    if r.returncode != 0:
        return None, (r.stdout + r.stderr)[-2000:]
    z = np.load(op)
    return [torch.from_numpy(z[f"logits_{i}"]) for i in range(len([k for k in z.files if k.startswith("logits_")]))], ""


@pytest.mark.parametrize("layers", [4, 28])
def test_product_vs_reference_gpu_forward_vs_fp32_truth(layers, tmp_path):
    import numpy as np
    from nanovllm import ops
    from nanovllm.models.qwen3 import Qwen3ForCausalLM
    from nanovllm.utils.context import reset_context, set_context
    from nanovllm.utils.synthetic import hf_config_dict, random_weights
    dims = _dims(layers)
    weights = random_weights(dims, seed=4321)
    script = make_script(dims["vocab_size"], scale=16)                 # 256-token pages: the reference's only page size
    gold = np.load(os.path.join(ROOT, "tests", "golden", f"ref_gpu_forward_L{layers}.npz"))
    cols = torch.from_numpy(gold["columns"])
    ref_mode = str(gold["ref_mode"])

    # ---- ours
    hf = SimpleNamespace(**hf_config_dict(dims))
    model = Qwen3ForCausalLM(hf, 0, 1, "cuda", max_position=4096)
    for name, w in weights.items():
        model.load_hf_tensor(name, w)
    kv = torch.zeros(ops.kv_cache_shape(layers, script["num_blocks"], model.num_kv_heads, script["block_size"], model.head_dim),
                     dtype=torch.bfloat16, device="cuda")
    ops.bind_kv_cache(kv)
    for i, a in enumerate(model.modules()):
        a.k_cache, a.v_cache, a.layer_id = kv[0, i], kv[1, i], i

    def gpu_step(ids, pos, c):
        set_context(c["is_prefill"], c.get("cu_seqlens_q"), c.get("cu_seqlens_k"), c.get("max_seqlen_q", 0),
                    c.get("max_seqlen_k", 0), c.get("slot_mapping"), c.get("context_lens"), c.get("block_tables"))
        out = model.compute_logits(model(ids, pos)).float().cpu()
        reset_context()
        return out

    ours = run_script(torch, script, gpu_step, device="cuda")
    del model, kv
    torch.cuda.empty_cache()

    # ---- truth: fp32 everywhere
    w32 = {k: v.float() for k, v in weights.items()}
    oracle = Qwen3Ref(RefDims.from_json(hf_config_dict(dims)), w32, rounding="fused", max_pos=4096)
    okv = alloc_logical_kv(oracle.d, script["num_blocks"], script["block_size"], dtype=torch.float32)

    def cpu_step(ids, pos, c):
        ctx = SimpleNamespace(is_prefill=c["is_prefill"], cu_seqlens_q=c.get("cu_seqlens_q"), cu_seqlens_k=c.get("cu_seqlens_k"),
                              max_seqlen_q=c.get("max_seqlen_q", 0), max_seqlen_k=c.get("max_seqlen_k", 0),
                              slot_mapping=c.get("slot_mapping"), context_lens=c.get("context_lens"), block_tables=c.get("block_tables"))
        return oracle.logits(oracle.forward(ids, pos, ctx, okv), ctx).float()

    truth = run_script(torch, script, cpu_step)

    rel = lambda a, b: ((a - b).norm() / b.norm()).item()
    steps = []
    rows = agree_all = decided = decided_ok = ours_eq_ref = 0
    for i, (o, t) in enumerate(zip(ours, truth)):
        r_sample = torch.from_numpy(gold[f"ref_sample_{i}"]).view(torch.bfloat16).float()
        r_argmax = torch.from_numpy(gold[f"ref_argmax_{i}"])
        assert o.shape == t.shape and o.shape[0] == r_sample.shape[0] and torch.isfinite(o).all()
        ulp = 2 ** -8 * t.abs().max().item()
        e_o, e_r = rel(o, t), float(gold[f"ref_vs_truth_{i}"])
        e_or = rel(o[:, cols], r_sample)
        steps.append(dict(step=i, rows=o.shape[0], ours_vs_truth=e_o, ref_vs_truth=e_r, ours_vs_ref_sampled=e_or,
                          ours_max_ulps=((o - t).abs().max().item() / ulp), ref_max_ulps=float(gold[f"ref_max_ulps_{i}"])))
        assert e_o <= 1.25 * e_r + 1e-3, f"step {i}: ours {e_o:.3e} vs truth, the reference's own GPU forward {e_r:.3e}"
        top2 = t.topk(2, dim=-1).values
        for row in range(o.shape[0]):
            a_o, a_r, a_t = int(o[row].argmax()), int(r_argmax[row]), int(t[row].argmax())
            rows += 1
            agree_all += a_o == a_r == a_t
            ours_eq_ref += a_o == a_r
            if (top2[row, 0] - top2[row, 1]).item() > 8 * ulp:
                decided += 1
                decided_ok += a_o == a_t and a_r == a_t
                assert a_o == a_t, f"step {i} row {row}: greedy token {a_o}, fp32 truth {a_t} (reference: {a_r})"
    worst_o = max(s["ours_vs_truth"] for s in steps)
    worst_r = max(s["ref_vs_truth"] for s in steps)
    record("reference_gpu_forward", dict(layers=layers, dims="qwen3-0.6b", ref_mode=ref_mode, worst_ours_vs_truth=worst_o,
                                         worst_ref_vs_truth=worst_r, worst_ours_vs_ref_sampled=max(s["ours_vs_ref_sampled"] for s in steps),
                                         greedy_rows=rows, all_three_agree=agree_all, ours_eq_ref=ours_eq_ref,
                                         rows_with_clear_fp32_winner=decided, of_which_all_agree=decided_ok, steps=steps))


def test_reference_tree_with_only_the_operator_swapped(tmp_path):
    """INTEGRATION.md option B, executed: the reference's own model (its linears, norms, RoPE, LM head; eager) with ONLY
    Attention.forward and the cache layout line changed to libb200attn.so (integration/b200_binding.py), against the
    unmodified reference (flash-attn + Triton store) on the same weights and the same serving script.  It runs the
    reference's own modules, so it needs the reference staged under oracle/_ref (oracle/install_reference.py) and skips
    without it."""
    if not os.path.isdir(REF):
        pytest.skip("oracle/_ref (the staged reference) is not present")
    from nanovllm.utils.synthetic import make_model_dir
    dims = _dims(4)
    model_dir = make_model_dir(str(tmp_path / "model"), dims, seed=99, tokenizer=False)
    script = make_script(dims["vocab_size"], scale=16)
    ref, err = _run_reference(model_dir, script, str(tmp_path), compiled=False)
    assert ref is not None, err
    got, err = _run_reference(model_dir, script, str(tmp_path), compiled=False, dropin=True)
    assert got is not None, err
    rows = same = 0
    worst = 0.0
    for i, (g, r) in enumerate(zip(got, ref)):
        assert g.shape == r.shape and torch.isfinite(g).all()
        rel = ((g - r).norm() / r.norm()).item()
        worst = max(worst, rel)
        # two bf16 pipelines that differ only in the attention arithmetic (flash-attn rounds P to bf16 and accumulates in
        # its own order): measured 1.0e-2 at 4 layers, the same distance each of them has from the fp32 truth (the
        # three-way test above records ~1.1e-2 for both); the bar is twice that
        assert rel < 2.5e-2, f"step {i}: logits of the reference with our operator vs the unmodified reference: relative L2 {rel}"
        ulp = 2 ** -8 * r.abs().max().item()
        top2 = r.topk(2, dim=-1).values
        for row in range(g.shape[0]):
            rows += 1
            eq = int(g[row].argmax()) == int(r[row].argmax())
            same += eq
            if (top2[row, 0] - top2[row, 1]).item() > 8 * ulp:
                assert eq, f"step {i} row {row}: greedy token differs from the unmodified reference"
    record("integration_option_b", dict(layers=4, dims="qwen3-0.6b", worst_rel_l2_vs_unmodified_reference=worst,
                                        greedy_rows=rows, greedy_equal=same))
