"""Generate tests/golden/ref_gpu_forward_L<layers>.npz: what the REFERENCE's own GPU forward computes on the serving script of
tests/test_gpu_reference_forward.py, so that the test compares the product against it without the reference present.

    python oracle/make_gpu_golden.py            # on a GPU, with the reference staged under oracle/_ref

For each layer count it runs tests/ref_gpu_forward.py (the unmodified reference: its nn.Modules, flash-attn, Triton
store_kvcache, torch.compile; eager if compiling fails) and the fp32 truth (oracle/qwen3_ref.py, fp32 end to end, CPU),
and stores per step: the reference's relative L2 error against the truth and its worst element in bf16 roundings of
the logit scale, per row: the reference's greedy token, and the reference's bf16 logits at a fixed, seeded sample of
SAMPLE_COLS vocabulary columns (the full logits would be megabytes).
"""
from __future__ import annotations

import os
import sys
import tempfile
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, "tests"), os.path.join(ROOT, "nano-vllm_b200"), ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

SAMPLE_COLS = 2048
MODEL_SEED = 4321


def sample_columns(vocab: int) -> np.ndarray:
    return np.sort(np.random.default_rng(2024).choice(vocab, SAMPLE_COLS, replace=False)).astype(np.int64)


def truth_logits(torch, dims: dict, weights: dict, script: dict) -> list:
    """The fp32 oracle over the script (no bf16 rounding anywhere)."""
    from nanovllm.utils.synthetic import hf_config_dict
    from oracle.model_script import run_script
    from oracle.qwen3_ref import Qwen3Ref, RefDims, alloc_logical_kv
    w32 = {k: v.float() for k, v in weights.items()}
    oracle = Qwen3Ref(RefDims.from_json(hf_config_dict(dims)), w32, rounding="fused", max_pos=4096)
    okv = alloc_logical_kv(oracle.d, script["num_blocks"], script["block_size"], dtype=torch.float32)

    def cpu_step(ids, pos, c):
        ctx = SimpleNamespace(is_prefill=c["is_prefill"], cu_seqlens_q=c.get("cu_seqlens_q"), cu_seqlens_k=c.get("cu_seqlens_k"),
                              max_seqlen_q=c.get("max_seqlen_q", 0), max_seqlen_k=c.get("max_seqlen_k", 0),
                              slot_mapping=c.get("slot_mapping"), context_lens=c.get("context_lens"), block_tables=c.get("block_tables"))
        return oracle.logits(oracle.forward(ids, pos, ctx, okv), ctx).float()

    return run_script(torch, script, cpu_step)


def main():
    import torch
    from test_gpu_reference_forward import _dims, _run_reference
    from nanovllm.utils.synthetic import make_model_dir, random_weights
    from oracle.model_script import make_script
    for layers in (4, 28):
        dims = _dims(layers)
        tmp = tempfile.mkdtemp(prefix="ref_gpu_golden_")
        model_dir = make_model_dir(os.path.join(tmp, "model"), dims, seed=MODEL_SEED, tokenizer=False)
        weights = random_weights(dims, seed=MODEL_SEED)
        script = make_script(dims["vocab_size"], scale=16)
        ref, err = _run_reference(model_dir, script, tmp, compiled=True)
        mode = "compiled"
        if ref is None:
            ref, err2 = _run_reference(model_dir, script, tmp, compiled=False)
            mode = "eager"
            assert ref is not None, err + "\n" + err2
        truth = truth_logits(torch, dims, weights, script)
        cols = sample_columns(dims["vocab_size"])
        out = {"columns": cols, "ref_mode": np.asarray(mode)}
        for i, (r, t) in enumerate(zip(ref, truth)):
            ulp = 2 ** -8 * t.abs().max().item()
            out[f"ref_vs_truth_{i}"] = np.asarray(((r - t).norm() / t.norm()).item())
            out[f"ref_max_ulps_{i}"] = np.asarray((r - t).abs().max().item() / ulp)
            out[f"ref_argmax_{i}"] = r.argmax(dim=-1).numpy().astype(np.int64)
            out[f"ref_sample_{i}"] = r[:, torch.from_numpy(cols)].to(torch.bfloat16).view(torch.int16).numpy()
        path = os.path.join(ROOT, "tests", "golden", f"ref_gpu_forward_L{layers}.npz")
        np.savez_compressed(path, **out)
        print("wrote", path, mode, [float(out[f"ref_vs_truth_{i}"]) for i in range(len(ref))])


if __name__ == "__main__":
    main()
