"""Runs the UNMODIFIED reference model (oracle/_ref: its Qwen3ForCausalLM, its flash-attn Attention.forward,
its Triton store_kvcache, its loader) on cuda:0 over a teacher-forced serving script and saves the logits.
TEST INFRASTRUCTURE ONLY -- executed as a subprocess by tests/test_gpu_reference_forward.py because the reference
and the product both own the package name ``nanovllm``.

    python tests/ref_gpu_forward.py <model_dir> <script.json> <out.npz> [--dropin]

With --dropin the same reference runs with INTEGRATION.md's option B applied (integration/b200_binding.py): only
Attention.forward and the cache allocation line change, every other module is the reference's own.

What it does is what the reference's ModelRunner does in eager mode (engine/model_runner.py:17-48,103-121,195-220):
process group of one, bf16 default dtype on cuda, load_model, one [2, L, nblk, bs, Hkv, D] cache bound to every
module that has k_cache/v_cache, then per step set_context(...) -> model(input_ids, positions) -> compute_logits.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")


def main():
    model_dir, script_path, out_path = sys.argv[1:4]
    dropin = "--dropin" in sys.argv[4:]
    sys.path.insert(0, REF)
    sys.path.insert(1, ROOT)
    import numpy as np
    import torch
    import torch.distributed as dist
    import nanovllm
    assert os.path.realpath(nanovllm.__file__).startswith(os.path.realpath(REF)), nanovllm.__file__
    from transformers import AutoConfig
    from nanovllm.models.qwen3 import Qwen3ForCausalLM
    from nanovllm.utils.context import reset_context, set_context
    from nanovllm.utils.loader import load_model
    from oracle.model_script import run_script

    script = json.load(open(script_path))
    port = int(os.environ.get("REF_FORWARD_PORT", "29731"))
    dist.init_process_group("nccl", f"tcp://127.0.0.1:{port}", world_size=1, rank=0)
    torch.cuda.set_device(0)
    hf = AutoConfig.from_pretrained(model_dir)
    torch.set_default_dtype(torch.bfloat16)
    torch.set_default_device("cuda")
    model = Qwen3ForCausalLM(hf)
    load_model(model, model_dir)
    head_dim = getattr(hf, "head_dim", hf.hidden_size // hf.num_attention_heads)
    if dropin:
        from integration import b200_binding as b200
        b200.init(0)
        b200.patch()
        kv = b200.allocate_kv_cache(model, hf.num_hidden_layers, script["num_blocks"], script["block_size"],
                                    hf.num_key_value_heads, head_dim, hf.num_attention_heads)
    else:
        kv = torch.zeros(2, hf.num_hidden_layers, script["num_blocks"], script["block_size"], hf.num_key_value_heads, head_dim)
        layer = 0
        for module in model.modules():                       # model_runner.py:116-121
            if hasattr(module, "k_cache") and hasattr(module, "v_cache"):
                module.k_cache = kv[0, layer]
                module.v_cache = kv[1, layer]
                layer += 1
        assert layer == hf.num_hidden_layers
    torch.set_default_device("cpu")

    @torch.inference_mode()
    def step(ids, pos, c):
        set_context(c["is_prefill"], c.get("cu_seqlens_q"), c.get("cu_seqlens_k"), c.get("max_seqlen_q", 0),
                    c.get("max_seqlen_k", 0), c.get("slot_mapping"), c.get("context_lens"), c.get("block_tables"))
        logits = model.compute_logits(model(ids, pos))
        reset_context()
        return logits.float().cpu().numpy()

    outs = run_script(torch, script, step, device="cuda")
    np.savez(out_path, **{f"logits_{i}": o for i, o in enumerate(outs)},
             compiled=np.asarray(os.environ.get("TORCH_COMPILE_DISABLE", "0") != "1"))
    dist.destroy_process_group()
    print("ref_gpu_forward ok", len(outs), "steps")


if __name__ == "__main__":
    main()
