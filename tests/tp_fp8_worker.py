"""Tensor-parallel check of a block-FP8 checkpoint (launched by tests/test_gpu_linear_fp8.py, two ranks on one GPU over
gloo): every rank builds LLM(..., tensor_parallel_size=world) on the same FP8 directory, generates greedily, and rank 0
checks that the ranks agree and that every token is the one-rank FP8 oracle's argmax or within its bf16 tie band."""
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "nano-vllm_b200"), os.path.join(ROOT, "tests")]


def main():
    import torch
    import torch.distributed as dist
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(0)
    dist.init_process_group(os.environ.get("B200_TP_BACKEND", "gloo"))
    from nanovllm import LLM, SamplingParams
    from nanovllm.utils.synthetic import PRESETS, hf_config_dict, make_model_dir, quantize_checkpoint, random_weights
    preset = "tiny-g4"
    mdir = f"/tmp/tp_fp8_model_{preset}_{os.getuid()}"
    if rank == 0:
        make_model_dir(mdir, preset, seed=1234, fp8=True)
    dist.barrier()
    llm = LLM(mdir, tensor_parallel_size=world, enforce_eager=True, max_model_len=256, max_num_seqs=8,
              max_num_batched_tokens=256, kvcache_block_size=16, num_kvcache_blocks=96)
    rnd = random.Random(3)
    vocab = PRESETS[preset]["vocab_size"]
    prompts = [[rnd.randint(2, vocab - 1) for _ in range(rnd.randint(4, 70))] for _ in range(8)]
    outs = llm.generate(prompts, SamplingParams(temperature=0.0, max_tokens=12, ignore_eos=True), use_tqdm=False)
    toks = [o["token_ids"] for o in outs]
    gathered = [None] * world
    dist.all_gather_object(gathered, toks)
    if rank == 0:
        assert all(g == toks for g in gathered), "ranks disagree on the sampled tokens"
        from fp8_ref import Qwen3RefFp8W
        from gpu_helpers import check_greedy_against_oracle
        from oracle.qwen3_ref import RefDims
        oracle = Qwen3RefFp8W(RefDims.from_json(hf_config_dict(PRESETS[preset])),
                              quantize_checkpoint(random_weights(PRESETS[preset], seed=1234)), rounding="fused")
        n = d = 0
        for p, t in zip(prompts, toks):
            a, b, _ = check_greedy_against_oracle(oracle, p, t, ulps=12.0)
            n, d = n + a, d + b
        print("TP_FP8_RESULT " + json.dumps(dict(world=world, greedy_tokens=n, differ_from_oracle_argmax=d, ok=True)), flush=True)
    llm.exit()


if __name__ == "__main__":
    main()
