"""Tensor-parallel check of a Qwen3 MoE checkpoint (launched by tests/test_gpu_moe.py, two ranks on one GPU over gloo):
every rank builds LLM(..., tensor_parallel_size=world) on the same tiny-moe directory (each expert sharded along
moe_intermediate_size), generates greedily, and rank 0 checks that the ranks agree and that the first token of every
prompt is the one-rank oracle's argmax or within its bf16 tie band.  The prompts route every token with a gap of at least
4 bf16 ulps (moe_ref.gap_safe_sequences), so the first token depends on no near-tied routing; later tokens can route
near a tie, where the sharded sums' bf16 roundings may pick the other expert, so those are counted, not checked."""
import json
import os
import random
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "nano-vllm_b200"), os.path.join(ROOT, "tests")]


def main():
    import torch
    import torch.distributed as dist
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(0)
    dist.init_process_group(os.environ.get("B200_TP_BACKEND", "gloo"))
    from nanovllm import LLM, SamplingParams
    from nanovllm.utils.synthetic import PRESETS, make_model_dir, random_weights
    preset = "tiny-moe"
    box = [tempfile.mkdtemp(prefix="tp_moe_model_") if rank == 0 else None]     # a fresh directory: no stale checkpoint
    dist.broadcast_object_list(box, src=0)
    mdir = box[0]
    if rank == 0:
        make_model_dir(mdir, preset, seed=1234)
    dist.barrier()
    llm = LLM(mdir, tensor_parallel_size=world, enforce_eager=True, max_model_len=256, max_num_seqs=8,
              max_num_batched_tokens=256, kvcache_block_size=16, num_kvcache_blocks=96)
    from moe_ref import Qwen3MoeRef, gap_safe_sequences
    vocab = PRESETS[preset]["vocab_size"]
    oracle = Qwen3MoeRef.from_preset(PRESETS[preset], random_weights(PRESETS[preset], seed=1234), rounding="fused")
    rnd = random.Random(3)
    prompts = gap_safe_sequences(oracle, vocab, [rnd.randint(4, 40) for _ in range(6)], seed=3, gap_ulps=6.0)
    outs = llm.generate(prompts, SamplingParams(temperature=0.0, max_tokens=12, ignore_eos=True), use_tqdm=False)
    toks = [o["token_ids"] for o in outs]
    gathered = [None] * world
    dist.all_gather_object(gathered, toks)
    if rank == 0:
        assert all(g == toks for g in gathered), "ranks disagree on the sampled tokens"
        from gpu_helpers import check_greedy_against_oracle, oracle_full_logits
        n = d = 0
        for p, t in zip(prompts, toks):
            a, b, _ = check_greedy_against_oracle(oracle, p, t[:1], ulps=12.0)
            n, d = n + a, d + b
            lg = oracle_full_logits(oracle, p + t[:-1])[len(p) - 1:]
            later = sum(int(lg[i].argmax()) != tok for i, tok in enumerate(t) if i > 0)
            d += later
        print("TP_MOE_RESULT " + json.dumps(dict(world=world, first_tokens_checked=n, tokens_differing_from_oracle_argmax=d, ok=True)), flush=True)
    llm.exit()
    if rank == 0:
        shutil.rmtree(mdir, ignore_errors=True)


if __name__ == "__main__":
    main()
