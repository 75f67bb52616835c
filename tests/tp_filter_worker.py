"""Tensor-parallel engine check of top-k / top-p / min-p sampling, one process per rank (launched by
tests/test_gpu_sampling_filters.py; gloo on one GPU there):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29567 tests/tp_filter_worker.py

Every rank generates with filtered requests (eager); rank 0 checks that top_k=1 requests are greedy against the CPU oracle
and that every rank returned the same tokens for the top_p=0.95, top_k=20 requests.
"""
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "nano-vllm_b200"), os.path.join(ROOT, "tests")]


def main():
    import torch
    import torch.distributed as dist
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    backend = os.environ.get("B200_TP_BACKEND", "nccl")
    if os.environ.get("B200_TP_ONE_DEVICE") == "1":
        local = 0
    torch.cuda.set_device(local)
    if backend == "nccl":
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    else:
        dist.init_process_group(backend)
    from nanovllm import LLM, SamplingParams
    from nanovllm.utils.synthetic import PRESETS, make_model_dir, random_weights
    preset = "tiny-g4"
    mdir = f"/tmp/tp_filter_model_{preset}"
    if local == 0:
        make_model_dir(mdir, preset, seed=1234)
    dist.barrier()
    llm = LLM(mdir, tensor_parallel_size=world, enforce_eager=True, max_model_len=256, max_num_seqs=8,
              max_num_batched_tokens=256, kvcache_block_size=16, num_kvcache_blocks=96)
    rnd = random.Random(4)
    vocab = PRESETS[preset]["vocab_size"]
    prompts = [[rnd.randint(2, vocab - 1) for _ in range(rnd.randint(4, 60))] for _ in range(10)]
    sps = [SamplingParams(temperature=1.0, max_tokens=6 + i, ignore_eos=True, top_k=1) if i % 2 else
           SamplingParams(temperature=0.6, max_tokens=6 + i, ignore_eos=True, top_p=0.95, top_k=20) for i in range(10)]
    toks = [o["token_ids"] for o in llm.generate(prompts, sps, use_tqdm=False)]
    gathered = [None] * world
    dist.all_gather_object(gathered, toks)
    if rank == 0:
        assert all(g == toks for g in gathered), "ranks disagree on the sampled tokens"
        from gpu_helpers import check_greedy_against_oracle, make_oracle
        oracle = make_oracle(PRESETS[preset], random_weights(PRESETS[preset], seed=1234), "fused")
        n = 0
        for p, sp, t in zip(prompts, sps, toks):
            assert len(t) == sp.max_tokens
            if sp.top_k == 1:
                n += check_greedy_against_oracle(oracle, p, t)[0]
        print("TP_FILTER_RESULT " + json.dumps(dict(world=world, backend=backend, greedy_tokens=n, ok=True)), flush=True)
    llm.exit()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
