"""Tensor-parallel engine check of the per-token logprobs, one process per rank (launched by tests/test_gpu_logprobs.py;
gloo on one GPU there):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29573 tests/tp_logprob_worker.py

Every rank generates with logprob requests (eager), greedy and sampled, some also filtered or penalised; rank 0 checks
that every rank returned the same tokens and bit-identical logprob dicts, and that the greedy requests' logprobs follow
the CPU oracle's log_softmax.
"""
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "nano-vllm_b200"), os.path.join(ROOT, "tests")]


def main():
    import numpy as np
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
    mdir = f"/tmp/tp_logprob_model_{preset}"
    if local == 0:
        make_model_dir(mdir, preset, seed=1234)
    dist.barrier()
    llm = LLM(mdir, tensor_parallel_size=world, enforce_eager=True, max_model_len=256, max_num_seqs=8,
              max_num_batched_tokens=256, kvcache_block_size=16, num_kvcache_blocks=96)
    rnd = random.Random(4)
    vocab = PRESETS[preset]["vocab_size"]
    pen = dict(repetition_penalty=1.3, presence_penalty=1.5, frequency_penalty=0.5)
    prompts = [[rnd.randint(2, vocab - 1) for _ in range(rnd.randint(4, 60))] for _ in range(10)]
    sps = [SamplingParams(temperature=0.0, max_tokens=12 + i, ignore_eos=True, logprobs=[5, 20, 0][i % 3]) if i % 2 else
           SamplingParams(temperature=0.6, max_tokens=12 + i, ignore_eos=True, top_k=20 if i % 4 else -1,
                          logprobs=None if i == 4 else 3, **(pen if i % 4 == 0 else {}))
           for i in range(10)]
    outs = llm.generate(prompts, sps, use_tqdm=False)
    mine = [(o["token_ids"], [[(t, lp.logprob, lp.rank) for t, lp in d.items()] for d in o.get("logprobs", [])])
            for o in outs]
    gathered = [None] * world
    dist.all_gather_object(gathered, mine)
    if rank == 0:
        assert all(g == mine for g in gathered), "ranks disagree on the tokens or the logprobs"
        from gpu_helpers import make_oracle, oracle_full_logits
        oracle = make_oracle(PRESETS[preset], random_weights(PRESETS[preset], seed=1234), "fused")
        n = 0
        for p, sp, o in zip(prompts, sps, outs):
            assert len(o["token_ids"]) == sp.max_tokens
            assert ("logprobs" in o) == (sp.logprobs is not None)
            if sp.temperature != 0.0:
                continue
            toks = o["token_ids"]
            lg = oracle_full_logits(oracle, p + toks[:-1]).numpy().astype(np.float64)
            for i, (t, d) in enumerate(zip(toks, o["logprobs"])):
                row = lg[len(p) - 1 + i]
                ref = row - row.max() - np.log(np.exp(row - row.max()).sum())
                tol = 6 * 2 ** -8 * np.abs(row).max()
                assert next(iter(d)) == t
                for tid, lp in d.items():
                    assert abs(lp.logprob - ref[tid]) <= tol, (i, tid, lp.logprob, ref[tid])
                n += 1
        print("TP_LOGPROB_RESULT " + json.dumps(dict(world=world, backend=backend, greedy_tokens=n, ok=True)), flush=True)
    llm.exit()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
