"""BASELINE.json configs[2] sanity + timing: Qwen3-8B dims (random init), block_size=16, prefix cache on, one GPU.

    NANOVLLM_ALLOW_RANDOM_INIT=1 python profiles/config3_8b.py [num_seqs] [max_tokens]

Requests share a 600-token prefix (so all but the first admitted batch hit the prefix cache: paged prefill with
len_q < len_k over 16-token pages), greedy, and a sample of the outputs is checked for internal consistency
(same prompt => same completion).  Prints one JSON line.
"""
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "nano-vllm_b200")]
os.environ.setdefault("NANOVLLM_ALLOW_RANDOM_INIT", "1")


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 192
    max_tokens = int(sys.argv[2]) if len(sys.argv) > 2 else 48
    import torch
    from nanovllm import LLM, SamplingParams
    from nanovllm.utils.synthetic import make_model_dir
    mdir = make_model_dir("/tmp/b200_models/qwen3-8b", "qwen3-8b", weights=False)
    t0 = time.time()
    llm = LLM(mdir, kvcache_block_size=16, max_model_len=4096, max_num_seqs=256, gpu_memory_utilization=0.85)
    init_s = time.time() - t0
    rnd = random.Random(0)
    prefix = [rnd.randint(2, 150000) for _ in range(600)]
    prompts = [prefix + [rnd.randint(2, 150000) for _ in range(rnd.randint(8, 200))] for _ in range(n - 2)]
    prompts += [list(prompts[0]), list(prompts[1])]                  # duplicates: must reproduce their twins
    sps = [SamplingParams(temperature=0.0, max_tokens=max_tokens, ignore_eos=True)] * n
    llm.generate(prompts[:4], sps[:4], use_tqdm=False)               # warm-up (also seeds the prefix cache)
    torch.cuda.synchronize()
    t = time.time()
    outs = llm.generate(prompts, sps, use_tqdm=False)
    torch.cuda.synchronize()
    dt = time.time() - t
    bm = llm.scheduler.block_manager
    def agree(a, b):                      # leading tokens on which two runs of the same prompt agree
        k = 0
        while k < len(a) and a[k] == b[k]:
            k += 1
        return k
    # identical prompts served in different batches (one of them through the prefix cache): with random-init
    # weights the logits are nearly flat, so a one-ulp difference between batch shapes can flip an argmax;
    # the agreement length is reported, not asserted
    same = [agree(outs[0]["token_ids"], outs[-2]["token_ids"]), agree(outs[1]["token_ids"], outs[-1]["token_ids"])]
    print(json.dumps({"config": "Qwen3-8B dims random-init bf16, block_size 16, prefix cache, 1 GPU", "seqs": n,
                      "max_tokens": max_tokens, "output_tok_s": n * max_tokens / dt, "seconds": dt, "init_s": init_s,
                      "kv_blocks": llm.config.num_kvcache_blocks, "cached_hashes": len(bm.hash_to_block_id),
                      "duplicate_prompt_agreement_tokens": same}))
    llm.exit()


if __name__ == "__main__":
    main()
