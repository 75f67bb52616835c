"""BASELINE.json configs[2..4] end to end through the public API, one process per GPU.

    python profiles/run_config.py 3                                   # Qwen3-8B, 512 seqs, block 16, prefix cache, 1 GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 4 --master-addr 127.0.0.1 --master-port 29640 profiles/run_config.py 4
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29650 profiles/run_config.py 5

  3  Qwen3-8B dims, 512 requests sharing a 600-token prefix + U[8,200] own tokens, 128 output tokens, kvcache_block_size 16
     (prefix cache: all but the first admitted batch take the paged-prefill path with len_q < len_k over 16-token pages)
  4  Qwen3-8B dims, tensor_parallel_size 4, 1 024 requests in/out U[100,1024] (the bench mix, twice as many): at most 512
     run at a time, so prefill and decode steps interleave as requests are admitted
  5  Qwen3-32B dims, tensor_parallel_size 8, 128 requests of 8 192 prompt tokens and 1 024 output tokens, max_model_len 9 472

Weights are random-init drawn on the device (utils/loader.py: one well-defined full model, each rank keeps its shard); there
are no checkpoints offline.  Prints one JSON line (rank 0) and, with an output path as second argument, writes it there:
throughput (wall clock around generate(), after a warm-up generate), the decode kernel's GB/s on this run's own decode
shapes (CUDA events, rank 0's shard), KV sizing, and a parity leg: greedy requests whose tokens must agree (a) between
all ranks, (b) between twin prompts served in different batches / through the prefix cache, and (c) -- configs 3 and 4 use
the same model and the same greedy prompts -- between the 1-GPU run and the TP4 run (tokens of config 3 are saved to
gpurun_out/r02_config3_greedy_tokens.json, committed as profiles/r02_config3_greedy_tokens.json and compared by config 4).
"""
import json
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "nano-vllm_b200")]
os.environ.setdefault("NANOVLLM_ALLOW_RANDOM_INIT", "1")
GREEDY_FILE = os.path.join(ROOT, "profiles", "r02_config3_greedy_tokens.json")          # committed copy, read by config 4
GREEDY_OUT = os.path.join(ROOT, "gpurun_out", "r02_config3_greedy_tokens.json")          # written by config 3 (gpurun merges gpurun_out/ back)


def requests_for(cfg: int):
    rnd = random.Random(0)
    if cfg == 3:
        prefix = [rnd.randint(2, 150000) for _ in range(600)]
        prompts = [prefix + [rnd.randint(2, 150000) for _ in range(rnd.randint(8, 200))] for _ in range(512)]
        return prompts, [128] * 512
    if cfg == 4:
        prompts = [[rnd.randint(0, 10000) for _ in range(rnd.randint(100, 1024))] for _ in range(1024)]
        return prompts, [rnd.randint(100, 1024) for _ in range(1024)]
    prompts = [[rnd.randint(0, 150000) for _ in range(8192)] for _ in range(128)]
    return prompts, [1024] * 128


def greedy_requests():
    """The shared greedy parity prompts of configs 3 and 4 (same model, same prompts -> same tokens expected)."""
    rnd = random.Random(77)
    base = [[rnd.randint(2, 150000) for _ in range(rnd.randint(30, 400))] for _ in range(6)]
    return base + [list(base[0]), list(base[1])]           # twins: served in another row of the batch


def agree_len(a, b):
    k = 0
    while k < min(len(a), len(b)) and a[k] == b[k]:
        k += 1
    return k


def main():
    cfg = int(sys.argv[1])
    out_path = sys.argv[2] if len(sys.argv) > 2 else None
    import torch
    import torch.distributed as dist
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    assert world == {3: 1, 4: 4, 5: 8}[cfg] or os.environ.get("RUN_CONFIG_ANY_WORLD"), f"config {cfg} runs on {({3: 1, 4: 4, 5: 8}[cfg])} GPUs"
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from nanovllm import LLM, SamplingParams
    from nanovllm.utils.synthetic import make_model_dir
    preset = "qwen3-32b" if cfg == 5 else "qwen3-8b"
    mdir = f"/tmp/b200_models/{preset}"
    if local == 0:
        make_model_dir(mdir, preset, weights=False)
    if world > 1:
        dist.barrier()
    kw = {3: dict(kvcache_block_size=16, max_model_len=4096, max_num_seqs=512),
          4: dict(max_model_len=4096, max_num_seqs=512),
          5: dict(max_model_len=9472, max_num_seqs=128)}[cfg]
    t0 = time.time()
    llm = LLM(mdir, tensor_parallel_size=world, **kw)
    init_s = time.time() - t0
    runner = llm.model_runner
    m = runner.model
    prompts, max_tokens = requests_for(cfg)
    sps = [SamplingParams(temperature=0.6, max_tokens=mt, ignore_eos=True) for mt in max_tokens]

    # warm-up: a small slice of the workload (different token values, so nothing lands in the prefix cache of the run)
    wn = {3: 16, 4: 32, 5: 2}[cfg]
    warm = [[(t + 7) % 150001 for t in p] for p in prompts[:wn]]
    llm.generate(warm, [SamplingParams(temperature=0.6, max_tokens=8, ignore_eos=True)] * wn, use_tqdm=False)

    def sync():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize()

    runner.begin_profile()
    sync()
    t = time.time()
    outs = llm.generate(prompts, sps, use_tqdm=False)
    sync()
    dt = time.time() - t
    prof = runner.end_profile()
    assert [len(o["token_ids"]) for o in outs] == max_tokens
    bm = llm.scheduler.block_manager
    cached_hashes = len(bm.hash_to_block_id)

    # ---- parity leg -------------------------------------------------------------------------------------------
    parity = {}
    if cfg in (3, 4):
        gp = greedy_requests()
        gs = [SamplingParams(temperature=0.0, max_tokens=16, ignore_eos=True)] * len(gp)
        g1 = [o["token_ids"] for o in llm.generate(gp, gs, use_tqdm=False)]
        g2 = [o["token_ids"] for o in llm.generate(gp[:3], gs[:3], use_tqdm=False)]      # again: now through the prefix cache
        parity["twin_prompt_agreement_tokens_of_16"] = [agree_len(g1[0], g1[6]), agree_len(g1[1], g1[7])]
        parity["prefix_cache_rerun_agreement_tokens_of_16"] = [agree_len(a, b) for a, b in zip(g1[:3], g2)]
        toks = g1
    else:
        gp = [prompts[0][:3000], prompts[1][:777], prompts[0][:3000]]
        gs = [SamplingParams(temperature=0.0, max_tokens=12, ignore_eos=True)] * 3
        toks = [o["token_ids"] for o in llm.generate(gp, gs, use_tqdm=False)]
        parity["twin_prompt_agreement_tokens_of_12"] = [agree_len(toks[0], toks[2])]
    if world > 1:
        gathered = [None] * world
        dist.all_gather_object(gathered, toks)
        parity["ranks_agree"] = all(g == toks for g in gathered)
        parity["ranks"] = world
        peer = getattr(m, "peer", None)
        parity["tp_exchange"] = "nccl" if peer is None else ("nvls" if peer.nvls else "peer-memory kernel")
    if rank == 0 and cfg == 3:
        os.makedirs(os.path.dirname(GREEDY_OUT), exist_ok=True)
        with open(GREEDY_OUT, "w") as f:
            json.dump({"what": "greedy tokens of profiles/run_config.py greedy_requests() on Qwen3-8B dims, 1 GPU", "tokens": toks}, f)
    if rank == 0 and cfg == 4 and os.path.exists(GREEDY_FILE):
        ref = json.load(open(GREEDY_FILE))["tokens"]
        parity["tp4_vs_1gpu_agreement_tokens_of_16"] = [agree_len(a, b) for a, b in zip(toks, ref)]
        parity["tp4_vs_1gpu_note"] = ("same model (seeded on-device init), same prompts; with random-init weights the logits are nearly "
                                      "flat, so one differently-rounded all-reduce can flip an argmax and everything after it")

    roof = None
    if rank == 0:
        import bench
        every = {3: 16, 4: 96, 5: 64}[cfg]
        roof = bench.decode_roofline(llm, sample_every=every, requests=(prompts, max_tokens))
    if rank == 0:
        hf = llm.config.hf_config
        line = {
            "config": {3: "Qwen3-8B dims random-init bf16, 512 seqs, kvcache_block_size 16, shared 600-token prefix (prefix cache on), 1 GPU",
                       4: "Qwen3-8B dims random-init bf16, tensor_parallel_size 4, 1024 seqs in/out U[100,1024], max_num_seqs 512 (mixed prefill+decode)",
                       5: "Qwen3-32B dims random-init bf16, tensor_parallel_size 8, 128 seqs, 8192-token prompts, 1024 output tokens, max_model_len 9472"}[cfg],
            "n_gpus": world, "output_tokens": sum(max_tokens), "prompt_tokens": sum(len(p) for p in prompts),
            "seconds": dt, "output_tok_s": sum(max_tokens) / dt, "total_tok_s": (sum(max_tokens) + sum(len(p) for p in prompts)) / dt,
            "device_busy_s": prof["device_ms"] / 1e3, "engine_steps": prof["engine_steps"], "kernel_launches": prof["kernel_launches"],
            "init_s": round(init_s, 1), "kv_blocks": llm.config.num_kvcache_blocks, "kvcache_block_size": llm.config.kvcache_block_size,
            "block_table_width": runner.max_blocks, "cached_hashes_after_run": cached_hashes,
            "q_heads_per_kv_head": hf.num_attention_heads // hf.num_key_value_heads, "kv_heads_per_rank": m.num_kv_heads,
            "decode_kernel": roof, "parity": parity,
        }
        print(json.dumps(line))
        if out_path:
            with open(out_path, "w") as f:
                json.dump(line, f, indent=1)
    llm.exit()
    if world > 1 and dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
