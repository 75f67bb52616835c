"""Per-token logprob cost, in one process.

    python profiles/logprobs_bench.py [--rounds 2] [--out profiles/h100_logprobs.json]

1. Each kernel of csrc/logprobs.cu alone (vocab 151 936): top-k + maximum, rank + mass (after the restore has read
   x_sampled) and finish at rows 1 / 16 / 128 / 256 / 512 and k = 0 / 5 / 20; save and restore of 1 024 penalised
   positions per row at k = 5.  Timed as in the decode graph: CUDA events around the replay of a graph of 50 back-to-back
   launches, median of the repetitions, divided by 50.
2. End to end: the benchmark's request mix (bench.py's bench_requests, Qwen3-0.6B-shaped synthetic weights) through one
   engine with CUDA graphs at temperature 0.6, alternating --rounds times: logprobs off, logprobs=0, 5 and 20.  Output
   tokens / device-busy time (CUDA events around each engine step, as bench.py's value) and / CUDA-event time around
   generate(), device-to-host bytes per step, and the engine's host-loop time (loop_stats: total minus the time blocked
   on the GPU).
3. Graph capture: cumulative seconds, the allocator's reserved bytes and the bytes of the graphs' shared private pool
   after each of the three graph sets (--rounds 0 records only this).
The GPU's name and power limit are read in the same run and written beside the numbers.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "nano-vllm_b200"), os.path.join(ROOT, "profiles")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402  (read-only: the request mix and the synthetic model directory)
from penalty_bench import _graph_time  # noqa: E402
from sampling_filter_bench import gpu_info  # noqa: E402


def kernels(reps: int, vocab: int = 151936) -> list:
    from nanovllm import ops
    lib = ops.nat.load()
    out = []
    for rows in (1, 16, 128, 256, 512):
        x = (torch.randn(rows, vocab, device="cuda") * 2.5).to(torch.bfloat16)
        tokens = torch.randint(0, vocab, (rows,), device="cuda")
        ws = ops.logprob_workspace(rows)
        keys = torch.zeros(rows * ops.LOGPROB_MAX_K, dtype=torch.int64, device="cuda")
        res_out = torch.zeros(rows, ops.LOGPROB_OUT_WORDS, dtype=torch.int32, device="cuda")
        for k in (0, 5, 20):
            kk = torch.full((rows,), k, dtype=torch.int32, device="cuda")
            ops.logprobs(x, kk, tokens, workspace=ws)                 # leaves the words a kernel reads valid below

            def topk():
                ops.logprobs_topk(x, kk, ws, keys)

            def rank():
                ops.nat.check(lib.b200_logprob_restore(x.data_ptr(), x.stride(0), kk.data_ptr(), rows, vocab, 0,
                                                       tokens.data_ptr(), ws.data_ptr(), None, 0, ops._stream()))
                ops.nat.check(lib.b200_logprob_rank(x.data_ptr(), x.stride(0), kk.data_ptr(), rows, vocab, ws.data_ptr(),
                                                    ops._stream()))

            def finish():
                ops.nat.check(lib.b200_logprob_finish(kk.data_ptr(), rows, tokens.data_ptr(), keys.data_ptr(), 1,
                                                      ws.data_ptr(), res_out.data_ptr(), res_out[:, 21:].data_ptr(),
                                                      res_out[:, 42:].data_ptr(), res_out.stride(0), ops._stream()))

            res = dict(rows=rows, k=k, topk_us=round(_graph_time(topk, reps), 1),
                       restore_plus_rank_us=round(_graph_time(rank, reps), 1), finish_us=round(_graph_time(finish, reps), 1))
            ws.zero_()
            out.append(res)
            print(json.dumps(res), flush=True)
        # save / restore of 1 024 penalised positions per row (k = 5)
        entries = 1024
        rng = np.random.default_rng(rows)
        hist, lens = ops.penalty_history(rows, entries + 1)
        toks = np.stack([np.sort(rng.choice(vocab, entries, replace=False)) for _ in range(rows)]).astype(np.int64)
        off = torch.arange(0, rows * entries + 1, entries, dtype=torch.int32, device="cuda")
        slots = torch.arange(rows, dtype=torch.int32, device="cuda")
        ops.penalty_load(hist, lens, torch.from_numpy(((toks << 32) | 1).reshape(-1)).cuda(), off, slots)
        saved = ops.logprob_saved_buffer(rows, entries + 1)
        kk = torch.full((rows,), 5, dtype=torch.int32, device="cuda")
        pending = torch.from_numpy(toks[:, 0].copy()).cuda()

        def save():
            ops.logprobs_save(x, kk, ws, saved, hist, lens, slots, pending)

        def restore():
            ops.nat.check(lib.b200_logprob_restore(x.data_ptr(), x.stride(0), kk.data_ptr(), rows, vocab, 0, tokens.data_ptr(),
                                                   ws.data_ptr(), saved.data_ptr(), entries + 1, ops._stream()))

        save_us = _graph_time(save, reps)
        save()
        ws_n = ops.logprob_words(ws, rows, 4, 5).clone()

        def restore_again():                                        # the restore clears the count: put it back each time
            ops.logprob_words(ws, rows, 4, 5).copy_(ws_n)
            restore()
        res = dict(rows=rows, k=5, penalised_entries=entries, save_us=round(save_us, 1),
                   restore_with_1024_saved_us=round(_graph_time(restore_again, reps), 1), note="restore timing includes "
                   "a [rows, 1] int64 copy that re-arms it")
        out.append(res)
        print(json.dumps(res), flush=True)
        del x, hist, saved
        torch.cuda.empty_cache()
    return out


SETTINGS = {"off": None, "logprobs0": 0, "logprobs5": 5, "logprobs20": 20}


def engine(rounds: int, settings: list) -> dict:
    from nanovllm import LLM, SamplingParams
    llm = LLM(bench.ensure_model_dir(0), enforce_eager=False, max_model_len=4096)
    runner = llm.model_runner

    def one_pass(k, name):
        prompts, max_tokens = bench.bench_requests(k)
        lp = SETTINGS[name]
        sps = [SamplingParams(temperature=0.6, ignore_eos=True, max_tokens=mt, **({} if lp is None else dict(logprobs=lp)))
               for mt in max_tokens]
        llm.loop_stats = {"steps": 0, "total_s": 0.0, "wait_s": 0.0}
        runner.begin_profile()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        outs = llm.generate(prompts, sps, use_tqdm=False)
        e1.record()
        torch.cuda.synchronize()
        prof = runner.end_profile()
        st = llm.loop_stats
        tokens = sum(max_tokens)
        assert sum(len(o["token_ids"]) for o in outs) == tokens
        return dict(setting=name, tokens=tokens, device_busy_tok_s=round(tokens / (prof["device_ms"] * 1e-3), 1),
                    e2e_tok_s=round(tokens / (e0.elapsed_time(e1) * 1e-3), 1), engine_steps=prof["engine_steps"],
                    d2h_bytes_per_step=round(prof["d2h_bytes"] / prof["engine_steps"], 1),
                    host_loop_s=round(st["total_s"] - st["wait_s"], 3), loop_total_s=round(st["total_s"], 3))

    if rounds == 0:                                              # capture cost only
        settings = []
    for i, name in enumerate(settings):                          # warm-up passes
        one_pass(1000 + i, name)
    runs = []
    for r in range(rounds):
        for name in settings:
            runs.append(dict(round=r, **one_pass(0, name)))
            print(json.dumps(runs[-1]), flush=True)
    cap = [dict(set=c["set"], cumulative_s=round(c["seconds"], 2), reserved_MiB=round(c["reserved"] / 2**20, 1),
                pool_MiB=round(c["pool"] / 2**20, 1) if "pool" in c else None) for c in getattr(runner, "capture_stats", [])]
    info = dict(kv_blocks=llm.config.num_kvcache_blocks, kernels_plain_bs256=runner.graph_kernels.get(256),
                kernels_second_set_bs256=runner.fgraph_kernels.get(256),
                kernels_third_set_bs256=runner.lgraph_kernels.get(256), capture=cap,
                saved_logits_MiB=round(runner.g_lp_saved.numel() * 8 / 2**20, 1))
    llm.exit()
    return dict(engine=info, runs=runs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2, help="0: build the engine and record its capture cost only")
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--skip-engine", action="store_true")
    ap.add_argument("--skip-kernels", action="store_true")
    ap.add_argument("--settings", default=",".join(SETTINGS), help="comma-separated subset of " + ", ".join(SETTINGS))
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_logprobs.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    os.environ.setdefault("B200_SAMPLE_SEED", "0")
    info = gpu_info()
    print(json.dumps(info), flush=True)
    res = dict(gpu=info, what="per-token logprobs; profiles/logprobs_bench.py",
               kernels=None if args.skip_kernels else kernels(args.reps))
    if not args.skip_engine:
        res["engine"] = engine(args.rounds, args.settings.split(","))
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
