"""Top-k / top-p / min-p sampling cost, in one process.

    python profiles/sampling_filter_bench.py [--rounds 2] [--out profiles/h100_sampling_filters.json]

1. Kernels alone: stages 0-3 and the masked race of ops.sample_filtered against ops.sample (b200_sample) at rows
   1 / 16 / 128 / 256 / 512, vocab 151 936, Qwen3's recommended setting (t 0.6, top_p 0.95, top_k 20) on every row,
   CUDA events per launch (median of the repetitions).  GB/s = algorithmic bytes (launches that read the row x rows x
   vocab x 2 B) / time.
2. End to end: the benchmark's request mix (bench.py's bench_requests, Qwen3-0.6B-shaped synthetic weights) through one
   engine at temperature 0.6, without and with top_p=0.95, top_k=20, alternating --rounds times.  Output tokens /
   device-busy time (CUDA events around each engine step, as bench.py's value) and / CUDA-event time around generate().
3. Capture cost of that engine: time in capture_cudagraph (both graph sets) and the graph pool's memory.
The GPU's name and power limit are read in the same run and written beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "nano-vllm_b200"), os.path.join(ROOT, "profiles")]

import torch  # noqa: E402

import bench  # noqa: E402  (read-only: the request mix and the synthetic model directory)


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [x.strip() for x in q[0].split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def _time(fn, reps):
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1000)
    ts.sort()
    return ts[len(ts) // 2]


def kernels(reps: int, vocab: int = 151936) -> list:
    from nanovllm import ops
    out = []
    for rows in (1, 16, 128, 256, 512):
        g = (torch.randn(rows, vocab, device="cuda") * 2.5).to(torch.bfloat16)
        t = torch.full((rows,), 0.6, device="cuda")
        k = torch.full((rows,), 20, dtype=torch.int32, device="cuda")
        p = torch.full((rows,), 0.95, device="cuda")
        mp = torch.zeros(rows, device="cuda")
        ws = ops.filter_workspace(rows)
        tok = torch.empty(rows, dtype=torch.int64, device="cuda")
        for _ in range(3):
            ops.sample_filtered(g, t, k, p, mp, 1, 1, ws, out=tok)
            ops.sample(g, t, 1, 1, out=tok)
        torch.cuda.synchronize()
        stage_us = [_time(lambda s=s: ops.sample_filter_stage(s, g, t, k, p, mp, ws), reps) for s in range(4)]
        race_us = _time(lambda: ops.sample_filter_race(g, t, k, p, mp, 1, 1, ws, out=tok), reps)
        total_us = _time(lambda: ops.sample_filtered(g, t, k, p, mp, 1, 1, ws, out=tok), reps)
        plain_us = _time(lambda: ops.sample(g, t, 1, 1, out=tok), reps)
        row_bytes = rows * vocab * 2
        r = dict(rows=rows, vocab=vocab, stage_us=[round(x, 1) for x in stage_us], race_us=round(race_us, 1),
                 filtered_total_us=round(total_us, 1), plain_sample_us=round(plain_us, 1),
                 filtered_GBps=round(5 * row_bytes / (total_us * 1e-6) / 1e9, 1),
                 plain_GBps=round(row_bytes / (plain_us * 1e-6) / 1e9, 1))
        out.append(r)
        print(json.dumps(r), flush=True)
        del g, ws
        torch.cuda.empty_cache()
    return out


def engine(rounds: int) -> dict:
    from nanovllm import LLM, SamplingParams
    from nanovllm.engine.model_runner import ModelRunner
    cap = {}
    orig = ModelRunner.capture_cudagraph

    def timed_capture(self):
        torch.cuda.synchronize()
        m0 = torch.cuda.memory_reserved()
        t0 = time.perf_counter()
        orig(self)
        torch.cuda.synchronize()
        cap.update(capture_s=round(time.perf_counter() - t0, 2), pool_reserved_MiB=round((torch.cuda.memory_reserved() - m0) / 2**20, 1),
                   graphs_plain=len(self.graphs), graphs_filtered=len(self.fgraphs),
                   kernels_plain_bs256=self.graph_kernels.get(256), kernels_filtered_bs256=self.fgraph_kernels.get(256))

    ModelRunner.capture_cudagraph = timed_capture
    llm = LLM(bench.ensure_model_dir(0), enforce_eager=False, max_model_len=4096)
    ModelRunner.capture_cudagraph = orig
    runner = llm.model_runner

    def one_pass(k, filtered):
        prompts, max_tokens = bench.bench_requests(k)
        extra = dict(top_p=0.95, top_k=20) if filtered else {}
        sps = [SamplingParams(temperature=0.6, ignore_eos=True, max_tokens=mt, **extra) for mt in max_tokens]
        runner.begin_profile()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        llm.generate(prompts, sps, use_tqdm=False)
        e1.record()
        torch.cuda.synchronize()
        prof = runner.end_profile()
        tokens = sum(max_tokens)
        return dict(filtered=filtered, tokens=tokens, device_busy_tok_s=round(tokens / (prof["device_ms"] * 1e-3), 1),
                    e2e_tok_s=round(tokens / (e0.elapsed_time(e1) * 1e-3), 1), engine_steps=prof["engine_steps"])

    one_pass(1000, False)
    one_pass(1001, True)                                         # warm-up passes
    runs = []
    for r in range(rounds):
        for filtered in (False, True):
            runs.append(dict(round=r, **one_pass(0, filtered)))
            print(json.dumps(runs[-1]), flush=True)
    llm.exit()
    return dict(capture=cap, runs=runs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--skip-engine", action="store_true")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_sampling_filters.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    os.environ.setdefault("B200_SAMPLE_SEED", "0")
    info = gpu_info()
    print(json.dumps(info), flush=True)
    res = dict(gpu=info, what="top-k / top-p / min-p sampling; profiles/sampling_filter_bench.py", kernels=kernels(args.reps))
    if not args.skip_engine:
        res["engine"] = engine(args.rounds)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
