"""Mixture-of-experts MLP on one H100, in one call (DESIGN.md 3.7).

    python profiles/moe_bench.py [--out profiles/h100_moe.json] [--skip-e2e]

(a) Kernels at Qwen3-30B-A3B dimensions (128 experts, top 8, hidden 2048, moe_intermediate_size 768) for T tokens: the two
    grouped wgmma GEMMs (gate_up + SiluAndMul, down) on a fixed routing, the whole MoE MLP (route, align, gather, the two
    GEMMs, combine), and a per-expert loop of cuBLAS F.linear + silu_mul + F.linear over the same permuted rows.  Routing
    from random bf16 router logits of std 2.  CUDA events around a CUDA graph of back-to-back calls, median of 5 replays.
    Decode sizes report distinct expert-weight bytes over time against 3.35 TB/s, prefill sizes FLOP/s against 989 TFLOP/s
    (H100 SXM data-sheet figures, dense bf16).
(b) End to end: bench.py's request mix through LLM.generate() on a random-init qwen3-30b-a3b directory at TP1, in a child
    process (it sizes its KV cache from the whole card): output tokens / s and num_kvcache_blocks.
The GPU's name and power limit are read in the same run and written beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "nano-vllm_b200"), os.path.join(ROOT, "profiles")]

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import bench  # noqa: E402  (read-only: the request mix)

HBM_TBPS, BF16_TFLOPS = 3.35, 989.0
TOKENS = [1, 8, 32, 128, 256, 512, 2048, 8192, 16384]
PRESET = "qwen3-30b-a3b"


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [x.strip() for x in q[0].split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def timed(fn, reps: int, windows: int = 5) -> float:
    """Median over `windows` of the mean device time of `reps` back-to-back calls captured in one CUDA graph, in seconds."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    out = []
    for _ in range(windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) * 1e-3 / reps)
    del g
    return sorted(out)[len(out) // 2]


def kernels() -> list:
    from nanovllm import ops
    from nanovllm.utils.synthetic import PRESETS
    d = PRESETS[PRESET]
    E, k, H, I = d["num_experts"], d["num_experts_per_tok"], d["hidden_size"], d["moe_intermediate_size"]
    g = torch.Generator(device="cuda").manual_seed(0)
    gu = (0.02 * torch.randn(E, 2 * I, H, generator=g, device="cuda")).to(torch.bfloat16)
    dn = (0.02 * torch.randn(E, H, I, generator=g, device="cuda")).to(torch.bfloat16)
    rows = []
    for T in TOKENS:
        x = torch.randn(T, H, generator=g, device="cuda").to(torch.bfloat16)
        lg = (2.0 * torch.randn(T, E, generator=g, device="cuda")).to(torch.bfloat16)
        ids, w = ops.moe_route(lg, k, True)
        perm, tiles = ops.moe_align(ids, E)
        xp = ops.moe_gather(x, k, perm)
        act = torch.empty(T * k, I, dtype=torch.bfloat16, device="cuda")
        y = torch.empty(T * k, H, dtype=torch.bfloat16, device="cuda")
        out = torch.empty(T, H, dtype=torch.bfloat16, device="cuda")
        counts = torch.bincount(ids.reshape(-1).long(), minlength=E).tolist()
        starts = [sum(counts[:e]) for e in range(E)]
        used = [e for e in range(E) if counts[e]]

        def grouped():
            ops.moe_linear(xp, gu, tiles, ops.EPI_SILU, 64, pdl=True, out=act)
            ops.moe_linear(act, dn, tiles, ops.EPI_BF16, 64, pdl=True, out=y)

        def full():
            ops.moe_mlp(x, lg, gu, dn, k, True, out=out)

        def loop():
            for e in used:
                s, n = starts[e], counts[e]
                torch.mm(ops.silu_mul(F.linear(xp[s:s + n], gu[e])), dn[e].t(), out=y[s:s + n])

        reps = 20 if T <= 512 else 3
        tg, tf, tl = timed(grouped, reps), timed(full, reps), timed(loop, max(1, reps // 4))
        wbytes = len(used) * 3 * H * I * 2
        flop = 2.0 * T * k * 3 * H * I
        row = dict(T=T, experts_used=len(used), grouped_gemms_us=tg * 1e6, moe_mlp_us=tf * 1e6, per_expert_cublas_loop_us=tl * 1e6,
                   speedup_vs_loop=tl / tg)
        if T <= 512:
            row.update(expert_weight_TBps=wbytes / tg / 1e12, share_of_hbm_datasheet=wbytes / tg / 1e12 / HBM_TBPS,
                       loop_expert_weight_TBps=wbytes / tl / 1e12)
        else:
            row.update(TFLOPs=flop / tg / 1e12, share_of_bf16_datasheet=flop / tg / 1e12 / BF16_TFLOPS, loop_TFLOPs=flop / tl / 1e12)
        rows.append(row)
        print(json.dumps(row), flush=True)
        del x, lg, xp, act, y, out
        torch.cuda.empty_cache()
    return rows


def e2e_arm() -> dict:
    os.environ["NANOVLLM_ALLOW_RANDOM_INIT"] = "1"
    from nanovllm import LLM, SamplingParams
    from nanovllm.utils.synthetic import make_model_dir
    path = make_model_dir(os.path.join(tempfile.gettempdir(), f"b200_moebench_{os.getuid()}", PRESET), PRESET, seed=0, weights=False)
    t = time.perf_counter()
    llm = LLM(path, enforce_eager=False, max_model_len=4096)
    init_s = time.perf_counter() - t
    prompts, max_tokens = bench.bench_requests(0)
    sps = [SamplingParams(temperature=0.6, ignore_eos=True, max_tokens=mt) for mt in max_tokens]
    llm.generate(prompts[:16], sps[:16], use_tqdm=False)                # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    llm.generate(prompts, sps, use_tqdm=False)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    row = dict(preset=PRESET, tp=1, requests=len(prompts), output_tokens=sum(max_tokens), output_tok_s=sum(max_tokens) / dt,
               seconds=dt, num_kvcache_blocks=llm.config.num_kvcache_blocks, weight_gb=torch.cuda.memory_allocated() / 1e9,
               init_s=round(init_s, 1))
    llm.exit()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_moe.json"))
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--arm", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    os.environ.setdefault("B200_SAMPLE_SEED", "0")
    if args.arm:
        print("ARM " + json.dumps(e2e_arm()), flush=True)
        return
    info = gpu_info()
    print(json.dumps(info), flush=True)
    res = dict(gpu=info, what="Qwen3-30B-A3B MoE MLP: grouped wgmma GEMMs vs a per-expert cuBLAS loop; profiles/moe_bench.py")
    res["kernels"] = kernels()
    if not args.skip_e2e:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--arm"], capture_output=True, text=True, timeout=2400)
        lines = [l for l in r.stdout.splitlines() if l.startswith("ARM ")]
        res["e2e"] = json.loads(lines[-1][4:]) if r.returncode == 0 and lines else dict(error=r.stdout[-1500:] + r.stderr[-1500:])
        print(json.dumps(res["e2e"]), flush=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
