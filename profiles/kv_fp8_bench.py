"""bf16 vs fp8 (e4m3) KV cache on the benchmark workload, in one process.

    python profiles/kv_fp8_bench.py [--rounds 2] [--passes 1] [--out profiles/h100_kv_fp8.json]

1. End to end: the benchmark's request mix (bench.py's bench_requests, Qwen3-0.6B-shaped synthetic weights) through
   LLM.generate() with kv_cache_dtype "auto" and "fp8", alternating, one engine at a time (each in a child process,
   so that it sizes its cache from the whole card) at the default memory utilisation.  Reports output tokens / device-busy time (CUDA events around each engine step, as bench.py's value),
   tokens / CUDA-event time around generate() (bench.py's e2e) and num_kvcache_blocks.
2. The decode attention launch alone at the benchmark's decode batches (profiles/decode_microbench.py's schedule, 28
   layers of distinct KV) for both cache dtypes: microseconds per launch, and bytes/s of the algorithmic K/V bytes of
   each dtype (sum of contexts x 2 x Hkv x D x element size).
3. Greedy agreement with the CPU oracle's fp8 mode: the seven-step model script (tests/kv_fp8_ref.py's oracle) on the
   Qwen3-0.6B shapes, product model with an fp8 cache on the GPU.
The GPU's name and power limit are read in the same run and written beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "nano-vllm_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "profiles")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402  (read-only: the request mix and the synthetic model directory)


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [x.strip() for x in q[0].split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def e2e_arm(mdir: str, dtype: str, passes: int, step0: int) -> dict:
    from nanovllm import LLM, SamplingParams
    t = time.perf_counter()
    llm = LLM(mdir, enforce_eager=False, max_model_len=4096, kv_cache_dtype=dtype)
    init_s = time.perf_counter() - t
    runner = llm.model_runner

    def one_pass(k):
        prompts, max_tokens = bench.bench_requests(k)
        sps = [SamplingParams(temperature=0.6, ignore_eos=True, max_tokens=mt) for mt in max_tokens]
        llm.generate(prompts, sps, use_tqdm=False)
        return sum(max_tokens)

    llm.generate(["t1 t2 t3"], SamplingParams(), use_tqdm=False)
    one_pass(1000 + step0)                                     # warm-up pass
    runner.begin_profile()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    tokens = sum(one_pass(step0 + k) for k in range(passes))
    e1.record()
    torch.cuda.synchronize()
    prof = runner.end_profile()
    row = dict(kv_cache_dtype=dtype, tokens=tokens, device_busy_tok_s=tokens / (prof["device_ms"] * 1e-3),
               e2e_tok_s=tokens / (e0.elapsed_time(e1) * 1e-3), num_kvcache_blocks=llm.config.num_kvcache_blocks,
               kv_block_bytes=runner.kv_block_bytes(), engine_steps=prof["engine_steps"], init_s=round(init_s, 1))
    llm.exit()
    return row


def e2e_child(dtype: str, passes: int) -> dict:
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--arm", dtype, "--passes", str(passes)],
                       capture_output=True, text=True, timeout=1800)
    lines = [l for l in r.stdout.splitlines() if l.startswith("ARM ")]
    assert r.returncode == 0 and lines, r.stdout[-3000:] + r.stderr[-3000:]
    return json.loads(lines[-1][4:])


def decode_launches(layers: int, reps: int, steps=(0, 500, 900, 1020), hq=16, hkv=8) -> list:
    from decode_microbench import schedule_decode_steps
    from nanovllm import ops
    metas = schedule_decode_steps(set(steps))
    nblk, bs = 800, 256
    flush = torch.empty(512 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    for dtype in ("bf16", "fp8"):
        shape = ops.kv_cache_shape(layers, nblk, hkv, bs, 128)
        if dtype == "bf16":
            kv = torch.empty(shape, dtype=torch.bfloat16, device="cuda").normal_()
        else:
            kv = torch.empty(shape, dtype=torch.bfloat16, device="cuda").normal_().to(torch.float8_e4m3fn)
        ops.bind_kv_cache(kv)
        elem = kv.element_size()
        for st in steps:
            a = metas[st]
            n = len(a["context_lens"])
            ctx = torch.from_numpy(a["context_lens"]).cuda()
            bt = torch.from_numpy(np.ascontiguousarray(a["block_tables"])).cuda()
            q = torch.randn(n, hq, 128, device="cuda").to(torch.bfloat16)
            out = torch.empty_like(q)
            for _ in range(2):
                for layer in range(layers):
                    ops.paged_decode(layer, q, bt, ctx, 0.0884, out=out)
            best = 1e9
            for _ in range(reps):
                flush.fill_(1)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for layer in range(layers):
                    ops.paged_decode(layer, q, bt, ctx, 0.0884, out=out)
                e1.record()
                torch.cuda.synchronize()
                best = min(best, e0.elapsed_time(e1) / layers)
            sctx = int(a["context_lens"].sum())
            kv_bytes = sctx * 2 * hkv * 128 * elem
            rows.append(dict(kv=dtype, step=st, batch=n, sum_ctx=sctx, us_per_launch=round(best * 1000, 2),
                             kv_bytes=kv_bytes, kv_GBps=round(kv_bytes / (best * 1e-3) / 1e9, 1)))
            print(json.dumps(rows[-1]), flush=True)
        del kv
        from nanovllm import _native as nat
        nat.handle().kv = None
        torch.cuda.empty_cache()
    return rows


def oracle_agreement(preset: str = "qwen3-0.6b") -> dict:
    from kv_fp8_ref import Qwen3RefFp8, alloc_logical_kv_fp8, oracle_fp8_step_fn
    from nanovllm import ops
    from nanovllm.layers.attention import KVGroup, kv_group_arrays, plan_kv_groups
    from nanovllm.models.qwen3 import Qwen3ForCausalLM
    from nanovllm.utils.context import reset_context, set_context
    from nanovllm.utils.synthetic import PRESETS, hf_config_dict, random_weights
    from oracle.model_script import make_script, run_script
    from oracle.qwen3_ref import RefDims
    weights = random_weights(PRESETS[preset], seed=1234)
    script = make_script(PRESETS[preset]["vocab_size"], max_token=10000)
    hf = SimpleNamespace(**hf_config_dict(PRESETS[preset]))
    model = Qwen3ForCausalLM(hf, 0, 1, "cuda", max_position=4096)
    for name, w in weights.items():
        model.load_hf_tensor(name, w.cuda())
    model.fused_decode_max_batch = 0
    kv8 = torch.zeros(ops.kv_cache_shape(hf.num_hidden_layers, script["num_blocks"], model.num_kv_heads, script["block_size"],
                                         model.head_dim), dtype=torch.uint8, device="cuda").view(torch.float8_e4m3fn)
    ops.bind_kv_cache(kv8)
    scratch = torch.empty(2, 256, model.num_kv_heads, model.head_dim, dtype=torch.bfloat16, device="cuda")
    for i, a in enumerate(model.modules()):
        a.k_cache, a.v_cache, a.layer_id, a.kv_scratch = kv8[0, i], kv8[1, i], i, scratch

    def gpu_step(ids, pos, c):
        groups = None
        if c["is_prefill"] and c.get("block_tables") is not None:
            cq, ck = c["cu_seqlens_q"].cpu().numpy(), c["cu_seqlens_k"].cpu().numpy()
            groups = [KVGroup(*g[:6], torch.from_numpy(g[6]).cuda(), torch.from_numpy(g[7]).cuda())
                      for g in kv_group_arrays(cq, ck, plan_kv_groups(ck, scratch.shape[1]))]
        set_context(c["is_prefill"], c.get("cu_seqlens_q"), c.get("cu_seqlens_k"), c.get("max_seqlen_q", 0),
                    c.get("max_seqlen_k", 0), c.get("slot_mapping"), c.get("context_lens"), c.get("block_tables"), groups)
        out = model.compute_logits(model(ids, pos)).float().cpu()
        reset_context()
        return out

    got = run_script(torch, script, gpu_step, device="cuda")
    oracle = Qwen3RefFp8(RefDims.from_json(hf_config_dict(PRESETS[preset])), weights, rounding="fused", max_pos=4096)
    want = [o.float() for o in run_script(torch, script, oracle_fp8_step_fn(
        oracle, alloc_logical_kv_fp8(oracle.d, script["num_blocks"], script["block_size"])))]
    rows = same = 0
    rel = []
    for g, w in zip(got, want):
        rel.append(((g - w).norm() / w.norm()).item())
        same += int((g.argmax(-1) == w.argmax(-1)).sum())
        rows += g.shape[0]
    return dict(preset=preset, steps=len(got), greedy_rows=rows, greedy_same_as_fp8_oracle=same,
                logits_rel_l2_per_step=[round(r, 5) for r in rel])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2, help="bf16 / fp8 alternations of the end-to-end runs")
    ap.add_argument("--passes", type=int, default=1, help="timed passes of the request mix per engine")
    ap.add_argument("--layers", type=int, default=28)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_kv_fp8.json"))
    ap.add_argument("--arm", default=None, help=argparse.SUPPRESS)         # child: one end-to-end arm
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    os.environ.setdefault("B200_SAMPLE_SEED", "0")
    if args.arm:
        print("ARM " + json.dumps(e2e_arm(bench.ensure_model_dir(0), args.arm, args.passes, 0)), flush=True)
        return
    info = gpu_info()
    print(json.dumps(info), flush=True)
    bench.ensure_model_dir(0)                                  # built once, before the children
    e2e = []
    for r in range(args.rounds):
        for dtype in ("auto", "fp8"):
            e2e.append(dict(round=r, **e2e_child(dtype, args.passes)))
            print(json.dumps(e2e[-1]), flush=True)
    launches = decode_launches(args.layers, args.reps)
    agree = oracle_agreement()
    print(json.dumps(agree), flush=True)
    res = dict(gpu=info, what="bf16 vs fp8 (e4m3, unit scales) KV cache; profiles/kv_fp8_bench.py", e2e=e2e,
               decode_launch=launches, oracle_fp8_agreement=agree)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
