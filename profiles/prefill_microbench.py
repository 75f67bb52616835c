"""Prefill attention kernel alone on the benchmark's prefill shapes (packed, causal, Hq16/Hkv8/D128).

    B200_PREFILL=tc|ws python profiles/prefill_microbench.py [--paged]

Sequence lengths are those of the benchmark's first prefill step (31 prompts, 15 705 tokens).
FLOPs = sum_s 4 * Hq * D * (len_q*len_k - len_q^2/2)   (SURVEY.md 8d).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "nano-vllm_b200")]

import torch  # noqa: E402

import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paged", action="store_true")
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    from nanovllm import ops
    prompts, _ = bench.bench_requests(0)
    lens, tot = [], 0
    for p in prompts:
        if tot + len(p) > 16384:
            break
        lens.append(len(p))
        tot += len(p)
    hq, hkv, d = 16, 8, 128
    qkv = torch.randn(tot, (hq + 2 * hkv) * d, device="cuda").to(torch.bfloat16)
    q = qkv[:, :hq * d].view(tot, hq, d)
    k = qkv[:, hq * d:(hq + hkv) * d].view(tot, hkv, d)
    v = qkv[:, (hq + hkv) * d:].view(tot, hkv, d)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device="cuda")
    flops = sum(4 * hq * d * (l * l - l * l / 2) for l in lens)
    kw = {}
    if args.paged:
        bs = 256
        nblk = sum((l + bs - 1) // bs for l in lens)
        kv = torch.randn(ops.kv_cache_shape(1, nblk, hkv, bs, d), device="cuda").to(torch.bfloat16)
        ops.bind_kv_cache(kv)
        bt = torch.full((len(lens), max((l + bs - 1) // bs for l in lens)), -1, dtype=torch.int32)
        u = 0
        for i, l in enumerate(lens):
            n = (l + bs - 1) // bs
            bt[i, :n] = torch.arange(u, u + n, dtype=torch.int32)
            u += n
        kw = dict(block_tables=bt.cuda(), num_kv_heads=hkv)
    out = torch.empty_like(q)
    for _ in range(3):
        ops.paged_prefill(0, q, k, v, cu, cu, max(lens), max(lens), d ** -0.5, out=out, **kw)
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ops.paged_prefill(0, q, k, v, cu, cu, max(lens), max(lens), d ** -0.5, out=out, **kw)
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    print(json.dumps(dict(impl=os.environ.get("B200_PREFILL", "tc"), paged=args.paged, seqs=len(lens), tokens=tot, us=best * 1000,
                          tflops=flops / (best * 1e-3) / 1e12)))


if __name__ == "__main__":
    main()
