"""Does a wgmma projection chain hide under the decode-attention kernel of ANOTHER stream on the same SMs?

    python profiles/dual_microbench.py [rows per half, default 128] [ring slots, default 3]

Times, per layer (CUDA events, graph replay of 28 layers, median of 20 replays), on Qwen3-0.6B shapes and the benchmark's
batch-256 context mix cut in two:
  attn     b200_paged_decode_fused of one half batch alone
  chain    the six non-attention kernels of one half batch alone (add+norm, qkv, o split-K, add+norm, gate_up+SiluAndMul,
           down split-K; wgmma with the given ring depth)
  both     the two on two streams at once (what one phase of the two-stream decode step does)
`both` ~ max(attn, chain) means the chain's CTAs do share the SMs with the attention CTAs; `both` ~ attn + chain means
they do not (shared memory / registers / carve-out) and the two-stream step cannot win.
"""
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "nano-vllm_b200")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402


def main():
    rows = int(sys.argv[1]) if len(sys.argv) > 1 else 128
    ring = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    cfgs = sys.argv[3] if len(sys.argv) > 3 else "64,64,64,8,64,8"
    bn_qkv, bn_gu, bn_o, s_o, bn_d, s_d = [int(v) for v in cfgs.split(",")]
    from nanovllm import ops
    from nanovllm.layers.rotary_embedding import build_cos_sin
    L, hq, hkv, d, hidden, inter, bs = 28, 16, 8, 128, 1024, 3072, 256
    prompts, _ = bench.bench_requests(0)
    lens = [len(p) + 1 for p in prompts][:rows]
    nblk = sum((c + bs - 1) // bs for c in lens)
    kv = torch.empty(ops.kv_cache_shape(L, nblk, hkv, bs, d), dtype=torch.bfloat16, device="cuda").normal_()
    ops.bind_kv_cache(kv)
    bt = torch.full((rows, 8), -1, dtype=torch.int32)
    u = 0
    for i, c in enumerate(lens):
        n = (c + bs - 1) // bs
        bt[i, :n] = torch.arange(u, u + n, dtype=torch.int32)
        u += n
    bt, ctx = bt.cuda(), torch.tensor(lens, dtype=torch.int32).cuda()
    dev = "cuda"
    rnd = lambda *s: (torch.randn(*s, device=dev) * 0.05).to(torch.bfloat16)
    W = [dict(qkv=rnd((hq + 2 * hkv) * d, hidden), o=rnd(hidden, hq * d), gu=rnd(2 * inter, hidden), down=rnd(hidden, inter))
         for _ in range(L)]
    ln = torch.ones(hidden, device=dev, dtype=torch.bfloat16)
    qn = torch.ones(d, device=dev, dtype=torch.bfloat16)
    cs = build_cos_sin(d, 4096, 1e6, dev)
    qkv_in = rnd(rows, (hq + 2 * hkv) * d)
    o_in = rnd(rows, hq * d)
    residual = rnd(rows, hidden)
    out_attn = torch.empty(rows, hq, d, device=dev, dtype=torch.bfloat16)

    def attn_layers():
        with ops.pdl_off():
            for li in range(L):
                ops.paged_decode_fused(li, qkv_in, hq, qn, qn, cs, 1e-6, bt, ctx, d ** -0.5, out=out_attn)

    def chain_layers():
        parts = None
        for li in range(L):
            w = W[li]
            if parts is None:
                x = ops.rmsnorm(residual, ln, 1e-6)
            else:
                x, _ = ops.add_rmsnorm_partials(parts, residual, ln, 1e-6, pdl=True)
            ops.linear(x, w["qkv"], ops.EPI_BF16, bn_qkv, pdl=True, stages=ring)
            parts = ops.linear(o_in, w["o"], ops.EPI_PARTIAL, bn_o, s_o, pdl=False, stages=ring)
            x, _ = ops.add_rmsnorm_partials(parts, residual, ln, 1e-6, pdl=True)
            act = ops.linear(x, w["gu"], ops.EPI_SILU, bn_gu, pdl=True, stages=ring)
            parts = ops.linear(act, w["down"], ops.EPI_PARTIAL, bn_d, s_d, pdl=True, stages=ring)

    side = torch.cuda.Stream()

    def both():
        main = torch.cuda.current_stream()
        ev = torch.cuda.Event()
        ev.record(main)
        side.wait_event(ev)
        with torch.cuda.stream(side):
            chain_layers()
        attn_layers()
        ev2 = torch.cuda.Event()
        ev2.record(side)
        main.wait_event(ev2)

    res = {"rows": rows, "ring_slots": ring, "cfg": cfgs, "sum_ctx": int(sum(lens)), "unit": "us per layer"}
    for name, fn in (("attn", attn_layers), ("chain", chain_layers), ("both", both)):
        fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        g.replay()
        torch.cuda.synchronize()
        ts = []
        for _ in range(20):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1000.0 / L)
        res[name] = round(statistics.median(ts), 2)
    res["kv_GBps_alone"] = round(sum(lens) * 2 * hkv * d * 2 / (res["attn"] * 1e-6) / 1e9, 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
