"""Staged wgmma linear (csrc/linear_tc.cu) against the library path it would replace, at Qwen3-0.6B decode shapes.

    python profiles/linear_microbench.py > linear_microbench.json

A configuration the library refuses (unsupported shape) is recorded as null; results are flushed per batch size.

Each measurement is one CUDA-graph replay of the op over 16 distinct weight sets (more bytes than the 50 MB L2 for the
large shapes, as in a real step where every layer has its own weights), CUDA events around the replay, best of 5.
"""
import itertools
import json
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, "nano-vllm_b200")
from nanovllm import ops  # noqa: E402

NSETS = 16
HID, INTER, QKV, OIN = 1024, 3072, 4096, 2048


def timed(fn_per_set, nsets=NSETS):
    try:
        return _timed(fn_per_set, nsets)
    except Exception as e:                      # e.g. an unsupported tile / cluster combination
        print(f"skipped: {type(e).__name__}: {str(e)[:80]}", file=sys.stderr, flush=True)
        return None


def _timed(fn_per_set, nsets):
    for i in range(nsets):
        fn_per_set(i)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(nsets):
            fn_per_set(i)
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) / nsets)
    return round(best * 1000, 2)


def rnd(*shape):
    return torch.randn(*shape, device="cuda").to(torch.bfloat16)


res = {}
for M in (256, 128, 64, 16, 1):
    r = {}
    x_h = rnd(M, HID); x_o = rnd(M, OIN); x_i = rnd(M, INTER)
    w_qkv = [rnd(QKV, HID) for _ in range(NSETS)]
    w_o = [rnd(HID, OIN) for _ in range(NSETS)]
    w_gu = [rnd(2 * INTER, HID) for _ in range(NSETS)]
    w_dn = [rnd(HID, INTER) for _ in range(NSETS)]
    resid = rnd(M, HID); wn = torch.ones(HID, dtype=torch.bfloat16, device="cuda")

    r["qkv_cublas"] = timed(lambda i: F.linear(x_h, w_qkv[i]))
    for bn, pdl, sh in itertools.product((16, 32, 64), (False, True), (False, True)):
        r[f"qkv_tc_bn{bn}{'_pdl' if pdl else ''}{'_shallow' if sh else ''}"] = timed(
            lambda i: ops.linear(x_h, w_qkv[i], ops.EPI_BF16, bn, pdl=pdl, shallow=sh))

    for bn, cl in itertools.product((32, 64), (2, 4)):
        r[f"qkv_tc_bn{bn}_cluster{cl}_pdl"] = timed(lambda i: ops.linear(x_h, w_qkv[i], ops.EPI_BF16, bn, pdl=True, cluster=cl))

    r["gate_up+silu_cublas"] = timed(lambda i: ops.silu_mul(F.linear(x_h, w_gu[i])))
    for bn, pdl in itertools.product((32, 64), (False, True)):
        r[f"gate_up+silu_tc_bn{bn}{'_pdl' if pdl else ''}"] = timed(lambda i: ops.linear(x_h, w_gu[i], ops.EPI_SILU, bn, pdl=pdl))

    for bn, cl in itertools.product((32, 64), (2, 4)):
        r[f"gate_up+silu_tc_bn{bn}_cluster{cl}_pdl"] = timed(lambda i: ops.linear(x_h, w_gu[i], ops.EPI_SILU, bn, pdl=True, cluster=cl))

    for name, xin, ws, k in (("o", x_o, w_o, OIN), ("down", x_i, w_dn, INTER)):
        r[f"{name}+addnorm_cublas"] = timed(lambda i: ops.add_rmsnorm(F.linear(xin, ws[i]), resid, wn, 1e-6))
        for bn, splits, pdl in itertools.product((32, 64, 128), (1, 2, 4, 8), (False, True)):
            if (k // 64) % splits:
                continue
            r[f"{name}+addnorm_tc_bn{bn}_s{splits}{'_pdl' if pdl else ''}"] = timed(
                lambda i: ops.add_rmsnorm_partials(ops.linear(xin, ws[i], ops.EPI_PARTIAL, bn, splits, pdl=pdl), resid, wn, 1e-6, pdl=pdl))

    # the MLP half of a layer as one chain (what a step would issue)
    def mlp_lib(i):
        a = ops.silu_mul(F.linear(x_h, w_gu[i]))
        return ops.add_rmsnorm(F.linear(a, w_dn[i]), resid, wn, 1e-6)

    def mlp_tc(i, pdl=True):
        a = ops.linear(x_h, w_gu[i], ops.EPI_SILU, 32, pdl=pdl)
        return ops.add_rmsnorm_partials(ops.linear(a, w_dn[i], ops.EPI_PARTIAL, 64, 8, pdl=pdl), resid, wn, 1e-6, pdl=pdl)

    r["mlp_chain_cublas"] = timed(mlp_lib)
    r["mlp_chain_tc_pdl"] = timed(mlp_tc)
    r["mlp_chain_tc_nopdl"] = timed(lambda i: mlp_tc(i, False))
    # LM head + sampling (tied Qwen3-0.6B head: 151 936 x 1024), two distinct weight sets (311 MB each)
    heads = [rnd(151936, HID) for _ in range(2)]
    temps = torch.full((M,), 0.6, device="cuda")
    kws = torch.zeros(M, dtype=torch.int64, device="cuda")
    r["lm_head+sample_cublas"] = timed(lambda i: ops.sample(F.linear(x_h, heads[i]), temps, 1, 0), nsets=2)
    for sh, cl in ((True, 1), (False, 1), (False, 2), (False, 4)):
        r[f"lm_head+sample_fused_{'shallow' if sh else 'deep'}_cluster{cl}"] = timed(
            lambda i: ops.lm_head_sample(x_h, heads[i], temps, 1, 0, kws, shallow=sh, cluster=cl), nsets=2)
    del heads
    res[f"M{M}"] = r
    print(f"M={M} done " + json.dumps(r), file=sys.stderr, flush=True)
print(json.dumps({"unit": "us per op (graph replay over 16 weight sets)", "results": res}, indent=1))
