"""Block-FP8 weights vs bf16 on one H100, in one call (DESIGN.md 3.6).

    python profiles/fp8_weights_bench.py [--out profiles/h100_fp8_weights.json] [--skip-e2e]

(a) GEMMs: the FP8 projection (activation quantization + the e4m3 wgmma GEMM, and the GEMM alone) against the bf16 path
    the engine runs for the same projection (decode batches <= 128 rows: cuBLAS for qkv / gate_up + SiluAndMul and the
    bf16 wgmma split-K kernel for o / down; above: cuBLAS everywhere), at Qwen3-0.6B / 8B / 32B projection shapes.
    Decode sizes report achieved weight bytes / s, prefill sizes TFLOP/s (against the 1979 TFLOP/s FP8 data-sheet figure).
    CUDA events around a CUDA graph of 20 (decode) or 5 (prefill) back-to-back calls, median of 5 replays.
(b) End to end: bench.py's request mix through LLM.generate() on random-init bf16 and FP8 directories at 0.6B and 8B
    dimensions, alternated, each engine in a child process (it sizes its KV cache from the whole card):
    num_kvcache_blocks and output tokens / s.
(c) Qwen3-32B dimensions in FP8 on one GPU: does it load, how many KV blocks, what tok/s on the same mix.
Quality: relative L2 error of FP8 last-token logits against bf16 logits of the same seed (the full Qwen3-0.6B-shaped
    random model, packed prefill of eight 256-token prompts), and how often their argmax agrees.
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "nano-vllm_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "profiles")]

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import bench  # noqa: E402  (read-only: the request mix)

FP8_PEAK_TFLOPS = 1979.0
DECODE_M = [1, 16, 64, 128, 256]
PREFILL_M = [2048, 8192, 16384]
MODELS = {"0.6b": "qwen3-0.6b", "8b": "qwen3-8b", "32b": "qwen3-32b"}


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [x.strip() for x in q[0].split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def timed(fn, reps: int, windows: int = 5) -> float:
    """Median over `windows` of the mean device time of `reps` back-to-back calls, in seconds.  The calls are captured in
    one CUDA graph and replayed, as the engine replays its decode steps, so that host launch overhead is not measured."""
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


def projection_shapes(d: dict) -> dict:
    q, kv, h, i = d["num_attention_heads"] * d["head_dim"], d["num_key_value_heads"] * d["head_dim"], d["hidden_size"], d["intermediate_size"]
    return dict(qkv=(q + 2 * kv, h), o=(h, q), gate_up=(2 * i, h), down=(h, i))


def gemms() -> list:
    from nanovllm import ops
    from nanovllm.utils.fp8 import quantize_weight
    from nanovllm.utils.synthetic import PRESETS
    rows = []
    for tag, preset in MODELS.items():
        for proj, (n, k) in projection_shapes(PRESETS[preset]).items():
            wb = (0.02 * torch.randn(n, k, device="cuda")).to(torch.bfloat16)
            wq, ws = quantize_weight(wb)
            kb = k // 128
            for m in DECODE_M + PREFILL_M:
                x = torch.randn(m, k, device="cuda").to(torch.bfloat16)
                xq, xs = ops.quant_fp8(x)
                decode = m <= 256
                epi = ops.EPI_SILU if proj == "gate_up" else (ops.EPI_PARTIAL if proj in ("o", "down") and m <= 128 else ops.EPI_BF16)
                bn = 64                                    # Qwen3ForCausalLM's policy
                splits = next(d for d in range(min(8, kb), 0, -1) if kb % d == 0) if epi == ops.EPI_PARTIAL else 1
                fp8_gemm = lambda: ops.linear_fp8(xq, xs, wq, ws, epi, bn, splits, pdl=True)
                fp8_full = lambda: (ops.linear_fp8(*ops.quant_fp8(x), wq, ws, epi, bn, splits, pdl=True))
                if proj in ("o", "down") and m <= 128:
                    tkb = k // 64
                    s16 = next(d for d in range(min(8, tkb), 0, -1) if tkb % d == 0)
                    bf16 = lambda: ops.linear(x, wb, ops.EPI_PARTIAL, 64, s16, pdl=True)
                    bf16_name = "wgmma split-K (bf16)"
                elif proj == "gate_up":
                    bf16 = lambda: ops.silu_mul(F.linear(x, wb))
                    bf16_name = "cuBLAS + silu_mul"
                else:
                    bf16 = lambda: F.linear(x, wb)
                    bf16_name = "cuBLAS"
                reps = 20 if decode else 5
                t8, t8q, t16 = timed(fp8_gemm, reps), timed(fp8_full, reps), timed(bf16, reps)
                flop = 2.0 * m * n * k
                row = dict(model=tag, proj=proj, n=n, k=k, m=m, bf16_path=bf16_name, fp8_gemm_us=t8 * 1e6,
                           fp8_quant_gemm_us=t8q * 1e6, bf16_us=t16 * 1e6, speedup_quant_gemm=t16 / t8q)
                if decode:
                    row.update(fp8_weight_TBps=n * k / t8q / 1e12, bf16_weight_TBps=2 * n * k / t16 / 1e12)
                else:
                    row.update(fp8_TFLOPs=flop / t8q / 1e12, fp8_gemm_only_TFLOPs=flop / t8 / 1e12, bf16_TFLOPs=flop / t16 / 1e12,
                               fp8_share_of_datasheet=flop / t8q / 1e12 / FP8_PEAK_TFLOPS)
                rows.append(row)
                print(json.dumps(row), flush=True)
                del x, xq, xs
            del wb, wq, ws
            torch.cuda.empty_cache()
    return rows


def model_dir(preset: str, fp8: bool) -> str:
    from nanovllm.utils.synthetic import make_model_dir
    return make_model_dir(os.path.join(tempfile.gettempdir(), f"b200_fp8bench_{os.getuid()}", f"{preset}_{'fp8' if fp8 else 'bf16'}"),
                          preset, seed=0, weights=False, fp8=fp8)


def e2e_arm(preset: str, fp8: bool) -> dict:
    os.environ["NANOVLLM_ALLOW_RANDOM_INIT"] = "1"
    from nanovllm import LLM, SamplingParams
    t = time.perf_counter()
    llm = LLM(model_dir(preset, fp8), enforce_eager=False, max_model_len=4096)
    init_s = time.perf_counter() - t
    prompts, max_tokens = bench.bench_requests(0)
    sps = [SamplingParams(temperature=0.6, ignore_eos=True, max_tokens=mt) for mt in max_tokens]
    llm.generate(prompts[:16], sps[:16], use_tqdm=False)                # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    llm.generate(prompts, sps, use_tqdm=False)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    row = dict(preset=preset, weights="fp8" if fp8 else "bf16", output_tokens=sum(max_tokens), output_tok_s=sum(max_tokens) / dt,
               num_kvcache_blocks=llm.config.num_kvcache_blocks, weight_gb=torch.cuda.memory_allocated() / 1e9, init_s=round(init_s, 1))
    llm.exit()
    return row


def child(preset: str, fp8: bool) -> dict:
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--arm", preset, *(["--fp8"] if fp8 else [])],
                       capture_output=True, text=True, timeout=2400)
    lines = [l for l in r.stdout.splitlines() if l.startswith("ARM ")]
    if r.returncode != 0 or not lines:
        return dict(preset=preset, weights="fp8" if fp8 else "bf16", error=(r.stdout[-1500:] + r.stderr[-1500:]))
    return json.loads(lines[-1][4:])


def quality(preset: str = "qwen3-0.6b", seqs: int = 8, seq_len: int = 256) -> dict:
    """Relative L2 of FP8 last-token logits vs bf16 logits of the same seed, packed prefill of `seqs` random prompts."""
    from types import SimpleNamespace
    from nanovllm.models.qwen3 import Qwen3ForCausalLM
    from nanovllm.utils.context import reset_context, set_context
    from nanovllm.utils.loader import load_model
    from nanovllm.utils.synthetic import PRESETS, hf_config_dict
    from nanovllm.utils import fp8 as fp8fmt
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(2, PRESETS[preset]["vocab_size"], (seqs * seq_len,), generator=g).cuda()
    pos = torch.arange(seq_len).repeat(seqs).cuda()
    cu = torch.arange(0, (seqs + 1) * seq_len, seq_len, dtype=torch.int32).cuda()
    out = {}
    for fp8 in (False, True):
        cfg = hf_config_dict(PRESETS[preset])
        if fp8:
            cfg["quantization_config"] = fp8fmt.quantization_config_dict()
        m = Qwen3ForCausalLM(SimpleNamespace(**cfg), 0, 1, "cuda", max_position=4096)
        load_model(m, tempfile.mkdtemp(), allow_random=True, seed=0)
        set_context(True, cu, cu, seq_len, seq_len, None, None, None)
        out[fp8] = m.compute_logits(m(ids, pos)).float()
        reset_context()
        del m
        torch.cuda.empty_cache()
    rel = ((out[True] - out[False]).norm(dim=-1) / out[False].norm(dim=-1))
    agree = (out[True].argmax(-1) == out[False].argmax(-1)).float().mean().item()
    return dict(preset=preset, prompts=seqs, prompt_len=seq_len, logits_rel_l2_mean=rel.mean().item(),
                logits_rel_l2_max=rel.max().item(), argmax_agreement=agree)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_fp8_weights.json"))
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--arm", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--fp8", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    os.environ.setdefault("B200_SAMPLE_SEED", "0")
    if args.arm:
        print("ARM " + json.dumps(e2e_arm(args.arm, args.fp8)), flush=True)
        return
    info = gpu_info()
    print(json.dumps(info), flush=True)
    res = dict(gpu=info, what="block-FP8 (e4m3, 128x128 weight blocks, dynamic 1x128 activations) vs bf16; profiles/fp8_weights_bench.py")
    res["quality"] = quality()
    print(json.dumps(res["quality"]), flush=True)
    res["gemm"] = gemms()
    if not args.skip_e2e:
        e2e = []
        for preset in ("qwen3-0.6b", "qwen3-8b"):
            for fp8 in (False, True):
                e2e.append(child(preset, fp8))
                print(json.dumps(e2e[-1]), flush=True)
        res["e2e"] = e2e
        res["one_gpu_32b_fp8"] = child("qwen3-32b", True)
        print(json.dumps(res["one_gpu_32b_fp8"]), flush=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
