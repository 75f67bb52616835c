"""Run the UNMODIFIED reference (staged under oracle/_ref by oracle/install_reference.py, git-ignored) on the GPU:
its own LLM / flash-attn 2.8.3 / Triton / torch.compile / CUDA-graph path, on the benchmark request mix.

    python baseline/run_reference_gpu.py [passes]

This is the "kernel to beat on the same box" of BASELINE.md section 4 -- context for the headline number, not
the driver's `--impl reference` arm (that one is the CPU port, as the task tier prescribes).
Prints one JSON line: {"impl": "reference-gpu", "value": tokens/s, ...}.
"""
import importlib.util
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")


def load_by_path(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    passes = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    if not os.path.isdir(os.path.join(REF, "nanovllm")):
        print(json.dumps({"impl": "reference-gpu", "unavailable": "oracle/_ref missing (oracle/install_reference.py)"}))
        return
    syn = load_by_path("b200_synthetic", os.path.join(ROOT, "nano-vllm_b200", "nanovllm", "utils", "synthetic.py"))
    mdir = syn.make_model_dir(os.environ.get("B200_BENCH_MODEL_DIR", "/tmp/b200_bench_models/qwen3-0.6b"), "qwen3-0.6b", seed=0)
    sys.path.insert(0, REF)                      # the reference owns the name `nanovllm` in this process
    import torch
    from nanovllm import LLM, SamplingParams
    import nanovllm
    assert os.path.realpath(nanovllm.__file__).startswith(os.path.realpath(REF))
    from random import randint, seed
    t0 = time.time()
    llm = LLM(mdir, enforce_eager=False, max_model_len=4096)
    init_s = time.time() - t0
    llm.generate(["t1 t2 t3"], SamplingParams())
    rates = []
    for p in range(passes):
        seed(0)                                   # reference bench.py:9-18
        prompts = [[randint(0, 10000) for _ in range(randint(100, 1024))] for _ in range(256)]
        sps = [SamplingParams(temperature=0.6, ignore_eos=True, max_tokens=randint(100, 1024)) for _ in range(256)]
        if p:
            prompts = [[(t + 17 * p) % 10001 for t in q] for q in prompts]
        torch.cuda.synchronize()
        t = time.time()
        llm.generate(prompts, sps, use_tqdm=False)
        torch.cuda.synchronize()
        dt = time.time() - t
        rates.append(sum(sp.max_tokens for sp in sps) / dt)
        print(f"[reference-gpu] pass {p}: {dt:.2f}s {rates[-1]:.0f} tok/s", file=sys.stderr, flush=True)
    print(json.dumps({"impl": "reference-gpu", "metric": "output tokens/s, Qwen3-0.6B 256 seqs in/out 100-1024", "value": max(rates),
                      "all_passes": rates, "unit": "tokens/s", "init_s": init_s,
                      "what": "unmodified GeeeekExplorer/nano-vllm @ bb823b3e, flash-attn 2.8.3, CUDA graphs on, same synthetic Qwen3-0.6B"}))
    os._exit(0)


if __name__ == "__main__":
    main()
