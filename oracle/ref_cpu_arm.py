"""The REFERENCE'S OWN classes on the host CPU: the `--impl reference` arm and the cpu_baseline leg of bench.py.
TEST INFRASTRUCTURE / REPORTED BASELINE ONLY (see oracle/__init__.py) -- nothing in the product imports this.

    python oracle/ref_cpu_arm.py <model_dir> <reps> <budget_seconds> [n_seqs]

Runs, in a process of its own (the reference and the product both own the package name ``nanovllm``), the unmodified
reference installed under oracle/_ref:
  * its Scheduler / BlockManager / Sequence                         (engine/scheduler.py, block_manager.py, sequence.py)
  * its ModelRunner.prepare_prefill / prepare_decode, unbound       (engine/model_runner.py:123-188; pin_memory/.cuda()
    neutralised, exactly like oracle/make_golden.py does)
  * its Qwen3ForCausalLM nn.Modules in bf16 on CPU, its loader       (models/qwen3.py, utils/loader.py)
  * its Sampler (temperature / exponential race)                     (layers/sampler.py:7-12)
  * the serving loop of LLMEngine.step                               (engine/llm_engine.py:49-55)
with ONE substitution: Attention.forward's flash-attn / Triton calls (GPU only, layers/attention.py:59-75) are replaced by
oracle/paged_attention_ref.attention_forward_ref, the CPU restatement of the same operator.  torch.compile is
disabled (TORCH_COMPILE_DISABLE=1): the decorated functions run as the eager PyTorch the reference wrote.

Workload: a bounded sample of the benchmark mix (reference bench.py:9-18, seed 0): its first `n_seqs` requests with
their own prompt and output lengths, temperature 0.6, ignore_eos; each repetition is cut off after `budget_seconds`.
Prints one JSON line: {"kind": "reference", "reps": [{"tokens": .., "seconds": .., "steps": ..}, ...], "threads": ..}.
"""
import itertools
import json
import os
import random
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")


def main():
    model_dir, reps, budget = sys.argv[1], int(sys.argv[2]), float(sys.argv[3])
    n_seqs = int(sys.argv[4]) if len(sys.argv) > 4 else 8
    os.environ["TORCH_COMPILE_DISABLE"] = "1"
    sys.path.insert(0, REF)
    sys.path.insert(1, ROOT)
    import torch
    import torch.distributed as dist
    import nanovllm
    assert os.path.realpath(nanovllm.__file__).startswith(os.path.realpath(REF)), nanovllm.__file__
    cores = os.cpu_count() or 1
    threads = min(cores, int(os.environ.get("B200_CPU_THREADS", "32")))
    torch.set_num_threads(threads)

    from transformers import AutoConfig
    from nanovllm.engine.model_runner import ModelRunner
    from nanovllm.engine.scheduler import Scheduler
    from nanovllm.engine.sequence import Sequence
    from nanovllm.layers import attention as ref_attn
    from nanovllm.layers.sampler import Sampler
    from nanovllm.models.qwen3 import Qwen3ForCausalLM
    from nanovllm.sampling_params import SamplingParams
    from nanovllm.utils.context import get_context, reset_context
    from nanovllm.utils.loader import load_model
    from oracle.paged_attention_ref import attention_forward_ref

    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{29800 + os.getpid() % 150}", world_size=1, rank=0)
    hf = AutoConfig.from_pretrained(model_dir)
    torch.set_default_dtype(torch.bfloat16)
    model = Qwen3ForCausalLM(hf)
    torch.set_default_dtype(torch.float32)
    load_model(model, model_dir)
    sampler = Sampler()

    def cpu_attention(self, q, k, v):                 # flash-attn has no CPU build: same operator, restated
        ctx = get_context()
        has = self.k_cache.numel() > 0
        return attention_forward_ref(q, k, v, self.k_cache if has else None, self.v_cache if has else None, ctx, self.scale)

    ref_attn.Attention.forward = cpu_attention

    # prepare_prefill / prepare_decode build pinned tensors and move them to the GPU: neutralise both calls
    real_tensor = torch.tensor

    def tensor_nopin(*a, **k):
        k.pop("pin_memory", None)
        return real_tensor(*a, **k)

    torch.tensor = tensor_nopin
    torch.Tensor.cuda = lambda self, *a, **k: self

    random.seed(0)                                    # reference bench.py:9-18
    prompts = [[random.randint(0, 10000) for _ in range(random.randint(100, 1024))] for _ in range(256)]
    max_tokens = [random.randint(100, 1024) for _ in range(256)]
    prompts, max_tokens = prompts[:n_seqs], max_tokens[:n_seqs]
    block = 256
    head_dim = getattr(hf, "head_dim", hf.hidden_size // hf.num_attention_heads)
    num_blocks = sum((len(p) + m + block - 1) // block for p, m in zip(prompts, max_tokens)) + 2
    for m in model.modules():
        if hasattr(m, "k_cache") and hasattr(m, "v_cache"):
            m.k_cache = torch.zeros(num_blocks, block, hf.num_key_value_heads, head_dim, dtype=torch.bfloat16)
            m.v_cache = torch.zeros_like(m.k_cache)
    stub = types.SimpleNamespace(block_size=block)
    stub.prepare_block_tables = lambda seqs: ModelRunner.prepare_block_tables(stub, seqs)

    out = []
    for r in range(reps):
        Sequence.block_size = block
        Sequence.counter = itertools.count()
        cfg = types.SimpleNamespace(max_num_seqs=512, max_num_batched_tokens=16384, eos=-1, kvcache_block_size=block,
                                    num_kvcache_blocks=num_blocks)
        sched = Scheduler(cfg)
        shift = 17 * r                                 # token values differ per repetition: no prefix-cache reuse
        for p, mt in zip(prompts, max_tokens):
            sched.add(Sequence([(t + shift) % 10001 for t in p], SamplingParams(temperature=0.6, max_tokens=mt, ignore_eos=True)))
        produced = steps = 0
        t0 = time.perf_counter()
        with torch.inference_mode():
            while not sched.is_finished() and time.perf_counter() - t0 < budget:
                seqs, is_prefill = sched.schedule()                          # llm_engine.py:49-55
                ids, pos = (ModelRunner.prepare_prefill if is_prefill else ModelRunner.prepare_decode)(stub, seqs)
                temps = torch.tensor([s.temperature for s in seqs], dtype=torch.float32)
                logits = model.compute_logits(model(ids, pos))
                tokens = sampler(logits, temps).tolist()
                reset_context()
                before = sum(s.num_completion_tokens for s in seqs)
                sched.postprocess(seqs, tokens, is_prefill)
                produced += sum(s.num_completion_tokens for s in seqs) - before
                steps += 1
        dt = time.perf_counter() - t0
        out.append(dict(tokens=produced, seconds=dt, steps=steps))
        print(f"[ref-cpu] rep {r}: {produced} tokens in {dt:.1f}s over {steps} engine steps", file=sys.stderr, flush=True)
    print(json.dumps(dict(kind="reference", reps=out, threads=threads, cores=cores, n_seqs=n_seqs,
                          prompt_tokens=sum(len(p) for p in prompts), budget_s=budget)))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
