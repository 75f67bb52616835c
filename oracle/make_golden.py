"""Generate tests/golden/* by running the REFERENCE's own code.

    TORCH_COMPILE_DISABLE=1 python oracle/make_golden.py            # needs the reference under oracle/_ref

The reference is Python and is staged under oracle/_ref (oracle/install_reference.py); nothing at test
time reads it, the tests read what this script stored.  What gets pinned:

1. hash_kat.json          BlockManager.compute_hash known answers          (block_manager.py:35-41)
2. trace_<workload>.json  step-by-step digests of the reference Scheduler / BlockManager /
                          Sequence driven by a deterministic fake sampler, plus the digests of the
                          arrays the reference's own ModelRunner.prepare_prefill / prepare_decode /
                          prepare_block_tables build for every step       (scheduler.py, block_manager.py,
                          sequence.py, model_runner.py:123-188)
3. model_<preset>.npz     logits of the reference's own nn.Modules (Qwen3ForCausalLM on CPU, gloo world
                          of 1, torch.compile disabled) with Attention.forward replaced by
                          oracle.paged_attention_ref (the reference's attention is flash-attn, GPU only)

The product's host code is tested against (1)-(2) bit for bit; oracle/qwen3_ref.py in "eager"
rounding mode is tested against (3) bit for bit, which is what entitles it to be the checker
for the CUDA kernels.
"""
from __future__ import annotations

import hashlib
import json
import os
import random
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref")   # oracle/install_reference.py
sys.path.insert(0, ROOT)


# --------------------------------------------------------------------------------------------
# shared with tests/: workload definitions and the digest format
# --------------------------------------------------------------------------------------------
MODEL_PRESETS = ("tiny", "tiny-g4", "tiny-g1", "tiny-g8")      # q/kv head ratios 2, 4, 1, 8; tied and untied LM heads


def fake_token(seq_id: int, num_tokens: int, vocab: int) -> int:
    return (seq_id * 7919 + num_tokens * 104729 + 13) % vocab


def workloads() -> dict:
    """name -> dict(engine cfg, prompts, sampling tuples (temperature, max_tokens, ignore_eos), vocab, eos)."""
    out = {}
    rnd = random.Random(0)
    # the benchmark's exact request mix (reference bench.py:9-18): seed(0), 256 seqs, in/out U[100, 1024]
    random.seed(0)
    prompts = [[random.randint(0, 10000) for _ in range(random.randint(100, 1024))] for _ in range(256)]
    sps = [(0.6, random.randint(100, 1024), True) for _ in range(256)]
    base = dict(max_num_seqs=512, max_num_batched_tokens=16384, kvcache_block_size=256)
    out["bench"] = dict(cfg=dict(base, num_kvcache_blocks=5000), prompts=prompts, sps=sps, vocab=50000, eos=-1)
    out["bench_tight"] = dict(cfg=dict(base, num_kvcache_blocks=400), prompts=prompts, sps=sps, vocab=50000, eos=-1)
    # shared prefix, small pages: prefix-cache hits, ref-counted shared blocks, revival of freed blocks
    prefix = [rnd.randint(0, 30000) for _ in range(600)]
    p3 = [prefix + [rnd.randint(0, 30000) for _ in range(rnd.randint(5, 120))] for _ in range(96)]
    s3 = [(0.0, rnd.randint(4, 48), True) for _ in range(96)]
    out["prefix16"] = dict(cfg=dict(max_num_seqs=24, max_num_batched_tokens=4096, kvcache_block_size=16,
                                    num_kvcache_blocks=1500), prompts=p3, sps=s3, vocab=50000, eos=-1)
    # long prompts against a small token budget: chunked prefill, plus block pressure
    p4 = [[rnd.randint(0, 30000) for _ in range(rnd.randint(300, 3000))] for _ in range(14)]
    s4 = [(1.0, rnd.randint(8, 64), True) for _ in range(14)]
    out["chunked32"] = dict(cfg=dict(max_num_seqs=8, max_num_batched_tokens=1024, kvcache_block_size=32,
                                     num_kvcache_blocks=420), prompts=p4, sps=s4, vocab=50000, eos=-1)
    # EOS termination (tiny vocab so the fake sampler hits it), repeated prompts
    p5 = [[rnd.randint(0, 40) for _ in range(rnd.randint(20, 200))] for _ in range(40)]
    p5 += [list(p5[i]) for i in range(10)]
    s5 = [(0.8, rnd.randint(16, 200), False) for _ in range(50)]
    out["eos64"] = dict(cfg=dict(max_num_seqs=16, max_num_batched_tokens=2048, kvcache_block_size=64,
                                 num_kvcache_blocks=60), prompts=p5, sps=s5, vocab=41, eos=7)
    # BASELINE config 4's request mix at the bookkeeping level: 1024 requests against 512 running slots, so prefill
    # and decode steps interleave for the whole run; the cache is sized to force preemptions
    r6 = random.Random(4)
    p6 = [[r6.randint(0, 150000) for _ in range(r6.randint(50, 800))] for _ in range(1024)]
    s6 = [(0.7, r6.randint(10, 200), True) for _ in range(1024)]
    out["mixed1024"] = dict(cfg=dict(max_num_seqs=512, max_num_batched_tokens=16384, kvcache_block_size=256,
                                     num_kvcache_blocks=1100), prompts=p6, sps=s6, vocab=151936, eos=-1)
    # BASELINE config 5's: 128 concurrent long-context requests (about 8k in, up to 1k out); every prompt is
    # longer than half the token budget, so prefill is chunked throughout, and blocks run out during decode
    r7 = random.Random(5)
    p7 = [[r7.randint(0, 150000) for _ in range(r7.randint(7000, 8192))] for _ in range(128)]
    s7 = [(0.7, r7.randint(300, 1024), True) for _ in range(128)]
    out["longctx128"] = dict(cfg=dict(max_num_seqs=128, max_num_batched_tokens=16384, kvcache_block_size=256,
                                      num_kvcache_blocks=4000), prompts=p7, sps=s7, vocab=151936, eos=-1)
    return out


def fuzz_workloads(seed: int, n: int) -> list:
    """Small random workloads for differential testing (tests/test_differential_fuzz.py): every knob the scheduler
    and the block manager branch on is drawn at random -- page size, token budget, running slots, cache size (tight
    enough to preempt), shared prefixes and exact duplicates (prefix-cache hits, block revival), EOS stops."""
    out = []
    for i in range(n):
        r = random.Random(seed * 100003 + i)
        bs = r.choice([2, 4, 8, 16, 32, 256])      # not 1: the reference's `len % block_size == 1` append rule needs >= 2
        nseq = r.randint(1, 40)
        max_len = r.choice([8, 40, 150, 600])
        vocab = r.choice([5, 37, 1000, 50000])
        prefixes = [[r.randrange(vocab) for _ in range(r.randint(0, 3 * bs + 5))] for _ in range(3)]
        prompts = []
        for _ in range(nseq):
            kind = r.random()
            if kind < 0.15 and prompts:
                prompts.append(list(r.choice(prompts)))                        # exact duplicate
            elif kind < 0.55:
                prompts.append(r.choice(prefixes) + [r.randrange(vocab) for _ in range(r.randint(1, max_len))])
            else:
                prompts.append([r.randrange(vocab) for _ in range(r.randint(1, max_len))])
        use_eos = r.random() < 0.4
        sps = [(r.choice([0.5, 0.8, 1.0]), r.randint(1, 40), not use_eos or r.random() < 0.3) for _ in range(nseq)]
        longest = max(len(p) + mt for p, (_, mt, _) in zip(prompts, sps))
        need = (longest + bs - 1) // bs + 1                                    # one sequence must always fit
        total = sum((len(p) + mt + bs - 1) // bs for p, (_, mt, _) in zip(prompts, sps))
        nblk = max(need, int(total * r.choice([0.15, 0.4, 1.0, 2.0])))
        budget = r.choice([16, 64, 256, 4096])
        cfg = dict(max_num_seqs=r.choice([1, 2, 5, 16, 64]), max_num_batched_tokens=budget, kvcache_block_size=bs,
                   num_kvcache_blocks=nblk)
        out.append(dict(cfg=cfg, prompts=prompts, sps=sps, vocab=vocab, eos=r.randrange(vocab) if use_eos else -1))
    return out


def digest(*arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(np.asarray(a, dtype=np.int64))
        h.update(np.asarray(a.shape, dtype=np.int64).tobytes())
        h.update(a.tobytes())
    return h.hexdigest()[:20]


def step_record(seqs, is_prefill: bool, meta: dict) -> list:
    """[is_prefill, n_seqs, n_tokens, bookkeeping digest, metadata digest]"""
    ntok = sum(s.num_scheduled_tokens for s in seqs)
    book = [np.asarray([s.seq_id for s in seqs]), np.asarray([s.num_scheduled_tokens for s in seqs]),
            np.asarray([s.num_cached_tokens for s in seqs]), np.asarray([len(s) for s in seqs])]
    book += [np.asarray(s.block_table) for s in seqs]
    keys = ["input_ids", "positions", "slot_mapping", "cu_seqlens_q", "cu_seqlens_k", "context_lens", "block_tables"]
    md = [np.zeros(0) if meta.get(k) is None else meta[k] for k in keys]
    md.append(np.asarray([meta.get("max_seqlen_q", 0), meta.get("max_seqlen_k", 0), int(meta.get("block_tables") is not None)]))
    return [int(is_prefill), len(seqs), int(ntok), digest(*book), digest(*md)]


COMPACT_CHUNK = 32


def compact_steps(steps) -> str:
    """A workload's step records as one string of 8-hex-digit hashes, one per chunk of COMPACT_CHUNK consecutive steps
    (keeps the fuzz fixtures small; a differing step still changes its chunk's hash)."""
    return "".join(hashlib.sha256(json.dumps(steps[i:i + COMPACT_CHUNK]).encode()).hexdigest()[:8]
                   for i in range(0, len(steps), COMPACT_CHUNK))


def drive(make_seq, scheduler, block_size, build_meta, w) -> dict:
    """Run one workload to completion; identical for the reference classes and the product's."""
    for p, (t, mt, ie) in zip(w["prompts"], w["sps"]):
        scheduler.add(make_seq(p, t, mt, ie))
    steps, preempt_proxy = [], 0
    outputs = {}
    while not scheduler.is_finished():
        seqs, is_prefill = scheduler.schedule()
        meta = build_meta(seqs, is_prefill)
        steps.append(step_record(seqs, is_prefill, meta))
        toks = [fake_token(s.seq_id, len(s), w["vocab"]) for s in seqs]
        scheduler.postprocess(seqs, toks, is_prefill)
        for s in seqs:
            if s.is_finished:
                outputs[s.seq_id] = list(s.completion_token_ids)
    bm = scheduler.block_manager
    final = digest(np.asarray(sorted(bm.free_block_ids)), np.asarray(list(bm.free_block_ids)),
                   np.asarray(sorted(bm.hash_to_block_id.values())),
                   np.asarray([h % (1 << 62) for h in sorted(bm.hash_to_block_id.keys())]))
    out_digest = digest(*[np.asarray(outputs[k]) for k in sorted(outputs)])
    return dict(steps=steps, final_state=final, outputs=out_digest, num_steps=len(steps),
                num_prefill_steps=sum(s[0] for s in steps), sum_decode_batch=sum(s[1] for s in steps if not s[0]))


# --------------------------------------------------------------------------------------------
# reference side
# --------------------------------------------------------------------------------------------
def import_reference():
    sys.path.insert(0, REF)
    import torch
    import nanovllm  # noqa: F401  (the reference package)
    assert os.path.realpath(nanovllm.__file__).startswith(os.path.realpath(REF)), nanovllm.__file__
    return torch


def reference_meta_builder(torch, block_size):
    """The reference's own prepare_* run unbound with a stub self (SURVEY.md section 4)."""
    from nanovllm.engine.model_runner import ModelRunner
    from nanovllm.utils.context import get_context
    real_tensor = torch.tensor

    def tensor_nopin(*a, **k):
        k.pop("pin_memory", None)
        return real_tensor(*a, **k)

    torch.tensor = tensor_nopin
    torch.Tensor.cuda = lambda self, *a, **k: self
    stub = types.SimpleNamespace(block_size=block_size)
    stub.prepare_block_tables = lambda seqs: ModelRunner.prepare_block_tables(stub, seqs)

    def build(seqs, is_prefill):
        if is_prefill:
            ids, pos = ModelRunner.prepare_prefill(stub, seqs)
        else:
            ids, pos = ModelRunner.prepare_decode(stub, seqs)
        c = get_context()
        g = lambda t: None if t is None else t.numpy()
        return dict(input_ids=ids.numpy(), positions=pos.numpy(), slot_mapping=g(c.slot_mapping),
                    cu_seqlens_q=g(c.cu_seqlens_q), cu_seqlens_k=g(c.cu_seqlens_k), context_lens=g(c.context_lens),
                    block_tables=g(c.block_tables), max_seqlen_q=c.max_seqlen_q, max_seqlen_k=c.max_seqlen_k)
    return build


def gen_traces(torch, only=None):
    import itertools
    from nanovllm.engine.scheduler import Scheduler
    from nanovllm.engine.sequence import Sequence
    from nanovllm.sampling_params import SamplingParams
    for name, w in workloads().items():
        if only and name not in only:
            continue
        cfg = types.SimpleNamespace(eos=w["eos"], **w["cfg"])
        Sequence.block_size = cfg.kvcache_block_size
        Sequence.counter = itertools.count()

        def make_seq(p, t, mt, ie):
            sp = SamplingParams(temperature=max(t, 0.5), max_tokens=mt, ignore_eos=ie)   # reference forbids t == 0
            return Sequence(p, sp)

        rec = drive(make_seq, Scheduler(cfg), cfg.kvcache_block_size,
                    reference_meta_builder(torch, cfg.kvcache_block_size), w)
        rec["workload"] = name
        with open(os.path.join(GOLD, f"trace_{name}.json"), "w") as f:
            json.dump(rec, f, separators=(",", ":"))
        print(name, {k: v for k, v in rec.items() if k != "steps"})


def fuzz_reference(torch, seed: int, n: int, out_path: str):
    """Reference side of the differential test: run the reference's classes over fuzz_workloads(seed, n); the step records
    are stored compacted (compact_steps)."""
    import itertools
    from nanovllm.engine.scheduler import Scheduler
    from nanovllm.engine.sequence import Sequence
    from nanovllm.sampling_params import SamplingParams
    results = []
    for w in fuzz_workloads(seed, n):
        cfg = types.SimpleNamespace(eos=w["eos"], **w["cfg"])
        Sequence.block_size = cfg.kvcache_block_size
        Sequence.counter = itertools.count()
        make_seq = lambda p, t, mt, ie: Sequence(p, SamplingParams(temperature=t, max_tokens=mt, ignore_eos=ie))
        rec = drive(make_seq, Scheduler(cfg), cfg.kvcache_block_size, reference_meta_builder(torch, cfg.kvcache_block_size), w)
        rec["steps"] = compact_steps(rec["steps"])
        results.append(rec)
    with open(out_path, "w") as f:
        json.dump(results, f, separators=(",", ":"))


def api_surface(pkg) -> dict:
    """Public API of a `nanovllm` package as plain data (same function runs on the reference and on the product)."""
    import dataclasses
    import inspect
    from nanovllm.config import Config
    from nanovllm.engine.llm_engine import LLMEngine
    from nanovllm.sampling_params import SamplingParams

    def fields(cls):
        out = []
        for f in dataclasses.fields(cls):
            default = repr(f.default) if f.default is not dataclasses.MISSING else "<required>"
            out.append([f.name, default])
        return out

    def params(fn):
        out = []
        for name, p in inspect.signature(fn).parameters.items():
            out.append([name, "<required>" if p.default is inspect.Parameter.empty else repr(p.default), p.kind.name])
        return out

    methods = {m: params(getattr(LLMEngine, m)) for m in ("__init__", "add_request", "step", "is_finished", "generate", "exit")}
    return dict(exports=sorted(n for n in ("LLM", "SamplingParams") if hasattr(pkg, n)),
                llm_is_engine=issubclass(pkg.LLM, LLMEngine),
                config=fields(Config), sampling_params=fields(SamplingParams), engine_methods=methods)


def gen_api_surface():
    import nanovllm
    with open(os.path.join(GOLD, "api_surface.json"), "w") as f:
        json.dump(api_surface(nanovllm), f, indent=1)
    print("api surface written")


def gen_hash_kat():
    from nanovllm.engine.block_manager import BlockManager
    rnd = random.Random(1)
    cases = []
    for n, prefix in ((256, -1), (256, 12345), (16, -1), (16, 2**63 + 5), (1, -1), (33, 987654321987654321)):
        toks = list(range(n)) if not cases else [rnd.randint(0, 151935) for _ in range(n)]
        cases.append(dict(tokens=toks, prefix=prefix, hash=BlockManager.compute_hash(toks, prefix)))
    assert cases[0]["hash"] == 5218229187174952702          # SURVEY.md section 4
    with open(os.path.join(GOLD, "hash_kat.json"), "w") as f:
        json.dump(cases, f)
    print("hash KATs:", len(cases))


# ---- model ------------------------------------------------------------------------------------
def load_product_synthetic():
    """The product's checkpoint writer, loaded by file path (the reference owns the name `nanovllm` here)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "b200_synthetic", os.path.join(ROOT, "nano-vllm_b200", "nanovllm", "utils", "synthetic.py"))
    syn = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(syn)
    return syn


def gen_model(torch, preset: str):
    """Run oracle/model_script.py through the reference's own nn.Modules on CPU and record the logits."""
    import torch.distributed as dist
    from oracle.model_script import make_script, run_script
    from oracle.paged_attention_ref import attention_forward_ref
    syn = load_product_synthetic()

    if not dist.is_initialized():
        dist.init_process_group("gloo", init_method="tcp://127.0.0.1:29511", world_size=1, rank=0)
    from transformers import AutoConfig
    from nanovllm.layers import attention as ref_attn
    from nanovllm.models.qwen3 import Qwen3ForCausalLM
    from nanovllm.utils.context import get_context, reset_context, set_context
    from nanovllm.utils.loader import load_model

    mdir = syn.make_model_dir(f"/tmp/golden_model_{preset}", preset, seed=1234, tokenizer=False)
    hf = AutoConfig.from_pretrained(mdir)
    torch.set_default_dtype(torch.bfloat16)
    model = Qwen3ForCausalLM(hf)
    torch.set_default_dtype(torch.float32)
    load_model(model, mdir)

    def patched_forward(self, q, k, v):            # the reference's attention is flash-attn (GPU only)
        ctx = get_context()
        has = self.k_cache.numel() > 0
        return attention_forward_ref(q, k, v, self.k_cache if has else None, self.v_cache if has else None,
                                     ctx, self.scale)

    ref_attn.Attention.forward = patched_forward
    dims = syn.PRESETS[preset]
    script = make_script(dims["vocab_size"])
    for m in model.modules():
        if hasattr(m, "k_cache") and hasattr(m, "v_cache"):
            m.k_cache = torch.zeros(script["num_blocks"], script["block_size"], dims["num_key_value_heads"],
                                    dims["head_dim"], dtype=torch.bfloat16)
            m.v_cache = torch.zeros_like(m.k_cache)

    def step_fn(input_ids, positions, c):
        set_context(c["is_prefill"], c.get("cu_seqlens_q"), c.get("cu_seqlens_k"), c.get("max_seqlen_q", 0),
                    c.get("max_seqlen_k", 0), c.get("slot_mapping"), c.get("context_lens"), c.get("block_tables"))
        with torch.inference_mode():
            logits = model.compute_logits(model(input_ids, positions))
        reset_context()
        return logits

    outs = run_script(torch, script, step_fn)
    np.savez_compressed(os.path.join(GOLD, f"model_{preset}.npz"),
                        **{f"logits_{i}": o.view(torch.int16).numpy() for i, o in enumerate(outs)})
    print("model", preset, [tuple(o.shape) for o in outs])


def main():
    os.environ.setdefault("TORCH_COMPILE_DISABLE", "1")
    os.makedirs(GOLD, exist_ok=True)
    torch = import_reference()
    only = sys.argv[1:]                      # e.g. `make_golden.py mixed1024 longctx128` regenerates just those traces
    if only and only[0] == "--api":
        gen_api_surface()
        return
    if only and only[0] == "--models":       # `make_golden.py --models tiny-g1 tiny-g8`: just those model fixtures
        for preset in only[1:]:
            gen_model(torch, preset)
        return
    if only and only[0] == "--fuzz":         # `make_golden.py --fuzz SEED 150 tests/golden/fuzz_seedSEED.json`
        fuzz_reference(torch, int(only[1]), int(only[2]), only[3])
        return
    if only:
        gen_traces(torch, only)
        return
    gen_hash_kat()
    gen_api_surface()
    gen_traces(torch)
    for preset in MODEL_PRESETS:
        gen_model(torch, preset)


if __name__ == "__main__":
    main()
