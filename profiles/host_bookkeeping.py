"""Host-side cost of one engine step, ours against the reference's own classes, on the SAME workloads (CPU only, no GPU).

    python profiles/host_bookkeeping.py                 # both sides; workloads bench, mixed1024, longctx128 -> one JSON object
    python profiles/host_bookkeeping.py ours|ref NAME   # one side, one workload (what the driver mode runs in subprocesses)

SURVEY.md 8(f) rows 1 and 4: once the GPU step is fast, what the host does per step -- Scheduler.schedule (+ BlockManager),
the metadata builders (prepare_prefill / prepare_decode / prepare_block_tables), Scheduler.postprocess (+ hash_blocks) --
bounds tokens/s unless it hides under the GPU step.  This replays a workload with fake tokens (oracle/make_golden.py's driver,
the one the golden traces were made with, so both sides take identical decisions) and times the three parts per step with
perf_counter.  "ref" = the unmodified reference from oracle/_ref (its prepare_* run unbound with pin_memory / .cuda()
neutralised: what it does on the host before the copies); "ours" = nanovllm/engine of this repo (flat-array BlockManager,
vectorised numpy builders writing one pinned staging buffer -- the staging copy itself is not part of this number).
Both sides run in this process's CPU, one thread, one after the other, each in its own interpreter (they share a package name).
"""
import itertools
import json
import os
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")


def run_side(side: str, name: str) -> dict:
    sys.path.insert(0, ROOT)
    if side == "ref":
        sys.path.insert(0, REF)
    else:
        sys.path.insert(0, os.path.join(ROOT, "nano-vllm_b200"))
    from oracle import make_golden as mg
    w = mg.workloads()[name]
    cfg = types.SimpleNamespace(eos=w["eos"], **w["cfg"])
    if side == "ref":
        import torch
        import nanovllm
        assert os.path.realpath(nanovllm.__file__).startswith(os.path.realpath(REF)), nanovllm.__file__
        build = mg.reference_meta_builder(torch, cfg.kvcache_block_size)
    else:
        import nanovllm
        assert not os.path.realpath(nanovllm.__file__).startswith(os.path.realpath(REF)), nanovllm.__file__
        from nanovllm.engine.model_runner import ModelRunner
        stub = types.SimpleNamespace(block_size=cfg.kvcache_block_size)
        stub.prepare_block_tables = lambda seqs: ModelRunner.prepare_block_tables(stub, seqs)
        build = lambda seqs, is_prefill: (ModelRunner.prefill_arrays(stub, seqs) if is_prefill else ModelRunner.decode_arrays(stub, seqs))
    from nanovllm.engine.scheduler import Scheduler
    from nanovllm.engine.sequence import Sequence
    from nanovllm.sampling_params import SamplingParams
    Sequence.block_size = cfg.kvcache_block_size
    Sequence.counter = itertools.count()
    sched = Scheduler(cfg)
    for p, (t, mt, ie) in zip(w["prompts"], w["sps"]):
        sched.add(Sequence(p, SamplingParams(temperature=max(t, 0.5), max_tokens=mt, ignore_eos=ie)))
    acc = {True: [0, 0.0, 0.0, 0.0, 0], False: [0, 0.0, 0.0, 0.0, 0]}       # steps, schedule, marshal, postprocess, rows
    pc = time.perf_counter
    seen = {True: False, False: False}
    while not sched.is_finished():
        t0 = pc()
        seqs, is_prefill = sched.schedule()
        t1 = pc()
        build(seqs, is_prefill)
        t2 = pc()
        toks = [mg.fake_token(s.seq_id, len(s), w["vocab"]) for s in seqs]
        t3 = pc()
        sched.postprocess(seqs, toks, is_prefill)
        t4 = pc()
        a = acc[bool(is_prefill)]
        if not seen[bool(is_prefill)]:                      # the first step of each kind pays one-time lazy initialisation: not counted
            seen[bool(is_prefill)] = True
            continue
        a[0] += 1
        a[1] += t1 - t0
        a[2] += t2 - t1
        a[3] += t4 - t3
        a[4] += len(seqs)
    out = {}
    for kind, a in (("prefill", acc[True]), ("decode", acc[False])):
        n = max(a[0], 1)
        out[kind] = {"steps": a[0], "avg_rows": round(a[4] / n, 1), "schedule_us": round(1e6 * a[1] / n, 1),
                     "marshal_us": round(1e6 * a[2] / n, 1), "postprocess_us": round(1e6 * a[3] / n, 1),
                     "total_us": round(1e6 * (a[1] + a[2] + a[3]) / n, 1)}
    return out


def main():
    if len(sys.argv) >= 3:
        print(json.dumps(run_side(sys.argv[1], sys.argv[2])))
        return
    res = {"what": __doc__.split("\n\n")[0], "cpu": os.cpu_count(), "unit": "microseconds per engine step (mean over the workload)", "workloads": {}}
    for name in ("bench", "mixed1024", "longctx128"):
        row = {}
        for side in ("ours", "ref"):
            if side == "ref" and not os.path.isdir(os.path.join(REF, "nanovllm")):
                row[side] = "oracle/_ref absent"
                continue
            env = dict(os.environ, OMP_NUM_THREADS="1")
            r = subprocess.run([sys.executable, os.path.abspath(__file__), side, name], capture_output=True, text=True, env=env)
            lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
            row[side] = json.loads(lines[-1]) if r.returncode == 0 and lines else {"error": (r.stderr or r.stdout)[-400:]}
        res["workloads"][name] = row
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
