"""Differential fuzzing of the host bookkeeping against the reference's own classes.

The committed golden traces (tests/golden/trace_*.json) pin seven hand-picked workloads.  This test adds a few hundred
random small workloads (page sizes 2..256, tight caches that force preemption, shared prefixes, duplicates, EOS stops,
tiny token budgets that force chunking): the REFERENCE's Scheduler / BlockManager / Sequence / prepare_* were run over
them by `oracle/make_golden.py --fuzz SEED 150 tests/golden/fuzz_seedSEED.json`, which stored the step-by-step digests
(one short hash per chunk of 32 steps), and the product must produce the same digests.
"""
import itertools
import json
import os
import types

import pytest

from oracle.make_golden import COMPACT_CHUNK, compact_steps, drive, fuzz_workloads

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("seed", [1, 2])
def test_random_workloads_match_reference(seed):
    from nanovllm.engine.scheduler import Scheduler
    from nanovllm.engine.sequence import Sequence
    from nanovllm.sampling_params import SamplingParams
    from test_bookkeeping_golden import product_meta_builder
    n = 150
    ref = json.load(open(os.path.join(ROOT, "tests", "golden", f"fuzz_seed{seed}.json")))
    assert len(ref) == n
    preempting = prefix_hits = 0
    for i, (w, gold) in enumerate(zip(fuzz_workloads(seed, n), ref)):
        cfg = types.SimpleNamespace(eos=w["eos"], **w["cfg"])
        Sequence.block_size = cfg.kvcache_block_size
        Sequence.counter = itertools.count()
        make = lambda p, t, mt, ie: Sequence(p, SamplingParams(temperature=t, max_tokens=mt, ignore_eos=ie))
        sched = Scheduler(cfg)
        count = [0]
        orig = sched.preempt

        def counting(seq, orig=orig, count=count):
            count[0] += 1
            return orig(seq)
        sched.preempt = counting
        hits = [0]
        orig_alloc = sched.block_manager.allocate

        def counting_alloc(seq, num_cached, orig_alloc=orig_alloc, hits=hits):
            hits[0] += num_cached > 0
            return orig_alloc(seq, num_cached)
        sched.block_manager.allocate = counting_alloc
        got = drive(make, sched, cfg.kvcache_block_size, product_meta_builder(cfg.kvcache_block_size), w)
        assert got["num_steps"] == gold["num_steps"], f"workload {i}: {w['cfg']}"
        mine = compact_steps(got["steps"])
        for c in range(0, len(mine), 8):
            k = c // 8 * COMPACT_CHUNK
            assert mine[c:c + 8] == gold["steps"][c:c + 8], \
                f"workload {i} ({w['cfg']}), steps {k}..{k + COMPACT_CHUNK - 1}: product {got['steps'][k:k + COMPACT_CHUNK]} differ from the reference"
        for key in ("final_state", "outputs", "num_prefill_steps", "sum_decode_batch"):
            assert got[key] == gold[key], f"workload {i}: {key}"
        preempting += count[0] > 0
        prefix_hits += hits[0] > 0
    # the fuzzer must actually reach the interesting branches (measured: ~50 preempting, ~130 prefix-hit workloads of 150)
    assert preempting >= 25 and prefix_hits >= 60, (preempting, prefix_hits)
