"""Per-token logprobs, host side (no GPU): SamplingParams, the float64 reference on hand-checked rows, the dict
construction, the runner's per-row k, the engine's attachment of result rows over both branches of the overlapped loop
(chunked prefill, preemption, EOS) and the C entry points' refusals."""
import ctypes
import itertools
import math
import types

import numpy as np
import pytest

from logprob_ref import logprobs_ref, vllm_dict
from nanovllm import SamplingParams
from nanovllm import _native as nat


# ---- SamplingParams ---------------------------------------------------------------------------------------------------
def test_sampling_params_logprobs_validation_and_surface():
    import copy
    import dataclasses
    import pickle
    import nanovllm
    from nanovllm.sampling_params import Logprob
    assert SamplingParams().logprobs is None
    assert SamplingParams(0.6, 10, False, -1, 1.0, 0.0, 0.0, 0.0, 1.0, 5).logprobs == 5     # positional, last
    for ok in (0, 1, 20):
        assert SamplingParams(logprobs=ok).logprobs == ok
    for bad in (-1, 21, True, False, 1.0, "3"):
        with pytest.raises(ValueError):
            SamplingParams(logprobs=bad)
    for kw in (dict(prompt_logprobs=1), dict(logprob_token_ids=[3]), dict(logprobs_mode="raw_logits"),
               dict(logprobs_mode="processed_logprobs")):
        with pytest.raises(ValueError):
            SamplingParams(**kw)
    SamplingParams(prompt_logprobs=None, logprob_token_ids=None, logprobs_mode="raw_logprobs")   # the defaults: accepted
    with pytest.raises(TypeError):
        SamplingParams(not_a_parameter=1)
    assert "logprobs" not in [f.name for f in dataclasses.fields(SamplingParams)]
    assert "Logprob" not in nanovllm.__all__
    sp = SamplingParams(temperature=0.6, logprobs=5, presence_penalty=1.0)
    assert sp == SamplingParams(temperature=0.6, logprobs=5, presence_penalty=1.0)
    assert sp != sp.replace(logprobs=4) and sp != sp.replace(logprobs=None)
    assert pickle.loads(pickle.dumps(sp)) == sp and copy.copy(sp) == sp and copy.deepcopy(sp) == sp
    assert sp.replace(max_tokens=3).logprobs == 5 and sp.__replace__(top_k=5).logprobs == 5
    assert sp.as_dict()["logprobs"] == 5 and len(sp.as_dict()) == 10 and "logprobs=5" in repr(sp)
    plain = SamplingParams()
    assert len(plain.as_dict()) == 9 and "logprobs" not in repr(plain)
    assert SamplingParams(logprobs=0).as_dict()["logprobs"] == 0
    with pytest.raises(ValueError):
        sp.replace(logprobs=-1)
    lp = Logprob(-0.5, 1)
    assert (lp.logprob, lp.rank) == (-0.5, 1) and lp == Logprob(-0.5, 1)
    with pytest.raises(dataclasses.FrozenInstanceError):
        lp.rank = 2


def test_sequence_carries_k():
    from nanovllm.engine.sequence import Sequence
    assert Sequence([1], SamplingParams(logprobs=3)).logprobs_k == 3
    s = Sequence([1])
    assert s.logprobs_k == -1 and s.logprob_rows is None


# ---- the reference ----------------------------------------------------------------------------------------------------
def test_reference_all_equal_row():
    lp, rank, top, tlp = logprobs_ref(np.zeros(8), 3, 5)
    assert rank == 8 and top.tolist() == [0, 1, 2] and np.allclose(tlp, -math.log(8)) and lp == pytest.approx(-math.log(8))


def test_reference_ties_at_the_boundary_and_at_the_top():
    x = np.array([1.0, 3.0, 2.0, 3.0, 2.0, 2.0, 0.0])
    _, rank, top, _ = logprobs_ref(x, 4, 5)
    assert top.tolist() == [1, 3, 2, 4]                           # ties at the top and at k: ascending ids
    assert rank == 5                                              # #{x >= 2}: ties raise the rank
    _, rank, top, _ = logprobs_ref(x, 1, 3)
    assert top.tolist() == [1] and rank == 2                      # the tied maximum with the larger id has rank 2


def test_reference_values_and_dicts():
    x = np.array([2.0, 1.0, 0.0, -1.0])
    z = np.log(np.exp(x).sum())
    lp, rank, top, tlp = logprobs_ref(x, 2, 3)                    # sampled outside the top 2
    assert lp == pytest.approx(-1.0 - z) and rank == 4 and top.tolist() == [0, 1]
    d = vllm_dict(3, lp, rank, top, tlp)
    assert list(d) == [3, 0, 1] and d[3][1] == 4 and [d[0][1], d[1][1]] == [1, 2]
    lp, rank, top, tlp = logprobs_ref(x, 2, 1)                    # sampled inside: its top-k entry, first position
    d = vllm_dict(1, lp, rank, top, tlp)
    assert list(d) == [1, 0] and d[1] == (pytest.approx(1.0 - z), 2) and len(d) == 2
    assert vllm_dict(2, -3.0, 3, [], []) == {2: (-3.0, 3)}       # logprobs=0: the sampled token only


def test_logprob_dicts_from_packed_rows():
    from nanovllm import ops
    from nanovllm.engine.llm_engine import logprob_dicts
    from nanovllm.sampling_params import Logprob

    def row(ids, lps, rank):
        r = np.zeros(ops.LOGPROB_OUT_WORDS, np.int32)
        r[:len(ids)] = ids
        r[ops.LOGPROB_LP_COL:ops.LOGPROB_LP_COL + len(lps)] = np.asarray(lps, np.float32).view(np.int32)
        r[ops.LOGPROB_RANK_COL] = rank
        return r

    rows = [row([7, 3, 7], [-2.5, -0.5, -2.5], 2), row([9, 3, 4], [-4.0, -0.25, -1.0], 6)]
    dicts, cum = logprob_dicts(rows, 2)
    assert dicts[0] == {7: Logprob(-2.5, 2), 3: Logprob(-0.5, 1)} and list(dicts[0]) == [7, 3]
    assert dicts[1] == {9: Logprob(-4.0, 6), 3: Logprob(-0.25, 1), 4: Logprob(-1.0, 2)} and list(dicts[1]) == [9, 3, 4]
    assert cum == -6.5 and isinstance(cum, float)
    dicts, cum = logprob_dicts(rows, 0)
    assert dicts == [{7: Logprob(-2.5, 2)}, {9: Logprob(-4.0, 6)}]


# ---- runner -----------------------------------------------------------------------------------------------------------
def test_runner_logprob_arrays():
    from nanovllm.engine.model_runner import ModelRunner
    from nanovllm.engine.sequence import Sequence
    a = Sequence(list(range(10, 30)), SamplingParams(logprobs=5))
    b = Sequence([1, 2, 3])
    c = Sequence([4, 5], SamplingParams(logprobs=0))
    assert ModelRunner.logprob_arrays([b], 4) is None
    a.num_cached_tokens, a.num_scheduled_tokens = 0, 8                # a prompt chunk that is not the last
    c.num_cached_tokens, c.num_scheduled_tokens = 0, 2
    assert ModelRunner.logprob_arrays([a, b], prefill=True) is None
    k = ModelRunner.logprob_arrays([a, b, c], prefill=True)
    assert k.dtype == np.int32 and k.tolist() == [-1, -1, 0]
    a.num_cached_tokens, a.num_scheduled_tokens = 8, 12
    assert ModelRunner.logprob_arrays([a, b, c], prefill=True).tolist() == [5, -1, 0]
    assert ModelRunner.logprob_arrays([a, b, c], 8).tolist() == [5, -1, 0] + [-1] * 5


# ---- engine attachment ------------------------------------------------------------------------------------------------
class _LogprobRunner:
    """test_engine_overlap's fake runner plus result rows: row i of a step carries the step's token for sequence i as its
    sampled id and len(sequence) at launch as its logprob, so every attached row names the position it belongs to."""

    def __init__(self, block_size, vocab):
        from test_engine_overlap import FakeRunner
        self.inner = FakeRunner(block_size, vocab)
        self.rows = []
        self.last_logprobs = None

    def call(self, name, *a):
        return getattr(self, name)(*a)

    def stage_decode(self, seqs):
        return self.inner.stage_decode(seqs)

    def launch(self, seqs, is_prefill, staged=None, src=None):
        from nanovllm import ops
        self.inner.launch(seqs, is_prefill, staged, src)
        r = np.zeros((len(seqs), ops.LOGPROB_OUT_WORDS), np.int32)
        r[:, 0] = self.inner.queue[-1]
        r[:, ops.LOGPROB_LP_COL] = np.asarray([len(s) for s in seqs], np.float32).view(np.int32)
        r[:, ops.LOGPROB_RANK_COL] = 1
        self.rows.append(r if any(s.logprobs_k >= 0 for s in seqs) else None)

    def collect(self):
        self.last_logprobs = self.rows.pop(0)
        return self.inner.collect()

    def check_peer_exchange(self):
        pass


@pytest.mark.parametrize("seed", [5])
def test_engine_attaches_one_row_per_completion_token(seed):
    """Random workloads (mixed ignore_eos / EOS batches, preemption, chunking, prefix hits) with every other request asking
    for logprobs: each finished request has exactly one dict per completion token, keyed by that token and carrying the
    length the sequence had when the token was sampled; the others get no logprobs."""
    from oracle.make_golden import fuzz_workloads
    from nanovllm.engine.llm_engine import LLMEngine
    from nanovllm.engine.scheduler import Scheduler
    from nanovllm.engine.sequence import Sequence
    checked = preempted = 0
    for w in fuzz_workloads(seed, 60):
        cfg = types.SimpleNamespace(eos=w["eos"], **w["cfg"])
        Sequence.block_size = cfg.kvcache_block_size
        Sequence.counter = itertools.count()
        eng = object.__new__(LLMEngine)
        eng.scheduler = Scheduler(cfg)
        eng.model_runner = _LogprobRunner(cfg.kvcache_block_size, w["vocab"])
        orig = eng.scheduler.preempt

        def preempt(seq, orig=orig):
            nonlocal preempted
            preempted += 1
            orig(seq)
        eng.scheduler.preempt = preempt
        seqs = []
        for i, (p, (t, mt, ie)) in enumerate(zip(w["prompts"], w["sps"])):
            seqs.append(Sequence(p, SamplingParams(temperature=t, max_tokens=mt, ignore_eos=ie,
                                                   logprobs=(i % 3) * 2 if i % 2 == 0 else None)))
            eng.scheduler.add(seqs[-1])
        finished = []
        eng._run_overlapped(lambda f, n, dt: finished.extend(f))
        assert len(finished) == len(seqs)
        for s in seqs:
            if s.logprob_rows is None:
                continue
            assert len(s.logprob_rows) == s.num_completion_tokens
            for i, (tok, row) in enumerate(zip(s.completion_token_ids, s.logprob_rows)):
                assert row[0] == tok
                assert row[21:22].view(np.float32)[0] == s.num_prompt_tokens + i
            checked += 1
    assert checked > 50 and preempted > 0


def test_generate_output_shape(monkeypatch):
    """generate() adds "logprobs" and "cumulative_logprob" to the requests that asked, and nothing to the others."""
    from nanovllm.engine.llm_engine import LLMEngine
    from nanovllm.engine.scheduler import Scheduler
    from nanovllm.engine.sequence import Sequence
    from nanovllm.sampling_params import Logprob
    cfg = types.SimpleNamespace(eos=-1, max_num_seqs=4, max_num_batched_tokens=64, kvcache_block_size=16,
                                num_kvcache_blocks=16)
    Sequence.block_size = 16
    eng = object.__new__(LLMEngine)
    eng.scheduler = Scheduler(cfg)
    eng.model_runner = _LogprobRunner(16, 100)
    eng.config = types.SimpleNamespace(hf_config=types.SimpleNamespace(vocab_size=100), max_model_len=64)
    eng.tokenizer = types.SimpleNamespace(decode=lambda toks: "")
    eng.rank, eng._mirrors = 0, False
    outs = eng.generate([[1, 2, 3], [4, 5]], [SamplingParams(max_tokens=3, ignore_eos=True, logprobs=0),
                                              SamplingParams(max_tokens=2, ignore_eos=True)], use_tqdm=False)
    assert set(outs[0]) == {"text", "token_ids", "logprobs", "cumulative_logprob"} and set(outs[1]) == {"text", "token_ids"}
    lps = outs[0]["logprobs"]
    assert [list(d) for d in lps] == [[t] for t in outs[0]["token_ids"]]
    assert [d[t] for d, t in zip(lps, outs[0]["token_ids"])] == [Logprob(3.0, 1), Logprob(4.0, 1), Logprob(5.0, 1)]
    assert outs[0]["cumulative_logprob"] == 12.0


# ---- C ABI refusals -----------------------------------------------------------------------------------------------------
def test_logprob_entry_points_refuse_bad_arguments_without_a_gpu():
    lib = nat.load()
    EINVAL, EUNSUP = -1, -2
    buf = ctypes.create_string_buffer(8192)
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16
    assert lib.b200_logprob_workspace_words(4) == 32
    assert lib.b200_logprob_workspace_words(0) == 0 and lib.b200_logprob_workspace_words(1025) == 0

    def refused(fn, ok, pointers, values, code=EINVAL):
        for i in pointers:
            args = list(ok)
            args[i] = None
            assert fn(*args) == code, (fn.__name__, i)
        for i, v in values:
            args = list(ok)
            args[i] = v
            assert fn(*args) == (v[1] if isinstance(v, tuple) else code), (fn.__name__, i, v)

    # logits, stride, k, rows, vocab, index_offset, workspace, topk_keys, stream
    topk = lib.b200_logprob_topk
    ok = [p, 64, p, 2, 64, 0, p, p, None]
    refused(topk, ok, (0, 2, 6, 7), ())
    for i, v, code in ((3, 0, EINVAL), (3, 1025, EINVAL), (4, 0, EINVAL), (5, -1, EINVAL), (0, p + 2, EINVAL),
                       (1, 60, EINVAL), (1, 32, EINVAL), (4, (1 << 18) + 8, EUNSUP), (5, (1 << 18) - 32, EUNSUP)):
        args = list(ok)
        args[i] = v
        if i == 4 and v > 64:
            args[1] = v                                            # a stride that fits the row
        assert topk(*args) == code, (i, v)
    # logits, stride, k, rows, vocab, index_offset, history, lengths, num_slots, capacity, slots, pending, ws, saved, stream
    save = lib.b200_logprob_save
    ok = [p, 64, p, 2, 64, 0, p, p, 4, 16, p, None, p, p, None]
    refused(save, ok, (0, 2, 6, 7, 10, 12, 13), ((8, 0), (9, 0), (5, -1), (3, 0), (3, 1025)))
    # logits, stride, k, rows, vocab, index_offset, tokens, ws, saved, capacity, stream
    restore = lib.b200_logprob_restore
    ok = [p, 64, p, 2, 64, 0, p, p, p, 16, None]
    refused(restore, ok, (0, 2, 6, 7), ((9, 0), (5, -1), (0, p + 8)))
    # logits, stride, k, rows, vocab, ws, stream
    rank = lib.b200_logprob_rank
    ok = [p, 64, p, 2, 64, p, None]
    refused(rank, ok, (0, 2, 5), ((3, 0), (3, 1025), (4, 0), (1, 12)))
    args = list(ok)
    args[1] = args[4] = (1 << 18) + 8
    assert rank(*args) == EUNSUP
    # k, rows, tokens, topk_keys, sources, ws, out_ids, out_logprobs, out_rank, out_stride, stream
    finish = lib.b200_logprob_finish
    ok = [p, 2, p, p, 1, p, p, p, p, 43, None]
    refused(finish, ok, (0, 2, 3, 5, 6, 7, 8), ((1, 0), (1, 1025), (4, 0), (4, 65), (9, 20)))
