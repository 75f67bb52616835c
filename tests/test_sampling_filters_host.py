"""Top-k / top-p / min-p sampling, host side (no GPU): SamplingParams, argument refusals of the C entry points, the
runner's per-row filter arrays and its _forward_and_sample(filters=...) glue.  Also the float64 reference of the kept
set that tests/test_gpu_sampling_filters.py checks the kernels against."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from nanovllm import SamplingParams
from nanovllm import _native as nat


# ---- float64 reference ------------------------------------------------------------------------------------------------
def kept_count_ref(x, t: float, k: int, p: float, min_p: float) -> int:
    """Number of tokens of one row that the filters keep, from the definitions (vLLM v1 semantics):
    probabilities are those of x / t; min_p keeps prob >= min_p * prob_max, top_k keeps x >= the k-th largest x,
    top_p keeps x_j iff the mass of the survivors of both with a strictly larger x is < p times their total mass.
    t, p and min_p are taken at fp32 precision, as the engine stores them."""
    x = np.asarray(x, dtype=np.float64)
    t, p, min_p = float(np.float32(t)), float(np.float32(p)), float(np.float32(min_p))
    keep = np.ones(x.shape, dtype=bool)
    if not t > 0 or not (k > 0 or p < 1.0 or min_p > 0.0):
        return int(keep.sum())
    m = x.max()
    if min_p > 0:
        keep &= np.exp((x - m) / t) >= min_p
    if 0 < k < x.size:
        keep &= x >= np.sort(x)[::-1][k - 1]
    if p < 1.0:
        vals, inv = np.unique(x[keep], return_inverse=True)              # ascending unique survivor values
        mass = np.bincount(inv, weights=np.exp((x[keep] - m) / t), minlength=vals.size)
        above = np.concatenate([np.cumsum(mass[::-1])[::-1][1:], [0.0]])  # mass strictly above each value
        ok = above < p * mass.sum()
        keep &= x >= vals[ok].min()
    return int(keep.sum())


def kept_count_range(x, t, k, p, min_p, rel=1e-6):
    """The kept counts a correct kernel may return: where the top-p mass lies within `rel` of p at two adjacent values,
    either value is accepted (the kernel sums fixed-point fp32 exponentials, the reference float64 ones)."""
    if p >= 1.0:
        c = kept_count_ref(x, t, k, p, min_p)
        return c, c
    return kept_count_ref(x, t, k, p * (1 - rel), min_p), kept_count_ref(x, t, k, min(p * (1 + rel), 1.0 - 1e-12), min_p)


def test_reference_on_a_hand_example():
    x = [3.0, 2.0, 2.0, 1.0, 0.0]
    assert kept_count_ref(x, 1.0, 1, 1.0, 0.0) == 1
    assert kept_count_ref(x, 1.0, 2, 1.0, 0.0) == 3                     # ties at the k-th are kept
    assert kept_count_ref(x, 1.0, 0, 1.0, 1.0) == 1                     # min_p = 1: the maximum only
    e = np.exp(np.array(x) - 3.0)
    z = e.sum()
    assert kept_count_ref(x, 1.0, -1, e[0] / z + 1e-6, 0.0) == 3        # mass above the 2.0s is < p: both 2.0s kept
    assert kept_count_ref(x, 1.0, -1, e[0] / z - 1e-6, 0.0) == 1
    assert kept_count_ref(x, 0.0, 1, 0.5, 0.5) == 5                     # greedy rows are not filtered
    assert kept_count_ref(x, 1.0, 5, 1.0, 0.0) == 5 and kept_count_ref(x, 1.0, 9, 1.0, 0.0) == 5


# ---- SamplingParams ---------------------------------------------------------------------------------------------------
def test_sampling_params_defaults_and_validation():
    sp = SamplingParams()
    assert (sp.top_k, sp.top_p, sp.min_p) == (-1, 1.0, 0.0) and not sp.filtered
    names = [f for f in SamplingParams.__dataclass_fields__]
    assert names == ["temperature", "max_tokens", "ignore_eos", "top_k", "top_p", "min_p"]
    assert SamplingParams(0.6, 512, False, 20, 0.95).filtered
    assert SamplingParams(top_k=0).filtered is False
    assert SamplingParams(min_p=0.05).filtered and SamplingParams(top_p=0.95).filtered
    for bad in (dict(top_k=-2), dict(top_k=1.5), dict(top_p=0.0), dict(top_p=1.01), dict(top_p=float("nan")),
                dict(min_p=-0.1), dict(min_p=1.5)):
        with pytest.raises(ValueError):
            SamplingParams(**bad)
    SamplingParams(top_k=10 ** 9, top_p=1e-6, min_p=1.0)                  # k >= vocab just means off


def test_api_surface_still_matches(golden_dir):
    import json
    import os
    import nanovllm
    from oracle.make_golden import api_surface
    ref = json.load(open(os.path.join(golden_dir, "api_surface.json")))
    got = dict(api_surface(nanovllm)["sampling_params"])
    names = [n for n, _ in api_surface(nanovllm)["sampling_params"]]
    assert names[:len(ref["sampling_params"])] == [n for n, _ in ref["sampling_params"]]
    assert names[len(ref["sampling_params"]):] == ["top_k", "top_p", "min_p"]
    assert (got["top_k"], got["top_p"], got["min_p"]) == ("-1", "1.0", "0.0")


def test_sequence_copies_the_filters():
    from nanovllm.engine.sequence import Sequence
    s = Sequence([1, 2], SamplingParams(temperature=0.6, top_k=20, top_p=0.95, min_p=0.01))
    assert (s.top_k, s.top_p, s.min_p) == (20, 0.95, 0.01)
    d = Sequence([1])
    assert (d.top_k, d.top_p, d.min_p) == (-1, 1.0, 0.0)


# ---- C ABI refusals -----------------------------------------------------------------------------------------------------
def test_filter_entry_points_refuse_bad_arguments_without_a_gpu():
    lib = nat.load()
    EINVAL, EUNSUPPORTED = -1, -2
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16
    assert lib.b200_sample_filter_workspace_words(4) == 4 * 1538
    assert lib.b200_sample_filter_workspace_words(0) == 0
    stage = lib.b200_sample_filter_stage
    assert stage(None, 16, p, p, p, p, 1, 16, 0, p, None) == EINVAL                 # logits
    assert stage(p, 16, None, p, p, p, 1, 16, 0, p, None) == EINVAL                 # temperatures
    assert stage(p, 16, p, p, p, p, 1, 16, 0, None, None) == EINVAL                 # workspace
    assert stage(p, 16, p, p, p, p, 0, 16, 0, p, None) == EINVAL                    # rows
    assert stage(p, 16, p, p, p, p, 1, 0, 0, p, None) == EINVAL                     # vocab
    assert stage(p, 16, p, p, p, p, 1, 16, -1, p, None) == EINVAL                   # stage
    assert stage(p, 16, p, p, p, p, 1, 16, 4, p, None) == EINVAL
    assert stage(p + 2, 16, p, p, p, p, 1, 16, 0, p, None) == EINVAL                # misaligned rows
    assert stage(p, 12, p, p, p, p, 2, 12, 0, p, None) == EINVAL                    # row stride not a multiple of 8
    assert stage(p, 8, p, p, p, p, 2, 16, 0, p, None) == EINVAL                     # rows overlap
    assert stage(p, 2 ** 18 + 8, p, p, p, p, 1, 2 ** 18 + 1, 0, p, None) == EUNSUPPORTED
    race = lib.b200_sample_filtered
    assert race(None, 16, p, p, p, p, 1, 16, 0, 0, 0, None, p, p, None, None) == EINVAL
    assert race(p, 16, None, p, p, p, 1, 16, 0, 0, 0, None, p, p, None, None) == EINVAL
    assert race(p, 16, p, p, p, p, 1, 16, 0, 0, 0, None, None, p, None, None) == EINVAL
    assert race(p, 16, p, p, p, p, 1, 16, 0, 0, 0, None, p, None, None, None) == EINVAL   # neither out nor out_keys
    assert race(p, 16, p, p, p, p, 0, 16, 0, 0, 0, None, p, p, None, None) == EINVAL
    assert race(p, 16, p, p, p, p, 1, -1, 0, 0, 0, None, p, p, None, None) == EINVAL
    assert race(p + 8, 16, p, p, p, p, 1, 16, 0, 0, 0, None, p, p, None, None) == EINVAL
    assert race(p, 16, p, p, p, p, 1, 16, -1, 0, 0, None, p, p, None, None) == EINVAL
    assert race(p, 16, p, p, p, p, 1, 16, 2 ** 32, 0, 0, None, p, p, None, None) == EUNSUPPORTED


# ---- runner: filter arrays and glue ------------------------------------------------------------------------------------
def _seq(t, k=-1, p=1.0, mp=0.0):
    from nanovllm.engine.sequence import Sequence
    return Sequence([1, 2, 3], SamplingParams(temperature=t, top_k=k, top_p=p, min_p=mp))


def test_runner_filter_arrays_mixed_batch():
    from nanovllm.engine.model_runner import ModelRunner
    runner = SimpleNamespace()
    seqs = [_seq(0.6, 20, 0.95), _seq(0.0, 5, 0.5, 0.1), _seq(1.0), _seq(1.0, 0, 1.0, 0.05), _seq(0.7, 10 ** 6)]
    k, p, mp = ModelRunner.filter_arrays(runner, seqs, 8)
    assert k.dtype == np.int32 and p.dtype == np.float32 and mp.dtype == np.float32 and k.shape == (8,)
    assert k.tolist() == [20, 0, 0, 0, 10 ** 6, 0, 0, 0]                 # greedy, default and padding rows: off
    assert p.tolist() == pytest.approx([0.95, 1, 1, 1, 1, 1, 1, 1])
    assert mp.tolist() == pytest.approx([0, 0, 0, 0.05, 0, 0, 0, 0])
    # no row filters: the step takes the plain sampler
    assert ModelRunner.filter_arrays(runner, [_seq(1.0), _seq(0.0, 5, 0.5), _seq(0.5, 0)], 4) is None
    assert ModelRunner.filter_arrays(runner, [_seq(0.0, 1)]) is None
    k, _, _ = ModelRunner.filter_arrays(runner, [_seq(0.5, 3)])
    assert k.tolist() == [3]


class _FakeOps:
    def __init__(self):
        self.calls = []

    def sample_filtered(self, logits, temps, top_k, top_p, min_p, seed, step, ws, out=None, index_offset=0, out_keys=None,
                        step_dev=None, reduce=None):
        self.calls.append(dict(rows=logits.shape[0], offset=index_offset, keys=out_keys is not None, reduce=reduce, ws=ws))
        if reduce is not None:
            for s in range(4):
                reduce(ws[:logits.shape[0] * 1538].view(logits.shape[0], 1538)[:, s:s + 1], "max" if s == 0 else "sum")
        tok = logits.float().argmax(-1)
        if out is not None:
            out.copy_(tok)
        if out_keys is not None:
            out_keys.copy_(0xffffffff - tok)
        return out

    @staticmethod
    def tokens_from_keys(keys):
        return 0xffffffff - (keys & 0xffffffff)

    def sample(self, *a, **k):
        raise AssertionError("the plain sampler must not run on a filtered step")

    def lm_head_sample(self, *a, **k):
        raise AssertionError("the fused LM head must not run on a filtered step")


def _runner(world_size, fused=True):
    logits = torch.randn(3, 50).to(torch.bfloat16)

    class Model:
        def __call__(self, ids, pos):
            return torch.zeros(3, 8)

        def compute_logits(self, h):
            return logits

    return SimpleNamespace(model=Model(), fused_lm_head=fused, world_size=world_size, sample_seed=7, vocab_offset=0,
                           g_keyws=torch.zeros(8, dtype=torch.int64), g_tokens=torch.zeros(8, dtype=torch.int64),
                           g_keys=torch.zeros(8, dtype=torch.int64), g_filter_ws=torch.zeros(8 * 1538, dtype=torch.int64)), logits


@pytest.mark.parametrize("world_size", [1, 2])
def test_forward_and_sample_filtered_glue(monkeypatch, world_size):
    import torch.distributed as dist
    import nanovllm.engine.model_runner as mr
    fake = _FakeOps()
    monkeypatch.setattr(mr, "ops", fake)
    reduced = []
    monkeypatch.setattr(dist, "all_reduce", lambda t, op=None: reduced.append((tuple(t.shape), op)))
    runner, logits = _runner(world_size)
    runner._sample_filtered = lambda *a: mr.ModelRunner._sample_filtered(runner, *a)
    runner._reduce_filter_words = mr.ModelRunner._reduce_filter_words
    filters = (torch.zeros(3, dtype=torch.int32), torch.ones(3), torch.zeros(3))
    mr.ModelRunner._forward_and_sample(runner, torch.zeros(3, dtype=torch.int64), torch.zeros(3, dtype=torch.int64),
                                       torch.ones(3), None, 3, filters=filters)
    assert len(fake.calls) == 1 and fake.calls[0]["rows"] == 3              # the logits path, though the fused head is on
    assert torch.equal(runner.g_tokens[:3], logits.float().argmax(-1))
    if world_size == 1:
        assert fake.calls[0]["reduce"] is None and not reduced
    else:
        # one all-reduce per stage (MAX, then SUM x 3) and the keys' MAX
        assert [op for _, op in reduced] == [dist.ReduceOp.MAX] + [dist.ReduceOp.SUM] * 3 + [dist.ReduceOp.MAX]
        assert fake.calls[0]["keys"]


def test_forward_and_sample_without_filters_touches_nothing_new(monkeypatch):
    """filters=None runs today's code: a runner without any filter attribute still works (fused head on)."""
    import nanovllm.engine.model_runner as mr
    seen = {}

    class Ops:
        @staticmethod
        def lm_head_sample(hidden, lm_head, temps, seed, step, key_ws, out=None, **kw):
            seen["fused"] = hidden.shape[0]
            out.zero_()

        @staticmethod
        def sample_filtered(*a, **k):
            raise AssertionError("no filters: the filtered sampler must not run")

    monkeypatch.setattr(mr, "ops", Ops)
    from nanovllm.utils.context import reset_context, set_context

    class Model:
        lm_head = torch.zeros(50, 8)

        def __call__(self, ids, pos):
            return torch.zeros(2, 8)

        def last_token_rows(self, h):
            return h

    runner = SimpleNamespace(model=Model(), fused_lm_head=True, world_size=1, sample_seed=3, vocab_offset=0,
                             g_keyws=torch.zeros(4, dtype=torch.int64), g_tokens=torch.ones(4, dtype=torch.int64),
                             g_keys=torch.zeros(4, dtype=torch.int64))
    set_context(False)
    mr.ModelRunner._forward_and_sample(runner, torch.zeros(2, dtype=torch.int64), torch.zeros(2, dtype=torch.int64),
                                       torch.ones(2), None, 2)
    reset_context()
    assert seen == {"fused": 2}
