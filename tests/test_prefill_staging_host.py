"""The prefill staging buffer holds prepare_prefill's whole plan at its limits (no GPU): S sequences, T new tokens, block
tables W wide, and every optional region staged at once (top-k / top-p / min-p, penalties, logprobs)."""
import types

import numpy as np
import pytest
import torch

from nanovllm import SamplingParams


def _host_staging(nbytes: int):
    """A _Staging whose 'device' buffer is a CPU tensor, so that prepare_prefill runs without a GPU."""
    from nanovllm.engine.model_runner import _Staging
    st = _Staging.__new__(_Staging)
    st.hosts = [torch.zeros(nbytes, dtype=torch.uint8)]
    st.dev = torch.zeros(nbytes, dtype=torch.uint8)
    st.host_nps = [h.numpy() for h in st.hosts]
    return st


def _runner(T, S, W, block_size):
    from nanovllm.engine.model_runner import ModelRunner
    r = ModelRunner.__new__(ModelRunner)
    r.config = types.SimpleNamespace(max_num_batched_tokens=T, max_num_seqs=S, max_model_len=W * block_size)
    r.block_size, r.cap_bs, r.max_blocks = block_size, S, W
    r.kv_fp8, r.kv_scratch, r.sample_step = False, None, 0
    r._init_penalty_slots(S)
    r._stage_penalty_entries = lambda seqs, load, which, prefill: (np.zeros(len(seqs) + 1, np.int32), 0)
    r._load_penalty_slots = lambda *a: None
    r.pstage = _host_staging(ModelRunner.prefill_staging_bytes(max(T, S), S, W, False))
    return r


@pytest.mark.parametrize("T,S,W,block_size", [(256, 16, 16, 16), (2048, 64, 16, 256), (64, 4, 8, 16)])
def test_worst_case_prefill_plan_fits(T, S, W, block_size):
    """One sequence with W blocks (a prefix hit on a prompt of max_model_len tokens), S - 1 one-token prompts, T tokens
    in all, every request filtered, penalised and asking for logprobs."""
    from nanovllm.engine.sequence import Sequence
    from nanovllm.utils.context import reset_context
    Sequence.block_size = block_size
    sp = SamplingParams(temperature=0.6, top_k=20, top_p=0.9, min_p=0.05, presence_penalty=1.0, logprobs=20)
    long_len = W * block_size
    head = Sequence(list(range(1, long_len + 1)), sp)
    head.block_table = list(range(W))
    head.num_scheduled_tokens = T - (S - 1)
    head.num_cached_tokens = long_len - head.num_scheduled_tokens
    assert head.num_cached_tokens >= 0
    seqs = [head]
    for i in range(S - 1):
        s = Sequence([7 + i], sp)
        s.block_table = [W + i]
        s.num_scheduled_tokens = 1
        seqs.append(s)
    r = _runner(T, S, W, block_size)
    try:
        ids, pos, temps, step = r.prepare_prefill(seqs)
    finally:
        reset_context()
    assert r.h2d_bytes_last <= r.pstage.dev.numel()
    assert ids.numel() == T and temps.numel() == S
    assert r.step_logprobs is not None and r.step_logprobs.tolist() == [20] * S
    assert r.step_filters is not None and r.step_penalties is not None
