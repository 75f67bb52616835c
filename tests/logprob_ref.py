"""Float64 reference of the per-token logprobs (DESIGN.md 3.3.2) that tests/test_gpu_logprobs.py checks the kernels against:
log_softmax over the full vocabulary of the raw bf16 logits, the top k by (value descending, token id ascending), the
sampled token's rank counted with >=, and vLLM's dict construction."""
import numpy as np


def logprobs_ref(x, k: int, sampled: int):
    """One row: (sampled logprob, rank, top-k ids, top-k logprobs), all from the float64 log_softmax of x."""
    x = np.asarray(x, dtype=np.float64)
    m = x.max()
    lp = (x - m) - np.log(np.exp(x - m).sum())
    top = np.lexsort((np.arange(x.size), -x))[:k]                 # value descending, then id ascending
    rank = int((x >= x[sampled]).sum())
    return float(lp[sampled]), rank, top.astype(np.int64), lp[top]


def vllm_dict(sampled: int, sampled_lp: float, rank: int, top_ids, top_lps) -> dict:
    """{token_id: (logprob, rank)} as vLLM builds it: the sampled token first, then the top k with ranks 1..k; a sampled
    token inside the top k ends up with its top-k entry, in the first position."""
    d = {int(sampled): (float(sampled_lp), int(rank))}
    for j, (t, v) in enumerate(zip(top_ids, top_lps)):
        d[int(t)] = (float(v), j + 1)
    return d


def logprob_tolerance(ref) -> np.ndarray:
    """The kernel bar: expf's 2 ulp, the 2^-40 fixed point over at most 2^18 tokens and one fp32 rounding."""
    return 1e-6 + 2.0 ** -22 * np.abs(np.asarray(ref, dtype=np.float64))
