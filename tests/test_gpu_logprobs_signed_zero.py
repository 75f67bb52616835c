"""Ties between +0 and -0 logits (csrc/logprobs.cu): -0 is folded onto +0 in the top-k keys, so equal logits order by
token id alone, as DESIGN.md 3.3.2 and the float64 reference of tests/logprob_ref.py specify."""
import numpy as np
import pytest
import torch

from logprob_ref import logprobs_ref

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("vocab,rows", [(151936, 1), (151936, 64), (1001, 3)])
def test_signed_zero_ties_order_by_id(vocab, rows):
    from nanovllm import ops
    width = (vocab + 7) // 8 * 8
    g = torch.Generator().manual_seed(vocab + rows)
    x = -(torch.rand(rows, width, generator=g) * 4 + 1)                         # every logit < 0 ...
    zeros = torch.arange(0, vocab, 37)                                          # ... but a spread of zeros, the maximum
    x[:, zeros] = torch.where(torch.arange(zeros.numel()) % 2 == 0, -0.0, 0.0)  # alternately -0 and +0
    x = x.to(torch.bfloat16).cuda()[:, :vocab]
    assert (x[:, zeros].view(torch.int16) != 0).any(), "no -0 in the row"
    ks = [20] * rows
    tokens = [int(zeros[(3 * r + 1) % zeros.numel()]) for r in range(rows)]     # a +0 or -0 token
    k = torch.tensor(ks, dtype=torch.int32, device="cuda")
    out = ops.logprobs(x, k, torch.tensor(tokens, dtype=torch.int64, device="cuda")).cpu().numpy()
    xs = x.float().cpu().numpy()
    for r in range(rows):
        ids, lps, rank = ops.unpack_logprobs(out[r], 20)
        lp, want_rank, top, tlp = logprobs_ref(xs[r], 20, tokens[r])
        assert ids[1:].tolist() == top.tolist() == zeros[:20].tolist()
        assert rank == want_rank == zeros.numel()
        assert np.abs(lps.astype(np.float64) - np.concatenate([[lp], tlp])).max() <= 1e-6 + 2.0 ** -22 * abs(lp)
