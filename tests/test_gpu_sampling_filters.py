"""Top-k / top-p / min-p sampling on the GPU (csrc/sample_filter.cu + sample_masked_kernel): the threshold tau against
the float64 reference of tests/test_sampling_filters_host.py, the draw, determinism, vocab sharding, and the engine."""
import os
import random
import subprocess
import sys

import pytest
import torch

from gpu_helpers import check_greedy_against_oracle, make_oracle
from test_sampling_filters_host import kept_count_range, kept_count_ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ops():
    from nanovllm import ops as _ops
    return _ops


def key16(x: torch.Tensor) -> torch.Tensor:
    """Order-preserving key of bf16 values (-0 folded onto +0), as the kernels compute it."""
    b = x.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF
    b = torch.where(b == 0x8000, torch.zeros_like(b), b)
    return torch.where((b & 0x8000) != 0, b ^ 0xFFFF, b ^ 0x8000)


def params(rows, seed, greedy_every=0):
    """Mixed per-row (t, k, p, min_p), every kind of row represented."""
    rnd = random.Random(seed)
    out = []
    for r in range(rows):
        t = rnd.choice([0.1, 0.6, 1.0, 2.0])
        if greedy_every and r % greedy_every == 0:
            t = 0.0
        kind = r % 5
        k = rnd.choice([1, 20, 1000]) if kind in (0, 3) else -1
        p = rnd.choice([0.5, 0.95]) if kind in (1, 3) else 1.0
        mp = rnd.choice([0.05, 0.2]) if kind in (2, 3) else 0.0
        out.append((t, k, p, mp))
    return out


def tensors(prm):
    t = torch.tensor([a[0] for a in prm], dtype=torch.float32, device="cuda")
    k = torch.tensor([max(a[1], 0) for a in prm], dtype=torch.int32, device="cuda")
    p = torch.tensor([a[2] for a in prm], dtype=torch.float32, device="cuda")
    mp = torch.tensor([a[3] for a in prm], dtype=torch.float32, device="cuda")
    return t, k, p, mp


def random_logits(rows, width, seed, scale=2.5):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(rows, width, generator=g) * scale).to(torch.bfloat16)


@pytest.mark.parametrize("vocab,width", [(151936, 151936), (75968, 75968), (1001, 1024)])
def test_tau_matches_float64_reference(ops, vocab, width):
    ks = [1, 20, 1000, vocab - 1, vocab, vocab + 7, -1]
    combos = [(t, k, p, mp) for t in (0.1, 0.6, 1.0, 2.0) for k in ks for p in (1e-6, 0.5, 0.95, 1.0) for mp in (0.0, 0.05, 1.0)]
    rows = len(combos)
    x = random_logits(rows, width, seed=vocab)
    x[:, vocab:] = float("nan")                                           # never read: the view is [:, :vocab]
    rnd = random.Random(1)
    for r, (_, k, _, _) in enumerate(combos):
        if r % 2 and k > 0:                                               # hundreds of equal values straddling the k-th
            kk = min(k, vocab)
            srt = x[r, :vocab].float().sort(descending=True).values
            val = srt[max(0, kk - 150)]
            cols = torch.tensor(rnd.sample(range(vocab), min(300, vocab // 3)))
            x[r, cols] = val.to(torch.bfloat16)
    t, k, p, mp = tensors(combos)
    g = x.cuda()
    view = g[:, :vocab]
    ws = ops.filter_workspace(rows)
    ops.sample_filtered(view, t, k, p, mp, seed=3, step=1, workspace=ws)
    tau = ops.filter_tau_keys(ws, rows).cpu()
    got = (key16(view.cpu()) >= tau[:, None].to(torch.int32)).sum(-1)
    bad = []
    for r, (tr, kr, pr, mr) in enumerate(combos):
        lo, hi = kept_count_range(x[r, :vocab].float().numpy(), tr, kr, pr, mr)
        if not lo <= int(got[r]) <= hi:
            bad.append((r, combos[r], int(got[r]), lo, hi))
    assert not bad, f"{len(bad)} rows off the reference, e.g. {bad[:5]}"
    w = ws.view(rows, -1).clone()
    w[:, 1] = 0
    assert not w.any(), "the workspace must be zero again after the race (tau words aside)"


def test_every_token_is_in_the_kept_set(ops):
    rows, vocab = 64, 151936
    prm = params(rows, seed=5)
    t, k, p, mp = tensors(prm)
    ws = ops.filter_workspace(rows)
    for step in range(12):
        x = random_logits(rows, vocab, seed=100 + step, scale=1.0 + step % 3)
        g = x.cuda()
        tok = ops.sample_filtered(g, t, k, p, mp, seed=11, step=step, workspace=ws).cpu()
        tau = ops.filter_tau_keys(ws, rows).cpu()
        keys = key16(x)
        assert (keys.gather(1, tok[:, None]).squeeze(1) >= tau.to(torch.int32)).all(), f"step {step}"
        if step < 2:
            for r in range(0, rows, 7):
                lo, hi = kept_count_range(x[r].float().numpy(), *prm[r])
                assert lo <= int((keys[r] >= int(tau[r])).sum()) <= hi


@pytest.mark.parametrize("cfg", [(0.7, 3, 1.0, 0.0), (0.7, -1, 0.8, 0.0), (1.0, -1, 1.0, 0.2), (0.7, 5, 0.9, 0.05)])
def test_distribution_is_the_renormalised_softmax(ops, cfg):
    t, k, p, mp = cfg
    base = torch.tensor([2.0, 1.0, 0.0, -1.0, 0.5, -3.0, 1.5, 0.2])
    rows = 40000
    logits = base.to(torch.bfloat16).repeat(rows, 1).cuda()
    tt, kk, pp, mm = tensors([cfg] * rows)
    ws = ops.filter_workspace(rows)
    got = ops.sample_filtered(logits, tt, kk, pp, mm, seed=123, step=7, workspace=ws).cpu()
    n_kept = kept_count_ref(base.numpy(), t, k, p, mp)
    kept = base.argsort(descending=True)[:n_kept]
    want = torch.zeros(8)
    want[kept] = torch.softmax(base[kept].double() / t, 0).float()
    freq = torch.bincount(got, minlength=8).float() / rows
    assert (freq - want).abs().max().item() < 0.012, (freq, want)
    assert freq[want == 0].sum().item() == 0.0, "an excluded token was drawn"


def test_unfiltered_and_greedy_rows_are_unchanged(ops):
    rows, vocab = 96, 151936
    prm = [((0.6, 20, 0.95, 0.0) if r % 3 == 0 else ((0.8, -1, 1.0, 0.0) if r % 3 == 1 else (0.0, 20, 0.5, 0.1)))
           for r in range(rows)]
    t, k, p, mp = tensors(prm)
    g = random_logits(rows, vocab, seed=9).cuda()
    ws = ops.filter_workspace(rows)
    for step in (1, 2, 3):
        got = ops.sample_filtered(g, t, k, p, mp, seed=77, step=step, workspace=ws).cpu()
        plain = ops.sample(g, t, seed=77, step=step).cpu()
        sel = torch.tensor([r % 3 != 0 for r in range(rows)])
        assert torch.equal(got[sel], plain[sel]), f"step {step}"


@pytest.mark.parametrize("shards", [2, 4])
def test_sharded_equals_unsharded_bit_for_bit(ops, shards):
    rows, vocab = 24, 151936
    prm = params(rows, seed=shards, greedy_every=7)
    t, k, p, mp = tensors(prm)
    g = random_logits(rows, vocab, seed=21).cuda()
    ws = ops.filter_workspace(rows)
    full = ops.sample_filtered(g, t, k, p, mp, seed=5, step=3, workspace=ws).cpu()
    tau_full = ops.filter_tau_keys(ws, rows).cpu()
    width = vocab // shards
    parts = [g[:, i * width:(i + 1) * width] for i in range(shards)]
    wss = [ops.filter_workspace(rows) for _ in range(shards)]
    for stage in range(4):                       # torch max / sum over the shards stand in for the all-reduces
        for part, w in zip(parts, wss):
            ops.sample_filter_stage(stage, part, t, k, p, mp, w)
        words = [ops.filter_stage_words(w, rows, stage) for w in wss]
        comb = torch.stack(words).amax(0) if stage == 0 else torch.stack(words).sum(0)
        for w in words:
            w.copy_(comb)
    keys = []
    for i, (part, w) in enumerate(zip(parts, wss)):
        kk = torch.empty(rows, dtype=torch.int64, device="cuda")
        ops.sample_filter_race(part, t, k, p, mp, 5, 3, w, index_offset=i * width, out_keys=kk)
        keys.append(kk)
    tokens = ops.tokens_from_keys(torch.stack(keys).amax(0)).cpu()
    assert torch.equal(tokens, full)
    for w in wss:
        assert torch.equal(ops.filter_tau_keys(w, rows).cpu(), tau_full)


def test_split_count_invariance_and_determinism(ops):
    rows, vocab = 1024, 151936
    prm = params(rows, seed=8, greedy_every=11)
    t, k, p, mp = tensors(prm)
    g = random_logits(rows, vocab, seed=31).cuda()
    ws = ops.filter_workspace(rows)
    full = ops.sample_filtered(g, t, k, p, mp, seed=9, step=4, workspace=ws).cpu()
    again = ops.sample_filtered(g, t, k, p, mp, seed=9, step=4, workspace=ws).cpu()
    other = ops.sample_filtered(g, t, k, p, mp, seed=9, step=5, workspace=ws).cpu()
    assert torch.equal(full, again), "a re-launch on the same workspace must be identical"
    assert not torch.equal(full, other)
    for r in (0, 1, 3, 17, 130, 511, 1023):
        n = r + 1
        sub = ops.sample_filtered(g[:n], t[:n], k[:n], p[:n], mp[:n], seed=9, step=4, workspace=ws).cpu()
        assert int(sub[r]) == int(full[r]), f"row {r} in a batch of {n}"


def test_fp32_logits_are_refused(ops):
    from nanovllm._native import B200Error
    t, k, p, mp = tensors([(1.0, 5, 1.0, 0.0)])
    with pytest.raises(B200Error, match="code -2"):
        ops.sample_filtered(torch.zeros(1, 64, device="cuda"), t, k, p, mp, 0, 0, ops.filter_workspace(1))


# ---- engine ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny_dir(tmp_path_factory):
    from nanovllm.utils.synthetic import make_model_dir
    return make_model_dir(str(tmp_path_factory.mktemp("models") / "tiny"), "tiny", seed=1234)


def _generate(tiny_dir, eager, prompts, sps, **kw):
    from nanovllm import LLM
    cfg = dict(max_model_len=256, max_num_seqs=16, max_num_batched_tokens=256, kvcache_block_size=16, num_kvcache_blocks=160)
    cfg.update(kw)
    llm = LLM(tiny_dir, enforce_eager=eager, **cfg)
    try:
        return [o["token_ids"] for o in llm.generate(prompts, sps, use_tqdm=False)]
    finally:
        llm.exit()


@pytest.mark.parametrize("eager", [True, False])
def test_engine_mixed_filters(tiny_dir, eager, monkeypatch):
    """Rows without filters get exactly the tokens of a run where no request filters, and top_k=1 rows at temperature 1
    are greedy; ignore_eos and varied max_tokens make the engine stage steps early and move rows between steps."""
    from nanovllm import SamplingParams
    from nanovllm.utils.synthetic import PRESETS, random_weights
    monkeypatch.setenv("B200_SAMPLE_SEED", "4242")
    vocab = PRESETS["tiny"]["vocab_size"]
    rnd = random.Random(2)
    prompts = [[rnd.randint(2, vocab - 1) for _ in range(rnd.randint(3, 60))] for _ in range(14)]
    plain = [SamplingParams(temperature=0.8, max_tokens=6 + (i * 5) % 23, ignore_eos=True) for i in range(14)]
    mixed = []
    for i, sp in enumerate(plain):
        if i % 3 == 0:
            mixed.append(SamplingParams(temperature=1.0, max_tokens=sp.max_tokens, ignore_eos=True, top_k=1))
        elif i % 3 == 1:
            mixed.append(SamplingParams(temperature=0.6, max_tokens=sp.max_tokens, ignore_eos=True, top_k=20, top_p=0.95,
                                        min_p=0.01))
        else:
            mixed.append(sp)
    want = _generate(tiny_dir, eager, prompts, plain)
    got = _generate(tiny_dir, eager, prompts, mixed)
    oracle = make_oracle(PRESETS["tiny"], random_weights(PRESETS["tiny"], seed=1234), "fused")
    for i, (w, g) in enumerate(zip(want, got)):
        assert len(g) == mixed[i].max_tokens
        if i % 3 == 2:
            assert g == w, f"unfiltered request {i} changed when other requests filter"
        elif i % 3 == 0:
            check_greedy_against_oracle(oracle, prompts[i], g)


def test_engine_qwen3_recommended_setting_at_batch_256(tiny_dir):
    from nanovllm import SamplingParams
    from nanovllm.utils.synthetic import PRESETS
    vocab = PRESETS["tiny"]["vocab_size"]
    rnd = random.Random(6)
    prompts = [[rnd.randint(2, vocab - 1) for _ in range(rnd.randint(3, 30))] for _ in range(256)]
    sps = [SamplingParams(temperature=0.6, max_tokens=24, top_p=0.95, top_k=20, ignore_eos=True) for _ in prompts]
    out = _generate(tiny_dir, False, prompts, sps, max_num_seqs=256, max_num_batched_tokens=8192, num_kvcache_blocks=1024)
    assert [len(o) for o in out] == [24] * 256
    assert all(0 <= t < vocab for o in out for t in o)


def test_tp2_on_one_gpu_over_gloo_with_filters():
    env = dict(os.environ, B200_TP_BACKEND="gloo", B200_TP_ONE_DEVICE="1", B200_TP_ALLREDUCE="nccl")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29567", os.path.join(ROOT, "tests", "tp_filter_worker.py")]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "TP_FILTER_RESULT" in r.stdout and '"ok": true' in r.stdout
