"""Per-token logprobs on the GPU (csrc/logprobs.cu): the kernels against the float64 reference of tests/logprob_ref.py,
adversarial rows, split-count invariance, determinism, vocab sharding, penalised rows, and the engine (eager against the
logits it computed, graphed against the CPU oracle, tokens unchanged by asking, default step unchanged, tensor
parallelism)."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from gpu_helpers import make_oracle, oracle_full_logits
from logprob_ref import logprob_tolerance, logprobs_ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ops():
    from nanovllm import ops as _ops
    return _ops


def check_rows(ops, x, ks, tokens, out):
    """Every logprob row of `out` (packed, numpy) against the reference on bf16 logits x [rows, vocab]."""
    xs = x.float().cpu().numpy()
    for r, k in enumerate(ks):
        if k < 0:
            continue
        ids, lps, rank = ops.unpack_logprobs(out[r], k)
        lp, want_rank, top, tlp = logprobs_ref(xs[r], k, int(tokens[r]))
        assert ids[0] == tokens[r] and rank == want_rank, (r, rank, want_rank)
        assert ids[1:].tolist() == top.tolist(), (r, ids[1:], top)
        got = lps.astype(np.float64)
        want = np.concatenate([[lp], tlp])
        assert (np.abs(got - want) <= logprob_tolerance(want)).all(), (r, got - want)


def _run(ops, x, ks, tokens):
    k = torch.tensor(ks, dtype=torch.int32, device="cuda")
    t = torch.as_tensor(tokens, dtype=torch.int64).cuda()
    ws = ops.logprob_workspace(x.shape[0])
    out = ops.logprobs(x, k, t, workspace=ws).cpu().numpy()
    assert int(ws.abs().sum()) == 0, "the workspace is not zero after the call"
    return out


@pytest.mark.parametrize("vocab", [151936, 1001])
@pytest.mark.parametrize("rows", [1, 7, 64, 512])
def test_kernels_match_reference(ops, vocab, rows):
    g = torch.Generator().manual_seed(vocab + rows)
    width = (vocab + 7) // 8 * 8
    full = (torch.randn(rows, width, generator=g) * 3).to(torch.bfloat16).cuda()
    x = full[:, :vocab]
    rnd = random.Random(rows)
    ks = [[-1, 0, 1, 5, 20][i % 5] for i in range(rows)]
    xs = x.float().cpu().numpy()
    tokens = [int(np.argmax(xs[i])) if i % 3 == 0 else rnd.randrange(vocab) for i in range(rows)]
    out = _run(ops, x, ks, tokens)
    check_rows(ops, x, ks, tokens, out)


def test_adversarial_rows(ops):
    vocab = 151936
    rows = []
    rows.append(torch.zeros(vocab))                                           # all equal
    r = torch.full((vocab,), -4.0)
    r[77777] = 30.0                                                            # one dominant token
    rows.append(r)
    r = torch.full((vocab,), -30.0)                                            # a long flat tail below 2^-33 of the max
    r[5] = 0.0
    rows.append(r)
    r = torch.randint(-3, 3, (vocab,)).float()                                # massive ties at the top and at the k boundary
    rows.append(r)
    r = torch.arange(vocab).float() * 1e-3                                     # ascending: every element enters the list
    rows.append(r)
    x = torch.stack(rows).to(torch.bfloat16).cuda()
    for k in (0, 1, 20):
        ks = [k] * x.shape[0]
        tokens = [3, 77777, 100, 9, vocab - 1]
        check_rows(ops, x, ks, tokens, _run(ops, x, ks, tokens))


def test_split_invariance_and_determinism(ops):
    """A row's result is the same bits whether it runs alone (16 splits) or in batches of 64, 512 and 1024 rows (down to
    one CTA per row), and from launch to launch."""
    vocab = 151936
    g = torch.Generator().manual_seed(11)
    x = (torch.randn(1024, vocab, generator=g) * 2).to(torch.bfloat16).cuda()
    x[1, :] = 0.5
    ks = [20, 5, 0, 17] * 256
    tokens = [(i * 7919) % vocab for i in range(1024)]
    ref = _run(ops, x, ks, tokens)
    assert np.array_equal(_run(ops, x, ks, tokens), ref)
    for n in (1, 64, 512):
        assert np.array_equal(_run(ops, x[:n], ks[:n], tokens[:n]), ref[:n]), n
    assert np.array_equal(_run(ops, x[2:3], ks[2:3], tokens[2:3]), ref[2:3])


@pytest.mark.parametrize("shards", [2, 4])
def test_sharded_equals_unsharded(ops, shards):
    vocab, rows = 151936, 33
    g = torch.Generator().manual_seed(shards)
    x = (torch.randn(rows, vocab, generator=g) * 3).to(torch.bfloat16).cuda()
    x[0, :] = 1.0
    ks = [(i * 3) % 21 for i in range(rows)]
    ks[5] = -1
    tokens = [(i * 10007) % vocab for i in range(rows)]
    want = _run(ops, x, ks, tokens)
    k = torch.tensor(ks, dtype=torch.int32, device="cuda")
    t = torch.tensor(tokens, dtype=torch.int64, device="cuda")
    width = vocab // shards
    parts = [x[:, s * width:(s + 1) * width].contiguous() for s in range(shards)]
    wss = [ops.logprob_workspace(rows) for _ in range(shards)]
    keys = [torch.zeros(rows * ops.LOGPROB_MAX_K, dtype=torch.int64, device="cuda") for _ in range(shards)]

    def allreduce(lo, hi, op):
        words = [ops.logprob_words(w, rows, lo, hi) for w in wss]
        comb = torch.stack(words).amax(0) if op == "max" else torch.stack(words).sum(0)
        for w in words:
            w.copy_(comb)

    for s in range(shards):
        ops.logprobs_topk(parts[s], k, wss[s], keys[s], index_offset=s * width)
    allreduce(0, 1, "max")
    lib = ops.nat.load()
    for s in range(shards):
        ops.nat.check(lib.b200_logprob_restore(parts[s].data_ptr(), parts[s].stride(0), k.data_ptr(), rows, width, s * width,
                                               t.data_ptr(), wss[s].data_ptr(), None, 0, None))
    allreduce(1, 2, "max")
    for s in range(shards):
        ops.nat.check(lib.b200_logprob_rank(parts[s].data_ptr(), parts[s].stride(0), k.data_ptr(), rows, width,
                                            wss[s].data_ptr(), None))
    allreduce(2, 4, "sum")
    gathered = torch.stack(keys)
    outs = []
    for s in range(shards):
        out = torch.zeros(rows, ops.LOGPROB_OUT_WORDS, dtype=torch.int32, device="cuda")
        ops.nat.check(lib.b200_logprob_finish(k.data_ptr(), rows, t.data_ptr(), gathered.data_ptr(), shards,
                                              wss[s].data_ptr(), out.data_ptr(), out[:, 21:].data_ptr(),
                                              out[:, 42:].data_ptr(), out.stride(0), None))
        outs.append(out.cpu().numpy())
    for s in range(shards):
        for r in range(rows):
            if ks[r] >= 0:
                n = 1 + ks[r]
                assert np.array_equal(outs[s][r, :n], want[r, :n]) and np.array_equal(outs[s][r, 21:21 + n], want[r, 21:21 + n])
                assert outs[s][r, 42] == want[r, 42]
        assert int(wss[s].abs().sum()) == 0


def test_penalised_rows_see_the_raw_logits(ops):
    """Top-k, save, apply, the filtered sampler, restore and finish: the logprobs are those of the logits before the
    penalties, the logits are raw again, the tokens are those of penalties + sampler without the logprob kernels, and the
    workspace is zero again."""
    from penalty_ref import entries_of, history
    vocab, rows, capacity = 151936, 24, 600
    rnd = random.Random(3)
    g = torch.Generator().manual_seed(3)
    x0 = (torch.randn(rows, vocab, generator=g) * 3).to(torch.bfloat16).cuda()
    hists = [history(rnd.sample(range(vocab), 200), [rnd.randrange(vocab) for _ in range(100)]) for _ in range(rows)]
    ents = [entries_of(h) for h in hists]
    off = np.zeros(rows + 1, np.int32)
    np.cumsum([e.size for e in ents], out=off[1:])
    cuda = dict(device="cuda")
    slots = torch.tensor([i if i % 3 else -1 for i in range(rows)], dtype=torch.int32, **cuda)
    pending = torch.tensor([rnd.randrange(vocab) for _ in range(rows)], dtype=torch.int64, **cuda)
    r = torch.full((rows,), 1.3, **cuda)
    f = torch.full((rows,), 0.5, **cuda)
    p = torch.full((rows,), 1.5, **cuda)
    temps = torch.tensor([0.0 if i % 3 == 0 else 0.7 for i in range(rows)], **cuda)
    top_k = torch.tensor([20 if i % 2 else 0 for i in range(rows)], dtype=torch.int32, **cuda)
    ks = [[-1, 0, 5, 20][i % 4] for i in range(rows)]
    k = torch.tensor(ks, dtype=torch.int32, **cuda)

    def fresh():
        hist, lens = ops.penalty_history(rows, capacity)
        ops.penalty_load(hist, lens, torch.from_numpy(np.concatenate(ents)).cuda(), torch.from_numpy(off).cuda(),
                         torch.arange(rows, dtype=torch.int32, **cuda))
        return hist, lens

    hist, lens = fresh()                                                       # without the logprob kernels
    xp = x0.clone()
    ops.penalty_apply(xp, hist, lens, slots, r, f, p, pending)
    want_tok = ops.sample_filtered(xp, temps, top_k, None, None, seed=9, step=4, workspace=ops.filter_workspace(rows))
    hist, lens = fresh()
    x = x0.clone()
    ws, keys = ops.logprob_workspace(rows), torch.zeros(rows * ops.LOGPROB_MAX_K, dtype=torch.int64, **cuda)
    saved = ops.logprob_saved_buffer(rows, capacity)
    out = torch.zeros(rows, ops.LOGPROB_OUT_WORDS, dtype=torch.int32, **cuda)
    ops.logprobs_topk(x, k, ws, keys)
    ops.logprobs_save(x, k, ws, saved, hist, lens, slots, pending)
    ops.penalty_apply(x, hist, lens, slots, r, f, p, pending)
    assert not torch.equal(x, x0)
    tok = ops.sample_filtered(x, temps, top_k, None, None, seed=9, step=4, workspace=ops.filter_workspace(rows))
    assert torch.equal(tok, want_tok)
    ops.logprobs_finish(x, k, tok, ws, keys, out, saved=saved, capacity=capacity)
    changed = (x != x0).any(1).cpu().numpy()
    for i in range(rows):                                                      # rows without logprobs stay penalised
        assert changed[i] == (ks[i] < 0 and i % 3 != 0), i
    assert int(ws.abs().sum()) == 0
    check_rows(ops, x0, ks, tok.cpu().numpy(), out.cpu().numpy())


# ---- engine ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    import tempfile
    from nanovllm.utils.synthetic import PRESETS, make_model_dir, random_weights
    d = tempfile.mkdtemp(prefix="logprob_tiny_")
    make_model_dir(os.path.join(d, "tiny"), "tiny", seed=1234)
    oracle = make_oracle(PRESETS["tiny"], random_weights(PRESETS["tiny"], seed=1234), "fused")
    return os.path.join(d, "tiny"), oracle, PRESETS["tiny"]["vocab_size"]


CFG = dict(max_model_len=256, max_num_seqs=16, max_num_batched_tokens=256, kvcache_block_size=16, num_kvcache_blocks=160)
PEN = dict(repetition_penalty=1.3, presence_penalty=1.5, frequency_penalty=0.5)


def _prompts(vocab, n, seed, shared_prefix=0):
    rnd = random.Random(seed)
    prefix = [rnd.randint(2, vocab - 1) for _ in range(shared_prefix)]
    return [prefix + [rnd.randint(2, vocab - 1) for _ in range(rnd.randint(3, 90))] for _ in range(n)]


def _mixed(n, max_tokens=12):
    from nanovllm import SamplingParams
    out = []
    for i in range(n):
        extra = [{}, dict(top_k=20, top_p=0.9), PEN, {}][i % 4]
        out.append(SamplingParams(temperature=0.0 if i % 3 == 0 else 0.8, max_tokens=max_tokens + i % 5, ignore_eos=True,
                                  logprobs=[5, None, 20, 0, None, 3][i % 6], **extra))
    return out


@pytest.mark.parametrize("setting", ["chunked+prefix", "preempt"])
def test_engine_eager_matches_the_logits_it_computed(tiny, setting):
    from nanovllm import LLM
    model_dir, _, vocab = tiny
    if setting == "chunked+prefix":
        prompts, kw = _prompts(vocab, 12, seed=3, shared_prefix=40), dict(max_num_batched_tokens=96)
    else:
        prompts, kw = _prompts(vocab, 12, seed=4), dict(num_kvcache_blocks=30)
    sps = _mixed(len(prompts), 30)
    llm = LLM(model_dir, enforce_eager=True, **{**CFG, **kw})
    try:
        runner = llm.model_runner
        model = runner.model
        logits_q, seqs_q, checked = [], [], [0]
        orig_logits, orig_launch, orig_collect = model.compute_logits, runner.launch, runner.collect

        def compute_logits(h):
            out = orig_logits(h)
            logits_q.append(out.clone())
            return out

        def launch(seqs, is_prefill, *a):
            seqs_q.append([(s, s.logprobs_k if not is_prefill or s.num_cached_tokens + s.num_scheduled_tokens >= s.num_tokens
                            else -1) for s in seqs])
            return orig_launch(seqs, is_prefill, *a)

        def collect():
            toks = orig_collect()
            x, rows = logits_q.pop(0), seqs_q.pop(0)
            ks = [k for _, k in rows]
            if any(k >= 0 for k in ks):
                check_rows(ops_mod(), x, ks, toks, runner.last_logprobs)
                checked[0] += sum(k >= 0 for k in ks)
            else:
                assert runner.last_logprobs is None
            return toks

        model.compute_logits, runner.launch, runner.collect = compute_logits, launch, collect
        outs = llm.generate(prompts, sps, use_tqdm=False)
    finally:
        llm.exit()
    assert checked[0] > 100
    for o, sp in zip(outs, sps):
        if sp.logprobs is None:
            assert set(o) == {"text", "token_ids"}
            continue
        assert len(o["logprobs"]) == len(o["token_ids"]) == sp.max_tokens
        for d, t in zip(o["logprobs"], o["token_ids"]):
            assert next(iter(d)) == t and len(d) in (sp.logprobs, sp.logprobs + 1)
        assert o["cumulative_logprob"] == sum(d[t].logprob for d, t in zip(o["logprobs"], o["token_ids"]))


def ops_mod():
    from nanovllm import ops
    return ops


def test_engine_graphed_tokens_unchanged_and_oracle(tiny, monkeypatch):
    from nanovllm import LLM, SamplingParams
    monkeypatch.setenv("B200_SAMPLE_SEED", "77")
    model_dir, oracle, vocab = tiny
    prompts = _prompts(vocab, 14, seed=5)
    sps = _mixed(len(prompts))
    plain = [sp.replace(logprobs=None) for sp in sps]
    llm = LLM(model_dir, enforce_eager=False, **CFG)                 # same seed, fresh engine: the same RNG steps
    try:
        base = [o["token_ids"] for o in llm.generate(prompts, plain, use_tqdm=False)]
    finally:
        llm.exit()
    llm = LLM(model_dir, enforce_eager=False, **CFG)
    try:
        runner = llm.model_runner
        assert all(runner.lgraph_kernels[b] == runner.fgraph_kernels[b] + 5 for b in runner.graph_bs)
        kernels = dict(runner.graph_kernels), dict(runner.fgraph_kernels)
        outs = llm.generate(prompts, sps, use_tqdm=False)
        # a default step after logprob requests: same graphs, same upload and read-back bytes as before any
        d = SamplingParams(temperature=0.7, max_tokens=8, ignore_eos=True)
        llm.generate(prompts[:5], [d] * 5, use_tqdm=False)
        assert runner.h2d_bytes_last == runner.d_off["bt"] + 8 * runner.max_blocks * 4 and runner.d2h_bytes_last == 5 * 8
        assert (dict(runner.graph_kernels), dict(runner.fgraph_kernels)) == kernels
        llm.generate(prompts[:5], [d.replace(logprobs=2)] * 5, use_tqdm=False)
        assert runner.h2d_bytes_last == runner.d_off["bt"] + 8 * runner.max_blocks * 4 + runner.f_bytes
        assert runner.d2h_bytes_last == 5 * 8 + 5 * 4 * 43
    finally:
        llm.exit()
    assert [o["token_ids"] for o in outs] == base, "asking for logprobs changed the sampled tokens"
    for p, sp, o in zip(prompts, sps, outs):
        if sp.logprobs is None:
            continue
        toks = o["token_ids"]
        lg = oracle_full_logits(oracle, p + toks[:-1]).numpy().astype(np.float64)
        for i, (t, d) in enumerate(zip(toks, o["logprobs"])):
            row = lg[len(p) - 1 + i]
            ref = row - row.max() - np.log(np.exp(row - row.max()).sum())
            tol = 6 * 2 ** -8 * np.abs(row).max()
            for tid, lp in d.items():
                assert abs(lp.logprob - ref[tid]) <= tol, (i, tid, lp.logprob, ref[tid])
            if sp.temperature == 0.0 and not sp.penalised and sp.logprobs > 0:
                assert d[t].rank == 1, "a greedy row's token is its top-1 entry"


def test_tp2_on_one_gpu_over_gloo_with_logprobs():
    env = dict(os.environ, B200_TP_BACKEND="gloo", B200_TP_ONE_DEVICE="1", B200_TP_ALLREDUCE="nccl")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29573", os.path.join(ROOT, "tests", "tp_logprob_worker.py")]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "TP_LOGPROB_RESULT" in r.stdout and '"ok": true' in r.stdout
