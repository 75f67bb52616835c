"""Qwen3 mixture-of-experts MLP on the GPU (DESIGN.md 3.7): the routing kernel exactly against the reference, the grouped
GEMMs and the combine against float64 under stated bars over adversarial routings and T = 1 .. 16384, determinism and
token-permutation equivariance, CUDA-graph replays with a new routing each time, the model against tests/moe_ref.py's
oracle, and the engine end to end (chunked prefill, prefix cache, preemption, fp8 KV cache, graphs, sampling features,
two tensor-parallel ranks)."""
import os
import random
import subprocess
import sys
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from gpu_helpers import check_greedy_against_oracle, record
from moe_ref import Qwen3MoeRef, gap_safe_sequences, prefill_ctx, route_ref, tile_table_ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BM = 128
# routing-weight bar: fp32 expf (<= 2 ulp), a tree sum of <= 256 terms and two correctly rounded divisions
ROUTE_REL = 2.0 ** -19


def _ops():
    from nanovllm import ops
    return ops


# ---- routing -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("norm", [True, False])
@pytest.mark.parametrize("E,k", [(16, 4), (128, 8), (256, 16), (8, 8)])
def test_route_exact_ids_and_weights(E, k, norm):
    ops = _ops()
    g = torch.Generator().manual_seed(E * 31 + k)
    T = 3001
    lg = (torch.randn(T, E, generator=g) * 3).to(torch.bfloat16)
    lg[::3] = (torch.randint(-4, 5, (len(lg[::3]), E), generator=g) * 0.5).to(torch.bfloat16)   # many exact ties
    lg[1, :] = 0.0                                                                                 # all tied
    ids, w = ops.moe_route(lg.cuda(), k, norm)
    rid, _ = route_ref(lg, k, norm)
    assert torch.equal(ids.cpu().long(), rid)
    p = torch.softmax(lg.double(), -1).gather(1, rid)
    if norm:
        p = p / p.sum(-1, keepdim=True)
    err = ((w.cpu().double() - p).abs() / p.clamp_min(1e-300)).max().item()
    assert err <= ROUTE_REL, err


# ---- grouped GEMMs and combine ------------------------------------------------------------------------------------------
def _routing(kind: str, T: int, E: int, k: int, g: torch.Generator) -> torch.Tensor:
    """int32 [T, k] expert ids (distinct per token) for an adversarial routing."""
    if kind == "random":
        return torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(T)]).int()
    if kind == "one_expert":                      # every token's rank 0 on expert 3, the rest on fixed neighbours
        return torch.tensor([[(3 + j) % E for j in range(k)]] * T, dtype=torch.int32)
    if kind == "one_token_per_expert":            # token t on experts t, t + T, ... (T * k == E)
        return torch.tensor([[(t + j * T) % E for j in range(k)] for t in range(T)], dtype=torch.int32)
    if kind == "mostly_empty":                    # only experts {0, 1, ..., k} in use
        return torch.stack([torch.randperm(k + 1, generator=g)[:k] for _ in range(T)]).int()
    if kind == "tile_edges":                      # segments of BM - 1, BM, BM + 1 and 2 BM + 1 rows (k = 1)
        ids = torch.cat([torch.full((c,), e) for e, c in ((1, BM - 1), (2, BM), (5, BM + 1), (7, 2 * BM + 1))])
        return ids[torch.randperm(len(ids), generator=g)].reshape(-1, 1).int()
    raise ValueError(kind)


def _bf16_bar(y, a):
    """bf16-rounded GEMM output: half an ulp of the result plus fp32 accumulation over k (2^-16 of sum |x w|)."""
    return 2.0 ** -8 * y.abs() + 2.0 ** -16 * a


def _check_rows(n):
    if n <= 4096:
        return torch.arange(n)
    return torch.tensor(sorted(set(range(0, n, 37)) | set(range(n - 200, n))))


CASES = [("random", 1, 4), ("random", 7, 4), ("random", 200, 4), ("random", 2048, 8), ("random", 16384, 4),
         ("one_expert", 300, 4), ("one_token_per_expert", 4, 4), ("mostly_empty", 500, 4), ("tile_edges", 641, 1)]


@pytest.mark.parametrize("dims", ["small", "tp2", "30b-a3b"])
@pytest.mark.parametrize("kind,T,k", CASES)
def test_grouped_gemms_and_combine_against_float64(kind, T, k, dims):
    ops = _ops()
    E, H, I = dict(small=(16, 256, 128), tp2=(16, 256, 64), **{"30b-a3b": (128, 2048, 768)})[dims]   # tp2: tiny-moe per rank
    if dims == "tp2" and kind not in ("random", "tile_edges"):
        pytest.skip("one k tile per down projection: random routings and tile edges")
    if dims == "30b-a3b" and T > 2048:
        pytest.skip("30B-A3B dims at up to 2048 tokens (the float64 reference is CPU-bound); 16384 runs at the small dims")
    g = torch.Generator().manual_seed(T * 7 + k)
    ids = _routing(kind, T, E, k, g)
    w = torch.rand(T, k, generator=g) + 0.05
    x = torch.randn(T, H, generator=g).to(torch.bfloat16)
    gu = (0.05 * torch.randn(E, 2 * I, H, generator=g)).to(torch.bfloat16)
    dn = (0.05 * torch.randn(E, H, I, generator=g)).to(torch.bfloat16)
    xd, gud, dnd, idsd, wd = x.cuda(), gu.cuda(), dn.cuda(), ids.cuda(), w.cuda()
    perm, tiles = ops.moe_align(idsd, E)
    xp = ops.moe_gather(xd, k, perm)
    act = ops.moe_linear(xp, gud, tiles, ops.EPI_SILU, 64)
    y = ops.moe_linear(act, dnd, tiles, ops.EPI_BF16, 64)
    out = ops.moe_combine(y, perm, wd)
    torch.cuda.synchronize()
    perm_c, tiles_c = perm.cpu().long(), tiles.cpu()
    # the tile table and the permutation
    segs, want_tiles = tile_table_ref(ids, E, BM)
    n_tiles = int(tiles_c[0, 0])
    assert n_tiles == len(want_tiles) and int(tiles_c[0, 1]) == T * k
    assert [tuple(r) for r in tiles_c[1:1 + n_tiles, :3].tolist()] == want_tiles
    flat = ids.reshape(-1).long()
    assert sorted(perm_c.tolist()) == list(range(T * k))
    starts = torch.tensor([s for s, _ in segs])
    counts = torch.tensor([c for _, c in segs])
    assert ((perm_c >= starts[flat]) & (perm_c < starts[flat] + counts[flat])).all()
    assert torch.equal(xp.cpu()[perm_c], x.repeat_interleave(k, 0))
    # gate_up + SiluAndMul, per permuted row, against float64 on the same bf16 operands
    sel = _check_rows(T * k)
    exp = torch.empty(T * k, dtype=torch.long)
    exp[perm_c] = flat
    xs, es = xp.cpu()[sel].double(), exp[sel]
    a_in = act.cpu()[sel].double()
    hy, ha = torch.empty(len(sel), 2 * I, dtype=torch.float64), torch.empty(len(sel), 2 * I, dtype=torch.float64)
    dy, da = torch.empty(len(sel), H, dtype=torch.float64), torch.empty(len(sel), H, dtype=torch.float64)
    for e in torch.unique(es).tolist():                  # one expert at a time: a per-row weight gather would not fit
        r = es == e
        we, de = gu[e].double(), dn[e].double()
        hy[r], ha[r] = xs[r] @ we.t(), xs[r].abs() @ we.abs().t()
        dy[r], da[r] = a_in[r] @ de.t(), a_in[r].abs() @ de.abs().t()      # down on the kernel's own activations
    gg, uu = hy[:, :I], hy[:, I:]
    eg, eu = _bf16_bar(gg, ha[:, :I]), _bf16_bar(uu, ha[:, I:])
    sg = gg * torch.sigmoid(gg)
    want = sg * uu
    tol = 2.0 ** -8 * want.abs() + 1.1 * eg * uu.abs() + sg.abs() * eu + eg * eu + 1e-30
    r_act = ((act.cpu()[sel].double() - want).abs() / tol).max().item()
    r_down = ((y.cpu()[sel].double() - dy).abs() / (_bf16_bar(dy, da) + 1e-30)).max().item()
    # combine on the kernel's own expert outputs: one bf16 rounding of an fp32 chain of k products
    yk = y.cpu().double()[perm_c].reshape(T, k, H)
    cw = (w.double()[:, :, None] * yk).sum(1)
    ca = (w.double()[:, :, None] * yk.abs()).sum(1)
    r_comb = ((out.cpu().double() - cw).abs() / (2.0 ** -8 * cw.abs() + k * 2.0 ** -23 * ca + 1e-30)).max().item()
    record(f"moe_gemm_{dims}_{kind}_T{T}_k{k}", dict(act_err_over_bar=r_act, down_err_over_bar=r_down, combine_err_over_bar=r_comb))
    assert r_act <= 1.0 and r_down <= 1.0 and r_comb <= 1.0, (r_act, r_down, r_comb)


def _mlp_inputs(T, E=128, H=2048, I=768, k=8, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(T, H, generator=g, device="cuda").to(torch.bfloat16)
    lg = (3 * torch.randn(T, E, generator=g, device="cuda")).to(torch.bfloat16)
    gu = (0.02 * torch.randn(E, 2 * I, H, generator=g, device="cuda")).to(torch.bfloat16)
    dn = (0.02 * torch.randn(E, H, I, generator=g, device="cuda")).to(torch.bfloat16)
    return x, lg, gu, dn, k


@pytest.mark.parametrize("T", [1, 33, 256, 3000])
def test_deterministic_and_permutation_equivariant(T):
    ops = _ops()
    x, lg, gu, dn, k = _mlp_inputs(T, seed=T)
    a = ops.moe_mlp(x, lg, gu, dn, k, True)
    for _ in range(3):
        assert torch.equal(ops.moe_mlp(x, lg, gu, dn, k, True), a)
    p = torch.randperm(T, device="cuda")
    b = ops.moe_mlp(x[p].contiguous(), lg[p].contiguous(), gu, dn, k, True)
    assert torch.equal(b, a[p])
    # a token's output does not depend on the rest of the batch
    one = ops.moe_mlp(x[T // 2:T // 2 + 1].contiguous(), lg[T // 2:T // 2 + 1].contiguous(), gu, dn, k, True)
    assert torch.equal(one, a[T // 2:T // 2 + 1])


@pytest.mark.parametrize("world", [2, 4])
def test_tensor_parallel_shards_sum_to_the_whole_mlp(world):
    """Each rank's MLP on its moe_intermediate_size shard of every expert; the shards' outputs sum to the unsharded MLP
    up to the bf16 roundings of the partial sums."""
    ops = _ops()
    T, E, H, I, k = 300, 16, 256, 256, 4
    x, lg, gu, dn, _ = _mlp_inputs(T, E, H, I, k, seed=world)
    whole = ops.moe_mlp(x, lg, gu, dn, k, True).double()
    s = I // world
    total = torch.zeros_like(whole)
    for r in range(world):
        gu_r = torch.cat([gu[:, r * s:(r + 1) * s], gu[:, I + r * s:I + (r + 1) * s]], 1).contiguous()
        total += ops.moe_mlp(x, lg, gu_r, dn[:, :, r * s:(r + 1) * s].contiguous(), k, True).double()
    rel = ((total - whole).norm() / whole.norm()).item()
    assert rel < 1e-2, rel


def test_graph_replays_follow_new_routings():
    ops = _ops()
    T = 256
    x, lg, gu, dn, k = _mlp_inputs(T, seed=5)
    sx, slg = x.clone(), lg.clone()
    out = torch.empty_like(x)
    ops.moe_mlp(sx, slg, gu, dn, k, True, out=out)          # warm-up outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.moe_mlp(sx, slg, gu, dn, k, True, out=out)
    for seed in range(4):
        x2, lg2, _, _, _ = _mlp_inputs(T, seed=100 + seed)
        if seed == 1:
            lg2[:, 7] = 100.0                                # every token on expert 7
        if seed == 2:
            lg2[:, :120] = -100.0                            # 8 experts take everything
        sx.copy_(x2)
        slg.copy_(lg2)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, ops.moe_mlp(x2, lg2, gu, dn, k, True)), seed


# ---- model and engine -----------------------------------------------------------------------------------------------------
GAP_ULPS = 4.0         # the oracle's k-th / (k+1)-th routing logit gap, in bf16 ulps of the token's largest |router logit|
# Candidate tokens are accepted at a wider gap: the CPU oracle's bf16 GEMMs round the router logits of a longer packed
# batch a little differently than those of the one growing sequence the workload is drawn with.
DRAW_GAP_ULPS = 6.0


def _moe_weights(preset, seed=1234):
    from nanovllm.utils.synthetic import PRESETS, random_weights
    return random_weights(PRESETS[preset], seed=seed)


@pytest.mark.parametrize("preset", ["tiny-moe", "tiny-moe-g8"])
def test_moe_forward_matches_oracle(preset):
    from nanovllm import ops
    from nanovllm.models.qwen3_moe import Qwen3MoeForCausalLM
    from nanovllm.utils.context import reset_context, set_context
    from nanovllm.utils.synthetic import PRESETS, hf_config_dict
    d = PRESETS[preset]
    weights = _moe_weights(preset)
    oracle = Qwen3MoeRef.from_preset(d, weights, rounding="fused", max_pos=4096)
    lens = [23, 61, 9]
    seqs = gap_safe_sequences(oracle, d["vocab_size"], lens, seed=3, gap_ulps=DRAW_GAP_ULPS)
    ids = torch.tensor(sum(seqs, []))
    pos = torch.cat([torch.arange(n) for n in lens])
    ctx = prefill_ctx(lens)
    cu, m = ctx.cu_seqlens_q, ctx.max_seqlen_q
    want = oracle.forward(ids, pos, ctx, None).float()
    gap = oracle.min_gap_over_ulp()
    assert gap >= GAP_ULPS, gap                            # the precondition: no selection is within bf16 reach of a flip
    model = Qwen3MoeForCausalLM(SimpleNamespace(**hf_config_dict(d)), 0, 1, "cuda", max_position=4096)
    for name, w in weights.items():
        model.load_hf_tensor(name, w)
    set_context(True, cu.cuda(), cu.cuda(), m, m, None, None, None)
    got = model(ids.cuda(), pos.cuda()).float().cpu()
    reset_context()
    rel = ((got - want).norm() / want.norm()).item()
    row = ((got - want).norm(dim=-1) / want.norm(dim=-1)).max().item()
    record(f"moe_forward_{preset}", dict(rel_l2=rel, worst_row_rel_l2=row, min_gap_ulps=gap, tokens=int(ids.numel())))
    assert torch.isfinite(got).all() and rel < 2e-2 and row < 5e-2, (rel, row)


@pytest.fixture(scope="module")
def moe_dir(tmp_path_factory):
    from nanovllm.utils.synthetic import make_model_dir
    return make_model_dir(str(tmp_path_factory.mktemp("moe") / "ckpt"), "tiny-moe", seed=1234)


def _generate(path, params=None, **kw):
    from nanovllm import LLM, SamplingParams
    from nanovllm.utils.synthetic import PRESETS
    rnd = random.Random(7)
    vocab = PRESETS["tiny-moe"]["vocab_size"]
    shared = [rnd.randint(2, vocab - 1) for _ in range(40)]                    # prefix-cache hits
    prompts = [shared + [rnd.randint(2, vocab - 1) for _ in range(rnd.randint(3, 90))] for _ in range(10)]
    kw.setdefault("num_kvcache_blocks", 64)        # not sized from free memory: earlier tests of the session hold some
    llm = LLM(path, max_model_len=256, max_num_seqs=8, kvcache_block_size=16, **kw)
    try:
        sp = params or SamplingParams(temperature=0.0, max_tokens=24, ignore_eos=True)
        outs = llm.generate(prompts, sp, use_tqdm=False)
        return prompts, [o["token_ids"] for o in outs], outs
    finally:
        llm.exit()


@pytest.mark.parametrize("variant", ["plain", "chunked_preempt", "fp8_kv", "eager"])
def test_engine_greedy_against_oracle(moe_dir, variant):
    """Chunked prefill (64-token budget) with preemption (18 blocks for 10 sequences), prefix-cache hits throughout, an fp8
    KV cache, CUDA graphs (all but "eager").  Every greedy token is the oracle's argmax or within its bf16 tie band."""
    from nanovllm.utils.synthetic import PRESETS
    kw = dict(plain=dict(), chunked_preempt=dict(max_num_batched_tokens=64, num_kvcache_blocks=18),
              fp8_kv=dict(kv_cache_dtype="fp8"), eager=dict(enforce_eager=True))[variant]
    prompts, toks, _ = _generate(moe_dir, **kw)
    assert all(len(t) == 24 for t in toks)
    if variant == "fp8_kv":
        return                                               # the oracle has no fp8 cache; covered by running to the end
    oracle = Qwen3MoeRef.from_preset(PRESETS["tiny-moe"], _moe_weights("tiny-moe"), rounding="fused")
    n = d = 0
    worst = 0.0
    for p, t in zip(prompts, toks):
        a, b, w = check_greedy_against_oracle(oracle, p, t, ulps=12.0)
        n, d, worst = n + a, d + b, max(worst, w)
    record(f"moe_engine_{variant}", dict(tokens=n, differ_from_oracle_argmax=d, worst_margin_over_tol=worst))


def test_graphs_equal_eager(moe_dir):
    _, graph, _ = _generate(moe_dir)
    _, eager, _ = _generate(moe_dir, enforce_eager=True)
    assert graph == eager


def test_engine_sampling_features(moe_dir):
    """One request each with top-k / top-p filters, penalties and logprobs, under CUDA graphs."""
    from nanovllm import SamplingParams
    for sp in (SamplingParams(temperature=0.8, top_k=20, top_p=0.9, max_tokens=16, ignore_eos=True),
               SamplingParams(temperature=0.0, repetition_penalty=1.3, presence_penalty=0.5, max_tokens=16, ignore_eos=True),
               SamplingParams(temperature=0.0, logprobs=3, max_tokens=16, ignore_eos=True)):
        _, toks, outs = _generate(moe_dir, sp)
        assert all(len(t) == 16 for t in toks)
        if sp.logprobs:
            lp = outs[0]["logprobs"]
            assert len(lp) == 16 and all(len(e) >= 1 for e in lp)


def test_tp2_on_one_gpu_over_gloo():
    env = dict(os.environ, TP_EAGER="1", B200_TP_BACKEND="gloo", B200_TP_ONE_DEVICE="1", B200_TP_ALLREDUCE="nccl")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29563", os.path.join(ROOT, "tests", "tp_moe_worker.py")]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "TP_MOE_RESULT" in r.stdout and '"ok": true' in r.stdout
