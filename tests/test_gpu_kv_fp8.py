"""The fp8 (e4m3) KV cache on the GPU: stores bit-exact to the contract, decode and paged prefill against float64
over the dequantized cache, the refusals, and the whole model against the oracle's fp8 mode.

Caches follow tests/test_gpu_dispatch_edges.py: block tables are views into a wider buffer whose spare columns name
poisoned pages, and every cache row no sequence owns holds the e4m3 NaN byte 0x7F, so a read past a sequence's end shows
up as a wrong value.  Each case asserts which kernel the profiler saw.
"""
import os
import random
import subprocess
import sys
from types import SimpleNamespace

import pytest
import torch

from gpu_helpers import record
from kv_fp8_ref import dequantize_e4m3, quantize_e4m3
from test_gpu_dispatch_edges import (D, EPS, SCALE, assert_close_bf16, assert_ran, assert_rows_close, assert_vectors_close,
                                     build_paged, cu, decode64, edge_rows, launched, mixed_lens, norm_weight, prefill64,
                                     randn)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

F8 = torch.float8_e4m3fn
NAN8 = 0x7F


@pytest.fixture(scope="module")
def ops():
    from nanovllm import ops as _ops
    return _ops


def to_fp8(kv, ks, vs):
    """bf16 physical [2, L, nblk, Hkv, bs, D] -> e4m3 with the contract's quantizer (NaN rows stay NaN: 0x7F)."""
    return torch.stack([quantize_e4m3(kv[0], ks), quantize_e4m3(kv[1], vs)]).contiguous()


def logical(kv8, layer, which, scale):
    """Dequantized float32 logical [nblk, bs, Hkv, D] view of one layer of an e4m3 physical cache."""
    return dequantize_e4m3(kv8[which, layer], scale).permute(0, 2, 1, 3)


def poisoned_fp8(shape):
    return torch.full(shape, NAN8, dtype=torch.uint8, device="cuda").view(F8)


def expect_code(fn, code):
    from nanovllm import _native as nat
    with pytest.raises(nat.B200Error, match=f"code {code}"):
        fn()


# ---------------------------------------------------------------------------------------------------------------------
# stores: bit-exact e4m3 of what the bf16 path stores, slot -1 skipped, every other row untouched
# ---------------------------------------------------------------------------------------------------------------------
def test_store_kv_fp8(ops):
    hkv, bs, nblk, n, layer = 8, 16, 64, 700, 1
    ks, vs = 0.375, 0.05
    k = randn(n, hkv, D, seed=1, scale=2.0)
    v = randn(n, hkv, D, seed=2, scale=2.0)
    k[::5] = (k[::5].float() * 200).to(torch.bfloat16)          # past +-448 * scale: saturates
    v[::7] = (v[::7].float() * 500).to(torch.bfloat16)
    rnd = random.Random(3)
    slots = torch.tensor(rnd.sample(range(nblk * bs), n), dtype=torch.int32)
    slots[::11] = -1
    slots = slots.cuda()
    kv16 = randn(2, 2, nblk, hkv, bs, D, seed=4)
    ops.bind_kv_cache(kv16)
    ops.store_kv(layer, k, v, slots)
    kv8 = poisoned_fp8(kv16.shape)
    ops.bind_kv_cache(kv8, k_scale=ks, v_scale=vs)
    _, names = launched(lambda: ops.store_kv(layer, k, v, slots))
    assert_ran(names, "store_kv_fp8_kernel", "store_kv fp8")
    want = to_fp8(kv16, ks, vs).view(torch.uint8)
    got = kv8.view(torch.uint8)
    written = torch.zeros(nblk * bs, dtype=torch.bool, device="cuda")
    written[slots[slots >= 0].long()] = True
    written = written.view(nblk, 1, bs, 1).expand(nblk, hkv, bs, D)
    for c in range(2):
        assert torch.equal(got[c, layer][written], want[c, layer][written]), f"{'kv'[c]} rows differ from the contract"
        assert bool((got[c, layer][~written] == NAN8).all()), "a row no slot names was written"
        assert bool((got[c, 0] == NAN8).all()), "the other layer was written"
    assert bool((got[0, layer][written] == 0x7E).any()), "no saturated element: the case does not reach 448"


@pytest.mark.parametrize("n", [2047, 2048])
def test_qknorm_rope_store_fp8(ops, n):
    from oracle.qwen3_ref import rope_table
    hq, hkv, bs, layer = 32, 8, 256, 1
    ks, vs = 0.01, 0.75                                          # k_scale small enough that normed keys saturate
    nblk = (n + bs - 1) // bs + 2
    qkv = randn(n, (hq + 2 * hkv) * D, seed=n + 1)
    qkv[::3, (hq + hkv) * D:] = (qkv[::3, (hq + hkv) * D:].float() * 1000).to(torch.bfloat16)
    qw, kw = norm_weight(D, seed=1), norm_weight(D, seed=2)
    table = rope_table(D, 40960, 1e6).cuda()
    rnd = random.Random(n)
    pos = [rnd.randrange(40960) for _ in range(n)]
    pos[0], pos[n - 1] = 40959, 0
    pos = torch.tensor(pos, dtype=torch.int64, device="cuda")
    slots = torch.tensor(rnd.sample(range(nblk * bs), n), dtype=torch.int32)
    slots[::37] = -1
    slots[n - 1] = -1
    slots = slots.cuda()
    kv16 = randn(2, 2, nblk, hkv, bs, D, seed=n)
    ops.bind_kv_cache(kv16)
    g16 = qkv.clone()
    ops.qknorm_rope_store(layer, g16, hq, hkv, pos, qw, kw, table, EPS, slots)
    kv8 = poisoned_fp8(kv16.shape)
    ops.bind_kv_cache(kv8, k_scale=ks, v_scale=vs)
    g8 = qkv.clone()
    _, names = launched(lambda: ops.qknorm_rope_store(layer, g8, hq, hkv, pos, qw, kw, table, EPS, slots))
    assert_ran(names, "qknorm_rope_store_tok_fp8_kernel<8>" if n >= 2048 else "qknorm_rope_store_fp8_kernel(",
               f"qknorm_rope_store fp8 n={n}")
    assert torch.equal(g8, g16), "q / k rewritten in place exactly as with a bf16 cache"
    want = to_fp8(kv16, ks, vs).view(torch.uint8)
    got = kv8.view(torch.uint8)
    written = torch.zeros(nblk * bs, dtype=torch.bool, device="cuda")
    written[slots[slots >= 0].long()] = True
    written = written.view(nblk, 1, bs, 1).expand(nblk, hkv, bs, D)
    for c in range(2):
        assert torch.equal(got[c, layer][written], want[c, layer][written])
        assert bool((got[c, layer][~written] == NAN8).all())
        assert bool((got[c, 0] == NAN8).all())
        assert bool((got[c, layer][written] & 0x7F == 0x7E).any()), "no saturated element"


# ---------------------------------------------------------------------------------------------------------------------
# decode: the tensor-core kernel's fp8 variant for every head group
# ---------------------------------------------------------------------------------------------------------------------
def fp8_paged(c, ks, vs):
    """e4m3 version of a build_paged cache (+ the dequantized logical K / V of its last layer for the reference)."""
    kv8 = to_fp8(c.kv, ks, vs)
    L = kv8.shape[1] - 1
    return kv8, logical(kv8, L, 0, ks), logical(kv8, L, 1, vs)


def permuted_pages(kv8, tables, seed):
    """The same cache with its pages moved to other page ids (and the tables rewritten to match)."""
    nblk = kv8.shape[2]
    perm = torch.randperm(nblk, generator=torch.Generator().manual_seed(seed)).cuda()
    out = torch.empty_like(kv8)
    out[:, :, perm] = kv8
    buf = tables.as_strided((tables.shape[0], tables.stride(0)), (tables.stride(0), 1))
    buf2 = perm[buf.long()].to(torch.int32)
    return out, buf2[:, :tables.shape[1]]


DEC_KS, DEC_VS = 0.5, 0.1875


@pytest.mark.parametrize("bs", [16, 256])
@pytest.mark.parametrize("G", [1, 2, 4, 8], ids=lambda G: f"G{G}")
def test_decode_fp8(ops, G, bs):
    from nanovllm import _native as nat
    hkv, batch = 2, 1024
    lens = mixed_lens(batch, seed=G + bs)
    c = build_paged(lens, bs, hkv, seed=G + bs)
    kv8, K, V = fp8_paged(c, DEC_KS, DEC_VS)
    ops.bind_kv_cache(kv8, k_scale=DEC_KS, v_scale=DEC_VS)
    q = randn(batch, G * hkv, D, seed=200 + G)
    ctx = torch.tensor(lens, dtype=torch.int32, device="cuda")
    got, names = launched(lambda: ops.paged_decode(0, q, c.tables, ctx, SCALE))
    assert_ran(names, f"paged_decode_mma_fp8_kernel<{G}>", f"decode fp8 G={G}")
    want = decode64(q, K, V, lens, c.tables)
    assert_vectors_close(got, want, f"decode fp8 G={G} bs={bs} batch {batch}")
    assert_rows_close(got, want, [i for i in edge_rows(batch, extra=range(16)) if lens[i]], f"decode fp8 G={G}")
    assert (got[ctx == 0] == 0).all(), "zero-context rows are exactly zero"
    for b in (1, 3, 256):                                   # smaller batches through the same workspace
        assert_vectors_close(ops.paged_decode(0, q[:b], c.tables[:b], ctx[:b], SCALE), want[:b], f"decode fp8 G={G} batch {b}")
    again = ops.paged_decode(0, q, c.tables, ctx, SCALE)
    nat.handle().workspace = None
    fresh = ops.paged_decode(0, q, c.tables, ctx, SCALE)
    assert torch.equal(again, got) and torch.equal(fresh, got), "relaunch must be bit-identical"
    kv8p, tables_p = permuted_pages(kv8, c.tables, seed=G)
    ops.bind_kv_cache(kv8p, k_scale=DEC_KS, v_scale=DEC_VS)
    assert torch.equal(ops.paged_decode(0, q, tables_p, ctx, SCALE), got), "page placement changed the result"


@pytest.mark.parametrize("G,nseq", [(1, 4), (8, 1)])
def test_decode_fp8_long_context(ops, G, nseq):
    """40960-token contexts whose keys lean more and more towards the query: the running maximum rises across every
    segment boundary, so each merge of partials has to rescale."""
    hkv, bs = 8, 256
    lens = [40960] * nseq
    if nseq > 1:
        lens[1] = 40959
    g = torch.Generator(device="cuda").manual_seed(nseq * 10 + G)
    u = torch.randn(hkv, D, generator=g, device="cuda", dtype=torch.float64)
    c = build_paged(lens, bs, hkv, seed=nseq * 10 + G,
                    key_shift=lambda pos: (3.0 * pos.double() / 40960)[:, None, None] * u[None])
    kv8, K, V = fp8_paged(c, DEC_KS, DEC_VS)
    ops.bind_kv_cache(kv8, k_scale=DEC_KS, v_scale=DEC_VS)
    q = (0.5 * u.repeat_interleave(G, 0)[None] + torch.randn(nseq, G * hkv, D, generator=g, device="cuda", dtype=torch.float64))
    q = q.to(torch.bfloat16)
    ctx = torch.tensor(lens, dtype=torch.int32, device="cuda")
    got, names = launched(lambda: ops.paged_decode(0, q, c.tables, ctx, SCALE))
    assert_ran(names, f"paged_decode_mma_fp8_kernel<{G}>", f"decode fp8 G={G} context 40960")
    want = decode64(q, K, V, lens, c.tables)
    assert_vectors_close(got, want, f"decode fp8 G={G} {nseq} x 40960")
    for i in range(nseq):
        assert_close_bf16(got[i], want[i], f"decode fp8 G={G} sequence {i}")


def test_bind_bf16_fp8_bf16_one_process(ops):
    """The tensor-core decode caches its bf16 tensor maps per binding: an fp8 binding in between must neither use them
    nor leave a stale map for the bf16 binding that follows."""
    G, hkv, bs = 4, 2, 64
    lens = [1, 100, 777, 2048]
    q = randn(len(lens), G * hkv, D, seed=5)
    ctx = torch.tensor(lens, dtype=torch.int32, device="cuda")
    a = build_paged(lens, bs, hkv, seed=11)
    ops.bind_kv_cache(a.kv)
    assert_vectors_close(ops.paged_decode(0, q, a.tables, ctx, SCALE), decode64(q, a.K, a.V, lens, a.tables), "bf16 bind 1")
    b = build_paged(lens, bs, hkv, seed=12)
    kv8, K, V = fp8_paged(b, 1.0, 1.0)
    ops.bind_kv_cache(kv8)
    got, names = launched(lambda: ops.paged_decode(0, q, b.tables, ctx, SCALE))
    assert_ran(names, f"paged_decode_mma_fp8_kernel<{G}>", "fp8 bind")
    assert_vectors_close(got, decode64(q, K, V, lens, b.tables), "fp8 bind")
    c = build_paged(lens, bs, hkv, seed=13)
    ops.bind_kv_cache(c.kv)
    got, names = launched(lambda: ops.paged_decode(0, q, c.tables, ctx, SCALE))
    assert_ran(names, f"paged_decode_mma_kernel<{G}>", "bf16 bind 2")
    assert_vectors_close(got, decode64(q, c.K, c.V, lens, c.tables), "bf16 bind 2")


def test_fp8_refusals(ops):
    hkv, bs = 2, 16
    c = build_paged([40, 5], bs, hkv, seed=21)
    kv8, _, _ = fp8_paged(c, 1.0, 1.0)
    ops.bind_kv_cache(kv8)
    q = randn(2, 2 * hkv, D, seed=22)
    ctx = torch.tensor([40, 5], dtype=torch.int32, device="cuda")
    qkv = randn(2, (2 * hkv + 2 * hkv) * D, seed=23)
    from oracle.qwen3_ref import rope_table
    table = rope_table(D, 64, 1e6).cuda()
    w = norm_weight(D, seed=1)
    expect_code(lambda: ops.paged_decode_fused(0, qkv, 2 * hkv, w, w, table, EPS, c.tables, ctx, SCALE), -2)
    qp = randn(8, 2 * hkv, D, seed=24)
    cq, ck = cu([4, 4]), cu([40, 5])
    expect_code(lambda: ops.paged_prefill(0, qp, None, None, cq, ck, 4, 40, SCALE, block_tables=c.tables, num_kv_heads=hkv), -2)
    ops.bind_kv_cache(c.kv)                                   # bf16 binding: nothing to gather
    kout = torch.empty(45, hkv, D, dtype=torch.bfloat16, device="cuda")
    expect_code(lambda: ops.kv_gather(0, c.tables, ck, kout, kout.clone(), 45), -2)
    with pytest.raises(Exception):
        ops.bind_kv_cache(c.kv, k_scale=0.5)                  # scales belong to an fp8 cache
    with pytest.raises(Exception):
        ops.bind_kv_cache(kv8, k_scale=float("nan"))


# ---------------------------------------------------------------------------------------------------------------------
# paged prefill over an fp8 cache: gather (dequantize to bf16) per group of sequences + the packed prefill kernel
# ---------------------------------------------------------------------------------------------------------------------
def device_groups(cu_q, cu_k, rows):
    from nanovllm.layers.attention import KVGroup, kv_group_arrays, plan_kv_groups
    cq, ck = cu_q.cpu().numpy(), cu_k.cpu().numpy()
    out = []
    for g in kv_group_arrays(cq, ck, plan_kv_groups(ck, rows)):
        out.append(KVGroup(*g[:6], torch.from_numpy(g[6]).cuda(), torch.from_numpy(g[7]).cuda()))
    return out


PREFILL_CASES = {
    "chunk512of4096-bs16": ([512], [4096], 16, 1 << 20),
    "chunk512of4096-bs256": ([512], [4096], 256, 1 << 20),
    "prefix-hit": ([50, 1000, 17, 100], [300, 1000, 17, 700], 16, 1 << 20),
    "three-groups": ([50, 1000, 17, 100], [300, 1000, 17, 700], 64, 1100),
}


@pytest.mark.parametrize("case", list(PREFILL_CASES))
def test_paged_prefill_fp8(ops, case):
    from nanovllm.layers.attention import Attention
    from nanovllm.utils.context import reset_context, set_context
    lq, lk, bs, rows = PREFILL_CASES[case]
    hq, hkv, ks, vs = 8, 2, 0.75, 1.5
    c = build_paged(lk, bs, hkv, seed=len(case))
    kv8 = to_fp8(c.kv, ks, vs)
    ops.bind_kv_cache(kv8, k_scale=ks, v_scale=vs)
    attn = Attention(hq, D, SCALE, hkv)
    attn.k_cache, attn.v_cache, attn.layer_id = kv8[0, 0], kv8[1, 0], 0
    attn.kv_scratch = torch.full((2, min(rows, sum(lk)), hkv, D), float("nan"), dtype=torch.bfloat16, device="cuda")
    q = randn(sum(lq), hq, D, seed=7)
    cq, ck = cu(lq), cu(lk)
    groups = device_groups(cq, ck, attn.kv_scratch.shape[1])
    assert len(groups) == (3 if case == "three-groups" else 1)
    set_context(True, cq, ck, max(lq), max(lk), None, None, c.tables, groups)
    try:
        got, names = launched(lambda: attn(q, None, None, kv_stored=True))
    finally:
        reset_context()
    assert_ran(names, "kv_gather_fp8_kernel", f"prefill fp8 {case}")
    cache = SimpleNamespace(K=logical(kv8, 0, 0, ks).to(torch.bfloat16), V=logical(kv8, 0, 1, vs).to(torch.bfloat16),
                            tables=c.tables)
    want = prefill64(q, cq, ck, cache=cache)
    assert_vectors_close(got, want, f"prefill fp8 {case}")
    ends = (torch.tensor(lq).cumsum(0) - 1).tolist()
    assert_rows_close(got, want, edge_rows(sum(lq), extra=ends), f"prefill fp8 {case}")


# ---------------------------------------------------------------------------------------------------------------------
# the whole model: the seven-step script against the oracle's fp8 mode, and the engine
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("preset", ["tiny", "tiny-g1", "tiny-g4", "tiny-g8"])
def test_model_script_fp8_vs_oracle(preset):
    from gpu_helpers import make_oracle
    from kv_fp8_ref import Qwen3RefFp8, alloc_logical_kv_fp8, oracle_fp8_step_fn
    from nanovllm import ops
    from nanovllm.models.qwen3 import Qwen3ForCausalLM
    from nanovllm.utils.context import reset_context, set_context
    from nanovllm.utils.synthetic import PRESETS, hf_config_dict, random_weights
    from oracle.model_script import make_script, run_script
    from oracle.qwen3_ref import alloc_logical_kv
    from test_oracle_golden import oracle_step_fn
    weights = random_weights(PRESETS[preset], seed=1234)
    script = make_script(PRESETS[preset]["vocab_size"])
    hf = SimpleNamespace(**hf_config_dict(PRESETS[preset]))
    model = Qwen3ForCausalLM(hf, 0, 1, "cuda", max_position=4096)
    for name, w in weights.items():
        model.load_hf_tensor(name, w)
    model.fused_decode_max_batch = 0
    kv8 = torch.zeros(ops.kv_cache_shape(hf.num_hidden_layers, script["num_blocks"], model.num_kv_heads,
                                         script["block_size"], model.head_dim), dtype=torch.uint8, device="cuda").view(F8)
    ops.bind_kv_cache(kv8)
    scratch = torch.empty(2, 256, model.num_kv_heads, model.head_dim, dtype=torch.bfloat16, device="cuda")
    for i, a in enumerate(model.modules()):
        a.k_cache, a.v_cache, a.layer_id, a.kv_scratch = kv8[0, i], kv8[1, i], i, scratch

    def gpu_step(ids, pos, c):
        groups = None
        if c["is_prefill"] and c.get("block_tables") is not None:
            groups = device_groups(c["cu_seqlens_q"], c["cu_seqlens_k"], scratch.shape[1])
        set_context(c["is_prefill"], c.get("cu_seqlens_q"), c.get("cu_seqlens_k"), c.get("max_seqlen_q", 0),
                    c.get("max_seqlen_k", 0), c.get("slot_mapping"), c.get("context_lens"), c.get("block_tables"), groups)
        out = model.compute_logits(model(ids, pos)).float().cpu()
        reset_context()
        return out

    got = run_script(torch, script, gpu_step, device="cuda")
    base = make_oracle(PRESETS[preset], weights, "fused")
    oracle = Qwen3RefFp8(base.d, weights, rounding="fused", max_pos=4096)
    want = [o.float() for o in run_script(torch, script, oracle_fp8_step_fn(oracle, alloc_logical_kv_fp8(oracle.d, script["num_blocks"], script["block_size"])))]
    bf16 = [o.float() for o in run_script(torch, script, oracle_step_fn(base, alloc_logical_kv(base.d, script["num_blocks"], script["block_size"])))]
    worst_rel, worst_vs_bf16, flips, rows = 0.0, 0.0, 0, 0
    for i, (g, w, b) in enumerate(zip(got, want, bf16)):
        assert g.shape == w.shape and torch.isfinite(g).all()
        rel = ((g - w).norm() / w.norm()).item()
        worst_rel = max(worst_rel, rel)
        worst_vs_bf16 = max(worst_vs_bf16, ((w - b).norm() / b.norm()).item())
        assert rel < 2e-2, f"step {i}: logits relative L2 {rel} against the fp8 oracle"
        tol = 6 * 2 ** -8 * w.abs().max().item()
        for r in range(g.shape[0]):
            tok = int(g[r].argmax())
            margin = (w[r].max() - w[r, tok]).item()
            assert margin <= tol, f"step {i} row {r}: greedy token {tok} loses by {margin} in the fp8 oracle (tol {tol})"
            flips += tok != int(w[r].argmax())
            rows += 1
    record("model_script_fp8", dict(preset=preset, worst_rel_l2=worst_rel, fp8_oracle_vs_bf16_oracle_rel_l2=worst_vs_bf16,
                                    greedy_rows=rows, greedy_differ=flips))


@pytest.fixture(scope="module")
def tiny_dir(tmp_path_factory):
    from nanovllm.utils.synthetic import make_model_dir
    return make_model_dir(str(tmp_path_factory.mktemp("models") / "tiny"), "tiny", seed=1234)


@pytest.mark.parametrize("eager", [True, False])
def test_engine_generate_fp8(tiny_dir, eager):
    """generate() with kv_cache_dtype="fp8_e4m3": the same run as the bf16 engine test (prompts with a shared prefix, so
    the prefix cache is hit), half the bytes per cache block, greedy tokens teacher-forced against the bf16 oracle with the
    bf16 engine's bar (within 6 bf16 roundings of the logit scale)."""
    from gpu_helpers import check_greedy_against_oracle, make_oracle
    from nanovllm import LLM, SamplingParams
    from nanovllm.utils.synthetic import PRESETS, random_weights
    from test_gpu_model import _prompts
    kw = dict(enforce_eager=eager, max_model_len=256, max_num_seqs=8, max_num_batched_tokens=128, kvcache_block_size=16,
              num_kvcache_blocks=64)
    llm = LLM(tiny_dir, kv_cache_dtype="fp8_e4m3", **kw)
    try:
        runner = llm.model_runner
        assert runner.kv_cache.dtype == F8
        block8 = runner.kv_block_bytes()
        prompts = _prompts(PRESETS["tiny"]["vocab_size"])
        sps = [SamplingParams(temperature=0.0, max_tokens=8 + (i % 5) * 6, ignore_eos=True) for i in range(len(prompts))]
        outs = llm.generate(prompts, sps, use_tqdm=False)
    finally:
        llm.exit()
    hf = runner.config.hf_config
    assert block8 * 2 == 2 * hf.num_hidden_layers * 16 * runner.model.num_kv_heads * runner.model.head_dim * 2
    oracle = make_oracle(PRESETS["tiny"], random_weights(PRESETS["tiny"], seed=1234), "fused")
    tot = diff = 0
    worst = 0.0
    for p, sp, o in zip(prompts, sps, outs):
        assert len(o["token_ids"]) == sp.max_tokens
        n, d, w = check_greedy_against_oracle(oracle, p, o["token_ids"])
        tot, diff, worst = tot + n, diff + d, max(worst, w)
    record("engine_greedy_fp8", dict(eager=eager, tokens=tot, differ_from_bf16_oracle_argmax=diff, worst_margin_over_tol=worst))


@pytest.mark.skipif(os.environ.get("B200_KV_FP8_CHILD") == "1", reason="already the child run")
def test_paged_prefill_fp8_under_ws_kernel():
    """The same paged prefills with B200_PREFILL=ws (read once per process, hence a child pytest)."""
    cmd = [sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu", "-k", "test_paged_prefill_fp8 and not ws",
           os.path.abspath(__file__)]
    env = dict(os.environ, B200_PREFILL="ws", B200_KV_FP8_CHILD="1")
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and " passed" in r.stdout and " failed" not in r.stdout, r.stdout[-4000:] + r.stderr[-2000:]
