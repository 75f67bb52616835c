"""Parity of every CUDA entry point (called through the C ABI) with the CPU oracle on seeded inputs.

Integer / byte work (KV scatter, embedding gather, greedy argmax) is bit-exact.  Floating point is
compared in bf16: the kernels accumulate in a different order than the oracle, so the bar is
"within one bf16 rounding of the output scale" element-wise and 4e-3 in relative L2.  Attention outputs are held to
two bf16 ulps of each (row, head) vector's own scale (assert_vectors_close).
"""
import math
import random

import pytest
import torch

from oracle.paged_attention_ref import (paged_decode_ref, store_kvcache_ref, to_logical, to_physical,
                                        varlen_prefill_ref)
from oracle.qwen3_ref import add_rmsnorm_ref, rmsnorm_ref, rope_ref, rope_table, silu_mul_ref
from test_gpu_dispatch_edges import assert_vectors_close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from nanovllm import ops as _ops
    return _ops


def bf(*shape, scale=1.0, seed=None):
    g = torch.Generator().manual_seed(seed if seed is not None else random.randrange(1 << 30))
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16)


def assert_close_bf16(got, want, what="", rel_l2=4e-3, ulps=2.0):
    got, want = got.float().cpu(), want.float().cpu()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    scale = max(want.abs().max().item(), 1e-3)
    err = (got - want).abs().max().item()
    assert err <= ulps * scale * 2 ** -8, f"{what}: max abs err {err} vs scale {scale}"
    l2 = ((got - want).norm() / max(want.norm().item(), 1e-6)).item()
    assert l2 <= rel_l2, f"{what}: relative L2 {l2}"


def bind_random_cache(ops, layers, nblk, hkv, bs, seed=0, poison=False):
    """Returns (kv_cache physical on GPU, logical CPU k list, logical CPU v list)."""
    ks = [bf(nblk, bs, hkv, 128, seed=seed + 2 * l) for l in range(layers)]
    vs = [bf(nblk, bs, hkv, 128, seed=seed + 2 * l + 1) for l in range(layers)]
    kv = torch.stack([torch.stack([to_physical(k) for k in ks]), torch.stack([to_physical(v) for v in vs])]).cuda()
    ops.bind_kv_cache(kv)
    return kv, ks, vs


def make_tables(ctx_lens, bs, nblk, seed=0):
    rnd = random.Random(seed)
    pages = list(range(nblk))
    rnd.shuffle(pages)
    w = max(1, max((c + bs - 1) // bs for c in ctx_lens))
    tables = torch.full((len(ctx_lens), w), -1, dtype=torch.int32)
    used = 0
    for i, c in enumerate(ctx_lens):
        n = (c + bs - 1) // bs
        tables[i, :n] = torch.tensor(pages[used:used + n], dtype=torch.int32)
        used += n
    assert used <= nblk
    return tables


# ---------------------------------------------------------------------------------------------
# K1 store_kvcache                                                  (bit-exact)
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bs,hkv", [(16, 2), (256, 8), (64, 1)])
def test_store_kv_bit_exact(ops, bs, hkv):
    nblk, n = 6, 37
    kv, ks, vs = bind_random_cache(ops, 2, nblk, hkv, bs, seed=3)
    row = torch.randn(n, (4 + 2 * hkv) * 128).to(torch.bfloat16)          # k, v are strided views of a wider row
    k = row[:, 4 * 128:(4 + hkv) * 128].view(n, hkv, 128)
    v = row[:, (4 + hkv) * 128:].view(n, hkv, 128)
    slots = torch.tensor(random.Random(1).sample(range(nblk * bs), n), dtype=torch.int32)
    slots[5] = -1
    slots[20] = -1
    rg = row.cuda()
    ops.store_kv(1, rg[:, 4 * 128:(4 + hkv) * 128].view(n, hkv, 128), rg[:, (4 + hkv) * 128:].view(n, hkv, 128), slots.cuda())
    store_kvcache_ref(k, v, ks[1], vs[1], slots)
    assert torch.equal(to_logical(kv[0, 1].cpu()), ks[1]) and torch.equal(to_logical(kv[1, 1].cpu()), vs[1])
    assert torch.equal(to_logical(kv[0, 0].cpu()), ks[0])                  # other layer untouched


# ---------------------------------------------------------------------------------------------
# K4 paged decode
# ---------------------------------------------------------------------------------------------
DECODE_CASES = [
    # (hq, hkv, block_size, context lens)
    (16, 8, 256, [1, 15, 16, 17, 255, 256, 257, 1000, 2048, 0, 3]),
    (4, 2, 16, [1, 16, 17, 33, 100, 0, 64]),
    (8, 2, 64, [700, 64, 65, 1]),                       # G = 4
    (8, 1, 32, [900, 31, 32, 33]),                      # G = 8
    (2, 2, 128, [129, 128, 5]),                         # G = 1
    (16, 8, 256, [4000]),                               # one long sequence: many segments per kv head
    (16, 8, 16, [random.Random(5).randint(1, 300) for _ in range(150)]),
]


@pytest.mark.parametrize("hq,hkv,bs,lens", DECODE_CASES)
def test_paged_decode_vs_oracle(ops, hq, hkv, bs, lens):
    nblk = sum((c + bs - 1) // bs for c in lens) + 3
    kv, ks, vs = bind_random_cache(ops, 2, nblk, hkv, bs, seed=11)
    tables = make_tables(lens, bs, nblk, seed=2)
    ctx = torch.tensor(lens, dtype=torch.int32)
    q = bf(len(lens), hq, 128, seed=9)
    scale = 128 ** -0.5
    want = paged_decode_ref(q, ks[1], vs[1], ctx, tables, scale)
    got = ops.paged_decode(1, q.cuda(), tables.cuda(), ctx.cuda(), scale)
    assert_vectors_close(got, want, f"decode hq={hq} hkv={hkv} bs={bs}")
    # zero-context rows are exactly zero (graph padding)
    for i, c in enumerate(lens):
        if c == 0:
            assert got[i].float().abs().max().item() == 0.0
    # second launch on the same workspace (counters must have been left clean) is bit-identical
    again = ops.paged_decode(1, q.cuda(), tables.cuda(), ctx.cuda(), scale)
    assert torch.equal(got, again)


def _poison_invalid_rows(ks, vs, tables, lens, bs, nblk):
    """NaN in every cache row that no sequence owns (stale rows after the last token, unused pages)."""
    valid = torch.zeros(nblk, bs, dtype=torch.bool)
    for i, c in enumerate(lens):
        for p in range(c):
            valid[int(tables[i, p // bs]), p % bs] = True
    nan = torch.tensor(float("nan"), dtype=torch.bfloat16)
    for t in (ks, vs):
        t[~valid] = nan
    return valid


@pytest.mark.parametrize("hq,hkv,bs,lens", [(8, 2, 64, [70, 5, 130, 17, 64]), (8, 1, 16, [33, 1, 47]), (32, 8, 256, [300, 1, 255, 513]),
                                            (2, 2, 32, [31, 65])])
def test_paged_decode_wide_groups_ignore_stale_rows(ops, hq, hkv, bs, lens):
    """The tensor-core decode kernel (G >= 4, decode_mma.cu) always fetches whole 16-row TMA boxes: rows past the
    context hold stale bytes.  Poison them with NaN -- P = 0 there, but 0 * NaN would poison the accumulator -- and
    require the clean result.  (G = 1 rides along for the FMA kernel.)"""
    nblk = sum((c + bs - 1) // bs for c in lens) + 2
    kv, ks, vs = bind_random_cache(ops, 1, nblk, hkv, bs, seed=23)
    tables = make_tables(lens, bs, nblk, seed=5)
    ctx = torch.tensor(lens, dtype=torch.int32)
    q = bf(len(lens), hq, 128, seed=3)
    want = paged_decode_ref(q, ks[0], vs[0], ctx, tables, 0.1)
    _poison_invalid_rows(ks[0], vs[0], tables, lens, bs, nblk)
    kvp = torch.stack([to_physical(ks[0]).unsqueeze(0), to_physical(vs[0]).unsqueeze(0)]).cuda()
    ops.bind_kv_cache(kvp)
    got = ops.paged_decode(0, q.cuda(), tables.cuda(), ctx.cuda(), 0.1)
    assert_vectors_close(got, want, f"decode G={hq // hkv} with NaN-poisoned stale rows")


@pytest.mark.parametrize("bs", [16, 64, 256])
def test_prefill_paged_ignores_stale_rows(ops, bs):
    """Paged prefill (prefill_tc.cu) stages whole 64-key tiles; keys >= len_k of the last tile are stale page rows (or
    page 0 when the tile runs past the block table).  NaN there must not reach the tensor-core accumulator."""
    hq, hkv = 8, 2
    len_k = [300, 77, 130, 40, 65]
    len_q = [44, 77, 1, 13, 65]
    nblk = sum((c + bs - 1) // bs for c in len_k) + 2
    kv, ks, vs = bind_random_cache(ops, 1, nblk, hkv, bs, seed=43)
    tables = make_tables(len_k, bs, nblk, seed=8)
    q = bf(sum(len_q), hq, 128, seed=7)
    cu_q = torch.tensor([0] + list(torch.tensor(len_q).cumsum(0)), dtype=torch.int32)
    cu_k = torch.tensor([0] + list(torch.tensor(len_k).cumsum(0)), dtype=torch.int32)
    scale = 128 ** -0.5
    want = varlen_prefill_ref(q, None, None, cu_q, cu_k, scale, tables, ks[0], vs[0], p_dtype=torch.bfloat16)
    _poison_invalid_rows(ks[0], vs[0], tables, len_k, bs, nblk)
    kvp = torch.stack([to_physical(ks[0]).unsqueeze(0), to_physical(vs[0]).unsqueeze(0)]).cuda()
    ops.bind_kv_cache(kvp)
    got = ops.paged_prefill(0, q.cuda(), None, None, cu_q.cuda(), cu_k.cuda(), max(len_q), max(len_k), scale,
                            block_tables=tables.cuda(), num_kv_heads=hkv)
    assert_vectors_close(got, want, f"paged prefill bs={bs} with NaN-poisoned stale rows")


def test_prefill_packed_ignores_neighbouring_rows(ops):
    """Packed prefill: the last 64-key tile of a sequence overlaps the NEXT sequence's rows (or runs past the end of
    the batch).  Inf/NaN there must not leak into this sequence."""
    hq, hkv = 4, 2
    lens = [70, 3, 129]
    tot = sum(lens)
    q, k, v = bf(tot, hq, 128, seed=11), bf(tot, hkv, 128, seed=12), bf(tot, hkv, 128, seed=13)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32)
    scale = 128 ** -0.5
    # sequence 1 (rows 70..72) is all NaN/Inf: sequences 0 and 2 must be unaffected
    k2, v2 = k.clone(), v.clone()
    k2[70:73] = float("nan")
    v2[70:73] = float("inf")
    want = varlen_prefill_ref(q, k, v, cu, cu, scale, p_dtype=torch.bfloat16)
    got = ops.paged_prefill(0, q.cuda(), k2.cuda(), v2.cuda(), cu.cuda(), cu.cuda(), max(lens), max(lens), scale).cpu()
    keep = torch.ones(tot, dtype=torch.bool)
    keep[70:73] = False
    assert_vectors_close(got[keep], want[keep], "packed prefill next to a NaN/Inf sequence")


def test_paged_decode_ignores_rows_beyond_context(ops):
    """Stale rows after the last valid token (and unused pages) may hold anything, even NaN."""
    hq, hkv, bs, lens = 4, 2, 64, [70, 5, 130]
    nblk = 8
    kv, ks, vs = bind_random_cache(ops, 1, nblk, hkv, bs, seed=21)
    tables = make_tables(lens, bs, nblk, seed=4)
    ctx = torch.tensor(lens, dtype=torch.int32)
    q = bf(3, hq, 128, seed=1)
    want = paged_decode_ref(q, ks[0], vs[0], ctx, tables, 0.1)
    valid = torch.zeros(nblk, bs, dtype=torch.bool)
    for i, c in enumerate(lens):
        for p in range(c):
            valid[int(tables[i, p // bs]), p % bs] = True
    nan = torch.tensor(float("nan"), dtype=torch.bfloat16)
    for t in (ks[0], vs[0]):
        t[~valid] = nan
    kvp = torch.stack([to_physical(ks[0]).unsqueeze(0), to_physical(vs[0]).unsqueeze(0)]).cuda()
    ops.bind_kv_cache(kvp)
    got = ops.paged_decode(0, q.cuda(), tables.cuda(), ctx.cuda(), 0.1)
    assert_vectors_close(got, want, "decode with NaN-poisoned stale rows")


def test_paged_decode_page_permutation_invariance(ops):
    """Moving pages around in HBM (and renaming them in the block table) must not change a single bit."""
    hq, hkv, bs = 16, 8, 256
    lens = [random.Random(8).randint(100, 2048) for _ in range(64)]
    nblk = sum((c + bs - 1) // bs for c in lens)
    kv, ks, vs = bind_random_cache(ops, 1, nblk, hkv, bs, seed=31)
    tables = make_tables(lens, bs, nblk, seed=6)
    ctx = torch.tensor(lens, dtype=torch.int32).cuda()
    q = bf(len(lens), hq, 128, seed=2).cuda()
    a = ops.paged_decode(0, q, tables.cuda(), ctx, 0.088)
    perm = torch.randperm(nblk, generator=torch.Generator().manual_seed(3))
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(nblk)
    kv2 = kv[:, :, perm].contiguous()                   # new page j holds old page perm[j]
    t2 = tables.clone()
    m = t2 >= 0
    t2[m] = inv[t2[m].long()].to(torch.int32)
    ops.bind_kv_cache(kv2)
    b = ops.paged_decode(0, q, t2.cuda(), ctx, 0.088)
    assert torch.equal(a, b)


@pytest.mark.parametrize("hq,hkv,bs,lens", [(16, 8, 256, [1, 16, 17, 300, 1024, 0, 33, 2048]), (4, 2, 16, [5, 16, 49, 1]),
                                            (2, 1, 64, [65, 64, 700]), (4, 4, 32, [31, 32, 33])])
def test_paged_decode_fused_vs_two_kernels_and_oracle(ops, hq, hkv, bs, lens):
    """b200_paged_decode_fused == b200_qknorm_rope_store + b200_paged_decode == the oracle, including what ends up in
    the cache for the step's own token (position ctx-1, slot from the block table)."""
    nblk = sum((c + bs - 1) // bs for c in lens) + 2
    tables = make_tables(lens, bs, nblk, seed=12)
    ctx = torch.tensor(lens, dtype=torch.int32)
    n = len(lens)
    qkv = bf(n, (hq + 2 * hkv) * 128, seed=17)
    qw, kw = (1 + 0.1 * torch.randn(128)).to(torch.bfloat16), (1 + 0.1 * torch.randn(128)).to(torch.bfloat16)
    table = rope_table(128, 4096, 1e6)
    pos = (ctx.long() - 1).clamp(min=0)
    slots = torch.tensor([(int(tables[i, (c - 1) // bs]) * bs + (c - 1) % bs) if c > 0 else -1 for i, c in enumerate(lens)],
                         dtype=torch.int32)
    scale = 128 ** -0.5
    # oracle: norm + rope on q/k, scatter, attend
    kv, ks, vs = bind_random_cache(ops, 1, nblk, hkv, bs, seed=71)
    q = qkv[:, :hq * 128].view(n, hq, 128)
    k = qkv[:, hq * 128:(hq + hkv) * 128].view(n, hkv, 128)
    v = qkv[:, (hq + hkv) * 128:].view(n, hkv, 128)
    q_o = rope_ref(table, pos, rmsnorm_ref(q, qw, 1e-6))
    k_o = rope_ref(table, pos, rmsnorm_ref(k, kw, 1e-6))
    ko, vo = ks[0].clone(), vs[0].clone()
    store_kvcache_ref(k_o, v, ko, vo, slots)
    want = paged_decode_ref(q_o, ko, vo, ctx, tables, scale)
    # two kernels
    g2 = qkv.cuda()
    ops.qknorm_rope_store(0, g2, hq, hkv, pos.cuda(), qw.cuda(), kw.cuda(), table.cuda(), 1e-6, slots.cuda())
    two = ops.paged_decode(0, g2[:, :hq * 128].view(n, hq, 128), tables.cuda(), ctx.cuda(), scale)
    cache_two = kv.clone()
    # fused, on a pristine copy of the cache
    kv2, _, _ = bind_random_cache(ops, 1, nblk, hkv, bs, seed=71)
    g1 = qkv.cuda()
    fused = ops.paged_decode_fused(0, g1, hq, qw.cuda(), kw.cuda(), table.cuda(), 1e-6, tables.cuda(), ctx.cuda(), scale)
    assert torch.equal(g1.cpu(), qkv), "the fused kernel must not modify the projection output"
    assert_vectors_close(fused, want, "fused decode vs oracle")
    assert_close_bf16(fused, two, "fused decode vs two-kernel path", ulps=1.01, rel_l2=2e-3)
    assert torch.equal(kv2[1], cache_two[1]), "V rows are plain copies: bit-exact"
    assert_close_bf16(kv2[0], cache_two[0], "appended K rows", ulps=1.01, rel_l2=1e-3)
    assert_close_bf16(to_logical(kv2[0, 0].cpu()), ko, "cache K vs oracle", ulps=1.01, rel_l2=1e-3)
    for i, c in enumerate(lens):
        if c == 0:
            assert fused[i].float().abs().max().item() == 0.0


# ---------------------------------------------------------------------------------------------
# K2/K3 prefill
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hq,hkv,lens", [(4, 2, [1, 63, 64, 65, 128, 300]), (8, 2, [200, 17]), (8, 1, [129]), (2, 2, [70, 5])])
def test_prefill_packed_vs_oracle(ops, hq, hkv, lens):
    tot = sum(lens)
    row = bf(tot, (hq + 2 * hkv) * 128, seed=5)
    q = row[:, :hq * 128].view(tot, hq, 128)
    k = row[:, hq * 128:(hq + hkv) * 128].view(tot, hkv, 128)
    v = row[:, (hq + hkv) * 128:].view(tot, hkv, 128)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32)
    scale = 128 ** -0.5
    want = varlen_prefill_ref(q, k, v, cu, cu, scale, p_dtype=torch.bfloat16)
    rg = row.cuda()
    got = ops.paged_prefill(0, rg[:, :hq * 128].view(tot, hq, 128), rg[:, hq * 128:(hq + hkv) * 128].view(tot, hkv, 128),
                            rg[:, (hq + hkv) * 128:].view(tot, hkv, 128), cu.cuda(), cu.cuda(), max(lens), max(lens), scale)
    assert_vectors_close(got, want, f"packed prefill hq={hq} hkv={hkv}")


@pytest.mark.parametrize("bs", [16, 256])
def test_prefill_paged_prefix_and_chunk(ops, bs):
    """len_q < len_k: the keys of the cached prefix come from pages, mask is bottom-right aligned."""
    hq, hkv = 8, 2
    len_k = [300, 77, 512, 40]
    len_q = [44, 77, 1, 13]
    nblk = sum((c + bs - 1) // bs for c in len_k) + 2
    kv, ks, vs = bind_random_cache(ops, 2, nblk, hkv, bs, seed=41)
    tables = make_tables(len_k, bs, nblk, seed=7)
    tq = sum(len_q)
    q = bf(tq, hq, 128, seed=6)
    cu_q = torch.tensor([0] + list(torch.tensor(len_q).cumsum(0)), dtype=torch.int32)
    cu_k = torch.tensor([0] + list(torch.tensor(len_k).cumsum(0)), dtype=torch.int32)
    scale = 128 ** -0.5
    want = varlen_prefill_ref(q, None, None, cu_q, cu_k, scale, tables, ks[1], vs[1], p_dtype=torch.bfloat16)
    got = ops.paged_prefill(1, q.cuda(), None, None, cu_q.cuda(), cu_k.cuda(), max(len_q), max(len_k), scale,
                            block_tables=tables.cuda(), num_kv_heads=hkv)
    assert_vectors_close(got, want, f"paged prefill bs={bs}")


def test_prefill_long_causal_and_rescale(ops):
    """Many key blocks per query tile, and scores whose running maximum keeps growing by far more than 2^8, so the
    register accumulator is rescaled repeatedly (the lazy-rescale path of the wgmma kernel)."""
    hq, hkv = 4, 2
    lens = [1500, 900, 257]
    tot = sum(lens)
    g = torch.Generator().manual_seed(77)
    q = (torch.randn(tot, hq, 128, generator=g) * 3.0).to(torch.bfloat16)
    k = torch.randn(tot, hkv, 128, generator=g)
    ramp = torch.cat([torch.linspace(0.2, 4.0, n) for n in lens]).view(tot, 1, 1)     # later keys score much higher
    k = (k * ramp).to(torch.bfloat16)
    v = torch.randn(tot, hkv, 128, generator=g).to(torch.bfloat16)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32)
    scale = 128 ** -0.5
    want = varlen_prefill_ref(q, k, v, cu, cu, scale, p_dtype=torch.bfloat16)
    got = ops.paged_prefill(0, q.cuda(), k.cuda(), v.cuda(), cu.cuda(), cu.cuda(), max(lens), max(lens), scale)
    assert_vectors_close(got, want, "long causal prefill with growing maxima", ulps=3.0, rel_l2=6e-3)


@pytest.mark.parametrize("bs", [32, 64, 128])
def test_prefill_paged_block_sizes(ops, bs):
    hq, hkv = 16, 2                                       # G = 8
    len_k = [700, 129, 64]
    len_q = [300, 129, 1]
    nblk = sum((c + bs - 1) // bs for c in len_k) + 1
    kv, ks, vs = bind_random_cache(ops, 1, nblk, hkv, bs, seed=61)
    tables = make_tables(len_k, bs, nblk, seed=9)
    q = bf(sum(len_q), hq, 128, seed=16)
    cu_q = torch.tensor([0] + list(torch.tensor(len_q).cumsum(0)), dtype=torch.int32)
    cu_k = torch.tensor([0] + list(torch.tensor(len_k).cumsum(0)), dtype=torch.int32)
    scale = 128 ** -0.5
    want = varlen_prefill_ref(q, None, None, cu_q, cu_k, scale, tables, ks[0], vs[0], p_dtype=torch.bfloat16)
    got = ops.paged_prefill(0, q.cuda(), None, None, cu_q.cuda(), cu_k.cuda(), max(len_q), max(len_k), scale,
                            block_tables=tables.cuda(), num_kv_heads=hkv)
    assert_vectors_close(got, want, f"paged prefill bs={bs} G=8")


# ---------------------------------------------------------------------------------------------
# K5-K8 fused elementwise ops
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols", [(1, 1024), (37, 1024), (5, 4096), (3, 5120), (300, 256)])
def test_rmsnorm(ops, rows, cols):
    x, w = bf(rows, cols, seed=1), (1 + 0.1 * torch.randn(cols)).to(torch.bfloat16)
    got = ops.rmsnorm(x.cuda(), w.cuda(), 1e-6)
    assert_close_bf16(got, rmsnorm_ref(x, w, 1e-6), "rmsnorm", ulps=1.01)
    wide = bf(rows, cols + 64, seed=2)                                   # row-strided input view
    got = ops.rmsnorm(wide.cuda()[:, :cols], w.cuda(), 1e-6)
    assert_close_bf16(got, rmsnorm_ref(wide[:, :cols], w, 1e-6), "rmsnorm strided", ulps=1.01)


@pytest.mark.parametrize("rows,cols", [(1, 1024), (64, 1024), (7, 5120)])
def test_add_rmsnorm(ops, rows, cols):
    x, r, w = bf(rows, cols, seed=3), bf(rows, cols, seed=4), (1 + 0.1 * torch.randn(cols)).to(torch.bfloat16)
    want_y, want_r = add_rmsnorm_ref(x, r, w, 1e-6)
    rg = r.cuda()
    got_y, got_r = ops.add_rmsnorm(x.cuda(), rg, w.cuda(), 1e-6)
    assert got_r.data_ptr() == rg.data_ptr()
    assert torch.equal(got_r.cpu(), want_r), "residual = bf16(x + residual) must be bit-exact"
    assert_close_bf16(got_y, want_y, "add_rmsnorm", ulps=1.01)


@pytest.mark.parametrize("n", [29, 2501])          # 2501: the token-major kernel used for prefill-size batches
@pytest.mark.parametrize("hq,hkv,bs,cached", [(4, 2, 16, True), (16, 8, 256, True), (8, 1, 64, False), (2, 1, 32, True)])
def test_qknorm_rope_store(ops, hq, hkv, bs, cached, n):
    nblk, theta = max(5, (n + bs - 1) // bs + 2), 1e6
    kv, ks, vs = bind_random_cache(ops, 2, nblk, hkv, bs, seed=51)
    qkv = bf(n, (hq + 2 * hkv) * 128, seed=8)
    qw, kw = (1 + 0.1 * torch.randn(128)).to(torch.bfloat16), (1 + 0.1 * torch.randn(128)).to(torch.bfloat16)
    table = rope_table(128, 4096, theta)
    rp = random.Random(3)
    pos = torch.tensor([rp.randrange(4096) for _ in range(n)], dtype=torch.int64)
    slots = torch.tensor(random.Random(4).sample(range(nblk * bs), n), dtype=torch.int32)
    slots[3] = -1
    q = qkv[:, :hq * 128].view(n, hq, 128)
    k = qkv[:, hq * 128:(hq + hkv) * 128].view(n, hkv, 128)
    v = qkv[:, (hq + hkv) * 128:].view(n, hkv, 128)
    want_q = rope_ref(table, pos, rmsnorm_ref(q, qw, 1e-6))
    want_k = rope_ref(table, pos, rmsnorm_ref(k, kw, 1e-6))
    g = qkv.cuda()
    ops.qknorm_rope_store(1, g, hq, hkv, pos.cuda(), qw.cuda(), kw.cuda(), table.cuda(), 1e-6,
                          slots.cuda() if cached else None)
    out = g.cpu()
    assert_close_bf16(out[:, :hq * 128].view(n, hq, 128), want_q, "q norm+rope", ulps=1.01)
    assert_close_bf16(out[:, hq * 128:(hq + hkv) * 128].view(n, hkv, 128), want_k, "k norm+rope", ulps=1.01)
    assert torch.equal(out[:, (hq + hkv) * 128:], qkv[:, (hq + hkv) * 128:]), "v must pass through untouched"
    got_k = to_logical(kv[0, 1].cpu())
    got_v = to_logical(kv[1, 1].cpu())
    if cached:
        k_dev = out[:, hq * 128:(hq + hkv) * 128].reshape(n, hkv, 128)
        store_kvcache_ref(k_dev, v, ks[1], vs[1], slots)                      # the scatter itself is a bit-exact copy
    assert torch.equal(got_k, ks[1]) and torch.equal(got_v, vs[1])


def test_silu_mul(ops):
    x = bf(33, 2 * 3072, seed=9, scale=2.0)
    assert_close_bf16(ops.silu_mul(x.cuda()), silu_mul_ref(x), "silu_mul", ulps=1.01)


def test_embedding_bit_exact(ops):
    table = bf(1000, 256, seed=10)
    ids = torch.tensor([0, 999, 5, 5, 123], dtype=torch.int64)
    assert torch.equal(ops.embedding(ids.cuda(), table.cuda()).cpu(), table[ids])


# ---------------------------------------------------------------------------------------------
# K9 sampler
# ---------------------------------------------------------------------------------------------
def test_sample_greedy_is_first_argmax(ops):
    logits = bf(64, 151936, seed=12)
    logits[3, 100] = logits[3, 50000] = 30.0            # exact tie: lowest index wins
    logits[4, 151935] = 31.0
    got = ops.sample(logits.cuda(), torch.zeros(64).cuda(), seed=0, step=1).cpu()
    want = logits.float().argmax(dim=-1)
    want[3] = 100
    assert torch.equal(got, want)
    got32 = ops.sample(logits.float().cuda(), None, seed=0, step=1).cpu()
    assert torch.equal(got32, want)


def test_sample_temperature_matches_softmax(ops):
    torch.manual_seed(0)
    base = torch.tensor([2.0, 1.0, 0.0, -1.0, 0.5, -3.0, 1.5, 0.2])
    rows = 40000
    logits = base.repeat(rows, 1).cuda()
    t = 0.7
    got = ops.sample(logits, torch.full((rows,), t).cuda(), seed=123, step=7).cpu()
    freq = torch.bincount(got, minlength=8).float() / rows
    want = torch.softmax(base / t, dim=0)
    assert (freq - want).abs().max().item() < 0.012
    again = ops.sample(logits, torch.full((rows,), t).cuda(), seed=123, step=7).cpu()
    other = ops.sample(logits, torch.full((rows,), t).cuda(), seed=123, step=8).cpu()
    assert torch.equal(got, again) and not torch.equal(got, other)


def test_sample_sharded_keys_combine(ops):
    """Vocab-parallel combine: max over shard keys == single-shard result (same seed => same noise)."""
    logits = bf(16, 4096, seed=13)
    temps = torch.tensor([0.0, 0.9] * 8).cuda()
    full = ops.sample(logits.cuda(), temps, seed=5, step=3).cpu()
    keys = []
    for r in range(4):
        k = torch.empty(16, dtype=torch.int64, device="cuda")
        ops.sample(logits[:, r * 1024:(r + 1) * 1024].contiguous().cuda(), temps, seed=5, step=3, index_offset=r * 1024, out_keys=k)
        keys.append(k)
    best = torch.stack(keys).max(dim=0).values
    assert torch.equal(ops.tokens_from_keys(best).cpu(), full)


def test_errors_are_loud(ops):
    from nanovllm._native import B200Error
    with pytest.raises(B200Error):
        ops.silu_mul(torch.zeros(2, 16, dtype=torch.bfloat16))            # CPU tensor
    with pytest.raises(B200Error):
        ops.rmsnorm(torch.zeros(2, 16, device="cuda"), torch.ones(16, device="cuda"), 1e-6)   # fp32
    assert math.isfinite(1.0)


# ---------------------------------------------------------------------------------------------
# the operator seam: Attention module + Context, used the way the reference's model uses it
# ---------------------------------------------------------------------------------------------
def test_attention_module_seam_vs_oracle(ops):
    """Attention(num_heads, head_dim, scale, num_kv_heads).forward(q, k, v) reading the global Context and doing its own
    store_kvcache (reference layers/attention.py:59-75), for a packed prefill, a paged prefill and a decode step."""
    from types import SimpleNamespace
    from nanovllm.layers.attention import Attention
    from nanovllm.layers.activation import SiluAndMul
    from nanovllm.layers.layernorm import RMSNorm
    from nanovllm.layers.sampler import Sampler
    from nanovllm.utils.context import reset_context, set_context
    from oracle.paged_attention_ref import attention_forward_ref
    hq, hkv, bs, nblk = 4, 2, 16, 12
    kv, ks, vs = bind_random_cache(ops, 1, nblk, hkv, bs, seed=81)
    attn = Attention(hq, 128, 128 ** -0.5, hkv)
    attn.k_cache, attn.v_cache, attn.layer_id = kv[0, 0], kv[1, 0], 0
    lens = [20, 7]
    tables = make_tables([40, 30], bs, nblk, seed=3)
    i32 = lambda x: torch.tensor(x, dtype=torch.int32)

    def both(q, k, v, ctx_cpu):
        want = attention_forward_ref(q, k, v, ks[0], vs[0], ctx_cpu, 128 ** -0.5, p_dtype=torch.bfloat16 if ctx_cpu.is_prefill else None)
        g = lambda t: None if t is None else t.cuda()
        set_context(ctx_cpu.is_prefill, g(ctx_cpu.cu_seqlens_q), g(ctx_cpu.cu_seqlens_k), ctx_cpu.max_seqlen_q, ctx_cpu.max_seqlen_k,
                    g(ctx_cpu.slot_mapping), g(ctx_cpu.context_lens), g(ctx_cpu.block_tables))
        got = attn(q.cuda(), k.cuda(), v.cuda())
        reset_context()
        return got.reshape(want.shape), want

    # 1. packed prefill of two prompts
    tot = sum(lens)
    q, k, v = bf(tot, hq, 128, seed=1), bf(tot, hkv, 128, seed=2), bf(tot, hkv, 128, seed=3)
    slots = [int(tables[s, p // bs]) * bs + p % bs for s, n in enumerate(lens) for p in range(n)]
    c = SimpleNamespace(is_prefill=True, cu_seqlens_q=i32([0, 20, 27]), cu_seqlens_k=i32([0, 20, 27]), max_seqlen_q=20, max_seqlen_k=20,
                        slot_mapping=i32(slots), context_lens=None, block_tables=None)
    got, want = both(q, k, v, c)
    assert_vectors_close(got, want, "Attention module: packed prefill")
    assert torch.equal(to_logical(kv[0, 0].cpu()), ks[0]) and torch.equal(to_logical(kv[1, 0].cpu()), vs[0])
    # 2. second chunk of the first prompt through the paged path (len_q 5 over 25 keys)
    q, k, v = bf(5, hq, 128, seed=4), bf(5, hkv, 128, seed=5), bf(5, hkv, 128, seed=6)
    slots = [int(tables[0, p // bs]) * bs + p % bs for p in range(20, 25)]
    c = SimpleNamespace(is_prefill=True, cu_seqlens_q=i32([0, 5]), cu_seqlens_k=i32([0, 25]), max_seqlen_q=5, max_seqlen_k=25,
                        slot_mapping=i32(slots), context_lens=None, block_tables=tables[:1])
    got, want = both(q, k, v, c)
    assert_vectors_close(got, want, "Attention module: paged prefill")
    # 3. decode of both sequences
    q, k, v = bf(2, hq, 128, seed=7), bf(2, hkv, 128, seed=8), bf(2, hkv, 128, seed=9)
    ctxl = [26, 8]
    slots = [int(tables[s, (n - 1) // bs]) * bs + (n - 1) % bs for s, n in enumerate(ctxl)]
    c = SimpleNamespace(is_prefill=False, cu_seqlens_q=None, cu_seqlens_k=None, max_seqlen_q=0, max_seqlen_k=0,
                        slot_mapping=i32(slots), context_lens=i32(ctxl), block_tables=tables)
    got, want = both(q, k, v, c)
    assert got.shape == want.shape
    assert_vectors_close(got, want, "Attention module: decode")
    assert torch.equal(to_logical(kv[0, 0].cpu()), ks[0])
    # the other drop-in modules
    x = bf(9, 512, seed=10)
    norm = RMSNorm(512).cuda().to(torch.bfloat16)
    assert_close_bf16(norm(x.cuda()), rmsnorm_ref(x, norm.weight.cpu(), 1e-6), "RMSNorm module", ulps=1.01)
    y, r = norm(x.cuda(), x.cuda().clone())
    wy, wr = add_rmsnorm_ref(x, x, norm.weight.cpu(), 1e-6)
    assert torch.equal(r.cpu(), wr)
    assert_close_bf16(SiluAndMul()(x.cuda()), silu_mul_ref(x), "SiluAndMul module", ulps=1.01)
    lg = bf(5, 4096, seed=11)
    assert torch.equal(Sampler()(lg.cuda(), torch.zeros(5).cuda()).cpu(), lg.float().argmax(-1))
