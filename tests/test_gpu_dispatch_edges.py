"""Both sides of every host-side kernel choice, against float64 restatements of the same operations.

Each C entry point picks a kernel variant on the host: by shape (norm rows and columns, token count, head-group size,
batch rows) or by an environment variable the library reads once per process.  The cases below sit on both sides of
each of those boundaries, at the shapes production reaches (Qwen3-8B/14B dimensions, 1024-row decode batches, 40960-token
contexts, 4096-token prefills), and each one asserts which kernel actually ran, so that a later change of the dispatch
cannot quietly move a case to the other side.  The variables are covered by re-running the relevant subset of this
file in a child pytest with the variable set (``test_switch_*``).

The references are plain float64 torch on the device.  They round only where the kernel and the reference model round:
P to bf16 before PV in prefill attention, every projection output to bf16, the stored residual to bf16, the q/k norm
output to bf16 before RoPE.  The bars are the suite's: two bf16 ulps of the output scale and 4e-3 relative L2
(``assert_close_bf16``), four ulps and 1e-2 for the multi-stage layer tail.

Paged caches hold NaN in every row no sequence owns, and block tables are views into a wider buffer whose unused
columns name NaN pages: a read past a sequence's end shows up as a wrong value, never as an out-of-bounds access.
"""
import os
import random
import subprocess
import sys
import warnings
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD_GUARD = "B200_DISPATCH_EDGES_CHILD"          # set in the child pytest runs: they never spawn children of their own
IN_CHILD = os.environ.get(CHILD_GUARD) == "1"
D = 128
EPS = 1e-6
SCALE = D ** -0.5


@pytest.fixture(scope="module")
def ops():
    from nanovllm import ops as _ops
    return _ops


def randn(*shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def norm_weight(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (1 + 0.1 * torch.randn(n, generator=g, device="cuda")).to(torch.bfloat16)


def assert_close_bf16(got, want, what="", rel_l2=4e-3, ulps=2.0):
    got, want = got.double(), want.double()
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    scale = max(want.abs().max().item(), 1e-3)
    err = (got - want).abs().max().item()
    assert err <= ulps * scale * 2 ** -8, f"{what}: max abs err {err} vs scale {scale}"
    l2 = ((got - want).norm() / max(want.norm().item(), 1e-6)).item()
    assert l2 <= rel_l2, f"{what}: relative L2 {l2}"


def close_tail(got, want, what, ulps=4.0):
    """The layer tail's bar (test_gpu_layer_tail.py): four ulps of the output scale, 1e-2 relative L2."""
    got, want = got.double(), want.double()
    assert torch.isfinite(got).all(), f"{what}: non-finite"
    scale = max(want.abs().max().item(), 1e-3)
    err = (got - want).abs().max().item()
    rel = ((got - want).norm() / want.norm().clamp_min(1e-6)).item()
    assert err <= ulps * 2 ** -8 * scale and rel < 1e-2, f"{what}: max abs {err} (scale {scale}), rel L2 {rel}"


def edge_rows(n, extra=()):
    """Rows at the 64/128-row tile edges, the last row, and any extra rows (the last row of each sequence)."""
    return sorted({r for r in (0, 63, 64, 127, 128, n - 1, *extra) if 0 <= r < n})


def assert_rows_close(got, want, rows, what, **kw):
    for r in rows:
        assert_close_bf16(got[r], want[r], f"{what}, row {r}", **kw)


# ---------------------------------------------------------------------------------------------------------------------
# which kernel ran
# ---------------------------------------------------------------------------------------------------------------------
def launched(fn):
    """Run fn under torch.profiler.  Returns (fn's result, names of the CUDA kernels it launched), or None for the names
    when the profiler recorded no kernel events at all."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if getattr(e, "device_type", None) == DeviceType.CUDA]
    return out, (names or None)


def assert_ran(names, want, what):
    if names is None:
        warnings.warn(f"{what}: the profiler recorded no CUDA kernel events, so which kernel ran is not checked "
                      "(the numerical check still runs)")
        return
    assert any(want in n for n in names), f"{what}: expected a launch of {want}, the profiler saw {sorted(set(names))}"


# The expected kernel for each host-side choice, restating the library's dispatch (including the variables it reads).
def norm_kernel(rows, cols, res):
    max_rows = int(os.environ.get("B200_NORM_WARP_MAX_ROWS", "4096"))
    b = "true" if res else "false"
    if cols % 256 == 0 and cols // 256 in (1, 2, 4, 8) and rows <= max_rows:
        return f"rmsnorm_warp_kernel<{b}, {cols // 256}>"
    return f"rmsnorm_kernel<{b}>"


def qknorm_kernel(n):
    return "qknorm_rope_store_tok_kernel<8>" if n >= int(os.environ.get("B200_QKNORM_TOK_MIN", "2048")) else "qknorm_rope_store_kernel("


def decode_kernel(G, fused=False):
    if fused:
        return f"paged_decode_kernel<{G}, 8, 2, true>"
    if G > 2 or os.environ.get("B200_DECODE") == "mma":
        return f"paged_decode_mma_kernel<{G}>"
    nw, ns = {"12x2": (12, 2), "10x2": (10, 2), "8x3": (8, 3), "6x2": (6, 2)}.get(os.environ.get("B200_DECODE_CFG", ""), (8, 2))
    return f"paged_decode_kernel<{G}, {nw}, {ns}, false>"


def prefill_kernel():
    if os.environ.get("B200_PREFILL", "").startswith("w"):
        poly = int(os.environ.get("B200_PREFILL_POLY", "1")) != 0
        return f"prefill_ws_kernel<{'true' if poly else 'false'}>"
    return "prefill_tc_kernel"


# ---------------------------------------------------------------------------------------------------------------------
# float64 references
# ---------------------------------------------------------------------------------------------------------------------
def rmsnorm64(x, w, eps=EPS):
    xf = x.double()
    return xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps) * w.double()


def silu_mul64(x):
    g, u = x.double().chunk(2, -1)
    return g * torch.sigmoid(g) * u


def qknorm_rope64(x, w, pos, cos_sin):
    """q/k-norm then neox RoPE; x [n, H, D].  The norm's output is a stored bf16 tensor in the reference model."""
    nv = rmsnorm64(x, w).to(torch.bfloat16).double()
    cs = cos_sin[pos].double()[:, None, :]
    cos, sin = cs[..., :D // 2], cs[..., D // 2:]
    x1, x2 = nv[..., :D // 2], nv[..., D // 2:]
    return torch.cat((x1 * cos - x2 * sin, x2 * cos + x1 * sin), dim=-1)


def attend64(q, k, v, scale=SCALE):
    """Causal attention of one sequence, bottom-right aligned: q [Lq, Hq, D], k/v [Lk, Hkv, D] -> float64 [Lq, Hq, D].
    P = exp(S - max) is rounded to bf16 before PV (the tensor-core kernels feed a bf16 P to the MMA); the normaliser is
    the unrounded sum."""
    lq, hq, _ = q.shape
    lk, hkv, _ = k.shape
    g = hq // hkv
    kf = k.double().permute(1, 0, 2).repeat_interleave(g, 0)
    vf = v.double().permute(1, 0, 2).repeat_interleave(g, 0)
    out = torch.empty(lq, hq, D, dtype=torch.float64, device=q.device)
    step = max(1, (1 << 26) // (hq * lk))
    j = torch.arange(lk, device=q.device)[None, :]
    for a in range(0, lq, step):
        b = min(lq, a + step)
        s = q[a:b].double().permute(1, 0, 2) @ kf.transpose(1, 2) * scale
        i = torch.arange(a, b, device=q.device)[:, None]
        s.masked_fill_(j > i + (lk - lq), float("-inf"))
        p = torch.exp(s - s.amax(-1, keepdim=True))
        l = p.sum(-1, keepdim=True)
        out[a:b] = ((p.to(torch.bfloat16).double() @ vf) / l).permute(1, 0, 2)
    return out


def gather_seq(cache, table_row, n):
    """Rows 0..n-1 of one sequence out of a logical paged cache [nblk, bs, Hkv, D]."""
    bs = cache.shape[1]
    pos = torch.arange(n, device=cache.device)
    return cache[table_row[pos // bs].long(), pos % bs]


def prefill64(q, cu_q, cu_k, k=None, v=None, cache=None):
    """Varlen causal prefill; packed (k, v [T, Hkv, D]) or paged (cache: the PagedCache the keys live in)."""
    out = torch.zeros(q.shape, dtype=torch.float64, device=q.device)
    cq, ck = cu_q.tolist(), cu_k.tolist()
    for s in range(len(cq) - 1):
        if cq[s + 1] == cq[s]:
            continue
        if cache is None:
            ks, vs = k[ck[s]:ck[s + 1]], v[ck[s]:ck[s + 1]]
        else:
            n = ck[s + 1] - ck[s]
            ks, vs = gather_seq(cache.K, cache.tables[s], n), gather_seq(cache.V, cache.tables[s], n)
        out[cq[s]:cq[s + 1]] = attend64(q[cq[s]:cq[s + 1]], ks, vs)
    return out


def decode64(q, K, V, lens, tables, scale=SCALE):
    """One query token per sequence over keys 0..lens[b]-1 of a logical paged cache; zero-context rows give zeros."""
    B, hq, _ = q.shape
    bs, hkv = K.shape[1], K.shape[2]
    g = hq // hkv
    lens_t = torch.tensor(lens, device=q.device)
    out = torch.zeros(B, hq, D, dtype=torch.float64, device=q.device)
    i0 = 0
    while i0 < B:
        i1, L = i0, 0
        while i1 < B:                                   # rows per chunk: keep the gathered K/V near 1 GB of float64
            L2 = max(L, lens[i1])
            if i1 > i0 and (i1 + 1 - i0) * L2 * hkv * D > (1 << 27):
                break
            L, i1 = L2, i1 + 1
        if L > 0:
            pos = torch.arange(L, device=q.device)
            pages = tables[i0:i1][:, pos // bs].long()
            live = pos[None, :] < lens_t[i0:i1, None]
            k = torch.where(live[..., None, None], K[pages, pos % bs].double(), 0.0)
            v = torch.where(live[..., None, None], V[pages, pos % bs].double(), 0.0)
            s = torch.einsum("bkgd,blkd->bkgl", q[i0:i1].double().view(i1 - i0, hkv, g, D), k) * scale
            s = s.masked_fill(~live[:, None, None, :], float("-inf"))
            o = torch.einsum("bkgl,blkd->bkgd", torch.softmax(s, -1), v).reshape(i1 - i0, hq, D)
            o[lens_t[i0:i1] == 0] = 0.0
            out[i0:i1] = o
        i0 = i1
    return out


# ---------------------------------------------------------------------------------------------------------------------
# paged caches
# ---------------------------------------------------------------------------------------------------------------------
def build_paged(lens, bs, hkv, seed, data_seed=None, spare_cols=3, poison_pages=2, layers=1, key_shift=None):
    """Random K/V for sequences of the given lengths in shuffled pages.

    Returns a namespace with kv (physical [2, layers, nblk, Hkv, bs, D], the layout bind_kv_cache takes), K and V (the
    logical [nblk, bs, Hkv, D] view of the last layer's pages, for the reference) and tables: int32 [B, w], a view into
    a buffer spare_cols wider.  Table entries past a sequence's last page, inside the view and in the spare columns,
    name extra pages full of NaN, and every row of a used page past its sequence's end is NaN too.
    key_shift(pos) -> [rows, Hkv, D] is added to the keys of valid rows at sequence positions pos."""
    rnd = random.Random(seed)
    need = [(c + bs - 1) // bs for c in lens]
    used = sum(need)
    nblk = used + poison_pages
    perm = list(range(used))
    rnd.shuffle(perm)
    w = max(1, max(need))
    buf = (used + torch.arange(len(lens) * (w + spare_cols)) % poison_pages).to(torch.int32).view(len(lens), w + spare_cols)
    pos_of_row = torch.full((nblk, bs), -1, dtype=torch.int64)
    at = 0
    for i, (c, n) in enumerate(zip(lens, need)):
        pages = torch.tensor(perm[at:at + n], dtype=torch.int32)
        at += n
        buf[i, :n] = pages
        if n:
            p = torch.arange(c)
            pos_of_row[pages[p // bs].long(), p % bs] = p
    ds = seed if data_seed is None else data_seed
    K = randn(layers, nblk, bs, hkv, D, seed=ds * 7 + 1)
    V = randn(layers, nblk, bs, hkv, D, seed=ds * 7 + 2)
    pos_dev = pos_of_row.cuda()
    valid = pos_dev >= 0
    if key_shift is not None:
        K[-1][valid] = (K[-1][valid].double() + key_shift(pos_dev[valid])).to(torch.bfloat16)
    nan = torch.tensor(float("nan"), dtype=torch.bfloat16, device="cuda")
    K[:, ~valid] = nan
    V[:, ~valid] = nan
    kv = torch.stack([K.permute(0, 1, 3, 2, 4), V.permute(0, 1, 3, 2, 4)]).contiguous()
    tables = buf.cuda()[:, :w]
    assert tables.stride(0) == w + spare_cols
    return SimpleNamespace(kv=kv, K=K[-1], V=V[-1], tables=tables, lens=list(lens), bs=bs, hkv=hkv, nblk=nblk)


def cu(lens):
    return torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device="cuda")


# ---------------------------------------------------------------------------------------------------------------------
# RMSNorm / add+RMSNorm: warp-per-row kernel (cols % 256 == 0, cols <= 2048, rows <= 4096) vs block-per-row kernel
# ---------------------------------------------------------------------------------------------------------------------
NORM_CASES = [(4096, 1024), (4097, 1024), (64, 2048), (64, 2304), (64, 1536), (16384, 1024)]


@pytest.mark.parametrize("rows,cols", NORM_CASES)
def test_norm_rmsnorm(ops, rows, cols):
    x, w = randn(rows, cols, seed=rows + cols), norm_weight(cols, seed=cols)
    got, names = launched(lambda: ops.rmsnorm(x, w, EPS))
    assert_ran(names, norm_kernel(rows, cols, False), f"rmsnorm {rows}x{cols}")
    want = rmsnorm64(x, w)
    assert_close_bf16(got, want, f"rmsnorm {rows}x{cols}")
    assert_rows_close(got, want, edge_rows(rows), f"rmsnorm {rows}x{cols}")


@pytest.mark.parametrize("rows,cols", NORM_CASES)
def test_norm_add_rmsnorm(ops, rows, cols):
    x, r, w = randn(rows, cols, seed=rows), randn(rows, cols, seed=cols, scale=4.0), norm_weight(cols, seed=cols + 1)
    s = x.double() + r.double()
    want_r, want_y = s.to(torch.bfloat16), rmsnorm64(s, w)       # the norm reads the unrounded sum
    res = r.clone()
    (got_y, got_r), names = launched(lambda: ops.add_rmsnorm(x, res, w, EPS))
    assert_ran(names, norm_kernel(rows, cols, True), f"add_rmsnorm {rows}x{cols}")
    assert got_r.data_ptr() == res.data_ptr()
    assert torch.equal(got_r, want_r), "residual = bf16(x + residual) must be bit-exact"
    assert_close_bf16(got_y, want_y, f"add_rmsnorm {rows}x{cols}")
    assert_rows_close(got_y, want_y, edge_rows(rows), f"add_rmsnorm {rows}x{cols}")


# ---------------------------------------------------------------------------------------------------------------------
# SiluAndMul: 16384 x 3072 needs more CTAs than the 16-per-SM cap, so the kernel grid-strides; 1 x 8 is one partial CTA
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,inter", [(16384, 3072), (1, 8)])
def test_silu_mul_grid(ops, rows, inter):
    x = randn(rows, 2 * inter, seed=inter, scale=2.0)
    got, names = launched(lambda: ops.silu_mul(x))
    assert_ran(names, "silu_mul_kernel", f"silu_mul {rows}x{inter}")
    want = silu_mul64(x)
    assert_close_bf16(got, want, f"silu_mul {rows}x{inter}")
    assert_rows_close(got, want, edge_rows(rows), f"silu_mul {rows}x{inter}")


# ---------------------------------------------------------------------------------------------------------------------
# q/k-norm + RoPE + KV store: per-(token, head) kernel below 2048 tokens, token-major kernel from 2048
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [2047, 2048])
def test_qknorm_rope_store_boundary(ops, n):
    from oracle.qwen3_ref import rope_table
    hq, hkv, bs, layer = 32, 8, 256, 1
    nblk = (n + bs - 1) // bs + 2
    kv = randn(2, 2, nblk, hkv, bs, D, seed=n)
    ops.bind_kv_cache(kv)
    qkv = randn(n, (hq + 2 * hkv) * D, seed=n + 1)
    qw, kw = norm_weight(D, seed=1), norm_weight(D, seed=2)
    table = rope_table(D, 40960, 1e6).cuda()
    rnd = random.Random(n)
    pos = [rnd.randrange(40960) for _ in range(n)]
    pos[0], pos[n - 1], pos[n // 2] = 40959, 40958, 0
    pos = torch.tensor(pos, dtype=torch.int64, device="cuda")
    slots = torch.tensor(rnd.sample(range(nblk * bs), n), dtype=torch.int32)
    slots[::37] = -1
    slots[n - 1] = -1
    slots = slots.cuda()
    q_in = qkv[:, :hq * D].view(n, hq, D)
    k_in = qkv[:, hq * D:(hq + hkv) * D].view(n, hkv, D)
    v_in = qkv[:, (hq + hkv) * D:].clone()
    want_q, want_k = qknorm_rope64(q_in, qw, pos, table), qknorm_rope64(k_in, kw, pos, table)
    before = kv.clone()
    g = qkv.clone()
    _, names = launched(lambda: ops.qknorm_rope_store(layer, g, hq, hkv, pos, qw, kw, table, EPS, slots))
    assert_ran(names, qknorm_kernel(n), f"qknorm_rope_store n={n}")
    got_q, got_k = g[:, :hq * D].view(n, hq, D), g[:, hq * D:(hq + hkv) * D].view(n, hkv, D)
    assert_close_bf16(got_q, want_q, f"q norm+rope n={n}")
    assert_close_bf16(got_k, want_k, f"k norm+rope n={n}")
    rows = edge_rows(n, extra=(n // 2,))
    assert_rows_close(got_q, want_q, rows, f"q norm+rope n={n}")
    assert_rows_close(got_k, want_k, rows, f"k norm+rope n={n}")
    assert torch.equal(g[:, (hq + hkv) * D:], v_in), "v must pass through untouched"
    # the scatter is a copy of the rotated k and the raw v into the slots; slot -1 and the other layer stay as they were
    want_kv = before.clone()
    keep = slots >= 0
    for c, src in ((0, got_k), (1, v_in.view(n, hkv, D))):
        flat = want_kv[c, layer].permute(0, 2, 1, 3).reshape(nblk * bs, hkv, D)
        flat[slots[keep].long()] = src[keep]
        want_kv[c, layer] = flat.view(nblk, bs, hkv, D).permute(0, 2, 1, 3)
    assert torch.equal(kv, want_kv)


# ---------------------------------------------------------------------------------------------------------------------
# paged decode: FMA kernel (G <= 2, variants by B200_DECODE_CFG) vs tensor-core kernel (G in {4, 8}, or B200_DECODE=mma)
# ---------------------------------------------------------------------------------------------------------------------
def mixed_lens(batch, seed):
    rnd = random.Random(seed)
    lens = [rnd.randint(1, 700) for _ in range(batch)]
    head = [0, 1, 15, 16, 17, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1000, 2048]
    lens[:len(head)] = head
    for i in range(40, batch, 97):
        lens[i] = 0
    lens[-1] = 0
    lens[-2] = 1999
    return lens


@pytest.mark.parametrize("G", [1, 2, 4, 8], ids=lambda G: f"G{G}")
def test_decode_batch_1024_mixed_and_workspace_reuse(ops, G):
    from nanovllm import _native as nat
    hkv, bs, batch = 2, 64, 1024
    lens = mixed_lens(batch, seed=G)
    c = build_paged(lens, bs, hkv, seed=G)
    ops.bind_kv_cache(c.kv)
    q = randn(batch, G * hkv, D, seed=100 + G)
    ctx = torch.tensor(lens, dtype=torch.int32, device="cuda")
    got, names = launched(lambda: ops.paged_decode(0, q, c.tables, ctx, SCALE))
    assert_ran(names, decode_kernel(G), f"decode G={G} batch {batch}")
    want = decode64(q, c.K, c.V, lens, c.tables)
    assert_close_bf16(got, want, f"decode G={G} batch {batch}")
    assert_rows_close(got, want, [i for i in edge_rows(batch, extra=range(16)) if lens[i]], f"decode G={G}")
    zero = ctx == 0
    assert (got[zero] == 0).all(), "zero-context rows are exactly zero"
    # one workspace through batch 1024 -> 3 -> 1024: the counters left behind must not change a bit
    small = ops.paged_decode(0, q[:3], c.tables[:3], ctx[:3], SCALE)
    assert_close_bf16(small, want[:3], f"decode G={G} batch 3")
    again = ops.paged_decode(0, q, c.tables, ctx, SCALE)
    nat.handle().workspace = None                         # a fresh zeroed workspace
    fresh = ops.paged_decode(0, q, c.tables, ctx, SCALE)
    assert torch.equal(again, got) and torch.equal(fresh, got)


@pytest.mark.parametrize("G", [2, 4], ids=lambda G: f"G{G}")
@pytest.mark.parametrize("nseq", [1, 4])
def test_decode_long_context_rising_max(ops, nseq, G):
    """Contexts of 40960 tokens: one (sequence, kv head) is split over many warps and merged from partials.  The keys
    lean more and more towards the queries along the sequence, so the running maximum keeps rising across every segment
    boundary and each merge has to rescale."""
    hkv, bs = 8, 256
    lens = [40960] * nseq
    if nseq > 1:
        lens[1] = 40959
    g = torch.Generator(device="cuda").manual_seed(nseq * 10 + G)
    u = torch.randn(hkv, D, generator=g, device="cuda", dtype=torch.float64)
    c = build_paged(lens, bs, hkv, seed=nseq * 10 + G,
                    key_shift=lambda pos: (3.0 * pos.double() / 40960)[:, None, None] * u[None])
    ops.bind_kv_cache(c.kv)
    q = (0.5 * u.repeat_interleave(G, 0)[None] + torch.randn(nseq, G * hkv, D, generator=g, device="cuda", dtype=torch.float64))
    q = q.to(torch.bfloat16)
    ctx = torch.tensor(lens, dtype=torch.int32, device="cuda")
    got, names = launched(lambda: ops.paged_decode(0, q, c.tables, ctx, SCALE))
    assert_ran(names, decode_kernel(G), f"decode G={G} context 40960")
    want = decode64(q, c.K, c.V, lens, c.tables)
    assert_close_bf16(got, want, f"decode G={G} {nseq} x 40960")
    for i in range(nseq):
        assert_close_bf16(got[i], want[i], f"decode G={G} sequence {i}")


@pytest.mark.parametrize("G", [1, 2], ids=lambda G: f"G{G}")
@pytest.mark.parametrize("batch", [128, 129])
def test_fused_decode_strided_table(ops, batch, G):
    """b200_paged_decode_fused: q/k-norm + RoPE of the step's token, its K/V append at position ctx-1 (slot from the
    block table, a view into a wider buffer), then attention over the updated cache."""
    from oracle.qwen3_ref import rope_table
    hkv, bs = 8, 64
    hq = G * hkv
    rnd = random.Random(batch + G)
    lens = [rnd.randint(1, 900) for _ in range(batch)]
    lens[:6] = [1, 63, 64, 65, 0, 128]
    lens[-1] = 129
    c = build_paged(lens, bs, hkv, seed=batch + G)
    qkv = randn(batch, (hq + 2 * hkv) * D, seed=batch * G)
    qw, kw = norm_weight(D, seed=3), norm_weight(D, seed=4)
    table = rope_table(D, 4096, 1e6).cuda()
    ctx = torch.tensor(lens, dtype=torch.int32, device="cuda")
    pos = (ctx.long() - 1).clamp(min=0)
    live = ctx > 0
    tab = c.tables.long()
    slots = tab[torch.arange(batch, device="cuda"), pos // bs] * bs + pos % bs
    q_o = qknorm_rope64(qkv[:, :hq * D].view(batch, hq, D), qw, pos, table).to(torch.bfloat16)
    k_o = qknorm_rope64(qkv[:, hq * D:(hq + hkv) * D].view(batch, hkv, D), kw, pos, table).to(torch.bfloat16)
    v_in = qkv[:, (hq + hkv) * D:].view(batch, hkv, D)
    K2, V2 = c.K.clone(), c.V.clone()
    K2.view(-1, hkv, D)[slots[live]] = k_o[live]
    V2.view(-1, hkv, D)[slots[live]] = v_in[live]
    want = decode64(q_o, K2, V2, lens, c.tables)
    ops.bind_kv_cache(c.kv)
    src = qkv.clone()
    got, names = launched(lambda: ops.paged_decode_fused(0, qkv, hq, qw, kw, table, EPS, c.tables, ctx, SCALE))
    assert_ran(names, decode_kernel(G, fused=True), f"fused decode G={G} batch {batch}")
    assert torch.equal(qkv, src), "the fused kernel must not modify the projection output"
    assert_close_bf16(got, want, f"fused decode G={G} batch {batch}")
    assert_rows_close(got, want, [i for i in edge_rows(batch, extra=range(6)) if lens[i]], f"fused decode G={G}")
    assert (got[~live] == 0).all()
    gotK, gotV = c.kv[0, 0].permute(0, 2, 1, 3), c.kv[1, 0].permute(0, 2, 1, 3)
    assert torch.equal(gotV.nan_to_num(7.0), V2.nan_to_num(7.0)), "V append is a copy; every other row is unchanged"
    assert_close_bf16(gotK.reshape(-1, hkv, D)[slots[live]], k_o[live], "appended K rows")
    untouched = torch.ones(c.nblk * bs, dtype=torch.bool, device="cuda")
    untouched[slots[live]] = False
    assert torch.equal(gotK.reshape(-1, hkv, D)[untouched].nan_to_num(7.0), c.K.reshape(-1, hkv, D)[untouched].nan_to_num(7.0))


# ---------------------------------------------------------------------------------------------------------------------
# paged / packed prefill: prefill_tc.cu, or prefill_ws.cu with B200_PREFILL=ws (odd groups mix two-head and one-head CTAs)
# ---------------------------------------------------------------------------------------------------------------------
def check_prefill(got, want, lens_q, what):
    assert_close_bf16(got, want, what)
    ends = torch.tensor(lens_q).cumsum(0) - 1
    assert_rows_close(got, want, edge_rows(got.shape[0], extra=ends.tolist()), what)


@pytest.mark.parametrize("paged", [False, True], ids=["packed", "paged"])
@pytest.mark.parametrize("hq", [24, 40])
def test_prefill_odd_group(ops, hq, paged):
    hkv = 8
    lens_q = [1, 63, 64, 65, 127, 128, 129, 300]
    q = randn(sum(lens_q), hq, D, seed=hq)
    if not paged:
        k, v = randn(sum(lens_q), hkv, D, seed=hq + 1), randn(sum(lens_q), hkv, D, seed=hq + 2)
        want = prefill64(q, cu(lens_q), cu(lens_q), k, v)
        got, names = launched(lambda: ops.paged_prefill(0, q, k, v, cu(lens_q), cu(lens_q), max(lens_q), max(lens_q), SCALE))
    else:
        lens_k = [a + b for a, b in zip(lens_q, [0, 5, 64, 100, 1, 200, 0, 37])]
        c = build_paged(lens_k, 16, hkv, seed=hq)
        ops.bind_kv_cache(c.kv)
        want = prefill64(q, cu(lens_q), cu(lens_k), cache=c)
        got, names = launched(lambda: ops.paged_prefill(0, q, None, None, cu(lens_q), cu(lens_k), max(lens_q), max(lens_k),
                                                        SCALE, block_tables=c.tables, num_kv_heads=hkv))
    assert_ran(names, prefill_kernel(), f"prefill G={hq // hkv}")
    check_prefill(got, want, lens_q, f"{'paged' if paged else 'packed'} prefill G={hq // hkv}")


def test_prefill_one_4096_token_sequence(ops):
    hq, hkv, n = 32, 8, 4096
    q, k, v = randn(n, hq, D, seed=1), randn(n, hkv, D, seed=2), randn(n, hkv, D, seed=3)
    got, names = launched(lambda: ops.paged_prefill(0, q, k, v, cu([n]), cu([n]), n, n, SCALE))
    assert_ran(names, prefill_kernel(), "prefill 4096 tokens")
    check_prefill(got, prefill64(q, cu([n]), cu([n]), k, v), [n], "packed prefill of 4096 tokens")


@pytest.mark.parametrize("bs", [16, 256])
def test_prefill_chunk_over_long_prefix(ops, bs):
    """Chunked prefill: 512 new tokens over a 4096-token context whose first 3584 keys are cached pages."""
    hq, hkv, lq, lk = 32, 8, 512, 4096
    c = build_paged([lk], bs, hkv, seed=bs)
    ops.bind_kv_cache(c.kv)
    q = randn(lq, hq, D, seed=bs + 1)
    want = prefill64(q, cu([lq]), cu([lk]), cache=c)
    got, names = launched(lambda: ops.paged_prefill(0, q, None, None, cu([lq]), cu([lk]), lq, lk, SCALE,
                                                    block_tables=c.tables, num_kv_heads=hkv))
    assert_ran(names, prefill_kernel(), f"chunked prefill bs={bs}")
    check_prefill(got, want, [lq], f"chunked prefill 512 over 4096, bs={bs}")


def test_prefill_512_short_sequences(ops):
    """A step of 512 sequences of 1-3 new tokens each over cached prefixes: 512 CTAs along grid.z."""
    hq, hkv = 32, 8
    rnd = random.Random(5)
    lens_q = [rnd.randint(1, 3) for _ in range(512)]
    lens_k = [a + rnd.choice([0, 0, 1, 15, 16, 63, 64, rnd.randint(0, 300)]) for a in lens_q]
    c = build_paged(lens_k, 16, hkv, seed=512)
    ops.bind_kv_cache(c.kv)
    q = randn(sum(lens_q), hq, D, seed=512)
    want = prefill64(q, cu(lens_q), cu(lens_k), cache=c)
    got, names = launched(lambda: ops.paged_prefill(0, q, None, None, cu(lens_q), cu(lens_k), max(lens_q), max(lens_k), SCALE,
                                                    block_tables=c.tables, num_kv_heads=hkv))
    assert_ran(names, prefill_kernel(), "prefill of 512 short sequences")
    check_prefill(got, want, lens_q, "prefill of 512 short sequences")


# ---------------------------------------------------------------------------------------------------------------------
# sampler: up to 16 vocabulary slices per row at <= 1024 rows, one slice above; bf16 scalar tail for vocab % 8 != 0
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 64, 1024, 1025])
def test_sample_greedy_first_index_ties(ops, rows):
    vocab = 151936
    logits = randn(rows, vocab, seed=rows)
    rnd = random.Random(rows)
    want = torch.empty(rows, dtype=torch.int64)
    for r in range(rows):
        a, b = sorted(rnd.sample(range(vocab), 2))
        if r % 5 == 1:
            a, b = 0, vocab - 1                      # tie between the first and the last id
        elif r % 5 == 2:
            b = a + 1                                # tie inside one 8-element vector
        logits[r, b] = logits[r, a] = 8.0 + (r % 3)
        want[r] = a
    want = want.cuda()
    got, names = launched(lambda: ops.sample(logits, torch.zeros(rows, device="cuda"), seed=0, step=1))
    assert_ran(names, "sample_kernel<false>", f"greedy sample of {rows} rows")
    assert torch.equal(got, want)
    assert torch.equal(ops.sample(logits.float(), None, seed=0, step=1), want)


def test_sample_split_count_independence(ops):
    """Row r gives the same token whether its batch has 1025 rows (one slice per row) or r + 1 rows (several slices)."""
    rows, vocab = 1025, 151936
    logits = randn(rows, vocab, seed=11, scale=2.0)
    temps = torch.tensor([0.0 if r % 4 == 0 else 0.9 for r in range(rows)], device="cuda")
    full = ops.sample(logits, temps, seed=7, step=3)
    for r in (0, 1, 63, 131, 263, 527, 1023):
        part = ops.sample(logits[:r + 1], temps[:r + 1], seed=7, step=3)
        assert torch.equal(part, full[:r + 1]), f"a batch of {r + 1} rows samples differently from the 1025-row batch"
    assert not torch.equal(ops.sample(logits, temps, seed=7, step=4)[temps > 0], full[temps > 0])


@pytest.mark.parametrize("rows", [16, 1025])
@pytest.mark.parametrize("vocab", [1003, 151939])
def test_sample_bf16_view_with_ragged_vocab(ops, rows, vocab):
    """bf16 logits as a view into a wider buffer with vocab % 8 != 0: the last ids go through the scalar tail loop, and
    nothing past the view is read."""
    stride = (vocab + 8) // 8 * 8
    buf = randn(rows, stride, seed=vocab + rows)
    buf[:, vocab:] = 100.0                                   # outside the view: must never win
    view = buf[:, :vocab]
    want = view.float().argmax(-1)
    want[0::3] = vocab - 1
    want[1::3] = vocab - 3
    idx = torch.arange(rows, device="cuda")
    buf[idx[0::3], vocab - 1] = 50.0
    buf[idx[1::3], vocab - 3] = 50.0
    got, names = launched(lambda: ops.sample(view, torch.zeros(rows, device="cuda"), seed=1, step=2))
    assert_ran(names, "sample_kernel<false>", "sample of a ragged bf16 view")
    assert torch.equal(got, want)
    temps = torch.full((rows,), 0.8, device="cuda")
    a = ops.sample(view, temps, seed=3, step=9)
    assert int(a.max()) < vocab
    assert torch.equal(a, ops.sample(view.float().contiguous(), temps, seed=3, step=9)), "bf16 view vs fp32 copy"


# ---------------------------------------------------------------------------------------------------------------------
# wgmma linear at Qwen3-8B shapes and their two-way tensor-parallel shards
# ---------------------------------------------------------------------------------------------------------------------
LINEAR_SHAPES = {            # name: (output columns, k, epilogue, block_n, k splits)
    "qkv_8b": (6144, 4096, 0, 32, 1),
    "qkv_8b_tp2": (3072, 4096, 0, 64, 1),
    "gate_up_8b": (12288, 4096, 1, 64, 1),
    "gate_up_8b_tp2": (6144, 4096, 1, 128, 1),
    "o_proj_8b": (4096, 4096, 2, 64, 8),
    "down_8b": (4096, 12288, 2, 64, 8),
    "down_8b_tp2": (4096, 6144, 2, 32, 8),
}


@pytest.mark.parametrize("rows", [1, 65, 128, 129, 256])
@pytest.mark.parametrize("shape", list(LINEAR_SHAPES))
def test_linear_8b_shapes(ops, shape, rows):
    n, k, epi, bn, splits = LINEAR_SHAPES[shape]
    x = randn(rows, k, seed=rows + k)
    w = randn(2 * n if epi == ops.EPI_SILU else n, k, seed=n + k, scale=k ** -0.5)
    got, names = launched(lambda: ops.linear(x, w, epi, bn, splits))
    assert_ran(names, f"linear_tc_kernel<{bn}, {epi}, ", f"linear {shape}")
    h = x.double() @ w.double().t()
    if epi == ops.EPI_BF16:
        want = h.to(torch.bfloat16)
        assert_close_bf16(got, want, f"linear {shape} rows={rows}")
        assert_rows_close(got, want, edge_rows(rows), f"linear {shape}")
    elif epi == ops.EPI_SILU:
        y = h.to(torch.bfloat16).double()
        want = y[:, :n] * torch.sigmoid(y[:, :n]) * y[:, n:]
        assert_close_bf16(got, want, f"linear+silu {shape} rows={rows}", ulps=4.0)      # test_gpu_linear.py's 2^-6 bar
        assert_rows_close(got, want, edge_rows(rows), f"linear+silu {shape}", ulps=4.0)
    else:
        assert got.shape == (splits, rows, n)
        err = (got.double().sum(0) - h).abs().max().item()
        assert err <= 1e-3 * max(1.0, h.abs().max().item()), f"split-K partials {shape} rows={rows}: max abs err {err}"


# ---------------------------------------------------------------------------------------------------------------------
# persistent layer tail at Qwen3-8B dimensions, 1 to 8 row blocks of 128
# ---------------------------------------------------------------------------------------------------------------------
TAIL_DIMS = (4096, 4096, 12288, 6144)            # hidden, q_size, intermediate, next qkv


@pytest.fixture(scope="module")
def tail_weights():
    hidden, q_size, inter, qkv_n = TAIL_DIMS
    return dict(wo=randn(hidden, q_size, seed=1, scale=q_size ** -0.5), ln_mid=norm_weight(hidden, seed=2),
                wgu=randn(2 * inter, hidden, seed=3, scale=hidden ** -0.5), wd=randn(hidden, inter, seed=4, scale=inter ** -0.5),
                ln_next=norm_weight(hidden, seed=5), wqkv=randn(qkv_n, hidden, seed=6, scale=hidden ** -0.5))


def layer_tail64(attn, resid, w):
    """o_proj -> add+RMSNorm -> gate_up + SiluAndMul -> down_proj -> add+RMSNorm -> next qkv_proj in float64, rounded to
    bf16 where the reference model stores a tensor: every projection output, the residual, the normed rows, the act."""
    bf = lambda t: t.to(torch.bfloat16).double()
    inter = w["wd"].shape[1]
    h1 = bf(attn.double() @ w["wo"].double().t())
    s1 = h1 + resid.double()
    x = bf(rmsnorm64(s1, w["ln_mid"]))
    gu = bf(x @ w["wgu"].double().t())
    act = bf(gu[:, :inter] * torch.sigmoid(gu[:, :inter]) * gu[:, inter:])
    s2 = bf(act @ w["wd"].double().t()) + bf(s1)
    xn = rmsnorm64(s2, w["ln_next"])
    return s2.to(torch.bfloat16), xn, bf(xn) @ w["wqkv"].double().t()


@pytest.mark.parametrize("rows", [1, 129, 256, 257, 512, 1024])
def test_layer_tail_8b_row_blocks(ops, tail_weights, rows):
    hidden, q_size, inter, _ = TAIL_DIMS
    w = tail_weights
    attn, resid = randn(rows, q_size, seed=rows), randn(rows, hidden, seed=rows + 1)
    want_r, want_x, want_qkv = layer_tail64(attn, resid, w)
    ws = ops.layer_tail_workspace(1024, hidden, inter, 8)
    r = resid.clone()
    (x_next, qkv), names = launched(lambda: ops.layer_tail(attn, r, w["wo"], w["ln_mid"], w["wgu"], w["wd"], w["ln_next"], EPS, ws,
                                                           w_qkv_next=w["wqkv"]))
    assert_ran(names, "layer_tail_kernel", f"layer tail rows={rows}")
    assert not ops.layer_tail_error(ws), "a grid barrier timed out"
    close_tail(r, want_r, f"residual rows={rows}")
    close_tail(x_next, want_x, f"x_next rows={rows}")
    close_tail(qkv, want_qkv, f"next qkv rows={rows}")
    for i in edge_rows(rows):
        close_tail(x_next[i], want_x[i], f"x_next row {i}")
        close_tail(qkv[i], want_qkv[i], f"next qkv row {i}")


# ---------------------------------------------------------------------------------------------------------------------
# host-side refusals: argument checks before any launch
# ---------------------------------------------------------------------------------------------------------------------
def test_refuse_unsupported_arguments(ops):
    from nanovllm._native import B200Error
    from oracle.qwen3_ref import rope_table
    hkv = 2
    c = build_paged([5], 16, hkv, seed=1)
    ops.bind_kv_cache(c.kv)
    tables = torch.zeros(1025, 1, dtype=torch.int32, device="cuda")
    ctx = torch.ones(1025, dtype=torch.int32, device="cuda")
    with pytest.raises(B200Error):                                    # more rows than the decode kernels' prefix table
        ops.paged_decode(0, randn(1025, 2 * hkv, D, seed=1), tables, ctx, SCALE)
    for G in (3, 5, 16):                                              # head groups without a decode kernel
        with pytest.raises(B200Error):
            ops.paged_decode(0, randn(2, G * hkv, D, seed=G), tables[:2], ctx[:2], SCALE)
    with pytest.raises(B200Error):                                    # the fused decode exists for G <= 2 only
        ops.paged_decode_fused(0, randn(2, (4 * hkv + 2 * hkv) * D, seed=4), 4 * hkv, norm_weight(D, 1), norm_weight(D, 2),
                               rope_table(D, 64, 1e6).cuda(), EPS, tables[:2], ctx[:2], SCALE)
    hidden, q_size, inter = 256, 512, 512
    ws = ops.layer_tail_workspace(1024, hidden, inter, 8)
    with pytest.raises(B200Error):                                    # the layer tail takes at most 1024 rows
        ops.layer_tail(randn(1025, q_size, seed=1), randn(1025, hidden, seed=2), randn(hidden, q_size, seed=3), norm_weight(hidden, 4),
                       randn(2 * inter, hidden, seed=5), randn(hidden, inter, seed=6), norm_weight(hidden, 7), EPS, ws)


# ---------------------------------------------------------------------------------------------------------------------
# the tensor-core decode's cached tensor maps across contexts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("G", [4, 2], ids=lambda G: f"G{G}")
def test_context_reset_body(ops, G):
    """reset -> bind cache X -> decode -> reset -> bind cache Y -> decode must read Y.  X and Y have the same shape and
    both stay alive, so maps left over from X would read valid memory and give X's values."""
    if not IN_CHILD:
        pytest.skip("needs a fresh process: test_context_reset_in_fresh_process runs it")
    from nanovllm import _native as nat
    hkv, bs = 2, 16
    lens = [37, 200, 1, 64, 0, 129]
    x = build_paged(lens, bs, hkv, seed=1, data_seed=1)
    y = build_paged(lens, bs, hkv, seed=1, data_seed=2)
    q = randn(len(lens), G * hkv, D, seed=3)
    ctx = torch.tensor(lens, dtype=torch.int32, device="cuda")
    for c in (x, y):
        nat.reset_handle()
        ops.bind_kv_cache(c.kv)
        got, names = launched(lambda: ops.paged_decode(0, q, c.tables, ctx, SCALE))
        assert_ran(names, decode_kernel(G), f"decode G={G} after a context reset")
        assert_close_bf16(got, decode64(q, c.K, c.V, lens, c.tables), f"decode G={G} of the cache bound after a reset")


def run_child(kexpr, env):
    cmd = [sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu", "-k", kexpr, os.path.abspath(__file__)]
    r = subprocess.run(cmd, env=dict(os.environ, **env, **{CHILD_GUARD: "1"}), cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and " failed" not in r.stdout, r.stdout[-2000:]


@pytest.mark.parametrize("decode", ["default", "mma"])
def test_context_reset_in_fresh_process(decode):
    if IN_CHILD:
        pytest.skip("already a child process")
    run_child("context_reset_body", {} if decode == "default" else {"B200_DECODE": "mma"})


# The library reads these variables once per process: each one reruns the cases of its branch in a child pytest.
SWITCHES = {
    "decode_mma": ({"B200_DECODE": "mma"}, "decode and not fused"),
    "decode_cfg_12x2": ({"B200_DECODE_CFG": "12x2"}, "decode and not fused and (G1 or G2)"),
    "decode_cfg_10x2": ({"B200_DECODE_CFG": "10x2"}, "decode and not fused and (G1 or G2)"),
    "decode_cfg_8x3": ({"B200_DECODE_CFG": "8x3"}, "decode and not fused and (G1 or G2)"),
    "decode_cfg_6x2": ({"B200_DECODE_CFG": "6x2"}, "decode and not fused and (G1 or G2)"),
    "decode_l2hint_off": ({"B200_DECODE_L2HINT": "0"}, "decode"),
    "norm_block_only": ({"B200_NORM_WARP_MAX_ROWS": "0"}, "test_norm"),
    "qknorm_token_major_only": ({"B200_QKNORM_TOK_MIN": "1"}, "qknorm"),
    "prefill_ws_poly": ({"B200_PREFILL": "ws", "B200_PREFILL_POLY": "1"}, "prefill"),
    "prefill_ws_mufu": ({"B200_PREFILL": "ws", "B200_PREFILL_POLY": "0"}, "prefill"),
}


@pytest.mark.parametrize("switch", list(SWITCHES))
def test_switch_variant(switch):
    if IN_CHILD:
        pytest.skip("already a child process")
    env, kexpr = SWITCHES[switch]
    run_child(kexpr, env)
