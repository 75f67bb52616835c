"""Needle cases for the attention kernels, shared by tests/test_gpu_attention_needles.py (the kernels) and
tests/test_attention_needles_host.py (the cases' power, on the CPU).

A defect at one key position deep inside a long context (a segment boundary of the stream-K decode split, the merge of
its partials, a page or 16-token chunk edge, the causal diagonal of a 64-key tile, the lazy rescale of prefill) moves a
random-input output by about 1/L of its size, far below a bf16 bar.  These cases make each such key carry a fixed,
large share of its query head's attention:

* every query head is one-hot, BETA along a dimension of its own (head g of a kv head uses dimension g), so the
  G heads of a kv head are orthogonal and each can have needles of its own;
* background keys are randn * BG, so background scores sit within a few tenths of a nat of 0 (or of a chosen base);
* a needle key has score ~ln(L / m) for its head (m needles in the head, L keys visible), so the needles hold about
  half of the head's mass together;
* a needle's V row is A in one dimension of its own and 0 elsewhere, so each needle owns one output dimension and
  dropping it, or reading another key in its place, moves that dimension by its whole share.

The bar is per (row, query head) vector of 128 values: max abs error <= 2 * 2^-8 * max|ref of that vector| (plus a
1e-6 floor for all-zero vectors), so a long row's small outputs are not judged at the scale of a short row's large ones.

Stale cache rows right past a sequence's end (same page) hold a trap: a key that scores above every needle of every
head and a V row in dimension TRAP_DIM.  Other stale rows and unused pages are NaN (build_paged).

Everything takes a device: the GPU file builds on cuda, the host file the very same cases on the CPU.
"""
import math
from types import SimpleNamespace

import torch

from kv_fp8_ref import dequantize_e4m3, quantize_e4m3
from test_gpu_dispatch_edges import (D, SCALE, assert_vectors_close, attend64, build_paged, decode64, gather_seq,  # noqa: F401
                                     randn, vector_ratio)

LOG2E = 1.4426950408889634
SCALE_LOG2 = float(torch.tensor(SCALE * LOG2E, dtype=torch.float32))     # the kernels' fp32 scale * log2(e)
CHUNK, MIN_CHUNKS = 16, 8               # decode_common.cuh: tokens per chunk, smallest range handed to one warp
H100_SMS = 132
BETA = 8.0                              # |q| of every query head (a power of two: q * k is exact for one-hot q)
BG = 0.125                              # background key scale
A = 16.0                                # a needle's V value
TRAP_DIM = 7                            # V dimension of the trap rows; needles use dimensions 8..127
FP8_SCALES = (0.5, 0.1875)              # k_scale, v_scale of the fp8 cases: needles and traps stay below 448
# Prefill's bar for needle vectors.  A needle owns one output dimension, so that value is a single term P * A / l.  The
# kernels round P to bf16 against their lazily updated reference maximum, prefill64 rounds exp(s - max) against the true
# maximum: two independent roundings, each up to half an ulp of P, i.e. 2^-8 relative at the bottom of a binade.  They
# differ by up to 2^-7 * |o| <= 2 ulps (2 * 2^-8) of the vector's maximum, on top of the suite's 2 ulps.  With random
# V these errors average out over many keys; a one-hot V row shows them whole.  Decode needs no such term: decode64 does
# not round P, and the MMA kernel's single bf16 rounding of P (2^-8) plus that of the output (2^-8) stay within 2 ulps.
PREFILL_ULPS = 4.0


# ---------------------------------------------------------------------------------------------------------------------
# the stream-K decode partition, restated (decode_attn.cu / decode_mma.cu)
# ---------------------------------------------------------------------------------------------------------------------
def decode_warps(kernel_name):
    """Warps per CTA of a decode kernel, from its name: paged_decode_kernel<G, NW, NS, F>, the bf16 tensor-core kernel
    (MMA_WARPS = 8) or its fp8 variant (F8_WARPS = 12)."""
    if "mma_fp8" in kernel_name:
        return 12
    if "mma" in kernel_name:
        return 8
    return int(kernel_name.split("<")[1].split(",")[1])


def decode_partition(lens, hkv, nwarps, sm_count):
    """C = hkv * sum(ceil(ctx / 16)) chunks in (sequence, kv head, chunk) order; TWe = min(ceil(C / 8), sm_count * NWARPS)
    workers; worker gw takes chunks [gw * C / TWe, (gw + 1) * C / TWe)."""
    n = [(max(c, 0) + CHUNK - 1) // CHUNK for c in lens]
    cum = [0]
    for x in n:
        cum.append(cum[-1] + x)
    C = hkv * cum[-1]
    TWe = min(-(-C // MIN_CHUNKS), sm_count * nwarps)
    return SimpleNamespace(C=C, TWe=TWe, cum=cum, n=n, hkv=hkv, lens=list(lens))


def pair_segments(part, b, h):
    """Token ranges [start, end) of the segments the pair (sequence b, kv head h) is cut into, one per worker."""
    C, T, L = part.C, part.TWe, part.lens[b]
    c0 = part.hkv * part.cum[b] + h * part.n[b]
    c1 = c0 + part.n[b]
    if c1 == c0:
        return []
    gw = c0 * T // C
    while (gw + 1) * C // T <= c0:
        gw += 1
    while gw * C // T > c0:
        gw -= 1
    segs = []
    while gw < T and gw * C // T < c1:
        s, e = max(gw * C // T, c0), min((gw + 1) * C // T, c1)
        if e > s:
            segs.append(((s - c0) * CHUNK, min((e - c0) * CHUNK, L)))
        gw += 1
    # the kernel's own count of the pair's segments (the merge waits for exactly this many)
    nseg = ((c1 * T - 1) // C) - (((c0 + 1) * T - 1) // C) + 1
    assert nseg == len(segs), (nseg, segs)
    return segs


def check_splits(case):
    """The pairs a case targets really are split into 3 or more segments by the kernel it runs on."""
    assert case.splits, "the case targets no split pair"
    for b, h, nseg in case.splits:
        assert nseg >= 3, f"sequence {b} kv head {h} ({case.lens[b]} tokens) is cut into {nseg} segments only"


# ---------------------------------------------------------------------------------------------------------------------
# cache rows
# ---------------------------------------------------------------------------------------------------------------------
def _slots(c, b, pos):
    pos = torch.as_tensor(pos, dtype=torch.long, device=c.tables.device)
    return c.tables[b].long()[pos // c.bs], pos % c.bs


def read_k(c, b, pos, h):
    pages, sl = _slots(c, b, pos)
    return c.K[pages, sl, h]


def write_rows(c, b, pos, h, k=None, v=None):
    """Cache rows of sequence b at positions pos, kv head h, in the logical view and the physical cache alike."""
    pages, sl = _slots(c, b, pos)
    if k is not None:
        k = k.to(torch.bfloat16).to(c.K.device)
        c.K[pages, sl, h] = k
        c.kv[0, -1, pages, h, sl] = k
    if v is not None:
        v = v.to(torch.bfloat16).to(c.K.device)
        c.V[pages, sl, h] = v
        c.kv[1, -1, pages, h, sl] = v


def one_hot_v(dim, device):
    v = torch.zeros(D, dtype=torch.float64, device=device)
    v[dim] = A
    return v


def paged_cache(lens, bs, hkv, seed, device):
    """build_paged with the background keys scaled by BG (exact in bf16; NaN rows stay NaN)."""
    c = build_paged(lens, bs, hkv, seed, device=device)
    c.kv[0].mul_(BG)
    c.K.mul_(BG)
    return c


# ---------------------------------------------------------------------------------------------------------------------
# decode cases
# ---------------------------------------------------------------------------------------------------------------------
DECODE_CASES = ("segments", "positions16", "positions256", "merge")


def _boundary_needles(segs, g, L):
    """Keys either side of some segment boundaries of a pair (different ones for each head g), and the pair's first and
    last key for head 0."""
    nseg = len(segs)
    out = set()
    if nseg >= 2:
        for k in {1 + g, nseg // 2 + g, nseg - 1 - g}:
            if 1 <= k < nseg:
                t = segs[k][0]
                out |= {t - 1, t}
    if g == 0:
        out |= {0, L - 1}
    return out


def _position_needles(L, bs):
    cand = {0, L - 1, bs - 1, bs, 2 * bs - 1, 2 * bs, 15, 16, 31, 32, 16 * (L // 32) - 1, 16 * (L // 32)}
    return sorted(p for p in cand if 0 <= p < L)


def decode_case(name, G, device="cuda", nwarps=8, sm_count=H100_SMS, fp8=False, seed=1):
    """A paged-decode launch with needles.  Returns q [B, G * hkv, D] and the cache (kv: physical, K / V: the logical
    view the reference reads), the checked rows, the needles {(b, h, g): [positions]} and the split pairs."""
    hkv = 2
    if name == "segments":
        lens, bs = [40960, 3, 16, 40951, 17, 12288, 1, 257, 0, 40960, 700], 256
    elif name in ("positions16", "positions256"):
        lens, bs = [1, 2, 15, 16, 17, 31, 32, 33, 255, 256, 257, 1000, 4097, 0, 511], int(name[9:])
    elif name == "merge":
        lens, bs = [40960, 40960, 40960, 5, 40944], 256
    else:
        raise ValueError(name)
    c = paged_cache(lens, bs, hkv, seed, device)
    part = decode_partition(lens, hkv, nwarps, sm_count)
    needles, bases, splits = {}, {}, []
    for b, L in enumerate(lens):
        if L == 0:
            continue
        for h in range(hkv):
            segs = pair_segments(part, b, h)
            if name == "segments":
                if L >= 4096:
                    splits.append((b, h, len(segs)))
                taken = set()
                for g in range(G):
                    ps = sorted(_boundary_needles(segs, g, L) - taken)
                    taken |= set(ps)
                    needles[(b, h, g)] = ps
            elif name.startswith("positions"):
                if L >= 4096:
                    splits.append((b, h, len(segs)))
                ps = _position_needles(L, bs)
                for g in range(G):
                    needles[(b, h, g)] = ps[(h * G + g)::hkv * G]
            else:
                if L < 4096:
                    needles[(b, h, 0)] = [0, L - 1]
                    continue
                splits.append((b, h, len(segs)))
                mid = lambda k, g: (segs[k][0] + segs[k][1]) // 2 + g
                base = [0.0] * G
                for g in range(G):
                    pattern = ((b * hkv + h) * G + g) % 6
                    n = len(segs)
                    if pattern == 0:                          # the maximum in the first segment
                        ps = [mid(0, g)]
                    elif pattern == 1:                        # in a middle segment
                        ps = [mid(n // 2, g)]
                    elif pattern == 2:                        # in the last segment
                        ps = [mid(n - 1, g)]
                    elif pattern == 3:                        # two segments tie for it
                        ps = [mid(1, g), mid(n - 2, g)]
                    elif pattern == 4:                        # every score about -100 nats
                        ps, base[g] = [mid(n // 2 - 1, g)], -100.0
                    else:                                     # every score about +100 nats
                        ps, base[g] = [mid(n // 2 + 1, g)], 100.0
                    needles[(b, h, g)] = ps
                bases[(b, h)] = base
    q = torch.zeros(len(lens), G * hkv, D, dtype=torch.float64, device=device)
    for h in range(hkv):
        for g in range(G):
            q[:, h * G + g, g] = BETA
    q = q.to(torch.bfloat16)
    kdir = lambda g: torch.eye(D, dtype=torch.float64, device=device)[g] / (BETA * SCALE)    # score 1 nat for head g
    _place(c, lens, hkv, G, needles, bases, kdir, device)
    case = SimpleNamespace(kind="decode", name=name, lens=lens, bs=bs, hkv=hkv, G=G, q=q, c=c, kv=c.kv, K=c.K, V=c.V,
                           tables=c.tables, needles=needles, splits=splits, part=part,
                           rows=[b for b, L in enumerate(lens) if L > 0], scales={})
    if fp8:
        ks, vs = FP8_SCALES
        case.kv = torch.stack([quantize_e4m3(c.kv[0], ks), quantize_e4m3(c.kv[1], vs)]).contiguous()
        case.K = dequantize_e4m3(case.kv[0, -1], ks).permute(0, 2, 1, 3)
        case.V = dequantize_e4m3(case.kv[1, -1], vs).permute(0, 2, 1, 3)
        case.scales = dict(k_scale=ks, v_scale=vs)
    case.ctx = torch.tensor(lens, dtype=torch.int32, device=device)
    return case


def _place(c, lens, hkv, G, needles, bases, kdir, device):
    """Write bases, needles and traps into the cache.  kdir(g) is the key direction that scores 1 nat for head g; a
    needle's key is its pair's base plus ln(L / m) along its head's direction."""
    for b, L in enumerate(lens):
        if L == 0:
            continue
        for h in range(hkv):
            base = bases.get((b, h), [0.0] * G)
            base_k = sum(base[g] * kdir(g) for g in range(G))
            if any(base):
                pos = torch.arange(L)
                write_rows(c, b, pos, h, k=read_k(c, b, pos, h).double() + base_k)
            ps_all = [p for g in range(G) for p in needles.get((b, h, g), [])]
            assert len(ps_all) == len(set(ps_all)), f"two heads share a needle key in sequence {b}"
            dim = 8
            for g in range(G):
                ps = needles.get((b, h, g), [])
                s = math.log(max(L, 2) / max(len(ps), 1))
                for p in ps:
                    write_rows(c, b, [p], h, k=(base_k + s * kdir(g))[None], v=one_hot_v(dim, device)[None])
                    dim = 8 + (dim - 7) % 120
            if L % c.bs:                                      # the stale row right past the end: a trap
                trap = base_k + (math.log(L) + 2) * sum(kdir(g) for g in range(G))
                write_rows(c, b, [L], h, k=trap[None], v=one_hot_v(TRAP_DIM, device)[None])


def decode_reference(case):
    """float64 decode of the checked rows."""
    r = case.rows
    return decode64(case.q[r], case.K, case.V, [case.lens[i] for i in r], case.tables[r])


# ---------------------------------------------------------------------------------------------------------------------
# fused decode cases: q/k-norm + RoPE + append happen in the kernel; the needle sits on the newest token
# ---------------------------------------------------------------------------------------------------------------------
FUSED_CASES = ("positions", "segments")
NEWEST_LOGIT = math.log(1000.0)


def fused_case(name, G, device="cuda", nwarps=8, sm_count=H100_SMS, seed=3):
    from oracle.qwen3_ref import rope_table
    from test_gpu_dispatch_edges import qknorm_rope64
    hkv = 2
    hq = G * hkv
    if name == "positions":
        lens, bs = [1, 2, 16, 17, 18, 33, 64, 65, 200, 257, 1000, 0], 16
    elif name == "segments":
        lens, bs = [40960, 18, 12289, 0, 1000, 40945], 256
    else:
        raise ValueError(name)
    B = len(lens)
    c = paged_cache(lens, bs, hkv, seed, device)
    part = decode_partition(lens, hkv, nwarps, sm_count)
    # raw projection rows: q heads one-hot; the step's k one-hot along the head it targets; v one-hot in dimension 8
    qkv = torch.zeros(B, (hq + 2 * hkv) * D, dtype=torch.float64, device=device)
    qraw = qkv[:, :hq * D].view(B, hq, D)
    kraw = qkv[:, hq * D:(hq + hkv) * D].view(B, hkv, D)
    vraw = qkv[:, (hq + hkv) * D:].view(B, hkv, D)
    for h in range(hkv):
        for g in range(G):
            qraw[:, h * G + g, g] = 1.0
        for b in range(B):
            kraw[b, h, (b + h) % G] = 1.0
        vraw[:, h, 8] = A
    qkv = qkv.to(torch.bfloat16)
    # RMSNorm of a one-hot row is sqrt(D) on its dimension: the newest token scores D * qw * kw * scale for its head
    qw = torch.ones(D, dtype=torch.float64, device=device)
    kw = torch.ones(D, dtype=torch.float64, device=device)
    kw[:G] = NEWEST_LOGIT / (D * SCALE)
    qw, kw = qw.to(torch.bfloat16), kw.to(torch.bfloat16)
    table = rope_table(D, 40960, 1e6).to(device)
    ctx = torch.tensor(lens, dtype=torch.int32, device=device)
    pos = (ctx.long() - 1).clamp(min=0)
    q_o = qknorm_rope64(qkv[:, :hq * D].view(B, hq, D), qw, pos, table).to(torch.bfloat16)
    needles, splits = {}, []
    for b, L in enumerate(lens):
        if L == 0:
            continue
        for h in range(hkv):
            if name == "segments":
                segs = pair_segments(part, b, h)
                if L >= 4096:
                    splits.append((b, h, len(segs)))
                taken = {L - 1}
                for g in range(G):
                    ps = sorted(_boundary_needles(segs, g, L) - taken)
                    taken |= set(ps)
                    needles[(b, h, g)] = ps
            else:
                ps = [p for p in _position_needles(L, bs) if p < L - 1]
                if L >= 2 and L - 2 not in ps:
                    ps.append(L - 2)
                for g in range(G):
                    needles[(b, h, g)] = sorted(ps[(h * G + g)::hkv * G])
    # cached needles point along the rotated query of their head: q_o . k = s / SCALE
    qd = q_o.double()
    for h in range(hkv):
        kdir = lambda g, b, h=h: qd[b, h * G + g] / (qd[b, h * G + g].pow(2).sum() * SCALE)
        _place_fused_head(c, lens, h, G, {(b, g): v for (b, hh, g), v in needles.items() if hh == h}, kdir, device)
    # the reference: the step's K (normed, rotated) and raw V appended at ctx - 1
    k_o = qknorm_rope64(qkv[:, hq * D:(hq + hkv) * D].view(B, hkv, D), kw, pos, table).to(torch.bfloat16)
    K2, V2 = c.K.clone(), c.V.clone()
    live = ctx > 0
    slots = c.tables.long()[torch.arange(B, device=device), pos // bs] * bs + pos % bs
    K2.view(-1, hkv, D)[slots[live]] = k_o[live]
    V2.view(-1, hkv, D)[slots[live]] = qkv[:, (hq + hkv) * D:].view(B, hkv, D)[live]
    for b, L in enumerate(lens):                               # the newest token is a needle of the head it targets
        for h in range(hkv):
            if L:
                needles.setdefault((b, h, (b + h) % G), []).append(L - 1)
    return SimpleNamespace(kind="fused", name=name, lens=lens, bs=bs, hkv=hkv, G=G, qkv=qkv, qw=qw, kw=kw, table=table,
                           q=q_o, c=c, kv=c.kv, K=K2, V=V2, tables=c.tables, ctx=ctx, needles=needles, splits=splits,
                           part=part, rows=[b for b, L in enumerate(lens) if L > 0], scales={})


def _place_fused_head(c, lens, h, G, needles, kdir, device):
    """Cached needles and traps of kv head h; needles {(b, g): positions}, all before the newest token (which carries
    its own needle, V dimension 8, in whichever head its raw k targets)."""
    for b, L in enumerate(lens):
        if L == 0:
            continue
        dim = 9
        seen = set()
        for g in range(G):
            ps = needles.get((b, g), [])
            s = NEWEST_LOGIT                                  # level with the newest token's needle
            for p in ps:
                assert p not in seen and p < L - 1
                seen.add(p)
                write_rows(c, b, [p], h, k=(s * kdir(g, b))[None], v=one_hot_v(dim, device)[None])
                dim = 9 + (dim - 8) % 119
        if L % c.bs:
            trap = (max(math.log(L), NEWEST_LOGIT) + 2) * sum(kdir(g, b) for g in range(G))
            write_rows(c, b, [L], h, k=trap[None], v=one_hot_v(TRAP_DIM, device)[None])


# ---------------------------------------------------------------------------------------------------------------------
# prefill cases: packed, paged and chunked over a prefix
# ---------------------------------------------------------------------------------------------------------------------
PREFILL_CASES = ("causal-packed", "causal-paged16", "causal-paged256", "chunk16", "chunk256", "rescale")
DIAG_OFFSETS = (0, 1, 15, 16, 63, 64, 65, 127)                # query offsets inside a 128-query tile
RESCALE_BASE = 3.0                                             # log2 units: the earlier maximum's score


def _cu(lens, device):
    return torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=device)


def prefill_case(name, device="cuda", seed=5):
    """Needles on the causal diagonal of every 128-query tile, or the lazy-rescale pairs; hq 32, hkv 8."""
    hq, hkv = 32, 8
    G = hq // hkv
    bs = None
    if name == "causal-packed":
        lens_q, lens_k = [4096, 129], [4096, 129]
    elif name.startswith("causal-paged"):
        lens_q, lens_k, bs = [4096, 129], [4096, 166], int(name[12:])
    elif name.startswith("chunk"):
        lens_q, lens_k, bs = [512], [4096], int(name[5:])
    elif name == "rescale":
        lens_q, lens_k = [1024], [1024]
    else:
        raise ValueError(name)
    paged = bs is not None
    T, Tk = sum(lens_q), sum(lens_k)
    q = torch.zeros(T, hq, D, dtype=torch.float64, device=device)
    for h in range(hkv):
        for g in range(G):
            q[:, h * G + g, g] = BETA
    q = q.to(torch.bfloat16)
    if paged:
        c = paged_cache(lens_k, bs, hkv, seed, device)
    else:
        k = (randn(Tk, hkv, D, seed=seed, device=device).double() * BG).to(torch.bfloat16)
        v = randn(Tk, hkv, D, seed=seed + 1, device=device)
    unit = torch.eye(D, dtype=torch.float64, device=device)
    needles, rows, gaps = {}, set(), []
    cq, ck = [0] + list(torch.tensor(lens_q).cumsum(0).tolist()), [0] + list(torch.tensor(lens_k).cumsum(0).tolist())
    for s, (lq, lk) in enumerate(zip(lens_q, lens_k)):
        off = lk - lq
        keyval = {}                                           # (h, position) -> (k row, v row)
        for h in range(hkv):
            dim = 8
            for g in range(G):
                ps = []
                if name == "rescale":
                    later, delta = g < 2, (7.9, 8.1)[g % 2]
                    if later:                                 # the earlier maximum in key tile 0, the needle later
                        a, bpos = 2 + g + 4 * h, 64 * (2 + h) + 5 + g
                    else:                                     # both in one tile
                        a = 64 * (9 + h % 6) + 3 + g + 8 * (h // 6)
                        bpos = a + 30
                    ka = round_bf16(RESCALE_BASE / (BETA * SCALE_LOG2))
                    sa = f32_score(ka)
                    kb = round_bf16((sa + delta) / (BETA * SCALE_LOG2))
                    gaps.append((s, h, g, later, delta, f32_score(kb) - sa))
                    for p, kv_ in ((a, ka), (bpos, kb)):
                        keyval[(h, p)] = (kv_ * unit[g], one_hot_v(dim, device))
                        dim += 1
                        ps.append(p)
                    for r in (bpos - off - 1, bpos - off, bpos - off + 1, lq - 1, a - off - 1, a - off, 128 * ((bpos - off) // 128 + 1) + 5):
                        if 0 <= r < lq:
                            rows.add(cq[s] + r)
                else:
                    xs = (DIAG_OFFSETS[(2 * g + h) % 8], DIAG_OFFSETS[(2 * g + h + 1) % 8])
                    for mb in range((lq + 127) // 128):
                        for x in xs:
                            r = 128 * mb + x
                            if r >= lq:
                                continue
                            j = r + off
                            sc = math.log(j + 1)
                            keyval[(h, j)] = (sc / (BETA * SCALE) * unit[g], one_hot_v(dim, device))
                            dim = 8 + (dim - 7) % 120
                            ps.append(j)
                            rows.update(cq[s] + rr for rr in (r - 1, r) if rr >= 0)
                needles[(s, h, g)] = ps
        assert len(keyval) == sum(len(needles[(s, h, g)]) for h in range(hkv) for g in range(G)), "shared needle key"
        for (h, p), (kr, vr) in keyval.items():
            if paged:
                write_rows(c, s, [p], h, k=kr[None], v=vr[None])
            else:
                k[ck[s] + p, h] = kr.to(torch.bfloat16)
                v[ck[s] + p, h] = vr.to(torch.bfloat16)
    case = SimpleNamespace(kind="prefill", name=name, lens_q=lens_q, lens_k=lens_k, bs=bs, hq=hq, hkv=hkv, G=G, q=q,
                           cu_q=_cu(lens_q, device), cu_k=_cu(lens_k, device), needles=needles, rows=sorted(rows),
                           gaps=gaps, paged=paged)
    if paged:
        case.c, case.kv, case.tables = c, c.kv, c.tables
    else:
        case.k, case.v = k, v
    return case


def round_bf16(x):
    return float(torch.tensor(x, dtype=torch.float64).to(torch.bfloat16))


def f32_score(kval):
    """The kernels' score of a one-hot key kval against a one-hot query BETA, in log2 units (fp32 product)."""
    return float(torch.tensor(BETA * kval, dtype=torch.float32) * torch.tensor(SCALE_LOG2, dtype=torch.float32))


def seq_kv(case, s):
    """float keys / values of prefill sequence s."""
    lk = case.lens_k[s]
    if case.paged:
        return gather_seq(case.K_ref, case.tables[s], lk), gather_seq(case.V_ref, case.tables[s], lk)
    k0 = int(case.cu_k[s])
    return case.k[k0:k0 + lk], case.v[k0:k0 + lk]


def prefill_reference(case, K=None, V=None):
    """float64 prefill (attend64: P rounded to bf16) of the checked rows, in the order of case.rows.  K / V: the logical
    cache the reference reads (default: the case's bf16 cache)."""
    if case.paged:
        case.K_ref = case.c.K if K is None else K
        case.V_ref = case.c.V if V is None else V
    out = torch.empty(len(case.rows), case.hq, D, dtype=torch.float64, device=case.q.device)
    cq = case.cu_q.tolist()
    at = 0
    for s in range(len(case.lens_q)):
        rs = [r - cq[s] for r in case.rows if cq[s] <= r < cq[s + 1]]
        ks, vs = seq_kv(case, s)
        off = case.lens_k[s] - case.lens_q[s]
        i = 0
        while i < len(rs):                                    # runs of consecutive rows: one attend64 call each
            j = i
            while j + 1 < len(rs) and rs[j + 1] == rs[j] + 1:
                j += 1
            a, b = rs[i], rs[j] + 1
            out[at:at + b - a] = attend64(case.q[cq[s] + a:cq[s] + b], ks[:b + off], vs[:b + off])
            at += b - a
            i = j + 1
    return out


# ---------------------------------------------------------------------------------------------------------------------
# designed defects, in float64: how far each one moves the checked vectors (tests/test_attention_needles_host.py)
# ---------------------------------------------------------------------------------------------------------------------
def edited_softmax(q, k, v, n, edits, ulps=2.0):
    """One query row q [Hq, D] over keys 0..n-1 of k, v [>= n, Hkv, D], unrounded float64.  Returns the clean output
    [Hq, D] and, for each edit, the defective output and its vector_ratio against the clean one (max over heads).
    Edits: ("drop", j) leaves key j out; ("swap", j, j2) reads key j2 in place of key j; ("admit", e) adds key e."""
    hq, hkv = q.shape[0], k.shape[1]
    G = hq // hkv
    kd, vd = k.double(), v.double()
    s = torch.einsum("kgd,lkd->kgl", q.double().view(hkv, G, D), kd) * SCALE
    m = s[..., :n].amax(-1, keepdim=True)
    p = torch.exp(s - m)
    N = torch.einsum("kgl,lkd->kgd", p[..., :n], vd[:n])
    l = p[..., :n].sum(-1, keepdim=True)
    clean = (N / l).reshape(hq, D)
    term = lambda j: (p[..., j, None] * vd[j][:, None, :], p[..., j, None])
    out = []
    for e in edits:
        if e[0] == "drop":
            (pv, pj) = term(e[1])
            bad = (N - pv) / (l - pj)
        elif e[0] == "swap":
            (pv, pj), (pv2, pj2) = term(e[1]), term(e[2])
            bad = (N - pv + pv2) / (l - pj + pj2)
        else:
            (pv, pj) = term(e[1])
            bad = (N + pv) / (l + pj)
        out.append((e, vector_ratio(bad.reshape(hq, D), clean, ulps).max().item()))
    return clean, out


def _neighbour(j, n):
    return j - 1 if j >= 1 else (j + 1 if j + 1 < n else None)


def decode_defects(case):
    """Per checked row: (row, clean output [Hq, D], [(edit, ratio)]) for every needle dropped or read as its neighbour,
    and for the key past the end admitted."""
    w = case.tables.shape[1]
    for b in case.rows:
        L = case.lens[b]
        n_have = min(L + 1, w * case.bs)
        k = gather_seq(case.K, case.tables[b], n_have).double()
        v = gather_seq(case.V, case.tables[b], n_have).double()
        if n_have == L:                                       # the key past the end lies past the table's view: NaN pages
            nan = torch.full((1,) + tuple(k.shape[1:]), math.nan, dtype=torch.float64, device=k.device)
            k, v = torch.cat([k, nan]), torch.cat([v, nan])
        edits = [("admit", L)]
        for (bb, h, g), ps in case.needles.items():
            if bb != b:
                continue
            for j in ps:
                edits.append(("drop", j))
                nb = _neighbour(j, L)
                if nb is not None:
                    edits.append(("swap", j, nb))
        clean, res = edited_softmax(case.q[b], k, v, L, edits)
        yield b, clean, res


def prefill_defects(case):
    """Per needle key j of sequence s: query j - off must see it (dropped, read as its neighbour), query j - off - 1 must
    not (admitted).  Yields (global row, clean output, [(edit, ratio against the PREFILL_ULPS bar)])."""
    if case.paged:
        case.K_ref, case.V_ref = case.c.K, case.c.V
    cq = case.cu_q.tolist()
    for s in range(len(case.lens_q)):
        lq, lk = case.lens_q[s], case.lens_k[s]
        off = lk - lq
        ks, vs = seq_kv(case, s)
        per_row = {}
        for (ss, h, g), ps in case.needles.items():
            if ss != s:
                continue
            for j in ps:
                r0 = j - off
                if 0 <= r0 < lq:
                    per_row.setdefault(r0, []).append(("drop", j))
                    nb = _neighbour(j, r0 + off + 1)
                    if nb is not None:
                        per_row[r0].append(("swap", j, nb))
                if 1 <= r0 <= lq:
                    per_row.setdefault(r0 - 1, []).append(("admit", j))
        for r, edits in sorted(per_row.items()):
            n = r + off + 1
            clean, res = edited_softmax(case.q[cq[s] + r], ks[:n + 1], vs[:n + 1], n, edits, PREFILL_ULPS)
            yield cq[s] + r, clean, res
