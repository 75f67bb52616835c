"""Exactly representable operands for the wgmma GEMMs (csrc/linear_tc.cu), their float64 reference, and the table of
GEMM launches the Qwen3 model makes.

Small integer operands with power-of-two block scales make every product exact and every partial sum an integer
multiple of the smallest scale product, far below 2^24.  A correct kernel then has exactly one answer whatever its
tiling, split, ring depth, cluster or PDL setting, and it equals float64 bit for bit; a dropped, repeated or misplaced
k tile, a wrong row, a wrong block scale or a wrong split range leaves a non-zero difference.  The block scales are
drawn so that no two neighbours share one (neighbouring k blocks, n blocks and rows, and the gate / up rows of the same
SiluAndMul column), so taking a neighbour's scale always changes the result.

This complements the float64-bar tests on Gaussian data (test_gpu_linear*.py), which measure precision; exact data
cannot.  Needs torch only: the CPU test (test_gemm_exact_host.py) and the GPU test (test_gpu_gemm_exact.py) share it.
"""
from __future__ import annotations

import zlib
from typing import NamedTuple

import torch

BLOCK = 128                     # FP8 scale block (both dims) and one FP8 k slot of the kernel
LK = 64                         # bf16 k tile of the kernel
HEAD_DIM = 128
EPI_BF16, EPI_SILU, EPI_PARTIAL = 0, 1, 2
EPI_NAMES = {EPI_BF16: "bf16", EPI_SILU: "silu", EPI_PARTIAL: "partial"}

# operand ranges; exactness_ratio() checks what they imply at every shape used
BF16_INT = 4                    # bf16 x and w entries in {-4 .. 4}
LM_HEAD_SCALE = 2.0 ** -6       # the LM head's entries are {-4 .. 4} * 2^-6: logits are multiples of 2^-6
FP8_INT = 2                     # e4m3 entries in {-2 .. 2}
X_EXPONENTS = (-1, 0, 1)        # x_scale[m, kb] = 2^e: left and upper neighbour excluded, 3 values suffice
W_EXPONENTS = (-1, 0, 1, 2)     # w_scale[nb, kb] = 2^e: left, upper and the gate partner of an up row, so 4 values

# Qwen3 dense models: (hidden, intermediate, q heads, kv heads), head_dim 128
QWEN3 = {
    "0.6b": (1024, 3072, 16, 8),
    "1.7b": (2048, 6144, 16, 8),
    "4b": (2560, 9728, 32, 8),
    "8b": (4096, 12288, 32, 8),
    "14b": (5120, 17408, 40, 8),
    "32b": (5120, 25600, 64, 8),
}
TP_SIZES = (1, 2, 4, 8)
DECODE_ROWS = (1, 64, 65, 128, 129, 256)
PREFILL_ROWS = 2048 + 37


class Launch(NamedTuple):
    """One GEMM launch: w is [n, k] (n = 2 * columns out for EPI_SILU), ``splits`` k ranges (fp32 partials)."""
    fp8: bool
    n: int
    k: int
    epi: int
    block_n: int
    splits: int

    def name(self) -> str:
        return f"{'fp8' if self.fp8 else 'bf16'}-{EPI_NAMES[self.epi]}-n{self.n}-k{self.k}-bn{self.block_n}-s{self.splits}"


def case_seed(*parts) -> int:
    return zlib.crc32(repr(parts).encode())


# ---- what the model launches ---------------------------------------------------------------------------------------------
def tp_ok(model: str, tp: int, fp8: bool) -> bool:
    """The model shards heads, kv heads and the MLP evenly; block-FP8 also needs whole 128-blocks per rank
    (utils/fp8.py:check_shapes)."""
    hidden, inter, hq, hkv = QWEN3[model]
    if hq % tp or hkv % tp or inter % tp:
        return False
    return not fp8 or all(v % BLOCK == 0 for v in (hq * HEAD_DIM // tp, hkv * HEAD_DIM // tp, hidden, inter // tp))


def projections(model: str, tp: int) -> dict:
    """(n, k) of the four projections of one tensor-parallel rank; gate_up is [2 * inter, hidden]."""
    hidden, inter, hq, hkv = QWEN3[model]
    q, kv, i = hq * HEAD_DIM // tp, hkv * HEAD_DIM // tp, inter // tp
    return dict(qkv=(q + 2 * kv, hidden), o=(hidden, q), gate_up=(2 * i, hidden), down=(hidden, i))


def largest_divisor(total: int, cap: int) -> int:
    """The largest d <= cap that divides total: the split-K count of a k extent of ``total`` tiles / blocks."""
    return next(d for d in range(max(1, min(cap, total)), 0, -1) if total % d == 0)


def model_launches(model: str, tp: int, fp8: bool, rows: int, prefill: bool = False) -> list[tuple[str, Launch]]:
    """The wgmma GEMMs one layer of ``model`` runs on a step of ``rows`` tokens, restated from models/qwen3.py:
      bf16 (B200_LINEAR=auto up to 128 rows, B200_LINEAR=rows up to 256; qkv / gate_up stay cuBLAS): o / down as fp32
        split-K partials at block_n 64 with up to 8 splits, up to 4 above 128 rows; under tensor parallelism EPI_BF16
        at block_n 32 into the peer buffer.  Prefill runs no wgmma GEMM.
      FP8 (every projection, decode and prefill): qkv EPI_BF16 and gate_up EPI_SILU at block_n 64; o / down as split-K
        partials (up to 8 splits over the 128-wide k blocks) on one GPU up to 128 rows, EPI_BF16 at block_n 32 into the
        peer buffer for decode steps under tensor parallelism, EPI_BF16 at block_n 64 otherwise."""
    p = projections(model, tp)
    out = []
    if not fp8:
        if prefill or rows > 256:
            return out
        for name in ("o", "down"):
            n, k = p[name]
            if tp == 1:
                out.append((name, Launch(False, n, k, EPI_PARTIAL, 64, largest_divisor(k // LK, 8 if rows <= 128 else 4))))
            else:
                out.append((name, Launch(False, n, k, EPI_BF16, 32, 1)))
        return out
    out.append(("qkv", Launch(True, *p["qkv"], EPI_BF16, 64, 1)))
    out.append(("gate_up", Launch(True, *p["gate_up"], EPI_SILU, 64, 1)))
    for name in ("o", "down"):
        n, k = p[name]
        if tp == 1 and rows <= 128 and not prefill:
            out.append((name, Launch(True, n, k, EPI_PARTIAL, 64, largest_divisor(k // BLOCK, 8))))
        elif tp > 1 and not prefill:
            out.append((name, Launch(True, n, k, EPI_BF16, 32, 1)))
        else:
            out.append((name, Launch(True, n, k, EPI_BF16, 64, 1)))
    return out


def launch_table() -> dict[tuple[Launch, int], list[str]]:
    """Every distinct (launch, rows) over the six models, TP 1/2/4/8, bf16 and FP8, the decode rows and one prefill
    (FP8 only: bf16 prefill is cuBLAS) -> where it comes from."""
    table: dict[tuple[Launch, int], list[str]] = {}
    for model in QWEN3:
        for fp8 in (False, True):
            for tp in TP_SIZES:
                if not tp_ok(model, tp, fp8):
                    continue
                steps = [(r, False) for r in DECODE_ROWS] + ([(PREFILL_ROWS, True)] if fp8 else [])
                for rows, prefill in steps:
                    for proj, launch in model_launches(model, tp, fp8, rows, prefill):
                        table.setdefault((launch, rows), []).append(f"{model}.tp{tp}.{proj}")
    return table


# ---- pipeline sweep on small synthetic shapes ----------------------------------------------------------------------------
# k tiles (bf16, 64 wide) / k blocks (FP8, 128 wide) per split: below, at and above the FP8 scale prefetch distance (4)
# and the ring depths (4 / 6 / 8 slots), 1 mod 4, and the 25 of Qwen3-32B's down_proj
SWEEP_NK = (1, 2, 3, 4, 5, 6, 7, 8, 9, 13, 25)
SWEEP_SPLITS = (1, 2, 8)
SWEEP_ROWS = 130                # one CTA with both m64 halves, one with a single ragged half
SWEEP_N = 256                   # output columns (two FP8 n blocks; gate_up has 2 x 256 weight rows)


def sweep_launches(fp8: bool, nk: int, splits: int) -> list[tuple[Launch, dict]]:
    """Every epilogue the split count allows, at every block_n, and at block_n 64 every ring / cluster / PDL variant."""
    k = nk * splits * (BLOCK if fp8 else LK)
    out = []
    for epi in ((EPI_PARTIAL,) if splits > 1 else (EPI_BF16, EPI_SILU, EPI_PARTIAL)):
        n = 2 * SWEEP_N if epi == EPI_SILU else SWEEP_N
        bns = (16, 32, 64) + (() if fp8 else (128,))
        for bn in bns:
            if epi == EPI_SILU and bn == 16:
                continue
            out.append((Launch(fp8, n, k, epi, bn, splits), {}))
        for kw in (dict(stages=2), dict(stages=3), dict(shallow=True), dict(cluster=2), dict(cluster=4), dict(pdl=True)):
            out.append((Launch(fp8, n, k, epi, 64, splits), kw))
    return out


# ---- operands ------------------------------------------------------------------------------------------------------------
def distinct_exponents(rows: int, cols: int, values, gen: torch.Generator, pair_offset: int | None = None) -> torch.Tensor:
    """int64 [rows, cols] drawn from ``values``; every entry differs from its left and upper neighbour and, for rows
    r >= pair_offset, from entry [r - pair_offset] (the gate block of an up block).  Filled one anti-diagonal at a time
    (both neighbours lie on the previous one), each entry uniform over the values its neighbours leave."""
    v = torch.tensor(values, dtype=torch.int64)
    e = torch.zeros(rows, cols, dtype=torch.int64)
    for d in range(rows + cols - 1):
        r = torch.arange(max(0, d - cols + 1), min(rows, d + 1))
        c = d - r
        allowed = torch.ones(len(r), len(v), dtype=torch.bool)
        allowed &= ~((c > 0)[:, None] & (e[r, (c - 1).clamp(min=0)][:, None] == v))
        allowed &= ~((r > 0)[:, None] & (e[(r - 1).clamp(min=0), c][:, None] == v))
        if pair_offset is not None:
            allowed &= ~((r >= pair_offset)[:, None] & (e[(r - pair_offset).clamp(min=0), c][:, None] == v))
        pick = ((torch.rand(len(r), len(v), generator=gen) + 1.0) * allowed).argmax(1)
        e[r, c] = v[pick]
    return e


def fp8_scales(rows: int, n: int, k: int, epi: int, seed: int) -> tuple[torch.Tensor, torch.Tensor]:
    """(x_scale [rows, k/128], w_scale [n/128, k/128]) fp32 powers of two, neighbour-distinct (CPU)."""
    gen = torch.Generator().manual_seed(seed)
    kb = k // BLOCK
    xs = torch.pow(2.0, distinct_exponents(rows, kb, X_EXPONENTS, gen).double()).float()
    pair = n // BLOCK // 2 if epi == EPI_SILU else None
    ws = torch.pow(2.0, distinct_exponents(n // BLOCK, kb, W_EXPONENTS, gen, pair).double()).float()
    return xs, ws


def _ints(shape, bound: int, seed: int, device) -> torch.Tensor:
    gen = torch.Generator(device=device).manual_seed(seed)
    return torch.randint(-bound, bound + 1, shape, generator=gen, device=device, dtype=torch.int8)


def bf16_operands(rows: int, n: int, k: int, seed: int, device="cuda", x_pad: int = 0):
    """x [rows, k] (a view with row stride k + x_pad) and w [n, k], bf16 integers in {-4 .. 4}."""
    xb = _ints((rows, k + x_pad), BF16_INT, seed, device).to(torch.bfloat16)
    return xb[:, :k], _ints((n, k), BF16_INT, seed + 1, device).to(torch.bfloat16)


def fp8_operands(rows: int, n: int, k: int, epi: int, seed: int, device="cuda", x_pad: int = 0, xs_pad: int = 0):
    """(xq, x_scale, w, w_scale): e4m3 integers in {-2 .. 2}, power-of-two block scales (fp8_scales).  ``x_pad`` /
    ``xs_pad``: xq / x_scale are views into wider buffers (x_scale a column slice starting at column 1)."""
    xq = _ints((rows, k + x_pad), FP8_INT, seed, device).to(torch.float8_e4m3fn)[:, :k]
    w = _ints((n, k), FP8_INT, seed + 1, device).to(torch.float8_e4m3fn)
    xs, ws = fp8_scales(rows, n, k, epi, seed + 2)
    if xs_pad:
        wide = torch.full((rows, k // BLOCK + xs_pad), float("nan"))
        wide[:, 1:1 + k // BLOCK] = xs
        xs = wide.to(device)[:, 1:1 + k // BLOCK]
    else:
        xs = xs.to(device)
    return xq, xs, w, ws.to(device)


def exactness_ratio(launch: Launch) -> float:
    """Worst-case |partial sum| over its granularity (the smallest product of scales), from the operand ranges alone;
    every fp32 sum the kernel forms is exact while this stays below 2^24."""
    if launch.fp8:
        kb = launch.k // BLOCK
        smax = 2.0 ** (max(X_EXPONENTS) + max(W_EXPONENTS))
        smin = 2.0 ** (min(X_EXPONENTS) + min(W_EXPONENTS))
        return kb * fp8_block_bound() * smax / smin
    return launch.k * BF16_INT * BF16_INT


def fp8_block_bound() -> int:
    """Worst-case |sum| of one 128-wide k block of e4m3 integer products (unit granularity): the fp8 wgmma chain, which
    accumulates with reduced precision, stays exact while this needs few bits."""
    return BLOCK * FP8_INT * FP8_INT


# ---- float64 reference ---------------------------------------------------------------------------------------------------
def _dequant(q: torch.Tensor, s: torch.Tensor | None, row_block: int) -> torch.Tensor:
    v = q.double()
    if s is None:
        return v
    s = s.double().repeat_interleave(BLOCK, 1)
    if row_block > 1:
        s = s.repeat_interleave(row_block, 0)
    return v * s


def reference(x, w, splits: int = 1, x_scale=None, w_scale=None, chunk_bytes: int = 1 << 27):
    """y = dequant(x) @ dequant(w)^T in float64 on x's device, chunked over the n rows of w, and each split's partial over
    exactly the k range that split owns.  Returns (full, partials [splits, rows, n]) as fp32, after checking that fp32
    holds every value exactly (so comparing a kernel's fp32 / bf16 output with them is comparing with float64)."""
    rows, k = x.shape
    n = w.shape[0]
    xd = _dequant(x, x_scale, 1)
    ks = k // splits
    full = torch.empty(rows, n, dtype=torch.float32, device=x.device)
    parts = torch.empty(splits, rows, n, dtype=torch.float32, device=x.device) if splits > 1 else None
    step = max(BLOCK, (chunk_bytes // (8 * max(k, rows))) // BLOCK * BLOCK)
    for n0 in range(0, n, step):
        n1 = min(n, n0 + step)
        wd = _dequant(w[n0:n1], w_scale[n0 // BLOCK:(n1 + BLOCK - 1) // BLOCK] if w_scale is not None else None, BLOCK)
        acc = torch.zeros(rows, n1 - n0, dtype=torch.float64, device=x.device)
        for s in range(splits):
            ys = xd[:, s * ks:(s + 1) * ks] @ wd[:, s * ks:(s + 1) * ks].t()
            acc += ys
            if parts is not None:
                p32 = ys.float()
                assert torch.equal(p32.double(), ys), "a split partial is not exact in fp32"
                parts[s, :, n0:n1] = p32
        f32 = acc.float()
        assert torch.equal(f32.double(), acc), "the product is not exact in fp32"
        full[:, n0:n1] = f32
    return full, parts


def silu_mul_reference(full: torch.Tensor) -> torch.Tensor:
    """float64 silu(bf16 g) * bf16 u of the exact [gate | up] product (the kernel rounds both to bf16 first, as the
    reference's F.linear output is bf16)."""
    half = full.shape[1] // 2
    g = full[:, :half].to(torch.bfloat16).double()
    u = full[:, half:].to(torch.bfloat16).double()
    return g * torch.sigmoid(g) * u


def bf16_ulp(v: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 at |v| (8 significant bits), for float64 v != 0."""
    _, e = torch.frexp(v)
    return torch.ldexp(torch.ones_like(v), (e - 8).to(torch.int32))


def describe_mismatch(bad: torch.Tensor, got: torch.Tensor, want: torch.Tensor, limit: int = 6) -> str:
    """Count of the flagged elements, the rows / columns they sit in, and the first few values."""
    idx = bad.nonzero()
    if idx.numel() == 0:
        return "0 elements differ"
    rows = torch.unique(idx[:, -2]).tolist()
    cols = torch.unique(idx[:, -1]).tolist()
    first = ", ".join(f"{tuple(i.tolist())}: got {got[tuple(i)].item()!r} want {want[tuple(i)].item()!r}" for i in idx[:limit])
    return (f"{idx.shape[0]} of {bad.numel()} elements differ; rows {rows[:8]}{'...' if len(rows) > 8 else ''} "
            f"({len(rows)}), columns {cols[:8]}{'...' if len(cols) > 8 else ''} ({len(cols)}); {first}")
