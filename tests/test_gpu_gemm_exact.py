"""The bf16 and block-FP8 wgmma GEMMs (csrc/linear_tc.cu) bit for bit against float64, on exactly representable operands
(tests/gemm_exact.py): small integers, power-of-two block scales with no two neighbours alike.  A correct kernel has
exactly one answer on such data, whatever its tiling, split, ring depth, cluster or PDL setting, so every check here is
an equality (EPI_SILU: one bf16 ulp, for expf and the division):

* every launch the Qwen3 models make (six dims sets, TP 1/2/4/8) at decode rows 1 .. 256 and one FP8 prefill;
* a pipeline sweep over 1 .. 25 k tiles per split, 1 / 2 / 8 splits, every block_n, ring depth, cluster size and PDL;
* strided x, a column-slice x_scale view and a strided bf16 output;
* the split-K add + RMSNorm on exact partials, and the fused LM head + sampling on exact logits with planted ties.

The float64-bar tests on Gaussian data (test_gpu_linear.py, test_gpu_linear_fp8.py) measure precision; these pin the
dataflow: which k blocks, rows, scales and splits go where.
"""
import pytest
import torch

import gemm_exact as ge

pytestmark = pytest.mark.gpu

TABLE = ge.launch_table()
TABLE_CASES = sorted(TABLE, key=lambda c: (c[0].fp8, c[0].n * c[0].k, c[0], c[1]))


def _ops():
    from nanovllm import ops
    return ops


def _operands(launch: ge.Launch, rows: int, seed: int, x_pad: int = 0, xs_pad: int = 0):
    if launch.fp8:
        return ge.fp8_operands(rows, launch.n, launch.k, launch.epi, seed, x_pad=x_pad, xs_pad=xs_pad)
    x, w = ge.bf16_operands(rows, launch.n, launch.k, seed, x_pad=x_pad)
    return x, None, w, None


def _run(launch: ge.Launch, x, xs, w, ws, out=None, **kw):
    ops = _ops()
    if launch.fp8:
        return ops.linear_fp8(x, xs, w, ws, launch.epi, launch.block_n, launch.splits, out=out, **kw)
    return ops.linear(x, w, launch.epi, launch.block_n, launch.splits, out=out, **kw)


def _compare(launch: ge.Launch, got: torch.Tensor, full: torch.Tensor, parts) -> str | None:
    """None when ``got`` is what float64 says, else the count and place of the differing elements."""
    if launch.epi == ge.EPI_PARTIAL:
        want = full[None] if launch.splits == 1 else parts
        bad = got != want
        if not bad.any():
            return None
        splits = torch.unique(bad.nonzero()[:, 0]).tolist()
        per = launch.k // launch.splits // (ge.BLOCK if launch.fp8 else ge.LK)
        return f"splits {splits} (each {per} k {'blocks' if launch.fp8 else 'tiles'}): " + ge.describe_mismatch(bad, got, want)
    if launch.epi == ge.EPI_BF16:
        want = full.to(torch.bfloat16)
        bad = got != want
        return ge.describe_mismatch(bad, got, want) if bad.any() else None
    # EPI_SILU: g and u are exact before the activation; expf, the division and the output rounding are left, so at most
    # one bf16 ulp of the float64 value.  Below 2^-100 (gates under -88, where expf(-g) overflows to inf and the kernel
    # returns 0) nothing is visible at bf16 resolution of any other element.
    want = ge.silu_mul_reference(full)
    bar = torch.where(want.abs() < 2.0 ** -100, torch.full_like(want, 2.0 ** -100), ge.bf16_ulp(want))
    g = got.double()
    bad = ~((g - want).abs() <= bar)
    if bad.any():
        return ge.describe_mismatch(bad, got, want)
    return None


def _not_bit_equal(launch, got, full) -> int:
    if launch.epi == ge.EPI_SILU:
        return int((got != ge.silu_mul_reference(full).to(torch.bfloat16)).sum())
    return 0


NOT_BIT_EQUAL = {}


@pytest.mark.parametrize("launch,rows", TABLE_CASES, ids=[f"{lc.name()}-r{r}" for lc, r in TABLE_CASES])
def test_model_launch_exact(launch, rows):
    x, xs, w, ws = _operands(launch, rows, ge.case_seed(launch, rows))
    got = _run(launch, x, xs, w, ws)
    full, parts = ge.reference(x, w, launch.splits, xs, ws)
    msg = _compare(launch, got, full, parts)
    NOT_BIT_EQUAL[f"{launch.name()}-r{rows}"] = _not_bit_equal(launch, got, full)
    assert msg is None, f"{launch.name()} rows={rows} ({', '.join(TABLE[(launch, rows)][:4])}): {msg}"


@pytest.mark.parametrize("splits", ge.SWEEP_SPLITS)
@pytest.mark.parametrize("nk", ge.SWEEP_NK)
@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
def test_pipeline_sweep_exact(fp8, nk, splits):
    """Every variant of the same launch must equal float64, not merely each other."""
    refs, failures = {}, []
    for launch, kw in ge.sweep_launches(fp8, nk, splits):
        key = (launch.n, launch.epi)
        if key not in refs:
            operands = _operands(launch, ge.SWEEP_ROWS, ge.case_seed("sweep", fp8, nk, splits, *key))
            refs[key] = (operands, ge.reference(operands[0], operands[2], launch.splits, operands[1], operands[3]))
        (x, xs, w, ws), (full, parts) = refs[key]
        got = _run(launch, x, xs, w, ws, **kw)
        msg = _compare(launch, got, full, parts)
        NOT_BIT_EQUAL[f"sweep-{launch.name()}-{kw}"] = _not_bit_equal(launch, got, full)
        if msg is not None:
            failures.append(f"{launch.name()} {kw}: {msg}")
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
def test_strided_operands_exact(fp8):
    """x as a view with row stride > k; FP8: x_scale a column slice of a wider buffer (stride k/128 + 3)."""
    for epi, splits in ((ge.EPI_BF16, 1), (ge.EPI_SILU, 1), (ge.EPI_PARTIAL, 4)):
        n = 512 if epi == ge.EPI_SILU else 256
        launch = ge.Launch(fp8, n, 2048, epi, 32, splits)
        x, xs, w, ws = _operands(launch, 100, ge.case_seed("strided", launch), x_pad=128, xs_pad=3 if fp8 else 0)
        assert x.stride(0) == 2048 + 128 and (not fp8 or (xs.stride(0) == 16 + 3 and not xs.is_contiguous()))
        got = _run(launch, x, xs, w, ws)
        full, parts = ge.reference(x, w, splits, xs, ws)
        msg = _compare(launch, got, full, parts)
        assert msg is None, f"{launch.name()}: {msg}"


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
def test_strided_bf16_output_exact(fp8):
    """EPI_BF16 into a view with row stride > n: the columns past n stay untouched."""
    rows, n, pad = 130, 256, 64
    launch = ge.Launch(fp8, n, 1024, ge.EPI_BF16, 64, 1)
    x, xs, w, ws = _operands(launch, rows, ge.case_seed("strided-out", launch))
    buf = torch.full((rows, n + pad), float("nan"), dtype=torch.bfloat16, device="cuda")
    got = _run(launch, x, xs, w, ws, out=buf[:, :n])
    assert got.stride(0) == n + pad
    full, parts = ge.reference(x, w, 1, xs, ws)
    msg = _compare(launch, got, full, parts)
    assert msg is None, msg
    assert torch.isnan(buf[:, n:]).all(), "the kernel wrote past the output columns"


ADD_NORM_CASES = sorted({(lc.n, lc.splits) for lc, _ in TABLE if lc.epi == ge.EPI_PARTIAL} | {(1024, 1)})


@pytest.mark.parametrize("rows", [1, 65, 128])
@pytest.mark.parametrize("cols,splits", ADD_NORM_CASES)
def test_add_rmsnorm_partials_exact(cols, splits, rows):
    """The split-K add + RMSNorm on exact partials (multiples of 2^-2, a different range per split): the residual
    bf16(bf16(sum of splits) + residual) is bit-exact against float64; the normed rows keep the bar of
    test_gpu_linear.py."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(ge.case_seed("addnorm", cols, splits, rows))
    scale = torch.tensor([2.0 ** (s % 5) for s in range(splits)], device="cuda")[:, None, None]
    parts = torch.randint(-256, 257, (splits, rows, cols), generator=g, device="cuda").float() * 2.0 ** -2 * scale
    residual = torch.randint(-64, 65, (rows, cols), generator=g, device="cuda").to(torch.bfloat16)
    weight = (1 + 0.1 * torch.randn(cols, generator=g, device="cuda")).to(torch.bfloat16)
    h = parts.double().sum(0)
    v = (h.to(torch.bfloat16).double() + residual.double()).to(torch.bfloat16)
    res = residual.clone()
    out, _ = ops.add_rmsnorm_partials(parts, res, weight, 1e-6)
    bad = res != v
    assert not bad.any(), ge.describe_mismatch(bad, res, v)
    vd = v.double()
    y = vd * torch.rsqrt((vd * vd).mean(-1, keepdim=True) + 1e-6) * weight.double()
    assert (out.double() - y).abs().max().item() <= 2.0 ** -7 * y.abs().max().item()


LM_CASES = [(151936, 128, 1), (18992, 128, 1), (18992, 64, 1), (4096, 32, 2), (151936, 128, 4)]


def _plant_ties(x, w, temps, block_n, cluster):
    """Give up to 8 greedy rows a maximal logit (w row = 4 * sign(x row) * 2^-6) at several vocabulary columns: the same
    CTA, the next CTA, the next cluster, and (one row) the ragged last column.  Returns {row: winning column}."""
    vocab = w.shape[0]
    greedy = [r for r in range(x.shape[0]) if temps[r] == 0][:8]
    stride = vocab // (len(greedy) + 1)
    assert stride > block_n * cluster + 1
    winners = {}
    for j, r in enumerate(greedy):
        pattern = (4 * torch.sign(x[r].float()) * ge.LM_HEAD_SCALE).to(torch.bfloat16)
        a = j * stride + (r * 7919) % (stride - block_n * cluster - 1)
        cols = [a + block_n, vocab - 1] if j == len(greedy) - 1 and j > 0 else [a, a + 1, a + block_n, a + block_n * cluster]
        for c in cols:
            w[c] = pattern
        winners[r] = min(cols)
    return winners


@pytest.mark.parametrize("offset", [0, 7], ids=["offset0", "offset7v"])
@pytest.mark.parametrize("rows", [1, 37, 256])
@pytest.mark.parametrize("vocab,block_n,cluster", LM_CASES)
def test_lm_head_sample_exact(vocab, block_n, cluster, rows, offset):
    """Greedy rows: the first-index argmax of the float64 logits rounded to bf16 (the kernel scores the bf16 logit, as
    the reference's F.linear output is bf16), ties planted across CTAs and clusters.  Every row: the two-kernel path
    (ops.sample) on those logits with the same seed and step."""
    ops = _ops()
    if (-(-vocab // block_n)) % cluster:
        pytest.skip("column blocks not divisible by the cluster size")
    k = 1024
    seed = ge.case_seed("lm_head", vocab, block_n, cluster, rows)
    x, w = ge.bf16_operands(rows, vocab, k, seed)
    w = (w.float() * ge.LM_HEAD_SCALE).to(torch.bfloat16)
    temps = torch.tensor([0.0 if i % 3 == 0 else 0.8 for i in range(rows)], dtype=torch.float32, device="cuda")
    winners = _plant_ties(x, w, temps, block_n, cluster)
    index_offset = offset * vocab
    full, _ = ge.reference(x, w)
    logits = full.to(torch.bfloat16)
    first = logits.float().argmax(-1)
    for r, c in winners.items():
        assert first[r].item() == c and (logits[r] == logits[r, c]).sum().item() >= 2      # the planted tie is the max
    want = ops.sample(logits, temps, seed=11, step=5, index_offset=index_offset)
    ws = torch.zeros(rows, dtype=torch.int64, device="cuda")
    got = ops.lm_head_sample(x, w, temps, 11, 5, ws, index_offset=index_offset, block_n=block_n, cluster=cluster)
    torch.cuda.synchronize()
    assert int(ws.abs().max()) == 0, "the key workspace must be left empty"
    greedy = temps == 0
    bad = greedy & (got != first + index_offset)
    assert not bad.any(), f"greedy rows {bad.nonzero().flatten().tolist()}: got {got[bad].tolist()} want {(first + index_offset)[bad].tolist()}"
    bad = got != want
    assert not bad.any(), f"{int(bad.sum())} of {rows} rows differ from ops.sample: rows {bad.nonzero().flatten().tolist()[:8]}"


def test_zz_report_not_bit_equal():
    """EPI_SILU outputs that are within the one-ulp bar but not bit-equal to float64 rounded to bf16, per case."""
    from gpu_helpers import record
    if NOT_BIT_EQUAL:
        record("gemm_exact_silu_not_bit_equal", dict(cases=len(NOT_BIT_EQUAL), total=sum(NOT_BIT_EQUAL.values()),
                                                     nonzero={k: v for k, v in NOT_BIT_EQUAL.items() if v}))
