"""The needle cases of tests/test_gpu_attention_needles.py, built on the CPU at full size: each one targets split pairs
that really are cut into 3 or more segments, and every designed defect (a needle dropped, a neighbour key read in its
place, the key past the end or past the causal diagonal admitted) moves some checked (row, head) vector by 4x its bar
or more.  The float64 model of the defects is checked against the suite's references on the same rows."""
import pytest
import torch

import attention_needles as an

POWER = 4.0
# warps per CTA of every decode kernel the GPU file runs: FMA default and its B200_DECODE_CFG variants, MMA, fp8 MMA
DECODE_WARPS = {"fma": (8, 12, 10, 6), "mma": (8,), "fp8": (12,)}


def assert_power(defects, what):
    n = 0
    for row, _, res in defects:
        for edit, ratio in res:
            assert ratio >= POWER, f"{what}: row {row}, {edit} moves the output by {ratio:.2f}x the bar only"
            n += 1
    assert n, f"{what}: no defect checked"


def model_matches(defects, want, rows, what, tol=0.25):
    """The defect model's clean rows are the reference's (within tol of the bar: prefill64 rounds P to bf16)."""
    got = {r: clean for r, clean, _ in defects}
    for i, r in enumerate(rows):
        if r in got:
            assert an.vector_ratio(got[r], want[i]).max().item() <= tol, f"{what}: the defect model's clean row {r}"


@pytest.mark.parametrize("case", an.DECODE_CASES)
@pytest.mark.parametrize("kind,G", [("fma", 1), ("fma", 2), ("mma", 4), ("mma", 8), ("fp8", 1), ("fp8", 2), ("fp8", 4),
                                    ("fp8", 8)], ids=lambda x: str(x))
def test_decode_needle_power(kind, G, case):
    for nw in DECODE_WARPS[kind]:
        cs = an.decode_case(case, G, device="cpu", nwarps=nw, fp8=kind == "fp8")
        if case != "positions16" and case != "positions256" or cs.splits:
            an.check_splits(cs)
        if nw == DECODE_WARPS[kind][0]:
            defects = list(an.decode_defects(cs))
            assert_power(defects, f"decode {case} {kind} G={G}")
            model_matches(defects, an.decode_reference(cs), cs.rows, f"decode {case} {kind} G={G}")


@pytest.mark.parametrize("case", an.FUSED_CASES)
@pytest.mark.parametrize("G", [1, 2])
def test_fused_decode_needle_power(G, case):
    cs = an.fused_case(case, G, device="cpu")
    if case == "segments":
        an.check_splits(cs)
    defects = list(an.decode_defects(cs))
    assert_power(defects, f"fused decode {case} G={G}")
    model_matches(defects, an.decode_reference(cs), cs.rows, f"fused decode {case} G={G}")
    for b, L in enumerate(cs.lens):                            # the newest token is a needle of every row
        if L:
            assert any(L - 1 in ps for (bb, _, _), ps in cs.needles.items() if bb == b)


@pytest.mark.parametrize("case", an.PREFILL_CASES)
def test_prefill_needle_power(case):
    cs = an.prefill_case(case, device="cpu")
    defects = list(an.prefill_defects(cs))
    assert_power(defects, f"prefill {case}")
    model_matches(defects, an.prefill_reference(cs), cs.rows, f"prefill {case}", tol=0.5)
    checked = set(cs.rows)
    assert all(r in checked for r, _, _ in defects), "a defect row is not among the checked rows"
    if case.startswith(("causal", "chunk")):               # a needle on the diagonal of every 128-query tile
        for s, lq in enumerate(cs.lens_q):
            off = cs.lens_k[s] - lq
            tiles = {(j - off) // 128 for (ss, _, _), ps in cs.needles.items() if ss == s for j in ps}
            assert tiles == set(range((lq + 127) // 128))
    if case == "rescale":                                  # gaps of 7.9 and 8.1 kernel log2 units, in one tile and later
        kinds = {(later, delta) for _, _, _, later, delta, _ in cs.gaps}
        assert kinds == {(a, b) for a in (True, False) for b in (7.9, 8.1)}
        for _, _, _, _, delta, gap in cs.gaps:
            assert abs(gap - delta) < 0.05, (delta, gap)


def test_partition_restatement():
    """pair_segments against a direct walk of every worker's chunk range."""
    lens = [40960, 3, 0, 257, 16, 17, 12288]
    for nw in (6, 8, 10, 12):
        part = an.decode_partition(lens, 2, nw, an.H100_SMS)
        owner = {}
        for gw in range(part.TWe):
            for c in range(gw * part.C // part.TWe, (gw + 1) * part.C // part.TWe):
                owner[c] = gw
        assert len(owner) == part.C
        for b, L in enumerate(lens):
            for h in range(2):
                segs = an.pair_segments(part, b, h)
                c0 = 2 * part.cum[b] + h * part.n[b]
                want = sorted({owner[c0 + t // 16] for t in range(0, L, 16)})
                assert len(segs) == len(want)
                assert all(owner[c0 + s // 16] == w for (s, _), w in zip(segs, want))
                assert sum(e - s for s, e in segs) == L
