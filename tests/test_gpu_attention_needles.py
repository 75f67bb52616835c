"""The attention kernels against float64 with needle keys at every split, page, chunk, tile and causal boundary
(tests/attention_needles.py builds the cases; tests/test_attention_needles_host.py proves on the CPU that each designed
defect at those keys moves a checked vector by 4x its bar or more).

Each (row, query head) output vector is held to 2 bf16 ulps of its own largest reference value (prefill: 4, derived at
attention_needles.PREFILL_ULPS), every case asserts which kernel ran, and every decode case asserts that the pairs it
targets are split into 3 or more segments by that kernel's stream-K partition.  Variables the library reads once per process (B200_DECODE, B200_DECODE_CFG, B200_PREFILL,
B200_PREFILL_POLY) are covered by child pytest runs of the matching subset (test_switch_*).
"""
import os

import pytest
import torch

import attention_needles as an
from test_gpu_dispatch_edges import IN_CHILD, EPS, SCALE, assert_ran, decode_kernel, launched, prefill_kernel, run_child

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from nanovllm import ops as _ops
    return _ops


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------------
# decode: FMA (G 1, 2), tensor-core (G 4, 8), fp8 tensor-core (G 1..8), fused (G 1, 2)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", an.DECODE_CASES)
@pytest.mark.parametrize("cache,G", [("bf16", 1), ("bf16", 2), ("bf16", 4), ("bf16", 8), ("fp8", 1), ("fp8", 2), ("fp8", 4),
                                     ("fp8", 8)], ids=lambda x: f"G{x}" if isinstance(x, int) else x)
def test_decode_needles(ops, cache, G, case):
    kernel = f"paged_decode_mma_fp8_kernel<{G}>" if cache == "fp8" else decode_kernel(G)
    cs = an.decode_case(case, G, device="cuda", nwarps=an.decode_warps(kernel), sm_count=sm_count(), fp8=cache == "fp8")
    if cs.splits or not case.startswith("positions"):
        an.check_splits(cs)
    ops.bind_kv_cache(cs.kv, **cs.scales)
    got, names = launched(lambda: ops.paged_decode(0, cs.q, cs.tables, cs.ctx, SCALE))
    what = f"decode needles {case} {cache} G={G}"
    assert_ran(names, kernel, what)
    an.assert_vectors_close(got[cs.rows], an.decode_reference(cs), what)
    assert (got[cs.ctx == 0] == 0).all(), "zero-context rows are exactly zero"


@pytest.mark.parametrize("case", an.FUSED_CASES)
@pytest.mark.parametrize("G", [1, 2], ids=lambda G: f"G{G}")
def test_fused_decode_needles(ops, G, case):
    kernel = decode_kernel(G, fused=True)
    cs = an.fused_case(case, G, device="cuda", nwarps=an.decode_warps(kernel), sm_count=sm_count())
    if case == "segments":
        an.check_splits(cs)
    ops.bind_kv_cache(cs.kv)
    got, names = launched(lambda: ops.paged_decode_fused(0, cs.qkv, G * cs.hkv, cs.qw, cs.kw, cs.table, EPS, cs.tables,
                                                         cs.ctx, SCALE))
    what = f"fused decode needles {case} G={G}"
    assert_ran(names, kernel, what)
    an.assert_vectors_close(got[cs.rows], an.decode_reference(cs), what)


# ---------------------------------------------------------------------------------------------------------------------
# prefill: packed, paged and chunked over a prefix (prefill_tc, or prefill_ws under B200_PREFILL=ws); fp8 paged prefill
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", an.PREFILL_CASES)
def test_prefill_needles(ops, case):
    cs = an.prefill_case(case, device="cuda")
    mq, mk = max(cs.lens_q), max(cs.lens_k)
    if cs.paged:
        ops.bind_kv_cache(cs.kv)
        run = lambda: ops.paged_prefill(0, cs.q, None, None, cs.cu_q, cs.cu_k, mq, mk, SCALE, block_tables=cs.tables,
                                        num_kv_heads=cs.hkv)
    else:
        run = lambda: ops.paged_prefill(0, cs.q, cs.k, cs.v, cs.cu_q, cs.cu_k, mq, mk, SCALE)
    got, names = launched(run)
    what = f"prefill needles {case}"
    assert_ran(names, prefill_kernel(), what)
    an.assert_vectors_close(got[cs.rows], an.prefill_reference(cs), what, ulps=an.PREFILL_ULPS)


@pytest.mark.parametrize("case", ["chunk16", "chunk256", "causal-paged16"])
def test_prefill_needles_fp8(ops, case):
    """Paged prefill over an e4m3 cache: the gather dequantizes to bf16, then the packed prefill kernel runs."""
    from nanovllm.layers.attention import Attention
    from nanovllm.utils.context import reset_context, set_context
    from test_gpu_kv_fp8 import device_groups, logical, to_fp8
    ks, vs = an.FP8_SCALES
    cs = an.prefill_case(case, device="cuda")
    kv8 = to_fp8(cs.kv, ks, vs)
    ops.bind_kv_cache(kv8, k_scale=ks, v_scale=vs)
    attn = Attention(cs.hq, an.D, SCALE, cs.hkv)
    attn.k_cache, attn.v_cache, attn.layer_id = kv8[0, 0], kv8[1, 0], 0
    attn.kv_scratch = torch.full((2, sum(cs.lens_k), cs.hkv, an.D), float("nan"), dtype=torch.bfloat16, device="cuda")
    groups = device_groups(cs.cu_q, cs.cu_k, attn.kv_scratch.shape[1])
    set_context(True, cs.cu_q, cs.cu_k, max(cs.lens_q), max(cs.lens_k), None, None, cs.tables, groups)
    try:
        got, names = launched(lambda: attn(cs.q, None, None, kv_stored=True))
    finally:
        reset_context()
    what = f"fp8 prefill needles {case}"
    assert_ran(names, "kv_gather_fp8_kernel", what)
    assert_ran(names, prefill_kernel(), what)
    want = an.prefill_reference(cs, K=logical(kv8, 0, 0, ks).to(torch.bfloat16), V=logical(kv8, 0, 1, vs).to(torch.bfloat16))
    an.assert_vectors_close(got[cs.rows], want, what, ulps=an.PREFILL_ULPS)


# ---------------------------------------------------------------------------------------------------------------------
# variables read once per process: the matching subset in a child pytest
# ---------------------------------------------------------------------------------------------------------------------
SWITCHES = {
    "decode_mma": ({"B200_DECODE": "mma"}, "test_decode_needles and bf16"),
    "decode_cfg_12x2": ({"B200_DECODE_CFG": "12x2"}, "test_decode_needles and bf16 and (G1 or G2)"),
    "decode_cfg_10x2": ({"B200_DECODE_CFG": "10x2"}, "test_decode_needles and bf16 and (G1 or G2)"),
    "decode_cfg_8x3": ({"B200_DECODE_CFG": "8x3"}, "test_decode_needles and bf16 and (G1 or G2)"),
    "decode_cfg_6x2": ({"B200_DECODE_CFG": "6x2"}, "test_decode_needles and bf16 and (G1 or G2)"),
    "prefill_ws_poly": ({"B200_PREFILL": "ws", "B200_PREFILL_POLY": "1"}, "prefill_needles"),
    "prefill_ws_mufu": ({"B200_PREFILL": "ws", "B200_PREFILL_POLY": "0"}, "prefill_needles"),
}


@pytest.mark.parametrize("switch", list(SWITCHES))
def test_switch_needles(switch):
    if IN_CHILD:
        pytest.skip("already a child process")
    env, kexpr = SWITCHES[switch]
    run_child(kexpr, env, path=os.path.abspath(__file__))
