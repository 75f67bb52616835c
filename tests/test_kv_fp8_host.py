"""The fp8 KV-cache option without a GPU: Config values, argument checks of the new C entry points, the oracle's e4m3
quantizer against a table of hand-computed values, and the engine's split of a paged prefill into gather groups."""
import ctypes
import math

import numpy as np
import pytest
import torch

from kv_fp8_ref import dequantize_e4m3, quantize_e4m3


def _config(**kw):
    from types import SimpleNamespace
    from nanovllm.config import Config
    hf = SimpleNamespace(max_position_embeddings=4096)
    return Config("unused", hf_config=hf, **kw)


@pytest.mark.parametrize("value", ["auto", "fp8", "fp8_e4m3"])
def test_config_accepts(value):
    assert _config(kv_cache_dtype=value).kv_cache_dtype == value
    assert _config().kv_cache_dtype == "auto"


@pytest.mark.parametrize("value", ["fp8_e5m2", "bf16", "float8", "", "FP8", None])
def test_config_rejects(value):
    with pytest.raises(ValueError):
        _config(kv_cache_dtype=value)


def test_config_field_is_last():
    from dataclasses import fields
    from nanovllm.config import Config
    names = [f.name for f in fields(Config)]
    assert names[-1] == "kv_cache_dtype"


def test_c_entry_points_validate_without_gpu():
    from nanovllm import _native as nat
    lib = nat.load()
    EINVAL = -1
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 128
    # null context, null pointers
    assert lib.b200_kv_bind_fp8(None, p, p, 1, 1, 16, 1, 128, 1.0, 1.0) == EINVAL
    assert lib.b200_kv_bind_fp8(None, None, p, 1, 1, 16, 1, 128, 1.0, 1.0) == EINVAL
    # scales that are not finite and > 0 are refused before anything else is looked at
    for ks, vs in ((0.0, 1.0), (1.0, -1.0), (math.nan, 1.0), (1.0, math.inf), (-0.0, 1.0), (1.0, math.nan)):
        assert lib.b200_kv_bind_fp8(None, p, p, 1, 1, 16, 1, 128, ks, vs) == EINVAL
    assert lib.b200_kv_gather(None, 0, p, 1, p, 1, p, 128, p, 128, 1, None) == EINVAL
    assert lib.b200_kv_gather(None, 0, None, 1, p, 1, p, 128, p, 128, 1, None) == EINVAL
    assert lib.b200_prefill_packed_kv(None, p, 128, p, 128, p, 128, p, p, p, 128, 1, 2, 1, 1, 1, 1, 0.1, None) == EINVAL


# (input, scale, expected e4m3 value): round-to-nearest-even ties, saturation at +-448, subnormals down to 2^-9
QUANT_TABLE = [
    (1.0, 1.0, 1.0),
    (1.0625, 1.0, 1.0),            # halfway between 1.0 and 1.125: even mantissa (1.0)
    (1.09375, 1.0, 1.125),         # past the halfway point: rounds up
    (1.1875, 1.0, 1.25),           # halfway between 1.125 (odd) and 1.25 (even)
    (-1.0625, 1.0, -1.0),
    (448.0, 1.0, 448.0),
    (464.0, 1.0, 448.0),           # past the largest finite value: saturates instead of NaN
    (1e6, 1.0, 448.0),
    (-1e6, 1.0, -448.0),
    (2.0 ** -9, 1.0, 2.0 ** -9),   # smallest subnormal
    (2.0 ** -10, 1.0, 0.0),        # half of it: tie to even (zero)
    (1.5 * 2.0 ** -10, 1.0, 2.0 ** -9),
    (3 * 2.0 ** -9, 1.0, 3 * 2.0 ** -9),
    (2.0 ** -6, 1.0, 2.0 ** -6),   # smallest normal
    (7 * 2.0 ** -9, 1.0, 7 * 2.0 ** -9),   # largest subnormal
    (240.0, 1.0, 240.0),
    (232.0, 1.0, 224.0),           # tie between 224 (even) and 240
    (3.0, 0.5, 6.0),               # x / scale
    (300.0, 0.5, 448.0),           # saturates after the division
    (0.75, 0.375, 2.0),
    (-1.0, 4.0, -0.25),
]


def test_oracle_quantizer_table():
    x = torch.tensor([r[0] for r in QUANT_TABLE], dtype=torch.float32)
    for i, (xv, s, want) in enumerate(QUANT_TABLE):
        got = quantize_e4m3(x[i:i + 1], s).float().item()
        assert got == want, f"e4m3({xv} / {s}) = {got}, expected {want}"
        assert dequantize_e4m3(quantize_e4m3(x[i:i + 1], s), s).item() == want * s


def test_oracle_quantizer_covers_every_code():
    """Every finite e4m3 value is a fixed point of quantize(dequantize()), for unit and non-unit scales."""
    codes = torch.arange(256, dtype=torch.int32).to(torch.uint8)
    vals = codes.view(torch.float8_e4m3fn).float()
    finite = torch.isfinite(vals)
    for s in (1.0, 0.5, 0.75):
        back = quantize_e4m3(dequantize_e4m3(codes[finite], s), s).view(torch.uint8)
        same = back == codes[finite]
        zero = vals[finite] == 0                  # -0 and +0 may swap
        assert bool((same | zero).all())


def test_gather_groups():
    from nanovllm.layers.attention import kv_group_arrays, plan_kv_groups
    cu_q = np.array([0, 50, 1050, 1067, 1167], dtype=np.int32)
    cu_k = np.array([0, 300, 1300, 1317, 2017], dtype=np.int32)
    groups = plan_kv_groups(cu_k, 1100)
    assert groups == [(0, 1), (1, 3), (3, 4)]
    arrs = kv_group_arrays(cu_q, cu_k, groups)
    assert [a[:6] for a in arrs] == [(0, 1, 0, 50, 300, 50), (1, 3, 50, 1067, 1017, 1000), (3, 4, 1067, 1167, 700, 100)]
    assert arrs[1][6].tolist() == [0, 1000, 1017] and arrs[1][7].tolist() == [0, 1000, 1017]
    assert plan_kv_groups(cu_k, 10 ** 6) == [(0, 4)]
    assert plan_kv_groups(cu_k, 1) == [(0, 1), (1, 2), (2, 3), (3, 4)]      # one sequence always makes a group
