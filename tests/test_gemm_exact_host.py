"""CPU side of the exact-operand GEMM tests (tests/gemm_exact.py, tests/test_gpu_gemm_exact.py), no library needed:

* every launch of the table and of the pipeline sweep stays exact in fp32 by its worst-case bound, not by the draw;
* no two neighbouring FP8 block scales are equal, so taking a neighbour's scale always changes the result;
* the launch table restated in gemm_exact.py is what models/qwen3.py launches: the model runs on the CPU at every Qwen3
  dims set with recording stand-ins for ``ops``, and the (n, k, epilogue, block_n, splits) of every wgmma call it makes
  must be the table's, so the table cannot drift from the model.
"""
from types import SimpleNamespace

import pytest
import torch

import gemm_exact as ge

EXACT = 2 ** 24


def test_table_covers_every_model_and_is_exact():
    table = ge.launch_table()
    seen = {src.split(".tp")[0] for srcs in table.values() for src in srcs}
    assert seen == set(ge.QWEN3)
    for (launch, rows), srcs in table.items():
        assert ge.exactness_ratio(launch) < EXACT, (launch, srcs)
        kt = launch.k // (ge.BLOCK if launch.fp8 else ge.LK)
        assert kt % launch.splits == 0 and launch.n % (launch.block_n // (2 if launch.epi == ge.EPI_SILU else 1)) == 0
    assert ge.fp8_block_bound() <= 2 ** 9
    # per-split block counts at the edges of the scale prefetch (nk < 4, nk = 1 mod 4) and hidden 5120 (40 k blocks)
    nks = {launch.k // ge.BLOCK // launch.splits for launch, _ in table if launch.fp8 and launch.epi == ge.EPI_PARTIAL}
    assert {2, 3, 12, 25} <= nks
    assert any(launch.fp8 and launch.k == 5120 for launch, _ in table)


def test_sweep_is_exact():
    for fp8 in (False, True):
        for nk in ge.SWEEP_NK:
            for splits in ge.SWEEP_SPLITS:
                launches = ge.sweep_launches(fp8, nk, splits)
                assert launches and {launch.splits for launch, _ in launches} == {splits}
                for launch, _ in launches:
                    assert ge.exactness_ratio(launch) < EXACT, launch
    # the LM head: x in {-4 .. 4}, w in {-4 .. 4} * 2^-6 over k = 1024; the 2^-6 cancels in the ratio
    assert ge.exactness_ratio(ge.Launch(False, 151936, 1024, ge.EPI_BF16, 128, 1)) < EXACT


def _assert_neighbours_distinct(e: torch.Tensor, pair_offset=None):
    assert (e[:, 1:] != e[:, :-1]).all()
    assert (e[1:] != e[:-1]).all()
    if pair_offset is not None:
        assert (e[pair_offset:] != e[:-pair_offset]).all()


@pytest.mark.parametrize("rows,n,k,epi", [(1, 1024, 2048, ge.EPI_PARTIAL), (130, 512, 3200, ge.EPI_SILU),
                                           (ge.PREFILL_ROWS, 51200, 5120, ge.EPI_SILU), (256, 5120, 25600, ge.EPI_BF16),
                                           (3, 256, 128, ge.EPI_SILU)])
def test_fp8_scales_neighbour_distinct(rows, n, k, epi):
    xs, ws = ge.fp8_scales(rows, n, k, epi, seed=ge.case_seed(rows, n, k, epi))
    assert xs.shape == (rows, k // 128) and ws.shape == (n // 128, k // 128)
    ex, ew = torch.log2(xs.double()), torch.log2(ws.double())
    assert torch.equal(ex, ex.round()) and torch.equal(ew, ew.round())                  # powers of two
    assert set(ex.unique().long().tolist()) <= set(ge.X_EXPONENTS) and set(ew.unique().long().tolist()) <= set(ge.W_EXPONENTS)
    _assert_neighbours_distinct(ex)
    _assert_neighbours_distinct(ew, n // 128 // 2 if epi == ge.EPI_SILU else None)
    if ex.numel() > 64:                                                                  # every allowed value is used
        assert set(ex.unique().long().tolist()) == set(ge.X_EXPONENTS)
    # deterministic for a seed
    assert torch.equal(xs, ge.fp8_scales(rows, n, k, epi, seed=ge.case_seed(rows, n, k, epi))[0])


def test_tp_rule_matches_the_fp8_shape_check():
    from nanovllm.utils import fp8 as fp8fmt
    for model, (hidden, inter, hq, hkv) in ge.QWEN3.items():
        for tp in ge.TP_SIZES:
            if not ge.tp_ok(model, tp, False):
                assert not ge.tp_ok(model, tp, True)
                continue
            try:
                fp8fmt.check_shapes(hq * 128 // tp, hkv * 128 // tp, hidden, inter // tp)
                ok = True
            except NotImplementedError:
                ok = False
            assert ge.tp_ok(model, tp, True) == ok, (model, tp)


# ---- the table against the model ---------------------------------------------------------------------------------------
class RecordingOps:
    """nanovllm.ops stand-ins that return tensors of the right shape and record every wgmma GEMM launch."""
    EPI_BF16, EPI_SILU, EPI_PARTIAL = ge.EPI_BF16, ge.EPI_SILU, ge.EPI_PARTIAL

    def __init__(self, hidden, head_dim):
        self.hidden, self.head_dim = hidden, head_dim
        self.launches: list[ge.Launch] = []

    class pdl_off:
        def __enter__(self):
            return self

        def __exit__(self, *exc):
            return False

    def embedding(self, ids, table, out=None):
        return torch.zeros(ids.shape[0], table.shape[1], dtype=table.dtype)

    def rmsnorm(self, x, weight, eps, out=None):
        return torch.zeros_like(x)

    def add_rmsnorm(self, x, residual, weight, eps, out=None):
        assert x.shape == residual.shape
        return torch.zeros_like(residual), residual

    def add_rmsnorm_partials(self, partials, residual, weight, eps, pdl=False, out=None):
        assert partials.dim() == 3 and partials.shape[1:] == residual.shape
        return (out if out is not None else torch.zeros_like(residual)), residual

    def silu_mul(self, x, out=None):
        return torch.zeros(x.shape[0], x.shape[1] // 2, dtype=x.dtype)

    def qknorm_rope_store(self, layer, qkv, *a, **k):
        return qkv

    def paged_decode_fused(self, layer, qkv, hq, *a, **k):
        return torch.zeros(qkv.shape[0], hq, self.head_dim, dtype=qkv.dtype)

    def paged_decode(self, layer, q, *a, **k):
        return torch.zeros_like(q)

    def paged_prefill(self, layer, q, *a, **k):
        return torch.zeros_like(q)

    def _out(self, rows, n, epi, splits, out, dtype):
        n_out = n // 2 if epi == ge.EPI_SILU else n
        if out is not None:
            assert out.shape == (rows, n_out)
            return out
        if epi == ge.EPI_PARTIAL:
            return torch.zeros(splits, rows, n_out, dtype=torch.float32)
        return torch.zeros(rows, n_out, dtype=dtype)

    def linear(self, x, w, epilogue=0, block_n=32, k_splits=1, pdl=False, out=None, shallow=False, cluster=1, stages=0):
        assert x.dtype == w.dtype == torch.bfloat16 and x.shape[1] == w.shape[1]
        self.launches.append(ge.Launch(False, w.shape[0], w.shape[1], epilogue, block_n, k_splits))
        return self._out(x.shape[0], w.shape[0], epilogue, k_splits, out, torch.bfloat16)

    def quant_fp8(self, x, out=None, scales=None):
        return (torch.zeros(x.shape, dtype=torch.float8_e4m3fn), torch.ones(x.shape[0], x.shape[1] // 128))

    def linear_fp8(self, xq, x_scale, w, w_scale, epilogue=0, block_n=64, k_splits=1, pdl=False, out=None, shallow=False,
                   cluster=1, stages=0):
        assert xq.dtype == w.dtype == torch.float8_e4m3fn and w_scale.shape == (w.shape[0] // 128, w.shape[1] // 128)
        assert x_scale.shape == (xq.shape[0], xq.shape[1] // 128)
        self.launches.append(ge.Launch(True, w.shape[0], w.shape[1], epilogue, block_n, k_splits))
        return self._out(xq.shape[0], w.shape[0], epilogue, k_splits, out, torch.bfloat16)


def _record_model(monkeypatch, model: str, fp8: bool, mode: str, rows: int, prefill: bool) -> list[ge.Launch]:
    import nanovllm.layers.attention as attn_mod
    import nanovllm.models.qwen3 as model_mod
    from nanovllm.utils import fp8 as fp8fmt
    from nanovllm.utils.context import reset_context, set_context
    from nanovllm.utils.synthetic import hf_config_dict
    for var in ("B200_LINEAR", "B200_LINEAR_CFG", "B200_LINEAR_MAX_ROWS", "B200_LINEAR_SPLITS_BIG", "B200_TAIL", "B200_DUAL"):
        monkeypatch.delenv(var, raising=False)
    monkeypatch.setenv("B200_LINEAR", mode)
    hidden, inter, hq, hkv = ge.QWEN3[model]
    cfg = hf_config_dict(dict(hidden_size=hidden, num_hidden_layers=1, num_attention_heads=hq, num_key_value_heads=hkv,
                              head_dim=ge.HEAD_DIM, intermediate_size=inter, vocab_size=1024, tie_word_embeddings=False))
    if fp8:
        cfg["quantization_config"] = fp8fmt.quantization_config_dict()
    fake = RecordingOps(hidden, ge.HEAD_DIM)
    monkeypatch.setattr(model_mod, "ops", fake)
    monkeypatch.setattr(attn_mod, "ops", fake)
    monkeypatch.setattr(model_mod, "F", SimpleNamespace(linear=lambda x, w: torch.zeros(x.shape[0], w.shape[0], dtype=x.dtype)))
    m = model_mod.Qwen3ForCausalLM(SimpleNamespace(**cfg), 0, 1, "cpu", max_position=4096)
    assert m.fp8 == fp8
    for a in m.modules():
        a.k_cache = a.v_cache = torch.zeros(1, hkv, 16, ge.HEAD_DIM, dtype=torch.bfloat16)     # "cache allocated"
    ids, pos = torch.zeros(rows, dtype=torch.int64), torch.arange(rows, dtype=torch.int64)
    if prefill:
        cu = torch.tensor([0, rows], dtype=torch.int32)
        set_context(True, cu, cu, rows, rows, torch.arange(rows, dtype=torch.int32), None, None)
    else:
        set_context(False, None, None, 0, 0, torch.arange(rows, dtype=torch.int32), torch.ones(rows, dtype=torch.int32),
                    torch.zeros(rows, 1, dtype=torch.int32))
    try:
        m(ids, pos)
    finally:
        reset_context()
    return fake.launches


STEPS = [(1, False), (128, False), (129, False), (ge.PREFILL_ROWS, True)]


@pytest.mark.parametrize("model", list(ge.QWEN3))
@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
def test_launch_table_is_what_the_model_launches(model, fp8, monkeypatch):
    """One decoder layer at TP 1 on decode steps of 1, 128 and 129 rows and one prefill: under B200_LINEAR=rows (o /
    down on wgmma up to 256 rows) the model's launches are exactly the table's, under the default auto policy they are
    the table's up to 128 rows and none above; FP8 ignores the policy."""
    table = ge.launch_table()
    for rows, prefill in STEPS:
        want = sorted(launch for _, launch in ge.model_launches(model, 1, fp8, rows, prefill))
        for launch in want:
            assert (launch, rows) in table
        for mode in ("rows", "auto"):
            got = sorted(_record_model(monkeypatch, model, fp8, mode, rows, prefill))
            if mode == "auto" and not fp8 and rows > 128:
                assert got == [], (rows, got)
            else:
                assert got == want, (mode, rows, prefill, got, want)
