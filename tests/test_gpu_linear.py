"""Parity tests for the wgmma linear layer (csrc/linear_tc.cu): the decode-size projections of the product path (o_proj /
down_proj split-K for batches <= 128 rows; all four in the two-stream decode step) and the fused LM-head + sampling kernel.

Reference for every case: torch fp32 matmul of the same bf16 inputs, rounded where the reference rounds
(F.linear output is bf16, layers/linear.py:51,73,153; SiluAndMul in fp32 on that, layers/activation.py:8-11).
Part of the default GPU suite.
"""
import pytest
import torch

pytestmark = [pytest.mark.gpu]


def _inputs(rows, n, k, seed=0, x_pad=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    xb = torch.randn(rows, k + x_pad, generator=g).to(torch.bfloat16).cuda()
    x = xb[:, :k]
    w = (torch.randn(n, k, generator=g) * k ** -0.5).to(torch.bfloat16).cuda()
    return x, w


@pytest.mark.parametrize("rows", [1, 37, 128, 129, 256])
@pytest.mark.parametrize("n,k,block_n", [(4096, 1024, 32), (4096, 1024, 64), (1024, 2048, 16), (1024, 3072, 128), (512, 64, 32)])
def test_linear_bf16(rows, n, k, block_n):
    from nanovllm import ops
    x, w = _inputs(rows, n, k, seed=rows + n)
    got = ops.linear(x, w, ops.EPI_BF16, block_n)
    torch.cuda.synchronize()
    want = (x.float() @ w.float().t())
    err = (got.float() - want).abs().max().item()
    # fp32 accumulation in a different order + one bf16 rounding of the output
    assert err <= 2.0 ** -7 * want.abs().max().item() + 1e-3, err


@pytest.mark.parametrize("block_n", [16, 32, 64, 128])
def test_linear_shallow_ring(block_n):
    from nanovllm import ops
    x, w = _inputs(200, 1024, 2048, seed=block_n)                 # 32 k tiles through a 3-4 slot ring: many wrap-arounds
    got = ops.linear(x, w, ops.EPI_BF16, block_n, shallow=True)
    want = x.float() @ w.float().t()
    assert (got.float() - want).abs().max().item() <= 2.0 ** -7 * want.abs().max().item() + 1e-3
    assert torch.equal(got, ops.linear(x, w, ops.EPI_BF16, block_n))      # ring depth does not change the arithmetic


@pytest.mark.parametrize("stages", [2, 3])
@pytest.mark.parametrize("block_n", [32, 64])
def test_linear_explicit_ring_depth(stages, block_n):
    """flags bits 4-7: the 2-3 slot rings of the two-stream decode step (a CTA that fits beside the attention kernel's);
    the ring depth changes the schedule, never the arithmetic."""
    from nanovllm import ops
    x, w = _inputs(128, 1024, 2048, seed=block_n + stages)
    assert torch.equal(ops.linear(x, w, ops.EPI_BF16, block_n, stages=stages, pdl=True), ops.linear(x, w, ops.EPI_BF16, block_n))
    xw, ww = _inputs(100, 2 * 3072, 1024, seed=7)
    assert torch.equal(ops.linear(xw, ww, ops.EPI_SILU, block_n, stages=stages), ops.linear(xw, ww, ops.EPI_SILU, block_n))
    xd, wd = _inputs(128, 1024, 3072, seed=8)
    assert torch.equal(ops.linear(xd, wd, ops.EPI_PARTIAL, block_n, 8, stages=stages), ops.linear(xd, wd, ops.EPI_PARTIAL, block_n, 8))


@pytest.mark.parametrize("cluster", [2, 4])
@pytest.mark.parametrize("rows", [1, 100, 256])
def test_linear_multicast_cluster(cluster, rows):
    """x tiles fetched once per cluster and multicast to its CTAs: bit-identical to the unclustered kernel."""
    from nanovllm import ops
    x, w = _inputs(rows, 4096, 1024, seed=rows + cluster)
    base = ops.linear(x, w, ops.EPI_BF16, 32)
    assert torch.equal(ops.linear(x, w, ops.EPI_BF16, 32, cluster=cluster), base)
    assert torch.equal(ops.linear(x, w, ops.EPI_BF16, 32, cluster=cluster, pdl=True), base)
    xw, ww = _inputs(rows, 2 * 3072, 1024, seed=7)
    assert torch.equal(ops.linear(xw, ww, ops.EPI_SILU, 32, cluster=cluster), ops.linear(xw, ww, ops.EPI_SILU, 32))
    xd, wd = _inputs(rows, 1024, 3072, seed=8)                                    # 48 k tiles, 8 splits, ring wraps
    assert torch.equal(ops.linear(xd, wd, ops.EPI_PARTIAL, 64, 2, cluster=cluster), ops.linear(xd, wd, ops.EPI_PARTIAL, 64, 2))


def test_linear_strided_x():
    from nanovllm import ops
    x, w = _inputs(100, 1024, 1024, seed=5, x_pad=64)       # row stride 1088: a view into a wider buffer
    got = ops.linear(x, w, ops.EPI_BF16, 32)
    want = x.float() @ w.float().t()
    assert (got.float() - want).abs().max().item() <= 2.0 ** -7 * want.abs().max().item() + 1e-3


@pytest.mark.parametrize("rows", [1, 64, 200, 256])
@pytest.mark.parametrize("block_n", [32, 64, 128])
def test_linear_silu(rows, block_n):
    from nanovllm import ops
    inter, k = 3072, 1024
    x, w = _inputs(rows, 2 * inter, k, seed=rows)
    got = ops.linear(x, w, ops.EPI_SILU, block_n)
    y = (x.float() @ w.float().t()).to(torch.bfloat16).float()
    g, u = y[:, :inter], y[:, inter:]
    want = (g * torch.sigmoid(g) * u)
    err = (got.float() - want).abs().max().item()
    assert err <= 2.0 ** -6 * want.abs().max().item() + 1e-3, err
    # and against the two-kernel path it replaces, which shares the rounding points exactly up to accumulation order
    two = ops.silu_mul((x @ w.t()).contiguous())
    assert (got.float() - two.float()).abs().max().item() <= 2.0 ** -6 * want.abs().max().item() + 1e-3


@pytest.mark.parametrize("rows", [1, 130, 256])
@pytest.mark.parametrize("k,splits,block_n", [(2048, 4, 64), (3072, 8, 64), (3072, 6, 32), (1024, 1, 16)])
def test_linear_splitk_add_rmsnorm(rows, k, splits, block_n):
    from nanovllm import ops
    n = 1024
    x, w = _inputs(rows, n, k, seed=rows + k)
    g = torch.Generator(device="cpu").manual_seed(9)
    residual = torch.randn(rows, n, generator=g).to(torch.bfloat16).cuda()
    weight = (1 + 0.1 * torch.randn(n, generator=g)).to(torch.bfloat16).cuda()
    parts = ops.linear(x, w, ops.EPI_PARTIAL, block_n, splits)
    assert parts.shape == (splits, rows, n)
    want_h = x.float() @ w.float().t()
    assert (parts.sum(0) - want_h).abs().max().item() <= 1e-3 * max(1.0, want_h.abs().max().item())
    res_a, res_b = residual.clone(), residual.clone()
    out_a, _ = ops.add_rmsnorm_partials(parts, res_a, weight, 1e-6)
    h = parts[0].clone()
    for s in range(1, splits):
        h += parts[s]
    out_b, _ = ops.add_rmsnorm(h.to(torch.bfloat16), res_b, weight, 1e-6)
    assert torch.equal(res_a, res_b)                                         # same rounding points, same order
    # the normalised rows may differ by one rounding: the two kernels add the squares in a different order
    assert (out_a.float() - out_b.float()).abs().max().item() <= 2.0 ** -7 * out_b.float().abs().max().item()
    # run-to-run determinism
    parts2 = ops.linear(x, w, ops.EPI_PARTIAL, block_n, splits)
    assert torch.equal(parts, parts2)


def test_linear_pdl_chain_in_graph():
    """Programmatic dependent launch: a chain of our kernels captured in a CUDA graph gives the eager result."""
    from nanovllm import ops
    rows, hidden, inter = 64, 1024, 3072
    x, w1 = _inputs(rows, 2 * inter, hidden, seed=1)
    _, w2 = _inputs(rows, hidden, inter, seed=2)
    g0 = torch.Generator(device="cpu").manual_seed(3)
    residual0 = torch.randn(rows, hidden, generator=g0).to(torch.bfloat16).cuda()
    weight = torch.ones(hidden, dtype=torch.bfloat16, device="cuda")

    def chain(pdl, residual):
        a = ops.linear(x, w1, ops.EPI_SILU, 32, pdl=pdl)
        p = ops.linear(a, w2, ops.EPI_PARTIAL, 64, 8, pdl=pdl)
        return ops.add_rmsnorm_partials(p, residual, weight, 1e-6, pdl=pdl)[0]

    want = chain(False, residual0.clone())
    torch.cuda.synchronize()
    res = residual0.clone()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        chain(True, res.clone())                      # warm-up outside capture (cudaFuncSetAttribute, map cache)
    s.synchronize()
    graph = torch.cuda.CUDAGraph()
    static_res = residual0.clone()
    with torch.cuda.graph(graph):
        got = chain(True, static_res)
    for _ in range(3):
        static_res.copy_(residual0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(got, want)


@pytest.mark.parametrize("preset", ["tiny", "tiny-g4"])
def test_model_with_tc_linear_matches_library_path(preset, monkeypatch):
    """B200_LINEAR=tc (every decode-size projection through linear_tc.cu) against the default cuBLAS path on the
    7-step teacher-forced script: same rounding points, so only accumulation order differs."""
    from oracle.model_script import make_script, run_script
    from nanovllm.utils.context import reset_context, set_context
    from nanovllm.utils.synthetic import PRESETS, random_weights
    from test_gpu_model import build_product_model
    weights = random_weights(PRESETS[preset], seed=1234)
    script = make_script(PRESETS[preset]["vocab_size"])

    def run(mode):
        monkeypatch.setenv("B200_LINEAR", mode)
        monkeypatch.setenv("B200_LINEAR_CFG", "32,32,64,4,64,4,0")
        model, _ = build_product_model(preset, weights, script["num_blocks"], script["block_size"])
        assert model.tc_linear == (mode == "tc")

        def step(ids, pos, c):
            set_context(c["is_prefill"], c.get("cu_seqlens_q"), c.get("cu_seqlens_k"), c.get("max_seqlen_q", 0),
                        c.get("max_seqlen_k", 0), c.get("slot_mapping"), c.get("context_lens"), c.get("block_tables"))
            out = model.compute_logits(model(ids, pos)).float().cpu()
            reset_context()
            return out
        return run_script(torch, script, step, device="cuda")

    want, got = run("cublas"), run("tc")
    for i, (g, w) in enumerate(zip(got, want)):
        rel = ((g - w).norm() / w.norm()).item()
        assert rel < 1e-2, f"step {i}: relative L2 {rel}"


@pytest.mark.parametrize("rows", [1, 37, 256])
@pytest.mark.parametrize("vocab,block_n,cluster", [(151936, 128, 1), (18992, 128, 1), (18992, 64, 1), (4096, 32, 2), (151936, 128, 4)])
def test_fused_lm_head_sampling_matches_the_two_kernel_path(rows, vocab, block_n, cluster):
    """hidden -> tokens without materialising logits, against F.linear + b200_sample on the same inputs: same RNG, same
    scoring, so tokens can differ only where two candidates are within the bf16 rounding of differently-ordered sums."""
    from nanovllm import ops
    k = 1024
    if (-(-vocab // block_n)) % cluster:
        pytest.skip("column blocks not divisible by the cluster size")
    x, w = _inputs(rows, vocab, k, seed=rows + vocab)
    w = (w.float() * 8).to(torch.bfloat16)                        # logits with a spread of a few units, like a real head
    temps = torch.tensor([0.0 if i % 3 == 0 else 0.8 for i in range(rows)], dtype=torch.float32, device="cuda")
    ws = torch.zeros(rows, dtype=torch.int64, device="cuda")
    offset = 7 * vocab
    logits = x @ w.t()
    want = ops.sample(logits, temps, seed=11, step=5, index_offset=offset)
    keys = torch.empty(rows, dtype=torch.int64, device="cuda")
    got = ops.lm_head_sample(x, w, temps, 11, 5, ws, index_offset=offset, out_keys=keys, out=torch.empty(rows, dtype=torch.int64, device="cuda"),
                             block_n=block_n, cluster=cluster)
    torch.cuda.synchronize()
    assert int(ws.abs().max()) == 0, "the key workspace must be left empty"
    assert ((got >= offset) & (got < offset + vocab)).all()
    assert torch.equal(ops.tokens_from_keys(keys), got)
    same = (got == want).float().mean().item()
    assert same >= 0.95, f"only {same:.3f} of the rows agree with the two-kernel path"
    lf = logits.float()
    tol = 2 * 2.0 ** -8 * lf.abs().max().item()
    for r in range(rows):
        if temps[r] == 0 and got[r] != want[r]:                  # greedy disagreement only on a near-tie
            assert (lf[r].max() - lf[r, got[r] - offset]).item() <= tol
    # deterministic, and fresh noise for another step
    again = ops.lm_head_sample(x, w, temps, 11, 5, ws, index_offset=offset, block_n=block_n, cluster=cluster)
    assert torch.equal(again, got)
    other = ops.lm_head_sample(x, w, temps, 11, 6, ws, index_offset=offset, block_n=block_n, cluster=cluster)
    sampled = temps > 0
    if rows >= 37:
        assert (other[sampled] != got[sampled]).any()
    assert torch.equal(other[~sampled], got[~sampled])
