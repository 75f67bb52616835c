"""The fused tensor-parallel exchange (csrc/tp_allreduce.cu, allreduce_add_rmsnorm_kernel<false>) on ONE GPU.

The kernel reaches the other ranks only through bases[p] + data_off (their partials) and bases[p] + flag_off (their
flag words).  So the ranks' slices of the symmetric allocation can be ordinary allocations on one device, laid out as
PeerReduce.__init__ lays them out: two data buffers of rows_cap x cols bf16, each rounded up to 256 bytes, then the
flag words.  A launch "as rank r at epoch e" finds the flags its peers would have announced (e + 1) already in place,
so it never waits: the data path and every side effect of the flag protocol are checked deterministically, without a
second GPU, torch.distributed or symmetric memory.  The last test runs two live ranks through PeerReduce on two
streams of the same GPU.

The references:
  * residual: bf16(((residual + p_0) + p_1) + ... + p_{w-1}), summed in float32 on the CPU in exactly that order, and
    compared bit for bit -- the fixed order is what makes every rank produce the same bits;
  * out: the float64 norm of that float32 sum times the weight, within the suite's bar (assert_close_bf16).
Every byte the kernel must not write holds a NaN pattern (0xff): the other data buffer, the rows of each buffer past
`rows`, the flag words nobody announces into, and the residual and output rows past `rows` (the kernel gets views into
taller buffers).
"""
import pytest
import torch

from test_gpu_dispatch_edges import (EPS, assert_close_bf16, assert_ran, assert_rows_close, edge_rows, launched,
                                     norm_weight, randn, rmsnorm64)

pytestmark = pytest.mark.gpu

FLAG_BYTES = 256                 # the flag area PeerReduce allocates behind the two data buffers (64 int32 words)
PAD = 2                          # poisoned rows past the last row of every buffer
INT_MAX, INT_MIN = 2 ** 31 - 1, -2 ** 31


def i32(x):
    """x wrapped to int32, as the device counters wrap."""
    return (x + 2 ** 31) % 2 ** 32 - 2 ** 31


def bits(t):
    return t.detach().cpu().contiguous().view(torch.int16)


def assert_bits_equal(got, want, what):
    g, w = bits(got), bits(want)
    bad = (g != w).nonzero()
    assert bad.numel() == 0, f"{what}: {bad.shape[0]} of {g.numel()} elements differ, first at {bad[0].tolist()}"


def poisoned(rows, cols):
    """bf16 NaN with every bit set, the pattern of the 0xff-filled slices."""
    return torch.full((rows, cols), -1, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def assert_poisoned(t, what):
    assert bool((bits(t) == -1).all()), f"{what}: the kernel wrote outside its rows"


class Ranks:
    """`world` emulated slices of a symmetric allocation, each a separate allocation, and every rank's private
    [epoch, done, err] words."""

    def __init__(self, world, rows_cap, cols):
        self.world, self.rows_cap, self.cols = world, rows_cap, cols
        self.buf_bytes = (rows_cap * cols * 2 + 255) // 256 * 256
        self.flag_off = 2 * self.buf_bytes
        self.raw = [torch.full((self.flag_off + FLAG_BYTES,), 0xFF, dtype=torch.uint8, device="cuda") for _ in range(world)]
        self.bases = torch.tensor([t.data_ptr() for t in self.raw], dtype=torch.int64, device="cuda")
        self.state = [torch.zeros(3, dtype=torch.int32, device="cuda") for _ in range(world)]

    def data(self, p, turn):
        a = turn * self.buf_bytes
        return self.raw[p][a:a + self.rows_cap * self.cols * 2].view(torch.bfloat16).view(self.rows_cap, self.cols)

    def flags(self, p):
        """flags_of(p): word q holds the last epoch rank q announced to rank p."""
        return self.raw[p][self.flag_off:].view(torch.int32)

    def load(self, turn, partials):
        """partials[p] into rank p's buffer `turn`; every other data byte of every slice becomes NaN."""
        for p, part in enumerate(partials):
            self.raw[p][:self.flag_off].fill_(0xFF)
            self.data(p, turn)[:part.shape[0]].copy_(part)

    def arm(self, r, ahead=()):
        """state_r = [e, 0, 0] with e the device epoch word as it is now, and flags_of(r)[p] = e + 1 for every peer p
        (e + 2 for the peers in `ahead`): what the peers would have announced.  Returns e."""
        e = int(self.state[r][0])
        self.state[r].copy_(torch.tensor([e, 0, 0], dtype=torch.int32))
        f = self.flags(r)
        for p in range(self.world):
            if p != r:
                f[p] = i32(e + (2 if p in ahead else 1))
        return e

    def launch(self, r, turn, residual, weight, out, rows):
        from nanovllm import _native as nat
        st = self.state[r].data_ptr()
        return nat.load().b200_allreduce_add_rmsnorm(self.bases.data_ptr(), turn * self.buf_bytes, self.flag_off, st, st + 4,
                                                     st + 8, r, self.world, residual.data_ptr(), weight.data_ptr(),
                                                     out.data_ptr(), rows, self.cols, EPS, torch.cuda.current_stream().cuda_stream)

    def snapshot(self):
        return [t.clone() for t in self.raw]

    def assert_launch_effects(self, r, e, before):
        """A launch as rank r at epoch e announced e + 1 into flags_of(p)[r] of every peer p, changed no other byte of any
        slice, advanced the epoch once and left done and err at zero."""
        for p in range(self.world):
            want = before[p].view(torch.int32).clone()
            if p != r:
                want[self.flag_off // 4 + r] = i32(e + 1)
            got = self.raw[p].view(torch.int32)
            bad = (got != want).nonzero().flatten().tolist()
            where = [f"flag {i - self.flag_off // 4}" if i >= self.flag_off // 4 else f"data byte {4 * i}" for i in bad[:4]]
            assert not bad, f"launch as rank {r} at epoch {e}: slice {p} differs at {where} ({len(bad)} words)"
        got = self.state[r].tolist()
        assert got == [i32(e + 1), 0, 0], f"launch as rank {r} at epoch {e}: [epoch, done, err] = {got}"


def rank_order_sum(residual, partials):
    """float32 on the CPU: ((residual + p_0) + p_1) + ... + p_{w-1}."""
    s = residual.float().cpu()
    for p in partials:
        s = s + p.float().cpu()
    return s


def reference(residual, partials, weight):
    s = rank_order_sum(residual, partials)
    return s.to(torch.bfloat16), rmsnorm64(s, weight.cpu())


def padded_weight(cols, seed):
    """Non-unit norm weights as a view into a buffer whose next 8 columns are NaN."""
    buf = torch.full((cols + 8,), float("nan"), dtype=torch.bfloat16, device="cuda")
    buf[:cols] = norm_weight(cols, seed)
    return buf[:cols]


def exchange(fab, r, turn, rows, weight, seed, ahead=(), partials=None, residual=None):
    """One launch as rank r over buffer `turn`, checked against the references and the protocol.  Random partials and
    residual (scale 4) unless given; with more than one row, row rows // 2 is all zero in every input.  Returns
    (epoch the launch ran at, residual, out)."""
    cols = fab.cols
    zero_row = rows // 2 if partials is None and rows > 1 else None
    if partials is None:
        partials = [randn(rows, cols, seed=seed * 16 + p) for p in range(fab.world)]
        residual = randn(rows, cols, seed=seed * 16 + 15, scale=4.0)
        if zero_row is not None:
            for t in (*partials, residual):
                t[zero_row] = 0.0
    fab.load(turn, partials)
    res_buf, out_buf = poisoned(rows + PAD, cols), poisoned(rows + PAD, cols)
    res_buf[:rows] = residual
    e = fab.arm(r, ahead)
    before = fab.snapshot()
    assert fab.launch(r, turn, res_buf[:rows], weight, out_buf[:rows], rows) == 0
    torch.cuda.synchronize()
    what = f"world {fab.world} rank {r} turn {turn} {rows}x{cols}"
    fab.assert_launch_effects(r, e, before)
    want_r, want_y = reference(residual, partials, weight)
    got_r, got_y = res_buf[:rows], out_buf[:rows]
    assert_bits_equal(got_r, want_r, f"{what}: residual vs the rank-order float32 sum")
    assert_close_bf16(got_y.cpu(), want_y, f"{what}: out")
    assert_rows_close(got_y.cpu(), want_y, edge_rows(rows), f"{what}: out")
    if zero_row is not None:
        assert bool((got_y[zero_row] == 0).all()), f"{what}: an all-zero row must normalise to finite zeros"
    assert_poisoned(res_buf[rows:], f"{what}: residual")
    assert_poisoned(out_buf[rows:], f"{what}: out")
    return e, got_r, got_y


# ---------------------------------------------------------------------------------------------------------------------
# 1. the data path: every world size, first / middle / last rank, both data buffers, row lengths around the 1024-column
#    step of the vector loop (8184 and 8192 are its last two), 1 to 1024 rows
# ---------------------------------------------------------------------------------------------------------------------
COLS = [8, 1024, 1032, 2560, 4096, 5120, 8184, 8192]
ROWS = [1, 7, 128, 1024]


@pytest.mark.parametrize("cols", COLS)
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_data_path_matches_reference(world, cols):
    fab = Ranks(world, max(ROWS) + PAD, cols)
    w = padded_weight(cols, seed=cols)
    i = world + COLS.index(cols)
    for r in sorted({0, world // 2, world - 1}):
        for turn in (0, 1):
            exchange(fab, r, turn, ROWS[i % len(ROWS)], w, seed=world * 100003 + cols * 17 + i)
            i += 1


# ---------------------------------------------------------------------------------------------------------------------
# 2. the summation order is observable, and it is the rank order on every rank
# ---------------------------------------------------------------------------------------------------------------------
def test_sum_order_is_rank_order_on_every_rank():
    """Partials of +-2^20 scale that cancel, with small ones between them: float32 keeps only 1/8 steps next to 2^20, so
    the order of the additions shows in the bf16 residual."""
    world, rows, cols, turn = 4, 64, 1024, 1
    g = torch.Generator(device="cuda").manual_seed(7)
    big = (2.0 ** 20 * (1 + torch.rand(rows, cols, generator=g, device="cuda"))
           * torch.where(torch.rand(rows, cols, generator=g, device="cuda") < 0.5, -1.0, 1.0)).to(torch.bfloat16)
    partials = [big, randn(rows, cols, seed=71), -big, randn(rows, cols, seed=72)]
    residual = randn(rows, cols, seed=73)
    want_r = rank_order_sum(residual, partials).to(torch.bfloat16)
    reverse = rank_order_sum(residual, partials[::-1]).to(torch.bfloat16)
    nccl_point = (sum(p.double().cpu() for p in partials).to(torch.bfloat16).float() + residual.float().cpu()).to(torch.bfloat16)
    assert bool((bits(want_r) != bits(reverse)).any()), "the case cannot tell rank order from reverse order"
    assert bool((bits(want_r) != bits(nccl_point)).any()), "the case cannot tell rank order from bf16(sum) + residual"
    fab = Ranks(world, rows + PAD, cols)
    w = padded_weight(cols, seed=3)
    first = None
    for r in range(world):
        _, got_r, got_y = exchange(fab, r, turn, rows, w, seed=0, partials=partials, residual=residual)
        if first is None:
            first = (got_r.clone(), got_y.clone())
        else:
            assert_bits_equal(got_r, first[0], f"rank {r} vs rank 0: residual")
            assert_bits_equal(got_y, first[1], f"rank {r} vs rank 0: out")


# ---------------------------------------------------------------------------------------------------------------------
# 3. one non-zero partial: the exchange reduces to add+RMSNorm, whose block-per-row kernel accumulates in the same order
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cols", [4096, 5120, 8192])
def test_single_partial_equals_add_rmsnorm(cols):
    from nanovllm import ops
    world, rows, turn, r = 4, 33, 1, 1
    x = randn(rows, cols, seed=cols + 1)
    residual = randn(rows, cols, seed=cols + 2, scale=4.0)
    w = padded_weight(cols, seed=cols + 3)
    res_ref = residual.clone()
    (want_y, want_r), names = launched(lambda: ops.add_rmsnorm(x, res_ref, w, EPS))
    assert_ran(names, "rmsnorm_kernel<true>", f"add_rmsnorm {rows}x{cols}")
    fab = Ranks(world, rows + PAD, cols)
    for k in (0, 2):
        partials = [x if p == k else torch.zeros_like(x) for p in range(world)]
        _, got_r, got_y = exchange(fab, r, turn, rows, w, seed=0, partials=partials, residual=residual)
        assert_bits_equal(got_r, want_r, f"x at rank {k}: residual vs add_rmsnorm")
        assert_bits_equal(got_y, want_y, f"x at rank {k}: out vs add_rmsnorm")


# ---------------------------------------------------------------------------------------------------------------------
# 4. the flag protocol's side effects
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 1024, 4096])
def test_protocol_consecutive_launches(rows):
    """Five launches in a row, alternating the data buffers as callers do: each announces once and advances the epoch
    once.  At 4096 rows the grid has more CTAs than can be resident at once, so most CTAs start after others have
    finished and the last CTA to finish is not among the first wave."""
    world, r, cols, n = 4, 2, 1024, 5
    if rows == 4096:
        props = torch.cuda.get_device_properties(0)
        assert rows > props.multi_processor_count * props.max_threads_per_multi_processor // 128
    fab = Ranks(world, rows + PAD, cols)
    w = padded_weight(cols, seed=rows)
    e0 = int(fab.state[r][0])
    for i in range(n):
        e, _, _ = exchange(fab, r, i % 2, rows, w, seed=rows * 8 + i)
        assert e == e0 + i
    assert fab.state[r].tolist() == [e0 + n, 0, 0]


def test_protocol_zero_rows_is_a_no_op():
    world, r, cols = 2, 1, 1024
    fab = Ranks(world, 4, cols)
    w = padded_weight(cols, seed=1)
    e = fab.arm(r)
    before = fab.snapshot()
    res, out = poisoned(4, cols), poisoned(4, cols)
    assert fab.launch(r, 0, res, w, out, 0) == 0
    torch.cuda.synchronize()
    for p in range(world):
        assert torch.equal(fab.raw[p], before[p]), f"slice {p} changed"
    assert fab.state[r].tolist() == [e, 0, 0]
    assert_poisoned(res, "residual")
    assert_poisoned(out, "out")


def test_protocol_peer_ahead_and_epoch_wrap():
    """A peer that has already announced the next epoch does not block; the epoch and the flags wrap from 2^31 - 1 to
    -2^31 and the wait compares across the wrap (the compare is a subtraction, not flag >= e + 1)."""
    world, r, rows, cols = 3, 1, 7, 1032
    fab = Ranks(world, rows + PAD, cols)
    w = padded_weight(cols, seed=2)
    exchange(fab, r, 0, rows, w, seed=1, ahead=(2,))
    fab.state[r][0] = INT_MAX
    e, _, _ = exchange(fab, r, 1, rows, w, seed=2)
    assert e == INT_MAX and fab.state[r].tolist() == [INT_MIN, 0, 0]
    fab.state[r][0] = INT_MAX - 1
    e, _, _ = exchange(fab, r, 0, rows, w, seed=3, ahead=(2,))
    assert e == INT_MAX - 1 and int(fab.flags(r)[2]) == INT_MIN
    assert fab.state[r].tolist() == [INT_MAX, 0, 0]


# ---------------------------------------------------------------------------------------------------------------------
# 5. inside a CUDA graph the epoch lives in device memory, so replays keep counting
# ---------------------------------------------------------------------------------------------------------------------
def test_graph_replays_keep_counting():
    world, r, rows, cols, turn, replays = 4, 3, 64, 2560, 1, 5
    fab = Ranks(world, rows + PAD, cols)
    w = padded_weight(cols, seed=4)
    parts_in = [torch.zeros(rows, cols, dtype=torch.bfloat16, device="cuda") for _ in range(world)]
    res_in = torch.zeros(rows, cols, dtype=torch.bfloat16, device="cuda")
    res_buf, out_buf = poisoned(rows + PAD, cols), poisoned(rows + PAD, cols)
    res, out = res_buf[:rows], out_buf[:rows]
    state, flags = fab.state[r], fab.flags(r)
    peers = torch.tensor([p < world and p != r for p in range(FLAG_BYTES // 4)], device="cuda")
    e0 = int(state[0])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for p in range(world):
            fab.data(p, turn)[:rows].copy_(parts_in[p])
        res.copy_(res_in)
        flags.copy_(torch.where(peers, state[:1] + 1, flags))      # the peers announce the epoch this replay runs at
        code = fab.launch(r, turn, res, w, out, rows)
    assert code == 0
    for i in range(replays):
        partials = [randn(rows, cols, seed=500 + 8 * i + p) for p in range(world)]
        residual = randn(rows, cols, seed=600 + i, scale=4.0)
        for p in range(world):
            parts_in[p].copy_(partials[p])
        res_in.copy_(residual)
        g.replay()
        torch.cuda.synchronize()
        want_r, want_y = reference(residual, partials, w)
        assert_bits_equal(res, want_r, f"replay {i}: residual")
        assert_close_bf16(out.cpu(), want_y, f"replay {i}: out")
        assert state.tolist() == [e0 + i + 1, 0, 0], f"replay {i}: [epoch, done, err] = {state.tolist()}"
        for p in range(world):
            if p != r:
                assert int(fab.flags(p)[r]) == e0 + i + 1
    assert_poisoned(res_buf[rows:], "residual")
    assert_poisoned(out_buf[rows:], "out")


# ---------------------------------------------------------------------------------------------------------------------
# 6. two live ranks on two streams of one GPU, through PeerReduce
# ---------------------------------------------------------------------------------------------------------------------
def peer_reduce_over(fab, rank):
    """A PeerReduce over an emulated slice, with the fields PeerReduce.__init__ sets (no symmetric memory)."""
    from nanovllm.engine.peer_reduce import PeerReduce
    pr = PeerReduce.__new__(PeerReduce)
    pr.rows_cap, pr.hidden, pr.rank, pr.world = fab.rows_cap, fab.cols, rank, fab.world
    pr.buf_bytes, pr.flag_off = fab.buf_bytes, fab.flag_off
    pr.raw = fab.raw[rank]
    pr.handle = None
    pr.bases_dev = fab.bases.data_ptr()
    pr.mc_ptr, pr.nvls = 0, False
    pr.state = fab.state[rank]
    pr.views = [fab.data(rank, i) for i in range(2)]
    pr.turn, pr.calls = 0, 0
    return pr


def test_live_two_ranks_through_peer_reduce():
    """64 exchanges of two ranks that really wait for each other.  Rank 1 sleeps before some of its exchanges, so rank 0
    runs ahead and writes its next partial while rank 1 still reads the previous one: the two alternating buffers must
    keep them apart.  At most 64 rows, so both grids are resident together; if they were not, the bounded wait would
    set err and the test would fail rather than hang."""
    from nanovllm.engine.peer_reduce import PeerExchangeTimeout
    world, cols, rows_cap, n_ex = 2, 1024, 64, 64
    fab = Ranks(world, rows_cap, cols)
    for p in range(world):
        fab.flags(p).zero_()                      # PeerReduce zeroes its slice once
    prs = [peer_reduce_over(fab, r) for r in range(world)]
    w = padded_weight(cols, seed=6)
    rows_of = [(1, 7, 64, 33, 64, 2)[n % 6] for n in range(n_ex)]
    partials = [[randn(rows, cols, seed=1000 + 2 * n + r) for r in range(world)] for n, rows in enumerate(rows_of)]
    residual = [randn(rows, cols, seed=2000 + n, scale=4.0) for n, rows in enumerate(rows_of)]
    res = [[t.clone() for t in residual] for _ in range(world)]
    outs = [[poisoned(rows, cols) for rows in rows_of] for _ in range(world)]
    streams = [torch.cuda.Stream() for _ in range(world)]
    # Every kernel the loop launches runs once before it.  Under lazy module loading the first launch of a kernel can
    # wait for the device to go idle, which it never does while one rank's grid spins waiting for the other: both ranks
    # share this process's context here, unlike ranks on separate GPUs.
    torch.cuda._sleep(1)
    exchange(Ranks(world, 1, cols), 0, 0, 1, w, seed=9)
    torch.cuda.synchronize()
    for n, rows in enumerate(rows_of):
        for r, pr in enumerate(prs):
            with torch.cuda.stream(streams[r]):
                if r == 1 and n % 4 in (1, 2):
                    torch.cuda._sleep(200_000)      # ~0.1 ms of skew
                pr.next_out(rows).copy_(partials[n][r])
                pr.reduce_add_norm(rows, res[r][n], w, EPS, out=outs[r][n])
    torch.cuda.synchronize()
    for r, pr in enumerate(prs):
        assert pr.state.tolist() == [n_ex, 0, 0], f"rank {r}: [epoch, done, err] = {pr.state.tolist()}"
        pr.raise_if_timed_out()
    for n in range(n_ex):
        want_r, want_y = reference(residual[n], partials[n], w)
        for r in range(world):
            assert_bits_equal(res[r][n], want_r, f"exchange {n}, rank {r}: residual")
            assert_close_bf16(outs[r][n].cpu(), want_y, f"exchange {n}, rank {r}: out")
    prs[0].state[2] = 1
    with pytest.raises(PeerExchangeTimeout):
        prs[0].raise_if_timed_out()
