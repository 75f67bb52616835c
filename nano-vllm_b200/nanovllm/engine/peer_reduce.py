"""Symmetric-memory workspace for the fused NVLink all-reduce + add + RMSNorm (csrc/tp_allreduce.cu).

Tensor-parallel decode steps exchange ``[batch, hidden]`` partial sums 2 x layers times per step; those messages
are at most a few hundred KB, so the exchange is latency bound.  Instead of ``dist.all_reduce`` (NCCL) followed by the
add+RMSNorm kernel, the row-parallel GEMM writes its partial straight into this rank's slice of a peer-mapped
allocation and ONE kernel does handshake + peer reads + reduction + residual update + normalisation.

PyTorch provides the plumbing (``torch.distributed._symmetric_memory``: allocation, handle exchange, the device array
of peer base pointers); the kernel and its flag protocol are ours.  If symmetric memory cannot be set up on the box,
``PeerReduce.create`` returns None and the model keeps NCCL.
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist

from .. import _native as nat
from .. import ops


class PeerExchangeTimeout(RuntimeError):
    pass


class PeerReduce:
    def __init__(self, rows_cap: int, hidden: int, rank: int, world: int, device: torch.device):
        import torch.distributed._symmetric_memory as symm
        self.rows_cap, self.hidden, self.rank, self.world = rows_cap, hidden, rank, world
        self.buf_bytes = (rows_cap * hidden * 2 + 255) // 256 * 256
        self.flag_off = 2 * self.buf_bytes
        self.raw = symm.empty(self.flag_off + 256, dtype=torch.uint8, device=device)
        self.raw.zero_()
        torch.cuda.synchronize()
        self.handle = symm.rendezvous(self.raw, dist.group.WORLD)
        self.bases_dev = int(self.handle.buffer_ptrs_dev)
        # Sum inside the NVSwitch (multimem.ld_reduce on the multicast mapping of the same buffer) when there is a multicast
        # mapping: every rank then pulls rows x hidden x 2 bytes per exchange instead of world x that, at the price of a
        # round trip through the switch, which only pays off with several peers, so the default (B200_TP_ALLREDUCE=auto)
        # uses it from 4 ranks up; "peer" / "nvls" force one of the two, "nccl" bypasses this module.
        self.mc_ptr = int(getattr(self.handle, "multicast_ptr", 0) or 0)
        mode = os.environ.get("B200_TP_ALLREDUCE", "auto")
        self.nvls = self.mc_ptr != 0 and (mode == "nvls" or (mode == "auto" and world >= 4))
        self.state = torch.zeros(3, dtype=torch.int32, device=device)           # [epoch, done counter, error flag]
        self.views = [self.raw[i * self.buf_bytes:i * self.buf_bytes + rows_cap * hidden * 2].view(torch.bfloat16).view(rows_cap, hidden)
                      for i in range(2)]
        self.turn = 0
        self.calls = 0
        torch.cuda.synchronize()                      # the caller's agreement all-reduce is the cross-rank barrier

    @staticmethod
    def _all_agree(ok: bool, device) -> bool:
        flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)              # also a barrier
        return int(flag.item()) == 1

    @classmethod
    def create(cls, rows_cap, hidden, rank, world, device):
        """The workspace, or None -- decided unanimously -- when peer memory cannot be set up or fails its self-test."""
        if os.environ.get("B200_TP_ALLREDUCE", "auto") not in ("auto", "peer", "nvls"):
            return None
        obj, why = None, ""
        try:
            obj = cls(rows_cap, hidden, rank, world, device)
        except Exception as e:                       # no P2P / fabric handles on this box, ...
            why = f"{type(e).__name__}: {e}"
        if not cls._all_agree(obj is not None, device):          # some rank could not map its peers: nobody uses it
            if rank == 0:
                print(f"[nanovllm] peer-memory all-reduce unavailable ({why or 'set-up failed on another rank'}); using NCCL", flush=True)
            return None
        try:
            ok = obj.self_test()
        except Exception as e:
            ok, why = False, f"{type(e).__name__}: {e}"
        if not cls._all_agree(ok, device):
            if rank == 0:
                print(f"[nanovllm] peer-memory all-reduce failed its self-test ({why or 'mismatch or timeout'}); using NCCL", flush=True)
            return None
        return obj

    def self_test(self, rounds: int = 4, rows: int = 8) -> bool:
        """A few real exchanges checked against an NCCL all-reduce of the same data; also trips the kernel's
        wait timeout (error flag) instead of hanging if a peer is unreachable."""
        gen = torch.Generator(device="cpu").manual_seed(1234 + self.rank)
        weight = torch.ones(self.hidden, dtype=torch.bfloat16, device=self.raw.device)
        good = True
        for _ in range(rounds):
            part = torch.randn(rows, self.hidden, generator=gen).to(torch.bfloat16).to(self.raw.device)
            self.next_out(rows).copy_(part)
            residual = torch.zeros(rows, self.hidden, dtype=torch.bfloat16, device=self.raw.device)
            _, got = self.reduce_add_norm(rows, residual, weight, 1e-6)
            want = part.float()
            dist.all_reduce(want)
            torch.cuda.synchronize()
            # never leave the loop early: every rank must issue the same collectives whatever it observes
            timed_out = int(self.state[2].item()) != 0
            err = (got.float() - want).abs().max().item()
            good = good and not timed_out and err <= 2.0 ** -7 * max(want.abs().max().item(), 1.0)   # one bf16 rounding
        return good

    def raise_if_timed_out(self) -> None:
        """The kernel gives up (error flag, undefined output) rather than spin forever when a peer never announces
        its epoch; callers check after each batch of work so that such a run fails loudly instead of returning junk."""
        if int(self.state[2].item()) != 0:
            raise PeerExchangeTimeout("tensor-parallel peer exchange timed out (a rank stopped or fell >10 s behind); "
                                      "results of this call are invalid -- rerun with B200_TP_ALLREDUCE=nccl to bypass")

    def next_out(self, rows: int) -> torch.Tensor:
        """Where the row-parallel GEMM of the next exchange must write its partial (the two buffers alternate)."""
        self.turn ^= 1
        return self.views[self.turn][:rows]

    def reduce_add_norm(self, rows: int, residual: torch.Tensor, weight: torch.Tensor, eps: float, out: torch.Tensor | None = None):
        """residual <- bf16(residual + sum over ranks of the partials in the current buffer); returns (normed, residual)."""
        if out is None:
            out = torch.empty_like(residual)
        lib = nat.load()
        if self.nvls:
            nat.check(lib.b200_allreduce_add_rmsnorm_nvls(self.bases_dev, self.mc_ptr, self.turn * self.buf_bytes, self.flag_off,
                                                          self.state.data_ptr(), self.state.data_ptr() + 4, self.state.data_ptr() + 8,
                                                          self.rank, self.world, residual.data_ptr(), weight.data_ptr(), out.data_ptr(),
                                                          rows, self.hidden, eps, ops._stream()))
            self.calls += 1
            return out, residual
        nat.check(lib.b200_allreduce_add_rmsnorm(self.bases_dev, self.turn * self.buf_bytes, self.flag_off,
                                                 self.state.data_ptr(), self.state.data_ptr() + 4, self.state.data_ptr() + 8,
                                                 self.rank, self.world, residual.data_ptr(), weight.data_ptr(), out.data_ptr(),
                                                 rows, self.hidden, eps, ops._stream()))
        self.calls += 1
        return out, residual
