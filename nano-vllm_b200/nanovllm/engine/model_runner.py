"""Per-GPU executor: device setup, KV-cache sizing/binding, step marshalling, CUDA graphs, sampling.

Same contract as the reference's ModelRunner (nanovllm/engine/model_runner.py:15-257):
``ModelRunner(config, rank, event)`` sets ``config.num_kvcache_blocks``; ``call("run", seqs,
is_prefill) -> list[int]`` returns one token id per sequence; one process per GPU, one thread,
everything on the current stream, one device->host sync per step.

Differences from the reference (DESIGN.md "runner"):
* per-step metadata travels in ONE pinned staging buffer (two of them, ping-pong, so step N+1 can be staged
  while step N runs) and ONE host->device copy into static device buffers (the reference builds seven pinned
  tensors and seven copies per step);
* launch() / collect() split a step into "enqueue everything" and "wait for its tokens"; up to two steps are in
  flight, a decode step's input ids are gathered on the device from the previous step's samples;
* the decode graph contains the whole step: embedding ... final norm, LM head, sampling and (under
  tensor parallelism) the all-reduces; the reference leaves logits and sampling outside;
* tensor-parallel ranks are SPMD replicas: every rank runs the same (deterministic) scheduler and
  this runner in lock-step, so there is no per-step RPC (the reference pickles the batch into shared
  memory every step, model_runner.py:61-89); ranks agree on the sampled tokens through the
  all-reduce(MAX) of packed (score, token) keys that replaces the reference's logits gather.
"""
from __future__ import annotations

import os
from collections import deque
from time import perf_counter

import numpy as np
import torch
import torch.distributed as dist

from .. import _native as nat
from .. import ops
from ..config import KV_CACHE_DTYPES, Config
from ..layers.attention import KVGroup, kv_group_arrays, plan_kv_groups
from ..models.qwen3_moe import model_class
from ..utils.context import reset_context, set_context
from ..utils.loader import load_model
from .sequence import Sequence, SequenceStatus

_ALIGN = 64


def _align(n: int) -> int:
    return (n + _ALIGN - 1) // _ALIGN * _ALIGN


class _Staging:
    """Pinned host byte buffers (ping-pong) mirrored by one device byte buffer; regions are typed views."""

    def __init__(self, nbytes: int, hosts: int = 1):
        self.hosts = [torch.empty(nbytes, dtype=torch.uint8, pin_memory=True) for _ in range(hosts)]
        self.dev = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        self.host_nps = [h.numpy() for h in self.hosts]

    def host_view(self, off: int, count: int, np_dtype, which: int = 0):
        nbytes = count * np.dtype(np_dtype).itemsize
        return self.host_nps[which][off:off + nbytes].view(np_dtype)

    def dev_view(self, off: int, count: int, np_dtype, torch_dtype):
        nbytes = count * np.dtype(np_dtype).itemsize
        return self.dev[off:off + nbytes].view(torch_dtype)

    def views(self, off: int, count: int, np_dtype, torch_dtype, which: int = 0):
        return self.host_view(off, count, np_dtype, which), self.dev_view(off, count, np_dtype, torch_dtype)

    def upload(self, nbytes: int, which: int = 0):
        self.dev[:nbytes].copy_(self.hosts[which][:nbytes], non_blocking=True)


class ModelRunner:
    def __init__(self, config: Config, rank: int = 0, event=None, sample_seed: int | None = None):
        self.config = config
        hf = config.hf_config
        self.block_size = config.kvcache_block_size
        self.kv_fp8 = KV_CACHE_DTYPES[config.kv_cache_dtype]
        # fp8 cache: rows of the bf16 scratch a paged prefill dequantizes keys / values into (one step's new tokens plus
        # the longest context fit, so one sequence always does; a step that needs more is cut into groups)
        self.kv_scratch_rows = config.max_num_batched_tokens + config.max_model_len
        self.kv_scratch = None
        self.enforce_eager = config.enforce_eager
        self.world_size = config.tensor_parallel_size
        self.rank = rank
        self.event = event
        self.sample_seed = sample_seed
        self.sample_step = 0
        self._prof = None
        self.graph_kernels: dict[int, int] = {}

        if not torch.cuda.is_available():
            raise nat.B200Error("ModelRunner needs a CUDA device: the GPU path has no CPU fallback")
        local = int(os.environ.get("LOCAL_RANK", rank))
        # Debug / CI knob: B200_TP_BACKEND=gloo with B200_TP_ONE_DEVICE=1 runs all tensor-parallel ranks on ONE GPU
        # (time-sliced processes, collectives through gloo, eager only): the sharding, the vocab-parallel sampling and
        # the SPMD engine can then be checked on a single-GPU box.  Never the fast path: NCCL is the default.
        backend = os.environ.get("B200_TP_BACKEND", "nccl")
        if os.environ.get("B200_TP_ONE_DEVICE") == "1":
            local = 0
        torch.cuda.set_device(local)
        self.device = torch.device("cuda", local)
        self._own_pg = False
        if self.world_size > 1 and not dist.is_initialized():
            addr = os.environ.get("MASTER_ADDR", "127.0.0.1")
            port = os.environ.get("MASTER_PORT", "2333")
            kw = dict(device_id=self.device) if backend == "nccl" else {}
            dist.init_process_group(backend, init_method=f"tcp://{addr}:{port}", world_size=self.world_size, rank=rank, **kw)
            self._own_pg = True
        if self.world_size > 1 and dist.get_backend() != "nccl" and not config.enforce_eager:
            raise ValueError("CUDA graphs need the NCCL backend (gloo collectives cannot be captured): pass enforce_eager=True")
        if self.world_size > 1:
            assert dist.get_world_size() == self.world_size, "tensor_parallel_size must equal the process-group size"
        self.native = nat.handle(local)
        # Sampling randomness: a fresh 63-bit seed per engine unless one is given (B200_SAMPLE_SEED or the argument);
        # every tensor-parallel rank must use the same one (each scores its own vocabulary shard with the RNG keyed by
        # the global token id), so rank 0's choice is broadcast.
        if sample_seed is None and os.environ.get("B200_SAMPLE_SEED"):
            sample_seed = int(os.environ["B200_SAMPLE_SEED"])
        if sample_seed is None:
            sample_seed = int.from_bytes(os.urandom(8), "little") >> 1
        if self.world_size > 1:
            t = torch.tensor([sample_seed], dtype=torch.int64, device=self.device)
            dist.broadcast(t, src=0)
            sample_seed = int(t.item())
        self.sample_seed = sample_seed

        self.model = model_class(hf)(hf, rank, self.world_size, self.device, max_position=hf.max_position_embeddings)
        load_model(self.model, config.model, allow_random=bool(os.environ.get("NANOVLLM_ALLOW_RANDOM_INIT")))
        self.vocab_offset = rank * self.model.vocab_shard
        if self.world_size > 1:
            from .peer_reduce import PeerReduce
            self.model.peer = PeerReduce.create(min(config.max_num_seqs, 1024), hf.hidden_size, rank, self.world_size, self.device)

        if config.max_num_seqs > 1024:
            raise ValueError("max_num_seqs > 1024 is not supported by the decode kernel's per-launch batch table")
        self.cap_bs = config.max_num_seqs                    # rows of the static decode buffers
        self.max_bs = min(config.max_num_seqs, 512)          # largest captured graph (model_runner.py:226)
        self.max_blocks = (config.max_model_len + self.block_size - 1) // self.block_size
        self._init_staging()
        self.warmup_model()
        self.allocate_kv_cache()
        self.allocate_penalty_history()
        self.graphs: dict[int, torch.cuda.CUDAGraph] = {}
        self.graph_bs: list[int] = []
        self.graph_pool = None
        if not self.enforce_eager:
            self.capture_cudagraph()

    def check_peer_exchange(self) -> None:
        """Raise if the fused NVLink all-reduce hit its wait timeout since the last check (peer_reduce.py)."""
        peer = getattr(self.model, "peer", None)
        if peer is not None:
            peer.raise_if_timed_out()

    # ---- measurement hooks (bench.py) ----------------------------------------------------------
    def begin_profile(self):
        """Record a CUDA-event pair around every step's GPU work until end_profile()."""
        self._prof = dict(events=[], h2d=0, d2h=0, steps=0, launches0=ops.LAUNCHES[0])

    def end_profile(self) -> dict:
        torch.cuda.synchronize()
        p, self._prof = self._prof, None
        return dict(device_ms=sum(a.elapsed_time(b) for a, b in p["events"]), h2d_bytes=p["h2d"], d2h_bytes=p["d2h"],
                    engine_steps=p["steps"], kernel_launches=ops.LAUNCHES[0] - p["launches0"])

    # ---- reference-compatible dispatch (model_runner.py:85-89) ------------------------------
    def call(self, method_name: str, *args):
        return getattr(self, method_name)(*args)

    def exit(self):
        self.graphs.clear()
        self.fgraphs.clear()
        self.lgraphs.clear()
        self.graph_pool = None
        torch.cuda.synchronize()
        if self._own_pg and dist.is_initialized():
            dist.destroy_process_group()

    # ---- staging layout -----------------------------------------------------------------------
    def _init_staging(self):
        cfg = self.config
        T = max(cfg.max_num_batched_tokens, self.cap_bs)
        S = self.cap_bs
        W = self.max_blocks
        # decode region: static offsets (they are baked into the CUDA graphs)
        o = 0
        self.d_off = {}
        mb = self.cap_bs
        for name, count, size in (("step", 1, 8), ("ids", mb, 8), ("pos", mb, 8), ("slot", mb, 4), ("ctx", mb, 4),
                                  ("temp", mb, 4), ("src", mb, 4), ("bt", mb * W, 4)):
            self.d_off[name] = o
            o = _align(o + count * size)
        self.d_bytes = o
        self.stage = _Staging(self.d_bytes, hosts=2)         # ping-pong: step N+1 is staged while step N runs
        self.pstage = _Staging(self.prefill_staging_bytes(T, S, W, self.kv_fp8))
        st = self.stage
        spec = (("step", 1, np.int64, torch.int64), ("ids", mb, np.int64, torch.int64), ("pos", mb, np.int64, torch.int64),
                ("slot", mb, np.int32, torch.int32), ("ctx", mb, np.int32, torch.int32), ("temp", mb, np.float32, torch.float32),
                ("src", mb, np.int32, torch.int32), ("bt", mb * W, np.int32, torch.int32))
        self.hd = [{name: st.host_view(self.d_off[name], cnt, npdt, k) for name, cnt, npdt, _ in spec} for k in range(2)]
        for h in self.hd:
            h["bt"] = h["bt"].reshape(mb, W)
            h["bt"][:] = 0
        g = {name: st.dev_view(self.d_off[name], cnt, npdt, tdt) for name, cnt, npdt, tdt in spec}
        self.g_step, self.g_ids, self.g_pos, self.g_slot = g["step"], g["ids"], g["pos"], g["slot"]
        self.g_ctx, self.g_temp, self.g_bt, self.g_src = g["ctx"], g["temp"], g["bt"].view(mb, W), g["src"]
        self.g_bt.zero_()
        self._host_k = 0
        self.g_tokens = torch.zeros(S, dtype=torch.int64, device="cuda")
        self.g_keys = torch.zeros(S, dtype=torch.int64, device="cuda")
        self.g_keyws = torch.zeros(S, dtype=torch.int64, device="cuda")      # running-max keys of the fused LM head (zero between steps)
        self.fused_lm_head = os.environ.get("B200_LM_HEAD", "gemm") == "fused"
        self.h_tokens = [torch.empty(S, dtype=torch.int64, pin_memory=True) for _ in range(2)]
        self.h_err = [torch.zeros(1, dtype=torch.int32, pin_memory=True) for _ in range(2)]   # peer-exchange error flag per step
        self.h_tokens_np = [t.numpy() for t in self.h_tokens]
        self.h2d_bytes_last = 0
        self.d2h_bytes_last = 0
        self._done = [torch.cuda.Event(), torch.cuda.Event()]
        self._launches = 0
        self._pending: deque = deque()            # (read-back buffer, rows) of steps launched but not collected
        # top-k / top-p / min-p and the penalties: per-row parameters in their own small ping-pong staging (same index as
        # the decode staging, uploaded only on a step where some row filters or penalises) and the filtered sampler's
        # workspace, sized for cap_bs rows
        # (plslot / ploff: the rows that reload their history slot in this step, and their entry-list offsets)
        fspec = (("topk", mb, np.int32, torch.int32), ("topp", mb, np.float32, torch.float32),
                 ("minp", mb, np.float32, torch.float32), ("pslot", mb, np.int32, torch.int32),
                 ("prep", mb, np.float32, torch.float32), ("pfreq", mb, np.float32, torch.float32),
                 ("ppres", mb, np.float32, torch.float32), ("plslot", mb, np.int32, torch.int32),
                 ("ploff", mb + 1, np.int32, torch.int32), ("lpk", mb, np.int32, torch.int32))
        self.f_off = {}
        o = 0
        for name, cnt, _, _ in fspec:
            self.f_off[name] = o
            o = _align(o + cnt * 4)
        self.f_bytes = o
        self.fstage = _Staging(self.f_bytes, hosts=2)
        self.hf = [{name: self.fstage.host_view(self.f_off[name], cnt, npdt, k) for name, cnt, npdt, _ in fspec}
                   for k in range(2)]
        for h in self.hf:
            h["pslot"][:] = -1
            h["lpk"][:] = -1
        self.f_any = [False, False]
        self.lp_any = [False, False]              # whether the step staged in buffer k has a logprob row
        self.p_load: list = [None, None]          # (entries, rows) of a decode step that reloads slots, per staging buffer
        gf = {name: self.fstage.dev_view(self.f_off[name], cnt, npdt, tdt) for name, cnt, npdt, tdt in fspec}
        self.g_topk, self.g_topp, self.g_minp = gf["topk"], gf["topp"], gf["minp"]
        self.g_pslot, self.g_prep, self.g_pfreq, self.g_ppres = gf["pslot"], gf["prep"], gf["pfreq"], gf["ppres"]
        self.g_plslot, self.g_ploff = gf["plslot"], gf["ploff"]
        self.g_lpk = gf["lpk"]
        self.g_lpk.fill_(-1)
        self.g_topk.zero_()
        self.g_topp.fill_(1.0)
        self.g_minp.zero_()
        self.g_pslot.fill_(-1)
        self.g_prep.fill_(1.0)
        self.g_pfreq.zero_()
        self.g_ppres.zero_()
        self.g_filter_ws = ops.filter_workspace(self.cap_bs)
        self.step_filters = None                  # the filter tensors of the step being launched (None: plain sampler)
        self.step_penalties = None                # its penalty tensors (slot, r, f, p, pending token), or None
        self.fgraphs: dict[int, torch.cuda.CUDAGraph] = {}
        self.fgraph_kernels: dict[int, int] = {}
        self._init_penalty_slots(self.cap_bs)
        # logprobs (DESIGN.md 3.3.2): the per-row k rides in the filter staging (-1 = off); workspace, top-k keys, the
        # packed result rows and the saved raw logits live on the device (allocate_penalty_history, after the KV cache is
        # sized), a pinned ping-pong copy of the result per read-back buffer, and a third graph set replayed only on a step
        # with a logprob row
        self.g_lp_ws = self.g_lp_keys = self.g_lp_out = self.g_lp_saved = None
        self.h_lp = [torch.zeros(S, ops.LOGPROB_OUT_WORDS, dtype=torch.int32, pin_memory=True) for _ in range(2)]
        self.h_lp_np = [t.numpy() for t in self.h_lp]
        self.step_logprobs = None                 # the k tensor of the step being launched, or None
        self.last_logprobs = None                 # packed result rows of the last collected step, or None
        self.lgraphs: dict[int, torch.cuda.CUDAGraph] = {}
        self.lgraph_kernels: dict[int, int] = {}

    @staticmethod
    def prefill_staging_bytes(T: int, S: int, W: int, kv_fp8: bool) -> int:
        """Bytes of the prefill staging buffer: room for prepare_prefill's plan at its limits, T new tokens of S sequences
        with block tables W wide, every optional region staged."""
        n = _align(8) + 2 * _align(T * 8) + _align(T * 4) + 2 * _align((S + 1) * 4) + _align(S * 4) + _align(S * W * 4)
        if kv_fp8:                                           # the rebased cu_seqlens_q/k of at most S gather groups
            n += 2 * (8 * S + _ALIGN * S)
        n += 3 * _align(S * 4)                               # top_k / top_p / min_p of a step where some request filters
        n += 4 * _align(S * 4) + _align((S + 1) * 4)         # penalty slot / r / f / p and entry-list offsets
        n += _align(S * 4)                                   # per-row logprobs k of a step where some request wants them
        return n

    # ---- presence / frequency / repetition penalties (DESIGN.md 3.3.1) ------------------------------------------------
    def _init_penalty_slots(self, num_slots: int):
        """Host side of the history pool: which sequence holds which slot.  The device pool itself is allocated after the
        KV cache (allocate_penalty_history), so that it does not change the cache's size."""
        self.pen_num_slots = num_slots
        self.pen_free = list(range(num_slots - 1, -1, -1))     # pop() hands out slot 0 first
        self.pen_slot: dict[int, int] = {}                     # seq_id -> slot
        self.pen_held: dict[int, Sequence] = {}                # seq_id -> the sequence holding it
        self.pen_used: dict[int, int] = {}                     # seq_id -> last staging that needed its slot
        self.pen_tick = 0
        self.pen_stats = dict(loads=0, evictions=0)
        self.pen_hist = self.pen_len = None
        # entry lists of the loading rows: pinned buffers 0 / 1 for the two decode stagings, 2 for a prefill; one device copy
        self.pen_ent_host: list = [None, None, None]
        self.pen_ent_dev = None

    @staticmethod
    def penalty_pool_shape(config: Config) -> tuple[int, int]:
        """(slots, entries per slot) of the history pool: one slot per row of a step, min(max_model_len, vocab) entries.
        The running set may outgrow max_num_seqs (admission is bounded by the KV cache, not by it); slots then act as a
        cache (penalty_arrays), so the pool's size never depends on the number of KV-cache blocks."""
        return config.max_num_seqs, min(config.max_model_len, config.hf_config.vocab_size)

    def allocate_penalty_history(self):
        """The penalty history pool, and the logprob kernels' device buffers (their saved-logits buffer has a slot's
        capacity plus one entry per row), all sized after the KV cache."""
        slots, capacity = self.penalty_pool_shape(self.config)
        self._init_penalty_slots(slots)
        self.pen_hist, self.pen_len = ops.penalty_history(slots, capacity)
        S = self.cap_bs
        self.g_lp_ws = ops.logprob_workspace(S)
        self.g_lp_keys = torch.zeros(S * ops.LOGPROB_MAX_K, dtype=torch.int64, device="cuda")
        self.g_lp_out = torch.zeros(S, ops.LOGPROB_OUT_WORDS, dtype=torch.int32, device="cuda")
        self.g_lp_saved = ops.logprob_saved_buffer(S, capacity)

    @staticmethod
    def penalty_entries(seq: Sequence, num_tokens: int | None = None) -> np.ndarray:
        """The history entries of the first `num_tokens` tokens of a sequence (all by default): one int64 per distinct
        token, token << 32 | in_prompt << 31 | the number of times it occurs after the prompt."""
        toks = np.asarray(seq.token_ids[:num_tokens], dtype=np.int64)
        uniq = np.unique(toks)
        in_prompt = np.isin(uniq, toks[:seq.num_prompt_tokens])
        gen, counts = np.unique(toks[seq.num_prompt_tokens:], return_counts=True)
        c = np.zeros(uniq.size, np.int64)
        c[np.searchsorted(uniq, gen)] = counts
        return (uniq << 32) | (in_prompt.astype(np.int64) << 31) | c

    def release_penalty_slots(self):
        """Give back the slots of sequences that finished, were preempted or were aborted.  Called when a step is staged;
        a released slot is reloaded only by a later step, after every step still using it in stream order."""
        for sid, s in list(self.pen_held.items()):
            if s.status is not SequenceStatus.RUNNING:
                self.pen_free.append(self.pen_slot.pop(sid))
                del self.pen_held[sid], self.pen_used[sid]

    def _acquire_penalty_slot(self, seq: Sequence, batch: set) -> int:
        """A free slot, else the one of the least recently used holder outside this step's batch.  A step has at most
        max_num_seqs rows, as many as there are slots, so such a holder exists.  The evicted sequence's history is rebuilt
        from its host tokens when it next needs a slot; a step still in flight that uses the slot runs before the reload
        in stream order."""
        if self.pen_free:
            s = self.pen_free.pop()
        else:
            out = [sid for sid in self.pen_held if sid not in batch]
            if not out:
                raise RuntimeError(f"a step with more penalised rows than the {self.pen_num_slots} history slots")
            victim = min(out, key=self.pen_used.__getitem__)
            s = self.pen_slot.pop(victim)
            del self.pen_held[victim], self.pen_used[victim]
            self.pen_stats["evictions"] += 1
        self.pen_slot[seq.seq_id] = s
        self.pen_held[seq.seq_id] = seq
        return s

    def penalty_arrays(self, seqs: list[Sequence], padded: int | None = None, prefill: bool = False):
        """Per-row slot (int32), repetition, frequency and presence penalty (fp32) and whether the row (re)loads its slot
        (bool), for a step over `padded` rows; None when no row penalises.  A prefill loads the slot of a penalised
        sequence whose prompt ends in this step (the step that samples for it) with all its tokens; a decode step gives a
        slot to a penalised sequence that holds none (its slot was taken while it sat outside the batch) and loads every
        token but the last, its input id, which the apply kernel absorbs.  Rows of earlier chunks, unpenalised rows and
        padding carry slot -1."""
        if not any(s.penalised for s in seqs):
            return None
        n = len(seqs)
        padded = n if padded is None else padded
        slot = np.full(padded, -1, np.int32)
        r = np.ones(padded, np.float32)
        f = np.zeros(padded, np.float32)
        p = np.zeros(padded, np.float32)
        load = np.zeros(padded, bool)
        self.pen_tick += 1
        batch = {s.seq_id for s in seqs}
        for i, s in enumerate(seqs):
            if not s.penalised:
                continue
            if prefill and s.num_cached_tokens + s.num_scheduled_tokens < s.num_tokens:
                continue
            load[i] = prefill or s.seq_id not in self.pen_slot
            slot[i] = self.pen_slot[s.seq_id] if s.seq_id in self.pen_slot else self._acquire_penalty_slot(s, batch)
            self.pen_used[s.seq_id] = self.pen_tick
            r[i], f[i], p[i] = s.repetition_penalty, s.frequency_penalty, s.presence_penalty
        if prefill and not (slot >= 0).any():
            return None
        return slot, r, f, p, load

    def _stage_penalty_entries(self, seqs: list[Sequence], load: np.ndarray, which: int, prefill: bool):
        """Entry lists of the loading rows into pinned buffer `which` (grown geometrically); returns (offsets, entries)."""
        lists = [self.penalty_entries(s, None if prefill else s.num_tokens - 1) if load[i] else np.zeros(0, np.int64)
                 for i, s in enumerate(seqs)]
        offsets = np.zeros(len(seqs) + 1, np.int32)
        np.cumsum([e.size for e in lists], out=offsets[1:])
        total = int(offsets[-1])
        host = self.pen_ent_host[which]
        if host is None or host.numel() < total:
            host = self.pen_ent_host[which] = torch.empty(max(total, 4096, 0 if host is None else 2 * host.numel()),
                                                          dtype=torch.int64, pin_memory=True)
        if self.pen_ent_dev is None or self.pen_ent_dev.numel() < total:
            self.pen_ent_dev = torch.empty(host.numel(), dtype=torch.int64, device="cuda")
        if total:
            host.numpy()[:total] = np.concatenate(lists)
        self.pen_stats["loads"] += int(load.sum())
        return offsets, total

    def _load_penalty_slots(self, which: int, total: int, offsets: torch.Tensor, slots: torch.Tensor) -> None:
        """Copy pinned entry buffer `which` to the device and load the slots of the rows with slots[r] >= 0."""
        self.pen_ent_dev[:total].copy_(self.pen_ent_host[which][:total], non_blocking=True)
        self.h2d_bytes_last += total * 8
        ops.penalty_load(self.pen_hist, self.pen_len, self.pen_ent_dev, offsets, slots)

    # ---- init-time passes -----------------------------------------------------------------------
    def warmup_model(self):
        """One maximum-size prefill without a cache, to find the activation peak (model_runner.py:91-101)."""
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        cfg = self.config
        seq_len = min(cfg.max_num_batched_tokens, cfg.max_model_len)
        num_seqs = min(cfg.max_num_batched_tokens // seq_len, cfg.max_num_seqs)
        seqs = [Sequence([0] * seq_len) for _ in range(num_seqs)]
        for s in seqs:
            s.num_scheduled_tokens = seq_len
        self.run(seqs, True)
        torch.cuda.empty_cache()

    def kv_block_bytes(self) -> int:
        hf = self.config.hf_config
        elem = 1 if self.kv_fp8 else 2
        return 2 * hf.num_hidden_layers * self.block_size * self.model.num_kv_heads * self.model.head_dim * elem

    def kv_scratch_bytes(self) -> int:
        """The fp8 cache's dequantization scratch (K and V, bf16); 0 for a bf16 cache."""
        return 2 * self.kv_scratch_rows * self.model.num_kv_heads * self.model.head_dim * 2 if self.kv_fp8 else 0

    def allocate_kv_cache(self):
        """Size the cache from free memory with the reference's formula (model_runner.py:103-113), allocate
        it head-major, bind it to the library and hand each attention operator its layer views (116-121)."""
        cfg = self.config
        hf = cfg.hf_config
        if cfg.num_kvcache_blocks is None or cfg.num_kvcache_blocks <= 0:
            free, total = torch.cuda.mem_get_info()
            used = total - free
            stats = torch.cuda.memory_stats()
            peak, current = stats["allocated_bytes.all.peak"], stats["allocated_bytes.all.current"]
            nblk = int(total * cfg.gpu_memory_utilization - used - peak + current - self.kv_scratch_bytes()) // self.kv_block_bytes()
            if self.world_size > 1:                      # replicas must agree on the block count
                t = torch.tensor([nblk], dtype=torch.int64, device="cuda")
                dist.all_reduce(t, op=dist.ReduceOp.MIN)
                nblk = int(t.item())
            cfg.num_kvcache_blocks = nblk
        if cfg.num_kvcache_blocks <= 0:
            raise RuntimeError("not enough GPU memory for a single KV-cache block")
        m = self.model
        shape = ops.kv_cache_shape(hf.num_hidden_layers, cfg.num_kvcache_blocks, m.num_kv_heads, self.block_size, m.head_dim)
        self.kv_scratch = None
        if self.kv_fp8:
            self.kv_cache = torch.zeros(shape, dtype=torch.uint8, device="cuda").view(torch.float8_e4m3fn)
            self.kv_scratch = torch.empty(2, self.kv_scratch_rows, m.num_kv_heads, m.head_dim, dtype=torch.bfloat16, device="cuda")
            m.fused_decode_max_batch = 0             # the fused decode front end has no quantized KV append
        else:
            self.kv_cache = torch.zeros(shape, dtype=torch.bfloat16, device="cuda")
        ops.bind_kv_cache(self.kv_cache)
        ops.ensure_workspace(self.cap_bs, m.num_heads)
        layer_id = 0
        for module in m.modules():
            if hasattr(module, "k_cache") and hasattr(module, "v_cache"):
                module.k_cache = self.kv_cache[0, layer_id]
                module.v_cache = self.kv_cache[1, layer_id]
                module.layer_id = layer_id
                module.kv_scratch = self.kv_scratch
                layer_id += 1

    # ---- step marshalling (host integer work; must match the reference bit for bit) ------------
    def prepare_block_tables(self, seqs: list[Sequence]) -> np.ndarray:
        """[len(seqs), max blocks in batch] int32, right-padded with -1 (model_runner.py:123-127)."""
        width = max(len(s.block_table) for s in seqs)
        bt = np.full((len(seqs), width), -1, dtype=np.int32)
        for i, s in enumerate(seqs):
            bt[i, :len(s.block_table)] = s.block_table
        return bt

    def prefill_arrays(self, seqs: list[Sequence]) -> dict:
        """Host arrays of a prefill step (model_runner.py:129-170): the scheduled token window of each
        sequence, its positions, cumulative q/k lengths, one cache slot per new token, and block tables
        only when some K/V comes from the cache (prefix hit or a later prompt chunk)."""
        bs = self.block_size
        ids, pos, slots = [], [], []
        cu_q, cu_k = [0], [0]
        max_q = max_k = 0
        for s in seqs:
            start = s.num_cached_tokens
            end = start + s.num_scheduled_tokens
            ids.append(np.asarray(s.token_ids[start:end], dtype=np.int64))
            p = np.arange(start, end, dtype=np.int64)
            pos.append(p)
            cu_q.append(cu_q[-1] + (end - start))
            cu_k.append(cu_k[-1] + end)
            max_q, max_k = max(max_q, end - start), max(max_k, end)
            if s.block_table:                                # absent only in the warm-up pass
                table = np.asarray(s.block_table, dtype=np.int64)
                slots.append((table[p // bs] * bs + p % bs).astype(np.int32))
        out = dict(input_ids=np.concatenate(ids) if ids else np.zeros(0, np.int64),
                   positions=np.concatenate(pos) if pos else np.zeros(0, np.int64),
                   cu_seqlens_q=np.asarray(cu_q, dtype=np.int32), cu_seqlens_k=np.asarray(cu_k, dtype=np.int32),
                   max_seqlen_q=max_q, max_seqlen_k=max_k,
                   slot_mapping=np.concatenate(slots) if slots else np.zeros(0, np.int32), block_tables=None)
        if cu_k[-1] > cu_q[-1]:
            out["block_tables"] = self.prepare_block_tables(seqs)
        return out

    def decode_arrays(self, seqs: list[Sequence]) -> dict:
        """Host arrays of a decode step (model_runner.py:172-188)."""
        bs = self.block_size
        n = len(seqs)
        ids = np.fromiter((s.last_token for s in seqs), dtype=np.int64, count=n)
        lens = np.fromiter((s.num_tokens for s in seqs), dtype=np.int64, count=n)
        last_blk = np.fromiter((s.block_table[-1] for s in seqs), dtype=np.int64, count=n)
        # last_block_num_tokens = len - (num_blocks - 1) * bs, so the slot of the newest token is:
        slots = last_blk * bs + (lens - 1) % bs
        return dict(input_ids=ids, positions=lens - 1, slot_mapping=slots.astype(np.int32),
                    context_lens=lens.astype(np.int32), block_tables=self.prepare_block_tables(seqs))

    def filter_arrays(self, seqs: list[Sequence], padded: int | None = None):
        """Per-row top_k (int32), top_p and min_p (fp32) of a step over `padded` rows, or None when no row filters.
        Greedy rows and graph-padding rows carry "off" (0, 1.0, 0.0)."""
        if not any(s.temperature > 0 and (s.top_k > 0 or s.top_p < 1.0 or s.min_p > 0.0) for s in seqs):
            return None
        n = len(seqs)
        padded = n if padded is None else padded
        k = np.zeros(padded, np.int32)
        p = np.ones(padded, np.float32)
        mp = np.zeros(padded, np.float32)
        for i, s in enumerate(seqs):
            if s.temperature > 0:
                k[i], p[i], mp[i] = max(s.top_k, 0), s.top_p, s.min_p
        return k, p, mp

    @staticmethod
    def logprob_arrays(seqs: list[Sequence], padded: int | None = None, prefill: bool = False):
        """Per-row requested logprobs k (int32, -1 = off) of a step over `padded` rows, or None when no row wants them.
        In a prefill only the rows whose prompt ends in this step (the ones that sample) get theirs."""
        if not any(s.logprobs_k >= 0 for s in seqs):
            return None
        n = len(seqs)
        k = np.full(n if padded is None else padded, -1, np.int32)
        k[:n] = [s.logprobs_k if not prefill or s.num_cached_tokens + s.num_scheduled_tokens >= s.num_tokens else -1
                 for s in seqs]
        return None if prefill and not (k >= 0).any() else k

    def prepare_prefill(self, seqs: list[Sequence]):
        a = self.prefill_arrays(seqs)
        filt = self.filter_arrays(seqs)
        lpk = self.logprob_arrays(seqs, prefill=True)
        self.release_penalty_slots()
        pen = self.penalty_arrays(seqs, prefill=True)
        st = self.pstage
        off = 0
        views = {}
        plan = [("step", np.asarray([self.sample_step], np.int64), torch.int64),
                ("input_ids", a["input_ids"], torch.int64), ("positions", a["positions"], torch.int64),
                ("slot_mapping", a["slot_mapping"], torch.int32),
                ("cu_seqlens_q", a["cu_seqlens_q"], torch.int32), ("cu_seqlens_k", a["cu_seqlens_k"], torch.int32),
                ("temps", np.fromiter((s.temperature for s in seqs), dtype=np.float32, count=len(seqs)), torch.float32)]
        groups = None
        if a["block_tables"] is not None:
            plan.append(("block_tables", np.ascontiguousarray(a["block_tables"]).reshape(-1), torch.int32))
            if self.kv_fp8 and self.kv_scratch is not None:
                groups = kv_group_arrays(a["cu_seqlens_q"], a["cu_seqlens_k"],
                                         plan_kv_groups(a["cu_seqlens_k"], self.kv_scratch_rows))
                for i, g in enumerate(groups):
                    plan += [(f"g{i}q", g[6], torch.int32), (f"g{i}k", g[7], torch.int32)]
        if filt is not None:
            plan += [("topk", filt[0], torch.int32), ("topp", filt[1], torch.float32), ("minp", filt[2], torch.float32)]
        if pen is not None:
            offsets, n_ent = self._stage_penalty_entries(seqs, pen[4], 2, prefill=True)
            plan += [("pslot", pen[0], torch.int32), ("prep", pen[1], torch.float32), ("pfreq", pen[2], torch.float32),
                     ("ppres", pen[3], torch.float32), ("poff", offsets, torch.int32)]
        if lpk is not None:
            plan.append(("lpk", lpk, torch.int32))
        for name, arr, tdt in plan:
            h, d = st.views(off, arr.size, arr.dtype, tdt)
            h[:] = arr
            views[name] = d
            off = _align(off + arr.nbytes)
        st.upload(off)
        self.h2d_bytes_last = off
        self.step_penalties = None
        if pen is not None:                                  # load the slots of the sequences this step samples for
            self._load_penalty_slots(2, n_ent, views["poff"], views["pslot"])
            self.step_penalties = (views["pslot"], views["prep"], views["pfreq"], views["ppres"], None)
        bt = views.get("block_tables")
        if bt is not None:
            bt = bt.view(len(seqs), -1)
        slot = views["slot_mapping"] if a["slot_mapping"].size else None
        kv_groups = None
        if groups is not None:
            kv_groups = [KVGroup(*g[:6], views[f"g{i}q"], views[f"g{i}k"]) for i, g in enumerate(groups)]
        set_context(True, views["cu_seqlens_q"], views["cu_seqlens_k"], a["max_seqlen_q"], a["max_seqlen_k"],
                    slot, None, bt, kv_groups)
        self.step_filters = None if filt is None else (views["topk"], views["topp"], views["minp"])
        self.step_logprobs = views.get("lpk")
        return views["input_ids"], views["positions"], views["temps"], views["step"]

    def _padded_rows(self, n: int) -> int:
        use_graph = (not self.enforce_eager) and n <= self.max_bs and bool(self.graphs)
        return next(b for b in self.graph_bs if b >= n) if use_graph else n

    def stage_decode(self, seqs: list[Sequence]) -> int:
        """Fill the next pinned decode buffer for this batch (graph-padded) WITHOUT touching the GPU; returns the
        buffer index.  input_ids / step are refreshed at launch, so this may run while the previous step is still
        executing and its sampled tokens are not known yet."""
        self._host_k ^= 1
        k = self._host_k
        h = self.hd[k]
        a = self.decode_arrays(seqs)
        n = len(seqs)
        padded = self._padded_rows(n)
        h["ids"][:n] = a["input_ids"]
        h["pos"][:n] = a["positions"]
        h["slot"][:n] = a["slot_mapping"]
        h["ctx"][:n] = a["context_lens"]
        h["temp"][:n] = np.fromiter((s.temperature for s in seqs), dtype=np.float32, count=n)
        if padded > n:                                       # graph padding rows (model_runner.py:206-208)
            h["ids"][n:padded] = 0
            h["pos"][n:padded] = 0
            h["slot"][n:padded] = -1
            h["ctx"][n:padded] = 0
            h["temp"][n:padded] = 0
        bt = a["block_tables"]
        h["bt"][:n, :bt.shape[1]] = bt
        filt = self.filter_arrays(seqs, padded)
        self.release_penalty_slots()
        pen = self.penalty_arrays(seqs, padded)
        lpk = self.logprob_arrays(seqs, padded)
        self.f_any[k] = filt is not None or pen is not None or lpk is not None
        self.lp_any[k] = lpk is not None
        self.p_load[k] = None
        if self.f_any[k]:
            hf = self.hf[k]
            if filt is None:
                filt = (0, 1.0, 0.0)
            hf["topk"][:padded], hf["topp"][:padded], hf["minp"][:padded] = filt
            if pen is None:
                pen = (-1, 1.0, 0.0, 0.0, np.zeros(padded, bool))
            hf["pslot"][:padded], hf["prep"][:padded], hf["pfreq"][:padded], hf["ppres"][:padded] = pen[:4]
            hf["lpk"][:padded] = -1 if lpk is None else lpk
            load = pen[4][:n]
            if load.any():                                   # sequences whose slot was taken while outside the batch
                offsets, total = self._stage_penalty_entries(seqs, load, k, prefill=False)
                hf["plslot"][:n] = np.where(load, pen[0][:n], -1)
                hf["ploff"][:n + 1] = offsets
                self.p_load[k] = (total, n)
        return k

    def prepare_decode(self, seqs: list[Sequence], padded: int, staged: int | None = None, src=None):
        """Upload a staged decode buffer (staging it now unless `staged` names one) and set the Context.

        `src` (optional, one int per row): row of the PREVIOUS step's sampled tokens that is this row's input id, or
        -1 when the id is already known on the host.  With it the step can be enqueued before the previous step's
        tokens have been read back: the ids are gathered on the device (b200_gather_tokens)."""
        n = len(seqs)
        if staged is None:
            k = self.stage_decode(seqs)
        else:                                                # staged early: only the token ids were unknown then
            k = staged
            self.hd[k]["ids"][:n] = np.fromiter((s.last_token for s in seqs), dtype=np.int64, count=n)
        self.hd[k]["step"][0] = self.sample_step
        if src is not None:
            self.hd[k]["src"][:n] = src
        nbytes = self.d_off["bt"] + padded * self.max_blocks * 4
        self.stage.upload(nbytes, k)
        self.h2d_bytes_last = nbytes
        self.step_filters = self.step_penalties = self.step_logprobs = None
        if self.f_any[k]:                                    # only a step where some row filters or penalises uploads them
            self.fstage.upload(self.f_bytes, k)
            self.h2d_bytes_last += self.f_bytes
            self.step_filters = (self.g_topk[:padded], self.g_topp[:padded], self.g_minp[:padded])
            # the pending token of a row is its input id: the token sampled one step earlier, absorbed into the history
            self.step_penalties = (self.g_pslot[:padded], self.g_prep[:padded], self.g_pfreq[:padded], self.g_ppres[:padded],
                                   self.g_ids[:padded])
            if self.lp_any[k]:
                self.step_logprobs = self.g_lpk[:padded]
            if self.p_load[k] is not None:
                total, rows = self.p_load[k]
                self._load_penalty_slots(k, total, self.g_ploff[:rows + 1], self.g_plslot[:rows])
        if src is not None:
            ops.gather_tokens(self.g_ids[:n], self.g_src[:n], self.g_tokens)
        set_context(False, slot_mapping=self.g_slot[:padded], context_lens=self.g_ctx[:padded],
                    block_tables=self.g_bt[:padded])

    # ---- model + sampling -------------------------------------------------------------------------
    def _forward_and_sample(self, input_ids, positions, temps, step_dev, rows: int, filters=None, penalties=None,
                            logprobs=None):
        """hidden -> shard logits -> sampled token ids in self.g_tokens[:rows] (all enqueued, no sync).
        ``filters``: (top_k, top_p, min_p) device tensors of the rows when some row filters; ``penalties``: (slot,
        repetition, frequency, presence, pending token or None) when some row filters or penalises.  The logits are then
        materialised (also under B200_LM_HEAD=fused), penalised and sampled by the filtered sampler.  ``logprobs``: the
        rows' requested k (int32, -1 = off) when some row wants logprobs; they go into self.g_lp_out[:rows]."""
        hidden = self.model(input_ids, positions)
        if filters is not None or penalties is not None or logprobs is not None:
            self._sample_filtered(hidden, temps, step_dev, rows, filters, penalties, logprobs)
            return
        if self.fused_lm_head and rows <= self.g_keyws.numel():
            # opt-in (B200_LM_HEAD=fused): LM head + sampling in one tensor-core kernel, logits never written; parity-green but
            # slower than the library GEMM + sample_kernel pair (DESIGN.md 3.4), hence not the default
            last = self.model.last_token_rows(hidden)
            if self.world_size == 1:
                ops.lm_head_sample(last, self.model.lm_head, temps, self.sample_seed, 0, self.g_keyws, out=self.g_tokens[:rows],
                                   step_dev=step_dev)
            else:
                keys = self.g_keys[:rows]
                ops.lm_head_sample(last, self.model.lm_head, temps, self.sample_seed, 0, self.g_keyws, out=self.g_tokens[:rows],
                                   index_offset=self.vocab_offset, out_keys=keys, step_dev=step_dev)
                dist.all_reduce(keys, op=dist.ReduceOp.MAX)
                self.g_tokens[:rows].copy_(ops.tokens_from_keys(keys))
            return
        logits = self.model.compute_logits(hidden)
        if self.world_size == 1:
            ops.sample(logits, temps, self.sample_seed, 0, out=self.g_tokens[:rows], step_dev=step_dev)
        else:
            keys = self.g_keys[:rows]
            ops.sample(logits, temps, self.sample_seed, 0, out=self.g_tokens[:rows], index_offset=self.vocab_offset,
                       out_keys=keys, step_dev=step_dev)
            dist.all_reduce(keys, op=dist.ReduceOp.MAX)
            self.g_tokens[:rows].copy_(ops.tokens_from_keys(keys))

    def _sample_filtered(self, hidden, temps, step_dev, rows: int, filters, penalties=None, logprobs=None):
        logits = self.model.compute_logits(hidden)
        tp = self.world_size > 1
        reduce = self._reduce_filter_words if tp else None
        if logprobs is not None:                 # on the raw logits: top k and maximum, then keep what the penalties rewrite
            ops.logprobs_topk(logits, logprobs, self.g_lp_ws, self.g_lp_keys, self.vocab_offset, reduce=reduce)
        if penalties is not None:                # every rank absorbs into its full copy of the history, penalises its shard
            slot, rep, freq, pres, pending = penalties
            if logprobs is not None:
                ops.logprobs_save(logits, logprobs, self.g_lp_ws, self.g_lp_saved, self.pen_hist, self.pen_len, slot, pending,
                                  self.vocab_offset)
            ops.penalty_apply(logits, self.pen_hist, self.pen_len, slot, rep, freq, pres, pending, self.vocab_offset)
        top_k, top_p, min_p = filters if filters is not None else (None, None, None)
        if not tp:
            ops.sample_filtered(logits, temps, top_k, top_p, min_p, self.sample_seed, 0, self.g_filter_ws,
                                out=self.g_tokens[:rows], step_dev=step_dev)
        else:
            # every rank launches every stage and every all-reduce, whatever its rows need, so the collectives match
            keys = self.g_keys[:rows]
            ops.sample_filtered(logits, temps, top_k, top_p, min_p, self.sample_seed, 0, self.g_filter_ws,
                                out=self.g_tokens[:rows], index_offset=self.vocab_offset, out_keys=keys, step_dev=step_dev,
                                reduce=reduce)
            dist.all_reduce(keys, op=dist.ReduceOp.MAX)
            self.g_tokens[:rows].copy_(ops.tokens_from_keys(keys))
        if logprobs is not None:                 # the logits are raw again after the restore
            ops.logprobs_finish(logits, logprobs, self.g_tokens[:rows], self.g_lp_ws, self.g_lp_keys, self.g_lp_out,
                                self.vocab_offset, saved=self.g_lp_saved if penalties is not None else None,
                                capacity=self.pen_hist.shape[1] if penalties is not None else 0, reduce=reduce,
                                gather=self._gather_logprob_keys if tp else None)

    def _gather_logprob_keys(self, keys: torch.Tensor) -> torch.Tensor:
        """Every tensor-parallel rank's top-k keys, [world, n] in rank order."""
        out = torch.empty(self.world_size, keys.numel(), dtype=keys.dtype, device=keys.device)
        dist.all_gather(list(out.unbind(0)), keys.contiguous())
        return out

    @staticmethod
    def _reduce_filter_words(words: torch.Tensor, op: str) -> None:
        """All-reduce one stage's words of the filter workspace over the tensor-parallel ranks (a strided view)."""
        buf = words.contiguous()
        dist.all_reduce(buf, op=dist.ReduceOp.MAX if op == "max" else dist.ReduceOp.SUM)
        words.copy_(buf)

    def run(self, seqs: list[Sequence], is_prefill: bool) -> list[int]:
        self.launch(seqs, is_prefill)
        return self.collect()

    @torch.inference_mode()
    def launch(self, seqs: list[Sequence], is_prefill: bool, staged: int | None = None, src=None) -> None:
        """Enqueue one step (metadata upload, forward, sampling, token read-back) without waiting for it.
        Up to two steps may be in flight; collect() returns them in launch order."""
        n = len(seqs)
        self.sample_step += 1
        prof = self._prof
        ev0 = None
        if is_prefill:
            ids, pos, temps, step_dev = self.prepare_prefill(seqs)
            if prof is not None:
                ev0 = torch.cuda.Event(enable_timing=True)
                ev0.record()
            self._forward_and_sample(ids, pos, temps, step_dev, n, filters=self.step_filters, penalties=self.step_penalties,
                                     logprobs=self.step_logprobs)
        else:
            if n > self.cap_bs:
                raise RuntimeError(f"decode batch {n} exceeds max_num_seqs = {self.cap_bs}")
            padded = self._padded_rows(n)
            self.prepare_decode(seqs, padded, staged, src)
            if prof is not None:
                ev0 = torch.cuda.Event(enable_timing=True)
                ev0.record()
            filt, lpk = self.step_filters, self.step_logprobs
            if padded in self.graphs and not self.enforce_eager and n <= self.max_bs:
                if lpk is not None:                          # the third graph: the second one plus the logprob kernels
                    self.lgraphs[padded].replay()
                    ops.LAUNCHES[0] += self.lgraph_kernels[padded]
                elif filt is None:
                    self.graphs[padded].replay()
                    ops.LAUNCHES[0] += self.graph_kernels[padded]
                else:                                        # the bucket's second graph: penalties, then the filtered sampler
                    self.fgraphs[padded].replay()
                    ops.LAUNCHES[0] += self.fgraph_kernels[padded]
            else:
                pen = self.step_penalties
                if filt is not None:
                    filt = tuple(t[:n] for t in filt)
                    pen = tuple(t[:n] for t in pen)
                    lpk = None if lpk is None else lpk[:n]
                self._forward_and_sample(self.g_ids[:n], self.g_pos[:n], self.g_temp[:n], self.g_step, n, filters=filt,
                                         penalties=pen, logprobs=lpk)
        if prof is not None:
            ev1 = torch.cuda.Event(enable_timing=True)
            ev1.record()
            prof["events"].append((ev0, ev1))
            prof["h2d"] += self.h2d_bytes_last
            prof["d2h"] += n * 8 + (n * ops.LOGPROB_OUT_WORDS * 4 if self.step_logprobs is not None else 0)
            prof["steps"] += 1
        kk = self._launches & 1
        self._launches += 1
        assert len(self._pending) < 2, "at most two steps in flight"
        self.h_tokens[kk][:n].copy_(self.g_tokens[:n], non_blocking=True)
        peer = getattr(self.model, "peer", None)
        if peer is not None:              # the exchange kernel's timeout flag rides along with the tokens: checked every step
            self.h_err[kk].copy_(peer.state[2:3], non_blocking=True)
        lp = self.step_logprobs is not None
        if lp:                            # only a step with a logprob row reads its result rows back
            self.h_lp[kk][:n].copy_(self.g_lp_out[:n], non_blocking=True)
        self._done[kk].record()
        self._pending.append((kk, n, lp))
        self.d2h_bytes_last = n * 8 + (n * ops.LOGPROB_OUT_WORDS * 4 if lp else 0)
        self.step_logprobs = None
        reset_context()

    def collect(self) -> list[int]:
        """Wait for the oldest step enqueued by launch() (that step's only host sync) and return its token ids.  The step's
        logprob result rows (int32 [n, ops.LOGPROB_OUT_WORDS], a copy) are left in self.last_logprobs, None when no row of
        the step asked for logprobs; rows that did not are undefined."""
        kk, n, lp = self._pending.popleft()
        self._done[kk].synchronize()
        if int(self.h_err[kk][0]) != 0:
            from .peer_reduce import PeerExchangeTimeout
            raise PeerExchangeTimeout("tensor-parallel peer exchange timed out in this step (a rank stopped or fell >10 s "
                                      "behind); its tokens are invalid -- rerun with B200_TP_ALLREDUCE=nccl to bypass")
        self.last_logprobs = self.h_lp_np[kk][:n].copy() if lp else None
        return self.h_tokens_np[kk][:n].tolist()

    def drain(self) -> None:
        """Forget steps that were launched but not collected (after a failed step)."""
        torch.cuda.synchronize()
        self._pending.clear()

    @torch.inference_mode()
    def capture_cudagraph(self):
        """One graph per batch-size bucket over the static buffers, largest first so they share one pool
        (model_runner.py:222-257; same bucket list)."""
        max_bs = self.max_bs
        self.graph_bs = [b for b in (1, 2, 4, 8) if b <= max_bs] + list(range(16, max_bs + 1, 16))
        if max_bs not in self.graph_bs:
            self.graph_bs.append(max_bs)
        h = self.hd[0]
        h["ctx"][:] = 0
        h["slot"][:] = -1
        h["ids"][:] = 0
        h["pos"][:] = 0
        h["temp"][:] = 0
        h["step"][0] = 0
        self.stage.upload(self.d_bytes, 0)
        torch.cuda.synchronize()
        # per graph set: cumulative capture seconds, bytes reserved by the caching allocator and bytes of the graphs' shared
        # private pool after it
        self.capture_stats: list[dict] = []
        t0 = perf_counter()

        def set_done(name: str):
            pool = tuple(self.graph_pool)
            pool_bytes = sum(seg["total_size"] for seg in torch.cuda.memory_snapshot()
                             if tuple(seg.get("segment_pool_id", ())) == pool)
            self.capture_stats.append(dict(set=name, seconds=perf_counter() - t0, reserved=torch.cuda.memory_reserved(),
                                           pool=pool_bytes))

        for bs in reversed(self.graph_bs):
            set_context(False, slot_mapping=self.g_slot[:bs], context_lens=self.g_ctx[:bs], block_tables=self.g_bt[:bs])
            args = (self.g_ids[:bs], self.g_pos[:bs], self.g_temp[:bs], self.g_step, bs)
            self._forward_and_sample(*args)                  # warm-up outside capture
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            before = ops.LAUNCHES[0]
            with torch.cuda.graph(graph, self.graph_pool):
                self._forward_and_sample(*args)
            self.graph_kernels[bs] = ops.LAUNCHES[0] - before
            if self.graph_pool is None:
                self.graph_pool = graph.pool()
            self.graphs[bs] = graph
            torch.cuda.synchronize()
            reset_context()
        set_done("plain")
        # second set, same pool: the same steps with the penalties and the top-k / top-p / min-p sampler, replayed when some
        # row filters or penalises (the slots are -1 here, so capturing touches no history)
        for bs in reversed(self.graph_bs):
            set_context(False, slot_mapping=self.g_slot[:bs], context_lens=self.g_ctx[:bs], block_tables=self.g_bt[:bs])
            args = (self.g_ids[:bs], self.g_pos[:bs], self.g_temp[:bs], self.g_step, bs)
            filters = (self.g_topk[:bs], self.g_topp[:bs], self.g_minp[:bs])
            penalties = (self.g_pslot[:bs], self.g_prep[:bs], self.g_pfreq[:bs], self.g_ppres[:bs], self.g_ids[:bs])
            self._forward_and_sample(*args, filters=filters, penalties=penalties)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            before = ops.LAUNCHES[0]
            with torch.cuda.graph(graph, self.graph_pool):
                self._forward_and_sample(*args, filters=filters, penalties=penalties)
            self.fgraph_kernels[bs] = ops.LAUNCHES[0] - before
            self.fgraphs[bs] = graph
            torch.cuda.synchronize()
            reset_context()
        set_done("filtered")
        # third set, same pool: the second set's step plus the logprob kernels, replayed when some row wants logprobs (k is
        # -1 in every row here, so capturing computes nothing)
        for bs in reversed(self.graph_bs):
            set_context(False, slot_mapping=self.g_slot[:bs], context_lens=self.g_ctx[:bs], block_tables=self.g_bt[:bs])
            args = (self.g_ids[:bs], self.g_pos[:bs], self.g_temp[:bs], self.g_step, bs)
            kw = dict(filters=(self.g_topk[:bs], self.g_topp[:bs], self.g_minp[:bs]),
                      penalties=(self.g_pslot[:bs], self.g_prep[:bs], self.g_pfreq[:bs], self.g_ppres[:bs], self.g_ids[:bs]),
                      logprobs=self.g_lpk[:bs])
            self._forward_and_sample(*args, **kw)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            before = ops.LAUNCHES[0]
            with torch.cuda.graph(graph, self.graph_pool):
                self._forward_and_sample(*args, **kw)
            self.lgraph_kernels[bs] = ops.LAUNCHES[0] - before
            self.lgraphs[bs] = graph
            torch.cuda.synchronize()
            reset_context()
        set_done("logprobs")
