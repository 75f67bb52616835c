"""The engine behind ``LLM`` (reference nanovllm/engine/llm_engine.py:15-90): same public methods
(``add_request``, ``step``, ``is_finished``, ``generate``, ``exit``), same return shapes.

Tensor parallelism is SPMD: each GPU process owns a full replica of the (deterministic) scheduler
and its own ModelRunner and executes the same steps in lock-step.  Two ways to get the ranks:

* launched by ``torchrun`` / any launcher that sets RANK, WORLD_SIZE (== tensor_parallel_size),
  LOCAL_RANK, MASTER_ADDR, MASTER_PORT: every process simply constructs ``LLM(...)`` and calls the
  same methods (this is how bench.py runs at N > 1);
* plain ``LLM(path, tensor_parallel_size=N)`` from one process, like the reference
  (llm_engine.py:24-30): ranks 1..N-1 are spawned and mirror rank 0's API calls, which are broadcast
  once per call (one message per ``generate``, not one per step).
"""
from __future__ import annotations

import atexit
import os
from dataclasses import fields
from time import perf_counter

from ..config import Config
from ..ops import LOGPROB_LP_COL, LOGPROB_RANK_COL
from ..sampling_params import Logprob, SamplingParams
from .model_runner import ModelRunner
from .scheduler import Scheduler
from .sequence import Sequence


def _free_port() -> int:
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def logprob_dicts(rows: list, k: int) -> tuple[list[dict], float]:
    """A finished sequence's logprob rows (one packed int32 row per completion token, ModelRunner.collect) -> one
    {token_id: Logprob} dict per token and the cumulative logprob of the sampled tokens.  Built like vLLM's: the sampled
    token first, with its rank, then the top k with ranks 1..k; a sampled token inside the top k takes its top-k entry."""
    import numpy as np
    a = np.stack(rows) if rows else np.zeros((0, LOGPROB_RANK_COL + 1), np.int32)
    ids = a[:, :1 + k].tolist()
    lps = a[:, LOGPROB_LP_COL:LOGPROB_LP_COL + 1 + k].view(np.float32).tolist()
    ranks = a[:, LOGPROB_RANK_COL].tolist()
    out = []
    for tid, tlp, rank in zip(ids, lps, ranks):
        d = {tid[0]: Logprob(tlp[0], rank)}
        for j in range(1, k + 1):
            d[tid[j]] = Logprob(tlp[j], j)
        out.append(d)
    return out, sum(t[0] for t in lps)


def _worker_main(model: str, kwargs: dict, rank: int, world: int, port: int):
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world),
                      MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    engine = LLMEngine(model, **kwargs)
    engine._serve()


class LLMEngine:
    def __init__(self, model: str, **kwargs):
        names = {f.name for f in fields(Config)}
        config = Config(model, **{k: v for k, v in kwargs.items() if k in names})   # unknown keys are ignored
        self.config = config
        Sequence.block_size = config.kvcache_block_size
        tp = config.tensor_parallel_size
        self.rank, self._procs, self._mirrors = 0, [], False
        saved_env = None
        if tp > 1:
            if int(os.environ.get("WORLD_SIZE", "1")) == tp and "RANK" in os.environ:
                self.rank = int(os.environ["RANK"])                                  # launcher-provided replicas
            else:
                # spawn mode: the rendezvous variables are set only while the ranks are being constructed and are put
                # back afterwards, so that a later LLM(...) in this process (or any child it starts) does not mistake
                # them for a launcher's and the launcher-vs-spawn decision above stays a function of the user's env
                import torch.multiprocessing as mp
                port = _free_port()
                keys = ("RANK", "LOCAL_RANK", "WORLD_SIZE", "MASTER_ADDR", "MASTER_PORT")
                saved_env = {k: os.environ.get(k) for k in keys}
                os.environ.update(RANK="0", LOCAL_RANK="0", WORLD_SIZE=str(tp), MASTER_ADDR="127.0.0.1",
                                  MASTER_PORT=str(port))
                ctx = mp.get_context("spawn")
                for r in range(1, tp):
                    p = ctx.Process(target=_worker_main, args=(model, dict(kwargs), r, tp, port), daemon=True)
                    p.start()
                    self._procs.append(p)
                self._mirrors = True
        try:
            self.model_runner = ModelRunner(config, self.rank, None)
        finally:
            if saved_env is not None:
                for k, v in saved_env.items():
                    if v is None:
                        os.environ.pop(k, None)
                    else:
                        os.environ[k] = v
        from transformers import AutoTokenizer
        self.tokenizer = AutoTokenizer.from_pretrained(config.model, use_fast=True)
        config.eos = self.tokenizer.eos_token_id if self.tokenizer.eos_token_id is not None else -1
        self.scheduler = Scheduler(config)            # after the runner: it needs num_kvcache_blocks
        self._closed = False
        # step-loop accounting (seconds): total wall time of the loop, and the part of it spent blocked on the GPU;
        # total - wait is the host's own work (scheduling, metadata staging, launches, detokenisation)
        self.loop_stats = {"steps": 0, "total_s": 0.0, "wait_s": 0.0}
        atexit.register(self.exit)

    # ---- rank-0 -> mirror ranks control channel (spawn mode only) --------------------------
    def _tell(self, *cmd):
        if self._mirrors:
            import torch.distributed as dist
            dist.broadcast_object_list([cmd], src=0)

    def _serve(self):
        import torch.distributed as dist
        while True:
            box = [None]
            dist.broadcast_object_list(box, src=0)
            cmd, *args = box[0]
            if cmd == "generate":
                self._generate(*args, use_tqdm=False)
            elif cmd == "add":
                self._add_request(*args)
            elif cmd == "step":
                self._step()
            elif cmd == "exit":
                self._close()
                return

    # ---- public API ------------------------------------------------------------------------
    def exit(self):
        if self._closed:
            return
        self._tell("exit")
        self._close()
        for p in self._procs:
            p.join(timeout=30)

    def _close(self):
        if not self._closed:
            self._closed = True
            self.model_runner.call("exit")

    def add_request(self, prompt: str | list[int], sampling_params: SamplingParams):
        if isinstance(prompt, str):
            prompt = self.tokenizer.encode(prompt)
        self._tell("add", prompt, sampling_params)
        self._add_request(prompt, sampling_params)

    def _add_request(self, prompt: list[int], sampling_params: SamplingParams):
        # the embedding gather indexes the table with these ids: refuse anything that is not a token of this model
        # (the reference's F.embedding device-asserts instead, embed_head.py:38)
        vocab = self.config.hf_config.vocab_size
        if len(prompt) == 0:
            raise ValueError("empty prompt")
        lo, hi = min(prompt), max(prompt)
        if lo < 0 or hi >= vocab:
            raise ValueError(f"prompt token id {lo if lo < 0 else hi} is outside the vocabulary [0, {vocab})")
        # a penalised sequence's token history lives in a fixed device slot of min(max_model_len, vocab) entries, and
        # nothing else bounds a sequence's length
        if sampling_params.penalised and len(prompt) + sampling_params.max_tokens > self.config.max_model_len:
            raise ValueError(f"a request with penalties needs len(prompt) + max_tokens <= max_model_len "
                             f"({len(prompt)} + {sampling_params.max_tokens} > {self.config.max_model_len})")
        self.scheduler.add(Sequence(prompt, sampling_params))

    def step(self):
        self._tell("step")
        return self._step()

    def _step(self):
        seqs, is_prefill = self.scheduler.schedule()
        num_tokens = sum(s.num_scheduled_tokens for s in seqs) if is_prefill else -len(seqs)
        before = [s.num_tokens for s in seqs]
        token_ids = self.model_runner.call("run", seqs, is_prefill)
        self.scheduler.postprocess(seqs, token_ids, is_prefill)
        lp = getattr(self.model_runner, "last_logprobs", None)
        if lp is not None:
            for i, (s, b) in enumerate(zip(seqs, before)):
                if s.num_tokens != b and s.logprob_rows is not None:
                    s.logprob_rows.append(lp[i].copy())   # not a view: it would keep the step's rows alive
        outputs = [(s.seq_id, s.completion_token_ids) for s in seqs if s.is_finished]
        return outputs, num_tokens

    def is_finished(self) -> bool:
        return self.scheduler.is_finished()

    def generate(self, prompts: list[str] | list[list[int]], sampling_params: SamplingParams | list[SamplingParams],
                 use_tqdm: bool = True) -> list[dict]:
        prompts = [self.tokenizer.encode(p) if isinstance(p, str) else list(p) for p in prompts]
        self._tell("generate", prompts, sampling_params)
        return self._generate(prompts, sampling_params, use_tqdm and self.rank == 0)

    def _generate(self, prompts, sampling_params, use_tqdm: bool):
        pbar = None
        if use_tqdm:
            from tqdm.auto import tqdm
            pbar = tqdm(total=len(prompts), desc="Generating", dynamic_ncols=True)
        if not isinstance(sampling_params, list):
            sampling_params = [sampling_params] * len(prompts)
        for prompt, sp in zip(prompts, sampling_params):
            self._add_request(prompt, sp)
        done: dict[int, dict] = {}
        stats = {"prefill": 0.0, "decode": 0.0}

        def on_step(finished, num_tokens, dt):
            if num_tokens > 0:
                stats["prefill"] = num_tokens / dt
            else:
                stats["decode"] = -num_tokens / dt
            for seq in finished:                  # detokenise now: the next step is already running on the GPU
                toks = seq.completion_token_ids
                done[seq.seq_id] = {"text": self.tokenizer.decode(toks), "token_ids": toks}
                if seq.logprob_rows is not None:
                    lp, cum = logprob_dicts(seq.logprob_rows, seq.logprobs_k)
                    done[seq.seq_id].update(logprobs=lp, cumulative_logprob=cum)
            if pbar is not None:
                pbar.set_postfix({"Prefill": f"{int(stats['prefill'])}tok/s", "Decode": f"{int(stats['decode'])}tok/s"})
                pbar.update(len(finished))

        try:
            self._run_overlapped(on_step)
            self.model_runner.check_peer_exchange()
        except Exception:
            # a step failed (e.g. the tensor-parallel exchange timed out and produced undefined data): nothing that step
            # or its successors wrote may survive -- drop in-flight steps, retire every sequence, forget the prefix
            # cache -- and let the error reach the caller
            self.model_runner.call("drain")
            self.scheduler.abort_all()
            raise
        finally:
            if pbar is not None:
                pbar.close()
        return [done[k] for k in sorted(done)]

    def _run_overlapped(self, on_step) -> None:
        """The reference's step loop (llm_engine.py:49-55, 73-86) with the host work of step N+1 done while the
        GPU runs step N.

        What the next schedule needs from a finished step is (a) which sequences ended and (b) the sampled
        token values.  (a) depends on the values only through EOS, so when no sequence of the batch can stop on
        EOS (ignore_eos) the whole postprocess -> schedule -> metadata staging of the next step is computed
        first with a placeholder token, a following decode step is even enqueued on the GPU (its input ids are
        gathered on the device from the running step's output), and the values are patched into the host state
        when they arrive: the bookkeeping is exactly the synchronous one, only earlier.  A batch that can hit EOS
        takes the synchronous order."""
        sched, runner = self.scheduler, self.model_runner
        PENDING = -1
        if sched.is_finished():
            return
        st = self.__dict__.setdefault("loop_stats", {"steps": 0, "total_s": 0.0, "wait_s": 0.0})   # host time: waiting vs own work
        seqs, is_prefill = sched.schedule()
        runner.call("launch", seqs, is_prefill)
        t0 = perf_counter()
        while True:
            num_tokens = sum(s.num_scheduled_tokens for s in seqs) if is_prefill else -len(seqs)
            nxt, launched = None, False
            if all(s.ignore_eos for s in seqs):
                before = [s.num_tokens for s in seqs]
                sched.postprocess(seqs, [PENDING] * len(seqs), is_prefill)
                if not sched.is_finished():
                    nxt = sched.schedule()
                    if not nxt[1]:
                        # a decode step: its metadata needs no token value and its input ids are gathered on the
                        # device from the step still running, so enqueue it now -- the GPU never waits for the host
                        row_of = {id(s): i for i, (s, b) in enumerate(zip(seqs, before)) if s.num_tokens != b}
                        src = [row_of.get(id(s), -1) for s in nxt[0]]
                        runner.launch(nxt[0], False, runner.stage_decode(nxt[0]), src)
                        launched = True
                tw = perf_counter()
                tokens = runner.call("collect")
                st["wait_s"] += perf_counter() - tw
                lp = getattr(runner, "last_logprobs", None)
                for i, (s, b, t) in enumerate(zip(seqs, before, tokens)):
                    if s.num_tokens != b:                       # a token was appended: give it its value
                        s.token_ids[-1] = t
                        s.last_token = t
                        if lp is not None and s.logprob_rows is not None:
                            s.logprob_rows.append(lp[i].copy())
            else:
                tw = perf_counter()
                tokens = runner.call("collect")
                st["wait_s"] += perf_counter() - tw
                lp = getattr(runner, "last_logprobs", None)
                before = None if lp is None else [s.num_tokens for s in seqs]
                sched.postprocess(seqs, tokens, is_prefill)
                if lp is not None:
                    for i, (s, b) in enumerate(zip(seqs, before)):
                        if s.num_tokens != b and s.logprob_rows is not None:
                            s.logprob_rows.append(lp[i].copy())
                if not sched.is_finished():
                    nxt = sched.schedule()
            now = perf_counter()
            on_step([s for s in seqs if s.is_finished], num_tokens, max(now - t0, 1e-9))
            st["steps"] += 1
            st["total_s"] += now - t0
            t0 = now
            if nxt is None:
                return
            seqs, is_prefill = nxt
            if not launched:
                runner.launch(seqs, is_prefill)
