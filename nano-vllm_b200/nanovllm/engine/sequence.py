"""Per-request state and block arithmetic (reference nanovllm/engine/sequence.py:14-83).

Attribute and property names are the reference's (the Scheduler, BlockManager and ModelRunner
contracts are written against them); the integers they hold must match the reference bit for
bit, which tests/test_bookkeeping_golden.py checks against traces of the reference's own classes.
"""
from __future__ import annotations

import itertools
from enum import Enum, auto

from ..sampling_params import SamplingParams


class SequenceStatus(Enum):
    WAITING = auto()
    RUNNING = auto()
    FINISHED = auto()


_DEFAULT_SP = SamplingParams()


class Sequence:
    block_size = 256                      # set by LLMEngine from Config.kvcache_block_size
    counter = itertools.count()           # ids are never reused within a process

    __slots__ = ("seq_id", "status", "token_ids", "last_token", "num_tokens", "num_prompt_tokens",
                 "num_cached_tokens", "num_scheduled_tokens", "is_prefill", "block_table",
                 "temperature", "max_tokens", "ignore_eos", "top_k", "top_p", "min_p")

    def __init__(self, token_ids: list[int], sampling_params: SamplingParams = _DEFAULT_SP):
        if not token_ids:
            raise ValueError("a sequence needs at least one prompt token")
        self.seq_id = next(Sequence.counter)
        self.status = SequenceStatus.WAITING
        self.token_ids = list(token_ids)
        self.last_token = self.token_ids[-1]
        self.num_tokens = self.num_prompt_tokens = len(self.token_ids)
        self.num_cached_tokens = 0        # tokens whose K/V already sit in the cache
        self.num_scheduled_tokens = 0     # tokens the current step computes
        self.is_prefill = True
        self.block_table: list[int] = []
        self.temperature = sampling_params.temperature
        self.max_tokens = sampling_params.max_tokens
        self.ignore_eos = sampling_params.ignore_eos
        self.top_k = sampling_params.top_k
        self.top_p = sampling_params.top_p
        self.min_p = sampling_params.min_p

    def __len__(self) -> int:
        return self.num_tokens

    def __getitem__(self, key):
        return self.token_ids[key]

    @property
    def is_finished(self) -> bool:
        return self.status is SequenceStatus.FINISHED

    @property
    def num_completion_tokens(self) -> int:
        return self.num_tokens - self.num_prompt_tokens

    @property
    def prompt_token_ids(self) -> list[int]:
        return self.token_ids[:self.num_prompt_tokens]

    @property
    def completion_token_ids(self) -> list[int]:
        return self.token_ids[self.num_prompt_tokens:]

    @property
    def num_blocks(self) -> int:
        return -(-self.num_tokens // self.block_size)

    @property
    def last_block_num_tokens(self) -> int:
        return self.num_tokens - (self.num_blocks - 1) * self.block_size

    def block(self, i: int) -> list[int]:
        if not 0 <= i < self.num_blocks:
            raise IndexError(i)
        bs = self.block_size
        return self.token_ids[i * bs:(i + 1) * bs]

    def append_token(self, token_id: int) -> None:
        self.token_ids.append(token_id)
        self.last_token = token_id
        self.num_tokens += 1

    # Slim transfer form for worker ranks (reference sequence.py:72-83): a decoding sequence
    # only needs its last token, a prefilling one its full token list.
    def __getstate__(self):
        tail = self.token_ids if self.is_prefill else self.last_token
        return (self.num_tokens, self.num_prompt_tokens, self.num_cached_tokens,
                self.num_scheduled_tokens, self.block_table, tail)

    def __setstate__(self, state):
        (self.num_tokens, self.num_prompt_tokens, self.num_cached_tokens,
         self.num_scheduled_tokens, self.block_table, tail) = state
        if isinstance(tail, list):
            self.token_ids, self.last_token, self.is_prefill = tail, tail[-1], True
        else:
            self.token_ids, self.last_token, self.is_prefill = [], tail, False
