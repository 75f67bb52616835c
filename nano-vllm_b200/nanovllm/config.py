"""Engine configuration (reference nanovllm/config.py:6-25): same fields, same defaults.

Differences, all widenings: ``kvcache_block_size`` may be any power of two in [16, 256]
(the reference's ``% 256`` assertion exists only for flash-attn's paged path, SURVEY.md S2),
``hf_config`` may be supplied pre-built (tests) instead of being read from ``model``, and
``kv_cache_dtype`` (vLLM's option) selects the KV-cache element type: "auto" = bf16, "fp8" / "fp8_e4m3" = e4m3
with unit scales (half the bytes per token, so twice the tokens in the same memory; DESIGN.md 3.5).
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Any

# accepted kv_cache_dtype values -> whether the cache holds fp8 (e4m3) elements
KV_CACHE_DTYPES = {"auto": False, "fp8": True, "fp8_e4m3": True}


@dataclass(slots=True)
class Config:
    model: str
    max_num_batched_tokens: int = 16384
    max_num_seqs: int = 512
    max_model_len: int = 4096
    gpu_memory_utilization: float = 0.9
    tensor_parallel_size: int = 1
    enforce_eager: bool = False
    hf_config: Any = None
    eos: int = -1
    kvcache_block_size: int = 256
    num_kvcache_blocks: int = -1
    kv_cache_dtype: str = "auto"

    def __post_init__(self):
        if self.kv_cache_dtype not in KV_CACHE_DTYPES:
            raise ValueError(f"kv_cache_dtype must be one of {sorted(KV_CACHE_DTYPES)}, got {self.kv_cache_dtype!r}")
        bs = self.kvcache_block_size
        if bs < 16 or bs > 256 or bs & (bs - 1):
            raise ValueError("kvcache_block_size must be a power of two in [16, 256]")
        if not 1 <= self.tensor_parallel_size <= 8:
            raise ValueError("tensor_parallel_size must be in 1..8")
        if self.hf_config is None:
            if not os.path.isdir(self.model):
                raise FileNotFoundError(f"model directory not found: {self.model}")
            from transformers import AutoConfig
            self.hf_config = AutoConfig.from_pretrained(self.model)
        self.max_model_len = min(self.max_model_len, self.hf_config.max_position_embeddings)
