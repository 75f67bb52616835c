"""Per-request sampling knobs (reference nanovllm/sampling_params.py:4-11).

Field names and defaults are the reference's.  One deliberate widening: temperature == 0 is
accepted and means greedy argmax (the reference asserts temperature > 1e-10; the north-star's
parity criterion needs greedy token ids).

Extras after the reference's fields, with vLLM's names, meanings and "off" defaults (DESIGN.md 3.3):
``top_k`` keeps the tokens whose logit is >= the k-th largest (-1 or 0: off), ``top_p`` keeps the smallest top set whose
probability reaches p (1.0: off), ``min_p`` keeps the tokens with prob >= min_p * max prob (0.0: off).  Ties at a
boundary are kept.  Greedy requests ignore them.
"""
from dataclasses import dataclass


@dataclass(slots=True)
class SamplingParams:
    temperature: float = 1.0
    max_tokens: int = 64
    ignore_eos: bool = False
    top_k: int = -1
    top_p: float = 1.0
    min_p: float = 0.0

    def __post_init__(self):
        if self.temperature < 0:
            raise ValueError("temperature must be >= 0 (0 selects greedy decoding)")
        if self.max_tokens < 1:
            raise ValueError("max_tokens must be >= 1")
        if self.top_k != int(self.top_k) or self.top_k < -1:
            raise ValueError("top_k must be an integer: -1 or 0 (off) or >= 1")
        if not 0.0 < self.top_p <= 1.0:
            raise ValueError("top_p must be in (0, 1] (1 = off)")
        if not 0.0 <= self.min_p <= 1.0:
            raise ValueError("min_p must be in [0, 1] (0 = off)")

    @property
    def greedy(self) -> bool:
        return self.temperature <= 1e-10

    @property
    def filtered(self) -> bool:
        """True when a top-k, top-p or min-p filter is on (it still has no effect on a greedy request)."""
        return self.top_k > 0 or self.top_p < 1.0 or self.min_p > 0.0
