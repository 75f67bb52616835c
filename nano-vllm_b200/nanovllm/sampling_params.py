"""Per-request sampling knobs (reference nanovllm/sampling_params.py:4-11).

Field names and defaults are the reference's.  One deliberate widening: temperature == 0 is
accepted and means greedy argmax (the reference asserts temperature > 1e-10; the north-star's
parity criterion needs greedy token ids).

Extras after the reference's fields, with vLLM's names, meanings and "off" defaults (DESIGN.md 3.3):
``top_k`` keeps the tokens whose logit is >= the k-th largest (-1 or 0: off), ``top_p`` keeps the smallest top set whose
probability reaches p (1.0: off), ``min_p`` keeps the tokens with prob >= min_p * max prob (0.0: off).  Ties at a
boundary are kept.  Greedy requests ignore them.

Then the penalties (DESIGN.md 3.3.1), applied to the logits before temperature and the filters, greedy requests
included: ``presence_penalty`` in [-2, 2] is subtracted from every token generated at least once (0.0: off),
``frequency_penalty`` in [-2, 2] times the number of times it was generated (0.0: off), and ``repetition_penalty`` > 0
divides the positive logits and multiplies the others of every token of the prompt or the output (1.0: off).  They are
keyword-or-positional arguments after ``min_p`` and attributes like the fields, but not dataclass fields:
``dataclasses.fields(SamplingParams)`` stays the published surface of the reference plus the filters.  ``repr``, ``==``,
pickling, ``copy.copy`` and ``copy.replace`` include them.  ``dataclasses.replace`` and ``dataclasses.asdict`` only see the
dataclass fields, so they drop the penalties (``replace`` resets them to off): use ``sp.replace(**changes)`` and
``sp.as_dict()`` instead.

Last, ``logprobs`` (DESIGN.md 3.3.2): None (off) or k in [0, 20].  Each generated token then gets the log_softmax of the raw
logits (before penalties, temperature and filters) for the sampled token, with its rank, and for the k most likely
tokens; ``generate()`` returns them as one ``{token_id: Logprob}`` dict per token.  It is handled like the penalties, but
``as_dict()`` and ``repr`` list it only when it is set.
"""
import math
from dataclasses import dataclass

MAX_LOGPROBS = 20
# vLLM parameters this engine does not implement; any value but "off" is refused
_UNSUPPORTED = {"prompt_logprobs": None, "logprob_token_ids": None, "logprobs_mode": "raw_logprobs"}


@dataclass(frozen=True, slots=True)
class Logprob:
    """One entry of a per-token logprobs dict: the log-probability under the raw logits and the rank (1 = most likely)."""
    logprob: float
    rank: int


class _Penalties:
    __slots__ = ("presence_penalty", "frequency_penalty", "repetition_penalty", "logprobs")


@dataclass(slots=True, init=False, repr=False, eq=False)
class SamplingParams(_Penalties):
    temperature: float = 1.0
    max_tokens: int = 64
    ignore_eos: bool = False
    top_k: int = -1
    top_p: float = 1.0
    min_p: float = 0.0

    def __init__(self, temperature: float = 1.0, max_tokens: int = 64, ignore_eos: bool = False, top_k: int = -1,
                 top_p: float = 1.0, min_p: float = 0.0, presence_penalty: float = 0.0, frequency_penalty: float = 0.0,
                 repetition_penalty: float = 1.0, logprobs: int | None = None, **unsupported):
        for name, value in unsupported.items():
            if name not in _UNSUPPORTED:
                raise TypeError(f"SamplingParams got an unexpected keyword argument {name!r}")
            if value != _UNSUPPORTED[name]:
                raise ValueError(f"{name}={value!r} is not supported (only {_UNSUPPORTED[name]!r})")
        self.temperature = temperature
        self.max_tokens = max_tokens
        self.ignore_eos = ignore_eos
        self.top_k = top_k
        self.top_p = top_p
        self.min_p = min_p
        self.presence_penalty = presence_penalty
        self.frequency_penalty = frequency_penalty
        self.repetition_penalty = repetition_penalty
        self.logprobs = logprobs
        self.__post_init__()

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
        if not -2.0 <= self.presence_penalty <= 2.0:
            raise ValueError("presence_penalty must be in [-2, 2] (0 = off)")
        if not -2.0 <= self.frequency_penalty <= 2.0:
            raise ValueError("frequency_penalty must be in [-2, 2] (0 = off)")
        if not (math.isfinite(self.repetition_penalty) and self.repetition_penalty > 0.0):
            raise ValueError("repetition_penalty must be finite and > 0 (1 = off)")
        lp = self.logprobs
        if lp is not None and (type(lp) is bool or not isinstance(lp, int) or not 0 <= lp <= MAX_LOGPROBS):
            raise ValueError(f"logprobs must be None (off) or an int in [0, {MAX_LOGPROBS}] (the full vocabulary, -1, "
                             "is not supported)")

    _NAMES = ("temperature", "max_tokens", "ignore_eos", "top_k", "top_p", "min_p", "presence_penalty",
              "frequency_penalty", "repetition_penalty")

    def _values(self) -> tuple:
        return tuple(getattr(self, n) for n in self._NAMES) + (self.logprobs,)

    def as_dict(self) -> dict:
        """Every parameter by name, penalties included (``dataclasses.asdict`` omits them); logprobs only when set."""
        d = {n: getattr(self, n) for n in self._NAMES}
        if self.logprobs is not None:
            d["logprobs"] = self.logprobs
        return d

    def replace(self, **changes) -> "SamplingParams":
        """A validated copy with `changes` applied, penalties kept (``dataclasses.replace`` resets them)."""
        unknown = set(changes) - set(self._NAMES) - {"logprobs"}
        if unknown:
            raise TypeError(f"unknown sampling parameters: {sorted(unknown)}")
        return SamplingParams(**{**self.as_dict(), **changes})

    __replace__ = replace                 # copy.replace (Python 3.13+)

    def __repr__(self) -> str:
        return "SamplingParams(" + ", ".join(f"{n}={v!r}" for n, v in self.as_dict().items()) + ")"

    def __eq__(self, other):
        if other.__class__ is not self.__class__:
            return NotImplemented
        return self._values() == other._values()

    @property
    def greedy(self) -> bool:
        return self.temperature <= 1e-10

    @property
    def filtered(self) -> bool:
        """True when a top-k, top-p or min-p filter is on (it still has no effect on a greedy request)."""
        return self.top_k > 0 or self.top_p < 1.0 or self.min_p > 0.0

    @property
    def penalised(self) -> bool:
        """True when a presence, frequency or repetition penalty is on (greedy requests are penalised too)."""
        return self.presence_penalty != 0.0 or self.frequency_penalty != 0.0 or self.repetition_penalty != 1.0
