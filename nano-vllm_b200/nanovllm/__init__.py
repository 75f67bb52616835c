"""nanovllm API (LLM / SamplingParams) on the H100-native paged-attention path.

Same public surface as the reference package (reference nanovllm/__init__.py:1-2), so
``from nanovllm import LLM, SamplingParams`` in the reference's bench.py / example.py keeps
working with ``nano-vllm_b200`` on the path instead.
"""
from .sampling_params import SamplingParams
from .llm import LLM

__all__ = ["LLM", "SamplingParams"]
__version__ = "0.1.0+b200"
