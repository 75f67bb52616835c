"""Qwen3 mixture-of-experts decoder (Qwen3-30B-A3B; HF ``Qwen3MoeForCausalLM``, DESIGN.md 3.7).

Attention, norms, embedding, LM head and tensor parallelism are the dense model's (models/qwen3.py); only the MLP of every
layer is a ``Qwen3MoeSparseMoeBlock``: a router picks the top k of E experts per token and the token's MLP output is the
routing-weighted sum of those experts' SwiGLU MLPs.  Per layer and step that is

    router GEMM (library) -> route -> align -> gather -> grouped gate_up + SiluAndMul -> grouped down -> combine

on the kernels of csrc/moe.cu and the grouped mode of csrc/linear_tc.cu (ops.moe_mlp).  Under tensor parallelism each
expert is sharded along moe_intermediate_size exactly like the dense MLP, and each rank's combined output goes through the
same all-reduce + add + RMSNorm as a dense down_proj.

The dense opt-in experiments B200_LINEAR=tc / gu (gate_up on wgmma), B200_TAIL=mega and B200_DUAL replace the dense MLP and
are ignored here; o_proj keeps its dense path, and B200_LM_HEAD=fused (the LM head) works as for dense models.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .. import ops
from .qwen3 import LayerWeights, Qwen3ForCausalLM

# k tile of the grouped GEMMs: hidden (gate_up's k) and moe_intermediate_size / tp (down's k, gate_up's n) are whole tiles
_TILE_K = 64


def check_moe_config(c, tp_size: int = 1) -> None:
    """Refuse, before any weight is read, what the MoE path does not implement (NotImplementedError)."""
    if getattr(c, "quantization_config", None) is not None:
        raise NotImplementedError("quantization_config on a Qwen3 MoE checkpoint: FP8 mixture-of-experts weights are not supported")
    if list(getattr(c, "mlp_only_layers", None) or []):
        raise NotImplementedError(f"mlp_only_layers {list(c.mlp_only_layers)}: every layer must be a mixture-of-experts layer")
    if getattr(c, "decoder_sparse_step", 1) != 1:
        raise NotImplementedError(f"decoder_sparse_step {c.decoder_sparse_step}: every layer must be a mixture-of-experts layer")
    e, k, inter = c.num_experts, c.num_experts_per_tok, c.moe_intermediate_size
    if not 1 <= e <= ops.MOE_MAX_EXPERTS or not 1 <= k <= min(e, ops.MOE_MAX_TOPK):
        raise NotImplementedError(f"num_experts {e} / num_experts_per_tok {k}: the kernels take at most "
                                  f"{ops.MOE_MAX_EXPERTS} experts and {ops.MOE_MAX_TOPK} per token")
    if inter % tp_size or (inter // tp_size) % _TILE_K or c.hidden_size % _TILE_K:
        raise NotImplementedError(f"moe_intermediate_size / tp = {inter} / {tp_size} and hidden_size {c.hidden_size} must be "
                                  f"multiples of {_TILE_K}")


def model_class(hf_config):
    """The decoder class of a config: Qwen3MoeForCausalLM for model_type "qwen3_moe", else the dense Qwen3ForCausalLM."""
    return Qwen3MoeForCausalLM if getattr(hf_config, "model_type", "qwen3") == "qwen3_moe" else Qwen3ForCausalLM


class Qwen3MoeForCausalLM(Qwen3ForCausalLM):
    def __init__(self, hf_config, tp_rank: int = 0, tp_size: int = 1, device="cuda", max_position: int | None = None):
        c = hf_config
        check_moe_config(c, tp_size)
        self.num_experts, self.top_k = c.num_experts, c.num_experts_per_tok
        self.norm_topk = bool(getattr(c, "norm_topk_prob", True))
        super().__init__(hf_config, tp_rank, tp_size, device, max_position)
        self.tc_gate_up = self.mega_tail = self.dual = False      # dense-MLP experiments (module docstring)
        for L in self.layers:
            L.gate = torch.empty(self.num_experts, self.hidden, dtype=torch.bfloat16, device=self.device)

    @staticmethod
    def _intermediate_size(c) -> int:
        return c.moe_intermediate_size

    def _mlp_shapes(self) -> list[tuple]:
        return [(self.num_experts, 2 * self.inter, self.hidden), (self.num_experts, self.hidden, self.inter)]

    def load_hf_tensor(self, name: str, w: torch.Tensor) -> None:
        """The router ``mlp.gate.weight`` and the Hub's per-expert ``mlp.experts.{e}.{gate,up,down}_proj.weight`` into the
        stacked tensors, each expert sliced to this rank's shard as the dense gate/up/down are; the rest as the dense model."""
        parts = name.split(".")
        if len(parts) < 5 or parts[:2] != ["model", "layers"] or parts[3] != "mlp":
            return super().load_hf_tensor(name, w)
        L, r, n, inter = self.layers[int(parts[2])], self.tp_rank, self.tp_size, self.inter
        leaf = ".".join(parts[4:])
        if leaf == "gate.weight":
            L.gate.copy_(w)
            return
        if len(parts) == 8 and parts[4] == "experts" and parts[7] == "weight" and 0 <= int(parts[5]) < self.num_experts:
            e, proj = int(parts[5]), parts[6]
            if proj == "gate_proj":
                L.gate_up[e, :inter].copy_(w.chunk(n, 0)[r])
                return
            if proj == "up_proj":
                L.gate_up[e, inter:].copy_(w.chunk(n, 0)[r])
                return
            if proj == "down_proj":
                L.down[e].copy_(w.chunk(n, 1)[r])
                return
        raise KeyError(f"unexpected checkpoint tensor {name}")

    def _mlp(self, L: LayerWeights, x: torch.Tensor, ctx, tc: bool, big: bool):
        """Qwen3MoeSparseMoeBlock on the normalised x; returns (partial, where) as the dense _mlp (no split-K partials)."""
        t, peer = x.shape[0], self.peer
        logits = F.linear(x, L.gate)
        out = peer.next_out(t) if peer is not None and t <= peer.rows_cap else None
        h = ops.moe_mlp(x, logits, L.gate_up, L.down, self.top_k, self.norm_topk, pdl=bool(self.tc_cfg[6]), out=out)
        return h, out is not None
