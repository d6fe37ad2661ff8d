"""FusedMoE layer composition (SURVEY 8f n4), mirroring xllm::layer::FusedMoEImpl on CUDA
(xllm/core/layers/cuda/fused_moe.cpp:28-117): replicated gate linear -> moe_fused_topk -> gated experts (bf16, unquantised:
all the reference's CUDA FusedMoE accepts, :39-42) -> all-reduce over the MoE-TP group, then over the MoE-EP group
(:116-117).  Any token count: decode batches run the expert GEMVs, prefill steps the grouped GEMMs (ops.cutlass_fused_moe).  Weights: w13 [E_local, 2 * I_local, H] in [up | gate] order (load_experts, :124-126), w2 [E_local, H, I_local];
expert e of the model lives on EP rank e // E_local; the intermediate dimension is split over the TP group."""
from typing import Optional

import torch

from . import ops

BF16 = torch.bfloat16


class FusedMoE:
    def __init__(self, gate_weight: torch.Tensor, w13: torch.Tensor, w2: torch.Tensor, topk: int, renormalize: bool = True,
                 scoring_func: str = "softmax", correction_bias: Optional[torch.Tensor] = None, ep_size: int = 1, ep_rank: int = 0,
                 tp_pg=None, ep_pg=None):
        self.gate_weight, self.w13, self.w2 = gate_weight, w13, w2
        self.topk, self.renormalize, self.scoring_func, self.correction_bias = topk, renormalize, scoring_func, correction_bias
        self.ep_size, self.ep_rank, self.tp_pg, self.ep_pg = ep_size, ep_rank, tp_pg, ep_pg
        self.num_experts = gate_weight.size(0)
        if w13.size(0) * ep_size != self.num_experts:
            raise ValueError("n_routed_experts must be divisible by ep_size (w13 holds this rank's experts)")

    def forward(self, hidden_states: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        # gate: ReplicatedLinear without bias (fused_moe.cpp:70-72); router logits in bf16 as the linear produces them
        router_logits = ops.matmul(hidden_states, self.gate_weight)
        scales, ids = ops.moe_fused_topk(router_logits, self.topk, self.renormalize, self.correction_bias, self.scoring_func)
        y = ops.cutlass_fused_moe(hidden_states, ids, scales, self.w13, self.w2, self.ep_size, self.ep_rank, out)
        if self.tp_pg is not None and self.tp_pg.world_size > 1:
            self.tp_pg.allreduce(y)
        if self.ep_pg is not None and self.ep_pg.world_size > 1:
            self.ep_pg.allreduce(y)
        return y
