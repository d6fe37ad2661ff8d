"""Per-expert, vectorised restatement of oracle.moe.fused_moe for the MoE prefill tests (test infrastructure).

oracle.moe.fused_moe walks the (token, expert) pairs one at a time, which is too slow on a CPU for prefill-sized checks
(thousands of tokens).  fused_moe_grouped computes the same arithmetic per expert, the way the grouped-GEMM path does: gather
each local expert's rows, fp32 matmuls for GEMM1, SwiGLU on the fp32 sums rounded once to bf16, GEMM2 rounded to bf16, then
the same fp32 combine in selection order.  Only the summation order inside the two GEMMs differs from fused_moe;
tests/test_moe_prefill_host_cpu.py pins the two against each other."""
import torch

BF16 = torch.bfloat16
F32 = torch.float32


def fused_moe_grouped(x, token_selected_experts, token_final_scales, fc1, fc2, expert_begin=0, return_abs=False, act=None,
                      return_act=False):
    """x [T, H] bf16, ids int32 [T, k], scales fp32 [T, k], fc1 [E_local, 2I, H] ([up | gate]), fc2 [E_local, H, I] -> [T, H]
    bf16, as oracle.moe.fused_moe (return_abs adds the same magnitude sum_k |scale_k y2_k|).  Experts outside
    [expert_begin, expert_begin + E_local) contribute zero.
    act: optional bf16 activations [T, k, I] to run GEMM2 and the combine from (so that a check of the second GEMM does not
    depend on which way the first one's bf16 roundings went); return_act appends the activations used ([T, k, I] bf16,
    zero for pairs of other experts) to the result."""
    T, H = x.shape
    El, I2, _ = fc1.shape
    inter = I2 // 2
    k = token_selected_experts.size(1)
    ids = token_selected_experts.long() - expert_begin
    y2 = torch.zeros(T, k, H, dtype=F32)
    acts = torch.zeros(T, k, inter, dtype=BF16)
    xf = x.to(F32)
    for e in range(El):
        t_idx, k_idx = (ids == e).nonzero(as_tuple=True)
        if t_idx.numel() == 0:
            continue
        if act is None:
            h1 = xf[t_idx] @ fc1[e].to(F32).t()
            up, gate = h1[:, :inter], h1[:, inter:]
            a = ((gate / (1.0 + torch.exp(-gate))) * up).to(BF16)
        else:
            a = act[t_idx, k_idx].to(BF16)
        acts[t_idx, k_idx] = a
        y2[t_idx, k_idx] = (a.to(F32) @ fc2[e].to(F32).t()).to(BF16).to(F32)
    sc = token_final_scales.to(F32)
    acc = torch.zeros(T, H, dtype=F32)
    mag = torch.zeros(T, H, dtype=F32)
    for kk in range(k):
        acc = torch.addcmul(acc, y2[:, kk], sc[:, kk:kk + 1])
        mag += y2[:, kk].abs() * sc[:, kk:kk + 1].abs()
    res = (acc.to(BF16), mag) if return_abs else (acc.to(BF16),)
    if return_act:
        res = res + (acts,)
    return res if len(res) > 1 else res[0]
