"""Read-back probes of the weight-only kernels' group indexing: weights whose every quantisation group dequantises
differently from its neighbours, read back one at a time through identity activations."""
import torch

from oracle import quant as Q

BF16 = torch.bfloat16
# K of the W4 small-M probe: long enough that every k split streams more slots than its ring holds, so both the ring
# prologue and the refill compute meta rows, at every group size from 64 to K (one group per row)
PROBE_K = 8192


def group_probe_weights(N: int, K: int, gs: int, bits: int, seed: int, device="cpu"):
    """(q, scales, zeros) of a weight-only linear for read-back probes: q uniform over the whole range, the scale of group g
    of row n is base_n * 2^(g mod 5) and its zero point (n + 7 g) mod 2^bits, so every group dequantises differently from
    its neighbours and a kernel that reads another group's meta row returns different bits."""
    g = torch.Generator(device=device).manual_seed(seed)
    G = K // gs
    q = torch.randint(0, 1 << bits, (N, K), generator=g, device=device, dtype=torch.uint8)
    base = torch.rand(N, 1, generator=g, device=device) * 0.01 + 0.001
    s = (base * torch.exp2((torch.arange(G, device=device) % 5).float())).to(BF16)
    z = ((torch.arange(N, device=device).unsqueeze(1) + 7 * torch.arange(G, device=device)) % (1 << bits)).to(torch.uint8)
    return q, s, z


def w4_probe(gs, rows=64, N=64, K=PROBE_K, dev="cuda"):
    """x = identity rows picks out single weights of the W4 small-M kernel: y[m, n] = bf16(w[n, k_m]) must equal the spec's
    dequantised weight bit-for-bit (one rounding in (q-z)*s); reading another group's meta row shows.  `rows` one-hot
    tokens per launch."""
    from xllm_b200 import ops, quant
    q, s, z = group_probe_weights(N, K, gs, 4, seed=11)
    wd = Q.dequantize(q, s, z, gs)
    qw, meta = quant.pack_w4(q, s, z, gs)
    qw, meta = qw.to(dev), meta.to(dev)
    eye = torch.eye(K, dtype=BF16, device=dev)
    y = torch.cat([ops.w4a16_linear_small_m(eye[k0:k0 + rows], qw, meta, gs) for k0 in range(0, K, rows)])
    bad = (y.cpu() != wd.t()).nonzero()
    assert bad.numel() == 0, f"gs={gs}: {bad.size(0)} weights differ, first at (k, n) = {tuple(bad[0].tolist())}"
