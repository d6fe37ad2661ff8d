"""Qwen3 dense on CPU: the oracle composition (tests/qwen3_parity.py) against transformers' Qwen3ForCausalLM; the prefill
runner's Qwen3 branch (xllm_b200/qwen2_prefill.py) with the library ops replaced by oracle arithmetic, one rank and
tensor-parallel over gloo; and the argument checks of xb_qk_norm_rope_and_cache_bf16 through the C ABI (no device)."""
import ctypes
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import batch as OB
from oracle import ops as O
from tests import qwen3_parity as Q3
from tests.test_parallel_cpu import _free_port
from tests.test_prefill_composition_cpu import OracleOps, _fresh_caches
from tests.test_tp_prefill_cpu import _shard
from xllm_b200 import parallel as P
from xllm_b200 import qwen2 as Q2
from xllm_b200.qwen2 import Qwen2Config
from xllm_b200.qwen2_prefill import Qwen2PrefillRunner

BF16 = torch.bfloat16
LENS = [5, 9, 1]
BLOCKS = [[3, 1], [6, 2, 5], [4]]
NBLOCKS = 8


class Qwen3OracleOps(OracleOps):
    @staticmethod
    def qk_norm_rope_and_cache(qkv, num_heads_q, num_heads_kv, head_dim, eps, q_weight, k_weight, cos_sin_cache,
                               position_ids, slot_ids, key_cache, value_cache):
        T, D, qs, kvs = qkv.size(0), head_dim, num_heads_q * head_dim, num_heads_kv * head_dim
        qkv.copy_(O.fused_qk_norm_rope(qkv, num_heads_q, num_heads_kv, num_heads_kv, D, eps, q_weight, k_weight,
                                       cos_sin_cache, False, position_ids))
        O.reshape_paged_cache(slot_ids, qkv[:, qs:qs + kvs].reshape(T, num_heads_kv, D),
                              qkv[:, qs + kvs:].reshape(T, num_heads_kv, D), key_cache, value_cache)


def _cfg(vocab=101):
    """q_size 256 over hidden 64: head_dim is not hidden / n_heads"""
    return Qwen2Config(hidden_size=64, num_layers=2, n_heads=4, n_kv_heads=2, head_dim=64, intermediate_size=96,
                       vocab_size=vocab, max_position_embeddings=64, block_size=4, quant="bf16", qkv_bias=False, qk_norm=True,
                       name="tiny-qwen3")


def _prompts(cfg):
    g = torch.Generator().manual_seed(3)
    return [torch.randint(0, cfg.vocab_size, (n,), generator=g).tolist() for n in LENS]


def _hf_state(cfg, W):
    qs, kvs, inter = cfg.q_size, cfg.kv_size, cfg.intermediate_size
    sd = {"model.embed_tokens.weight": W["embed"], "model.norm.weight": W["final_norm"], "lm_head.weight": W["lm_head"]}
    for i, L in enumerate(W["layers"]):
        p = f"model.layers.{i}."
        w = L["qkv"]["w"]
        for name, sl in (("q", slice(0, qs)), ("k", slice(qs, qs + kvs)), ("v", slice(qs + kvs, qs + 2 * kvs))):
            sd[p + f"self_attn.{name}_proj.weight"] = w[sl]
        sd[p + "self_attn.q_norm.weight"], sd[p + "self_attn.k_norm.weight"] = L["q_norm"], L["k_norm"]
        sd[p + "self_attn.o_proj.weight"] = L["o"]["w"]
        sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"] = L["gate_up"]["w"][:inter], L["gate_up"]["w"][inter:]
        sd[p + "mlp.down_proj.weight"] = L["down"]["w"]
        sd[p + "input_layernorm.weight"], sd[p + "post_attention_layernorm.weight"] = L["input_norm"], L["post_norm"]
    return sd


def test_qwen3_oracle_prefill_matches_transformers():
    """pins the q / k norm placement (per head, before RoPE), the bias-free projections and head_dim != hidden / n_heads
    against the published implementation; the bf16 rounding order differs between the stacks, hence a relative-L2 bar"""
    tf = pytest.importorskip("transformers")
    cfg = _cfg(vocab=128)
    W, _, _, _ = Q3.build_case(cfg, 1, [1], seed=7)
    try:
        hf_cfg = tf.Qwen3Config(vocab_size=128, hidden_size=64, intermediate_size=96, num_hidden_layers=2, num_attention_heads=4,
                                num_key_value_heads=2, head_dim=64, max_position_embeddings=64, rms_norm_eps=cfg.rms_norm_eps,
                                rope_theta=float(cfg.rope_theta), tie_word_embeddings=False, attention_bias=False,
                                attention_dropout=0.0, use_sliding_window=False)
        hf_cfg._attn_implementation = "eager"
        model = tf.Qwen3ForCausalLM(hf_cfg).to(BF16).eval()
        res = model.load_state_dict(_hf_state(cfg, W), strict=False)
    except Exception as e:                                                 # constructor surface differs between transformers versions
        pytest.skip(f"transformers Qwen3 not constructible here: {e}")
    assert not res.missing_keys and not res.unexpected_keys, res
    toks = _prompts(cfg)
    meta = OB.build_paged_meta([OB.SeqState(b, 0, n) for b, n in zip(BLOCKS, LENS)], cfg.block_size)
    mk = lambda: [torch.zeros(NBLOCKS, cfg.block_size, cfg.n_kv_heads, cfg.head_dim, dtype=BF16) for _ in range(cfg.num_layers)]
    ours = Q3.oracle_prefill(cfg, W, mk(), mk(), [t for s in toks for t in s], meta, chunked=False)
    with torch.no_grad():
        theirs = torch.stack([model(input_ids=torch.tensor([s])).logits[0, -1] for s in toks])
    rel = ((ours.float() - theirs.float()).norm() / theirs.float().norm()).item()
    assert rel <= 1e-2, f"qwen3: oracle vs transformers logits rel-L2 {rel:.3e}"
    assert torch.equal(ours.float().argmax(-1), theirs.float().argmax(-1))


def _runner_forward(cfg, w, kcs, vcs, tokens, meta, chunked, pg=None):
    r = Qwen2PrefillRunner(cfg, w, kcs, vcs, Q2.make_cos_sin_cache(cfg, "cpu"), device="cpu", pg=pg)
    i32 = lambda v: torch.tensor(v, dtype=torch.int32)
    return r.forward(i32(tokens), torch.tensor(meta.positions, dtype=torch.int64), i32(meta.new_cache_slots),
                     i32(meta.q_cu_seq_lens), i32(meta.kv_cu_seq_lens), i32(meta.paged_kv_indptr), i32(meta.paged_kv_indices),
                     i32(meta.paged_kv_last_page_len), chunked=chunked)


def _one_shot_and_chunked(cfg, w, mk, pg=None):
    """(logits, tokens, caches) of a one-shot prefill of the three prompts, and whether the same prompts in two chunks
    ([first 3 | rest]; prompt 2 finishes in chunk 1) reproduce them exactly."""
    toks, bs = _prompts(cfg), cfg.block_size
    meta = OB.build_paged_meta([OB.SeqState(b, 0, n) for b, n in zip(BLOCKS, LENS)], bs)
    kcs, vcs = mk(), mk()
    logits, tokens = _runner_forward(cfg, w, kcs, vcs, [t for s in toks for t in s], meta, False, pg)
    cut = [3, 3, 1]
    kc2, vc2 = mk(), mk()
    m1 = OB.build_paged_meta([OB.SeqState(b[: (c + bs - 1) // bs], 0, c) for b, c in zip(BLOCKS, cut)], bs)
    _runner_forward(cfg, w, kc2, vc2, [t for s, c in zip(toks, cut) for t in s[:c]], m1, False, pg)
    m2 = OB.build_paged_meta([OB.SeqState(b, c, n) for b, c, n in zip(BLOCKS, cut, LENS) if n > c], bs)
    logits2, tokens2 = _runner_forward(cfg, w, kc2, vc2, [t for s, c, n in zip(toks, cut, LENS) if n > c for t in s[c:]], m2,
                                       True, pg)
    chunk_ok = bool(torch.equal(logits2, logits[:2]) and torch.equal(tokens2, tokens[:2]) and
                    all(torch.equal(a, b) for a, b in zip(kc2 + vc2, kcs + vcs)))
    return logits, tokens, kcs, vcs, chunk_ok


def _oracle(cfg, W):
    toks = _prompts(cfg)
    meta = OB.build_paged_meta([OB.SeqState(b, 0, n) for b, n in zip(BLOCKS, LENS)], cfg.block_size)
    kc_o, vc_o = _fresh_caches(cfg, NBLOCKS)
    ref = Q3.oracle_prefill(cfg, W, kc_o, vc_o, [t for s in toks for t in s], meta, chunked=False)
    return ref, kc_o, vc_o


def test_qwen3_prefill_composition_matches_oracle_and_chunking_is_exact(monkeypatch):
    monkeypatch.setattr(Q2, "ops", Qwen3OracleOps)        # Linear.forward and the runner both resolve ops through qwen2
    cfg = _cfg()
    W, _, _, _ = Q3.build_case(cfg, 1, [1], seed=7)
    ref, kc_o, vc_o = _oracle(cfg, W)
    w = Q3.upload(cfg, W, device="cpu")
    logits, tokens, kcs, vcs, chunk_ok = _one_shot_and_chunked(cfg, w, lambda: _fresh_caches(cfg, NBLOCKS)[0])
    assert torch.equal(logits, ref), "runner composition differs from the oracle composition"
    assert torch.equal(tokens.long(), ref.float().argmax(-1))
    for a, b in zip(kcs + vcs, kc_o + vc_o):
        assert torch.equal(a, b), "KV cache contents differ"
    assert chunk_ok, "chunked prefill must reproduce one-shot prefill exactly"


def _tp_worker(rank, world, port, out_q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    Q2.ops = Qwen3OracleOps                              # Linear.forward and the runner resolve ops through qwen2
    cfg = _cfg(vocab=128)
    W, _, _, _ = Q3.build_case(cfg, 1, [1], seed=7)
    w, hp = _shard(cfg, W, rank, world, shard_embedding=False)
    for L, d in zip(w.layers, W["layers"]):
        L["q_norm"], L["k_norm"] = d["q_norm"], d["k_norm"]   # replicated on every rank, like every other norm weight
    mk = lambda: [torch.zeros(NBLOCKS, cfg.block_size, hp.num_kv_heads, cfg.head_dim, dtype=BF16) for _ in range(cfg.num_layers)]
    logits, tokens, kcs, vcs, chunk_ok = _one_shot_and_chunked(cfg, w, mk, P.ProcessGroup())
    out_q.put((rank, logits.float().numpy(), tokens.numpy(), [k.float().numpy() for k in kcs], [v.float().numpy() for v in vcs],
               chunk_ok))
    dist.barrier()
    dist.destroy_process_group()


def test_qwen3_tp2_prefill_composition_matches_single_rank_oracle():
    """heads partition as for Qwen2 and the norm weights are replicated: two gloo ranks reproduce the single-rank oracle"""
    cfg = _cfg(vocab=128)
    W, _, _, _ = Q3.build_case(cfg, 1, [1], seed=7)
    ref, kc_o, vc_o = _oracle(cfg, W)
    world, ctx = 2, mp.get_context("spawn")
    q, port = ctx.Queue(), _free_port()
    procs = [ctx.Process(target=_tp_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict()
    for _ in range(world):
        item = q.get(timeout=180)
        got[item[0]] = item[1:]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    l0, l1 = torch.from_numpy(got[0][0]), torch.from_numpy(got[1][0])
    assert torch.equal(l0, l1), "ranks disagree on the gathered logits"
    rel = ((l0 - ref.float()).norm() / ref.float().norm()).item()
    # per-rank partial sums are rounded to bf16 before the exchange (the reference's NCCL all-reduce does the same)
    assert rel <= 2e-2, f"TP2 Qwen3 prefill logits rel-L2 {rel:.3e}"
    assert torch.equal(torch.from_numpy(got[0][1]).long(), ref.float().argmax(-1))
    assert got[0][4] and got[1][4], "TP chunked prefill differs from TP one-shot prefill"
    for rank in (0, 1):
        sl = slice(rank, rank + 1)                                   # one kv head per rank
        k0, v0 = torch.from_numpy(got[rank][2][0]), torch.from_numpy(got[rank][3][0])
        assert torch.equal(k0, kc_o[0][:, :, sl].float()) and torch.equal(v0, vc_o[0][:, :, sl].float()), \
            "layer-0 K/V of this rank's heads must be bit-identical to the oracle's"


def test_qk_norm_rope_and_cache_argument_checks(built_lib):
    """rejected before any device access, with a message; num_tokens == 0 is a no-op"""
    from xllm_b200 import _lib
    lib = _lib.lib()
    nz = ctypes.c_void_p(16)          # stands in for a device pointer: never dereferenced on these paths
    f = lib.xb_qk_norm_rope_and_cache_bf16
    call = lambda D, qw, kw, cs, T: f(None, 8, 2, D, ctypes.c_float(1e-6), qw, kw, cs, None, None, None, None, T, None)
    for D in (32, 96, 256):
        assert call(D, nz, nz, nz, 4) != 0 and b"head_dim" in lib.xb_last_error(), D
    for qw, kw, cs in ((None, nz, nz), (nz, None, nz), (nz, nz, None)):
        assert call(128, qw, kw, cs, 4) != 0 and b"null" in lib.xb_last_error()
    assert call(128, nz, nz, nz, 0) == 0
    assert call(64, nz, nz, nz, 0) == 0
    assert call(128, nz, nz, nz, 3) != 0 and b"null pointer" in lib.xb_last_error()     # qkv / positions / caches NULL
