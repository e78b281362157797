"""GPU: prompt-lookup speculative decoding (include/emu_b200_spec.h).  The verify attention against an fp32 reference, the
draft and accept kernels against the host restatement, emu_llm_verify rows against teacher-forced emu_llm_decode steps (tiny
model and one LLaMA-33B-width layer), generate(prompt_lookup_num_tokens=k) against plain greedy, graphed against eager, and
the engine's refusals."""
import os
import random

import pytest
import torch

from helpers import assert_bf16_parity
from oracle import emu_oracle as O
from oracle import spec_oracle as S

pytestmark = pytest.mark.gpu


# ---- the verify attention ---------------------------------------------------------------------------------------------------
def _attn_ref(q, kc, vc, row, L, start, indir, scale):
    """fp32: query j of q [n, H, D] over positions start .. L + j of the sequence in cache row `row` (through indir)"""
    n, H, D = q.shape
    T = L + n
    rows = indir[:T].long() if indir is not None else torch.full((T,), row, dtype=torch.long, device=q.device)
    t = torch.arange(T, device=q.device)
    k = kc[rows, :, t].float()                                   # [T, H, D]
    v = vc[rows, :, t].float()
    s = torch.einsum("jhd,thd->hjt", q.float(), k) * scale
    vis = (t[None, :] >= start) & (t[None, :] <= L + torch.arange(n, device=q.device)[:, None])
    s = s.masked_fill(~vis[None], float("-inf"))
    return torch.einsum("hjt,thd->jhd", s.softmax(-1), v).reshape(n, H * D)


@pytest.mark.parametrize("D,H", [(64, 4), (128, 52)])
@pytest.mark.parametrize("ctx", [1, 300, 4096])
def test_attn_verify_matches_fp32(cuda, D, H, ctx):
    from emu_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(ctx + D)
    t_max = ctx + 8 + 5
    for n in range(1, 9):
        L = ctx
        start = 0 if n % 2 else min(L - 1, 3 + n)
        kc = torch.randn(3, H, t_max, D, generator=g, device="cuda").to(torch.bfloat16)
        vc = torch.randn(3, H, t_max, D, generator=g, device="cuda").to(torch.bfloat16)
        indir = None
        row = 1
        if n % 3 == 0:                                           # a scattered row table
            indir = torch.randint(0, 3, (t_max,), generator=g, device="cuda").to(torch.int32)
            indir[L:] = row
        kc[:, :, L + n:] = float("nan")                          # never part of any output
        vc[:, :, L + n:] = float("nan")
        q = torch.randn(n, 3 * H * D, generator=g, device="cuda").to(torch.bfloat16)  # q|k|v rows, q first
        pos = torch.tensor([L], dtype=torch.int32, device="cuda")
        st = torch.tensor([start], dtype=torch.int32, device="cuda")
        scale = D ** -0.5
        out = _lib.op_attn_verify(q, kc, vc, pos, scale, row=row, start=st, indir=indir)
        ref = _attn_ref(q[:, :H * D].view(n, H, D), kc, vc, row, L, start, indir, scale)
        err = ((out.float() - ref).abs().max() / ref.abs().max()).item()   # the kernel-level bf16 bound of the decode ops
        assert err <= 6e-3, (n, D, H, ctx, err)


# ---- draft and accept kernels -----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny(cuda):
    from test_regress_slots_gpu import _tiny_model
    m = _tiny_model(max_batch=8, max_seq=128)
    yield m
    m.engine.close()


def test_draft_and_accept_kernels_match_restatement(tiny):
    eng = tiny.engine
    rng = random.Random(1)
    i32 = dict(dtype=torch.int32, device="cuda")
    for _ in range(200):
        n = rng.randint(1, 300)
        vocab = rng.choice([3, 7, 40])
        h = [rng.randrange(vocab) for _ in range(n)]
        k, gsz, eos = rng.randint(1, 7), rng.randint(1, 3), rng.randrange(vocab)
        max_length = rng.choice([n + 1, n + 3, n + 400, max(1, n - 2)])
        hist = torch.tensor(h + [0] * 16, **i32)
        hist_len = torch.tensor([n], **i32)
        out = torch.full((k + 1,), -1, **i32)
        out_len = torch.zeros(1, **i32)
        eng.spec_draft(hist, hist_len, k, gsz, max_length, eos, out, out_len)
        d = S.prompt_lookup_draft(h, k, gsz, max_length, eos)
        assert int(out_len) == len(d) and out[:1 + len(d)].tolist() == [h[-1]] + d, (h, k, gsz, max_length, eos)
        # accept against arg-max rows that follow the draft for a random number of tokens
        nv = len(d) + 1
        nxt = [d[j] if j < len(d) and rng.random() < 0.7 else rng.randrange(vocab) for j in range(nv)]
        cap = n + rng.randint(1, 10)
        stats = torch.zeros(2, **i32)
        eng.spec_accept(hist, hist_len, out, torch.tensor(nxt, **i32), nv, eos, cap, stats)
        hh = list(h)
        m, done = S.accept(hh, d, nxt, eos, cap)
        assert stats.tolist() == [m, int(done)] and int(hist_len) == len(hh) and hist[:len(hh)].tolist() == hh


# ---- verify against teacher-forced decode -----------------------------------------------------------------------------------
def _teacher_forced(eng, emb, mask, toks):
    """prefill + one decode step per token: the logits after each token and the K/V the steps wrote"""
    eng.llm_reset()
    eng.llm_prefill(emb, mask, hf_positions=True, want_logits=True)
    L = eng.cur_len()
    buf = torch.empty(1, eng.cfg.llm_vocab, dtype=torch.float32, device="cuda")
    outs = []
    for t in toks:
        eng.llm_decode(token_ids=torch.tensor([t], dtype=torch.int32, device="cuda"), logits=buf, B=1)
        outs.append(buf[0].clone())
    return torch.stack(outs), eng.kv_cache()[:, :, 0, :, L:L + len(toks)].clone()


def _verified(eng, emb, mask, toks):
    eng.llm_reset()
    eng.llm_prefill(emb, mask, hf_positions=True, want_logits=True)
    L = eng.cur_len()
    n = len(toks)
    lg = torch.empty(n, eng.cfg.llm_vocab, dtype=torch.float32, device="cuda")
    nxt = torch.empty(n, dtype=torch.int32, device="cuda")
    eng.llm_verify(torch.tensor(toks, dtype=torch.int32, device="cuda"), n, logits=lg, next_ids=nxt)
    assert eng.cur_len() == L
    assert torch.equal(nxt.long(), lg.argmax(-1))
    eng.llm_commit(n)
    assert eng.cur_len() == L + n
    return lg, eng.kv_cache()[:, :, 0, :, L:L + n].clone()


def test_verify_rows_match_decode_tiny(tiny):
    eng = tiny.engine
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(0, 32000, (1, 20), generator=g)
    emb = eng.llm_embed(ids.cuda())
    mask = torch.ones(1, 20, dtype=torch.long, device="cuda")
    mask[0, :3] = 0
    toks = torch.randint(0, 32000, (8,), generator=g).tolist()
    for n in (1, 3, 8):
        ref, kv_ref = _teacher_forced(eng, emb, mask, toks[:n])
        got, kv_got = _verified(eng, emb, mask, toks[:n])
        assert O.rel_err(got, ref) <= 2e-2, (n, O.rel_err(got, ref))
        assert O.rel_err(kv_got.float(), kv_ref.float()) <= 2e-2


def test_verify_llama33b_layer(cuda):
    from helpers import VOCAB, StubTokenizer, TINY_VISION
    from test_realshape_gpu import LLAMA_33B_1L, _bf16, _llama_sd, _oracle_llama_steps
    from emu_b200.emu2.conf import CLIPVisionCfg, TextDecoderCfg
    from emu_b200.emu2.emu import EmuModel
    cfg = LLAMA_33B_1L
    sd = _llama_sd(cfg, VOCAB, seed=21)
    m = EmuModel(CLIPVisionCfg(**dict(TINY_VISION, layers=1)), TextDecoderCfg(), tokenizer=StubTokenizer(), llama_config=cfg,
                 max_batch=8, max_seq=96)
    for k, v in sd.items():
        m.engine.load_tensor(k, v)
    g = torch.Generator().manual_seed(22)
    N, n = 75, 6
    emb = torch.randn(1, N, cfg["hidden_size"], generator=g).to(torch.bfloat16)
    mask = torch.ones(1, N, dtype=torch.long)
    mask[0, :7] = 0
    toks = torch.randint(100, 31000, (1, n), generator=g)
    with torch.no_grad():
        ref32 = _oracle_llama_steps(sd, emb.float(), mask, toks, cfg["num_attention_heads"])
        ref16 = _oracle_llama_steps(_bf16(sd), emb, mask, toks, cfg["num_attention_heads"])
    eng = m.engine
    dec, kv_dec = _teacher_forced(eng, emb.cuda(), mask.cuda(), toks[0].tolist())
    got, kv_got = _verified(eng, emb.cuda(), mask.cuda(), toks[0].tolist())
    for j in range(n):
        assert_bf16_parity("llama33b layer verify row %d" % j, got[j:j + 1].cpu(), ref32[j + 1], ref16[j + 1])
        assert_bf16_parity("llama33b layer decode step %d" % j, dec[j:j + 1].cpu(), ref32[j + 1], ref16[j + 1])
    assert O.rel_err(kv_got.float(), kv_dec.float()) <= 2e-2
    eng.close()


# ---- end to end ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 4, 7])
def test_generate_equals_plain_greedy(tiny, k):
    from emu_b200 import generation
    eng = tiny.engine
    g = torch.Generator().manual_seed(7)
    base = torch.randint(0, 32000, (1, 6), generator=g)
    ids = torch.cat([base] * 4, 1).cuda()                   # repetitive: the prompt offers drafts
    emb = eng.llm_embed(ids)
    mask = torch.ones_like(ids)
    plain = generation.generate(eng, emb, mask, 40, 2, 32000, num_beams=1)
    spec = generation.generate(eng, emb, mask, 40, 2, 32000, num_beams=1, prompt_lookup_num_tokens=k, prompt_ids=ids)
    guided = generation.generate(eng, emb, mask, 40, 2, 32000, num_beams=1, prompt_lookup_num_tokens=k,
                                 prompt_ids=torch.cat((ids, plain.to(ids.dtype)), 1))
    for out in (spec, guided):
        if torch.equal(out, plain):
            continue
        # a divergence is allowed only at a near tie of the teacher-forced logits
        t = int((out[0, :min(out.shape[1], plain.shape[1])] != plain[0, :min(out.shape[1], plain.shape[1])]).nonzero()[0])
        lg, _ = _teacher_forced(eng, emb, mask, plain[0, :t].tolist()) if t > 0 else (None, None)
        row = lg[-1] if t > 0 else eng.llm_prefill(emb, mask)[1][0]
        lp = torch.log_softmax(row.float(), -1)
        assert float(lp[plain[0, t]] - lp[out[0, t]]) <= 1e-2 * float(lp.abs().max()), (k, t)


def test_graphed_verify_equals_eager(tiny):
    eng = tiny.engine
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(0, 32000, (1, 12), generator=g).cuda()
    emb = eng.llm_embed(ids)
    mask = torch.ones_like(ids)
    toks = torch.randint(0, 32000, (5,), generator=g).tolist()
    graphed, kv_g = _verified(eng, emb, mask, toks)
    os.environ["EMU_NO_GRAPH"] = "1"
    try:
        eager, kv_e = _verified(eng, emb, mask, toks)
    finally:
        del os.environ["EMU_NO_GRAPH"]
    assert torch.equal(graphed, eager) and torch.equal(kv_g, kv_e)


def test_engine_refusals(tiny):
    from emu_b200._lib import EmuError
    eng = tiny.engine
    toks = torch.zeros(9, dtype=torch.int32, device="cuda")
    nxt = torch.zeros(9, dtype=torch.int32, device="cuda")
    eng.llm_reset()
    with pytest.raises(EmuError, match="before prefill"):
        eng.llm_verify(toks, 2, next_ids=nxt)
    with pytest.raises(EmuError, match="commit without a verify"):
        eng.llm_commit(1)
    emb = eng.llm_embed(torch.zeros(2, 120, dtype=torch.long, device="cuda"))
    eng.llm_prefill(emb, None)
    with pytest.raises(EmuError, match="batch 1"):
        eng.llm_verify(toks, 2, next_ids=nxt)
    eng.llm_reset()
    eng.llm_prefill(emb[:1], None)
    with pytest.raises(EmuError, match="outside"):
        eng.llm_verify(toks, 9, next_ids=nxt)
    eng.llm_verify(toks, 4, next_ids=nxt)
    with pytest.raises(EmuError, match="outside"):
        eng.llm_commit(5)
    eng.llm_commit(4)
    with pytest.raises(EmuError, match="KV cache full"):
        eng.llm_verify(toks, 5, next_ids=nxt)
    with pytest.raises(EmuError, match="commit without a verify"):
        eng.llm_commit(1)
    eng.slots_begin(2)
    with pytest.raises(EmuError, match="slot mode") as ei:
        eng.llm_verify(toks, 2, next_ids=nxt)
    assert "state" in str(ei.value).lower()
    eng.llm_reset()
