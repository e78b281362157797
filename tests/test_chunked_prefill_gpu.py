"""GPU: chunked prefill in slot mode (include/emu_b200_chunked.h) — the mixed decode + prefill step.

The stand-alone kernels must match their torch restatements (and write nothing they do not own); a mixed step's segments
must agree with the fp32 oracle as closely as a bf16 run does, in one chunk or several; its decode rows must agree with
emu_llm_decode of the same tokens; every cache position outside the step's writes must stay bitwise as it was; and the
scheduler with prefill_chunk must agree with a teacher-forced replay."""
import math

import pytest
import torch

from helpers import TINY_LLAMA, TINY_VISION, VOCAB, StubTokenizer, assert_bf16_parity, make_emu2_state_dict
from oracle import emu_oracle as O

pytestmark = pytest.mark.gpu
L, NH = TINY_LLAMA["num_hidden_layers"], TINY_LLAMA["num_attention_heads"]


@pytest.fixture(scope="module")
def sd():
    return make_emu2_state_dict()


@pytest.fixture(scope="module")
def refs(sd):
    return {k: v.to(torch.bfloat16) for k, v in sd.items()}


@pytest.fixture(scope="module")
def model(cuda, sd):
    from emu_b200.emu2.conf import CLIPVisionCfg, TextDecoderCfg
    from emu_b200.emu2.emu import EmuModel
    m = EmuModel(CLIPVisionCfg(**TINY_VISION), TextDecoderCfg(), tokenizer=StubTokenizer(), llama_config=TINY_LLAMA,
                 max_batch=16, max_seq=384)
    m.load_state_dict(sd)
    return m


def _emb(n, seed, H=TINY_LLAMA["hidden_size"]):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(1, n, H, generator=g) * 0.5).to(torch.bfloat16)


def _oracle_last(sd, emb, heads=NH, layers=L, cache=None):
    m = torch.ones(1, emb.shape[1], dtype=torch.long)
    h = O.llama_forward(sd, emb, m, layers=layers, heads=heads, position_ids=O.hf_position_ids(m), cache=cache)
    return O.lm_logits(sd, h[:, -1]).float()


def _interleave(t, kv):
    if kv == 1:
        return t
    half = t.shape[-1] // 2
    return torch.stack([t[..., :half], t[..., half:]], dim=-1).flatten(-2)


def _i32(x):
    return torch.tensor(x, dtype=torch.int32, device="cuda")


def _chunks(n, k):
    """n tokens in k chunks as even as possible"""
    base, extra = divmod(n, k)
    return [base + (1 if i < extra else 0) for i in range(k)]


# ---- the stand-alone kernels ----
def _rot(x, c, s_):
    a, b = x[..., 0::2].float(), x[..., 1::2].float()
    r = lambda t: t.to(torch.bfloat16).float()
    lo, hi = (r(a * c) + r(-b * s_)).to(torch.bfloat16), (r(b * c) + r(a * s_)).to(torch.bfloat16)
    return torch.stack([lo, hi], -1).flatten(-2)


# B = 0: a join or an extend, segments only, each at its own cache row, first slot and position offset
@pytest.mark.parametrize("D,B", [(64, 4), (128, 4), (64, 0), (128, 0)], ids=["64", "128", "segments64", "segments128"])
def test_packed_rope_kv_write_matches_a_torch_restatement(cuda, D, B):
    """decode rows rotated at pos - pos_off, q compact, k / v written only for live rows; segment rows rotated at q0 + j -
    posoff, q in place, k / v at their slots; rows past the last segment and every other cache position untouched"""
    from emu_b200 import _lib
    g = torch.Generator().manual_seed(D if B else D + 1)
    H, T, rows = 2, 64, 6
    half, max_pos = D // 2, T + 8
    ang = torch.arange(max_pos)[:, None].float() / (10000 ** (torch.arange(half).float() * 2 / D))
    cos, sin = ang.cos().to(torch.bfloat16), ang.sin().to(torch.bfloat16)
    if B:
        pos, pos_off, active = [12, 30, 7, 20], [0, 3, 0, 5], [1, 0, 1, 0]        # rows 1 and 3 are not live
        seg_row, seg_q0, seg_new, seg_posoff = [1, 5, 3], [30, 0, 20], [5, 1, 9], [3, 0, 2]
    else:
        pos = pos_off = active = []
        seg_row, seg_q0, seg_new, seg_posoff = [4, 1, 2], [10, 0, 40], [9, 1, 5], [2, 0, 7]
    M = B + sum(seg_new) + 2                                                      # two rows past the last segment
    qkv = torch.randn(M, 3 * H * D, generator=g).to(torch.bfloat16)
    kc = torch.randn(rows, H, T, D, generator=g).to(torch.bfloat16)
    vc = torch.randn(rows, H, T, D, generator=g).to(torch.bfloat16)
    q_out = torch.zeros(B, H * D, dtype=torch.bfloat16)
    got_q, got_k, got_v, got_o = qkv.cuda(), kc.cuda(), vc.cuda(), q_out.cuda()
    dec = (_i32(pos), _i32(pos_off), _i32(active), got_o) if B else (None, None, None, None)
    _lib.op_rope_kv_write_packed(got_q, H, D, cos.cuda(), sin.cuda(), got_k, got_v, B, *dec, _i32(seg_row), _i32(seg_q0),
                                 _i32(seg_new), _i32(seg_posoff))
    want_q, want_k, want_v, want_o = qkv.clone(), kc.clone(), vc.clone(), q_out.clone()
    for b in range(B):
        p = pos[b]
        c, s_ = cos[p - pos_off[b]].float(), sin[p - pos_off[b]].float()
        t = qkv[b].view(3, H, D)
        want_o[b] = _rot(t[0], c, s_).flatten()
        if active[b]:
            want_k[b, :, p] = _rot(t[1], c, s_)
            want_v[b, :, p] = t[2]
    m = B
    for i in range(len(seg_row)):
        for j in range(seg_new[i]):
            p = seg_q0[i] + j
            c, s_ = cos[p - seg_posoff[i]].float(), sin[p - seg_posoff[i]].float()
            t = qkv[m].view(3, H, D)
            want_q[m, :H * D] = _rot(t[0], c, s_).flatten()
            want_k[seg_row[i], :, p] = _rot(t[1], c, s_)
            want_v[seg_row[i], :, p] = t[2]
            m += 1
    assert torch.equal(got_o.cpu(), want_o)
    assert torch.equal(got_k.cpu(), want_k) and torch.equal(got_v.cpu(), want_v)   # nothing for rows 1 and 3, nothing else
    assert torch.equal(got_q.cpu()[B:], want_q[B:])                                  # segments in place, the tail untouched


def _attn_ref(q, k, v, q_off, kv_start, scale):
    Nq, H, D = q.shape
    s = torch.einsum("qhd,khd->hqk", q.float(), k.float()) * scale
    i = torch.arange(Nq)[:, None] + q_off
    j = torch.arange(k.shape[0])[None, :]
    s = s.masked_fill((j > i) | (j < kv_start), float("-inf"))
    return torch.einsum("hqk,khd->qhd", torch.softmax(s, -1).nan_to_num(), v.float())


# NqX: segments of X, X - 3 and X / 2 queries (a join or an extend's suffixes); below 128 queries the mma.sync kernel runs
@pytest.mark.parametrize("lens", [(1, 7, 64), (129, 1, 7, 64), (7, 4, 3), (64, 61, 32), (129, 126, 64), (200, 197, 100)],
                         ids=["mma", "wgmma", "Nq7", "Nq64", "Nq129", "Nq200"])
@pytest.mark.parametrize("D", [64, 128])
def test_packed_attention_matches_torch(cuda, lens, D):
    """segments packed with gaps between them into one q view at their own key offsets; K/V read through kv_row with NaN in
    every key at or past a segment's end; each segment's rows equal the reference, the gaps stay as they were"""
    from emu_b200 import _lib
    g = torch.Generator().manual_seed(D + len(lens))
    H, rows = 4, 6
    n = len(lens)
    q_off = [0, 50, 131, 9][:n]
    kv_start = [0, 3, 17, 0][:n]
    kv_row = [4, 0, 2, 5][:n]
    q_row0, r = [], 3
    for k in lens:
        q_row0.append(r)
        r += k + 2                                                  # two rows of gap after each segment
    Mrows = r
    Nk = max(o + k for o, k in zip(q_off, lens)) + 5
    q = torch.randn(Mrows, H, D, generator=g).to(torch.bfloat16)
    k = torch.randn(rows, Nk, H, D, generator=g).to(torch.bfloat16)
    v = torch.randn(rows, Nk, H, D, generator=g).to(torch.bfloat16)
    for b in range(n):
        end = q_off[b] + lens[b]
        k[kv_row[b], end:] = float("nan")
        v[kv_row[b], end:] = float("nan")
    scale = 1 / math.sqrt(D)
    sentinel = torch.full((Mrows, H, D), 7.0, dtype=torch.bfloat16, device="cuda")
    got = _lib.op_attn_prefill_packed(q.cuda(), k.cuda(), v.cuda(), scale, _i32(q_row0), _i32(list(lens)), _i32(q_off),
                                      _i32(kv_start), _i32(kv_row), Nq=max(lens), out=sentinel).float().cpu()
    covered = torch.zeros(Mrows, dtype=torch.bool)
    for b in range(n):
        r0, m = q_row0[b], lens[b]
        covered[r0:r0 + m] = True
        want = _attn_ref(q[r0:r0 + m], k[kv_row[b]].nan_to_num(0.0), v[kv_row[b]].nan_to_num(0.0), q_off[b], kv_start[b], scale)
        assert torch.isfinite(got[r0:r0 + m]).all(), b
        err = (got[r0:r0 + m] - want).abs().max().item()
        assert err < 2e-2, (b, err)
    assert (got[~covered] == 7.0).all()                             # rows outside every segment are never written


# ---- the mixed step against its parts ----
@pytest.mark.parametrize("chunks", [1, 2, 5])
@pytest.mark.parametrize("n", [37, 150])
def test_step_segments_match_the_oracle(model, sd, refs, n, chunks):
    """a prompt prefilled by `chunks` mixed steps (a live slot decoding in every one) gives last-token logits and K / V within
    the bf16 bound of the fp32 oracle; until its last chunk the slot is kept at the length prefilled so far"""
    eng = model.engine
    x = _emb(n, 10 * n + chunks)
    c32, c16 = O.KVCache(L), O.KVCache(L)
    ref32 = _oracle_last(sd, x.float(), cache=c32)
    ref16 = _oracle_last(refs, x, cache=c16)
    eng.slots_begin(6)
    eng.join([4], _emb(20, 3).cuda())                                # a live neighbour above the segment's slot
    tok = torch.full((6,), 11, dtype=torch.int32, device="cuda")
    buf = torch.empty(6, VOCAB, dtype=torch.float32, device="cuda")
    done = 0
    for i, k in enumerate(_chunks(n, chunks)):
        final = i == chunks - 1
        got = eng.step([2], [done], [k], [final], x[0, done:done + k].cuda(), token_ids=tok, B=5, logits=buf)
        done += k
        if not final:
            assert eng.slot_len(2) == 0 and eng.slot_kept(2) == done
    assert eng.slot_len(2) == n and eng.slot_kept(2) == 0 and eng.slot_len(4) == 20 + chunks
    assert_bf16_parity("step n=%d chunks=%d" % (n, chunks), got.cpu(), ref32, ref16)
    new = eng.kv_cache()[:, :, 2, :, :n].float().cpu()
    for kv, name in ((0, "K"), (1, "V")):
        want32 = torch.stack([_interleave((c32.k if kv == 0 else c32.v)[l][0], kv) for l in range(L)])
        want16 = torch.stack([_interleave((c16.k if kv == 0 else c16.v)[l][0], kv) for l in range(L)]).float()
        assert_bf16_parity("step %s n=%d chunks=%d" % (name, n, chunks), new[:, kv], want32, want16)


def _live_state(eng, n_slots=8):
    """slot 1 live, a 3-beam group in slots 4..6 (joined into 4, forked), slot 0 kept (mid-prefill of 40 tokens)"""
    eng.slots_begin(n_slots)
    eng.join([1], _emb(33, 1).cuda())
    eng.join([4], _emb(21, 2).cuda())
    eng.fork(4, [5, 6])
    eng.step([0], [0], [40], [False], _emb(40, 3)[0].cuda())


def test_decode_rows_match_emu_llm_decode(model):
    eng = model.engine
    tok = torch.tensor([7, 8, 9, 10, 11, 12, 13, 14], dtype=torch.int32, device="cuda")
    src = torch.tensor([0, 1, 2, 3, 5, 4, 4, 7], dtype=torch.int32, device="cuda")
    ref = torch.empty(8, VOCAB, dtype=torch.float32, device="cuda")
    _live_state(eng)
    eng.llm_decode(token_ids=tok, beam_src=src, logits=ref, B=7)
    got = torch.empty(8, VOCAB, dtype=torch.float32, device="cuda")
    _live_state(eng)
    eng.step([0, 3], [40, 0], [9, 17], [False, True], torch.cat([_emb(9, 4), _emb(17, 5)], 1)[0].cuda(), token_ids=tok, B=7,
             beam_src=src, logits=got)
    for s in (1, 4, 5, 6):                                          # the live rows; the others are meaningless
        err = float((got[s] - ref[s]).abs().max() / ref[s].abs().max())
        assert err < 2e-2, (s, err)


def test_every_position_outside_the_steps_writes_is_unchanged(model):
    """a mid-prefill slot (0) below live slots, a live beam group re-parented in the same step, a fresh segment (3) and free
    and kept rows below B: the step writes K / V only at each live slot's next position and each segment's new positions"""
    eng = model.engine
    _live_state(eng, 10)
    eng.join([8], _emb(12, 6).cuda())
    eng.leave_keep([8], [12])                                       # a kept row below B, not in the step
    lens = {s: eng.slot_len(s) for s in range(10)}
    written = [(s, lens[s], lens[s] + 1) for s in (1, 4, 5, 6)] + [(0, 40, 49), (3, 0, 17)]
    for s, a, b in written:                                          # a sentinel where the step must write (nothing reads
        eng.kv_cache()[:, :, s, :, a:b] = 7.0                        # those positions before the step writes them)
    before = eng.kv_cache().clone()
    tok = torch.arange(10, dtype=torch.int32, device="cuda") + 5
    src = torch.tensor([0, 1, 2, 3, 6, 4, 5, 7, 8, 9], dtype=torch.int32, device="cuda")
    logits = torch.empty(10, VOCAB, dtype=torch.float32, device="cuda")
    eng.step([0, 3], [40, 0], [9, 17], [True, False], torch.cat([_emb(9, 4), _emb(17, 5)], 1)[0].cuda(), token_ids=tok, B=10,
             beam_src=src, logits=logits)
    after = eng.kv_cache()
    for s, a, b in written:
        assert not (after[:, :, s, :, a:b] == 7.0).any(), s
        after[:, :, s, :, a:b] = before[:, :, s, :, a:b]
    assert torch.equal(after, before)
    assert eng.slot_len(0) == 49 and eng.slot_kept(3) == 17 and eng.slot_kept(8) == 12
    assert [eng.slot_len(s) for s in (1, 4, 5, 6)] == [lens[s] + 1 for s in (1, 4, 5, 6)]


def test_step_refuses_what_it_cannot_do(model):
    from emu_b200._lib import EmuError
    eng = model.engine
    _live_state(eng)
    x = _emb(4, 9)[0].cuda()
    tok = torch.zeros(8, dtype=torch.int32, device="cuda")
    with pytest.raises(EmuError, match="slot 1 is occupied"):
        eng.step([1], [0], [4], [True], x)
    with pytest.raises(EmuError, match="highest live slot 6"):
        eng.step([2], [0], [4], [True], x, token_ids=tok, B=5)
    with pytest.raises(EmuError, match="slot 0 keeps 40"):
        eng.step([0], [41], [4], [True], x)
    with pytest.raises(EmuError, match="slot 2"):
        eng.step([2], [0], [384], [False], _emb(384, 1)[0].cuda())     # a kept slot holds at most llm_max_seq - 1


# ---- one real LLaMA-33B layer ----
@pytest.mark.parametrize("P,S", [(75, 37), (133, 129)])
def test_llama33b_layer_step(cuda, P, S):
    """the prompt in two mixed steps (P tokens, then S), a live slot decoding in both"""
    from test_realshape_gpu import LLAMA_33B_1L, _llama_sd
    from emu_b200.emu2.conf import CLIPVisionCfg, TextDecoderCfg
    from emu_b200.emu2.emu import EmuModel
    cfg = LLAMA_33B_1L
    sd = _llama_sd(cfg, VOCAB, seed=21)
    m = EmuModel(CLIPVisionCfg(**dict(TINY_VISION, layers=1)), TextDecoderCfg(), tokenizer=StubTokenizer(), llama_config=cfg,
                 max_batch=2, max_seq=320)
    for k, v in sd.items():
        m.engine.load_tensor(k, v)
    x = (torch.randn(1, P + S, cfg["hidden_size"], generator=torch.Generator().manual_seed(P)) * 0.5).to(torch.bfloat16)
    heads = cfg["num_attention_heads"]
    with torch.no_grad():
        ref32 = _oracle_last(sd, x.float(), heads=heads, layers=1)
        ref16 = _oracle_last({k: v.to(torch.bfloat16) for k, v in sd.items()}, x, heads=heads, layers=1)
    eng = m.engine
    eng.slots_begin(2)
    eng.join([0], x[:, :16].cuda())
    tok = torch.tensor([5, 6], dtype=torch.int32, device="cuda")
    buf = torch.empty(2, VOCAB, dtype=torch.float32, device="cuda")
    eng.step([1], [0], [P], [False], x[0, :P].cuda(), token_ids=tok, B=1, logits=buf)
    got = eng.step([1], [P], [S], [True], x[0, P:].cuda(), token_ids=tok, B=1, logits=buf).cpu()
    assert torch.isfinite(buf[0]).all()
    assert_bf16_parity("llama33b layer step %d+%d" % (P, S), got, ref32, ref16)
    eng.close()


# ---- the scheduler on the engine ----
@pytest.mark.parametrize("chunk", [16, 128])
def test_staggered_chunked_schedule_agrees_with_a_teacher_forced_replay(model, chunk):
    """greedy and 5-beam requests with pictures arriving while others decode, prefilled in chunks inside their decode steps:
    the logits every greedy request selects from are within the bf16 bound of a plain prefill + decode of its own tokens"""
    import os
    from emu_b200.batching import SlotRequest, SlotScheduler
    gold = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "emu2_tiny.pt"))
    eng = model.engine
    ids, img = gold["gen_input_ids"], gold["image"].cuda()
    sched = SlotScheduler(model, 16, prefill_chunk=chunk)
    seen, pick = {}, sched._select_one

    def spy(r):
        if r.num_beams == 1:
            seen.setdefault(r.tag, []).append(r.logits.clone())
        return pick(r)
    sched._select_one = spy
    EOS, PAD = 2, 32000
    specs = {0: [("g0", ids[0:1], img[0:1], 1), ("b0", ids[1:2], img[1:2], 5)], 2: [("g1", ids[1:2], img[1:2], 1)],
             3: [("g2", ids[0:1, -7:], None, 1)], 5: [("g3", ids[0:1], img[0:1], 1), ("b1", ids[0:1, -9:], None, 5)]}
    reqs, step = {}, 0
    while step <= max(specs) or sched.busy():
        for tag, prompt, im, nb in specs.get(step, []):
            reqs[tag] = (prompt, im, sched.submit(SlotRequest(prompt, image=im, num_beams=nb, max_new_tokens=10, min_len=0,
                                                              eos_token_id=EOS, pad_token_id=PAD, tag=tag)))
        sched.step()
        step += 1
    assert sched.prefill_chunks > 0 and any(B > 0 for B, _ in sched.mixed_sizes)
    for tag, (prompt, im, r) in reqs.items():
        assert r.error is None, (tag, r.error)
        if r.num_beams != 1:
            continue
        toks = r.result[0].to(torch.int32).cuda()
        eng.llm_reset()
        _, lg = eng.llm_prefill(model.embed_prompt(prompt.cuda(), im), None, hf_positions=True, want_logits=True)
        buf = torch.empty(1, VOCAB, dtype=torch.float32, device="cuda")
        replay = [lg.clone()]
        for t in range(len(toks) - 1):
            eng.llm_decode(token_ids=toks[t:t + 1].contiguous(), logits=buf, B=1)
            replay.append(buf.clone())
        assert len(seen[tag]) == len(toks)
        for t, (x, y) in enumerate(zip(seen[tag], replay)):
            err = float((x - y).abs().max() / y.abs().max())
            assert err < 2e-2, (tag, t, err)
    eng.llm_reset()
