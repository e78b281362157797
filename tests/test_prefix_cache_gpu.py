"""GPU: prefix caching in slot mode (include/emu_b200_prefix.h) — kept slots, prefix copies and per-slot continuation.

An extend from nothing must compute what a join computes; a join of a prefix plus an extend of the suffix must agree with the
fp32 oracle on the whole prompt as closely as a bf16 run does; a kept prefix must not feel the decode steps of other slots;
and the stand-alone kernels must match their torch restatements."""

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
    """the oracle's K ([H, T, D], rotate-half layout) in the engine's pair-interleaved head layout (element 2j = j,
    2j + 1 = j + D/2); V is stored as it is"""
    if kv == 1:
        return t
    half = t.shape[-1] // 2
    return torch.stack([t[..., :half], t[..., half:]], dim=-1).flatten(-2)


def _bf16(sd):
    return {k: v.to(torch.bfloat16) for k, v in sd.items()}


def test_extend_from_nothing_equals_join_bitwise(model):
    eng = model.engine
    x = torch.cat([_emb(37, 1), _emb(37, 2)]).cuda()
    buf = torch.empty(4, VOCAB, dtype=torch.float32, device="cuda")
    tok = torch.tensor([5, 6, 7, 8], dtype=torch.int32, device="cuda")
    eng.slots_begin(4)
    a = eng.join([1, 3], x)
    kv_join = eng.kv_cache()[:, :, [1, 3], :, :37].clone()
    eng.llm_decode(token_ids=tok, logits=buf, B=4)
    step_a = buf.clone()
    eng.slots_begin(4)
    b = eng.extend([1, 3], [0, 0], [37, 37], x)
    assert torch.equal(eng.kv_cache()[:, :, [1, 3], :, :37], kv_join)
    eng.llm_decode(token_ids=tok, logits=buf, B=4)
    assert torch.equal(a, b)
    assert torch.equal(step_a[[1, 3]], buf[[1, 3]])           # same cache rows: the next step is bitwise the same


@pytest.fixture(scope="module")
def refs(sd):
    return _bf16(sd)


@pytest.mark.parametrize("S", [1, 7, 64, 129])
@pytest.mark.parametrize("P", [1, 63, 64, 65, 127, 128, 129, 200])
def test_join_prefix_then_extend_suffix_matches_the_oracle(model, sd, refs, P, S):
    """suffixes of 1 / 7 / 64 tokens take the mma.sync attention, 129 the wgmma one.  The logits and the K / V the extend
    writes at [P, P + S) are within the bf16 bound of the fp32 oracle; every other cache position, of this slot and of every
    other row, is bitwise what it was"""
    eng = model.engine
    x = _emb(P + S, 100 * P + S)
    c32, c16 = O.KVCache(L), O.KVCache(L)
    ref32 = _oracle_last(sd, x.float(), cache=c32)
    ref16 = _oracle_last(refs, x, cache=c16)
    eng.slots_begin(4)
    eng.join([0], _emb(50, 9).cuda())                           # a live neighbour
    eng.join([2], x[:, :P].cuda())
    eng.leave_keep([2], [P])
    assert eng.slot_kept(2) == P
    before = eng.kv_cache().clone()
    got = eng.extend([2], [P], [S], x[:, P:].cuda())
    assert eng.slot_len(2) == P + S and eng.slot_kept(2) == 0
    assert_bf16_parity("extend P=%d S=%d" % (P, S), got.cpu(), ref32, ref16)
    after = eng.kv_cache()
    new = after[:, :, 2, :, P:P + S].float().cpu()
    for kv, name in ((0, "K"), (1, "V")):
        want32 = torch.stack([_interleave((c32.k if kv == 0 else c32.v)[l][0, :, P:P + S], kv) for l in range(L)])
        want16 = torch.stack([_interleave((c16.k if kv == 0 else c16.v)[l][0, :, P:P + S], kv) for l in range(L)]).float()
        assert_bf16_parity("extend %s[P, P+S) P=%d S=%d" % (name, P, S), new[:, kv], want32, want16)
    after[:, :, 2, :, P:P + S] = before[:, :, 2, :, P:P + S]
    assert torch.equal(after, before)                          # [0, P), past P + S and the other rows: untouched


def test_rows_with_different_prefixes_and_suffixes_in_one_extend(model, sd, refs):
    eng = model.engine
    cases = [(1, 129), (64, 7), (200, 1), (0, 33), (129, 64)]
    xs = [_emb(P + S, 7 + i) for i, (P, S) in enumerate(cases)]
    eng.slots_begin(8)
    slots = [0, 3, 4, 6, 7]
    for s, (P, _), x in zip(slots, cases, xs):
        if P:
            eng.join([s], x[:, :P].cuda())
            eng.leave_keep([s], [P])
    N = max(S for _, S in cases)
    emb = torch.zeros(len(cases), N, xs[0].shape[-1], dtype=torch.bfloat16)
    for i, ((P, S), x) in enumerate(zip(cases, xs)):
        emb[i, :S] = x[0, P:]
    got = eng.extend(slots, [P for P, _ in cases], [S for _, S in cases], emb.cuda()).cpu()
    for i, ((P, S), x) in enumerate(zip(cases, xs)):
        assert_bf16_parity("multi-row extend P=%d S=%d" % (P, S), got[i:i + 1], _oracle_last(sd, x.float()),
                           _oracle_last(refs, x))


@pytest.mark.parametrize("B", [6, 12], ids=["gemv", "wide"])
def test_a_kept_slot_is_untouched_by_twenty_decode_steps_of_others(model, B):
    eng = model.engine
    a, suffix = _emb(90, 3).cuda(), _emb(9, 4).cuda()
    others = [_emb(20 + s, 50 + s).cuda() for s in range(B)]
    buf = torch.empty(B, VOCAB, dtype=torch.float32, device="cuda")

    def resume(decode_steps):
        eng.slots_begin(B)
        eng.join([2], a)
        eng.leave_keep([2], [90])
        if decode_steps:
            for s in range(B):
                if s != 2:
                    eng.join([s], others[s])
            for t in range(decode_steps):
                eng.llm_decode(token_ids=torch.full((B,), 11 + t, dtype=torch.int32, device="cuda"), logits=buf, B=B)
            eng.leave([s for s in range(B) if s != 2])
        return eng.extend([2], [90], [9], suffix)
    assert torch.equal(resume(0), resume(20))


def test_copy_prefix_equals_resuming_in_place_and_leaves_the_source_alone(model):
    eng = model.engine
    a, suffix = _emb(70, 5).cuda(), _emb(12, 6).cuda()
    buf = torch.empty(8, VOCAB, dtype=torch.float32, device="cuda")
    tok = torch.full((8,), 9, dtype=torch.int32, device="cuda")
    eng.slots_begin(8)
    eng.join([0], a)
    eng.leave_keep([0], [64])
    in_place = eng.extend([0], [64], [12], suffix)
    eng.slots_begin(8)
    eng.join([0], a)
    eng.llm_decode(token_ids=tok, logits=buf, B=8)
    solo = buf[0].clone()
    eng.slots_begin(8)
    eng.join([0], a)
    eng.copy_prefix(0, 5, 64)                                   # from a live slot
    assert eng.slot_kept(5) == 64
    copied = eng.extend([5], [64], [12], suffix)
    assert torch.equal(copied, in_place)
    eng.llm_decode(token_ids=tok, logits=buf, B=8)
    assert torch.equal(buf[0], solo)                           # the live source decodes as if nothing happened
    eng.leave([0, 5])


def test_leave_keep_refuses_positions_a_slot_does_not_own(model):
    from emu_b200._lib import EmuError
    eng = model.engine
    x = _emb(30, 8).cuda()
    eng.slots_begin(6)
    eng.join([1], x)
    eng.fork(1, [2, 3])
    buf = torch.empty(6, VOCAB, dtype=torch.float32, device="cuda")
    eng.llm_decode(token_ids=torch.full((6,), 4, dtype=torch.int32, device="cuda"),
                   beam_src=torch.arange(6, dtype=torch.int32, device="cuda"), logits=buf, B=6)
    with pytest.raises(EmuError, match="slot 2 may keep"):
        eng.leave_keep([1, 2, 3], [30, 5, 0])                   # a forked slot owns nothing
    with pytest.raises(EmuError, match="slot 1 may keep"):
        eng.leave_keep([1, 2, 3], [31, 0, 0])                   # the group's first slot owns its prompt only
    eng.leave_keep([1, 2, 3], [30, 0, 0])
    assert [eng.slot_kept(s) for s in (1, 2, 3)] == [30, 0, 0]
    with pytest.raises(EmuError, match="keeps 30 positions"):
        eng.extend([1], [31], [1], x[:, :1])
    with pytest.raises(EmuError, match="occupied"):
        eng.join([4], x)
        eng.copy_prefix(1, 4, 10)


# ---- the stand-alone kernels ----
def test_prefix_copy_equals_a_slice_copy(cuda):
    from emu_b200 import _lib
    g = torch.Generator().manual_seed(1)
    cache = torch.randn(3, 5, 4, 64, 128, generator=g).to(torch.bfloat16).cuda()
    for src, dst, P in ((1, 3, 37), (4, 0, 64), (0, 2, 1)):
        want = cache.clone()
        want[:, dst, :, :P] = want[:, src, :, :P]
        _lib.op_kv_prefix_copy(cache, src, dst, P)
        assert torch.equal(cache, want)


# ---- one real LLaMA-33B layer ----
@pytest.mark.parametrize("P,S", [(75, 37), (133, 129)])
def test_llama33b_layer_extend(cuda, P, S):
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
        ref16 = _oracle_last(_bf16(sd), x, heads=heads, layers=1)
    eng = m.engine
    eng.slots_begin(2)
    eng.join([1], x[:, :P].cuda())
    eng.leave_keep([1], [P])
    got = eng.extend([1], [P], [S], x[:, P:].cuda()).cpu()
    assert_bf16_parity("llama33b layer extend %d+%d" % (P, S), got, ref32, ref16)
    eng.close()


# ---- the scheduler on the engine ----
def test_conversations_interleaved_with_other_requests_agree_with_a_replay(model):
    """3-turn conversations (the whole history resent each turn, a picture in turn 1) interleaved with greedy and 5-beam
    requests through SlotScheduler(prefix_cache=True): kept-slot parking under decode, resumes in place and through a copy,
    extend followed by a fork.  The logits every greedy turn selects from are within the bf16 bound of a plain prefill +
    decode of its own prompt and tokens."""
    import os
    from emu_b200.batching import SlotRequest, SlotScheduler
    gold = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "emu2_tiny.pt"))
    eng = model.engine
    ids, img = gold["gen_input_ids"], gold["image"].cuda()
    sched = SlotScheduler(model, 16, prefix_cache=True)
    seen, pick = {}, sched._select_one

    def spy(r):
        if r.num_beams == 1:
            seen.setdefault(r.tag, []).append(r.logits.clone())
        return pick(r)
    sched._select_one = spy
    EOS, PAD = 2, 32000
    convs = {"c0": (ids[0:1], img[0:1], ["pic0"], 1), "c1": (ids[1:2], img[1:2], ["pic1"], 1),
             "c5": (ids[0:1, -7:], None, None, 5)}
    done = []
    for turn in range(3):
        reqs = {}
        for name, (prompt, im, keys, nb) in convs.items():
            tag = "%s.%d" % (name, turn)
            beams = nb if turn != 1 else 1                        # the beam conversation's middle turn is greedy
            reqs[tag] = sched.submit(SlotRequest(prompt, image=im, image_keys=keys, num_beams=beams, max_new_tokens=6,
                                                 min_len=0, eos_token_id=EOS, pad_token_id=PAD, tag=tag))
        other = sched.submit(SlotRequest(ids[1:2, -5:], num_beams=5 if turn % 2 else 1, max_new_tokens=9, min_len=0,
                                         eos_token_id=EOS, pad_token_id=PAD, tag="o%d" % turn))
        for _ in range(2):                                        # a request arriving while the turn is decoding
            sched.step()
        late = sched.submit(SlotRequest(ids[0:1, -5:], num_beams=1, max_new_tokens=4, min_len=0, eos_token_id=EOS,
                                        pad_token_id=PAD, tag="l%d" % turn))
        sched.run_until_idle()
        for tag, r in list(reqs.items()) + [("o", other), ("l", late)]:
            assert r.error is None, (tag, r.error)
        for name, (prompt, im, keys, nb) in convs.items():
            r = reqs["%s.%d" % (name, turn)]
            done.append((r.tag, prompt, im, r))
            nxt = torch.cat([prompt, r.result.cpu()[:, :6].to(prompt.dtype), torch.tensor([[101 + turn, 102, 103]])], 1)
            convs[name] = (nxt, im, keys, nb)
    assert sched.prefix_hits >= 6 and sched.vit_pictures == 2
    for tag, prompt, im, r in done:
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
