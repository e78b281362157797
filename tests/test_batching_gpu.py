"""GPU: slot mode of the engine (include/emu_b200_slots.h) and the continuous-batching scheduler on it (tiny model).

A join must compute what a plain prefill computes, a slot's row must not feel what happens in the other slots, and one
request alone in the scheduler must get the ids EmuModel.generate_from_ids gives it."""
import os

import pytest
import torch

from helpers import TINY_LLAMA, TINY_VISION, StubTokenizer, make_emu2_state_dict

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "emu2_tiny.pt")
EOS, PAD, V = 2, 32000, 32272


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD)


@pytest.fixture(scope="module")
def model(cuda):
    from emu_b200.emu2.conf import CLIPVisionCfg, TextDecoderCfg
    from emu_b200.emu2.emu import EmuModel
    m = EmuModel(CLIPVisionCfg(**TINY_VISION), TextDecoderCfg(), tokenizer=StubTokenizer(), llama_config=TINY_LLAMA,
                 max_batch=16, max_seq=128)
    m.load_state_dict(make_emu2_state_dict())
    return m


def _prompts(model, gold):
    """embeddings [1, N, H] of four prompts of different lengths: the two golden rows with their pictures, two text tails"""
    ids, img = gold["gen_input_ids"].cuda(), gold["image"].cuda()
    out = [model.embed_prompt(ids[0:1], img[0:1]), model.embed_prompt(ids[1:2], img[1:2])]
    out += [model.embed_prompt(ids[0:1, -7:]), model.embed_prompt(ids[1:2, -5:])]
    return out


def _pad(embs):
    """left-pad [1, N_i, H] prompts into one batch + mask"""
    N = max(e.shape[1] for e in embs)
    x = torch.zeros(len(embs), N, embs[0].shape[-1], dtype=embs[0].dtype, device="cuda")
    m = torch.zeros(len(embs), N, dtype=torch.int32, device="cuda")
    for i, e in enumerate(embs):
        x[i, N - e.shape[1]:] = e[0]
        m[i, N - e.shape[1]:] = 1
    return x, m


def _tok(vals, n):
    t = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    for s, v in vals.items():
        t[s] = v
    return t


def test_join_equals_prefill_bitwise(model, gold):
    """join two prompts into scattered slots while two other slots hold live sequences at other lengths: the join's
    logits equal a plain prefill of the same prompts, the joined rows then decode exactly as they do without neighbours, and
    the live slots' next step is the one they take without the join"""
    eng, P = model.engine, _prompts(model, gold)
    x, m = _pad([P[2], P[1]])
    B = 10
    buf = torch.empty(B, V, dtype=torch.float32, device="cuda")
    _, plain = eng.llm_prefill(x, m, hf_positions=True, want_logits=True)
    plain = plain.clone()

    def live_schedule(with_join):
        eng.slots_begin(12)
        eng.join([1], P[0])
        eng.llm_decode(token_ids=_tok({1: 11}, B), logits=buf, B=B)
        eng.join([4], P[3])
        eng.llm_decode(token_ids=_tok({1: 12, 4: 13}, B), logits=buf, B=B)
        lg = eng.join([7, 2], x, m) if with_join else None
        eng.llm_decode(token_ids=_tok({1: 14, 4: 15, 7: 16, 2: 17}, B), logits=buf, B=B)
        return lg, buf.clone()
    joined, step_with = live_schedule(True)
    assert torch.equal(joined, plain)
    assert [eng.slot_len(s) for s in (1, 4, 7, 2, 0)] == [17, 7, 15, 15, 0]
    _, step_without = live_schedule(False)
    for s in (1, 4):                                              # the live slots' KV was left alone
        assert torch.equal(step_with[s], step_without[s]), s
    eng.slots_begin(12)                                           # the joined rows, alone
    assert torch.equal(eng.join([7, 2], x, m), plain)
    eng.llm_decode(token_ids=_tok({7: 16, 2: 17}, B), logits=buf, B=B)
    for s in (7, 2):
        assert torch.equal(step_with[s], buf[s]), s
    eng.llm_reset()


@pytest.mark.parametrize("B,slot", [(6, 1), (12, 9)])
def test_a_slot_does_not_feel_its_neighbours_bitwise(model, gold, B, slot):
    """a teacher-forced request's per-step logits, with other requests joining, forking (beam re-parenting included) and
    leaving around it, equal those of the same request alone in the same slot at the same B — on the GEMV path (B <= 8) and
    on the wide path (B > 8, whose RoPE / KV append reads every row's own position).  Likewise the beam group: re-parented
    while a LONGER sequence is live next to it, its rows must equal the group alone, which holds only if every row's table
    is rewritten up to its own length (past it, a beam's entries must keep pointing at its own row, where its new tokens go)"""
    eng, P = model.engine, _prompts(model, gold)
    buf = torch.empty(B, V, dtype=torch.float32, device="cuda")
    forced = [101, 2044, 530, 31000, 77, 9, 4242, 15]
    others = [s for s in range(B) if s != slot]
    a, b3 = others[0], others[-3:]

    def run(mode):          # "crowd": everything; "slot": the teacher-forced request alone; "group": the beam group alone
        eng.slots_begin(B)
        out_slot, out_group = [], []
        if mode != "group":
            out_slot.append(eng.join([slot], P[0]).clone())
        for t, tok in enumerate(forced):
            src = torch.arange(B, dtype=torch.int32, device="cuda")
            if mode == "crowd" and t == 1:
                eng.join([a], P[3])
            if mode != "slot":
                if t == 2:
                    out_group.append(eng.join([b3[0]], P[1]).clone())       # 14 tokens: shorter than `slot` by now
                    eng.fork(b3[0], b3[1:])
                if t in (3, 4):
                    src[b3[0]], src[b3[1]], src[b3[2]] = b3[2], b3[0], b3[0]
                if t == 6:
                    eng.leave(b3)
            if mode == "crowd" and t == 5:
                eng.leave([a])
            if mode == "group" and not 2 <= t < 6:
                continue
            toks = {slot: tok, a: 40 + t, b3[0]: 60 + t, b3[1]: 70 + t, b3[2]: 80 + t}
            eng.llm_decode(token_ids=_tok(toks, B), beam_src=src if mode != "slot" and t in (3, 4) else None, logits=buf, B=B)
            if mode != "group":
                out_slot.append(buf[slot].clone())
            if 2 <= t < 6:
                out_group.append(buf[b3].clone())
        return out_slot, out_group
    crowd_slot, crowd_group = run("crowd")
    alone_slot, _ = run("slot")
    _, alone_group = run("group")
    assert len(crowd_slot) == len(alone_slot) == len(forced) + 1
    for t, (x, y) in enumerate(zip(crowd_slot, alone_slot)):
        assert torch.equal(x.view(-1), y.view(-1)), ("slot", t)
    assert len(crowd_group) == len(alone_group) == 5
    for t, (x, y) in enumerate(zip(crowd_group, alone_group)):
        assert torch.equal(x, y), ("beam group", t)
    eng.llm_reset()


def test_a_long_join_into_a_scattered_slot_equals_prefill_bitwise(model, gold):
    """a join of 128 tokens runs the wgmma flash-attention kernel (shorter ones take the mma.sync kernel): its K/V tensor map
    spans every cache row and each query batch reads the row it was joined into.  Two prompts, one left-padded, join slots
    9 and 3 while slot 1 is live; logits equal a plain prefill, and slot 1's next step is untouched by the join"""
    eng, P = model.engine, _prompts(model, gold)
    long_ = torch.cat([P[0], P[1]] * 5, dim=1)[:, :128]
    x, m = _pad([long_, P[2]])
    assert x.shape[1] == 128
    _, plain = eng.llm_prefill(x, m, hf_positions=True, want_logits=True)
    plain = plain.clone()
    B = 10
    buf = torch.empty(B, V, dtype=torch.float32, device="cuda")

    def live_schedule(with_join):
        eng.slots_begin(12)
        eng.join([1], P[3])
        eng.llm_decode(token_ids=_tok({1: 11}, B), logits=buf, B=B)
        lg = None
        if with_join:
            lg = eng.join([9, 3], x, m)
            assert [eng.slot_len(s) for s in (9, 3)] == [128, 128]
            eng.leave([9, 3])                                     # full: no room to decode, but they were written
        eng.llm_decode(token_ids=_tok({1: 12}, B), logits=buf, B=B)
        return lg, buf[1].clone()
    joined, with_join = live_schedule(True)
    assert torch.equal(joined, plain)
    _, without = live_schedule(False)
    assert torch.equal(with_join, without)
    eng.llm_reset()


def test_one_request_gets_the_ids_of_generate_from_ids(model, gold):
    from emu_b200.batching import SlotRequest, SlotScheduler
    ids, img = gold["gen_input_ids"][:1], gold["image"][:1].cuda()
    for spec, n in ((dict(num_beams=1), 1), (dict(num_beams=5, length_penalty=-1), 5),
                    (dict(num_beams=1, do_sample=True, temperature=0.9, top_k=40, seed=7), 1)):
        kw = {k: v for k, v in spec.items() if k != "seed"}
        gen = lambda: torch.Generator(device="cuda").manual_seed(spec["seed"]) if "seed" in spec else None
        want = model.generate_from_ids(ids, torch.ones_like(ids), image=img, max_new_tokens=12, min_len=1, eos_token_id=EOS,
                                       pad_token_id=PAD, generator=gen(), **kw)
        sched = SlotScheduler(model, n)
        r = sched.submit(SlotRequest(ids, image=img, max_new_tokens=12, min_len=1, eos_token_id=EOS, pad_token_id=PAD,
                                     generator=gen(), **kw))
        sched.run_until_idle()
        assert r.error is None, r.error
        assert torch.equal(r.result.cpu(), want.cpu()), (spec, r.result.tolist(), want.tolist())
    model.engine.llm_reset()


def test_staggered_schedule_agrees_with_a_teacher_forced_replay(model, gold):
    """mixed knobs, staggered arrivals, left-padded joins: the logits every greedy / sampled request selects from are within
    the bf16 bound of a plain prefill + decode of its own tokens"""
    from emu_b200.batching import SlotRequest, SlotScheduler
    eng = model.engine
    ids = gold["gen_input_ids"]
    img = gold["image"].cuda()
    sched = SlotScheduler(model, 16)
    seen = {}
    pick = sched._select_one

    def spy(r):
        if r.num_beams == 1:
            seen.setdefault(r.tag, []).append(r.logits.clone())
        return pick(r)
    sched._select_one = spy
    specs = {0: [("g0", ids[0:1], img[0:1], dict(num_beams=1, max_new_tokens=10, min_len=0)),
                 ("b5", ids[1:2], img[1:2], dict(num_beams=5, max_new_tokens=8))],
             2: [("s1", ids[1:2, -5:], None, dict(num_beams=1, do_sample=True, top_k=20, max_new_tokens=9, min_len=0,
                                                  generator=torch.Generator(device="cuda").manual_seed(1)))],
             3: [("g2", ids[0:1, -7:], None, dict(num_beams=1, max_new_tokens=6, min_len=0)),
                 ("b3", ids[0:1], img[0:1], dict(num_beams=3, max_new_tokens=7, do_sample=True,
                                                 generator=torch.Generator(device="cuda").manual_seed(2)))]}
    reqs, step = {}, 0
    while step <= max(specs) or sched.busy():
        for tag, i, im, kw in specs.get(step, []):
            reqs[tag] = (i, im, sched.submit(SlotRequest(i, image=im, eos_token_id=EOS, pad_token_id=PAD, tag=tag, **kw)))
        sched.step()
        step += 1
    assert all(r.error is None for _, _, r in reqs.values())
    assert max(sched.batch_sizes) > 8
    for tag in ("g0", "s1", "g2"):
        i, im, r = reqs[tag]
        toks = r.result[0].to(torch.int32)
        eng.llm_reset()
        _, lg = eng.llm_prefill(model.embed_prompt(i.cuda(), im), None, hf_positions=True, want_logits=True)
        buf = torch.empty(1, V, dtype=torch.float32, device="cuda")
        replay = [lg.clone()]
        for t in range(len(toks) - 1):
            eng.llm_decode(token_ids=toks[t:t + 1].contiguous(), logits=buf, B=1)
            replay.append(buf.clone())
        assert len(seen[tag]) == len(toks)
        for t, (x, y) in enumerate(zip(seen[tag], replay)):
            err = float((x - y).abs().max() / y.abs().max())
            assert err < 2e-2, (tag, t, err)
    eng.llm_reset()


def test_free_slots_stay_frozen_and_a_full_cache_names_its_slot(model, gold):
    from emu_b200._lib import EmuError
    eng, P = model.engine, _prompts(model, gold)
    B = 4
    buf = torch.empty(B, V, dtype=torch.float32, device="cuda")
    eng.slots_begin(B)
    long = torch.cat([P[0]] * 9, dim=1)[:, :120]                 # 120 tokens of a 128-token cache
    eng.join([2], long)
    first = None
    for t in range(8):                                           # slot 0 is free: same token each step, same position 0
        eng.llm_decode(token_ids=_tok({0: 5, 2: 100 + t}, B), logits=buf, B=B)
        first = buf[0].clone() if first is None else first
        assert torch.equal(buf[0], first), t
        assert eng.slot_len(0) == 0
    assert eng.slot_len(2) == 128
    with pytest.raises(EmuError, match="KV cache full at slot 2"):
        eng.llm_decode(token_ids=_tok({2: 1}, B), logits=buf, B=B)
    eng.llm_reset()


def test_slot_mode_refuses_what_it_cannot_do(model, gold):
    from emu_b200._lib import EmuError
    eng, P = model.engine, _prompts(model, gold)
    with pytest.raises(EmuError, match="EMU_ERR_INVALID"):
        eng.slots_begin(17)                                      # more slots than llm_max_batch
    eng.slots_begin(4)
    eng.join([1], P[2])
    with pytest.raises(EmuError, match="EMU_ERR_STATE.*slot 1 is occupied"):
        eng.join([1], P[3])
    with pytest.raises(EmuError, match="EMU_ERR_INVALID.*out of range"):
        eng.join([4], P[3])
    with pytest.raises(EmuError, match="EMU_ERR_STATE"):
        eng.llm_prefill(P[2], None)
    with pytest.raises(EmuError, match="EMU_ERR_STATE"):
        eng.llm_expand(torch.zeros(2, dtype=torch.int32, device="cuda"), 2)
    eng.fork(1, [2, 3])
    with pytest.raises(EmuError, match="EMU_ERR_STATE.*leave with it"):
        eng.leave([2])
    with pytest.raises(EmuError, match="EMU_ERR_INVALID"):
        eng.llm_decode(token_ids=_tok({}, 4), B=3)               # B must cover the highest live slot
    eng.leave([1, 2, 3])
    assert [eng.slot_len(s) for s in range(4)] == [0, 0, 0, 0]
    eng.llm_reset()                                              # leaves slot mode: a plain prefill works again
    eng.llm_prefill(P[2], None)
    assert eng.slot_len(0) == -1
    eng.llm_reset()
