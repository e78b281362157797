"""CPU: prefix caching in the continuous-batching scheduler (SlotScheduler(prefix_cache=True)) over a slot oracle double that
keeps, copies and continues slot caches: every request's ids equal the run without the cache, while the counters show what
was not recomputed; the serving shell's --prefix-cache and its routing; and the C entry points of include/emu_b200_prefix.h
refusing bad arguments without a GPU."""
import ctypes
import io
import os
import re

import pytest
import torch

from helpers import make_emu2_state_dict
from oracle import emu_oracle as O
from test_batching_cpu import SlotOracleEngine, _chat, _model, _prompts
from test_generation_cpu import GOLD, L, NH

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class PrefixOracleEngine(SlotOracleEngine):
    """SlotOracleEngine + include/emu_b200_prefix.h: a leaving slot may keep a prefix of its oracle cache, a prefix can be
    copied into another slot, and a free slot can continue its kept prefix with right-padded new tokens."""

    def slots_begin(self, n_slots):
        super().slots_begin(n_slots)
        self.kept = [None] * n_slots                   # (oracle cache of the unpadded positions, pad, kept length)
        self.own = [0] * n_slots
        self.calls = []

    def _discard(self, slots):
        for s in slots:
            self.kept[s] = None

    def join(self, slots, embeds, attention_mask=None, want_logits=True):
        out = super().join(slots, embeds, attention_mask, want_logits)
        self._discard(slots)
        for s in slots:
            self.own[s] = self.lens[s]
        return out

    def fork(self, src, dst):
        super().fork(src, dst)
        self._discard(dst)
        for d in dst:
            self.own[d] = 0
        self.own[src] = -self.own[src]                 # frozen at its join length (negative: does not grow)

    def llm_decode(self, *a, **kw):
        live = [s for s in range(self.n_slots) if self.group[s] >= 0]
        super().llm_decode(*a, **kw)
        for s in live:
            if self.own[s] > 0:
                self.own[s] += 1

    def leave(self, slots):
        super().leave(slots)
        self._discard(slots)

    @staticmethod
    def _cut(cache, n):
        c = O.KVCache(L)
        c.k, c.v = [t[:, :, :n] for t in cache.k], [t[:, :, :n] for t in cache.v]
        return c

    def leave_keep(self, slots, keep):
        self.calls.append(("leave_keep", list(slots), list(keep)))
        held = []
        for s, k in zip(slots, keep):
            own = abs(self.own[s])
            assert 0 <= k <= min(own, self.cfg.llm_max_seq - 1), ("keep beyond the own row", s, k, own)
            pad = self.lens[s] - self.masks[s].shape[1]
            held.append((s, (self._cut(self.caches[s], k - pad), pad, k) if k else None))
        self.leave(slots)
        for s, kept in held:
            self.kept[s] = kept

    def slot_kept(self, s):
        return self.kept[s][2] if self.kept[s] is not None else 0

    def copy_prefix(self, src, dst, P):
        self.calls.append(("copy_prefix", src, dst, P))
        assert self.group[dst] < 0 and dst != src
        if self.group[src] >= 0:
            pad = self.lens[src] - self.masks[src].shape[1]
            assert P <= abs(self.own[src])
            self.kept[dst] = (self._cut(self.caches[src], P - pad), pad, P)
        else:
            cache, pad, k = self.kept[src]
            assert P <= k
            self.kept[dst] = (self._cut(cache, P - pad), pad, P)

    def extend(self, slots, prefix, new, embeds, want_logits=True):
        self.calls.append(("extend", list(slots), list(prefix), list(new)))
        self._slots(slots, True)
        out = []
        for i, s in enumerate(slots):
            assert 1 <= new[i] <= embeds.shape[1] and prefix[i] <= self.slot_kept(s)
            if prefix[i]:
                cache, pad, _ = self.kept[s]
                cache = self._cut(cache, prefix[i] - pad)
            else:
                cache, pad = O.KVCache(L), 0
            past = prefix[i] - pad
            h = O.llama_forward(self.sd, embeds[i:i + 1, :new[i]].float(), torch.ones(1, past + new[i], dtype=torch.long),
                                layers=L, heads=NH, position_ids=torch.arange(past, past + new[i]).unsqueeze(0), cache=cache)
            self.caches[s], self.masks[s] = cache, torch.ones(1, past + new[i], dtype=torch.long)
            self.group[s], self.lens[s], self.own[s], self.kept[s] = s, prefix[i] + new[i], prefix[i] + new[i], None
            out.append(O.lm_logits(self.sd, h[:, -1]).float())
        return torch.cat(out)


@pytest.fixture(scope="module")
def sd():
    return make_emu2_state_dict()


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD)


def _sched(sd, n_slots=8, max_seq=512, prefix_cache=True):
    from emu_b200.batching import SlotScheduler
    eng = PrefixOracleEngine(sd, max_batch=max(n_slots, 8), max_seq=max_seq)
    return eng, SlotScheduler(_model(eng), n_slots, prefix_cache=prefix_cache)


def _req(ids, image=None, keys=None, **spec):
    from emu_b200.batching import SlotRequest
    spec.setdefault("num_beams", 1)
    spec.setdefault("max_new_tokens", 6)
    return SlotRequest(ids, torch.ones_like(ids), image=image, image_keys=keys, **spec)


def _run(sched, r):
    sched.submit(r)
    sched.run_until_idle()
    assert r.error is None, r.error
    return r.result


def _uncached(sd, ids, image=None, keys=None, **spec):
    _, sched = _sched(sd, prefix_cache=False)
    return _run(sched, _req(ids, image, keys, **spec))


# ---- the demo's conversation: the whole history is resent on every turn ----
def _turns(pic):
    return [[[pic, "what is this?"]],
            [[pic, "what is this?"], None, ["and its colour?"]],
            [[pic, "what is this?"], None, ["and its colour?"], None, ["why?"]]]


def _conversation(sd, chat_engine_kwargs, prefix_cache, pic, knobs):
    from emu_b200.batching import SlotScheduler, chat_request
    eng = PrefixOracleEngine(sd, **chat_engine_kwargs)
    chat = _chat(eng)
    sched = SlotScheduler(chat.emu_model, 4, prefix_cache=prefix_cache)
    answers, counters = [], []
    for turn in _turns(pic):
        inputs = [m if m is not None else [answers[(i - 1) // 2]] for i, m in enumerate(turn)]
        r = chat_request(chat, inputs, prefix_keys=prefix_cache, **knobs)
        answers.append(_run(sched, r))
        counters.append((sched.vit_pictures, sched.prefill_tokens, sched.prefix_hits, sched.prefix_tokens_reused,
                         len(r.input_ids[0])))
    return answers, counters, eng


@pytest.mark.parametrize("knobs", [dict(num_beams=1, max_new_tokens=6), dict(num_beams=3, max_new_tokens=5)],
                         ids=["greedy", "beam3"])
def test_a_three_turn_conversation_reuses_its_history(sd, knobs):
    from PIL import Image
    pic = Image.new("RGB", (60, 40), (200, 30, 90))
    on, c_on, eng = _conversation(sd, dict(max_batch=8), True, pic, knobs)
    off, c_off, _ = _conversation(sd, dict(max_batch=8), False, pic, knobs)
    assert on == off
    assert c_on[0][0] == 1 and c_on[2][0] == 1                   # turns 2 and 3 ran no ViT ...
    assert c_off[2][0] == 3
    assert c_on[2][2] == 2                                       # ... resumed from the kept slot ...
    for t in (1, 2):                                             # ... and prefilled only their suffix
        prefilled = c_on[t][1] - c_on[t - 1][1]
        reused = c_on[t][3] - c_on[t - 1][3]
        assert prefilled + reused == c_on[t][4] and prefilled < c_on[t][4] - c_on[t - 1][4] + 8
    assert sum(1 for c in eng.calls if c[0] == "extend") == 2


def test_same_ids_with_a_different_picture_stop_before_it(sd, gold):
    ids, img = _prompts(gold)[0]
    first = int((ids[0] == 32003).nonzero()[0])
    eng, sched = _sched(sd)
    _run(sched, _req(ids, img, ["pic-a"]))
    other = img.flip(-1)
    got = _run(sched, _req(ids, other, ["pic-b"]))
    assert sched.prefix_hits == 1 and sched.prefix_tokens_reused == first
    assert sched.vit_pictures == 2
    assert torch.equal(got, _uncached(sd, ids, other, ["pic-b"]))
    # without picture keys nothing at or past the first picture ever matches
    _run(sched, _req(ids, img, None))
    assert sched.prefix_tokens_reused == 2 * first


def test_a_prefix_never_splits_a_picture_and_the_last_token_is_recomputed(sd, gold):
    ids, img = _prompts(gold)[0]
    pos = (ids[0] == 32003).nonzero()[:, 0]
    end = int(pos[-1]) + 1                                       # a prompt that ends with its picture
    eng, sched = _sched(sd)
    _run(sched, _req(ids, img, ["p"]))
    got = _run(sched, _req(ids, img, ["p"]))                     # the same prompt again: its last token is recomputed
    assert eng.calls[-2][:1] == ("extend",) and eng.calls[-2][3] == [1]
    assert torch.equal(got, _uncached(sd, ids, img, ["p"]))
    got = _run(sched, _req(ids[:, :end], img, ["p"]))
    assert sched.prefix_tokens_reused == ids.shape[1] - 1 + int(pos[0])   # cut back to the picture's first slot
    assert torch.equal(got, _uncached(sd, ids[:, :end], img, ["p"]))


def test_a_beam_request_keeps_its_prompt_and_the_next_turn_reuses_it(sd, gold):
    ids, _ = _prompts(gold)[2]
    eng, sched = _sched(sd, n_slots=6)
    _run(sched, _req(ids, num_beams=3, max_new_tokens=5))
    assert [eng.slot_kept(s) for s in range(6)] == [ids.shape[1], 0, 0, 0, 0, 0]
    more = torch.cat([ids, torch.tensor([[11, 12, 13]])], 1)
    got = _run(sched, _req(more, num_beams=3, max_new_tokens=5))
    assert sched.prefix_tokens_reused == ids.shape[1]
    assert torch.equal(got, _uncached(sd, more, num_beams=3, max_new_tokens=5))


def test_a_five_beam_request_that_cannot_start_at_its_prefix_copies_it(sd, gold):
    prompts = _prompts(gold)
    eng, sched = _sched(sd, n_slots=6)
    rs = [sched.submit(_req(p, i, ["k%d" % j], max_new_tokens=3)) for j, (p, i) in enumerate(prompts)]
    sched.run_until_idle()
    assert [r.slots for r in rs] == [[0], [1], [2], [3]]
    ids = torch.cat([prompts[3][0], torch.tensor([[21, 22]])], 1)    # continues the prompt kept in slot 3
    got = _run(sched, _req(ids, num_beams=5, max_new_tokens=4))
    copies = [c for c in eng.calls if c[0] == "copy_prefix"]
    assert len(copies) == 1 and copies[0][1] == 3 and copies[0][3] == rs[3].left_pad + prompts[3][0].shape[1]
    assert torch.equal(got, _uncached(sd, ids, num_beams=5, max_new_tokens=4))


def test_a_kept_row_from_a_left_padded_join_resumes(sd, gold):
    prompts = _prompts(gold)
    eng, sched = _sched(sd)
    long_ = sched.submit(_req(*prompts[0], keys=["x"], max_new_tokens=3))
    short = sched.submit(_req(prompts[3][0], max_new_tokens=4))
    sched.run_until_idle()
    pad = prompts[0][0].shape[1] - prompts[3][0].shape[1]
    assert short.left_pad == pad > 0
    ids = torch.cat([prompts[3][0], short.result[:, :3], torch.tensor([[31, 32]])], 1)
    got = _run(sched, _req(ids, max_new_tokens=5))
    assert sched.prefix_tokens_reused == prompts[3][0].shape[1] + 3
    assert torch.equal(got, _uncached(sd, ids, max_new_tokens=5))


def test_least_recently_used_kept_slot_is_overwritten_and_retention_never_delays(sd, gold):
    prompts = _prompts(gold)
    eng, sched = _sched(sd, n_slots=2)
    a = _req(prompts[2][0], max_new_tokens=2)
    _run(sched, a)
    b = _run(sched, _req(prompts[3][0], max_new_tokens=2)) is not None
    assert b and set(sched.kept) == {0, 1}                      # both slots keep a prefix, both count as free
    # a resume touches slot 0's prefix: slot 1 becomes the least recently used
    _run(sched, _req(torch.cat([prompts[2][0], torch.tensor([[7]])], 1), max_new_tokens=2))
    c = sched.submit(_req(torch.tensor([[40, 41, 42]]), max_new_tokens=2))
    sched.step()
    assert c.slots == [1] and 0 in sched.kept                   # admitted at once, over the LRU prefix
    sched.run_until_idle()
    assert c.error is None


def test_a_failing_extend_gives_its_slots_back(sd, gold):
    prompts = _prompts(gold)
    eng, sched = _sched(sd, n_slots=3)
    _run(sched, _req(prompts[2][0], max_new_tokens=2))

    def broken(*a, **kw):
        raise RuntimeError("extend failed")
    real, eng.extend = eng.extend, broken
    ids = torch.cat([prompts[2][0], torch.tensor([[9, 9]])], 1)
    bad = sched.submit(_req(ids, max_new_tokens=2))
    sched.run_until_idle()
    assert isinstance(bad.error, RuntimeError) and sched.owner == [None] * 3 and not sched.kept
    eng.extend = real
    assert torch.equal(_run(sched, _req(ids, max_new_tokens=2)), _uncached(sd, ids, max_new_tokens=2))


@pytest.mark.parametrize("prefix_cache", [False, True])
def test_a_requests_pad_token_id_reaches_its_selector(sd, gold, prefix_cache):
    """the scheduler's own bookkeeping (a slot's left padding) never takes the place of the request's pad token id"""
    import emu_b200.generation as G
    prompts = _prompts(gold)
    eng, sched = _sched(sd, prefix_cache=prefix_cache)
    seen, real = [], G.selector

    def spy(engine, batch, max_new_tokens, eos, pad, *a, **kw):
        seen.append(pad)
        return real(engine, batch, max_new_tokens, eos, pad, *a, **kw)
    G.selector = spy
    try:
        _run(sched, _req(prompts[0][0], prompts[0][1], max_new_tokens=2))          # joins with left padding 0 ...
        short = sched.submit(_req(prompts[3][0], max_new_tokens=2, pad_token_id=777))
        long_ = sched.submit(_req(prompts[1][0], prompts[1][1], max_new_tokens=2))   # ... and with left padding 9
        sched.run_until_idle()
    finally:
        G.selector = real
    assert sorted(seen) == [777, 32000, 32000] and (prefix_cache or short.left_pad > 0)


def test_chat_requests_carry_picture_keys_only_when_asked(sd):
    from PIL import Image
    from emu_b200.batching import chat_request
    chat = _chat(PrefixOracleEngine(sd))
    pic = Image.new("RGB", (60, 40), (1, 2, 3))
    plain = chat_request(chat, [pic, "hi"], num_beams=1)
    keyed = chat_request(chat, [pic, "hi"], prefix_keys=True, num_beams=1)
    assert plain.image_keys is None and plain.signature is None
    assert keyed.image_keys == [pic._emu_prefix_key] and keyed.signature == [pic._emu_prefix_key, "hi"]


# ---- the serving shell ----
def test_prefix_cache_needs_continuous_batching():
    from emu_b200 import serve
    from test_serve_cpu import FakeChat
    with pytest.raises(SystemExit):
        serve.main(["--prefix-cache", "--disable-generate", "--disable-chat"])
    with pytest.raises(ValueError, match="continuous"):
        serve.EmuServer(chat=FakeChat(), host="127.0.0.1", port=0, chat_prefix_cache=True)


def _serve_conversation(sd, prefix_cache, n_workers=1):
    from emu_b200 import serve
    from test_serve_cpu import png_bytes, post_chat
    srv = serve.EmuServer(chat=[_chat(PrefixOracleEngine(sd, max_batch=8)) for _ in range(n_workers)], host="127.0.0.1",
                          port=0, chat_scheduler="continuous", chat_prefix_cache=prefix_cache).start()
    url = "http://127.0.0.1:%d" % srv.port
    key = "[<IMAGE0>]"
    answers = []
    prompt = [["IMAGE", key], ["TEXT", "what is this?"]]
    for q in ("and its colour?", "why?"):
        files = {key: (key, io.BytesIO(png_bytes((60, 40))), "image/png")}
        a = post_chat(url, prompt, files=files, num_beams=1, max_new_tokens=6).json()
        answers.append(a)
        prompt = prompt + [["TEXT", a["data"]], ["TEXT", q]]
    return answers, srv


def test_the_demo_form_gives_the_same_answers_with_the_cache(sd):
    on, srv = _serve_conversation(sd, True)
    hits = srv.chat_workers[0].scheduler.prefix_hits
    srv.shutdown()
    off, srv = _serve_conversation(sd, False)
    srv.shutdown()
    assert on == off and all(a["code"] == 0 for a in on) and hits == 1


def test_a_request_goes_to_the_worker_holding_its_prefix(sd):
    from PIL import Image
    from emu_b200.batching import prompt_signature
    answers, srv = _serve_conversation(sd, True, n_workers=2)
    w0, w1 = srv.chat_workers
    holder = w0 if w0.scheduler.kept else w1
    other = w1 if holder is w0 else w0
    pic = Image.open(io.BytesIO(__import__("test_serve_cpu").png_bytes((60, 40)))).convert("RGB")
    inputs = [pic, "what is this?", answers[0]["data"], "and its colour?", answers[1]["data"], "more"]
    assert holder.scheduler.cached_prefix(prompt_signature(inputs)) >= 4
    from emu_b200.batching import SlotRequest
    holder.scheduler.submit(SlotRequest(torch.tensor([[5, 6, 7]]), num_beams=1))   # the holder is busier ...
    assert holder.load() > other.load()
    assert srv._pick(srv.chat_workers, "chat", inputs) is holder                     # ... and still gets it
    assert srv._pick(srv.chat_workers, "chat", ["unrelated"]) is other
    holder.scheduler.waiting.clear()                         # the stand-in load must not run while the server stops
    srv.shutdown()


# ---- the C entry points ----
HEADER = os.path.join(ROOT, "include", "emu_b200_prefix.h")


@pytest.fixture(scope="module")
def lib():
    from emu_b200 import build, _lib
    build.build()
    return _lib.load()


def test_prefix_header_symbols_are_bound_exported_and_disjoint(lib):
    from emu_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(emu_[a-z0-9_]+)\s*\(", src)))
    assert sorted(_lib.PREFIX_SYMBOLS) == syms
    assert all(hasattr(lib, s) for s in syms)
    others = set(_lib.SYMBOLS + _lib.SAFETY_SYMBOLS + _lib.SLOT_SYMBOLS + _lib.OPS_SYMBOLS + _lib.GEN_SLOT_SYMBOLS +
                 _lib.DIFFUSION_OPS_SYMBOLS)
    assert not others & set(syms)


def test_prefix_entry_points_refuse_null_arguments_without_a_gpu(lib):
    N = None
    one = (ctypes.c_int32 * 1)(0)
    V = ctypes.c_void_p(16)
    for name, args in {"emu_llm_leave_keep": [(N, one, one, 1, N)],
                       "emu_llm_copy_prefix": [(N, 0, 1, 4, N)],
                       "emu_llm_extend": [(N, one, one, one, 1, V, 4, N, N)],
                       "emu_op_kv_prefix_copy": [(N, 2, 4, 2, 64, 16, 0, 1, 4, N), (V, 2, 4, 2, 64, 16, 1, 1, 4, N),
                                                 (V, 2, 4, 2, 64, 16, 0, 1, 17, N),
                                                 (ctypes.c_void_p(24), 2, 4, 2, 64, 16, 0, 1, 4, N)],
                       "emu_llm_kv_cache": [(N, ctypes.byref(ctypes.c_void_p()), (ctypes.c_int64 * 5)())]}.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = ctypes.c_int, None
        for a in args:
            assert fn(*a) == -1, (name, a)
    assert lib.emu_llm_slot_kept(N, 0) == -1
