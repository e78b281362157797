"""CPU: continuous batching (emu_b200/batching.py) over a slot-capable oracle double of the engine — every request's ids equal
`generate` on that request alone, whatever joins, forks and leaves around it; the serving shell's ContinuousWorker behind the
demo's form; and the C entry points of slot mode refusing bad arguments without a GPU."""
import ctypes
import os
import re
import threading

import pytest
import torch
import torch.nn.functional as F

from helpers import StubTokenizer, make_emu2_state_dict
from oracle import emu_oracle as O
from test_generation_cpu import CTRL, GOLD, L, NH, OracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class SlotOracleEngine(OracleEngine):
    """OracleEngine + slot mode (include/emu_b200_slots.h): one oracle KV cache per slot.  A decode step runs every beam
    group as one batch and every other live slot on its own — the batches a request would have alone."""

    def __init__(self, sd, max_batch=8, max_seq=512):
        super().__init__(sd, max_batch)
        self.cfg.llm_max_seq = max_seq
        self.n_slots = 0
        self.decode_B = []

    def slots_begin(self, n_slots):
        if not 1 <= n_slots <= self.cfg.llm_max_batch:
            raise ValueError("n_slots out of range")
        self.n_slots = n_slots
        self.caches, self.masks = [None] * n_slots, [None] * n_slots
        self.group, self.lens = [-1] * n_slots, [0] * n_slots
        self.hf = True

    def _slots(self, slots, free):
        for s in slots:
            assert 0 <= s < self.n_slots and (self.group[s] < 0) == free, (s, self.group)
        assert len(set(slots)) == len(slots)

    @staticmethod
    def _copy(cache):
        c = O.KVCache(L)
        c.k, c.v = list(cache.k), list(cache.v)
        return c

    def join(self, slots, embeds, attention_mask=None, want_logits=True):
        self._slots(slots, True)
        out = []
        N = embeds.shape[1]
        for i, s in enumerate(slots):
            m = attention_mask[i] if attention_mask is not None else torch.ones(N, dtype=torch.int32)
            p = int((m == 0).sum())                    # left padding: masked, it changes nothing of the sequence
            mm = torch.ones(1, N - p, dtype=torch.long)
            cache = O.KVCache(L)
            h = O.llama_forward(self.sd, embeds[i:i + 1, p:].float(), mm, layers=L, heads=NH,
                                position_ids=O.hf_position_ids(mm), cache=cache)
            self.caches[s], self.masks[s], self.group[s], self.lens[s] = cache, mm, s, N
            out.append(O.lm_logits(self.sd, h[:, -1]).float())
        return torch.cat(out)

    def fork(self, src, dst):
        assert self.group[src] >= 0
        self._slots(dst, True)
        for d in dst:
            self.caches[d], self.masks[d] = self._copy(self.caches[src]), self.masks[src].clone()
            self.group[d], self.lens[d] = self.group[src], self.lens[src]

    def leave(self, slots):
        self._slots(slots, False)
        groups = {self.group[s] for s in slots}
        assert all(s in slots for s in range(self.n_slots) if self.group[s] in groups), "a beam group leaves together"
        for s in slots:
            self.caches[s] = self.masks[s] = None
            self.group[s], self.lens[s] = -1, 0

    def slot_len(self, s):
        return self.lens[s]

    def llm_decode(self, token_ids=None, embeds=None, beam_src=None, logits=None, hidden=None, next_ids=None, ban_id=-1, B=None):
        if not self.n_slots:
            return super().llm_decode(token_ids, embeds, beam_src, logits, hidden, next_ids, ban_id, B)
        live = [s for s in range(self.n_slots) if self.group[s] >= 0]
        assert live and max(live) < B <= self.n_slots
        self.decode_B.append(B)
        if beam_src is not None:
            old = [(self.caches[s], self.masks[s]) for s in range(self.n_slots)]
            for s in live:
                src = int(beam_src[s])
                assert self.group[src] == self.group[s], "beam_src maps a slot out of its group"
                self.caches[s], self.masks[s] = self._copy(old[src][0]), old[src][1].clone()
        for g in sorted({self.group[s] for s in live}):
            rows = [s for s in live if self.group[s] == g]
            assert all(self.lens[s] + 1 <= self.cfg.llm_max_seq for s in rows), "KV cache full"
            cache = O.KVCache(L)
            cache.k = [torch.cat([self.caches[s].k[l] for s in rows]) for l in range(L)]
            cache.v = [torch.cat([self.caches[s].v[l] for s in rows]) for l in range(L)]
            mask = torch.cat([self.masks[s] for s in rows])
            mask = torch.cat((mask, torch.ones(len(rows), 1, dtype=mask.dtype)), dim=1)
            e = F.embedding(token_ids[rows].long(), self.sd["decoder.lm.model.embed_tokens.weight"]).unsqueeze(1)
            h = O.llama_forward(self.sd, e, mask, layers=L, heads=NH, position_ids=mask.long().sum(-1, keepdim=True) - 1,
                                cache=cache)
            lg = O.lm_logits(self.sd, h[:, -1]).float()
            for i, s in enumerate(rows):
                c = O.KVCache(L)
                c.k, c.v = [t[i:i + 1] for t in cache.k], [t[i:i + 1] for t in cache.v]
                self.caches[s], self.masks[s] = c, mask[i:i + 1]
                self.lens[s] += 1
                logits[s] = lg[i]


def _model(engine):
    """EmuModel's host code over a CPU engine double (as tests/test_generation_cpu.py::_emu2_model)"""
    from types import SimpleNamespace as NS
    from emu_b200.emu2.emu import EmuModel
    sd = engine.sd
    m = EmuModel.__new__(EmuModel)
    engine.llm_embed = lambda ids: F.embedding(ids.long(), sd["decoder.lm.model.embed_tokens.weight"])
    m.engine, m.device_ = engine, torch.device("cpu")
    m.decoder, m.n_query, m.v_query = NS(tokenizer=StubTokenizer()), 4, 4
    m.image_placeholder = "[IMG]" + "<image>" * 4 + "[/IMG]"
    m.video_placeholder = "[IMG]" + "[gIMG]" * 4 + "[/IMG]"

    def encode(image, n_query=None):
        if image.shape[-1] != 56:
            raise ValueError("picture of the wrong size")
        return O.encode_image(sd, image.float(), patch=14, num_heads=4, layers=2, n_query=n_query or 4)
    m.encode_image = encode
    m._project_up = lambda x: F.linear(x, sd["project_up.weight"])
    return m


@pytest.fixture(scope="module")
def sd():
    return make_emu2_state_dict()


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD)


def _prompts(gold):
    """four prompts of different lengths: the two golden rows with their pictures, two text-only tails"""
    ids, img = gold["gen_input_ids"], gold["image"]
    out = [(ids[0:1], img[0:1]), (ids[1:2], img[1:2])]
    for row, n in ((0, 7), (1, 5)):
        tail = ids[row:row + 1, -n:]
        assert not (tail == 32003).any()
        out.append((tail, None))
    return out


def _solo(sd, ids, image, spec):
    """the request alone, through EmuModel.generate_from_ids -> generation.generate"""
    kw = {k: v for k, v in spec.items() if k != "seed"}
    if "seed" in spec:
        kw["generator"] = torch.Generator().manual_seed(spec["seed"])
    return _model(OracleEngine(sd, max_batch=8)).generate_from_ids(ids, torch.ones_like(ids), image=image, **kw)


def _request(ids, image, spec):
    from emu_b200.batching import SlotRequest
    kw = {k: v for k, v in spec.items() if k != "seed"}
    if "seed" in spec:
        kw["generator"] = torch.Generator().manual_seed(spec["seed"])
    return SlotRequest(ids, torch.ones_like(ids), image=image, **kw)


SPECS = [
    ("greedy", 0, dict(num_beams=1, max_new_tokens=12, min_len=1)),
    ("beam5", 0, dict(num_beams=5, max_new_tokens=12, min_len=1, length_penalty=-1)),            # gen_ids_beam5
    ("greedy_rep_ngram", 2, dict(num_beams=1, max_new_tokens=9, repetition_penalty=1.3, no_repeat_ngram_size=3)),
    ("beamsample2_topk", 0, dict(num_beams=2, max_new_tokens=12, min_len=1, do_sample=True, top_k=8, length_penalty=-1,
                                 seed=5)),
    ("sample", 3, dict(num_beams=1, max_new_tokens=10, do_sample=True, temperature=0.9, top_k=40, seed=11)),
    ("beam3_rep", 1, dict(num_beams=3, max_new_tokens=8, min_len=1, length_penalty=1.0, repetition_penalty=1.4,
                          no_repeat_ngram_size=2)),
    ("beamsample5_demo", 0, dict(num_beams=5, max_new_tokens=12, min_len=1, do_sample=True, top_k=3, top_p=0.9,
                                 temperature=0.7, length_penalty=1.0, seed=9)),
    ("greedy_short", 2, dict(num_beams=1, max_new_tokens=3)),
    ("sample_rep_ngram", 1, dict(num_beams=1, max_new_tokens=10, do_sample=True, temperature=0.8, top_k=20,
                                 repetition_penalty=1.3, no_repeat_ngram_size=2, seed=13)),
    ("greedy_min_len", 3, dict(num_beams=1, max_new_tokens=9, min_len=6)),
]


def test_scheduler_matches_each_request_alone(sd, gold):
    """staggered arrivals, mixed knobs sharing decode steps: each request's ids == generate on it alone; the batch-1 goldens of
    the reference's own lm.generate are reproduced too"""
    from emu_b200.batching import SlotScheduler
    ctrl = torch.load(CTRL)
    prompts = _prompts(gold)
    eng = SlotOracleEngine(sd, max_batch=16)
    sched = SlotScheduler(_model(eng), 16)
    reqs = {}
    arrivals = {0: SPECS[:2], 2: SPECS[2:4], 3: SPECS[4:5], 6: SPECS[5:7], 9: SPECS[7:]}
    step = 0
    while step <= max(arrivals) or sched.busy():
        for name, p, spec in arrivals.get(step, []):
            reqs[name] = (p, spec, sched.submit(_request(*prompts[p], spec)))
        sched.step()
        step += 1
    assert max(eng.decode_B) > 8                       # several requests (and beam groups) shared steps
    for name, (p, spec, r) in reqs.items():
        assert r.done.is_set() and r.error is None, (name, r.error)
        want = _solo(sd, *prompts[p], spec)
        assert torch.equal(r.result, want), (name, r.result.tolist(), want.tolist())
    assert torch.equal(reqs["beam5"][2].result, gold["gen_ids_beam5"])
    assert torch.equal(reqs["beamsample2_topk"][2].result, ctrl["beamsample2_topk"])
    assert torch.equal(reqs["beamsample5_demo"][2].result, ctrl["beamsample5_demo"])


def test_slots_are_reused_and_beam_groups_stay_contiguous(sd, gold):
    from emu_b200.batching import SlotScheduler
    prompts = _prompts(gold)
    eng = SlotOracleEngine(sd, max_batch=8)
    sched = SlotScheduler(_model(eng), 6)
    a = sched.submit(_request(*prompts[2], dict(num_beams=1, max_new_tokens=2)))
    b = sched.submit(_request(*prompts[0], dict(num_beams=3, max_new_tokens=12, min_len=12)))
    c = sched.submit(_request(*prompts[3], dict(num_beams=1, max_new_tokens=12, min_len=12)))
    sched.step()
    assert (a.slots, b.slots, c.slots) == ([0], [1, 2, 3], [4])
    assert eng.group[1:4] == [1, 1, 1] and eng.lens[1:4] == [eng.lens[1]] * 3
    while not a.done.is_set():
        sched.step()
    assert eng.group[0] == -1 and eng.lens[0] == 0      # a left: its slot is free again
    # two slots wanted: 0 and 5 are free but not adjacent, so the group waits (first come, first served) ...
    d = sched.submit(_request(*prompts[2], dict(num_beams=2, max_new_tokens=3)))
    e = sched.submit(_request(*prompts[3], dict(num_beams=1, max_new_tokens=2)))
    sched.step()
    assert not d.slots and not e.slots
    sched.run_until_idle()
    assert d.slots == [0, 1] and e.slots == [2]                 # freed slots are taken again, lowest first
    for r in (a, b, c, d, e):
        assert r.error is None
    assert eng.group == [-1] * 6
    for r, p, spec in ((d, 2, dict(num_beams=2, max_new_tokens=3)), (c, 3, dict(num_beams=1, max_new_tokens=12, min_len=12))):
        assert torch.equal(r.result, _solo(sd, *prompts[p], spec))


def test_a_failing_request_does_not_disturb_the_others(sd, gold):
    from emu_b200.batching import SlotScheduler
    prompts = _prompts(gold)
    sched = SlotScheduler(_model(SlotOracleEngine(sd)), 8)
    good = [sched.submit(_request(*prompts[0], dict(num_beams=3, max_new_tokens=6, min_len=1)))]
    sched.step()
    bad = sched.submit(_request(prompts[1][0], torch.zeros(1, 3, 8, 8), dict(num_beams=1, max_new_tokens=4)))
    good.append(sched.submit(_request(*prompts[3], dict(num_beams=1, max_new_tokens=5))))
    sched.run_until_idle()
    assert isinstance(bad.error, ValueError) and bad.result is None
    assert torch.equal(good[0].result, _solo(sd, *prompts[0], dict(num_beams=3, max_new_tokens=6, min_len=1)))
    assert torch.equal(good[1].result, _solo(sd, *prompts[3], dict(num_beams=1, max_new_tokens=5)))
    assert sched.engine.group == [-1] * 8


def test_a_request_failing_after_its_join_gives_its_slots_back(sd, gold):
    """the join succeeded but the fork after it failed: the slot the engine holds must leave, so the next request can take it"""
    from emu_b200.batching import SlotScheduler
    prompts = _prompts(gold)
    eng = SlotOracleEngine(sd)
    sched = SlotScheduler(_model(eng), 4)
    real_fork, calls = eng.fork, []

    def flaky_fork(src, dst):
        calls.append(src)
        if len(calls) == 1:
            raise RuntimeError("fork failed")
        return real_fork(src, dst)
    eng.fork = flaky_fork
    bad = sched.submit(_request(*prompts[2], dict(num_beams=3, max_new_tokens=4)))
    ok = sched.submit(_request(*prompts[3], dict(num_beams=1, max_new_tokens=4)))
    sched.step()
    assert isinstance(bad.error, RuntimeError) and bad.slots == [0, 1, 2] and ok.slots == [3]
    assert eng.group[:3] == [-1, -1, -1]                          # the joined first slot left the engine again
    again = sched.submit(_request(*prompts[2], dict(num_beams=3, max_new_tokens=4)))
    sched.run_until_idle()
    assert again.error is None and again.slots == [0, 1, 2] and ok.error is None
    assert torch.equal(again.result, _solo(sd, *prompts[2], dict(num_beams=3, max_new_tokens=4)))
    assert eng.group == [-1] * 4


def test_left_padding_never_takes_room_from_a_short_prompt(sd, gold):
    """close to llm_max_seq a short prompt is not joined together with a long one if the padding would cut its answer"""
    from emu_b200.batching import SlotScheduler
    prompts = _prompts(gold)
    eng = SlotOracleEngine(sd, max_seq=20)
    sched = SlotScheduler(_model(eng), 4)
    joins = []
    real_join = eng.join
    eng.join = lambda slots, embeds, mask=None, want_logits=True: (joins.append(embeds.shape[1]),
                                                                   real_join(slots, embeds, mask, want_logits))[1]
    long_ = sched.submit(_request(*prompts[0], dict(num_beams=1, max_new_tokens=5, min_len=5)))     # 14 tokens
    short = sched.submit(_request(*prompts[3], dict(num_beams=1, max_new_tokens=12, min_len=12)))   # 5 tokens
    sched.run_until_idle()
    assert joins == [14, 5]
    assert long_.result.shape == (1, 5) and short.result.shape == (1, 12)
    assert torch.equal(short.result, _solo(sd, *prompts[3], dict(num_beams=1, max_new_tokens=12, min_len=12)))


def test_requests_go_to_the_least_loaded_continuous_worker(sd, gold):
    from emu_b200 import serve
    from emu_b200.batching import SlotRequest
    srv = serve.EmuServer(chat=[_chat(SlotOracleEngine(sd)), _chat(SlotOracleEngine(sd))], host="127.0.0.1", port=0,
                          chat_scheduler="continuous").start()
    w0, w1 = srv.chat_workers
    # the worker thread blocks on its queue while idle, so this request stays waiting in w0's scheduler
    w0.scheduler.submit(SlotRequest(torch.tensor([[5, 6, 7]]), num_beams=1))
    assert (w0.load(), w1.load()) == (1, 0)
    assert srv._pick(srv.chat_workers, "chat") is w1
    srv.shutdown()


def test_a_worker_whose_engine_cannot_enter_slot_mode_fails_at_start(sd):
    from emu_b200 import serve
    eng = SlotOracleEngine(sd)

    def refuse(n):
        raise RuntimeError("EMU_ERR_UNSUPPORTED: slot mode with EMU_KV_COPY=1")
    eng.slots_begin = refuse
    srv = serve.EmuServer(chat=_chat(eng), host="127.0.0.1", port=0, chat_scheduler="continuous")
    with pytest.raises(RuntimeError, match="EMU_KV_COPY"):
        srv.start()
    srv.httpd.server_close()


def test_requests_the_form_cannot_send_are_refused():
    from emu_b200.batching import SlotRequest
    ids = torch.tensor([[5, 6, 7]])
    with pytest.raises(ValueError, match="contrastive"):
        SlotRequest(ids, num_beams=1, penalty_alpha=0.6, top_k=4)
    with pytest.raises(ValueError, match="prefix_allowed_tokens_fn"):
        SlotRequest(ids, prefix_allowed_tokens_fn=lambda b, i: [1])
    with pytest.raises(ValueError, match="num_return_sequences"):
        SlotRequest(ids, num_beams=3, num_return_sequences=2)


def test_max_new_tokens_is_capped_so_a_slot_cannot_overflow(sd, gold):
    from emu_b200.batching import SlotScheduler
    prompts = _prompts(gold)
    eng = SlotOracleEngine(sd, max_seq=20)                          # 14-token prompt: room for 7 new tokens
    sched = SlotScheduler(_model(eng), 4)
    r = sched.submit(_request(*prompts[0], dict(num_beams=1, max_new_tokens=50, min_len=50)))
    sched.run_until_idle()
    assert r.error is None and r.result.shape == (1, 7) and max(eng.lens) == 0


# ---- the serving shell: ContinuousWorker behind EmuServer, the demo's form as tests/test_serve_cpu.py posts it ----
def _fake_tokenize(texts):
    ids = []
    for piece in re.split(r"(\[IMG\]|\[/IMG\]|<image>)", texts[0]):
        ids += {"[IMG]": [32001], "[/IMG]": [32002], "<image>": [32003]}.get(piece, [100 + ord(ch) % 500 for ch in piece])
    t = torch.tensor([ids])
    return t, torch.ones_like(t)


def _chat(engine):
    from emu_b200.emu2.chat import EmuChatGeneration
    m = _model(engine)
    m._tokenize = _fake_tokenize
    return EmuChatGeneration(m, eva_size=56)


def test_continuous_worker_answers_the_demo_form(sd):
    from emu_b200 import serve
    from test_serve_cpu import png_bytes, post_chat
    import io
    srv = serve.EmuServer(chat=_chat(SlotOracleEngine(sd, max_batch=12)), host="127.0.0.1", port=0,
                          chat_scheduler="continuous").start()
    url = "http://127.0.0.1:%d" % srv.port
    key = "[<IMAGE0>]"
    posts = [
        dict(prompt=[["IMAGE", key], ["TEXT", "what is this?"]], files=True,
             data=dict(do_sample=False, max_new_tokens=8, temperature=0.7, top_k=3, top_p=0.9, length_penalty=1, num_beams=5,
                       repetition_penalty=1.0)),
        dict(prompt=[["TEXT", "hello there"]], files=False, data=dict(num_beams=1, max_new_tokens=6)),
        dict(prompt=[["TEXT", "and you"]], files=False, data=dict(num_beams=3, max_new_tokens=5, repetition_penalty=1.3)),
        dict(prompt=[["IMAGE", "missing"]], files=False, data={}),
    ]
    answers = {}

    def client(i):
        p = posts[i]
        files = {key: (key, io.BytesIO(png_bytes((60, 40))), "image/png")} if p["files"] else None
        answers[i] = post_chat(url, p["prompt"], files=files, **p["data"]).json()
    ts = [threading.Thread(target=client, args=(i,)) for i in range(len(posts))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    srv.shutdown()
    assert answers[3]["code"] == -1
    # each answer == EmuChatGeneration.forward of that request alone on the plain engine double
    from PIL import Image
    alone = _chat(OracleEngine(sd, max_batch=8))
    pic = Image.open(io.BytesIO(png_bytes((60, 40)))).convert("RGB")
    inputs = [[pic, "what is this?"], ["hello there"], ["and you"]]
    for i in range(3):
        knobs = serve.chat_knobs({k: str(v) for k, v in posts[i]["data"].items()})
        assert answers[i] == {"code": 0, "data": alone(inputs[i], **knobs)}, (i, answers[i])


def test_continuous_batching_is_opt_in():
    from emu_b200 import serve
    from test_serve_cpu import FakeChat
    srv = serve.EmuServer(chat=FakeChat(), host="127.0.0.1", port=0)
    assert isinstance(srv.chat_workers[0], serve.BatchingWorker)
    srv.httpd.server_close()
    with pytest.raises(ValueError):
        serve.EmuServer(chat=FakeChat(), host="127.0.0.1", port=0, chat_scheduler="continuous", announce=lambda *a: None)
    with pytest.raises(SystemExit):
        os.environ["WORLD_SIZE"] = "2"
        try:
            serve.main(["--continuous-batching", "--disable-generate"])
        finally:
            del os.environ["WORLD_SIZE"]


# ---- the C entry points of slot mode ----
HEADER = os.path.join(ROOT, "include", "emu_b200_slots.h")


@pytest.fixture(scope="module")
def lib():
    from emu_b200 import build, _lib
    build.build()
    return _lib.load()


def test_slot_header_symbols_are_bound_and_exported(lib):
    from emu_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(emu_[a-z0-9_]+)\s*\(", src)))
    assert sorted(_lib.SLOT_SYMBOLS) == syms
    assert all(hasattr(lib, s) for s in syms)


def test_slot_entry_points_refuse_bad_arguments_without_a_gpu(lib):
    """a NULL engine, NULL slot lists and empty lists are EMU_ERR_INVALID before anything is touched.  The checks that need
    engine state — a slot out of range, a join into an occupied slot, prefill / expand in slot mode, n_slots > llm_max_batch,
    a beam group leaving in part — are made on the host before any CUDA call too, but an engine cannot be created without a
    GPU: tests/test_batching_gpu.py::test_slot_mode_refuses_what_it_cannot_do covers them."""
    N = None
    one = (ctypes.c_int32 * 1)(0)
    for name, args in {"emu_llm_slots_begin": (N, 4, N),
                       "emu_llm_join": (N, one, 1, N, N, 4, N, N),
                       "emu_llm_fork": (N, 0, one, 1, N),
                       "emu_llm_leave": (N, one, 1, N)}.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = ctypes.c_int, None
        assert fn(*args) == -1, name
    assert lib.emu_llm_slot_len(N, 0) == -1
