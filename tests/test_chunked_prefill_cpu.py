"""CPU: chunked prefill in the continuous-batching scheduler (SlotScheduler(prefill_chunk=C)) over an oracle double of
emu_llm_step: every request's ids equal the unchunked scheduler's at any chunk size, live requests never stall while a prompt
is prefilled, left-padded prompts still join whole; the serving shell's --prefill-chunk; and the C entry points of
include/emu_b200_chunked.h refusing bad arguments without a GPU."""
import ctypes
import os
import re

import pytest
import torch

from helpers import make_emu2_state_dict
from test_batching_cpu import SPECS, _model, _prompts, _request
from test_generation_cpu import GOLD
from test_prefix_cache_cpu import PrefixOracleEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class ChunkOracleEngine(PrefixOracleEngine):
    """PrefixOracleEngine + include/emu_b200_chunked.h: emu_llm_step is the decode step of the live slots below B, then one
    emu_llm_extend per packed segment; a segment that is not final leaves its slot kept at its new length."""

    def slots_begin(self, n_slots):
        super().slots_begin(n_slots)
        self.steps = []

    def step(self, slots, prefix, new, final, embeds, token_ids=None, B=0, beam_src=None, logits=None, want_logits=True):
        assert len(slots) >= 1 and len(slots) == len(prefix) == len(new) == len(final)
        assert embeds.dim() == 2 and embeds.shape[0] == sum(new)
        self.steps.append((B, list(slots), list(prefix), list(new), list(final)))
        live = [s for s in range(self.n_slots) if self.group[s] >= 0]
        if B:
            assert live and max(live) < B <= self.n_slots
            self.llm_decode(token_ids=token_ids, beam_src=beam_src, logits=logits, B=B)
        else:
            assert beam_src is None and logits is None
        self._slots(slots, True)
        out, row = [], 0
        for s, p, k, f in zip(slots, prefix, new, final):
            assert 1 <= k and p + k <= self.cfg.llm_max_seq - (0 if f else 1)
            pad = self.kept[s][1] if p else 0
            out.append(self.extend([s], [p], [k], embeds[row:row + k].unsqueeze(0)))
            row += k
            if not f:                                  # kept at p + k: free, not decoded, continued by the next chunk
                cache = self.caches[s]
                self.caches[s] = self.masks[s] = None
                self.group[s], self.lens[s], self.own[s] = -1, 0, 0
                self.kept[s] = (cache, pad, p + k)
        return torch.cat(out)


@pytest.fixture(scope="module")
def sd():
    return make_emu2_state_dict()


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD)


def _run_trace(sd, gold, chunk, prefix_cache=False, n_slots=16, arrivals=None):
    from emu_b200.batching import SlotScheduler
    prompts = _prompts(gold)
    eng = ChunkOracleEngine(sd, max_batch=n_slots)
    sched = SlotScheduler(_model(eng), n_slots, prefix_cache=prefix_cache, prefill_chunk=chunk)
    reqs, step = {}, 0
    while step <= max(arrivals) or sched.busy():
        for name, p, spec, extra in arrivals.get(step, []):
            ids, img = prompts[p]
            if extra is not None:
                ids = torch.cat([ids, extra], 1)
            reqs[name] = sched.submit(_request(ids, img, spec))
        sched.step()
        step += 1
    for name, r in reqs.items():
        assert r.done.is_set() and r.error is None, (name, r.error)
    return {name: r.result for name, r in reqs.items()}, eng, sched


# greedy, sampling with a generator, 5-beam (its prompt spans several chunks at small C), beam-sample; staggered
ARRIVALS = {0: [(n, p, s, None) for n, p, s in SPECS[:2]], 1: [(n, p, s, None) for n, p, s in SPECS[4:5]],
            3: [(n, p, s, None) for n, p, s in SPECS[3:4] + SPECS[7:8]], 5: [(n, p, s, None) for n, p, s in SPECS[8:10]]}


@pytest.mark.parametrize("chunk", [1, 7, 64, "prompt"])
def test_chunked_requests_get_the_unchunked_ids(sd, gold, chunk):
    longest = max(p[0].shape[1] for p in _prompts(gold))
    got, eng, sched = _run_trace(sd, gold, longest if chunk == "prompt" else chunk, arrivals=ARRIVALS)
    want, eng0, _ = _run_trace(sd, gold, None, arrivals=ARRIVALS)
    for name in want:
        assert torch.equal(got[name], want[name]), (name, got[name].tolist(), want[name].tolist())
    C = longest if chunk == "prompt" else chunk
    assert sched.prefill_chunks == len(eng.steps) > 0
    assert all(sum(new) <= C for _, _, _, new, _ in eng.steps)
    assert all(t <= C for _, t in sched.mixed_sizes)
    if chunk == 1:                                   # a 5-beam prompt spanned many steps before it forked
        beam = [s for s in eng.steps if 0 in s[1]]
        assert len(beam) > 5 and beam[-1][4] == [1] and all(f == [0] for *_, f in beam[:-1])


def test_prefix_cache_resumes_start_their_first_chunk_at_the_prefix(sd, gold):
    prompts = _prompts(gold)
    base = prompts[2][0]
    more = torch.tensor([[11, 12, 13, 14, 15, 16, 17, 18, 19]])
    arrivals = {0: [("first", 2, dict(num_beams=1, max_new_tokens=4), None)],
                12: [("resume", 2, dict(num_beams=1, max_new_tokens=5), more),
                     ("resume_beam", 2, dict(num_beams=3, max_new_tokens=4), torch.cat([more, more], 1))]}
    got, eng, sched = _run_trace(sd, gold, 4, prefix_cache=True, n_slots=8, arrivals=arrivals)
    want, _, sched0 = _run_trace(sd, gold, None, prefix_cache=True, n_slots=8, arrivals=arrivals)
    for name in want:
        assert torch.equal(got[name], want[name]), name
    assert sched.prefix_hits == sched0.prefix_hits >= 1 and sched.prefix_tokens_reused == sched0.prefix_tokens_reused
    assert base.shape[1] in [p for st in eng.steps for p in st[2]]   # a resume's first chunk starts at its prefix


def test_live_requests_advance_every_step_while_a_long_prompt_prefills(sd, gold):
    from emu_b200.batching import SlotScheduler
    prompts = _prompts(gold)
    eng = ChunkOracleEngine(sd, max_batch=8)
    sched = SlotScheduler(_model(eng), 8, prefill_chunk=3)
    live = sched.submit(_request(*prompts[3], dict(num_beams=1, max_new_tokens=40, min_len=40)))
    while live not in sched.live:
        sched.step()
    sched.step()
    newcomer = sched.submit(_request(*prompts[0], dict(num_beams=1, max_new_tokens=3)))
    n_prompt = prompts[0][0].shape[1]
    seen, before_steps = [], len(sched.mixed_sizes)
    while newcomer not in sched.live and not newcomer.done.is_set():
        before = live.step
        sched.step()
        seen.append(live.step - before)
    assert len(seen) >= (n_prompt + 2) // 3 and seen == [1] * len(seen)    # one token per step, no stall step
    assert all(B >= 1 for B, _ in list(sched.mixed_sizes)[before_steps:])   # the live row rode on every chunk
    sched.run_until_idle()
    assert torch.equal(newcomer.result, _run_trace(sd, gold, None, arrivals={0: [("x", 0, dict(num_beams=1, max_new_tokens=3),
                                                                                     None)]})[0]["x"])


def test_a_masked_prompt_takes_the_join_path(sd, gold):
    from emu_b200.batching import SlotRequest, SlotScheduler
    prompts = _prompts(gold)
    eng = ChunkOracleEngine(sd, max_batch=8)
    sched = SlotScheduler(_model(eng), 8, prefill_chunk=4)
    ids = prompts[3][0]
    padded = torch.cat([torch.zeros(1, 3, dtype=ids.dtype), ids], 1)
    mask = torch.cat([torch.zeros(1, 3, dtype=torch.long), torch.ones_like(ids)], 1)
    r = sched.submit(SlotRequest(padded, mask, num_beams=1, max_new_tokens=4))
    plain = sched.submit(_request(ids, None, dict(num_beams=1, max_new_tokens=4)))
    sched.run_until_idle()
    assert r.error is None and plain.error is None
    assert [s for s in eng.steps if r.slots[0] in s[1]] == []             # never a segment of a mixed step ...
    assert [s for s in eng.steps if plain.slots[0] in s[1]]               # ... the unpadded prompt was
    assert torch.equal(r.result, plain.result)


def test_a_failing_mixed_step_fails_its_requests_and_the_scheduler_goes_on(sd, gold):
    from emu_b200.batching import SlotScheduler
    prompts = _prompts(gold)
    eng = ChunkOracleEngine(sd, max_batch=8)
    sched = SlotScheduler(_model(eng), 4, prefill_chunk=5)
    real = eng.step

    def broken(*a, **kw):
        raise RuntimeError("mixed step failed")
    eng.step = broken
    bad = sched.submit(_request(*prompts[0], dict(num_beams=1, max_new_tokens=3)))
    sched.step()
    assert isinstance(bad.error, RuntimeError) and sched.owner == [None] * 4 and not sched.prefilling and not sched.busy()
    eng.step = real
    spec = dict(num_beams=3, max_new_tokens=4)
    good = sched.submit(_request(*prompts[0], spec))
    sched.run_until_idle()
    assert good.error is None
    assert torch.equal(good.result, _run_trace(sd, gold, None, arrivals={0: [("x", 0, spec, None)]})[0]["x"])


def test_prefill_chunk_must_be_positive(sd):
    from emu_b200.batching import SlotScheduler
    with pytest.raises(ValueError, match="prefill_chunk"):
        SlotScheduler(_model(ChunkOracleEngine(sd)), 4, prefill_chunk=0)


# ---- the serving shell ----
def test_prefill_chunk_needs_continuous_batching():
    from emu_b200 import serve
    from test_serve_cpu import FakeChat
    with pytest.raises(SystemExit):
        serve.main(["--prefill-chunk", "64", "--disable-generate", "--disable-chat"])
    with pytest.raises(ValueError, match="continuous"):
        serve.EmuServer(chat=FakeChat(), host="127.0.0.1", port=0, chat_prefill_chunk=64)


def test_the_server_builds_a_chunking_scheduler(sd):
    from emu_b200 import serve
    from test_batching_cpu import _chat
    srv = serve.EmuServer(chat=_chat(ChunkOracleEngine(sd, max_batch=8)), host="127.0.0.1", port=0,
                          chat_scheduler="continuous", chat_prefill_chunk=32, chat_prefix_cache=True).start()
    try:
        sched = srv.chat_workers[0].scheduler
        assert sched.prefill_chunk == 32 and sched.prefix_cache
    finally:
        srv.shutdown()


# ---- the C entry points ----
HEADER = os.path.join(ROOT, "include", "emu_b200_chunked.h")


@pytest.fixture(scope="module")
def lib():
    from emu_b200 import build, _lib
    build.build()
    return _lib.load()


def test_chunked_header_symbols_are_bound_exported_and_disjoint(lib):
    from emu_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(emu_[a-z0-9_]+)\s*\(", src)))
    assert sorted(_lib.CHUNKED_SYMBOLS) == syms
    assert all(hasattr(lib, s) for s in syms)
    others = set(_lib.SYMBOLS + _lib.SAFETY_SYMBOLS + _lib.SLOT_SYMBOLS + _lib.OPS_SYMBOLS + _lib.PREFIX_SYMBOLS +
                 _lib.GEN_SLOT_SYMBOLS + _lib.DIFFUSION_OPS_SYMBOLS)
    assert not others & set(syms)


def test_chunked_entry_points_refuse_bad_arguments_without_a_gpu(lib):
    N = None
    one = (ctypes.c_int32 * 1)(0)
    st = (ctypes.c_int64 * 10)(*([8] * 10))
    V = ctypes.c_void_p(16)
    f = ctypes.c_float(1.0)
    cases = {
        # engine, token_ids, beam_src, B, logits, slots, prefix, new, final, n, embeds, logits_last, stream
        "emu_llm_step": [(N, V, N, 1, N, one, one, one, one, 1, V, N, N),
                         (V, V, N, 1, N, N, one, one, one, 1, V, N, N),
                         (V, V, N, 1, N, one, one, one, N, 1, V, N, N),
                         (V, V, N, 1, N, one, one, one, one, 0, V, N, N),       # n = 0 is emu_llm_decode
                         (V, V, N, 1, N, one, one, one, one, 1, N, N, N),
                         (V, N, N, 1, N, one, one, one, one, 1, V, N, N),       # decode rows without tokens
                         (V, V, N, -1, N, one, one, one, one, 1, V, N, N),
                         (V, N, V, 0, N, one, one, one, one, 1, V, N, N)],      # re-parenting with no decode rows
        # qkv, M, B, n, H, D, cos, sin, pos, pos_off, active, q_out, seg_row, seg_q0, seg_new, seg_posoff, k, v, t_max, s
        "emu_op_rope_kv_write_packed": [(N, 4, 1, 1, 2, 64, V, V, V, V, V, V, V, V, V, N, V, V, 16, N),
                                        (V, 4, 1, 1, 2, 64, V, V, N, V, V, V, V, V, V, N, V, V, 16, N),
                                        (V, 4, 1, 1, 2, 64, V, V, V, V, V, N, V, V, V, N, V, V, 16, N),
                                        (V, 4, 1, 1, 2, 64, V, V, V, V, V, V, V, N, V, N, V, V, 16, N),
                                        (V, 1, 1, 1, 2, 64, V, V, V, V, V, V, V, V, V, N, V, V, 16, N),
                                        (V, 4, 0, 0, 2, 64, V, V, V, V, V, V, V, V, V, N, V, V, 16, N),
                                        (V, 99, 33, 1, 2, 64, V, V, V, V, V, V, V, V, V, N, V, V, 16, N),
                                        (V, 4, 1, 1, 2, 48, V, V, V, V, V, V, V, V, V, N, V, V, 16, N)],
        # q, k, v, out, rows, B, H, Nq, Nk, D, st10, scale, q_row0, q_len, q_off, kv_start, kv_row, kv_rows, s
        "emu_op_attn_prefill_packed": [(V, V, V, V, 8, 1, 2, 4, 8, 64, st, f, N, V, V, N, N, 0, N),
                                       (V, V, V, V, 8, 1, 2, 4, 8, 64, st, f, V, N, V, N, N, 0, N),
                                       (V, V, V, V, 8, 1, 2, 4, 8, 64, st, f, V, V, N, N, N, 0, N),
                                       (V, V, V, V, 8, 1, 2, 4, 8, 96, st, f, V, V, V, N, N, 0, N),
                                       (V, V, V, V, 0, 1, 2, 4, 8, 64, st, f, V, V, V, N, N, 0, N),
                                       (V, V, V, V, 8, 33, 2, 4, 8, 64, st, f, V, V, V, N, N, 0, N),
                                       (V, V, V, V, 8, 1, 2, 4, 8, 64, st, f, V, V, V, N, V, 0, N)],
    }
    for name, args in cases.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = ctypes.c_int, None
        for a in args:
            assert fn(*a) == -1, (name, a)
