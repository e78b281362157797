"""CPU: prompt-lookup speculative decoding (generation.speculative_greedy_search) — the draft restated in oracle/spec_oracle.py
against transformers' PromptLookupCandidateGenerator, and the driver over engine doubles whose verify / commit are the CPU
oracle (or a tiny transformers LlamaForCausalLM): the ids must be those of plain greedy search."""
import random
from types import MethodType, SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from oracle import emu_oracle as O
from oracle import spec_oracle as S
from test_generation_cpu import L, NH, OracleEngine, _emu1_model, setup  # noqa: F401  (setup is a fixture)


# ---- the draft against transformers 5.5 -------------------------------------------------------------------------------------
def _hf_draft(hist, k, g, max_length, eos):
    from transformers.generation.candidate_generator import PromptLookupCandidateGenerator
    gen = PromptLookupCandidateGenerator(eos_token_id=torch.tensor([eos]), num_output_tokens=k, max_matching_ngram_size=g,
                                         max_length=max_length)
    ids = torch.tensor([hist])
    cand, _ = gen.get_candidates(ids)
    return cand[0, len(hist):].tolist()


def _histories():
    rng = random.Random(0)
    cases = []
    for _ in range(300):
        n = rng.randint(1, 40)
        vocab = rng.choice([3, 5, 12, 50])                       # small vocabularies repeat n-grams often
        hist = [rng.randrange(vocab) for _ in range(n)]
        k, g = rng.randint(1, 7), rng.randint(1, 3)
        max_length = rng.choice([n + 1, n + 2, n + 5, n + 50, max(1, n - 3)])
        cases.append((hist, k, g, max_length, rng.randrange(vocab)))
    cases += [([1, 2, 3, 4], 3, 2, 20, 9),                        # no match
              ([5, 6, 7, 5, 6, 2, 8, 5, 6], 4, 2, 30, 2),         # EOS in the continuation: cut before it
              ([5, 6, 2, 8, 5, 6], 4, 2, 30, 2),                  # ... right at its start: no draft
              ([1, 2, 3, 9, 9, 9, 1, 2, 3], 7, 3, 30, 0),         # 3-gram
              ([4, 1, 2, 7, 7, 7, 4, 1, 2], 7, 3, 8, 0),          # max_length inside the continuation
              ([4, 1, 2, 7, 7, 7, 4, 1], 7, 3, 9, 0)]             # max_length == len + 1: none
    return cases


def test_draft_restatement_matches_transformers():
    kinds = set()
    for hist, k, g, max_length, eos in _histories():
        mine = S.prompt_lookup_draft(list(hist), k, g, max_length, eos)
        assert mine == _hf_draft(hist, k, g, max_length, eos), (hist, k, g, max_length, eos)
        kinds.add("draft" if mine else "none")
        if mine and len(mine) < k:
            kinds.add("short")
    assert kinds == {"draft", "none", "short"}


def test_accept_restatement():
    hist = [1, 2]
    assert S.accept(hist, [3, 4, 5], [3, 4, 9, 6], eos_id=0, max_len=50) == (3, False) and hist == [1, 2, 3, 4, 9]
    hist = [1]
    assert S.accept(hist, [3, 0, 5], [3, 0, 5, 6], eos_id=0, max_len=50) == (2, True) and hist == [1, 3, 0]
    hist = [1]
    assert S.accept(hist, [3, 4, 5], [3, 4, 5, 6], eos_id=0, max_len=3) == (2, True) and hist == [1, 3, 4]
    hist = [1]
    assert S.accept(hist, [], [7], eos_id=0, max_len=9) == (1, False) and hist == [1, 7]


# ---- engine doubles ---------------------------------------------------------------------------------------------------------
def _spec_draft(self, hist, hist_len, k, max_ngram, max_length, eos, out, out_len):
    h = hist[:int(hist_len)].tolist()
    d = S.prompt_lookup_draft(h, k, max_ngram, max_length, eos)
    out[0] = h[-1]
    out[1:1 + len(d)] = torch.tensor(d, dtype=out.dtype)
    out_len[0] = len(d)


def _spec_accept(self, hist, hist_len, tokens, next_ids, n, eos, max_len, stats):
    h = hist[:int(hist_len)].tolist()
    m, done = S.accept(h, tokens[1:n].tolist(), next_ids[:n].tolist(), eos, max_len)
    hist[:len(h)] = torch.tensor(h, dtype=hist.dtype)
    hist_len[0] = len(h)
    stats[0], stats[1] = m, int(done)
    self.calls.append(("accept", n, m))


def _with_spec_ops(eng):
    eng.spec_draft, eng.spec_accept = MethodType(_spec_draft, eng), MethodType(_spec_accept, eng)
    eng.calls = []
    return eng


class SpecOracleEngine(OracleEngine):
    """OracleEngine + emu_llm_verify / emu_llm_commit by the oracle, and the draft / accept restatements"""

    def __init__(self, sd, max_batch=8, max_seq=512):
        super().__init__(sd, max_batch)
        self.cfg.llm_max_seq = max_seq
        _with_spec_ops(self)

    def llm_verify(self, tokens, n, logits=None, next_ids=None, ban_id=-1, ban_rows=0):
        assert self.mask.shape[0] == 1 and 1 <= n <= min(8, self.cfg.llm_max_batch)
        assert self.cache.length() + n <= self.cfg.llm_max_seq, "KV cache full"
        self.len0 = self.cache.length()
        e = F.embedding(tokens[:n].long(), self.sd["decoder.lm.model.embed_tokens.weight"])[None]
        self.mask = torch.cat((self.mask, torch.ones(1, n, dtype=self.mask.dtype)), dim=1)
        pos = (self.mask.long().cumsum(-1) - 1)[:, -n:] if self.hf else None
        h = O.llama_forward(self.sd, e, self.mask, layers=L, heads=NH, position_ids=pos, cache=self.cache)
        lg = O.lm_logits(self.sd, h[0]).float()
        if logits is not None:
            logits[:n].copy_(lg)
        if ban_id >= 0:
            lg[:ban_rows, ban_id] = float("-inf")
        next_ids[:n].copy_(lg.argmax(-1).to(next_ids.dtype))
        self.calls.append(("verify", n))

    def llm_commit(self, m):
        keep = self.len0 + m
        self.cache.k = [t[:, :, :keep] for t in self.cache.k]
        self.cache.v = [t[:, :, :keep] for t in self.cache.v]
        self.mask = self.mask[:, :keep]


def _greedy(eng, emb, mask, n, eos=2, min_length=0):
    from emu_b200 import generation
    return generation.greedy_search(eng, emb, mask, n, eos, 32000, min_length=min_length)


def _spec(eng, emb, mask, n, k, eos=2, min_length=0, prompt_ids=None):
    from emu_b200 import generation
    return generation.generate(eng, emb, mask, n, eos, 32000, num_beams=1, min_length=min_length,
                               prompt_lookup_num_tokens=k, prompt_ids=prompt_ids)


@pytest.mark.parametrize("k", [1, 3, 7])
def test_emu2_golden_greedy(setup, k):  # noqa: F811
    gold, sd, emb = setup
    mask = gold["gen_attention_mask"]
    for b in range(emb.shape[0]):
        ids = _spec(SpecOracleEngine(sd), emb[b:b + 1], mask[b:b + 1], 12, k, min_length=1,
                    prompt_ids=gold["gen_input_ids"][b:b + 1])
        assert torch.equal(ids, _greedy(OracleEngine(sd), emb[b:b + 1], mask[b:b + 1], 12, min_length=1))
        assert torch.equal(ids[0], gold["gen_ids_greedy"][b])


@pytest.mark.parametrize("k", [1, 3, 7])
def test_emu1_golden_greedy(k):
    import os
    gold = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "emu1_generate_tiny.pt"))
    m, sd = _emu1_model(torch.float32)
    m.engine.cfg.llm_max_seq = 512
    m.engine.llm_verify = MethodType(SpecOracleEngine.llm_verify, m.engine)
    m.engine.llm_commit = MethodType(SpecOracleEngine.llm_commit, m.engine)
    _with_spec_ops(m.engine)
    for b in range(gold["input_ids"].shape[0]):
        kw = dict(image=gold["image"][b:b + 1], max_new_tokens=12, min_length=1, eos_token_id=2, pad_token_id=32000,
                  num_beams=1)
        plain = m.generate_from_ids(gold["input_ids"][b:b + 1], gold["attention_mask"][b:b + 1], **kw)
        spec = m.generate_from_ids(gold["input_ids"][b:b + 1], gold["attention_mask"][b:b + 1], prompt_lookup_num_tokens=k,
                                   **kw)
        assert torch.equal(spec, plain)
        assert any(c[0] == "verify" for c in m.engine.calls)


def _plain_run(sd, n=24):
    """a prompt, its embeddings and the plain greedy continuation (no EOS among the first n tokens with eos = -1)"""
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, 32000, (1, 9), generator=g)
    emb = F.embedding(ids, sd["decoder.lm.model.embed_tokens.weight"])
    mask = torch.ones(1, 9, dtype=torch.long)
    return ids, emb, mask, _greedy(OracleEngine(sd), emb, mask, n, eos=32001)


@pytest.mark.parametrize("k", [1, 3, 7])
def test_repetitive_prompt_accepts_most_drafts(setup, k):  # noqa: F811
    """the draft source holds the continuation itself: almost every draft is accepted, and the ids do not change"""
    _, sd, _ = setup
    ids, emb, mask, plain = _plain_run(sd)
    eng = SpecOracleEngine(sd)
    out = _spec(eng, emb, mask, 24, k, eos=32001, prompt_ids=torch.cat((ids, plain), 1))
    assert torch.equal(out, plain)
    verifies = [c for c in eng.calls if c[0] == "verify"]
    assert len(verifies) <= -(-23 // (k + 1)) + 1, eng.calls
    unguided = SpecOracleEngine(sd)
    assert torch.equal(_spec(unguided, emb, mask, 24, k, eos=32001, prompt_ids=ids), plain)


@pytest.mark.parametrize("k", [1, 3, 7])
@pytest.mark.parametrize("case", ["eos_in_run", "max_new_mid_run", "min_length"])
def test_stops_like_greedy(setup, k, case):  # noqa: F811
    _, sd, _ = setup
    ids, emb, mask, plain = _plain_run(sd)
    guide = torch.cat((ids, plain), 1)
    eos, n, min_length = 32001, 24, 0
    if case == "eos_in_run":
        eos = int(plain[0, 6])                    # inside the first accepted run of a draft copied from the guide
    elif case == "max_new_mid_run":
        n = 10
    else:
        eos, min_length = int(plain[0, 2]), 5     # banned in the first rows: the plain run changes after it
    ref = _greedy(OracleEngine(sd), emb, mask, n, eos=eos, min_length=min_length)
    out = _spec(SpecOracleEngine(sd), emb, mask, n, k, eos=eos, min_length=min_length, prompt_ids=guide)
    assert torch.equal(out, ref), (out, ref)
    if case == "eos_in_run":
        assert out.shape[1] <= 7 and int(out[0, -1]) == eos


def test_refusals(setup):  # noqa: F811
    from emu_b200 import generation
    gold, sd, emb = setup
    e1, m1 = emb[:1], gold["gen_attention_mask"][:1]
    eng = SpecOracleEngine(sd)

    def gen(e=e1, m=m1, engine=eng, **kw):
        kw.setdefault("prompt_lookup_num_tokens", 3)
        return generation.generate(engine, e, m, 8, 2, 32000, **kw)

    for kw, exc, what in ((dict(do_sample=True), ValueError, "greedy"), (dict(num_beams=2), ValueError, "greedy"),
                          (dict(repetition_penalty=1.2), NotImplementedError, "repetition_penalty"),
                          (dict(no_repeat_ngram_size=2), NotImplementedError, "no_repeat_ngram_size"),
                          (dict(prefix_allowed_tokens_fn=lambda b, s: [1]), NotImplementedError, "prefix_allowed"),
                          (dict(prompt_lookup_num_tokens=8), ValueError, "[1, 7]"),
                          (dict(prompt_lookup_num_tokens=0), ValueError, "[1, 7]"),
                          (dict(penalty_alpha=0.6, top_k=4), ValueError, "contrastive"),
                          (dict(max_matching_ngram_size=0), ValueError, "max_matching_ngram_size")):
        with pytest.raises(exc, match=None) as ei:
            gen(**kw)
        assert what in str(ei.value), (kw, str(ei.value))
    with pytest.raises(ValueError, match="batch=2"):
        gen(e=emb, m=gold["gen_attention_mask"])
    with pytest.raises(ValueError, match="llm_max_batch = 4"):
        gen(engine=SpecOracleEngine(sd, max_batch=4), prompt_lookup_num_tokens=4)
    assert eng.calls == []


# ---- the driver over transformers' own LlamaForCausalLM --------------------------------------------------------------------
class HFEngine:
    """prefill / verify / commit on a transformers LlamaForCausalLM with a DynamicCache (no padding)"""

    def __init__(self, model, max_seq=256):
        self.m = model
        self.cfg = SimpleNamespace(llm_vocab=model.config.vocab_size, llm_max_batch=8, llm_max_seq=max_seq)
        _with_spec_ops(self)

    def llm_reset(self):
        self.cache = None

    def llm_prefill(self, embeds, attention_mask, hf_positions=True, want_hidden=False, want_logits=True):
        from transformers import DynamicCache
        self.cache = DynamicCache()
        out = self.m(inputs_embeds=embeds, attention_mask=attention_mask, past_key_values=self.cache, use_cache=True)
        return None, out.logits[:, -1].float()

    def llm_verify(self, tokens, n, logits=None, next_ids=None, ban_id=-1, ban_rows=0):
        self.len0 = self.cache.get_seq_length()
        lg = self.m(input_ids=tokens[None, :n].long(), past_key_values=self.cache, use_cache=True).logits[0].float()
        if ban_id >= 0:
            lg[:ban_rows, ban_id] = float("-inf")
        next_ids[:n].copy_(lg.argmax(-1).to(next_ids.dtype))
        self.calls.append(("verify", n))

    def llm_commit(self, m):
        self.cache.crop(self.len0 + m)


@pytest.mark.parametrize("k", [1, 3, 7])
def test_driver_matches_transformers_prompt_lookup(k):
    from transformers import LlamaConfig, LlamaForCausalLM
    from emu_b200 import generation
    torch.manual_seed(0)
    cfg = LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=4,
                      vocab_size=50, max_position_embeddings=256, eos_token_id=3, pad_token_id=0, bos_token_id=1)
    model = LlamaForCausalLM(cfg).eval()
    # a small vocabulary and a repeating prompt make the random model repeat itself, so drafts do get accepted
    ids = torch.tensor([[1] + [5, 9, 11, 7, 13, 21] * 5])
    with torch.no_grad():
        ref = model.generate(ids, attention_mask=torch.ones_like(ids), do_sample=False, max_new_tokens=30,
                             prompt_lookup_num_tokens=k, eos_token_id=3, pad_token_id=0)[:, ids.shape[1]:]
        plain = model.generate(ids, attention_mask=torch.ones_like(ids), do_sample=False, max_new_tokens=30,
                               eos_token_id=3, pad_token_id=0)[:, ids.shape[1]:]
        eng = HFEngine(model)
        out = generation.generate(eng, model.get_input_embeddings()(ids), torch.ones_like(ids), 30, 3, 0, num_beams=1,
                                  prompt_lookup_num_tokens=k, prompt_ids=ids)
    assert torch.equal(out, ref), (out, ref)
    assert torch.equal(out, plain)
    assert len([c for c in eng.calls if c[0] == "verify"]) < out.shape[1]
