"""Autoregressive generation control on top of the engine's prefill/decode steps.

Restates the two HF `GenerationMixin` strategies the reference drives through `lm.generate(inputs_embeds=...)`
(Emu2/emu/emu.py:213-229; Emu1/models/modeling_emu.py:162-179): greedy search and beam search
(num_beams=5, length_penalty=-1 are the reference defaults), plus sampling.  Token selection runs on the GPU; the
greedy loop never synchronises with the host inside the loop (token ids are chained device-to-device through the
CUDA-graphed decode step), and neither does beam search: its per-step hypothesis bookkeeping is a device kernel
(emu_beam_step) and the host reads the "finished" flag every few steps only.

When driven by inputs_embeds HF returns only the NEW tokens; so do these functions.

Strategies (the combinations `lm.generate` picks from do_sample / num_beams / penalty_alpha, and which callers reach them):
  greedy_search        num_beams=1                         README image captioning; + logits processors (repetition_penalty,
                                                           no_repeat_ngram_size, prefix_allowed_tokens_fn) like HF `_sample`
  sample_search        do_sample, num_beams=1              chat demo (Emu2/demo/backend/pytorch_model/backend.py:196-214)
  beam_search          num_beams>1 (reference default 5)   every default call; do_sample=True -> HF beam-sample (what the demo
                                                           runs when "do_sample" is ticked with its default num_beams=5)
  contrastive_search   penalty_alpha>0, top_k>1, 1 beam    Emu2/emu/emu.py:166,222 / Emu1 modeling_emu.py:110 forward the knob
  speculative_greedy_  prompt_lookup_num_tokens=k, greedy, HF prompt-lookup assisted generation (lm.generate's **kwargs): the
    search             batch 1                             greedy ids, several drafted tokens checked per weight pass
`num_return_sequences` (Emu1 `num_captions`, modeling_emu.py:113,177) is honoured by beam search (n best hypotheses per prompt) and
sampling (n independent draws per prompt, one prefill).

How greedy (with processors), sampling and beam search pick their tokens lives in one selector per strategy, which holds
the per-call state (`selector` maps the knobs to one).  `select(logits, step)`, `done()` and `output()` drive the solo
loops here and the continuous-batching scheduler (batching.py), which runs one selector per request on its own rows.
"""
import torch


def decoding_knobs(num_beams, repetition_penalty, no_repeat_ngram_size, num_return_sequences):
    """the knobs callers may pass as None, normalised as `generate` takes them:
    (num_beams, repetition_penalty, no_repeat_ngram_size, num_return_sequences)"""
    if num_beams is None or num_beams < 1:
        raise ValueError("num_beams has to be an integer >= 1")
    return (int(num_beams), 1.0 if repetition_penalty is None else float(repetition_penalty), int(no_repeat_ngram_size or 0),
            max(1, int(num_return_sequences or 1)))


def _allowed_mask(prefix_allowed_tokens_fn, seqs, V, device):
    """PrefixConstrainedLogitsProcessor's mask: seqs [rows_outer, rows_inner, cur_len] (host int64) -> uint8 [rows, V], 1 = allowed.
    The callback is host Python by construction (Emu1/mm_eval/models/emu.py:97-109), so this path reads the tokens back."""
    Bt, nb = seqs.shape[0], seqs.shape[1]
    allowed = torch.zeros(Bt * nb, V, dtype=torch.uint8)
    for b in range(Bt):
        for k in range(nb):
            ok = prefix_allowed_tokens_fn(b, seqs[b, k])
            allowed[b * nb + k, torch.as_tensor(list(ok), dtype=torch.long)] = 1
    return allowed.to(device)


def _finish_rows(toks, eos_token_id, pad_token_id):
    """HF `_sample` output form: after a row's first EOS every later token is pad; trimmed to the step at which the last
    row finished (the loop may have run a few steps past it between two host checks)."""
    is_eos = toks == eos_token_id
    after = (is_eos.cumsum(1) - is_eos.long()) > 0
    toks = toks.masked_fill(after, pad_token_id)
    if bool(is_eos.any(1).all()):
        last = int((is_eos.float().argmax(1)).max()) + 1
        toks = toks[:, :last]
    return toks


def _prefill(engine, inputs_embeds, attention_mask, n):
    """the prompts' last logits, each prompt's cache row mapped to n rows.  HF expands the inputs n times and prefills every
    copy; here each prompt is prefilled ONCE (same cache contents, 1 / n of the work)."""
    engine.llm_reset()
    _, logits = engine.llm_prefill(inputs_embeds, attention_mask, hf_positions=True, want_logits=True)
    if n > 1:
        B = inputs_embeds.shape[0] * n
        engine.llm_expand(torch.arange(B, device=inputs_embeds.device, dtype=torch.int32) // n, B)
        logits = logits.repeat_interleave(n, dim=0).contiguous()
    return logits


def _decode_loop(engine, sel, logits, max_new_tokens, check_every):
    """select -> poll the finish flag every `check_every` steps -> decode, for at most max_new_tokens steps.  The tensors
    handed to the decode step keep their addresses for the whole call (CUDA graphs / plans are keyed by their pointers)."""
    logits_buf = torch.empty_like(logits)
    for step in range(max_new_tokens):
        ids = sel.select(logits, step)
        if step + 1 == max_new_tokens or (check_every and (step + 1) % check_every == 0 and bool(sel.done())):
            break
        engine.llm_decode(token_ids=ids, beam_src=sel.beam_src, logits=logits_buf, B=logits.shape[0])
        logits = logits_buf
    return sel.output()


class _Selector:
    """What the strategies share: HF's logits processors (`_topk`) and `n`, the steps selected so far."""

    beam_src = None

    def __init__(self, engine, eos_token_id, device, min_length, repetition_penalty, no_repeat_ngram_size,
                 prefix_allowed_tokens_fn):
        self.engine, self.eos, self.device, self.min_length = engine, eos_token_id, device, min_length
        self.repetition_penalty, self.ngram, self.prefix_fn = repetition_penalty, no_repeat_ngram_size, prefix_allowed_tokens_fn
        self.n = 0

    def _topk(self, logits, running_scores, beams, step, prev, seqs, penalty_on_logits):
        """emu_beam_topk with the processors (`prev`: the rows' tokens for the penalty and n-gram ban, or None; `seqs`
        [prompts, beams, >= step]: the same for the prefix callback); leaves the processed log-probabilities in `logits`"""
        allowed = None
        if self.prefix_fn is not None:
            allowed = _allowed_mask(self.prefix_fn, seqs[:, :, :step].to("cpu", torch.int64), self.engine.cfg.llm_vocab,
                                    self.device)
        return self.engine.beam_topk(logits, running_scores, logits.shape[0] // beams, beams, 2 * beams,
                                     ban_id=self.eos if step < self.min_length else -1, prev_tokens=prev, prev_len=step,
                                     repetition_penalty=self.repetition_penalty, penalty_on_logits=penalty_on_logits,
                                     no_repeat_ngram=self.ngram, allowed=allowed)


class GreedySelector(_Selector):
    """Greedy search over `rows` rows with HF's logits processors, in `_sample`'s order: RepetitionPenalty on the RAW logits
    -> NoRepeatNGram -> MinLength -> PrefixConstrained -> argmax; a finished row emits pad.  The processors and the selection
    are the device kernels of emu_beam_topk run with one beam (log_softmax is monotone per row, so its top-1 is the processed
    logits' argmax); `input_ids` for the processors is what HF sees when generation is driven by inputs_embeds: the tokens
    generated so far, pads included.  Without processors the arg-max is taken from the logits with EOS banned below
    min_length (what greedy_search's in-graph arg-max does)."""

    def __init__(self, engine, rows, max_new_tokens, eos_token_id, pad_token_id, device, min_length=0, repetition_penalty=1.0,
                 no_repeat_ngram_size=0, prefix_allowed_tokens_fn=None):
        super().__init__(engine, eos_token_id, device, min_length, repetition_penalty, no_repeat_ngram_size,
                         prefix_allowed_tokens_fn)
        self.pad = pad_token_id
        self.processed = repetition_penalty != 1.0 or bool(no_repeat_ngram_size) or prefix_allowed_tokens_fn is not None
        i32 = dict(dtype=torch.int32, device=device)
        self.prev = torch.full((rows, max_new_tokens), pad_token_id, **i32)     # the tokens so far: processor input, output
        self.tokens = torch.empty(rows, **i32)                                  # the decode step's token_ids (fixed address)
        self.pad_t = torch.full((rows,), pad_token_id, **i32)
        self.finished = torch.zeros(rows, dtype=torch.bool, device=device)
        self.zero_run = torch.zeros(rows, 1, dtype=torch.float32, device=device)

    def _process(self, logits, step):
        return self._topk(logits, self.zero_run, 1, step, self.prev if step > 0 else None, self.prev[:, None], True)[1]

    def _pick(self, logits, step):
        if self.processed:
            return self._process(logits, step)[:, 0]                   # one beam: flat index == token id
        if step < self.min_length:
            logits[:, self.eos] = float("-inf")
        return logits.argmax(-1).to(torch.int32)

    def select(self, logits, step):
        """the next token of every row from its logits [rows, V] (overwritten): int32 [rows], always the same buffer"""
        nxt = torch.where(self.finished, self.pad_t, self._pick(logits, step), out=self.tokens)
        self.prev[:, step] = nxt
        self.finished |= nxt == self.eos
        self.n = step + 1
        return nxt

    def done(self):
        """device flag: every row has produced EOS"""
        return self.finished.all()

    def output(self):
        return _finish_rows(self.prev[:, :self.n].to(torch.int64), self.eos, self.pad)


class SampleSelector(GreedySelector):
    """Multinomial sampling, HF `_sample` order: the logits processors as GreedySelector runs them (they leave the processed
    log-probabilities in place; softmax(log_softmax(x) / T) == softmax(x / T), so the warpers see what HF's see) -> warpers
    temperature -> top_k -> top_p -> one draw per row, all in emu_sample_tokens.  Returns every step's tokens, pads after
    a row's EOS, untrimmed."""

    def __init__(self, *args, temperature=None, top_k=None, top_p=None, generator=None, **kwargs):
        super().__init__(*args, **kwargs)
        self.temperature, self.top_k, self.top_p = temperature or 1.0, top_k or 0, 1.0 if top_p is None else top_p
        # one fresh seed per call, DRAWN from the generator so that its state advances like torch.multinomial's would:
        # two do_sample calls with the same prompt differ, a re-seeded generator reproduces
        g = generator
        self.seed = int(torch.randint(0, 2 ** 62, (1,), generator=g, device="cpu" if g is None else g.device))

    def _pick(self, logits, step):
        if self.processed:
            self._process(logits, step)
        return self.engine.sample_tokens(logits, self.temperature, self.top_k, self.top_p,
                                         self.eos if step < self.min_length else -1, self.seed, step)

    def output(self):
        return self.prev[:, :self.n].to(torch.int64)


def _warp_log_probs(lp, temperature, top_k, top_p, min_keep):
    """HF's sampling warpers on [rows, V] scores, in GenerationMixin's order (TemperatureLogitsWarper -> TopKLogitsWarper ->
    TopPLogitsWarper); under beam search they keep at least `min_keep` = 2 tokens per row so a beam can always continue."""
    if temperature is not None and temperature != 1.0:
        lp = lp / temperature
    if top_k:
        k = min(max(int(top_k), min_keep), lp.shape[-1])
        kth = torch.topk(lp, k)[0][..., -1, None]
        lp = lp.masked_fill(lp < kth, float("-inf"))
    if top_p is not None and top_p < 1.0:
        s_sorted, s_idx = torch.sort(lp, descending=False)
        remove = s_sorted.softmax(-1).cumsum(-1) <= (1 - top_p)
        remove[..., -min_keep:] = False
        lp = lp.masked_fill(remove.scatter(1, s_idx, remove), float("-inf"))
    return lp


class BeamSelector(_Selector):
    """HF (transformers >= 4.50 vectorised) beam search over `batch` prompts x `num_beams` rows, decoder_prompt_len = 0
    because generation is driven by inputs_embeds.  A step never leaves the device: engine.beam_topk (emu_beam_topk:
    log_softmax, logits processors, running score, top 2*beams over beams x vocab) -> engine.beam_step (emu_beam_step: running
    / finished hypothesis bookkeeping, next tokens and KV-cache reorder indices `beam_src`).  Steps made after the search
    has finished are no-ops on the beam state.  `prefix_allowed_tokens_fn(batch_id, ids)` is a host callback by construction
    (Emu1/mm_eval/models/emu.py:97-109): when it is given, the running sequences are read back every step to build the
    allowed-token mask.

    do_sample=True is HF's beam-sample (`_get_top_k_continuations`): the processor kernels leave the processed
    log-probabilities in place, the sampling warpers and "+ running beam score" follow, and the 2*beams candidates are DRAWN
    without replacement (with `generator`, every step) from softmax over beams x vocab instead of taken by top-k; the
    bookkeeping is the same device step.  (do_sample with top_k < 2 * num_beams — the chat demo's defaults, top_k = 3 with
    5 beams — leaves the first step fewer live candidates than the 2 * num_beams it draws: torch.multinomial then returns
    zero-probability entries, whose accumulated score is -inf; those beams are dead from the start, exactly as in HF.)

    The output is the best `num_return_sequences` finished hypotheses per prompt ([batch * n, T], best first), padded."""

    def __init__(self, engine, batch, num_beams, max_new_tokens, eos_token_id, pad_token_id, device, min_length=0,
                 length_penalty=1.0, early_stopping=False, repetition_penalty=1.0, no_repeat_ngram_size=0,
                 prefix_allowed_tokens_fn=None, penalty_on_logits=False, num_return_sequences=1, do_sample=False,
                 temperature=None, top_k=None, top_p=None, generator=None):
        super().__init__(engine, eos_token_id, device, min_length, repetition_penalty, no_repeat_ngram_size,
                         prefix_allowed_tokens_fn)
        self.length_penalty, self.early_stopping, self.penalty_on_logits = length_penalty, early_stopping, penalty_on_logits
        self.n_ret, self.do_sample, self.generator = num_return_sequences, do_sample, generator
        self.temperature, self.top_k, self.top_p = temperature, top_k, top_p
        self.st = engine.beam_state(batch, num_beams, max_new_tokens, pad_token_id, device)
        self.need_prev = repetition_penalty != 1.0 or bool(no_repeat_ngram_size)
        self.zero_run = torch.zeros(batch, num_beams, dtype=torch.float32, device=device) if do_sample else None

    @property
    def beam_src(self):
        return self.st.beam_src

    def select(self, logits, step):
        """one beam-search step from the logits [batch * beams, V] (overwritten): the next tokens int32 [batch * beams]
        (`st.next_tokens`) and their cache rows `beam_src`"""
        st = self.st
        Bt, nb, V = st.batch, st.beams, logits.shape[-1]
        live = st.running_seq[st.live(step)]                       # [Bt, nb, max_length] tokens generated so far
        topk_lp, topk_i = self._topk(logits, self.zero_run if self.do_sample else st.running_scores, nb, step,
                                     live.view(Bt * nb, st.max_length) if self.need_prev and step > 0 else None, live,
                                     self.penalty_on_logits)
        if self.do_sample:
            lp = _warp_log_probs(logits.view(Bt * nb, V), self.temperature, self.top_k, self.top_p, min_keep=2)
            acc = (lp.view(Bt, nb, V) + st.running_scores.view(Bt, nb, 1)).view(Bt, nb * V)
            pick = torch.multinomial(torch.softmax(acc, dim=-1), num_samples=2 * nb, generator=self.generator)
            topk_lp, topk_i = torch.gather(acc, 1, pick).contiguous(), pick.to(torch.int32).contiguous()
        self.engine.beam_step(st, topk_lp, topk_i, step, self.eos, self.length_penalty, self.early_stopping)
        self.n = step + 1
        return st.next_tokens

    def done(self):
        """device flag: the search has finished"""
        return self.st.done

    def output(self):
        return self.st.result(self.n, self.n_ret).to(self.device)


def selector(engine, batch, max_new_tokens, eos_token_id, pad_token_id, device, num_beams=1, do_sample=False, min_length=0,
             length_penalty=1.0, early_stopping=False, repetition_penalty=1.0, no_repeat_ngram_size=0, temperature=None,
             top_k=None, top_p=None, generator=None):
    """the selector `generate` runs for these knobs (as `decoding_knobs` leaves them) on `batch` prompts, one sequence each:
    beam search / beam-sample, sampling or greedy search (contrastive search has no selector)"""
    common = dict(min_length=min_length, repetition_penalty=repetition_penalty, no_repeat_ngram_size=no_repeat_ngram_size)
    if num_beams > 1:
        return BeamSelector(engine, batch, num_beams, max_new_tokens, eos_token_id, pad_token_id, device,
                            length_penalty=length_penalty, early_stopping=early_stopping, do_sample=do_sample,
                            temperature=temperature, top_k=top_k, top_p=top_p, generator=generator, **common)
    if do_sample:
        return SampleSelector(engine, batch, max_new_tokens, eos_token_id, pad_token_id, device, temperature=temperature,
                              top_k=top_k, top_p=top_p, generator=generator, **common)
    return GreedySelector(engine, batch, max_new_tokens, eos_token_id, pad_token_id, device, **common)


@torch.no_grad()
def greedy_search(engine, inputs_embeds, attention_mask, max_new_tokens, eos_token_id, pad_token_id, min_length=0,
                  check_every=16, repetition_penalty=1.0, no_repeat_ngram_size=0, prefix_allowed_tokens_fn=None):
    """HF greedy: argmax; finished rows emit pad; stop when every row has produced EOS.  With a repetition penalty, an n-gram
    ban or a prefix constraint the per-step argmax goes through the processor kernels (`GreedySelector`)."""
    B = inputs_embeds.shape[0]
    dev = inputs_embeds.device
    logits = _prefill(engine, inputs_embeds, attention_mask, 1)
    if repetition_penalty != 1.0 or no_repeat_ngram_size or prefix_allowed_tokens_fn is not None:
        sel = GreedySelector(engine, B, max_new_tokens, eos_token_id, pad_token_id, dev, min_length, repetition_penalty,
                             no_repeat_ngram_size or 0, prefix_allowed_tokens_fn)
        return _decode_loop(engine, sel, logits, max_new_tokens, check_every)
    if min_length > 0:
        logits[:, eos_token_id] = float("-inf")
    out = torch.empty(max_new_tokens, B, dtype=torch.int32, device=dev)
    # two fixed token buffers used alternately, so the engine sees only two argument sets (CUDA graphs / plans are
    # keyed by their pointers); each step's ids are also copied into `out` device-to-device
    ping = [torch.empty(B, dtype=torch.int32, device=dev), torch.empty(B, dtype=torch.int32, device=dev)]
    ping[0].copy_(logits.argmax(-1))
    out[0].copy_(ping[0])
    n_done = 1
    for step in range(1, max_new_tokens):
        ban = eos_token_id if step < min_length else -1
        src, dst = ping[(step - 1) & 1], ping[step & 1]
        engine.llm_decode(token_ids=src, next_ids=dst, ban_id=ban, B=B)
        out[step].copy_(dst)
        n_done = step + 1
        if check_every and step % check_every == 0:
            if bool((out[:n_done] == eos_token_id).any(0).all()):
                break
    return _finish_rows(out[:n_done].t().to(torch.int64), eos_token_id, pad_token_id)


@torch.no_grad()
def sample_search(engine, inputs_embeds, attention_mask, max_new_tokens, eos_token_id, pad_token_id, min_length=0,
                  temperature=None, top_k=None, top_p=None, generator=None, repetition_penalty=1.0, no_repeat_ngram_size=0,
                  prefix_allowed_tokens_fn=None, num_return_sequences=1):
    """Multinomial sampling (`SampleSelector`).  num_return_sequences = n draws n independent continuations per prompt (HF
    expands the inputs n times; here each prompt is prefilled once and its cache row mapped to n rows); returns [B * n, T].
    The host reads the finish flag every step, so T is the step at which the last row produced EOS."""
    n = max(1, int(num_return_sequences or 1))
    B = inputs_embeds.shape[0] * n
    if B > engine.cfg.llm_max_batch:
        raise ValueError("batch x num_return_sequences = %d exceeds the engine's llm_max_batch = %d" % (B, engine.cfg.llm_max_batch))
    logits = _prefill(engine, inputs_embeds, attention_mask, n)
    sel = SampleSelector(engine, B, max_new_tokens, eos_token_id, pad_token_id, inputs_embeds.device, min_length,
                         repetition_penalty, no_repeat_ngram_size or 0, prefix_allowed_tokens_fn, temperature=temperature,
                         top_k=top_k, top_p=top_p, generator=generator)
    return _decode_loop(engine, sel, logits, max_new_tokens, check_every=1)


@torch.no_grad()
def beam_search(engine, inputs_embeds, attention_mask, num_beams, max_new_tokens, eos_token_id, pad_token_id,
                min_length=0, length_penalty=1.0, early_stopping=False, repetition_penalty=1.0, no_repeat_ngram_size=0,
                prefix_allowed_tokens_fn=None, penalty_on_logits=False, check_every=8, num_return_sequences=1,
                do_sample=False, temperature=None, top_k=None, top_p=None, generator=None):
    """HF beam search / beam-sample (`BeamSelector`).  Returns the best `num_return_sequences` finished hypotheses per batch
    row ([B * n, T], best first), new tokens only, padded.  The step chains through device buffers into the CUDA-graphed
    decode step; the host reads the `done` flag every `check_every` steps only.

    With num_beams=1, early_stopping=True and penalty_on_logits=True this is HF greedy search with logits processors."""
    Bt = inputs_embeds.shape[0]
    nb = num_beams
    n_ret = max(1, int(num_return_sequences or 1))
    if n_ret > nb:
        raise ValueError("num_return_sequences = %d has to be <= num_beams = %d" % (n_ret, nb))
    if Bt * nb > engine.cfg.llm_max_batch:
        raise ValueError("batch x num_beams = %d exceeds the engine's llm_max_batch = %d" % (Bt * nb, engine.cfg.llm_max_batch))
    logits = _prefill(engine, inputs_embeds, attention_mask, nb)
    sel = BeamSelector(engine, Bt, nb, max_new_tokens, eos_token_id, pad_token_id, inputs_embeds.device, min_length,
                       length_penalty, early_stopping, repetition_penalty, no_repeat_ngram_size or 0, prefix_allowed_tokens_fn,
                       penalty_on_logits, n_ret, do_sample, temperature, top_k, top_p, generator)
    return _decode_loop(engine, sel, logits, max_new_tokens, check_every)


@torch.no_grad()
def contrastive_search(engine, inputs_embeds, attention_mask, max_new_tokens, eos_token_id, pad_token_id, top_k,
                       penalty_alpha, min_length=0, repetition_penalty=1.0, no_repeat_ngram_size=0, check_every=16):
    """Contrastive search (Su et al. 2022) as transformers 4.31 — the version the reference pins, Emu2/requirements.txt:2 —
    runs it when `penalty_alpha > 0`, `top_k > 1`, one beam and no sampling (Emu2/emu/emu.py:166,222 forward the knob):

        candidates  = top_k tokens of softmax(processed logits)            (one look-ahead decode step for all of them)
        degeneration(v) = max_j cos(h_v, h_j) over the hidden states h_j of the context            (`_ranking_fast`)
        next        = argmax_v (1 - alpha) * p(v) - alpha * degeneration(v)

    `h` are the last hidden states (post final norm = HF hidden_states[-1]).  Engine mapping: the k candidates of every row
    are decoded as k cache rows (emu_llm_expand maps the row to k, one emu_llm_decode step returns their logits and hidden
    states), then the chosen candidate's row becomes the row again (emu_llm_expand with the selected indices) — the cache
    itself never moves, only the row table the decode attention reads through.  Left-pad positions of the prompt take no
    part in the similarity (they hold no token).  Parity: restated from the published algorithm; the installed transformers
    (5.5) no longer ships contrastive search, so this strategy is pinned only by the literal restatement in the CPU tests."""
    B = inputs_embeds.shape[0]
    k = int(top_k)
    dev = inputs_embeds.device
    if k < 2 or not penalty_alpha or penalty_alpha <= 0:
        raise ValueError("contrastive search needs top_k > 1 and penalty_alpha > 0")
    if B * k > engine.cfg.llm_max_batch:
        raise ValueError("batch x top_k = %d exceeds the engine's llm_max_batch = %d" % (B * k, engine.cfg.llm_max_batch))
    V, H = engine.cfg.llm_vocab, inputs_embeds.shape[-1]
    alpha = float(penalty_alpha)
    engine.llm_reset()
    hidden, logits = engine.llm_prefill(inputs_embeds, attention_mask, hf_positions=True, want_hidden=True, want_logits=True)
    N = hidden.shape[1]
    ctx = torch.zeros(B, N + max_new_tokens, H, dtype=torch.float32, device=dev)        # unit-norm context hidden states
    ctx[:, :N] = torch.nn.functional.normalize(hidden.float(), dim=-1)
    valid = torch.zeros(B, N + max_new_tokens, dtype=torch.bool, device=dev)
    valid[:, :N] = attention_mask.to(dev) != 0
    processed = repetition_penalty != 1.0 or bool(no_repeat_ngram_size)
    prev = torch.full((B, max_new_tokens), pad_token_id, dtype=torch.int32, device=dev)
    zero_run = torch.zeros(B, 1, dtype=torch.float32, device=dev)
    expand_idx = torch.arange(B * k, device=dev, dtype=torch.int32) // k
    row_base = torch.arange(B, device=dev) * k
    cand_logits = torch.empty(B * k, V, dtype=torch.float32, device=dev)
    cand_hidden = torch.empty(B * k, H, dtype=torch.bfloat16, device=dev)
    cand_tok = torch.empty(B * k, dtype=torch.int32, device=dev)
    finished = torch.zeros(B, dtype=torch.bool, device=dev)
    pad_t = torch.full((B,), pad_token_id, dtype=torch.int64, device=dev)
    n_done = 0
    for step in range(max_new_tokens):
        ban = eos_token_id if step < min_length else -1
        if processed or ban >= 0:
            engine.beam_topk(logits, zero_run, B, 1, 2, ban_id=ban, prev_tokens=prev if step > 0 else None, prev_len=step,
                             repetition_penalty=repetition_penalty, penalty_on_logits=True,
                             no_repeat_ngram=no_repeat_ngram_size or 0)
        top_p_, top_ids = torch.topk(torch.softmax(logits.float(), dim=-1), k)                # [B, k]
        # look-ahead: every candidate as its own cache row
        engine.llm_expand(expand_idx, B * k)
        cand_tok.copy_(top_ids.reshape(-1))
        engine.llm_decode(token_ids=cand_tok, logits=cand_logits, hidden=cand_hidden, B=B * k)
        h = torch.nn.functional.normalize(cand_hidden.float(), dim=-1).view(B, k, H)
        cos = torch.einsum("bkh,bsh->bks", h, ctx[:, :N + step])
        cos = cos.masked_fill(~valid[:, None, :N + step], float("-inf"))
        score = (1.0 - alpha) * top_p_ - alpha * cos.max(dim=-1)[0]
        sel = score.argmax(dim=-1)                                                           # [B]
        nxt = torch.where(finished, pad_t, top_ids.gather(1, sel[:, None])[:, 0])
        prev[:, step] = nxt.to(torch.int32)
        ctx[:, N + step] = h[torch.arange(B, device=dev), sel]
        valid[:, N + step] = True
        finished |= nxt == eos_token_id
        n_done = step + 1
        # the chosen candidate's row (its look-ahead step is the sequence's real step) becomes row b again
        engine.llm_expand((row_base + sel).to(torch.int32), B)
        logits = cand_logits.view(B, k, V)[torch.arange(B, device=dev), sel].contiguous()
        if n_done == max_new_tokens:
            break
        if check_every and n_done % check_every == 0 and bool(finished.all()):
            break
    return _finish_rows(prev[:, :n_done].to(torch.int64), eos_token_id, pad_token_id)


@torch.no_grad()
def speculative_greedy_search(engine, inputs_embeds, attention_mask, max_new_tokens, eos_token_id, pad_token_id, k,
                              max_matching_ngram_size=2, prompt_ids=None, min_length=0):
    """Greedy search at batch 1 with prompt-lookup speculative decoding (HF assisted generation with
    `prompt_lookup_num_tokens=k`): the same ids as greedy_search, in fewer passes over the weights.

    The history is prompt_ids (the prompt's token ids, picture positions holding their placeholder ids; may be None) followed
    by the generated tokens, on the device.  After the prefill every step runs emu_llm_verify over the last committed token
    and up to k drafted tokens (n = d + 1 rows, one weight pass), emu_spec_accept (the drafts equal to the arg-max before them,
    then the arg-max after the last of them), emu_spec_draft for the next step, ONE read-back of {tokens appended, finished,
    next draft length}, and emu_llm_commit of the appended positions.  A draft only changes how many tokens a pass yields:
    every kept token is the arg-max of the verify row that produced it."""
    dev = inputs_embeds.device
    N = inputs_embeds.shape[1]
    i32 = dict(dtype=torch.int32, device=dev)
    P = 0 if prompt_ids is None else int(prompt_ids.shape[-1])
    cap = P + max_new_tokens
    hist = torch.zeros(cap, **i32)
    if P:
        hist[:P].copy_(prompt_ids.reshape(-1))
    logits = _prefill(engine, inputs_embeds, attention_mask, 1)
    if min_length > 0:
        logits[:, eos_token_id] = float("-inf")
    hist[P:P + 1].copy_(logits.argmax(-1))
    hist_len = torch.full((1,), P + 1, **i32)
    # fixed addresses: the verify's CUDA graphs are keyed by their arguments
    tokens = torch.zeros(k + 1, **i32)      # the verify's rows: the last committed token, then the draft
    next_ids = torch.zeros(k + 1, **i32)
    stats = torch.zeros(3, **i32)           # tokens appended, finished, next draft length
    stats[1:2].copy_((hist[P:P + 1] == eos_token_id) | (max_new_tokens <= 1))
    engine.spec_draft(hist, hist_len, k, max_matching_ngram_size, cap, eos_token_id, tokens, stats[2:])
    _, done, d = stats.tolist()
    n_gen, max_seq = 1, engine.cfg.llm_max_seq
    while not done:
        # the cache holds the prompt and every generated token but the last; no row past max_new_tokens or llm_max_seq
        L = N + n_gen - 1
        n = 1 + max(0, min(d, max_new_tokens - n_gen - 1, max_seq - L - 1))
        engine.llm_verify(tokens, n, next_ids=next_ids, ban_id=eos_token_id, ban_rows=max(0, min(n, min_length - n_gen)))
        engine.spec_accept(hist, hist_len, tokens, next_ids, n, eos_token_id, cap, stats)
        engine.spec_draft(hist, hist_len, k, max_matching_ngram_size, cap, eos_token_id, tokens, stats[2:])
        m, done, d = stats.tolist()
        n_gen += m
        if not done:
            engine.llm_commit(m)
    return _finish_rows(hist[None, P:P + n_gen].to(torch.int64), eos_token_id, pad_token_id)


def _speculative_knobs(engine, batch, k, max_matching_ngram_size, do_sample, num_beams, penalty_alpha, top_k, rp, ngram,
                       prefix_allowed_tokens_fn):
    """the refusals of prompt-lookup decoding, as HF's assisted generation makes them where it has them: (k, n-gram size)"""
    if do_sample or num_beams != 1 or batch != 1:
        raise ValueError("prompt_lookup_num_tokens needs greedy search at batch 1 (no sampling, num_beams = 1), got "
                         "do_sample=%s, num_beams=%d, batch=%d" % (bool(do_sample), num_beams, batch))
    if penalty_alpha is not None and penalty_alpha > 0 and top_k is not None and top_k > 1:
        raise ValueError("prompt_lookup_num_tokens cannot be combined with contrastive search (penalty_alpha)")
    if rp != 1.0 or ngram or prefix_allowed_tokens_fn is not None:
        raise NotImplementedError("prompt_lookup_num_tokens with logits processors (repetition_penalty, "
                                  "no_repeat_ngram_size, prefix_allowed_tokens_fn)")
    k = int(k)
    limit = min(7, int(engine.cfg.llm_max_batch) - 1)
    if k < 1 or k > limit:
        raise ValueError("prompt_lookup_num_tokens = %d outside [1, %d]: a verify checks at most min(8, llm_max_batch = %d) "
                         "rows, the last token and k drafts" % (k, limit, engine.cfg.llm_max_batch))
    g = 2 if max_matching_ngram_size is None else int(max_matching_ngram_size)
    if g < 1:
        raise ValueError("max_matching_ngram_size has to be >= 1, got %d" % g)
    return k, g


def generate(engine, inputs_embeds, attention_mask, max_new_tokens, eos_token_id, pad_token_id, do_sample=False, num_beams=1,
             min_length=0, length_penalty=1.0, repetition_penalty=1.0, penalty_alpha=None, top_k=None, top_p=None,
             temperature=None, no_repeat_ngram_size=0, prefix_allowed_tokens_fn=None, num_return_sequences=1,
             early_stopping=False, generator=None, check_every=None, prompt_lookup_num_tokens=None, max_matching_ngram_size=2,
             prompt_ids=None):
    """`lm.generate(inputs_embeds=...)` as the reference calls it (Emu2/emu/emu.py:213-229, Emu1/models/modeling_emu.py:162-179):
    picks the decoding strategy from the knobs the way GenerationMixin (transformers 4.31, the pinned version) does

        num_beams == 1, no sampling, penalty_alpha > 0 and top_k > 1   -> contrastive search
        num_beams == 1, no sampling, prompt_lookup_num_tokens = k      -> speculative greedy search (batch 1; prompt_ids,
                                                                          the prompt's token ids, are drafted from too)
        num_beams == 1, no sampling                                    -> greedy search
        num_beams == 1, do_sample                                      -> multinomial sampling
        num_beams  > 1                                                 -> beam search / beam-sample (do_sample)

    and returns the new token ids [B * num_return_sequences, T]."""
    num_beams, rp, ngram, n_ret = decoding_knobs(num_beams, repetition_penalty, no_repeat_ngram_size, num_return_sequences)
    ce = {} if check_every is None else {"check_every": check_every}
    if prompt_lookup_num_tokens is not None:
        k, g = _speculative_knobs(engine, inputs_embeds.shape[0], prompt_lookup_num_tokens, max_matching_ngram_size, do_sample,
                                  num_beams, penalty_alpha, top_k, rp, ngram, prefix_allowed_tokens_fn)
        if n_ret != 1:
            raise ValueError("num_return_sequences has to be 1 when doing greedy / contrastive search, got %d" % n_ret)
        return speculative_greedy_search(engine, inputs_embeds, attention_mask, max_new_tokens, eos_token_id, pad_token_id, k,
                                         max_matching_ngram_size=g, prompt_ids=prompt_ids, min_length=min_length)
    if num_beams == 1 and not do_sample:
        if n_ret != 1:
            raise ValueError("num_return_sequences has to be 1 when doing greedy / contrastive search, got %d" % n_ret)
        if penalty_alpha is not None and penalty_alpha > 0 and top_k is not None and top_k > 1:
            if prefix_allowed_tokens_fn is not None:
                raise NotImplementedError("prefix_allowed_tokens_fn under contrastive search")
            return contrastive_search(engine, inputs_embeds, attention_mask, max_new_tokens, eos_token_id, pad_token_id,
                                      top_k=top_k, penalty_alpha=penalty_alpha, min_length=min_length, repetition_penalty=rp,
                                      no_repeat_ngram_size=ngram, **ce)
        return greedy_search(engine, inputs_embeds, attention_mask, max_new_tokens, eos_token_id, pad_token_id,
                             min_length=min_length, repetition_penalty=rp, no_repeat_ngram_size=ngram,
                             prefix_allowed_tokens_fn=prefix_allowed_tokens_fn, **ce)
    if num_beams == 1:
        return sample_search(engine, inputs_embeds, attention_mask, max_new_tokens, eos_token_id, pad_token_id,
                             min_length=min_length, temperature=temperature, top_k=top_k, top_p=top_p, generator=generator,
                             repetition_penalty=rp, no_repeat_ngram_size=ngram,
                             prefix_allowed_tokens_fn=prefix_allowed_tokens_fn, num_return_sequences=n_ret)
    return beam_search(engine, inputs_embeds, attention_mask, num_beams, max_new_tokens, eos_token_id, pad_token_id,
                       min_length=min_length, length_penalty=length_penalty, early_stopping=early_stopping,
                       repetition_penalty=rp, no_repeat_ngram_size=ngram, prefix_allowed_tokens_fn=prefix_allowed_tokens_fn,
                       num_return_sequences=n_ret, do_sample=bool(do_sample), temperature=temperature, top_k=top_k,
                       top_p=top_p, generator=generator, **ce)
