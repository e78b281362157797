"""Continuous batching for chat: requests join and leave the decode batch between steps (iteration-level scheduling).

`SlotScheduler` drives the engine's slot mode (include/emu_b200_slots.h): every KV-cache row is a slot holding one sequence of
its own length.  One `step()` is one iteration:

  1. admit: waiting requests take free slots, lowest first (a beam request takes `num_beams` contiguous slots); their
     pictures go through the ViT, their prompts are embedded and spliced, and ONE emu_llm_join prefills all of them
     (left-padded to the longest) while the live slots keep their cache.  A beam request joins into its first slot and is
     forked to the others.  The join stalls the live requests for one ViT + prefill;
  2. select: every live request picks its next tokens from ITS OWN rows of the logits with ITS OWN knobs, through the
     selector generation.generate runs for those knobs (generation.selector, one prompt: num_beams rows), so a request's
     tokens are the ones it would get alone;
  3. retire: finished requests leave (their slots are freed) and are answered;
  4. decode: ONE emu_llm_decode over B = highest occupied slot + 1 advances every live request by one token (free slots
     below B are computed and ignored).

Prefix caching (`SlotScheduler(prefix_cache=True)`, opt-in): a finished request leaves with emu_llm_leave_keep, so its slot keeps
the KV of its prompt and answer (a beam search: its prompt).  A newcomer whose key sequence (token ids; a picture slot keyed by
the picture's digest and its index within the picture) starts like a kept or live slot's resumes from it: in place when that
kept slot can be its first slot, else through emu_llm_copy_prefix.  Only the suffix is embedded (pictures inside the prefix do
not go through the ViT) and ONE emu_llm_extend prefills the suffixes of all resuming newcomers.  Kept slots count as free: a
newcomer that needs room overwrites the least recently used one, so retention never delays admission.

Chunked prefill (`SlotScheduler(prefill_chunk=C)`, opt-in): a newcomer takes its slots, has its pictures encoded and its prompt
embedded at admission as above, but is not joined: it is queued as prefilling.  While any request is prefilling, the decode of
step 4 becomes ONE emu_llm_step (include/emu_b200_chunked.h): the live slots' next tokens and at most C prompt tokens of the
prefilling requests (first come, first served), packed without padding into one weight pass.  A request's last chunk makes
its first slot live (a beam request then forks, as after a join); its earlier chunks leave that slot kept at its length, owned
by the request, so it is never a prefix source nor evicted.  No live request waits longer than one such step for a newcomer.
A prompt with left padding (zeros in its attention_mask) still joins whole.

Each step reads ONE small tensor back to the host: the finish flag of every live request (EOS of a greedy / sampled request,
`done` of a beam search), which is what lets a request leave as soon as it is finished.

Strategies: greedy, sampling, beam search and beam-sample with min_len, repetition_penalty, no_repeat_ngram_size,
temperature / top_k / top_p and length_penalty — what the demo's /v1/mmc form can send.  Requests with different knobs share
a decode step.  A request's output is what generation.generate returns for it alone (beam search: its best hypothesis;
greedy / sampling: its tokens up to EOS).  Contrastive search, prefix_allowed_tokens_fn and num_return_sequences > 1 are
refused.  Sampled requests reproduce their solo draws when they carry a `generator`; without one they draw from torch's
global generator, shared with whatever else runs in the process.
"""
import collections
import threading

import torch

from . import generation


class SlotRequest:
    """One generate call's worth of work: a one-row prompt (token ids, optional pictures) and its decoding knobs, with
    EmuModel.generate_from_ids' names and defaults.  `result` (token ids [1, T] or the decoded text) or `error` is set
    when it is finished, then `done` is set and `on_done(request)` is called."""

    def __init__(self, input_ids, attention_mask=None, image=None, video=None, image_token_id=32003, video_token_id=32004,
                 num_beams=5, max_new_tokens=10, min_len=1, do_sample=False, temperature=None, top_k=None, top_p=None,
                 length_penalty=-1, repetition_penalty=1.0, no_repeat_ngram_size=0, early_stopping=False, penalty_alpha=None,
                 num_return_sequences=1, prefix_allowed_tokens_fn=None, generator=None, eos_token_id=None,
                 pad_token_id=None, finish=None, on_done=None, tag=None, image_keys=None, signature=None):
        ids = torch.as_tensor(input_ids)
        self.input_ids = ids.view(1, -1) if ids.dim() == 1 else ids
        if self.input_ids.shape[0] != 1:
            raise ValueError("a request holds one prompt, got input_ids of shape %s" % (tuple(self.input_ids.shape),))
        self.attention_mask = (torch.ones_like(self.input_ids) if attention_mask is None
                               else torch.as_tensor(attention_mask).view(1, -1))
        self.image, self.video = image, video
        self.image_token_id, self.video_token_id = image_token_id, video_token_id
        self.num_beams, rp, ngram, n_ret = generation.decoding_knobs(num_beams, repetition_penalty, no_repeat_ngram_size,
                                                                     num_return_sequences)
        self.max_new_tokens = int(max_new_tokens)
        self.knobs = dict(do_sample=bool(do_sample), min_length=int(min_len or 0), length_penalty=length_penalty,
                          early_stopping=early_stopping, repetition_penalty=rp, no_repeat_ngram_size=ngram,
                          temperature=temperature, top_k=top_k, top_p=top_p, generator=generator)
        self.eos, self.pad = eos_token_id, pad_token_id
        self.finish, self.on_done, self.tag = finish, on_done, tag
        # prefix caching: one digest per picture of `image` (None: a picture never matches), and the front end's view of the
        # prompt (its elements; pictures as digests) that the serving shell routes by
        self.image_keys = None if image_keys is None else list(image_keys)
        self.signature = signature
        self.done = threading.Event()
        self.result = self.error = None
        if self.max_new_tokens < 1:
            raise ValueError("max_new_tokens has to be >= 1")
        if self.num_beams == 1 and not do_sample and penalty_alpha is not None and penalty_alpha > 0 \
                and top_k is not None and top_k > 1:
            raise ValueError("continuous batching does not run contrastive search (penalty_alpha with top_k > 1)")
        if prefix_allowed_tokens_fn is not None:
            raise ValueError("continuous batching does not take prefix_allowed_tokens_fn")
        if n_ret != 1:
            raise ValueError("continuous batching returns one sequence per request (num_return_sequences = 1)")
        # set at admission
        self.slots = []
        self.engine_slots = []      # the slots the engine holds for this request (joined / forked): they must leave
        self.step = 0
        self.logits = None
        self.selector = None        # generation's token selector for this request
        self.keys = None            # prefix caching: the prompt's key sequence
        self.left_pad = 0           # ... its left padding in its slot's row
        self.resume = None          # ... (prefix keys, prefix cache positions, source slot, in place) when it resumes


class _RequestQueue:
    """The request life cycle both slot schedulers share.  `submit` (from any thread) queues a request; the subclass's
    `step` (from one thread) admits, advances and retires.  A request is answered once: with `_result(r)` when it retires,
    or with an error; either way it leaves its slots first (`_release`).  `_live()` lists the admitted requests."""

    def __init__(self):
        self.waiting = collections.deque()
        self._lock = threading.Lock()

    def submit(self, request):
        with self._lock:
            self.waiting.append(request)
        return request

    def busy(self):
        return bool(self._live()) or bool(self.waiting)

    def load(self):
        """requests admitted or waiting"""
        return len(self._live()) + len(self.waiting)

    def abort(self, ex):
        """fail every live and waiting request with `ex` (the scheduler itself stays usable)"""
        for r in self._live():
            self._fail(r, ex)
        with self._lock:
            waiting, self.waiting = list(self.waiting), collections.deque()
        for r in waiting:
            self._fail(r, ex)

    def run_until_idle(self):
        out = []
        while self.busy():
            out += self.step()
        return out

    def _retire(self, r):
        try:
            r.result = self._result(r)
        except Exception as ex:
            r.error = ex
        self._answer(r)

    def _fail(self, r, ex):
        r.error = ex
        self._answer(r)

    def _answer(self, r):
        self._release(r)
        r.done.set()
        if r.on_done is not None:
            r.on_done(r)


class SlotScheduler(_RequestQueue):
    """Continuous batching over `emu_model` (an EmuModel: its engine, tokenizer ids, ViT and projection) with `n_slots`
    KV-cache slots (at most the engine's llm_max_batch).  Owns the engine while it lives: nothing else may use the engine's
    LLM between steps.  Single-threaded: `submit` may be called from any thread, `step` from one."""

    def __init__(self, emu_model, n_slots=None, prefix_cache=False, prefill_chunk=None):
        super().__init__()
        self.prefix_cache = bool(prefix_cache)
        self.prefill_chunk = None if prefill_chunk is None else int(prefill_chunk)
        if self.prefill_chunk is not None and self.prefill_chunk < 1:
            raise ValueError("prefill_chunk must be >= 1, got %d" % self.prefill_chunk)
        self.prefilling = []                                # chunked prefill: admitted requests not yet live, in admission order
        self.kept = {}                                      # kept slot -> _Kept (prefix caching)
        self._signatures = ()                               # front-end signatures of the kept and live slots (routing)
        self._clock = 0
        # prefix-caching observability (the tests read them): admissions that reused a prefix, the prompt tokens they did not
        # prefill, the prompt tokens prefilled, the pictures encoded
        self.prefix_hits = self.prefix_tokens_reused = self.prefill_tokens = self.vit_pictures = 0
        self.model = emu_model
        self.engine = emu_model.engine
        cfg = self.engine.cfg
        self.n_slots = int(n_slots or cfg.llm_max_batch)
        if not 1 <= self.n_slots <= cfg.llm_max_batch:
            raise ValueError("n_slots = %d must be in [1, llm_max_batch = %d]" % (self.n_slots, cfg.llm_max_batch))
        self.max_seq = int(getattr(cfg, "llm_max_seq", 0) or 0)
        self.V = cfg.llm_vocab
        self.device = torch.device(emu_model.device())
        tok = getattr(getattr(emu_model, "decoder", None), "tokenizer", None)
        self.eos = getattr(tok, "eos_token_id", None)
        self.pad = getattr(tok, "pad_token_id", None)
        self.live = []                                      # admitted requests, in admission order
        self.owner = [None] * self.n_slots                  # slot -> request
        self.steps = 0
        self.batch_sizes = collections.deque(maxlen=1024)   # B of the recent decode steps (observability; the tests read it)
        self.prefill_chunks = 0                             # chunked prefill: mixed steps run, and their recent sizes
        self.mixed_sizes = collections.deque(maxlen=1024)   # ... (decode rows B, prompt tokens prefilled)
        i32 = dict(dtype=torch.int32, device=self.device)
        self.tok_buf = torch.zeros(self.n_slots, **i32)      # fixed buffers: the decode graphs are keyed by their pointers
        self.ident = torch.arange(self.n_slots, **i32)
        self.src_buf = self.ident.clone()                    # identity except the rows of live beam groups
        self.logits_buf = torch.zeros(self.n_slots, self.V, dtype=torch.float32, device=self.device)
        with _on_device(self.device):
            self.engine.slots_begin(self.n_slots)

    # ---- producer side ----
    def submit(self, request: SlotRequest):
        if request.eos is None:
            request.eos = self.eos
        if request.pad is None:
            request.pad = self.pad
        if request.num_beams > self.n_slots:
            raise ValueError("num_beams = %d exceeds the scheduler's %d slots" % (request.num_beams, self.n_slots))
        n_prompt = request.input_ids.shape[1]
        if self.max_seq and n_prompt > self.max_seq:
            raise ValueError("prompt of %d tokens exceeds llm_max_seq = %d" % (n_prompt, self.max_seq))
        return super().submit(request)

    def _live(self):
        return list(self.live) + list(self.prefilling)

    # ---- one iteration ----
    @torch.no_grad()
    def step(self):
        """admit -> select -> retire -> decode (module docstring); returns the requests finished in this step"""
        with _on_device(self.device):
            return self._step()

    def _step(self):
        self._admit()
        finished = self._select()
        for r in finished:
            self._retire(r)
        if self.prefilling:
            self._mixed()
        elif self.live:
            self._decode()
        self.steps += 1
        if self.prefix_cache:                               # one assignment: readers on other threads see old or new
            self._signatures = tuple(e.signature for e in self.kept.values()) + tuple(r.signature for r in self.live)
        return finished

    # ---- admission ----
    def _free_run(self, n):
        """lowest first slot of n contiguous free slots, or None"""
        run = 0
        for s in range(self.n_slots):
            run = run + 1 if self.owner[s] is None else 0
            if run == n:
                return s - n + 1
        return None

    def _admit(self):
        batch = []
        with self._lock:
            while self.waiting:
                r = self.waiting[0]
                first = self._place(r) if self.prefix_cache else self._free_run(r.num_beams)
                if first is None:
                    break                                   # first come, first served: the head waits for room
                self.waiting.popleft()
                r.slots = list(range(first, first + r.num_beams))
                for s in r.slots:
                    self.owner[s] = r
                    self.kept.pop(s, None)                  # whatever a kept slot held is overwritten or resumed now
                batch.append(r)
        if not batch:
            return
        ready = []
        for r in batch:                                     # a prompt that cannot be embedded fails on its own
            try:
                ready.append((r, self._embed(r)))
            except Exception as ex:
                self._fail(r, ex)
        if self.prefix_cache:
            ready = self._resume(ready)
        if self.prefill_chunk is not None:
            ready = self._queue_prefill(ready)
        for group in self._join_groups(ready):
            try:
                self._join(group)
            except Exception as ex:                         # nothing of this group was joined
                if len(group) == 1:
                    self._fail(group[0][0], ex)
                    continue
                for item in group:                          # a shared join failed: join one by one, only the culprit fails
                    try:
                        self._join([item])
                    except Exception as ex1:
                        self._fail(item[0], ex1)

    def _cap(self, r, n):
        """r's max_new_tokens in a slot that holds n prompt positions: the last token is never fed back, so the slot ends
        at n + max_new_tokens - 1 positions, which must fit llm_max_seq"""
        return min(r.max_new_tokens, self.max_seq - n + 1) if self.max_seq else r.max_new_tokens

    def _join_groups(self, ready):
        """split the admitted prompts into joins (usually one) such that left-padding a prompt to its join's length never
        leaves it less room than it has alone"""
        groups = []
        for item in ready:
            for g in groups:
                N = max(e.shape[1] for _, (e, _) in g + [item])
                if all(self._cap(r, N) == self._cap(r, e.shape[1]) for r, (e, _) in g + [item]):
                    g.append(item)
                    break
            else:
                groups.append([item])
        return groups

    def _embed(self, r):
        m = self.model
        ids, image = r.input_ids, r.image
        if r.resume is not None:                            # the suffix only: pictures inside the prefix skip the ViT
            P = r.resume[0]
            k0 = int((ids[0, :P] == r.image_token_id).sum()) // self._per_picture(r) if image is not None else 0
            ids, image = ids[:, P:], (image[k0:] if image is not None and k0 < image.shape[0] else None)
        self.vit_pictures += (0 if image is None else image.shape[0]) + (0 if r.video is None else r.video.shape[0])
        self.prefill_tokens += int(r.attention_mask[0].sum()) - (r.resume[0] if r.resume is not None else 0)
        ids = ids.to(self.device)
        mask = torch.ones_like(ids) if r.resume is not None else r.attention_mask.to(self.device)
        return m.embed_prompt(ids, image, r.video, r.image_token_id, r.video_token_id), mask

    # ---- prefix caching ----
    @staticmethod
    def _per_picture(r):
        n_img = int((r.input_ids == r.image_token_id).sum())
        return max(1, n_img // r.image.shape[0]) if r.image is not None and r.image.shape[0] else max(1, n_img)

    def _key_sequence(self, r):
        """token ids, with every picture slot keyed by (picture digest, index within the picture); a picture without a digest
        (and every video frame) gets a key equal to nothing else"""
        ids = r.input_ids[0].tolist()
        per = self._per_picture(r)
        keys, k = [], 0
        for t in ids:
            if t == r.image_token_id:
                pic, j = divmod(k, per)
                ok = r.image_keys is not None and r.image is not None and pic < len(r.image_keys)
                keys.append((r.image_keys[pic], j) if ok else object())
                k += 1
            elif t == r.video_token_id:
                keys.append(object())
            else:
                keys.append(t)
        return keys

    def _sources(self):
        """(slot, keys, pad, kept) of every kept slot and every live request's first slot (its prompt is its own row)"""
        out = [(s, e.keys, e.left_pad, True) for s, e in self.kept.items()]
        out += [(r.slots[0], r.keys, r.left_pad, False) for r in self.live if r.keys is not None]
        return out

    def _match(self, r):
        """(prefix keys, source slot, its pad, kept) of the longest usable prefix of r's keys, or (0, None, 0, False)"""
        keys, best = r.keys, (0, None, 0, False)
        n = len(keys)
        for s, ks, pad, kept in self._sources():
            P = 0
            for a, b in zip(keys, ks):
                if a != b:
                    break
                P += 1
            P = min(P, n - 1)                               # the last prompt token is recomputed for its logits
            if P < n and isinstance(keys[P], tuple):        # never split a picture: cut back to its first slot
                P -= keys[P][1]
            if P <= best[0] or (self.max_seq and pad + n > self.max_seq) or self._cap(r, pad + n) != self._cap(r, n):
                continue
            best = (P, s, pad, kept)
        return best

    def _place(self, r):
        """the first slot for r (prefix caching on), or None; sets r.keys and r.resume"""
        nb = r.num_beams
        r.keys = self._key_sequence(r) if bool((r.attention_mask != 0).all()) else None
        r.resume = None
        P, src, pad, kept = self._match(r) if r.keys is not None else (0, None, 0, False)
        if P > 0 and kept and all(t < self.n_slots and self.owner[t] is None for t in range(src, src + nb)):
            first, in_place = src, True
        else:
            first, in_place = self._pick_run(nb), False      # the copy runs before anything overwrites the source
        if first is None:
            return None
        if P > 0:
            r.resume, r.left_pad = (P, pad + P, src, in_place), pad
            if src in self.kept:
                self._clock += 1
                self.kept[src].used = self._clock
        return first

    def _pick_run(self, n):
        """first slot of n contiguous unowned slots, preferring runs that hold no kept prefix, then the least recently used"""
        best = None
        for first in range(self.n_slots - n + 1):
            run = range(first, first + n)
            if any(self.owner[t] is not None for t in run):
                continue
            cost = max([self.kept[t].used for t in run if t in self.kept], default=-1)
            if best is None or cost < best[0]:
                best = (cost, first)
        return None if best is None else best[1]

    def _resume(self, ready):
        """copy the prefixes that cannot resume in place, then ONE emu_llm_extend for every resuming newcomer; returns the
        items that join from nothing"""
        joins, ext = [], []
        for item in ready:
            r = item[0]
            if r.resume is None:
                joins.append(item)
                continue
            P, Pc, src, in_place = r.resume
            try:
                if not in_place:
                    self.engine.copy_prefix(src, r.slots[0], Pc)
            except Exception as ex:
                self._fail(r, ex)
                continue
            ext.append(item)
        if ext and self.prefill_chunk is not None:          # chunked prefill: the first chunk starts at the resumed prefix
            for r, (e, _) in ext:
                self.prefix_hits += 1
                self.prefix_tokens_reused += r.resume[0]
                self._prefilling(r, e, r.resume[1])
        elif ext:
            try:
                self._extend(ext)
            except Exception as ex:
                if len(ext) == 1:
                    self._extend_failed(ext[0][0], ex)
                else:
                    for item in ext:                        # a shared extend failed: one by one, only the culprit fails
                        try:
                            self._extend([item])
                        except Exception as ex1:
                            self._extend_failed(item[0], ex1)
        return joins

    def _extend_failed(self, r, ex):
        for s in r.slots:
            self.kept.pop(s, None)
        self._fail(r, ex)

    def _extend(self, items):
        N = max(e.shape[1] for _, (e, _) in items)
        embeds = torch.zeros(len(items), N, items[0][1][0].shape[-1], dtype=items[0][1][0].dtype, device=self.device)
        for i, (_, (e, _)) in enumerate(items):            # right padding: every row continues its own slot
            embeds[i, :e.shape[1]] = e[0]
        logits = self.engine.extend([r.slots[0] for r, _ in items], [r.resume[1] for r, _ in items],
                                    [e.shape[1] for _, (e, _) in items], embeds)
        for r, _ in items:
            self.prefix_hits += 1
            self.prefix_tokens_reused += r.resume[0]
        self._start(items, logits, [r.left_pad + len(r.keys) for r, _ in items])

    # ---- chunked prefill ----
    def _queue_prefill(self, ready):
        """queue the unpadded prompts for chunked prefill; returns the left-padded ones, which join whole"""
        joins = []
        for item in ready:
            r, (e, m) = item
            if bool((m != 0).all()):
                r.left_pad = 0
                self._prefilling(r, e, 0)
            else:
                joins.append(item)
        return joins

    def _prefilling(self, r, embeds, start):
        """r prefills embeds [1, T, hidden] into its first slot from cache position `start` on, a chunk per step"""
        r.pf_embeds, r.pf_start, r.pf_done = embeds[0], int(start), 0
        self.prefilling.append(r)

    def _mixed(self):
        """ONE emu_llm_step: the live slots' decode rows and up to prefill_chunk prompt tokens of the prefilling requests"""
        segs, budget = [], self.prefill_chunk
        for r in self.prefilling:
            if budget == 0:
                break
            T = r.pf_embeds.shape[0]
            k = min(budget, T - r.pf_done)
            segs.append((r, r.pf_start + r.pf_done, k, r.pf_done + k == T))
            budget -= k
        B = max(s for r in self.live for s in r.slots) + 1 if self.live else 0
        beams = any(r.num_beams > 1 for r in self.live)
        embeds = torch.cat([r.pf_embeds[r.pf_done:r.pf_done + k] for r, _, k, _ in segs])
        try:
            last = self.engine.step([r.slots[0] for r, _, _, _ in segs], [p for _, p, _, _ in segs], [k for _, _, k, _ in segs],
                                    [f for _, _, _, f in segs], embeds, token_ids=self.tok_buf if B else None, B=B,
                                    beam_src=self.src_buf if beams else None, logits=self.logits_buf if B else None)
        except Exception as ex:       # the requests in the step fail, the scheduler stays usable
            for r in list(self.live) + [r for r, _, _, _ in segs]:
                self._fail(r, ex)
            return
        self.prefill_chunks += 1
        self.mixed_sizes.append((B, sum(k for _, _, k, _ in segs)))
        if B:
            self.batch_sizes.append(B)
        for r in self.live:
            r.logits = self.logits_buf[r.slots[0]:r.slots[0] + r.num_beams]
        started, rows, lengths = [], [], []
        for i, (r, p, k, final) in enumerate(segs):
            r.pf_done += k
            if final:
                self.prefilling.remove(r)
                r.pf_embeds = None
                started.append((r, None))
                rows.append(i)
                lengths.append(p + k)
        if started:
            self._start(started, last[rows], lengths)

    def _keep(self, r):
        """what r's first slot keeps when it retires: the prompt and every answer token whose KV was written (beam search:
        the prompt, its generated positions are scattered over the group's rows), or None"""
        if r.keys is None:
            return None
        keys = list(r.keys)
        if r.num_beams == 1 and r.step > 1:
            keys += r.selector.prev[0, :r.step - 1].tolist()
        if self.max_seq:
            keys = keys[:self.max_seq - 1 - r.left_pad]
        if not keys:
            return None
        self._clock += 1
        return _Kept(keys, r.left_pad, r.left_pad + len(keys), self._clock)

    def cached_prefix(self, signature):
        """how many leading elements of a prompt's front-end signature a kept or live slot of this scheduler holds (the
        serving shell sends a request to the worker where this is longest).  Reads the snapshot `step()` publishes, so it
        may be called from any thread."""
        best = 0
        for sig in self._signatures:
            n = 0
            for a, b in zip(signature or (), sig or ()):
                if a != b:
                    break
                n += 1
            best = max(best, n)
        return best

    def _join(self, items):
        """one emu_llm_join for `items`; raises only if nothing was joined.  After the join every request is on its own: a
        request that fails later leaves the slots the engine holds for it."""
        N = max(e.shape[1] for _, (e, _) in items)
        embeds = torch.zeros(len(items), N, items[0][1][0].shape[-1], dtype=items[0][1][0].dtype, device=self.device)
        mask = torch.zeros(len(items), N, dtype=torch.int32, device=self.device)
        for i, (_, (e, m)) in enumerate(items):            # left padding, as the tokenizer pads a batch
            embeds[i, N - e.shape[1]:] = e[0]
            mask[i, N - e.shape[1]:] = m[0].to(torch.int32)
        logits = self.engine.join([r.slots[0] for r, _ in items], embeds, mask)
        for r, (e, _) in items:
            r.left_pad = N - e.shape[1]
        self._start(items, logits, [N] * len(items))

    def _start(self, items, logits, lengths):
        """the joined / resumed first slots (lengths: their cache lengths) become live requests: beam groups fork"""
        for r, _ in items:
            r.engine_slots = [r.slots[0]]
        for i, (r, _) in enumerate(items):
            try:
                r.max_new_tokens = self._cap(r, lengths[i])  # the room it has alone (_join_groups, _match)
                if r.num_beams > 1:
                    self.engine.fork(r.slots[0], r.slots[1:])
                    r.engine_slots = list(r.slots)
                r.logits = logits[i:i + 1].repeat(r.num_beams, 1).contiguous() if r.num_beams > 1 else logits[i:i + 1]
                r.selector = generation.selector(self.engine, 1, r.max_new_tokens, r.eos, r.pad, self.device,
                                                 r.num_beams, **r.knobs)
            except Exception as ex:
                self._fail(r, ex)
                continue
            self.live.append(r)

    # ---- selection ----
    def _select(self):
        flags, order = [], []
        for r in list(self.live):
            try:
                flags.append(self._select_one(r))
                order.append(r)
            except Exception as ex:
                self._fail(r, ex)
        if not order:
            return []
        hit = torch.stack([f.reshape(()).to(torch.int32) for f in flags]).tolist()   # the one read-back of the step
        done = []
        for r, h in zip(order, hit):
            if h or r.step >= r.max_new_tokens:
                done.append(r)
        return done

    def _select_one(self, r):
        """r's next tokens from r.logits ([num_beams, V]); writes them (and the beam re-parenting) into the decode inputs
        of r's slots and returns a device flag: r is finished"""
        first, nb = r.slots[0], r.num_beams
        self.tok_buf[first:first + nb] = r.selector.select(r.logits, r.step)
        if nb > 1:
            self.src_buf[first:first + nb] = r.selector.beam_src + first
        r.step += 1
        return r.selector.done()

    # ---- retirement ----
    def _result(self, r):
        ids = r.selector.output()
        return r.finish(ids) if r.finish is not None else ids

    def _release(self, r):
        if r in self.live:
            self.live.remove(r)
        if r in self.prefilling:                            # a kept slot the engine holds for it is simply overwritten later
            self.prefilling.remove(r)
            r.pf_embeds = None
        for s in r.slots:
            if self.owner[s] is r:
                self.owner[s] = None
        if r.num_beams > 1 and r.slots:                       # its rows of the re-parenting input go back to identity
            self.src_buf[r.slots[0]:r.slots[-1] + 1] = self.ident[r.slots[0]:r.slots[-1] + 1]
        held, r.engine_slots = r.engine_slots, []
        if held:
            keep = self._keep(r) if self.prefix_cache and r.error is None and r.selector is not None else None
            try:
                if keep is None:
                    self.engine.leave(held)
                else:
                    self.engine.leave_keep(held, [keep.length] + [0] * (len(held) - 1))
                    keep.signature = r.signature
                    self.kept[held[0]] = keep
            except Exception:
                try:
                    self.engine.leave(held)
                except Exception:
                    pass

    # ---- decode ----
    def _decode(self):
        B = max(s for r in self.live for s in r.slots) + 1
        beams = any(r.num_beams > 1 for r in self.live)
        try:
            self.engine.llm_decode(token_ids=self.tok_buf, beam_src=self.src_buf if beams else None, logits=self.logits_buf, B=B)
        except Exception as ex:       # an engine-level failure: every live request fails, the scheduler stays usable
            for r in list(self.live):
                self._fail(r, ex)
            return
        self.batch_sizes.append(B)
        for r in self.live:
            r.logits = self.logits_buf[r.slots[0]:r.slots[0] + r.num_beams]


class _Kept:
    """a kept slot of the prefix cache: its key sequence, left padding, kept length (cache positions) and last use"""

    def __init__(self, keys, pad, length, used):
        self.keys, self.left_pad, self.length, self.used = keys, pad, length, used
        self.signature = None


def _on_device(device):
    """the engine enqueues on the current stream of the current device: make that the scheduler's device"""
    import contextlib
    return torch.cuda.device(device) if device.type == "cuda" else contextlib.nullcontext()


def chat_request(chat, inputs, is_grounding=False, skip_special_tokens=True, prefix_keys=False, **knobs):
    """one EmuChatGeneration call (`chat(inputs, **knobs)`) as a SlotRequest whose result is the decoded answer: the same
    prompt assembly, tokenisation and picture transform as `forward`, and the same `skip_special_tokens` decoding"""
    model = chat.emu_model
    text, image, video, iph, vph = chat.prepare(inputs, is_grounding)
    input_ids, mask, IMAGE, VIDEO = model.tokenize_prompt(text, iph, vph)
    tok = model.decoder.tokenizer
    knobs = dict(knobs)
    knobs.pop("synced_gpus", None)
    keys = sig = None
    if prefix_keys:                                         # only a prefix-caching scheduler reads them
        pics = _pictures(inputs)
        keys = [picture_key(p) for p in pics] if image is not None and len(pics) == image.shape[0] else None
        sig = prompt_signature(inputs)
    return SlotRequest(input_ids, mask, image=image, video=video, image_token_id=IMAGE, video_token_id=VIDEO,
                       finish=lambda ids: tok.batch_decode(ids, skip_special_tokens=skip_special_tokens)[0],
                       image_keys=keys, signature=sig, **knobs)


def picture_key(picture):
    """the prefix-cache key of a picture: a blake2b digest of its RGB pixels and their shape, taken before any transform"""
    key = getattr(picture, "_emu_prefix_key", None)        # computed once per picture object (routing, then the request)
    if key is not None:
        return key
    import hashlib
    import numpy as np
    a = np.ascontiguousarray(np.asarray(picture.convert("RGB"), dtype=np.uint8))
    h = hashlib.blake2b(digest_size=32)
    h.update(repr(a.shape).encode())
    h.update(a.tobytes())
    key = h.hexdigest()
    try:
        picture._emu_prefix_key = key
    except AttributeError:
        pass
    return key


def prompt_signature(inputs):
    """the front end's view of a prompt: its elements in order, strings as they are and pictures as their digests"""
    return [picture_key(x) if hasattr(x, "convert") else x for x in _flatten(inputs)]


def _flatten(inputs):
    for x in inputs:
        if isinstance(x, (list, tuple)):
            yield from _flatten(x)
        else:
            yield x


def _pictures(inputs):
    return [x for x in _flatten(inputs) if hasattr(x, "convert")]


# ---- continuous batching for image generation ----
class ImageRequest:
    """One EmuVisualGeneration.forward call's worth of work: `inputs` (the interleaved prompt) or precomputed
    `prompt_embeds` ([2, L, Cc] = [cond; uncond] with guidance > 1, [1, L, Cc] without, as _prepare_and_encode_inputs returns
    them), with forward's knobs and defaults; height / width None take the scheduler's size.  `result` (an EmuVisualGenerationPipelineOutput, or the final latents
    [1, C, h, w] fp32 with output_type="latent") or `error` is set when it is finished, then `done` is set and
    `on_done(request)` is called."""

    def __init__(self, inputs=None, prompt_embeds=None, height=None, width=None, num_inference_steps=50, guidance_scale=3.,
                 crop_info=(0, 0), original_size=(1024, 1024), generator=None, latents=None, output_type="pil",
                 on_done=None, tag=None):
        if (inputs is None) == (prompt_embeds is None):
            raise ValueError("an image request carries either inputs or prompt_embeds")
        self.inputs = inputs if inputs is None or isinstance(inputs, list) else [inputs]
        self.prompt_embeds = prompt_embeds
        self.height, self.width = height, width
        self.steps = int(num_inference_steps)
        self.guidance = float(guidance_scale)
        self.crop_info, self.original_size = list(crop_info), list(original_size)
        self.generator, self.latents, self.output_type = generator, latents, output_type
        self.on_done, self.tag = on_done, tag
        self.done = threading.Event()
        self.result = self.error = None
        if self.steps < 1:
            raise ValueError("num_inference_steps has to be >= 1")
        if output_type not in ("pil", "latent"):
            raise ValueError("output_type must be 'pil' or 'latent', got %r" % (output_type,))
        # set at admission
        self.slot = None
        self.step = 0
        self.regressing = False     # encode_steps: its prompt is in its LLaMA regression slot (the slot index is the same)
        self.n_regressed = 0        # ... its embeddings regressed so far
        self.encoded = None         # the prompt embeddings [cond; uncond] (or [cond]) its latent slot was conditioned with


class DenoiseSlotScheduler(_RequestQueue):
    """Continuous batching of EmuVisualGeneration requests over `n_slots` latent slots (include/emu_b200_gen_slots.h): each
    slot holds one request at its own denoise step, with its own step count, guidance, time ids and latents.  One `step()`:

      1. admit: waiting requests take the lowest free slots.  Each is encoded alone through _prepare_and_encode_inputs (so
         the cached unconditional branch is reused) unless it carries prompt_embeds; its conditioning rows and initial
         latents are written into its slot.  Encoding stalls the live slots;
      2. step: the [n_slots][4] step parameters and the live mask go to the device from a pinned staging buffer, and ONE
         emu_denoise_step_slots over B = highest live slot + 1 moves every live request one step along its own schedule;
      3. retire: a request that has run all its steps is decoded (VAE, uint8, safety stage), answered and leaves its slot.

    A request that fails answers with its own error and frees its slot; the others continue.  Each request's latents are the
    ones `denoise` gives it alone (bitwise while the UNet's row count 2B stays within the GEMV path of its small linears, 8).
    height / width are fixed per scheduler: the buffers, and the CUDA graph of each B, are made for one latent size.
    Owns the pipeline's engine while it lives.  Single-threaded: `submit` may be called from any thread, `step` from one.

    Regression slots (`encode_steps=R`, opt-in): a generation-mode request's prompt is encoded in the engine's LLaMA slot mode
    (include/emu_b200_regress.h) instead of by one generate_image call while every live slot waits.  Its latent slot index is
    also its LLaMA slot, so n_slots <= llm_max_batch, and every regression step runs at B = n_slots.  Admission runs the ViT
    for the newcomers' pictures, embeds their prompts (EmuModel.image_prompt_ids / image_prompt_embeds, as generate_image) and
    prefills all of them in ONE emu_llm_regress_join; then each step() runs up to R emu_llm_regress_step while any prompt is
    regressing.  A request whose L embeddings are done leaves its LLaMA slot, is conditioned ([cond; cached uncond]) into its
    latent slot and denoises from that step's UNet step on.  Requests with prompt_embeds and autoencoding-mode requests
    (pictures only) are encoded at admission as before.  A request's embeddings are those of its prompt regressed alone in the
    same slot of a pool of the same size, bit for bit, and its image is the one it gets from this scheduler alone."""

    def __init__(self, pipeline, n_slots=4, height=1024, width=1024, n_tokens=None, encode_steps=None):
        super().__init__()
        self.pipe, self.engine = pipeline, pipeline.engine
        self.n_slots = int(n_slots)
        if not 1 <= self.n_slots <= 32:
            raise ValueError("n_slots = %d must be in [1, 32]" % self.n_slots)
        self.height, self.width = int(height), int(width)
        f = pipeline.vae_scale_factor
        if self.height % f or self.width % f:
            raise ValueError("height and width must be multiples of %d" % f)
        ucfg = pipeline.unet_config
        self.L = int(n_tokens or pipeline.multimodal_encoder.n_query)
        self.device = torch.device(pipeline.device_)
        n, dev = self.n_slots, self.device
        self.latents = torch.zeros(n, ucfg["in_channels"], self.height // f, self.width // f, dtype=torch.float32, device=dev)
        self.ctx = torch.zeros(2 * n, self.L, ucfg["cross_attention_dim"], dtype=torch.bfloat16, device=dev)
        self.text_embeds = torch.zeros(2 * n, ucfg["cross_attention_dim"], dtype=torch.bfloat16, device=dev)
        self.time_ids = torch.zeros(2 * n, 6, dtype=torch.int32, device=dev)
        # params [n][4] fp32 and live [n] int32 travel in ONE copy: both are views of one byte buffer on each side
        nbytes = n * 4 * 4 + n * 4
        self._stage = torch.zeros(nbytes, dtype=torch.uint8, pin_memory=dev.type == "cuda")
        self._dev = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
        self.params, self.live = self._dev[:n * 16].view(torch.float32).view(n, 4), self._dev[n * 16:].view(torch.int32)
        self._stage_params = self._stage[:n * 16].view(torch.float32).view(n, 4)
        self._stage_live = self._stage[n * 16:].view(torch.int32)
        self._copied = None                                  # event: the last staging copy has run
        self.owner = [None] * n
        self.steps = 0
        self.batch_sizes = collections.deque(maxlen=1024)   # B of the recent UNet steps (observability; the tests read it)
        self.encode_steps = None if encode_steps is None else int(encode_steps)
        self.regress_steps = 0                              # encode_steps: regression steps run, and the recent joins' sizes
        self.join_sizes = collections.deque(maxlen=1024)
        if self.encode_steps is not None:
            self._begin_regression(n)
        # every workspace at its largest size now: a later growth would drop every captured graph
        with _on_device(dev):
            self._unet_step(n)

    def _begin_regression(self, n):
        if self.encode_steps < 1:
            raise ValueError("encode_steps must be >= 1, got %d" % self.encode_steps)
        enc, cfg = self.pipe.multimodal_encoder, self.engine.cfg
        if n > cfg.llm_max_batch:
            raise ValueError("encode_steps: the %d latent slots are LLaMA slots too, at most llm_max_batch = %d"
                             % (n, cfg.llm_max_batch))
        if self.L != enc.n_query:
            raise ValueError("encode_steps: the encoder regresses %d embeddings, the slots hold %d" % (enc.n_query, self.L))
        self.max_seq = int(cfg.llm_max_seq)
        self.embeds = torch.zeros(n, self.L, self.ctx.shape[2], dtype=torch.bfloat16, device=self.device)
        with _on_device(self.device):
            # generate_image resets the LLM (it leaves slot mode): the unconditional branch is made first, once
            self.uncond = self.pipe._unconditional("", lambda: enc.generate_image(text=[""]))
            self.engine.slots_begin(n)

    # ---- producer side ----
    def submit(self, request: ImageRequest):
        if request.height is None and request.width is None:
            request.height, request.width = self.height, self.width
        if (request.height, request.width) != (self.height, self.width):
            raise ValueError("this scheduler generates %dx%d images; a %dx%d request needs a scheduler of its own size"
                             % (self.width, self.height, request.width, request.height))
        text = self._pool_text(request)
        if text is not None:                                # the prompt and L - 1 regressed positions must fit a slot
            n = self.pipe.multimodal_encoder.image_prompt_ids([text])[0].shape[1]
            if n + self.L - 1 > self.max_seq:
                raise ValueError("prompt of %d tokens and %d regressed embeddings exceed llm_max_seq = %d"
                                 % (n, self.L, self.max_seq))
        return super().submit(request)

    def _live(self):
        return [r for r in self.owner if r is not None]

    def _denoising(self):
        return [r for r in self.owner if r is not None and not r.regressing]

    def _pool_text(self, r):
        """encode_steps: the text of r's generation-mode prompt, which regression slots encode; None for a request that is
        encoded at admission (prompt_embeds, autoencoding mode, or encode_steps unset)"""
        if self.encode_steps is None or r.prompt_embeds is not None:
            return None
        from .emu2.constants import DEFAULT_IMG_PLACEHOLDER
        text, pictures, saw_text = self.pipe._prompt_text(r.inputs, DEFAULT_IMG_PLACEHOLDER)
        return None if pictures and not saw_text else text

    # ---- one iteration ----
    @torch.no_grad()
    def step(self):
        """admit -> (regress) -> step -> retire (class docstring); returns the requests finished in this step"""
        with _on_device(self.device):
            self._admit()
            if self.encode_steps is not None:
                self._regress()
            live = self._denoising()
            if not live:
                return []
            try:
                self._unet_step(max(r.slot for r in live) + 1)
            except Exception as ex:       # an engine-level failure: every live request fails, the scheduler stays usable
                for r in live:
                    self._fail(r, ex)
                return live
            self.steps += 1
            self.batch_sizes.append(max(r.slot for r in live) + 1)
            finished = []
            for r in live:
                r.step += 1
                if r.step == r.steps:
                    self._retire(r)
                    finished.append(r)
            return finished

    def _admit(self):
        pool = []
        while True:
            with self._lock:
                if not self.waiting or None not in self.owner:
                    break
                r = self.waiting.popleft()
                r.slot = self.owner.index(None)
                self.owner[r.slot] = r
            try:
                text = self._pool_text(r)
                if text is None:
                    self._fill_slot(r)
                else:
                    pool.append((r, self._pool_prompt(r, text)))
            except Exception as ex:         # a prompt that cannot be encoded fails on its own
                self._fail(r, ex)
        if pool:
            self._regress_join(pool)

    def _fill_slot(self, r):
        pe = r.prompt_embeds
        if pe is None:
            pe = self.pipe._prepare_and_encode_inputs(r.inputs, r.guidance > 1.0)
        self._condition(r, pe)

    def _condition(self, r, pe):
        """r's latent slot from its prompt embeddings pe [2 or 1, L, Cc]: conditioning rows, schedule, initial latents"""
        pipe, s = self.pipe, r.slot
        cfg = r.guidance > 1.0
        pe = pe.to(self.device, torch.bfloat16)
        if pe.dim() != 3 or pe.shape[0] != (2 if cfg else 1) or tuple(pe.shape[1:]) != tuple(self.ctx.shape[1:]):
            raise ValueError("prompt embeddings of shape %s do not fit a slot: expected [%d, %d, %d]"
                             % (tuple(pe.shape), 2 if cfg else 1, self.L, self.ctx.shape[2]))
        ctx, te, tid = pipe.conditioning(pe, self.height, self.width, r.crop_info, r.original_size)
        ts, sig, init_noise_sigma = pipe.schedule(r.steps)
        lat = pipe.initial_latents(1, self.height, self.width, init_noise_sigma, generator=r.generator, latents=r.latents)
        u = 1 if cfg else 0                  # without guidance the unconditional row repeats the conditional one (ignored)
        self.ctx[2 * s], self.ctx[2 * s + 1] = ctx[0], ctx[u]
        self.text_embeds[2 * s], self.text_embeds[2 * s + 1] = te[0], te[u]
        self.time_ids[2 * s], self.time_ids[2 * s + 1] = tid[0], tid[u]
        self.latents[s] = lat[0]
        r.timesteps, r.sigmas = [float(t) for t in ts], [float(v) for v in sig]
        r.encoded = pe

    # ---- regression slots (encode_steps) ----
    def _pool_prompt(self, r, text):
        """r's prompt as generate_image builds it: tokenised with [IMG] appended, its pictures through the ViT, spliced ->
        embeddings [N, hidden]"""
        from .emu2.constants import DEFAULT_IMG_PLACEHOLDER
        enc = self.pipe.multimodal_encoder
        _, pictures, _ = self.pipe._split_prompt(r.inputs, DEFAULT_IMG_PLACEHOLDER)
        ids, mask, image_id = enc.image_prompt_ids([text])
        return enc.image_prompt_embeds(ids, pictures, image_id)[0]

    def _regress_join(self, items):
        """ONE emu_llm_regress_join for the newcomers (two when some prompts are shorter than 128 tokens and some are not: the
        prefill attention kernel is picked by a join's longest prompt, so each prompt joins with its own kind and keeps its
        bits); if a join fails, its prompts join one by one, so that only the culprit fails"""
        for group in ([it for it in items if it[1].shape[0] < 128], [it for it in items if it[1].shape[0] >= 128]):
            if not group:
                continue
            try:
                self._join(group)
            except Exception as ex:
                if len(group) == 1:
                    self._fail(group[0][0], ex)
                    continue
                for item in group:
                    try:
                        self._join([item])
                    except Exception as ex1:
                        self._fail(item[0], ex1)

    def _join(self, items):
        self.engine.regress_join([r.slot for r, _ in items], [e.shape[0] for _, e in items], torch.cat([e for _, e in items]),
                                 self.embeds)
        self.join_sizes.append(len(items))
        for r, _ in items:
            r.regressing, r.n_regressed = True, 1
        for r, _ in items:
            if r.n_regressed == self.L:
                self._regressed(r)

    def _regress(self):
        """up to encode_steps regression steps while any prompt is regressing; a finished prompt conditions its latent slot"""
        for _ in range(self.encode_steps):
            busy = [r for r in self.owner if r is not None and r.regressing]
            if not busy:
                return
            try:
                self.engine.regress_step(self.n_slots, self.embeds)
            except Exception as ex:        # the prompts in the step fail, the scheduler stays usable
                for r in busy:
                    self._fail(r, ex)
                return
            self.regress_steps += 1
            for r in busy:
                r.n_regressed += 1
                if r.n_regressed == self.L:
                    self._regressed(r)

    def _regressed(self, r):
        """r's L embeddings are done: it leaves its LLaMA slot and its latent slot is conditioned"""
        r.regressing = False
        try:
            self.engine.leave([r.slot])
            cond = self.embeds[r.slot:r.slot + 1].clone()
            self._condition(r, torch.cat([cond, self.uncond.to(self.device, torch.bfloat16)]) if r.guidance > 1.0 else cond)
        except Exception as ex:
            self._fail(r, ex)

    def _unet_step(self, B):
        if self._copied is not None:
            self._copied.synchronize()       # the staging buffer is rewritten only after its last copy has run
        self._stage.zero_()
        for r in self._denoising():
            i = r.step
            self._stage_params[r.slot] = torch.tensor([r.sigmas[i], r.sigmas[i + 1], r.timesteps[i], r.guidance])
            self._stage_live[r.slot] = 1
        self._dev.copy_(self._stage, non_blocking=True)
        if self.device.type == "cuda":
            self._copied = torch.cuda.Event()
            self._copied.record()
        self.engine.denoise_step_slots(self.latents, self.params, self.live, self.ctx, self.text_embeds, self.time_ids, B)

    # ---- retirement ----
    def _result(self, r):
        lat = self.latents[r.slot:r.slot + 1].clone()
        if r.output_type == "latent":
            return lat
        from PIL import Image
        from .emu2.diffusion import EmuVisualGenerationPipelineOutput
        u8, flags = self.pipe.decode_and_check(lat)
        return EmuVisualGenerationPipelineOutput(image=Image.fromarray(u8[0]),
                                                 nsfw_content_detected=None if flags is None else flags[0])

    def _release(self, r):
        if r.slot is not None and self.owner[r.slot] is r:
            self.owner[r.slot] = None
            if r.regressing:                 # its LLaMA slot is the same index
                r.regressing = False
                try:
                    self.engine.leave([r.slot])
                except Exception:
                    pass
