"""Prompt-lookup speculative decoding restated on host lists: the draft (transformers 5.5
`PromptLookupCandidateGenerator.get_candidates`, without logits processors) and the acceptance step, as emu_spec_draft and
emu_spec_accept compute them on the device."""


def prompt_lookup_draft(hist, k, max_ngram, max_length, eos_id):
    """the draft (a list, possibly empty) that follows hist (a list of token ids, len >= 1)"""
    n = len(hist)
    if max_length == n + 1:
        return []
    for g in range(min(max_ngram, n - 1), 0, -1):
        tail = hist[n - g:]
        for idx in range(0, n - g + 1):
            if hist[idx:idx + g] != tail:
                continue
            s = idx + g
            e = min(s + k, n, max_length)
            if s < e:
                draft = hist[s:e]
                if eos_id in draft:
                    draft = draft[:draft.index(eos_id)]
                return draft
    return []


def accept(hist, draft, next_ids, eos_id, max_len):
    """after a verify of [last token] + draft with arg-max next_ids: (tokens appended to hist in place, finished)"""
    a = 0
    while a < len(draft) and draft[a] == next_ids[a]:
        a += 1
    m, done = 0, False
    for t in next_ids[:a + 1]:
        if len(hist) >= max_len:
            break
        hist.append(t)
        m += 1
        if t == eos_id:
            done = True
            break
    return m, done or len(hist) >= max_len
