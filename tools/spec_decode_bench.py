"""Prompt-lookup speculative decoding on one GPU: LLaMA-33B at its real shape (60 layers, random-init weights like bench.py),
batch 1, greedy.  The card's name and power limit are read in the same call.  Times are CUDA events, medians of --iters runs
after a warm-up of every shape.

`--micro`: one emu_llm_verify of n rows against one emu_llm_decode step at B = 1, for n = 1..8 at contexts 128, 1024 and 4096
(the engine holds 8 cache rows, so at 4096 the 60 layers' weights and cache exceed 80 GB: `--layers` builds fewer, and the
JSON says how many ran);
and the verify attention kernel (n queries, each K / V row read once) against the decode attention at B = n with every row's
table pointing at the same cache row (the context read n times), one layer (52 heads x 128).

Default: controlled acceptance.  Random-init weights say nothing about how often a real draft is right, so the tool supplies
the drafts itself through verify / commit: the plain greedy run's own next tokens, each replaced by a wrong token with
probability 1 - p.  tok/s for p in {0, 0.25, 0.5, 0.75, 1} and k in {2, 4, 7} against plain greedy, and the ids checked
against plain greedy.  p = 0 is the worst case (every pass yields one token).  Then generate(prompt_lookup_num_tokens=k) on
the random-init model, whose drafts come from the prompt: reported, and NOT representative of real prompts.

    python tools/spec_decode_bench.py --micro [--iters 10] [--out f.json]
    python tools/spec_decode_bench.py [--iters 10] [--tokens 32] [--out f.json]
"""
import argparse
import json
import os
import random
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.gen_batching_bench import card  # noqa: E402


def model(max_seq, layers):
    from bench import emu2_cfgs
    from emu_b200.emu2 import synthetic
    from emu_b200.emu2.conf import TextDecoderCfg
    from emu_b200.emu2.emu import EmuModel
    from tools.gen_encode_bench import WordTokenizer
    vc, lc = emu2_cfgs()
    vc.layers = 1                                       # text-only prompts never run the ViT
    lc = dict(lc, num_hidden_layers=layers)
    m = EmuModel(vc, TextDecoderCfg(), tokenizer=WordTokenizer(), llama_config=lc, max_batch=8, max_seq=max_seq)
    synthetic.load_random_weights(m, vc, lc, synthetic.VOCAB_EMU2, seed=0)
    return m, lc


def timed(fn, iters, warmup=2):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def prompt_embeds(eng, n, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(100, 31000, (1, n), generator=g).cuda()
    return ids, eng.llm_embed(ids)


def micro(m, iters, contexts):
    from emu_b200 import _lib
    eng = m.engine
    res = {"verify_vs_decode_ms": {}, "attention_us": {}}
    i32 = dict(dtype=torch.int32, device="cuda")
    for ctx in contexts:
        _, emb = prompt_embeds(eng, ctx)
        mask = torch.ones(1, ctx, dtype=torch.long, device="cuda")
        eng.llm_reset()
        eng.llm_prefill(emb, mask)
        ping = [torch.zeros(1, **i32), torch.zeros(1, **i32)]
        state = [0]

        def decode():
            s = state[0]
            eng.llm_decode(token_ids=ping[s & 1], next_ids=ping[(s + 1) & 1], B=1)
            state[0] += 1

        row = {"decode_B1": timed(decode, iters)}       # the cache grows by iters + 2 positions: < 2% of 128
        eng.llm_reset()
        eng.llm_prefill(emb, mask)
        toks, nxt = torch.zeros(8, **i32), torch.zeros(8, **i32)
        for n in range(1, 9):
            row["verify_n%d" % n] = timed(lambda: eng.llm_verify(toks, n, next_ids=nxt), iters)
        res["verify_vs_decode_ms"][ctx] = row
        # the attention kernels alone on one layer's cache: verify (one read) against decode at B = n over one shared row
        H, D = 52, 128
        t_max = ctx + 8
        kc = torch.randn(8, H, t_max, D, device="cuda").to(torch.bfloat16)
        vc = torch.randn_like(kc)
        arow = {}
        for n in (1, 2, 4, 8):
            q = torch.randn(n, H * D, device="cuda").to(torch.bfloat16)
            pos1 = torch.tensor([ctx], **i32)
            posn = torch.arange(ctx, ctx + n, **i32)
            indir = torch.zeros(n, t_max, **i32)
            v_ms = timed(lambda: _lib.op_attn_verify(q, kc, vc, pos1, D ** -0.5), iters * 5)
            d_ms = timed(lambda: _lib.op_attn_decode_rows(q, kc, vc, posn, None, D ** -0.5, t_max, indir=indir), iters * 5)
            arow["n%d" % n] = {"verify_us": 1e3 * v_ms, "decode_rows_us": 1e3 * d_ms}
        res["attention_us"][ctx] = arow
        del kc, vc
        print(json.dumps({ctx: {"layers_ms": row, "attention_us": arow}}), flush=True)
    return res


def plain_greedy(eng, emb, n_tok):
    from emu_b200 import generation
    mask = torch.ones(1, emb.shape[1], dtype=torch.long, device="cuda")
    return generation.greedy_search(eng, emb, mask, n_tok, -1, 0, check_every=0)[0].tolist()


def controlled(eng, emb, plain, k, p, rng):
    """greedy with drafts = the plain run's next tokens, each wrong with probability 1 - p; returns (ids, passes)"""
    i32 = dict(dtype=torch.int32, device="cuda")
    mask = torch.ones(1, emb.shape[1], dtype=torch.long, device="cuda")
    eng.llm_reset()
    _, lg = eng.llm_prefill(emb, mask)
    out = [int(lg.argmax(-1))]
    toks, nxt = torch.zeros(k + 1, **i32), torch.zeros(k + 1, **i32)
    host = torch.zeros(k + 1, dtype=torch.int32).pin_memory()
    passes = 0
    while len(out) < len(plain):
        j = len(out)
        d = min(k, len(plain) - j - 1)
        draft = [plain[j + i] if rng.random() < p else (plain[j + i] + 1 + rng.randrange(1000)) % 32000 for i in range(d)]
        host[:d + 1] = torch.tensor([out[-1]] + draft, dtype=torch.int32)
        toks[:d + 1].copy_(host[:d + 1], non_blocking=True)
        eng.llm_verify(toks, d + 1, next_ids=nxt)
        got = nxt[:d + 1].tolist()
        passes += 1
        a = 0
        while a < d and draft[a] == got[a]:
            a += 1
        out += got[:a + 1]
        eng.llm_commit(a + 1)
    return out[:len(plain)], passes


def divergence(eng, emb, plain, got):
    """where `got` first departs from the plain run, the plain decode step's logit gap between the two tokens there (a near tie
    when it is within the bf16 rounding of the logits) and the spread of that row's logits"""
    t = next((i for i, (a, b) in enumerate(zip(plain, got)) if a != b), None)
    if t is None:
        return None
    mask = torch.ones(1, emb.shape[1], dtype=torch.long, device="cuda")
    eng.llm_reset()
    _, lg = eng.llm_prefill(emb, mask)
    for i in range(t):
        eng.llm_decode(token_ids=torch.tensor([plain[i]], dtype=torch.int32, device="cuda"), logits=lg, B=1)
    row = lg[0].float()
    return {"step": t, "logit_gap": float(row[plain[t]] - row[got[t]]), "logit_max": float(row.max()),
            "logit_std": float(row.std())}


def acceptance(m, iters, n_tok):
    from emu_b200 import generation
    eng = m.engine
    ids, emb = prompt_embeds(eng, 128, seed=1)
    plain = plain_greedy(eng, emb, n_tok)
    base_ms = timed(lambda: plain_greedy(eng, emb, n_tok), iters, warmup=1)
    res = {"tokens": n_tok, "plain_greedy_tok_s": 1e3 * n_tok / base_ms, "controlled": {}}
    ok = True
    for k in (2, 4, 7):
        for p in (0.0, 0.25, 0.5, 0.75, 1.0):
            rng = random.Random(0)
            got, passes = controlled(eng, emb, plain, k, p, rng)
            ok &= got == plain
            ms = timed(lambda: controlled(eng, emb, plain, k, p, random.Random(0)), iters, warmup=1)
            res["controlled"]["k%d_p%.2f" % (k, p)] = {"tok_s": 1e3 * n_tok / ms, "speedup": base_ms / ms,
                                                        "passes": passes, "ids_equal_plain": got == plain}
            print(json.dumps({"k": k, "p": p, **res["controlled"]["k%d_p%.2f" % (k, p)]}), flush=True)
    res["controlled_ids_equal_plain"] = ok
    res["first_divergence_k2_p0"] = divergence(eng, emb, plain, controlled(eng, emb, plain, 2, 0.0, random.Random(0))[0])
    # prompt lookup itself on the random-init model: its drafts come from a random prompt, NOT representative
    mask = torch.ones_like(ids)
    pl = {}
    for k in (2, 4, 7):
        def run():
            return generation.generate(eng, emb, mask, n_tok, -1, 0, num_beams=1, prompt_lookup_num_tokens=k, prompt_ids=ids)
        out = run()[0].tolist()
        ms = timed(run, iters, warmup=1)
        pl["k%d" % k] = {"tok_s": 1e3 * n_tok / ms, "speedup": base_ms / ms, "ids_equal_plain": out == plain}
    res["prompt_lookup_random_init_not_representative"] = pl
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--micro", action="store_true")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--tokens", type=int, default=32)
    ap.add_argument("--out", default=None)
    ap.add_argument("--contexts", default="128,1024,4096", help="--micro: prompt lengths")
    ap.add_argument("--layers", type=int, default=60,
                    help="decoder layers (60 = LLaMA-33B; with 8 cache rows a 4096 context only fits 80 GB with fewer)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spec_decode_bench needs a GPU")
    name, power = card()
    contexts = [int(c) for c in args.contexts.split(",")]
    m, lc = model(max(contexts) + 16 if args.micro else 128 + args.tokens + 16, args.layers)
    res = {"tool": "spec_decode_bench", "card": name, "power_limit": power, "llm_layers": lc["num_hidden_layers"]}
    with torch.no_grad():
        res.update(micro(m, args.iters, contexts) if args.micro else acceptance(m, args.iters, args.tokens))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
