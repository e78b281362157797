"""Chunked prefill on one GPU, on the real-shape Emu2 model (EVA-CLIP ViT + LLaMA-33B) with random-init weights like bench.py.

`--micro`: on an engine of its own (9 rows, 520 positions; a one-layer ViT, which is not timed, so the cache fits the card),
times one mixed step `step(B decode rows, one segment of C tokens)` against what the scheduler runs without chunking,
`decode(B)` + `extend(C)`, for B in {1, 4, 8} and C in {64, 256, 512}.  The B live rows hold 64-token prompts.  CUDA events,
median of `--iters`.

Trace (default): a seeded mix of short chats (one 448 x 448 picture, 8-24 text tokens, 32-64 answer tokens) and interleaved
few-shot requests (3 pictures and ~100 text tokens, about 300 prompt tokens, 32 answer tokens), arriving over a few seconds,
through SlotScheduler with chunking off and with C in `--chunks`, alternating in each round (8 slots, 400 positions).
Reported per run: generated tokens/s, time to first token p50 / p90, and the live requests' inter-token gap p50 / p99 (the
wall time between two consecutive token selections of one request: the stall a newcomer causes).  The card's name and power
limit are read in the same call.

    python tools/chunked_prefill_bench.py --micro [--iters 10] [--out f.json]
    python tools/chunked_prefill_bench.py [--rounds 2] [--chunks 128,256] [--out f.json]
"""
import argparse
import json
import os
import random
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.batching_bench import card  # noqa: E402


def _model(rows, max_seq, small, vit_layers=None):
    from bench import emu2_cfgs
    from emu_b200.emu2 import synthetic
    from emu_b200.emu2.conf import TextDecoderCfg
    from emu_b200.emu2.emu import EmuModel
    vc, lc = emu2_cfgs(small)
    if vit_layers is not None:
        vc.layers = vit_layers
    model = EmuModel(vc, TextDecoderCfg(), tokenizer=synthetic.SyntheticTokenizer(synthetic.VOCAB_EMU2), llama_config=lc,
                     max_batch=rows, max_seq=max_seq)
    synthetic.load_random_weights(model, vc, lc, synthetic.VOCAB_EMU2, seed=0)
    return model, vc


def micro(model, iters, Bs, Cs):
    eng = model.engine
    H, V = eng.cfg.llm_hidden, eng.cfg.llm_vocab
    g = torch.Generator().manual_seed(1)
    emb = (torch.randn(1, 640, H, generator=g) * 0.5).to(torch.bfloat16).cuda()
    tok = torch.arange(9, dtype=torch.int32, device="cuda") + 100
    buf = torch.empty(9, V, dtype=torch.float32, device="cuda")

    def timed(fn):
        ts = []
        for i in range(iters + 2):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            run = fn()
            torch.cuda.synchronize()
            a.record()
            run()
            b.record()
            torch.cuda.synchronize()
            if i >= 2:
                ts.append(a.elapsed_time(b))
        return round(statistics.median(ts), 3)

    res = []
    for B in Bs:
        for C in Cs:
            def live():
                eng.slots_begin(9)
                eng.join(list(range(B)), emb[:, :64].expand(B, -1, -1).contiguous())

            def separate():
                live()
                return lambda: (eng.llm_decode(token_ids=tok, logits=buf, B=B), eng.extend([B], [0], [C], emb[:, :C]))

            def mixed():
                live()
                return lambda: eng.step([B], [0], [C], [True], emb[0, :C], token_ids=tok, B=B, logits=buf)
            sep, mix = timed(separate), timed(mixed)
            res.append(dict(B=B, C=C, decode_plus_extend_ms=sep, step_ms=mix, saved_ms=round(sep - mix, 3)))
            print(json.dumps(res[-1]), file=sys.stderr, flush=True)
    eng.llm_reset()
    return dict(step_vs_decode_plus_extend=res)


def _picture_ids(n_query, rnd, n_text):
    from emu_b200.emu2.synthetic import IDS
    return [IDS["[IMG]"]] + [IDS["<image>"]] * n_query + [IDS["[/IMG]"]] + [rnd.randrange(100, 31000) for _ in range(n_text)]


def requests(n, seed, n_query, S):
    """a seeded mix: 2 of 3 short chats, 1 of 3 few-shot requests; arrival times over ~n / 2 seconds"""
    from emu_b200.emu2.synthetic import IDS
    rnd = random.Random(seed)
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        few = i % 3 == 2
        pics = 3 if few else 1
        ids = [IDS["bos"]]
        for p in range(pics):
            ids += _picture_ids(n_query, rnd, rnd.randrange(25, 40) if few else rnd.randrange(8, 25))
        out.append(dict(ids=torch.tensor([ids]), image=torch.randn(pics, 3, S, S, generator=g).to(torch.bfloat16),
                        answer=32 if few else rnd.choice([32, 48, 64]), kind="few_shot" if few else "chat",
                        start=rnd.uniform(0.0, n / 2.0)))
    return out


def run_trace(model, reqs, rows, chunk):
    from emu_b200.batching import SlotRequest, SlotScheduler
    sched = SlotScheduler(model, rows, prefill_chunk=chunk)
    stamps = {}
    pick = sched._select_one

    def spy(r):
        stamps.setdefault(r.tag, []).append(time.time())
        return pick(r)
    sched._select_one = spy
    submitted, live_reqs, tokens = {}, [], 0
    order = sorted(range(len(reqs)), key=lambda i: reqs[i]["start"])
    t0 = time.time()
    while True:
        now = time.time() - t0
        while order and reqs[order[0]]["start"] <= now:
            i = order.pop(0)
            q = reqs[i]
            live_reqs.append(sched.submit(SlotRequest(q["ids"], image=q["image"].cuda(), num_beams=1, max_new_tokens=q["answer"],
                                                      min_len=q["answer"], tag=i)))
            submitted[i] = time.time()
        if not order and all(r.done.is_set() for r in live_reqs):
            break
        if sched.busy():
            sched.step()
        else:
            time.sleep(0.002)
    wall = time.time() - t0
    for r in live_reqs:
        if r.error is not None:
            raise r.error
        tokens += int(r.result.shape[1])
    q = lambda xs, p: sorted(xs)[min(len(xs) - 1, int(p * len(xs)))]
    ttft = [stamps[i][0] - submitted[i] for i in submitted]
    gaps = [b - a for ts in stamps.values() for a, b in zip(ts, ts[1:])]
    return dict(prefill_chunk=chunk, tok_per_s=round(tokens / wall, 1), wall_s=round(wall, 2),
                ttft_ms=dict(p50=round(1e3 * q(ttft, 0.5), 1), p90=round(1e3 * q(ttft, 0.9), 1)),
                gap_ms=dict(p50=round(1e3 * q(gaps, 0.5), 1), p99=round(1e3 * q(gaps, 0.99), 1), max=round(1e3 * max(gaps), 1)),
                mixed_steps=sched.prefill_chunks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--micro", action="store_true")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--requests", type=int, default=12)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--chunks", default="128,256")
    ap.add_argument("--rows", type=int, default=8, help="KV-cache slots of the trace")
    ap.add_argument("--small", action="store_true", help="tiny shapes (a functional check, not a measurement)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    name, pl = card()
    if a.micro:
        model, _ = _model(9, 520, a.small, vit_layers=1)
        Cs = (64, 256, 512) if not a.small else (16, 64)
        out = dict(tool="chunked_prefill_bench", mode="micro", card=name, power_limit=pl, small=a.small,
                   **micro(model, a.iters, (1, 4, 8), Cs))
    else:
        model, vc = _model(a.rows, 400, a.small)
        reqs = requests(a.requests, 7, vc.n_query, vc.image_size)
        runs = []
        for r in range(a.rounds):
            for chunk in [None] + [int(c) for c in a.chunks.split(",")]:
                runs.append(dict(round=r, **run_trace(model, reqs, a.rows, chunk)))
                print(json.dumps(runs[-1]), file=sys.stderr, flush=True)
        out = dict(tool="chunked_prefill_bench", mode="trace", card=name, power_limit=pl, small=a.small, rows=a.rows,
                   kinds=[q["kind"] for q in reqs], prompt_tokens=[int(q["ids"].shape[1]) for q in reqs], runs=runs)
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
