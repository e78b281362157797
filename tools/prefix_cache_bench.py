"""Chat prefix caching on one GPU: multi-turn conversations through SlotScheduler with the cache on and off, alternating, on the
real-shape Emu2 model (EVA-CLIP ViT + LLaMA-33B) with random-init weights like bench.py.

Trace (seeded): `--convs` conversations x 3 turns.  Turn 1 is one 448 x 448 picture + text; every later turn resends the whole
history (the previous prompt, the answer's tokens, a few new user tokens), as the demo front end does.  Answers of 32 or 64
tokens (min_len = max_new_tokens), a mix of greedy and 5-beam conversations, about `--think` seconds between an answer and the
next turn.  Reported per run: time to first token p50 / p90 per turn index, generated tokens/s, ViT pictures encoded, prompt
tokens prefilled, and the live rows' stall per admission (wall time of an admission that ran while other requests were live,
ending in a device synchronise).  The card's name and power limit are read in the same call.

`--micro` instead times, on an engine of its own (2 rows, 1100 positions): extend(P, n) against join(P + n) for
P in {100, 400, 1000}, n in {16, 64} (CUDA events, median of `--iters`), and copy_prefix bandwidth at P = 1000 against the
3.35 TB/s data sheet.

    python tools/prefix_cache_bench.py [--convs 8] [--rounds 2] [--think 2.0] [--out f.json]
    python tools/prefix_cache_bench.py --micro [--out f.json]
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

KV_BYTES_PER_POS = 60 * 52 * 128 * 2 * 2  # Emu2 LLaMA-33B: layers x heads x head dim x (K, V) x bf16 = 1.597 MB


def _model(rows, max_seq, small):
    from bench import emu2_cfgs
    from emu_b200.emu2 import synthetic
    from emu_b200.emu2.conf import TextDecoderCfg
    from emu_b200.emu2.emu import EmuModel
    vc, lc = emu2_cfgs(small)
    model = EmuModel(vc, TextDecoderCfg(), tokenizer=synthetic.SyntheticTokenizer(synthetic.VOCAB_EMU2), llama_config=lc,
                     max_batch=rows, max_seq=max_seq)
    synthetic.load_random_weights(model, vc, lc, synthetic.VOCAB_EMU2, seed=0)
    ids, _ = synthetic.image_prompt_ids(n_query=vc.n_query, n_text=8)
    return model, ids, vc.image_size


def conversations(n, seed, S):
    rnd = random.Random(seed)
    g = torch.Generator().manual_seed(seed)
    return [dict(image=torch.randn(1, 3, S, S, generator=g).to(torch.bfloat16), key="pic%d" % i,
                 num_beams=rnd.choice([1, 1, 1, 5]), answers=[rnd.choice([32, 64]) for _ in range(3)],
                 user=[[rnd.randrange(1000, 30000) for _ in range(8)] for _ in range(3)], start=rnd.uniform(0.0, 2.0))
            for i in range(n)]


def run_trace(model, ids, convs, rows, prefix_cache, think):
    from emu_b200.batching import SlotRequest, SlotScheduler
    sched = SlotScheduler(model, rows, prefix_cache=prefix_cache)
    first_tok, stalls = {}, []
    pick, admit = sched._select_one, sched._admit

    def spy_select(r):
        first_tok.setdefault(r.tag, time.time())
        return pick(r)

    def timed_admit():
        live = bool(sched.live)
        t = time.time()
        admit()
        if live and len(sched.live) > 0:
            torch.cuda.synchronize()
            stalls.append(time.time() - t)
    sched._select_one, sched._admit = spy_select, timed_admit
    state = [dict(turn=0, prompt=ids.clone(), due=c["start"], req=None) for c in convs]
    submitted, tokens = {}, 0
    t0 = time.time()
    while True:
        now = time.time() - t0
        for i, (c, st) in enumerate(zip(convs, state)):
            if st["req"] is None and st["turn"] < 3 and now >= st["due"]:
                n = c["answers"][st["turn"]]
                tag = (i, st["turn"])
                st["req"] = sched.submit(SlotRequest(st["prompt"], image=c["image"].cuda(), image_keys=[c["key"]],
                                                     num_beams=c["num_beams"], max_new_tokens=n, min_len=n, length_penalty=-1,
                                                     tag=tag))
                submitted[tag] = time.time()
            r = st["req"]
            if r is not None and r.done.is_set():
                if r.error is not None:
                    raise r.error
                out = r.result.cpu()
                tokens += int(out.shape[1])
                st["prompt"] = torch.cat([st["prompt"], out.to(st["prompt"].dtype),
                                          torch.tensor([c["user"][st["turn"]]], dtype=st["prompt"].dtype)], 1)
                st["turn"] += 1
                st["req"], st["due"] = None, time.time() - t0 + think
        if all(st["turn"] == 3 for st in state):
            break
        if sched.busy():
            sched.step()
        else:
            time.sleep(0.005)
    wall = time.time() - t0
    ttft = {}
    for (i, turn), t in submitted.items():
        ttft.setdefault(turn, []).append(first_tok[(i, turn)] - t)
    q = lambda xs, p: sorted(xs)[min(len(xs) - 1, int(p * len(xs)))]
    return dict(prefix_cache=prefix_cache, tok_per_s=round(tokens / wall, 1), wall_s=round(wall, 2),
                ttft_ms={t + 1: dict(p50=round(1e3 * q(v, 0.5), 1), p90=round(1e3 * q(v, 0.9), 1)) for t, v in sorted(ttft.items())},
                vit_pictures=sched.vit_pictures, prefill_tokens=sched.prefill_tokens, prefix_hits=sched.prefix_hits,
                prefix_tokens_reused=sched.prefix_tokens_reused,
                stall_ms=dict(n=len(stalls), p50=round(1e3 * q(stalls, 0.5), 1) if stalls else None,
                              max=round(1e3 * max(stalls), 1) if stalls else None))


def micro(model, iters):
    eng = model.engine
    H = eng.cfg.llm_hidden
    g = torch.Generator().manual_seed(1)
    emb = (torch.randn(1, 1064, H, generator=g) * 0.5).to(torch.bfloat16).cuda()

    def timed(fn):
        ts = []
        for i in range(iters + 2):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            setup = fn()
            a.record()
            setup()
            b.record()
            torch.cuda.synchronize()
            if i >= 2:
                ts.append(a.elapsed_time(b))
        return round(statistics.median(ts), 3)
    res = []
    for P in (100, 400, 1000):
        for n in (16, 64):
            def join_all():
                eng.slots_begin(2)
                return lambda: eng.join([0], emb[:, :P + n])

            def extend():
                eng.slots_begin(2)
                eng.join([0], emb[:, :P])
                eng.leave_keep([0], [P])
                torch.cuda.synchronize()
                return lambda: eng.extend([0], [P], [n], emb[:, P:P + n])
            res.append(dict(P=P, n=n, join_ms=timed(join_all), extend_ms=timed(extend)))
    P = 1000

    def copy():
        eng.slots_begin(2)
        eng.join([0], emb[:, :P])
        torch.cuda.synchronize()
        return lambda: eng.copy_prefix(0, 1, P)
    ms = timed(copy)
    gbs = 2 * P * KV_BYTES_PER_POS / (ms * 1e-3) / 1e9
    eng.llm_reset()
    return dict(extend_vs_join=res, copy_prefix=dict(P=P, ms=ms, GB_per_s=round(gbs, 1), frac_of_3350=round(gbs / 3350, 3)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--convs", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--think", type=float, default=2.0)
    ap.add_argument("--rows", type=int, default=10, help="KV-cache slots")
    ap.add_argument("--micro", action="store_true")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--small", action="store_true", help="tiny shapes (a functional check, not a measurement)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    name, pl = card()
    if a.micro:
        model, _, _ = _model(2, 1100, a.small)
        out = dict(tool="prefix_cache_bench", mode="micro", card=name, power_limit=pl, small=a.small, **micro(model, a.iters))
    else:
        model, ids, S = _model(a.rows, 320, a.small)
        convs = conversations(a.convs, 11, S)
        runs = []
        for r in range(a.rounds):
            for on in (False, True):
                runs.append(dict(round=r, **run_trace(model, ids, convs, a.rows, on, a.think)))
                print(json.dumps(runs[-1]), file=sys.stderr, flush=True)
        out = dict(tool="prefix_cache_bench", mode="trace", card=name, power_limit=pl, small=a.small, convs=a.convs,
                   beams=[c["num_beams"] for c in convs], think_s=a.think, rows=a.rows, runs=runs)
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
