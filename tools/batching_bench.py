"""Admission batching vs continuous batching for chat on one GPU: a seeded synthetic trace of image + text requests (one
448 x 448 picture each, arrivals spread over time, max_new_tokens from {16, 64, 128}, num_beams 1 or 5) run through
serve.BatchingWorker and serve.ContinuousWorker, alternating, on the real-shape Emu2 model (EVA-CLIP ViT + LLaMA-33B) with
random-init weights like bench.py.  Every request generates exactly its max_new_tokens (min_len = max_new_tokens).  Prints
one JSON line: generated tokens/s and p50 / p90 request latency per scheduler and round, the slot-mode decode step time at
B = 1..8 (CUDA events), and the card's name and power limit read in the same call.

    python tools/batching_bench.py [--requests 16] [--rounds 2] [--span 6.0] [--small] [--out results/batching.json]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import threading
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in q.split(",")]
        return name, pl
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


class IdChat:
    """a chat pipeline at the token-id level (no tokenizer file): inputs = (prompt ids [1, N], picture [1, 3, S, S])"""

    def __init__(self, model):
        self.emu_model = model

    def forward_batch(self, batch_inputs, num_beams, max_new_tokens):
        ids = torch.cat([i for i, _ in batch_inputs]).cuda()
        img = torch.cat([p for _, p in batch_inputs]).cuda()
        out = self.emu_model.generate_from_ids(ids, torch.ones_like(ids), image=img, num_beams=num_beams,
                                               max_new_tokens=max_new_tokens, min_len=max_new_tokens, length_penalty=-1)
        return [out[b:b + 1] for b in range(len(batch_inputs))]

    def __call__(self, inputs, **knobs):
        return self.forward_batch([inputs], **knobs)[0]

    def max_requests_per_batch(self, num_beams=5):
        return max(1, int(self.emu_model.engine.cfg.llm_max_batch) // max(1, int(num_beams)))


def slot_request(pipe, inputs, knobs):
    from emu_b200.batching import SlotRequest
    ids, img = inputs
    return SlotRequest(ids, image=img.cuda(), num_beams=knobs["num_beams"], max_new_tokens=knobs["max_new_tokens"],
                       min_len=knobs["max_new_tokens"], length_penalty=-1)


def trace(n, span, seed, ids, S):
    rnd = random.Random(seed)
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        img = torch.randn(1, 3, S, S, generator=g).to(torch.bfloat16)
        knobs = dict(num_beams=rnd.choice([1, 1, 5]), max_new_tokens=rnd.choice([16, 64, 128]))
        out.append((rnd.uniform(0.0, span), (ids, img), knobs))
    return sorted(out, key=lambda t: t[0])


def run(worker, reqs):
    worker.start()
    done = {}
    t0 = time.time() + 0.5

    def client(i, at, inputs, knobs):
        time.sleep(max(0.0, t0 + at - time.time()))
        t_in = time.time()
        out = worker.submit(inputs, knobs)
        done[i] = (t_in, time.time(), int(out.shape[1]))
    ts = [threading.Thread(target=client, args=(i, *r)) for i, r in enumerate(reqs)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    worker.stop()
    worker.join(timeout=600)
    lat = sorted(b - a for a, b, _ in done.values())
    first, last = min(a for a, _, _ in done.values()), max(b for _, b, _ in done.values())
    toks = sum(n for _, _, n in done.values())
    q = lambda p: lat[min(len(lat) - 1, int(p * len(lat)))]
    return dict(tokens=toks, wall_s=round(last - first, 3), tok_per_s=round(toks / (last - first), 1),
                p50_s=round(q(0.5), 3), p90_s=round(q(0.9), 3))


def step_times(model, ids, img, iters=20):
    """ms per slot-mode decode step at B = 1..8 (B live slots, each holding the prompt)"""
    eng = model.engine
    emb = model.embed_prompt(ids.cuda(), img.cuda())
    tok = torch.full((8,), 100, dtype=torch.int32, device="cuda")
    lg = torch.empty(8, eng.cfg.llm_vocab, dtype=torch.float32, device="cuda")
    res = {}
    for B in range(1, 9):
        eng.slots_begin(8)
        eng.join(list(range(B)), emb.expand(B, -1, -1).contiguous())
        for _ in range(3):
            eng.llm_decode(token_ids=tok, logits=lg, B=B)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            eng.llm_decode(token_ids=tok, logits=lg, B=B)
        b.record()
        torch.cuda.synchronize()
        res[B] = round(a.elapsed_time(b) / iters, 3)
    eng.llm_reset()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--span", type=float, default=6.0, help="arrivals spread uniformly over this many seconds")
    ap.add_argument("--rows", type=int, default=10, help="KV-cache rows (slots)")
    ap.add_argument("--small", action="store_true", help="tiny shapes (a functional check, not a measurement)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    from bench import emu2_cfgs
    from emu_b200 import serve
    from emu_b200.emu2 import synthetic
    from emu_b200.emu2.conf import TextDecoderCfg
    from emu_b200.emu2.emu import EmuModel
    name, pl = card()
    vc, lc = emu2_cfgs(a.small)
    ids, _ = synthetic.image_prompt_ids(n_query=vc.n_query, n_text=8)
    model = EmuModel(vc, TextDecoderCfg(), tokenizer=synthetic.SyntheticTokenizer(synthetic.VOCAB_EMU2), llama_config=lc,
                     max_batch=a.rows, max_seq=ids.shape[1] + 128 + 8)
    synthetic.load_random_weights(model, vc, lc, synthetic.VOCAB_EMU2, seed=0)
    chat = IdChat(model)
    reqs = trace(a.requests, a.span, 7, ids, vc.image_size)
    rounds = []
    for r in range(a.rounds):
        for kind in ("batching", "continuous"):
            if kind == "batching":
                w = serve.BatchingWorker(chat, "chat", lambda k: chat.max_requests_per_batch(k["num_beams"]), 0.0)
            else:
                w = serve.ContinuousWorker(chat, a.rows, make_request=slot_request)
            rounds.append(dict(round=r, scheduler=kind, **run(w, reqs)))
            print(json.dumps(rounds[-1]), file=sys.stderr, flush=True)
    steps = step_times(model, ids, reqs[0][1][1])
    mix = dict(beams={b: sum(1 for _, _, k in reqs if k["num_beams"] == b) for b in (1, 5)},
               max_new={n: sum(1 for _, _, k in reqs if k["max_new_tokens"] == n) for n in (16, 64, 128)})
    out = dict(tool="batching_bench", card=name, power_limit=pl, small=a.small, requests=a.requests, span_s=a.span,
               rows=a.rows, trace=mix, rounds=rounds, decode_step_ms=steps)
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
