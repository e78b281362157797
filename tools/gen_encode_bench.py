"""Prompt encoding for continuous image generation on one GPU: Emu2-Gen's regression (EmuModel.generate_image: one prefill of
`text + [IMG]`, then 63 single-row LLaMA-33B steps fed with project_up(project_down(h))) one prompt at a time, against
regression slots (include/emu_b200_regress.h: one emu_llm_regress_join for all newcomers, then emu_llm_regress_step for every
slot at once).  Random-init weights like bench.py; text-only prompts; the card's name and power limit are read in the same call.

`--micro`: LLaMA-33B at its real shape (60 layers; a one-layer ViT, which text-only prompts never run), prompts of about 20
tokens, L = 64.  k prompts through generate_image one after another, against one regress_join + 63 regress_steps in a pool of
k slots, for k = 1, 2, 4, 8; and the time of one regress_step at B = 1..8.  CUDA events, median of --iters after a warm-up of
every shape.

Trace (default): encoder + Emu2-Gen UNet + VAE decoder in one engine.  --requests text-only requests at 1024 x 1024 arriving
over --span seconds, steps from {25, 50}, guidance 3, through serve.BatchingWorker (admission batching) and a ContinuousWorker
over DenoiseSlotScheduler with encode_steps off and each R of --encode-steps, --slots latent slots.  The whole model does not
fit 80 GB next to the UNet and VAE workspaces (at 60 layers the VAE decode of a 4-image batch runs out of memory on an
80 GB card): the encoder is built with max_seq = prompt + 64 and --llm-layers decoder layers, 48 by default (fewer are tried
if the engine cannot be built; the JSON says what ran, and no number is scaled to 60 layers).  Reported per scheduler:
images/s, p50 / p90 latency, and the longest gap between two consecutive UNet steps of a live request.

    python tools/gen_encode_bench.py --micro [--iters 5] [--out f.json]
    python tools/gen_encode_bench.py [--requests 12] [--span 8] [--slots 4] [--encode-steps 8,64] [--out f.json]
"""
import argparse
import json
import os
import random
import statistics
import sys
import time
import zlib

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.gen_batching_bench import EMU2_VAE, card, run_round, vae_decoder_shapes  # noqa: E402

PROMPT_WORDS = 18


class WordTokenizer:
    """BOS + one id per word (a stable hash into the text range) + the special tokens as themselves, left padding"""
    pad_token_id, bos_token_id, eos_token_id = 32000, 1, 2
    padding_side = truncation_side = "left"
    _special = {"[IMG]": 32001, "[/IMG]": 32002, "<image>": 32003, "[gIMG]": 32004}

    def __len__(self):
        return 32272

    def convert_tokens_to_ids(self, toks):
        return [self._special[t] for t in toks]

    def batch_decode(self, ids, skip_special_tokens=True):
        return [" ".join(str(int(i)) for i in row) for row in ids]

    def __call__(self, texts, padding="longest", return_tensors="pt"):
        from types import SimpleNamespace as NS
        rows = []
        for t in texts:
            for k in self._special:
                t = t.replace(k, " %s " % k)
            rows.append([1] + [self._special.get(w, 100 + zlib.crc32(w.encode()) % 30000) for w in t.split()])
        n = max(map(len, rows))
        return NS(input_ids=torch.tensor([[self.pad_token_id] * (n - len(r)) + r for r in rows]),
                  attention_mask=torch.tensor([[0] * (n - len(r)) + [1] * len(r) for r in rows]))


def prompt(i):
    rnd = random.Random(1000 + i)
    return " ".join("w%d" % rnd.randrange(100000) for _ in range(PROMPT_WORDS))


def encoder(layers, rows, max_seq):
    from bench import emu2_cfgs
    from emu_b200.emu2 import synthetic
    from emu_b200.emu2.conf import TextDecoderCfg
    from emu_b200.emu2.emu import EmuModel
    vc, lc = emu2_cfgs()
    vc.layers = 1
    lc = dict(lc, num_hidden_layers=layers)
    m = EmuModel(vc, TextDecoderCfg(), tokenizer=WordTokenizer(), llama_config=lc, max_batch=rows, max_seq=max_seq)
    synthetic.load_random_weights(m, vc, lc, synthetic.VOCAB_EMU2, seed=0)
    return m


def timed(fn, iters):
    """fn() prepares and returns the callable to time; the first call is the warm-up"""
    ts = []
    for i in range(iters + 1):
        run = fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        torch.cuda.synchronize()
        if i:
            ts.append(a.elapsed_time(b))
    return round(statistics.median(ts), 3)


def micro(iters):
    m = encoder(60, 8, 128)
    eng, L, W = m.engine, m.n_query, m.vision_cfg.width
    prompts = []
    for i in range(8):
        ids, mask, image_id = m.image_prompt_ids([prompt(i)])
        prompts.append((ids, mask, m.image_prompt_embeds(ids, None, image_id)[0]))
    out = torch.zeros(8, L, W, dtype=torch.bfloat16, device="cuda")
    res = {"prompt_tokens": [int(p[0].shape[1]) for p in prompts], "L": L, "solo_vs_pool": [], "regress_step_ms": {}}
    for k in (1, 2, 4, 8):
        def solo():
            return lambda: [m.generate_image_from_ids(ids, mask, image_token_id=32003) for ids, mask, _ in prompts[:k]]

        def pool():
            eng.slots_begin(k)
            es = [e for _, _, e in prompts[:k]]

            def run():
                eng.regress_join(list(range(k)), [e.shape[0] for e in es], torch.cat(es), out)
                for _ in range(L - 1):
                    eng.regress_step(k, out)
            return run
        a, b = timed(solo, iters), timed(pool, iters)
        res["solo_vs_pool"].append(dict(k=k, generate_image_one_after_another_ms=a, regress_join_plus_steps_ms=b,
                                        speedup=round(a / b, 2)))
        print(json.dumps(res["solo_vs_pool"][-1]), file=sys.stderr, flush=True)
    for B in range(1, 9):
        def step():
            eng.slots_begin(B)
            es = [e for _, _, e in prompts[:B]]
            eng.regress_join(list(range(B)), [e.shape[0] for e in es], torch.cat(es), out)
            eng.regress_step(B, out)                       # the graph of this B is captured before the timed call
            return lambda: eng.regress_step(B, out)
        res["regress_step_ms"][str(B)] = timed(step, iters)
    eng.llm_reset()
    return res


class GapSpy:
    """wraps a DenoiseSlotScheduler's UNet step: per request, the wall time between two consecutive UNet steps it took part in"""

    def __init__(self, sched):
        self.sched, self.last, self.max_gap = sched, {}, 0.0
        inner = sched._unet_step

        def wrapped(B):
            inner(B)
            if sched.device.type == "cuda":
                torch.cuda.current_stream().synchronize()
            now = time.time()
            for r in sched._denoising():
                if id(r) in self.last:
                    self.max_gap = max(self.max_gap, now - self.last[id(r)])
                self.last[id(r)] = now
        sched._unet_step = wrapped

    def take(self):
        g, self.max_gap, self.last = self.max_gap, 0.0, {}
        return g


def pipeline(layers, slots, max_seq):
    import bench
    from emu_b200.emu2.diffusion import EmuVisualGeneration
    from emu_b200.emu2.scheduler import EulerDiscreteScheduler
    m = encoder(layers, slots, max_seq)
    pipe = EmuVisualGeneration(m, EulerDiscreteScheduler(), bench.emu2_unet_json(), EMU2_VAE)
    pipe._warned_unfiltered = True
    eng = pipe.engine
    g = torch.Generator(device="cuda").manual_seed(1)
    for prefix, shapes in (("unet.", bench.unet_param_shapes(pipe.unet_config)), ("vae.", vae_decoder_shapes(EMU2_VAE))):
        for k, shp in shapes:
            if k.endswith(".bias"):
                t = torch.zeros(shp, device="cuda", dtype=torch.bfloat16)
            elif len(shp) == 1:
                t = torch.ones(shp, device="cuda", dtype=torch.bfloat16)
            else:
                fan = 1
                for d in shp[1:]:
                    fan *= d
                t = (torch.randn(shp, generator=g, device="cuda") * fan ** -0.5).to(torch.bfloat16)
            eng.load_tensor(prefix + k, t)
            del t
    return pipe


def trace_run(args):
    from emu_b200 import serve
    from emu_b200.batching import DenoiseSlotScheduler
    rnd = random.Random(args.seed)
    arrivals = sorted(rnd.uniform(0, args.span) for _ in range(args.requests))
    reqs = [(t, [prompt(i)], dict(guidance_scale=3.0, num_inference_steps=rnd.choice([25, 50])))
            for i, t in enumerate(arrivals)]
    warm = [(0.0, [prompt(100 + i)], dict(guidance_scale=3.0, num_inference_steps=2)) for i in range(args.slots)]
    max_seq = PROMPT_WORDS + 3 + 64
    pipe, layers, tried = None, None, []
    for n in [args.llm_layers] + [n for n in (48, 40, 32) if n < args.llm_layers]:
        try:
            pipe = pipeline(n, args.slots, max_seq)
            scheds = {"continuous": DenoiseSlotScheduler(pipe, args.slots, 1024, 1024)}
            for R in args.encode_steps:
                scheds["encode_R%d" % R] = DenoiseSlotScheduler(pipe, args.slots, 1024, 1024, encode_steps=R)
            layers = n
            break
        except Exception as ex:                            # out of memory: fewer decoder layers
            tried.append({"llm_layers": n, "error": str(ex)[:200]})
            pipe = scheds = None
            torch.cuda.empty_cache()
    if pipe is None:
        return {"error": "the model did not fit", "tried": tried}
    spies = {k: GapSpy(s) for k, s in scheds.items()}
    workers = {"admission_batching": serve.BatchingWorker(pipe, "generate", lambda knobs: args.slots, 0.0, None, "gen-batching")}
    for k, s in scheds.items():
        workers[k] = serve.ContinuousWorker(pipe, args.slots, "gen-" + k, serve.generate_slot_request,
                                            (lambda sc: lambda p, n: sc)(s), "generate")
    rounds = {k: [] for k in workers}
    for k, w in workers.items():
        w.start()
    for _ in range(args.rounds):
        for k, w in workers.items():                       # one scheduler at a time: they share the engine
            if k in scheds:                                # a scheduler that regresses re-enters slot mode for its turn
                s = scheds[k]
                if s.encode_steps is not None:
                    s.engine.slots_begin(s.n_slots)
            try:
                run_round(w, warm)
                if k in spies:
                    spies[k].take()
                r = run_round(w, reqs)
            except Exception as ex:                        # a request failed (its answer carries no timing)
                r = {"error": "%s: %s" % (type(ex).__name__, ex)}
            r["max_unet_gap_s"] = spies[k].take() if k in spies else None
            rounds[k].append(r)
            print(k, json.dumps(r), file=sys.stderr, flush=True)
    for w in workers.values():
        w.stop()
        w.join(timeout=600)
    med = lambda xs: sorted(xs)[len(xs) // 2]
    return {"llm_layers": layers, "llm_max_seq": max_seq, "vit_layers": 1, "tried": tried,
            "requests": args.requests, "span_s": args.span, "slots": args.slots, "size": "1024x1024", "guidance": 3.0,
            "steps": [k["num_inference_steps"] for _, _, k in reqs], "rounds": rounds,
            "images_per_s": {k: med([r.get("images_per_s", 0.0) for r in v]) for k, v in rounds.items()},
            "latency_p50_s": {k: med([r.get("latency_p50_s", 0.0) for r in v]) for k, v in rounds.items()},
            "latency_p90_s": {k: med([r.get("latency_p90_s", 0.0) for r in v]) for k, v in rounds.items()},
            "max_unet_gap_s": {k: max(r["max_unet_gap_s"] for r in v) for k, v in rounds.items() if k in spies}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--micro", action="store_true")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--requests", type=int, default=12)
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--span", type=float, default=8.0)
    ap.add_argument("--slots", type=int, default=4)
    ap.add_argument("--encode-steps", default="8,64")
    ap.add_argument("--llm-layers", type=int, default=48)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    args.encode_steps = [int(x) for x in args.encode_steps.split(",") if x]
    if not torch.cuda.is_available():
        sys.exit("gen_encode_bench needs a CUDA device")
    name, power = card()
    res = {"tool": "gen_encode_bench", "card": name, "power_limit": power}
    res.update({"micro": micro(args.iters)} if args.micro else {"trace": trace_run(args)})
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
