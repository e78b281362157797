"""Admission batching vs continuous batching for image generation on one GPU: a seeded trace of 1024 x 1024 requests (arrivals
spread over --span seconds, num_inference_steps from {25, 50}, guidance 3.0) run through serve.BatchingWorker and a
serve.ContinuousWorker driving a DenoiseSlotScheduler, alternating, on the Emu2-Gen UNet and VAE decoder with random-init
weights like bench.make_unet_engine.  Requests carry random conditioning: prompt encoding is excluded (the LLaMA-33B encoder,
64.6 GB, and the ViT, 8.7 GB, next to the 5.05 GB UNet leave almost nothing of 80 GB for UNet workspaces at 8 rows), and so is
the safety checker.  Prints one JSON line: images/s and p50 / p90 request latency per scheduler and round, the slot step time
at B = 1..n_slots (CUDA events), the time one retirement (VAE decode + uint8 + copy to the host) stalls the live slots, and
the card's name and power limit read in the same call.

    python tools/gen_batching_bench.py [--requests 12] [--rounds 2] [--span 8.0] [--slots 4] [--out results/gen_batching.json]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import threading
import time
from types import SimpleNamespace as NS

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

EMU2_VAE = dict(latent_channels=4, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                norm_num_groups=32, scaling_factor=0.13025)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in q.split(",")]
        return name, pl
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def vae_decoder_shapes(cfg):
    """(key, shape) of the AutoencoderKL decoder half, diffusers naming"""
    boc, lpb, lc = cfg["block_out_channels"], cfg["layers_per_block"], cfg["latent_channels"]
    out = []
    cv = lambda p, o, i, k=3: out.extend([(p + ".weight", (o, i, k, k)), (p + ".bias", (o,))])
    nrm = lambda p, c: out.extend([(p + ".weight", (c,)), (p + ".bias", (c,))])

    def resnet(p, cin, cout):
        nrm(p + "norm1", cin); cv(p + "conv1", cout, cin); nrm(p + "norm2", cout); cv(p + "conv2", cout, cout)
        if cin != cout:
            cv(p + "conv_shortcut", cout, cin, 1)
    top = boc[-1]
    cv("post_quant_conv", lc, lc, 1)
    cv("decoder.conv_in", top, lc)
    resnet("decoder.mid_block.resnets.0.", top, top)
    nrm("decoder.mid_block.attentions.0.group_norm", top)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        out.extend([("decoder.mid_block.attentions.0.%s.weight" % n, (top, top)), ("decoder.mid_block.attentions.0.%s.bias" % n, (top,))])
    resnet("decoder.mid_block.resnets.1.", top, top)
    cin = top
    rev = list(reversed(boc))
    for i, cout in enumerate(rev):
        for j in range(lpb + 1):
            resnet("decoder.up_blocks.%d.resnets.%d." % (i, j), cin, cout)
            cin = cout
        if i < len(rev) - 1:
            cv("decoder.up_blocks.%d.upsamplers.0.conv" % i, cout, cout)
    nrm("decoder.conv_norm_out", boc[0])
    cv("decoder.conv_out", cfg["out_channels"], boc[0])
    return out


def make_pipeline(L=64):
    """EmuVisualGeneration over the real-shape UNet + VAE decoder; `inputs` = ["<name>"] -> random conditioning"""
    import bench
    from emu_b200.emu2.diffusion import EmuVisualGeneration, vae_config_from_json
    from emu_b200.emu2.scheduler import EulerDiscreteScheduler
    eng, ucfg = bench.make_unet_engine(seed=0)
    eng.vae_configure(vae_config_from_json(EMU2_VAE))
    g = torch.Generator(device="cuda").manual_seed(1)
    for k, shp in vae_decoder_shapes(EMU2_VAE):
        if len(shp) == 1:
            t = torch.zeros(shp, device="cuda") if k.endswith(".bias") else torch.ones(shp, device="cuda")
        else:
            fan = 1
            for d in shp[1:]:
                fan *= d
            t = torch.randn(shp, generator=g, device="cuda") * fan ** -0.5
        eng.load_tensor("vae." + k, t.to(torch.bfloat16))
    p = EmuVisualGeneration.__new__(EmuVisualGeneration)
    p.engine, p.unet_config, p.vae_config = eng, ucfg, EMU2_VAE
    p.scheduler = EulerDiscreteScheduler()
    p.vae_scale_factor, p.vae_scaling = 8, EMU2_VAE["scaling_factor"]
    p.multimodal_encoder, p.device_ = NS(n_query=L), "cuda"
    p.safety_checker, p._warned_unfiltered, p.negative_prompt = None, True, {}

    def encode(inputs, do_cfg):
        gg = torch.Generator(device="cuda").manual_seed(sum(map(ord, inputs[0])))
        return torch.randn(2 if do_cfg else 1, L, ucfg["cross_attention_dim"], generator=gg, device="cuda")
    p._prepare_and_encode_inputs = encode
    return p


def trace(n, span, seed):
    rnd = random.Random(seed)
    arrivals = sorted(rnd.uniform(0, span) for _ in range(n))
    return [(t, ["request-%d" % i], dict(guidance_scale=3.0, num_inference_steps=rnd.choice([25, 50])))
            for i, t in enumerate(arrivals)]


def run_round(worker, reqs):
    lat = [None] * len(reqs)
    t0 = time.time()

    def one(i):
        at, inputs, knobs = reqs[i]
        time.sleep(max(0.0, t0 + at - time.time()))
        t_in = time.time()
        worker.submit(inputs, dict(knobs), "r%d" % i)
        lat[i] = (t_in, time.time())
    ts = [threading.Thread(target=one, args=(i,)) for i in range(len(reqs))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    torch.cuda.synchronize()
    wall = max(b for _, b in lat) - min(a for a, _ in lat)
    ls = sorted(b - a for a, b in lat)
    pct = lambda q: ls[min(len(ls) - 1, int(round(q * (len(ls) - 1))))]
    return {"images_per_s": len(reqs) / wall, "wall_s": wall, "latency_p50_s": pct(0.5), "latency_p90_s": pct(0.9)}


def slot_step_times(sched, reps=5):
    out = {}
    live = torch.zeros(sched.n_slots, dtype=torch.int32, device="cuda")   # dead slots cost the same UNet rows as live ones
    for B in range(1, sched.n_slots + 1):
        for _ in range(2):                          # eager, then the graph capture
            sched.engine.denoise_step_slots(sched.latents, sched.params, live, sched.ctx, sched.text_embeds, sched.time_ids, B)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            sched.engine.denoise_step_slots(sched.latents, sched.params, live, sched.ctx, sched.text_embeds, sched.time_ids, B)
        e1.record()
        torch.cuda.synchronize()
        out[str(B)] = e0.elapsed_time(e1) / reps
    return out


def retire_ms(pipe, sched, reps=3):
    lat = sched.latents[:1].clone()
    pipe.decode_and_check(lat)
    torch.cuda.synchronize()
    t = time.time()
    for _ in range(reps):
        pipe.decode_and_check(lat)
    return (time.time() - t) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=12)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--span", type=float, default=8.0)
    ap.add_argument("--slots", type=int, default=4)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", type=str, default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gen_batching_bench needs a CUDA device")
    from emu_b200 import serve
    from emu_b200.batching import DenoiseSlotScheduler
    name, power = card()
    pipe = make_pipeline()
    sched = DenoiseSlotScheduler(pipe, args.slots, 1024, 1024)
    steps_ms = slot_step_times(sched)
    stall = retire_ms(pipe, sched)
    make = {"batching": lambda: serve.BatchingWorker(pipe, "generate", lambda knobs: args.slots, 0.0, None, "gen-batching"),
            "continuous": lambda: serve.ContinuousWorker(pipe, args.slots, "gen-continuous", serve.generate_slot_request,
                                                         lambda p, n: sched, "generate")}
    reqs = trace(args.requests, args.span, args.seed)
    warm = [(0.0, ["warm-%d" % i], dict(guidance_scale=3.0, num_inference_steps=s)) for i, s in enumerate((2, 3, 2, 3))]
    rounds = {"batching": [], "continuous": []}
    workers = {}
    for mode in ("batching", "continuous"):
        workers[mode] = make[mode]()
        workers[mode].start()
        run_round(workers[mode], warm)              # every batch size's graph captured before the timed rounds
    for _ in range(args.rounds):
        for mode in ("batching", "continuous"):
            rounds[mode].append(run_round(workers[mode], reqs))
    for w in workers.values():
        w.stop()
        w.join(timeout=600)
    med = lambda xs: sorted(xs)[len(xs) // 2]
    res = {
        "tool": "gen_batching_bench", "card": name, "power_limit": power,
        "trace": {"requests": args.requests, "span_s": args.span, "steps": [k["num_inference_steps"] for _, _, k in reqs],
                  "guidance": 3.0, "size": "1024x1024", "slots": args.slots, "seed": args.seed},
        "excluded": "prompt encoding (random conditioning) and the safety checker: UNet + VAE decoder + uint8 only",
        "admission_stall": "not measured (prompt encoding excluded)",
        "rounds": rounds,
        "images_per_s": {m: med([r["images_per_s"] for r in rounds[m]]) for m in rounds},
        "slot_step_ms": steps_ms,
        "retire_stall_ms": stall,
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
