"""emu_vae_decode time for the Emu2-Gen VAE decoder (SDXL AutoencoderKL, 128/256/512/512, random-init weights) at 128 x 128
latents -> 1024 x 1024 images, B = 1 and 4, from CUDA events after warm-up.  Prints one JSON line with the per-batch median
and min over the timed repeats, the sha1 of the B = 1 image, and the card's name and power limit read in the same call.
--lib times another build of libemu_b200.so (same C ABI), so two builds can be run alternately on the same card.

    python tools/vae_decode_bench.py [--batches 1,4] [--warmup 2] [--iters 5] [--lib path/to/libemu_b200.so]
"""
import argparse
import hashlib
import json
import os
import statistics
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,4")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--lib", default=None, help="another build of libemu_b200.so to time instead of the in-tree one")
    args = ap.parse_args()
    from emu_b200 import _lib
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    from emu_b200.emu2.diffusion import vae_config_from_json
    from gen_batching_bench import EMU2_VAE, card, vae_decoder_shapes
    eng = _lib.Engine(_lib.EmuConfig())
    eng.vae_configure(vae_config_from_json(EMU2_VAE))
    g = torch.Generator(device="cuda").manual_seed(1)
    for k, shp in vae_decoder_shapes(EMU2_VAE):
        if len(shp) == 1:
            t = (0.05 * torch.randn(shp, generator=g, device="cuda")) if k.endswith(".bias") else \
                (1 + 0.1 * torch.randn(shp, generator=g, device="cuda"))
        else:
            fan = 1
            for d in shp[1:]:
                fan *= d
            t = torch.randn(shp, generator=g, device="cuda") * fan ** -0.5
        eng.load_tensor("vae." + k, t.to(torch.bfloat16))
    name, power = card()
    res = {"tool": "vae_decode_bench", "lib": args.lib or "in-tree", "card": name, "power_limit": power, "latent_hw": 128,
           "ms": {}}
    for B in [int(b) for b in args.batches.split(",")]:
        z = torch.randn(B, 4, 128, 128, generator=torch.Generator(device="cuda").manual_seed(2), device="cuda")
        z = z.to(torch.bfloat16)
        for _ in range(args.warmup):
            img = eng.vae_decode(z)
        times = []
        for _ in range(args.iters):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            img = eng.vae_decode(z)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        res["ms"][str(B)] = {"median": statistics.median(times), "min": min(times)}
        if B == 1:
            res["image_sha1"] = hashlib.sha1(img.cpu().numpy().tobytes()).hexdigest()[:16]
            res["finite"] = bool(torch.isfinite(img).all())
    eng.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
