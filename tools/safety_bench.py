"""Milliseconds per safety check (emu_safety_check: CLIP pre-processing, ViT-L/14 tower, scores, black-out) on 1024 x 1024 uint8
images, for B = 1 and 4, timed with CUDA events; seeded random weights in the published shapes.  Prints one JSON line with the
card's name and power limit next to the times and the shape-derived lower bounds (FLOP at the data sheet's dense BF16 rate,
weight bytes at its HBM bandwidth).

    python tools/safety_bench.py [--iters 50] [--warmup 5] [--out results/safety_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_BF16, PEAK_HBM = 989e12, 3.35e12   # H100 SXM data sheet (dense BF16, HBM3); a bound, not a measurement


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in q.split(",")]
        return name, pl
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def flops_per_image(W=1024, L=24, M=4096, N=257, proj=768, P=14):
    lin = 2 * N * (3 * W * W + W * W + 2 * W * M) * L + 2 * 256 * 3 * P * P * W + 2 * W * proj
    attn = 2 * 2 * N * N * W * L
    return lin, attn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    from emu_b200 import _lib
    from emu_b200.safety import SafetyChecker
    assert torch.cuda.is_available(), "safety_bench needs a GPU"
    ck = SafetyChecker()
    g = torch.Generator().manual_seed(0)
    from oracle.safety_oracle import param_shapes
    n_param = 0
    for k, shp in param_shapes().items():
        t = torch.randn(shp, generator=g) * (0.02 if len(shp) > 1 else 0.05)
        if k.endswith("_weights"):
            t = t.abs() + 0.2
        ck.load_tensor(k, t.to(torch.bfloat16))
        n_param += t.numel()
    res = {}
    for B in (1, 4):
        imgs = torch.randint(0, 256, (B, 1024, 1024, 3), dtype=torch.uint8, device="cuda")
        work = imgs.clone()
        for _ in range(a.warmup):
            work.copy_(imgs)
            ck.check_device(work)
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        ck.check_device(work)
        launches = _lib.launch_count() - n0
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(a.iters):
            ck.check_device(work)
        ev1.record()
        torch.cuda.synchronize()
        res["B%d" % B] = dict(ms_per_check=ev0.elapsed_time(ev1) / a.iters, launches_per_check=launches)
    lin, attn = flops_per_image()
    name, pl = card()
    out = dict(tool="safety_bench", card=name, power_limit=pl, image="1024x1024 uint8", iters=a.iters, results=res,
               gflop_per_image=dict(projections=lin / 1e9, attention=attn / 1e9),
               bound_ms_compute_per_image=(lin + attn) / PEAK_BF16 * 1e3,
               bound_ms_weights=n_param * 2 / PEAK_HBM * 1e3,
               bounds_note="H100 SXM data-sheet peaks (989 TFLOP/s dense BF16, 3.35 TB/s); not measured")
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
