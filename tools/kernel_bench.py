"""Micro-benchmark of the decode-loop kernels at the LLaMA-33B shapes (run on the GPU box).

Each GEMV shape is timed with CUDA events over a ring of distinct weight buffers (> 126 MB L2 in total, so every
launch streams from HBM like the real decode loop), alone and as the PDL-chained sequence of one decoder layer.
"""
import json
import sys
import os

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from emu_b200 import _lib  # noqa: E402


def time_gemv(N, K, B, mode=0, norm=False, residual=False, iters=40, pdl=False):
    nbuf = max(2, int(600e6 // (N * K * 2)) + 1)
    Ws = [torch.randn(N, K, device="cuda", dtype=torch.bfloat16) * 0.02 for _ in range(nbuf)]
    x = torch.randn(B, K, device="cuda", dtype=torch.bfloat16)
    nw = torch.ones(K, device="cuda", dtype=torch.bfloat16) if norm else None
    n_out = N // 2 if mode == 2 else N
    r = torch.randn(B, n_out, device="cuda", dtype=torch.bfloat16) if residual else None
    for i in range(5):
        _lib.op_gemv(Ws[i % nbuf], x, norm_w=nw, mode=mode, residual=r, pdl=pdl)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for i in range(iters):
        _lib.op_gemv(Ws[i % nbuf], x, norm_w=nw, mode=mode, residual=r, pdl=pdl)
    ev1.record()
    torch.cuda.synchronize()
    us = ev0.elapsed_time(ev1) * 1000 / iters
    return us, N * K * 2 / us / 1e3  # GB/s


def main():
    H, F, V = 6656, 17920, 32272
    out = {}
    for B in (1, 5, 8):
        for name, (N, K, mode, norm, res) in {
            "qkv": (3 * H, H, 0, True, False), "o": (H, H, 0, False, True), "gate_up": (2 * F, H, 2, True, False),
            "down": (H, F, 0, False, True), "lm_head": (V, H, 0, True, False)}.items():
            for pdl in (False, True):
                us, gbs = time_gemv(N, K, B, mode, norm, res, pdl=pdl)
                out["%s_B%d_%s" % (name, B, "pdl" if pdl else "plain")] = {"us": round(us, 2), "GBps": round(gbs, 1)}
                print(name, B, pdl, "%.1f us  %.0f GB/s" % (us, gbs), flush=True)
    json.dump(out, open("gpurun_out/kernel_bench.json", "w"), indent=1)


if __name__ == "__main__":
    main()


def chain_bench(B=1, layers=8, iters=5):
    """One decoder layer's four GEMVs back to back (PDL chained), distinct weights per layer so nothing hits in L2."""
    H, F = 6656, 17920
    Ws = []
    for _ in range(layers):
        Ws.append([torch.randn(3 * H, H, device="cuda", dtype=torch.bfloat16) * 0.02,
                   torch.randn(H, H, device="cuda", dtype=torch.bfloat16) * 0.02,
                   torch.randn(2 * F, H, device="cuda", dtype=torch.bfloat16) * 0.02,
                   torch.randn(H, F, device="cuda", dtype=torch.bfloat16) * 0.02])
    x = torch.randn(B, H, device="cuda", dtype=torch.bfloat16)
    xf = torch.randn(B, F, device="cuda", dtype=torch.bfloat16)
    nw = torch.ones(H, device="cuda", dtype=torch.bfloat16)

    def run():
        for w in Ws:
            _lib.op_gemv(w[0], x, norm_w=nw, pdl=True)
            _lib.op_gemv(w[1], x, residual=x, pdl=True)
            _lib.op_gemv(w[2], x, norm_w=nw, mode=2, pdl=True)
            _lib.op_gemv(w[3], xf, residual=x, pdl=True)
    run()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(iters):
        run()
    ev1.record()
    torch.cuda.synchronize()
    us = ev0.elapsed_time(ev1) * 1000 / (iters * layers)
    nbytes = 2 * (4 * H * H + 3 * H * F)
    print("chain B=%d: %.1f us per layer (4 GEMVs), %.0f GB/s" % (B, us, nbytes / us / 1e3), flush=True)


if __name__ == "__main__" and os.environ.get("EMU_CHAIN", "1") == "1":
    chain_bench(1)
    chain_bench(5)
    chain_bench(8)
