"""Micro-benchmark of emu_op_attn_prefill on the hot-path shapes (run twice: default = wgmma kernel, EMU_ATTN=legacy =
mma.sync kernel).  CUDA events, 3 warm-ups, inputs re-used (they fit L2 for the small shapes; stated in the output)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from emu_b200 import _lib  # noqa: E402

SHAPES = [  # name, B, N, H, D, causal
    ("vit_448 (EVA-CLIP-E)", 1, 1025, 16, 112, False),
    ("unet_64x64 (SDXL level 1, CFG)", 2, 4096, 10, 64, False),
    ("unet_32x32 (SDXL level 2, CFG)", 2, 1024, 20, 64, False),
    ("llama33b prefill 4k causal", 1, 4096, 52, 128, True),
    ("llama33b prefill 1k causal", 1, 1024, 52, 128, True),
]
CROSS = [  # name, B, Nq, Nk, H, D   (UNet cross-attention over the 64 regressed visual tokens)
    ("unet_64x64 cross-attn 64 keys", 2, 4096, 64, 10, 64),
    ("unet_32x32 cross-attn 64 keys", 2, 1024, 64, 20, 64),
]


def graph_us(fn, reps=20):
    """launch-to-launch time inside a CUDA graph (no host launch overhead; inputs stay in L2 like inside the model)"""
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for _ in range(reps):
                fn()
        g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (5 * reps) * 1000.0


def main():
    g = torch.Generator().manual_seed(0)
    for name, B, N, H, D, causal in SHAPES:
        qkv = (torch.randn(B, N, 3, H, D, generator=g) * 0.5).to(torch.bfloat16).cuda()
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
        for _ in range(3):
            _lib.op_attn_prefill(q, k, v, D ** -0.5, causal=causal)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = 20
        e0.record()
        for _ in range(iters):
            _lib.op_attn_prefill(q, k, v, D ** -0.5, causal=causal)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        flops = 4.0 * B * H * N * N * D * (0.5 if causal else 1.0)
        out = torch.empty(B, N, H, D, dtype=torch.bfloat16, device="cuda")
        us = graph_us(lambda: _lib.op_attn_prefill(q, k, v, D ** -0.5, causal=causal))
        print("%-34s %8.3f ms  %7.1f TFLOP/s | in-graph %8.1f us %7.1f TFLOP/s  [%s]"
              % (name, ms, flops / ms / 1e9, us, flops / us / 1e6, os.environ.get("EMU_ATTN", "wgmma")), flush=True)
    for name, B, Nq, Nk, H, D in CROSS:
        q = (torch.randn(B, Nq, H, D, generator=g) * 0.5).to(torch.bfloat16).cuda()
        kv = (torch.randn(B, Nk, 2, H, D, generator=g) * 0.5).to(torch.bfloat16).cuda()
        us = graph_us(lambda: _lib.op_attn_prefill(q, kv[:, :, 0], kv[:, :, 1], D ** -0.5))
        flops = 4.0 * B * H * Nq * Nk * D
        print("%-34s in-graph %8.1f us %7.1f TFLOP/s" % (name, us, flops / us / 1e6), flush=True)


if __name__ == "__main__":
    main()
