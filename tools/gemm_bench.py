"""Micro-benchmark of the wgmma GEMM / implicit-GEMM conv on the hot-path shapes (UNet levels, ViT, LLaMA prefill).
CUDA events, 3 warm-ups, 20 timed launches back to back (weights + activations of one launch fit L2 for the small shapes)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from emu_b200 import _lib  # noqa: E402

GEMMS = [  # name, M, N, K, epi  (epi -1 = bias + residual epilogue)
    ("unet L2 attn q/o (1024 tok x2)", 2048, 1280, 1280, 0),
    ("unet L2 attn o +bias+residual", 2048, 1280, 1280, -1),
    ("unet L2 ff2 +bias+residual", 2048, 1280, 5120, -1),
    ("unet L1 attn o +bias+residual", 8192, 640, 640, -1),
    ("unet L2 qkv", 2048, 3840, 1280, 0),
    ("unet L2 geglu ff1", 2048, 10240, 1280, _lib.EPI_GEGLU),
    ("unet L2 ff2", 2048, 1280, 5120, 0),
    ("unet L1 attn q/o (4096 tok x2)", 8192, 640, 640, 0),
    ("unet L1 qkv", 8192, 1920, 640, 0),
    ("unet L1 geglu ff1", 8192, 5120, 640, _lib.EPI_GEGLU),
    ("unet L1 ff2", 8192, 640, 2560, 0),
    ("vit qkv (1025 tok)", 1025, 5376, 1792, 0),
    ("vit proj", 1025, 1792, 1792, 0),
    ("vit fc1 gelu", 1025, 15360, 1792, _lib.EPI_GELU),
    ("vit fc2", 1025, 1792, 15360, 0),
    ("llama prefill qkv (4096 tok)", 4096, 19968, 6656, 0),
    ("llama prefill down", 4096, 6656, 17920, 0),
]
CONVS = [  # name, NB, H, W, Cin, Cout
    ("unet conv L0 320->320 @128", 2, 128, 128, 320, 320),
    ("unet conv L1 640->640 @64", 2, 64, 64, 640, 640),
    ("unet conv L2 1280->1280 @32", 2, 32, 32, 1280, 1280),
    ("unet conv up L2 2560->1280 @32", 2, 32, 32, 2560, 1280),
    ("unet conv up L1 1280->640 @64", 2, 64, 64, 1280, 640),
    ("unet conv up L0 640->320 @128", 2, 128, 128, 640, 320),
]


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, M, N, K, epi in GEMMS:
        A = (torch.randn(M, K, generator=g, device="cuda") * 0.1).to(torch.bfloat16)
        W = (torch.randn(N, K, generator=g, device="cuda") * 0.1).to(torch.bfloat16)
        if epi == -1:
            bias = torch.randn(N, generator=g, device="cuda").to(torch.bfloat16)
            res = torch.randn(M, N, generator=g, device="cuda").to(torch.bfloat16)
            ms = timeit(lambda: _lib.op_gemm(A, W, bias=bias, residual=res))
            print("%-36s M=%5d N=%5d K=%5d  %7.3f ms %7.1f TFLOP/s" % (name, M, N, K, ms, 2.0 * M * N * K / ms / 1e9), flush=True)
            continue
        ms = timeit(lambda: _lib.op_gemm(A, W, epi=epi))
        extra = ""
        if os.environ.get("GEMM_BENCH_SWEEP"):
            for bn in (64, 96, 128, 160, 192, 224, 256):
                t = timeit(lambda: _lib.op_gemm(A, W, epi=epi, force_bn=bn))
                extra += " bn%d=%.1fus" % (bn, t * 1000)
        print("%-36s M=%5d N=%5d K=%5d  %7.3f ms %7.1f TFLOP/s%s" % (name, M, N, K, ms, 2.0 * M * N * K / ms / 1e9, extra),
              flush=True)
    for name, NB, H, Wd, Cin, Cout in CONVS:
        x = (torch.randn(NB, H, Wd, Cin, generator=g, device="cuda") * 0.1).to(torch.bfloat16)
        w = (torch.randn(Cout, 9 * Cin, generator=g, device="cuda") * 0.02).to(torch.bfloat16)
        ms = timeit(lambda: _lib.op_conv3x3(x, w))
        fl = 2.0 * NB * H * Wd * Cout * 9 * Cin
        print("%-36s M=%5d N=%5d K=%5d  %7.3f ms %7.1f TFLOP/s" % (name, NB * H * Wd, Cout, 9 * Cin, ms, fl / ms / 1e9), flush=True)


if __name__ == "__main__":
    main()
