"""Where the time of a wgmma GEMM launch goes: per-CTA phase stamps (emu_debug_gemm_phases) on the UNet / ViT shapes, plus
the launch-to-launch time of the same GEMM replayed inside a CUDA graph (no host launch overhead, L2-warm like the model)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from emu_b200 import _lib  # noqa: E402

SHAPES = [  # name, M, N, K, epi (-1 = bias + residual)
    ("L2 attn o +res", 2048, 1280, 1280, -1),
    ("L2 q (plain)", 2048, 1280, 1280, 0),
    ("L2 qkv", 2048, 3840, 1280, 0),
    ("L2 geglu ff1", 2048, 10240, 1280, _lib.EPI_GEGLU),
    ("L2 ff2 +res", 2048, 1280, 5120, -1),
    ("L1 attn o +res", 8192, 640, 640, -1),
    ("L1 qkv", 8192, 1920, 640, 0),
    ("L1 geglu ff1", 8192, 5120, 640, _lib.EPI_GEGLU),
    ("L1 ff2 +res", 8192, 640, 2560, -1),
    ("vit fc1 gelu", 1025, 15360, 1792, _lib.EPI_GELU),
]


def graph_time(fn, reps=20):
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
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
    return e0.elapsed_time(e1) / (5 * reps) * 1000.0  # us per launch


def main():
    gen = torch.Generator(device="cuda").manual_seed(0)
    print("%-18s %5s %5s %5s | graph us/launch  TFLOP/s | median CTA cycles: setup  first-TMA  fill  mainloop  epi-wait  epilogue | total us @clk" % ("shape", "M", "N", "K"))
    for name, M, N, K, epi in SHAPES:
        A = (torch.randn(M, K, generator=gen, device="cuda") * 0.1).to(torch.bfloat16)
        W = (torch.randn(N, K, generator=gen, device="cuda") * 0.1).to(torch.bfloat16)
        bias = res = None
        e = epi
        n_out = N // 2 if epi in (_lib.EPI_GEGLU, _lib.EPI_SWIGLU) else N
        if epi == -1:
            bias = torch.randn(N, generator=gen, device="cuda").to(torch.bfloat16)
            res = torch.randn(M, N, generator=gen, device="cuda").to(torch.bfloat16)
            e = 0
        out = torch.empty(M, n_out, dtype=torch.bfloat16, device="cuda")
        lib = _lib.load()

        def run():
            _lib.check(lib.emu_op_gemm(_lib._ptr(A), K, _lib._ptr(W), K, M, N, K, _lib._ptr(bias), _lib._ptr(res),
                                       N if res is not None else 0, e, _lib._ptr(out), n_out, 0, 0, _lib._stream()))
        us = graph_time(run)
        for _ in range(2):
            _, st = _lib.debug_gemm_phases(A, W, bias=bias, residual=res, epi=e)
        torch.cuda.synchronize()
        st = st[st[:, 1] > 0].double()
        d = lambda a, b: float((st[:, a] - st[:, b]).median())
        total_ns = float((st[:, 0].max() - st[:, 0].min()))
        print("%-18s %5d %5d %5d | %8.2f  %8.1f | %6.0f %6.0f %6.0f %8.0f %6.0f %8.0f | ctas %d entry-skew %.1f us"
              % (name, M, N, K, us, 2.0 * M * N * K / us / 1e6, d(2, 1), d(3, 2), d(4, 3), d(5, 4), d(6, 5), d(7, 6), st.shape[0],
                 total_ns / 1000.0), flush=True)


if __name__ == "__main__":
    main()
