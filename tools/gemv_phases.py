"""Where the time of a decode-loop GEMV launch goes: per-CTA phase stamps (emu_debug_gemv_phases) for the four projections of
one LLaMA-33B decoder layer at tensor-parallel degree 1 / 2 / 8 shard sizes, launched as the PDL chain of a layer inside a
CUDA graph (distinct weights per layer so that nothing hits in L2) — plus the chain's time per layer."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from emu_b200 import _lib  # noqa: E402

H, F = 6656, 17920


def main():
    lib = _lib.load()
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 1       # batch rows (5 = the reference's default beam search)
    tps = [int(v) for v in sys.argv[2].split(",")] if len(sys.argv) > 2 else [1, 2, 8]
    print("batch rows = %d, EMU_GEMV_XBULK=%s" % (B, os.environ.get("EMU_GEMV_XBULK", "1")))
    for tp in tps:
        Hl = (52 + tp - 1) // tp * 128
        Fl = F // tp
        shapes = [("qkv", 3 * Hl, H, True, 0), ("o", H, Hl, False, 0), ("gate_up", 2 * Fl, H, True, 2), ("down", H, Fl, False, 0)]
        layers = 6
        Ws = [[torch.randn(n, k, device="cuda", dtype=torch.bfloat16) * 0.02 for _, n, k, _, _ in shapes] for _ in range(layers)]
        xh = torch.randn(B, H, device="cuda", dtype=torch.bfloat16)
        xs = {H: xh, Hl: torch.randn(B, Hl, device="cuda", dtype=torch.bfloat16), Fl: torch.randn(B, Fl, device="cuda", dtype=torch.bfloat16)}
        nw = torch.ones(H, device="cuda", dtype=torch.bfloat16)
        outs = {n: torch.empty(B, n, device="cuda", dtype=torch.bfloat16) for _, n, _, _, _ in shapes}
        outs[Fl] = torch.empty(B, Fl, device="cuda", dtype=torch.bfloat16)
        stamps = [[torch.zeros(2 * 132, 8, dtype=torch.int64, device="cuda") for _ in shapes] for _ in range(layers)]

        def run():
            for l in range(layers):
                for j, (name, n, k, norm, mode) in enumerate(shapes):
                    n_out = n // 2 if mode == 2 else n
                    _lib.check(lib.emu_debug_gemv_phases(_lib._ptr(Ws[l][j]), n, k, _lib._ptr(xs[k]), k, B,
                                                         _lib._ptr(nw if norm else None), _lib.C.c_float(1e-6), mode, None, 0,
                                                         _lib._ptr(outs[n_out]), n_out, 1, _lib._ptr(stamps[l][j]),
                                                         _lib._stream()))
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            run()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=st):
                run()
            g.replay()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
        us_layer = e0.elapsed_time(e1) / (5 * layers) * 1000.0
        nbytes = sum(n * k * 2 for _, n, k, _, _ in shapes)
        print("== TP%d shard: chain %.1f us per layer (4 GEMVs), %.0f GB/s; pure streaming at 6.48 TB/s = %.1f us"
              % (tp, us_layer, nbytes / us_layer / 1e3, nbytes / 6.4846e6), flush=True)
        print("   %-8s %6s %6s | ideal us | median CTA cycles: init  dep-wait  x-stage  first-chunk  consume+flush  tail | start gap us (entry - previous kernel's last exit)" % ("gemv", "N", "K"))
        prev_end = None
        l = layers - 1
        for j, (name, n, k, norm, mode) in enumerate(shapes):
            s = stamps[l][j].cpu()
            s = s[s[:, 1] > 0].double()
            d = lambda a, b: float((s[:, a] - s[:, b]).median())
            dur_cyc = float((s[:, 7] - s[:, 1]).median())
            start_ns = float(s[:, 0].median())
            gap = (start_ns - prev_end) / 1000.0 if prev_end is not None else float("nan")
            # estimate this kernel's end in globaltimer terms: entry + duration at ~1.9 GHz
            prev_end = float(s[:, 0].max()) + float((s[:, 7] - s[:, 1]).max()) / 1.9
            print("   %-8s %6d %6d | %7.1f | %6.0f %8.0f %8.0f %10.0f %12.0f %6.0f | total %6.0f cyc, gap %.1f us"
                  % (name, n, k, n * k * 2 / 6.4846e6, d(2, 1), d(3, 2), d(4, 3), d(5, 4), d(6, 5), d(7, 6), dur_cyc, gap), flush=True)


if __name__ == "__main__":
    main()
