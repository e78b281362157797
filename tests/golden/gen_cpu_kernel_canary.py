"""Generates tests/golden/cpu_kernel_canary.json — SHA-256 digests of the fp32 / bf16 CPU torch ops the oracles are built
from (linear, batched matmul, softmax, layer norm, the T5 norm, GELU, SiLU, the patch convolution), on seeded inputs at the
shapes of the Causal-Former and EVA ViT goldens.

The reference goldens (emu1_cformer_tiny.pt, emu1_tiny.pt, live_reference.pt) hold fp32 results of the reference modules,
which the oracles reproduce bit for bit only when the CPU runs the same kernels: MKL and ATen pick their vector code by
instruction set and vendor, so another CPU sums in another order and differs in the last bits.  tests/test_oracle_cpu.py
recomputes these ops: if every digest matches, the CPU reproduces the kernels that made the goldens and the oracle tests
demand bit equality; otherwise they hold the oracle to the fp32 reordering bound instead.

Run on a CPU where the reference goldens reproduce bit for bit:  python tests/golden/gen_cpu_kernel_canary.py
"""
import hashlib
import json
import os

import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "cpu_kernel_canary.json")


def canary_outputs():
    """name -> output tensor of one op on fixed seeded inputs"""
    g = torch.Generator().manual_seed(1234)
    r = lambda *s: torch.randn(*s, generator=g)
    x, w, b = r(2, 257, 1408), r(768, 1408) * 0.03, r(768)
    q, k = r(2, 12, 257, 64), r(2, 12, 32, 64)
    h = r(2, 197, 176)
    out = {}
    for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        xd, wd, bd, qd, kd = x.to(dt), w.to(dt), b.to(dt), q.to(dt), k.to(dt)
        out["linear_" + name] = F.linear(xd, wd)
        out["linear_bias_" + name] = F.linear(xd, wd, bd)
        s = torch.matmul(qd, kd.transpose(3, 2))
        out["matmul_" + name] = s
        p = F.softmax(s.float(), dim=-1).type_as(s)
        out["softmax_" + name] = p
        out["matmul_pv_" + name] = torch.matmul(p, kd)
        hd = h.to(dt)
        out["t5_norm_" + name] = hd * torch.rsqrt(hd.to(torch.float32).pow(2).mean(-1, keepdim=True) + 1e-6)
    out["layer_norm"] = F.layer_norm(h, (176,), r(176), r(176), 1e-6)
    out["gelu"] = F.gelu(h)
    out["silu"] = F.silu(h)
    out["conv_patch"] = F.conv2d(r(2, 3, 56, 56), r(176, 3, 14, 14) * 0.03, r(176), stride=14)
    return out


def digests():
    return {k: hashlib.sha256(v.contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()
            for k, v in canary_outputs().items()}


if __name__ == "__main__":
    with open(OUT, "w") as f:
        json.dump(digests(), f, indent=1, sort_keys=True)
    print("wrote", OUT)
