"""Tiny driver for `ncu --set full` on one wgmma GEMM shape: python tools/ncu_gemm.py M N K [force_bn] [epi]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from emu_b200 import _lib  # noqa: E402

M, N, K = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3])
bn = int(sys.argv[4]) if len(sys.argv) > 4 else 0
epi = int(sys.argv[5]) if len(sys.argv) > 5 else 0
A = (torch.randn(M, K, device="cuda") * 0.1).to(torch.bfloat16)
W = (torch.randn(N, K, device="cuda") * 0.1).to(torch.bfloat16)
for _ in range(4):
    _lib.op_gemm(A, W, epi=epi, force_bn=bn)
torch.cuda.synchronize()
