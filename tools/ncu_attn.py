"""Tiny driver for `ncu --set full` on the wgmma attention kernel: python tools/ncu_attn.py B N H D [causal]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from emu_b200 import _lib  # noqa: E402

B, N, H, D = (int(v) for v in sys.argv[1:5])
causal = len(sys.argv) > 5 and sys.argv[5] == "1"
qkv = (torch.randn(B, N, 3, H, D, device="cuda") * 0.5).to(torch.bfloat16)
for _ in range(4):
    _lib.op_attn_prefill(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], D ** -0.5, causal=causal)
torch.cuda.synchronize()
