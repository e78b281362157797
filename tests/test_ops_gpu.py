"""Kernel parity: every CUDA operator, called through the C ABI, against the CPU oracle on the same seeded inputs.

Tolerances (relative max-abs error, oracle.emu_oracle.rel_err):
  * fp32 outputs (logits)      : 1e-3   (north_star tolerance; observed ~1e-6: same bf16 inputs, fp32 accumulate)
  * bf16 outputs               : 6e-3   (one bf16 rounding of the largest element is 2^-9 = 2e-3)
"""
import math

import pytest
import torch

from oracle import emu_oracle as O

pytestmark = pytest.mark.gpu

TOL_F32 = 1e-3
TOL_BF16 = 6e-3


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(torch.bfloat16)


@pytest.mark.parametrize("M,N,K,bn", [
    (128, 128, 64, 128), (1, 64, 64, 64), (75, 320, 192, 0), (1025, 5376, 1792, 0), (300, 1000, 584, 64),
    (257, 768, 1408, 128), (4096, 640, 640, 256), (64, 6656, 1792, 0), (513, 264, 72, 0),
    (2048, 1280, 1280, 0), (2048, 1280, 640, 160), (300, 1000, 584, 96), (700, 900, 320, 192), (257, 1344, 256, 224),
    # 2048 = force the 2-CTA cluster (W tile TMA-multicast), 1024 = force it off; ragged / odd tile-row counts included
    (2048, 1280, 1280, 2048 + 160), (2048, 1280, 1280, 1024 + 160), (385, 520, 448, 2048 + 128), (1025, 1792, 1792, 2048),
    (100, 200, 136, 2048 + 64), (4096, 640, 640, 2048 + 256),
])
def test_gemm_plain(cuda, M, N, K, bn):
    from emu_b200 import _lib
    A, W = _rand((M, K), 1), _rand((N, K), 2, 0.05)
    ref = O.op_linear(A, W)
    out32 = _lib.op_gemm(A.cuda(), W.cuda(), out_fp32=True, force_bn=bn).cpu()
    assert O.rel_err(out32, ref) < TOL_F32
    out16 = _lib.op_gemm(A.cuda(), W.cuda(), force_bn=bn).cpu()
    assert O.rel_err(out16, ref) < TOL_BF16


@pytest.mark.parametrize("M,N,K", [(200, 384, 256), (2048, 1280, 1280), (700, 1000, 320), (4100, 640, 192), (129, 72, 64)])
@pytest.mark.parametrize("bn", [0, 64, 96, 128, 160, 192, 4096 + 160, 256])
def test_gemm_staged_epilogue(cuda, M, N, K, bn):
    """bf16 outputs leave through shared memory + TMA stores and the residual arrives by TMA load (bn <= 192); bn = 256 and
    4096 + bn (forced) take the direct register path.  Every epilogue flavour, ragged M / N, several tiles per CTA, and the
    in-place form x = x + lin(a) that the models use."""
    from emu_b200 import _lib
    A, W, b, r = _rand((M, K), 11), _rand((N, K), 12, 0.05), _rand((N,), 13), _rand((M, N), 14)
    lin = O.op_linear(A, W, b)
    bf = lambda t: t.to(torch.bfloat16)
    Ac, Wc, bc = A.cuda(), W.cuda(), b.cuda()
    assert O.rel_err(_lib.op_gemm(Ac, Wc, force_bn=bn).cpu(), O.op_linear(A, W)) < TOL_BF16
    assert O.rel_err(_lib.op_gemm(Ac, Wc, bias=bc, force_bn=bn).cpu(), lin) < TOL_BF16
    assert O.rel_err(_lib.op_gemm(Ac, Wc, bias=bc, epi=_lib.EPI_GELU, force_bn=bn).cpu(),
                     torch.nn.functional.gelu(bf(lin))) < TOL_BF16
    want = bf(lin).float() + r.float()
    assert O.rel_err(_lib.op_gemm(Ac, Wc, bias=bc, residual=r.cuda(), force_bn=bn).cpu(), want) < TOL_BF16
    # in place: C aliases the residual (h = h + o_proj(attn)), every tile reads its own residual before it is overwritten
    h = r.cuda().clone()
    lib = _lib.load()
    _lib.check(lib.emu_op_gemm(_lib._ptr(Ac), K, _lib._ptr(Wc), K, M, N, K, _lib._ptr(bc), _lib._ptr(h), N, 0, _lib._ptr(h), N,
                               0, bn, _lib._stream()))
    assert O.rel_err(h.cpu(), want) < TOL_BF16


@pytest.mark.parametrize("M,N,K", [(200, 384, 256), (2048, 2560, 640), (300, 400, 128)])
@pytest.mark.parametrize("bn", [0, 64, 128, 192, 224, 256])
def test_gemm_pair_epilogues_all_widths(cuda, M, N, K, bn):
    """SwiGLU / GEGLU with interleaved weight rows at every tile width (staged for multiples of 64, direct at 224)."""
    from emu_b200 import _lib
    A, W, b = _rand((M, K), 21), _rand((N, K), 22, 0.05), _rand((N,), 23)
    bf = lambda t: t.to(torch.bfloat16)
    g, u = O.op_linear(A, W[0::2]), O.op_linear(A, W[1::2])
    assert O.rel_err(_lib.op_gemm(A.cuda(), W.cuda(), epi=_lib.EPI_SWIGLU, force_bn=bn).cpu(),
                     torch.nn.functional.silu(bf(g)) * bf(u)) < TOL_BF16
    hb, gb = O.op_linear(A, W[0::2], b[0::2]), O.op_linear(A, W[1::2], b[1::2])
    assert O.rel_err(_lib.op_gemm(A.cuda(), W.cuda(), bias=b.cuda(), epi=_lib.EPI_GEGLU, force_bn=bn).cpu(),
                     bf(hb) * torch.nn.functional.gelu(bf(gb))) < TOL_BF16


def test_gemm_epilogues(cuda):
    from emu_b200 import _lib
    M, N, K = 200, 384, 256
    A, W, b, r = _rand((M, K), 3), _rand((N, K), 4, 0.05), _rand((N,), 5), _rand((M, N), 6)
    lin = O.op_linear(A, W, b)
    assert O.rel_err(_lib.op_gemm(A.cuda(), W.cuda(), bias=b.cuda()).cpu(), lin) < TOL_BF16
    # fused activations follow the reference's bf16 rounding points: Linear -> bf16 -> act -> bf16 (-> mul -> bf16)
    bf = lambda t: t.to(torch.bfloat16)
    assert O.rel_err(_lib.op_gemm(A.cuda(), W.cuda(), bias=b.cuda(), epi=_lib.EPI_GELU).cpu(),
                     torch.nn.functional.gelu(bf(lin))) < TOL_BF16
    assert O.rel_err(_lib.op_gemm(A.cuda(), W.cuda(), bias=b.cuda(), residual=r.cuda()).cpu(), lin + r.float()) < TOL_BF16
    # interleaved pair epilogues: rows (2j, 2j+1) = (gate_j, up_j) / (hidden_j, gate_j)
    g, u = O.op_linear(A, W[0::2]), O.op_linear(A, W[1::2])
    assert O.rel_err(_lib.op_gemm(A.cuda(), W.cuda(), epi=_lib.EPI_SWIGLU).cpu(),
                     torch.nn.functional.silu(bf(g)) * bf(u)) < TOL_BF16
    hb, gb = O.op_linear(A, W[0::2], b[0::2]), O.op_linear(A, W[1::2], b[1::2])
    assert O.rel_err(_lib.op_gemm(A.cuda(), W.cuda(), bias=b.cuda(), epi=_lib.EPI_GEGLU).cpu(),
                     bf(hb) * torch.nn.functional.gelu(bf(gb))) < TOL_BF16


@pytest.mark.parametrize("B,N,K", [
    (20, 6656, 2240), (5, 2688, 6656), (32, 4480, 1664), (1, 300, 72), (11, 768, 256), (20, 6656, 896), (13, 1000, 4104),
])
def test_gemm_skinny(cuda, B, N, K):
    """The wide-decode projection kernel (weights as the 128-row MMA operand, K-split partial sums through the workspace):
    plain fp32 / bf16, in-place residual (h = h + W a), SwiGLU with interleaved rows; TP-shard shapes of LLaMA-33B, ragged N / K,
    1..32 activation rows.  Run twice: the split counters must reset themselves."""
    from emu_b200 import _lib
    X, W, r = _rand((B, K), 31), _rand((N, K), 32, 0.05), _rand((B, N), 33)
    bf = lambda t: t.to(torch.bfloat16)
    ref = O.op_linear(X, W)
    Xc, Wc = X.cuda(), W.cuda()
    for _ in range(2):
        assert O.rel_err(_lib.op_gemm_skinny(Xc, Wc, out_fp32=True).cpu(), ref) < TOL_F32
    assert O.rel_err(_lib.op_gemm_skinny(Xc, Wc).cpu(), ref) < TOL_BF16
    want = bf(ref).float() + r.float()
    assert O.rel_err(_lib.op_gemm_skinny(Xc, Wc, residual=r.cuda()).cpu(), want) < TOL_BF16
    h = r.cuda().clone()
    lib = _lib.load()
    _lib.check(lib.emu_op_gemm_skinny(_lib._ptr(Xc), K, _lib._ptr(Wc), K, B, N, K, _lib._ptr(h), N, 0, _lib._ptr(h), N, 0,
                                      _lib._stream()))
    assert O.rel_err(h.cpu(), want) < TOL_BF16
    if N % 2 == 0:
        g, u = O.op_linear(X, W[0::2]), O.op_linear(X, W[1::2])
        got = _lib.op_gemm_skinny(Xc, Wc, epi=_lib.EPI_SWIGLU).cpu()
        assert O.rel_err(got, torch.nn.functional.silu(bf(g)) * bf(u)) < TOL_BF16
    # same rounding points as the general GEMM: bf16 outputs agree to the last bit except where the fp32 sums differ by
    # summation order right at a rounding boundary
    a, b = _lib.op_gemm_skinny(Xc, Wc).float().cpu(), _lib.op_gemm(Xc, Wc).float().cpu()
    assert O.rel_err(a, b) < TOL_BF16


@pytest.mark.parametrize("NB,H,W,Cin,Cout", [(1, 16, 8, 64, 64), (2, 32, 32, 128, 320), (1, 64, 64, 8, 96),
                                              (1, 8, 128, 320, 32)])
def test_conv3x3(cuda, NB, H, W, Cin, Cout):
    from emu_b200 import _lib
    x = _rand((NB, Cin, H, W), 7)
    w = _rand((Cout, Cin, 3, 3), 8, 0.05)
    b = _rand((Cout,), 9)
    ref = torch.nn.functional.conv2d(x.float(), w.float(), b.float(), padding=1).permute(0, 2, 3, 1)
    x_nhwc = x.permute(0, 2, 3, 1).contiguous().cuda()
    wk = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous().cuda()  # k = (r*3+s)*Cin + c
    out = _lib.op_conv3x3(x_nhwc, wk, bias=b.cuda()).cpu()
    assert O.rel_err(out, ref) < TOL_BF16


@pytest.mark.parametrize("NB,H,W,Cin,Cout", [(2, 32, 32, 128, 320), (1, 64, 64, 64, 640), (2, 16, 16, 256, 1280)])
def test_conv3x3_residual(cuda, NB, H, W, Cin, Cout):
    """ResnetBlock2D's conv2 + shortcut: the residual tile arrives by TMA load into the staged epilogue (Cout multi-tile)"""
    from emu_b200 import _lib
    x, w, b = _rand((NB, Cin, H, W), 27), _rand((Cout, Cin, 3, 3), 28, 0.05), _rand((Cout,), 29)
    r = _rand((NB, H, W, Cout), 30)
    ref = torch.nn.functional.conv2d(x.float(), w.float(), b.float(), padding=1).permute(0, 2, 3, 1)
    ref = ref.to(torch.bfloat16).float() + r.float()
    x_nhwc = x.permute(0, 2, 3, 1).contiguous().cuda()
    wk = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).contiguous().cuda()
    out = _lib.op_conv3x3(x_nhwc, wk, bias=b.cuda(), residual=r.cuda()).cpu()
    assert O.rel_err(out, ref) < TOL_BF16


@pytest.mark.parametrize("N,K,B", [(6656, 6656, 1), (1024, 256, 5), (32272, 512, 3), (2000, 1792, 8), (48, 64, 2),
                                   (35840, 6656, 1), (6656, 17920, 5), (1024, 6656, 8), (512, 17920, 8), (640, 2304, 7)])
def test_gemv_plain(cuda, N, K, B):
    from emu_b200 import _lib
    W, x = _rand((N, K), 10, 0.05), _rand((B, K), 11)
    ref = O.op_linear(x, W)
    assert O.rel_err(_lib.op_gemv(W.cuda(), x.cuda(), out_fp32=True).cpu(), ref) < TOL_F32
    assert O.rel_err(_lib.op_gemv(W.cuda(), x.cuda(), pdl=True).cpu(), ref) < TOL_BF16


def test_gemv_segmented_x_with_norm(cuda):
    """batch x K too large for shared memory: x is staged in K segments (fused RMSNorm statistics span all segments).
    K = 5664 pads to 23 chunks of 256 staged as 21 + 2, so the last segment is ragged and zero filled past K."""
    from emu_b200 import _lib
    B = 8
    bf = lambda t: t.to(torch.bfloat16)
    for N, K in [(2048, 6656), (1024, 5664)]:
        W, x, nw = _rand((N, K), 16, 0.05), _rand((B, K), 17), (1 + 0.1 * _rand((K,), 18).float()).to(torch.bfloat16)
        r = _rand((B, N), 19)
        xn = O.rms_norm(x, nw, 1e-6)
        ref = O.op_linear(xn, W)
        assert O.rel_err(_lib.op_gemv(W.cuda(), x.cuda(), norm_w=nw.cuda(), out_fp32=True).cpu(), ref) < TOL_F32, (N, K)
        assert O.rel_err(_lib.op_gemv(W.cuda(), x.cuda(), norm_w=nw.cuda(), residual=r.cuda()).cpu(),
                         bf(ref).float() + r.float()) < TOL_BF16, (N, K)
        g, u = O.op_linear(xn, W[0::2]), O.op_linear(xn, W[1::2])
        assert O.rel_err(_lib.op_gemv(W.cuda(), x.cuda(), norm_w=nw.cuda(), mode=_lib.EPI_SWIGLU).cpu(),
                         torch.nn.functional.silu(bf(g)) * bf(u)) < TOL_BF16, (N, K)


def test_gemv_fused(cuda):
    from emu_b200 import _lib
    N, K, B = 1024, 512, 4
    W, x, nw, r = _rand((N, K), 12, 0.05), _rand((B, K), 13), 1 + 0.1 * _rand((K,), 14).float(), _rand((B, N), 15)
    nw = nw.to(torch.bfloat16)
    xn = O.rms_norm(x, nw, 1e-6)          # bf16 rounding points of HF LlamaRMSNorm
    ref = O.op_linear(xn, W)
    assert O.rel_err(_lib.op_gemv(W.cuda(), x.cuda(), norm_w=nw.cuda(), out_fp32=True).cpu(), ref) < TOL_F32
    assert O.rel_err(_lib.op_gemv(W.cuda(), x.cuda(), norm_w=nw.cuda(), residual=r.cuda()).cpu(),
                     ref + r.float()) < TOL_BF16
    g, u = O.op_linear(xn, W[0::2]), O.op_linear(xn, W[1::2])
    bf = lambda t: t.to(torch.bfloat16)
    assert O.rel_err(_lib.op_gemv(W.cuda(), x.cuda(), norm_w=nw.cuda(), mode=_lib.EPI_SWIGLU).cpu(),
                     torch.nn.functional.silu(bf(g)) * bf(u)) < TOL_BF16


@pytest.mark.parametrize("B,Nq,Nk,H,D,causal", [
    (1, 1025, 1025, 16, 112, False), (2, 257, 257, 4, 88, False), (2, 75, 75, 4, 128, True),
    (1, 32, 257, 12, 64, False), (2, 40, 100, 3, 128, True), (1, 300, 300, 2, 64, True), (1, 17, 17, 2, 32, False),
])
def test_attn_prefill(cuda, B, Nq, Nk, H, D, causal):
    from emu_b200 import _lib
    q, k, v = _rand((B, Nq, H, D), 20), _rand((B, Nk, H, D), 21), _rand((B, Nk, H, D), 22)
    kv_start = torch.tensor([0, 7][:B], dtype=torch.int32) if causal else None
    ref = O.op_attention(q, k, v, D ** -0.5, causal=causal, kv_start=kv_start)
    out = _lib.op_attn_prefill(q.cuda(), k.cuda(), v.cuda(), D ** -0.5, causal=causal,
                               kv_start=None if kv_start is None else kv_start.cuda()).cpu()
    if kv_start is not None:  # fully masked (left-pad) query rows are don't-care
        for b in range(B):
            s = int(kv_start[b]) - (Nk - Nq)
            if s > 0:
                out[b, :s] = 0
                ref[b, :s] = 0
    assert O.rel_err(out, ref) < TOL_BF16


@pytest.mark.parametrize("B,Nq,Nk,H,D,causal,qscale,fused", [
    (2, 512, 512, 3, 64, False, 1.0, True), (1, 1024, 1024, 2, 64, False, 6.0, False), (2, 300, 400, 2, 128, True, 1.0, False),
    (1, 640, 640, 2, 128, True, 6.0, True), (1, 130, 700, 2, 64, False, 1.0, False), (1, 4096, 4096, 1, 64, False, 3.0, True),
    (1, 1025, 1025, 2, 112, False, 6.0, True), (2, 256, 64, 2, 64, False, 1.0, False),
])
def test_attn_prefill_tc(cuda, B, Nq, Nk, H, D, causal, qscale, fused):
    """wgmma flash attention (attention_tc.cu): multi-tile, ragged, causal with Nk > Nq and left padding, large score
    ranges (exercises the online max / O rescale), and head-interleaved fused-QKV strides."""
    from emu_b200 import _lib
    if fused and Nq == Nk:
        qkv = _rand((B, Nq, 3, H, D), 27)
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    else:
        q, k, v = _rand((B, Nq, H, D), 20), _rand((B, Nk, H, D), 21), _rand((B, Nk, H, D), 22)
    q = (q.float() * qscale).to(torch.bfloat16)
    kv_start = torch.tensor([0, 7][:B], dtype=torch.int32) if causal else None
    ref = O.op_attention(q, k, v, D ** -0.5, causal=causal, kv_start=kv_start)
    if fused and Nq == Nk:
        dq = (qkv.float() * torch.tensor([qscale, 1.0, 1.0]).view(1, 1, 3, 1, 1)).to(torch.bfloat16).cuda()
        qc, kc, vc = dq[:, :, 0], dq[:, :, 1], dq[:, :, 2]
    else:
        qc, kc, vc = q.cuda(), k.cuda(), v.cuda()
    out = _lib.op_attn_prefill(qc, kc, vc, D ** -0.5, causal=causal,
                               kv_start=None if kv_start is None else kv_start.cuda()).cpu()
    if kv_start is not None:
        for b in range(B):
            s = int(kv_start[b]) - (Nk - Nq)
            if s > 0:
                out[b, :s] = 0
                ref[b, :s] = 0
    assert torch.isfinite(out.float()).all()
    assert O.rel_err(out, ref) < TOL_BF16


def test_attn_prefill_bias(cuda):
    from emu_b200 import _lib
    B, N, H, D = 2, 32, 12, 64
    q, k, v = _rand((B, N, H, D), 23, 0.3), _rand((B, N, H, D), 24, 0.3), _rand((B, N, H, D), 25)
    bias = torch.randn(H, N, N, generator=torch.Generator().manual_seed(26))
    ref = O.op_attention(q, k, v, 1.0, causal=True, bias=bias)
    out = _lib.op_attn_prefill(q.cuda(), k.cuda(), v.cuda(), 1.0, causal=True, bias=bias.cuda()).cpu()
    assert O.rel_err(out, ref) < TOL_BF16


@pytest.mark.parametrize("B,H,D,T,lens,starts", [(1, 52, 128, 512, [200], [0]), (5, 4, 128, 96, [90, 90, 90, 90, 90], [0, 3, 0, 10, 1]),
                                                  (2, 12, 64, 2048, [1999, 1999], [0, 100]), (1, 2, 128, 64, [1], [0])])
def test_attn_decode(cuda, B, H, D, T, lens, starts):
    from emu_b200 import _lib
    q = _rand((B, H * D), 30)
    kc, vc = _rand((B, H, T, D), 31), _rand((B, H, T, D), 32)
    pos = torch.tensor([l - 1 for l in lens], dtype=torch.int32)
    start = torch.tensor(starts, dtype=torch.int32)
    out = _lib.op_attn_decode(q.cuda(), kc.cuda(), vc.cuda(), pos.cuda(), start.cuda(), D ** -0.5, T).cpu()
    for b in range(B):
        kk = kc[b, :, starts[b]:lens[b]].transpose(0, 1)[None]
        vv = vc[b, :, starts[b]:lens[b]].transpose(0, 1)[None]
        ref = O.op_attention(q[b].view(1, 1, H, D), kk, vv, D ** -0.5)
        assert O.rel_err(out[b].view(1, 1, H, D), ref) < TOL_BF16


def test_norms(cuda):
    from emu_b200 import _lib
    x, w, b, r = _rand((300, 1792), 40), (1 + 0.1 * _rand((1792,), 41).float()).to(torch.bfloat16), _rand((1792,), 42), _rand((300, 1792), 43)
    ref = torch.nn.functional.layer_norm(x.float(), (1792,), w.float(), b.float(), 1e-6)
    assert O.rel_err(_lib.op_layernorm(x.cuda(), w.cuda(), b.cuda(), 1e-6).cpu(), ref) < TOL_BF16
    assert O.rel_err(_lib.op_layernorm(x.cuda(), w.cuda(), b.cuda(), 1e-6, residual=r.cuda()).cpu(), ref + r.float()) < TOL_BF16
    assert O.rel_err(_lib.op_rmsnorm(x.cuda(), w.cuda(), 1e-6).cpu(), O.rms_norm(x.float(), w.float(), 1e-6)) < TOL_BF16


def test_gemv_rope_qkv(cuda):
    """fused RMSNorm + QKV + RoPE + KV-cache append vs the HF formulation (oracle.rotate_half path)."""
    from emu_b200 import _lib
    Hh, D, K, B, T = 4, 128, 256, 3, 32
    Wq, Wk, Wv = _rand((Hh * D, K), 50, 0.05), _rand((Hh * D, K), 51, 0.05), _rand((Hh * D, K), 52, 0.05)
    x, nw = _rand((B, K), 53), (1 + 0.1 * _rand((K,), 54).float()).to(torch.bfloat16)
    pos = torch.tensor([5, 9, 20], dtype=torch.int32)
    off = torch.tensor([0, 2, 7], dtype=torch.int32)
    xn = O.rms_norm(x, nw, 1e-6)
    q = O.op_linear(xn, Wq).view(B, Hh, D)
    k = O.op_linear(xn, Wk).view(B, Hh, D)
    v = O.op_linear(xn, Wv).view(B, Hh, D)
    # HF applies RoPE in the activation dtype: bf16 linear output, bf16 cos/sin, every op rounded to bf16
    cos, sin = O.rope_cos_sin((pos - off).long()[:, None], D, 10000.0, torch.bfloat16)   # [B,1,D]
    qb, kb = q.to(torch.bfloat16), k.to(torch.bfloat16)
    qr = (qb * cos + O.rotate_half(qb) * sin).float()
    kr = (kb * cos + O.rotate_half(kb) * sin).float()

    def interleave(w):  # row 2j <- j, 2j+1 <- j + D/2 inside each head
        w = w.view(Hh, D, K)
        return torch.stack((w[:, :D // 2], w[:, D // 2:]), dim=2).reshape(Hh * D, K)
    W = torch.cat((interleave(Wq), interleave(Wk), Wv), dim=0).contiguous()
    tab_pos = torch.arange(64)[None]
    ct, st_ = O.rope_cos_sin(tab_pos, D, 10000.0, torch.bfloat16)
    ct, st_ = ct[0, :, :D // 2].contiguous(), st_[0, :, :D // 2].contiguous()
    kc = torch.zeros(B, Hh, T, D, dtype=torch.bfloat16, device="cuda")
    vc = torch.zeros_like(kc)
    qo = _lib.op_gemv_rope_qkv(W.cuda(), Hh, D, x.cuda(), nw.cuda(), 1e-6, ct.cuda(), st_.cuda(), pos.cuda(), off.cuda(),
                               kc, vc, T).cpu().view(B, Hh, D)

    def deinterleave(t):  # [.., D] interleaved -> original order
        return torch.cat((t[..., 0::2], t[..., 1::2]), dim=-1)
    assert O.rel_err(deinterleave(qo), qr) < TOL_BF16
    for b in range(B):
        assert O.rel_err(deinterleave(kc[b, :, int(pos[b])].cpu()), kr[b]) < TOL_BF16
        assert O.rel_err(vc[b, :, int(pos[b])].cpu(), v[b]) < TOL_BF16


@pytest.mark.parametrize("Bt,nb,V,prev_len,ban,raw,ngram,mask", [
    (1, 5, 32272, 0, -1, False, 0, False), (2, 3, 32272, 7, 2, False, 0, False), (1, 1, 1000, 3, -1, True, 0, False),
    (3, 4, 517, 0, 5, False, 0, True), (2, 3, 517, 9, -1, False, 2, False), (1, 2, 300, 12, 1, True, 3, True)])
def test_beam_topk(cuda, Bt, nb, V, prev_len, ban, raw, ngram, mask):
    """emu_beam_topk vs the torch formulation of one HF _beam_search step (log_softmax -> repetition penalty -> no-repeat
    n-gram -> EOS ban -> prefix-allowed mask -> + running score -> topk(2*beams) over beams*vocab), incl. the greedy /
    sampling order (penalty on the raw logits)."""
    from emu_b200 import _lib
    from test_generation_cpu import torch_beam_topk
    g = torch.Generator().manual_seed(70)
    logits = torch.randn(Bt * nb, V, generator=g) * 3
    running = torch.randn(Bt, nb, generator=g)
    running[:, -1] = -1e9 if nb > 1 else running[:, -1]
    L = prev_len + 5
    prev = torch.randint(0, 40 if ngram else V, (Bt * nb, L), generator=g, dtype=torch.int32) if prev_len else None
    if prev is not None:
        prev[:, prev_len - 1] = prev[:, 0]  # a duplicate: the penalty must apply once; also closes a repeated n-gram
    allowed = (torch.rand(Bt * nb, V, generator=g) < 0.6).to(torch.uint8) if mask else None
    keep, pen = 2 * nb, 1.3
    ref_v, ref_i = torch_beam_topk(logits, running, Bt, nb, keep, ban, prev, prev_len, pen, raw, ngram, allowed)
    out_v, out_i = _lib.op_beam_topk(logits.cuda(), running.cuda(), Bt, nb, keep, ban_id=ban,
                                     prev_tokens=None if prev is None else prev.cuda(), prev_len=prev_len,
                                     repetition_penalty=pen, penalty_on_logits=raw, no_repeat_ngram=ngram,
                                     allowed=None if allowed is None else allowed.cuda())
    real = ref_v > -1e8  # candidates of a dead (-1e9) beam tie at fp32 resolution: order is don't-care
    assert torch.allclose(out_v.cpu()[real], ref_v[real], rtol=1e-5, atol=1e-4)
    assert torch.equal(out_i.cpu()[real], ref_i[real])


@pytest.mark.parametrize("Bt,nb,L,lp,es,eos_rate", [(1, 5, 24, -1.0, False, 0.15), (2, 3, 16, 1.0, False, 0.3),
                                                    (3, 4, 12, 0.0, True, 0.3), (1, 1, 20, 1.0, True, 0.1),
                                                    (2, 5, 10, 2.0, "never", 0.2)])
def test_beam_step_matches_torch_formulation(cuda, Bt, nb, L, lp, es, eos_rate):
    """emu_beam_step (device hypothesis bookkeeping) against the torch formulation that tests/test_generation_cpu.py pins to
    the reference's own lm.generate: random candidate streams (with EOS hits) are fed to both, every step's outputs that can
    influence the search must agree exactly — next tokens, cache reorder indices, running / finished scores, finished flags,
    lengths, the done flag — and so must the final hypotheses."""
    from types import SimpleNamespace
    from emu_b200 import _lib
    from test_generation_cpu import TorchBeamState
    V, eos, pad = 977, 2, 0
    g = torch.Generator().manual_seed(1234 + Bt * 100 + nb)
    eng = SimpleNamespace(lib=_lib.load(), cfg=SimpleNamespace(llm_vocab=V), h=None)
    dev_st = _lib.BeamState(Bt, nb, L, pad, "cuda")
    ref_st = TorchBeamState(Bt, nb, L, pad)
    for cur in range(L):
        # 2*nb distinct candidates per row, scores descending like a top-k output; some of them EOS
        sc = ref_st.running_scores.max(dim=1, keepdim=True)[0] - torch.rand(Bt, 2 * nb, generator=g).cumsum(1)
        beam = torch.randint(0, nb, (Bt, 2 * nb), generator=g)
        tok = torch.randint(3, V, (Bt, 2 * nb), generator=g)
        e = torch.rand(Bt, 2 * nb, generator=g) < eos_rate
        e &= e.long().cumsum(1) <= nb       # top-k over beams x vocab holds at most one EOS per beam
        tok[e] = eos
        idx = (beam * V + tok).to(torch.int32)
        ref_st.step(sc, idx, V, cur, eos, lp, es)
        _lib.Engine.beam_step(eng, dev_st, sc.cuda(), idx.cuda(), cur, eos, lp, es)
        assert int(dev_st.done.item()) == int(ref_st.done.item()), cur
        last = cur + 1 >= L                 # every candidate "hits" on the last step: the running beams tie at -1e9 (unused)
        if not last:
            assert torch.equal(dev_st.next_tokens.cpu(), ref_st.next_tokens), cur
            assert torch.equal(dev_st.beam_src.cpu(), ref_st.beam_src), cur
            assert torch.equal(dev_st.running_scores.cpu(), ref_st.running_scores), cur
        fin = ref_st.is_finished.bool()
        assert torch.equal(dev_st.is_finished.cpu().bool(), fin), cur
        assert torch.equal(dev_st.beam_scores.cpu()[fin], ref_st.beam_scores[fin]), cur
        assert torch.equal(dev_st.fin_len.cpu()[fin], ref_st.fin_len[fin]), cur
        assert torch.equal(dev_st.unsat.cpu(), ref_st.unsat), cur
        p = (cur + 1) & 1
        if not last:
            assert torch.equal(dev_st.running_seq[p].cpu(), ref_st.running_seq[p]), cur
        assert torch.equal(dev_st.sequences[p].cpu()[fin], ref_st.sequences[p][fin]), cur
        if ref_st.is_done():
            break
    assert ref_st.is_done() and dev_st.is_done()
    assert torch.equal(dev_st.result(cur + 1).cpu(), ref_st.result(cur + 1))


@pytest.mark.parametrize("H,W,S", [(37, 53, 16), (500, 333, 448), (448, 448, 448), (1024, 768, 448), (31, 97, 224),
                                   (448, 300, 448), (2160, 3840, 448)])
def test_preprocess_image(cuda, H, W, S):
    """emu_preprocess_image (Pillow-exact fixed-point bicubic + ToTensor + Normalize) is BIT-EXACT against the oracle,
    which is pinned bit-exactly to torchvision + Pillow on the CPU side."""
    import numpy as np
    from emu_b200 import _lib
    from oracle import preprocess_oracle as P
    mean, std = (0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)
    rng = np.random.default_rng(H * 1000 + W)
    img = (rng.random((H, W, 3)) * 255).astype(np.uint8)
    ref = torch.from_numpy(P.image_transform(img, S, mean, std))
    out = _lib.op_preprocess_image(torch.from_numpy(img).cuda(), S, S, mean, std, dtype=torch.float32).cpu()
    assert torch.equal(out, ref)
    out16 = _lib.op_preprocess_image(torch.from_numpy(img).cuda(), S, S, mean, std, dtype=torch.bfloat16).cpu()
    assert torch.equal(out16, ref.to(torch.bfloat16))


def test_image_to_uint8(cuda):
    """device uint8 conversion == numpy_to_pil's (images * 255).round().astype("uint8") incl. exact .5 ties"""
    import numpy as np
    from emu_b200 import _lib
    g = torch.Generator().manual_seed(80)
    x = torch.rand(3, 64, 64, 3, generator=g)
    x.view(-1)[:512] = (torch.arange(512) % 256 + 0.5) / 255.0   # products landing on (or next to) .5 ties
    x = x.clamp(0, 1).to(torch.bfloat16).float()                 # the VAE path hands over bf16-rounded values
    ref = (x.numpy() * 255).round().astype("uint8")
    out = _lib.op_image_to_uint8(x.cuda()).cpu().numpy()
    assert np.array_equal(out, ref)


def _hf_support(scores, top_k, top_p):
    """kept-token mask of HF's TopK / TopP warpers (the torch formulation in emu_b200/generation.py)"""
    s = scores.clone()
    if top_k:
        kth = torch.topk(s, min(top_k, s.shape[-1]))[0][..., -1, None]
        s = s.masked_fill(s < kth, float("-inf"))
    if top_p < 1.0:
        ss, si = torch.sort(s, descending=False)
        cum = ss.softmax(-1).cumsum(-1)
        rem = cum <= (1 - top_p)
        rem[..., -1:] = False
        s = s.masked_fill(rem.scatter(1, si, rem), float("-inf"))
    return s


@pytest.mark.parametrize("V,top_k,top_p,temp", [(64, 0, 1.0, 1.0), (64, 8, 1.0, 0.7), (64, 0, 0.8, 1.0), (1000, 50, 0.9, 1.3),
                                                 (32272, 50, 0.9, 1.0)])
def test_sample_tokens(cuda, V, top_k, top_p, temp):
    """emu_sample_tokens: every draw lies in HF's top-k/top-p support and the empirical distribution matches the filtered
    softmax (total-variation distance within sampling noise)."""
    from emu_b200 import _lib
    g = torch.Generator().manual_seed(90)
    R = 4096 if V <= 1000 else 2048
    base = torch.randn(1, V, generator=g) * 2.0
    logits = base.repeat(R, 1).contiguous()
    kept = _hf_support(base / temp, top_k, top_p)
    probs = kept.softmax(-1)[0]
    ids = _lib.op_sample_tokens(logits.cuda(), temperature=temp, top_k=top_k, top_p=top_p, seed=1234, offset=7).cpu().long()
    assert ids.min() >= 0 and ids.max() < V
    # tokens whose cumulative mass sits within 1e-3 of the top-p cut may legitimately fall on either side (fp32 sums)
    border = torch.zeros(V, dtype=torch.bool)
    if top_p < 1.0:
        sp, si = torch.sort((base / temp)[0].softmax(-1) if not top_k else _hf_support(base / temp, top_k, 1.0)[0].softmax(-1),
                            descending=True)
        before = sp.cumsum(0) - sp
        border[si[(before - top_p).abs() < 1e-3]] = True
    ok = (probs[ids] > 0) | border[ids]
    assert bool(ok.all()), ids[~ok][:10]
    emp = torch.bincount(ids, minlength=V).float() / R
    tv = 0.5 * (emp - probs).abs().sum()
    n_support = int((probs > 0).sum())
    assert tv < 0.5 * (n_support / R) ** 0.5 + 0.02, (float(tv), n_support)
    # different offsets give different draws, same (seed, offset) is reproducible
    ids2 = _lib.op_sample_tokens(logits.cuda(), temperature=temp, top_k=top_k, top_p=top_p, seed=1234, offset=7).cpu().long()
    assert torch.equal(ids, ids2)
    ids3 = _lib.op_sample_tokens(logits.cuda(), temperature=temp, top_k=top_k, top_p=top_p, seed=1234, offset=8).cpu().long()
    assert not torch.equal(ids, ids3) or n_support == 1
