"""GPU: the diffusion kernels through their stand-alone entry points (include/emu_b200_diffusion_ops.h), each against a plain
reference of the same operation at the shapes Emu2-Gen and the Emu1 pipeline serve: the SDXL UNet at 320 / 640 / 1280
channels on 128^2 / 64^2 / 32^2 latents and its up-block concat widths, the SDXL VAE decoder at 128..512 channels on planes
up to 1024^2 (and four images at once, 2^31 bytes per tensor), its mid-block attention over 16384 tokens of width 512, and
the SD-1.5 levels of Emu1 down to 8^2.

* GroupNorm(+SiLU): fp64 F.group_norm over the same bf16 inputs, relative max-abs error <= TOL_BF16, with per-group
  mean/std up to 300 (where a one-pass E[x^2] - mean^2 in fp32 cancels).  torch's own CUDA bf16 group_norm is held to the
  same bound on the groups of the same inputs that carry no offset, so the bound is one the reference's path meets; with
  the offsets torch's bf16 path is itself 0.07 - 0.2 off on an H100 (printed), the engine is not allowed to be.
* VAE attention: fp64 softmax(q k^T / sqrt(C)) v over the same bf16 inputs; the bound is TOL_BF16 or 1.5x what torch SDPA
  in bf16 costs on the same inputs, whichever is larger.
* time embeddings: within one bf16 ulp of fp64 cos / sin at the fp32 argument the reference forms (plus that argument's
  own fp32 ulp: the frequency table's exp may round the other way on the device).
* data movement, the token mean, the VAE post-process and the PNDM glue: bit for bit against a torch restatement (the
  token mean within its fp32 summation error of the fp64 mean).

Sentinels: every output element a kernel must not write holds bf16 NaN (or a known pattern), and the outputs are NaN
before the call, so a stray or a missing write fails the test without any fault.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL_BF16 = 6e-3
NAN = float("nan")


def _lib():
    from emu_b200 import _lib as L
    return L


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _guarded(shape, dtype, guard=4096):
    """an output tensor followed by `guard` NaN elements: returns (view, tail)"""
    n = math.prod(shape)
    buf = torch.full((n + guard,), NAN, dtype=dtype, device="cuda")
    return buf[:n].view(*shape), buf[n:]


def _check_guard(out, tail):
    assert bool(torch.isnan(tail).all()), "a kernel wrote past the end of its output"
    assert not bool(torch.isnan(out).any()), "an output element was not written"


def _rel_err(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


def _bf16_ulp(r):
    """spacing of bf16 numbers at |r| (8 significant bits)"""
    e = torch.floor(torch.log2(r.double().abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


# ------------------------------------------------------------------------------------------------------------------------
# GroupNorm (+SiLU)
# ------------------------------------------------------------------------------------------------------------------------
RATIOS = (0.0, 30.0, 100.0, 300.0)     # per-group |mean| / std, cycled over the groups of every case

# (name, C, H, W, NB, eps, channel-varying offsets)
GN_CASES = [
    # SDXL UNet: the level widths, then the up-block concat widths (cpg 80, 60, 40, 30, 20, 10: 8-channel vectors straddle
    # group edges where cpg % 8 != 0); NB 2 = one request with CFG, NB 8 = four CFG latent slots
    ("unet 320@128^2", 320, 128, 128, 2, 1e-5, False),
    ("unet 320@128^2 x8", 320, 128, 128, 8, 1e-5, True),
    ("unet 640@64^2", 640, 64, 64, 2, 1e-5, False),
    ("unet 1280@32^2", 1280, 32, 32, 2, 1e-5, False),
    ("unet 1280@32^2 x8", 1280, 32, 32, 8, 1e-5, False),
    ("unet cat 2560@32^2", 2560, 32, 32, 2, 1e-5, False),
    ("unet cat 2560@32^2 x8", 2560, 32, 32, 8, 1e-5, True),
    ("unet cat 1920@32^2", 1920, 32, 32, 2, 1e-5, True),
    ("unet cat 1920@64^2", 1920, 64, 64, 2, 1e-5, False),
    ("unet cat 1280@64^2", 1280, 64, 64, 2, 1e-5, False),
    ("unet cat 960@64^2", 960, 64, 64, 2, 1e-5, True),
    ("unet cat 960@128^2", 960, 128, 128, 2, 1e-5, False),
    ("unet cat 640@128^2", 640, 128, 128, 2, 1e-5, False),
    # SDXL VAE decoder (eps 1e-6), one image; 128^2 latents -> 1024^2 image
    ("vae 512@128^2", 512, 128, 128, 1, 1e-6, False),
    ("vae 512@256^2", 512, 256, 256, 1, 1e-6, True),
    ("vae 512@512^2", 512, 512, 512, 1, 1e-6, False),
    ("vae 256@512^2", 256, 512, 512, 1, 1e-6, False),
    ("vae 256@1024^2", 256, 1024, 1024, 1, 1e-6, True),
    ("vae 128@1024^2", 128, 1024, 1024, 1, 1e-6, False),
    ("vae 128@1024^2 x2", 128, 1024, 1024, 2, 1e-6, False),
    # SD-1.5 (Emu1) levels down to 8^2: HW 64 < the 128 partial-sum chunks, so some chunks are empty; one ragged plane
    ("sd15 320@64^2", 320, 64, 64, 2, 1e-5, False),
    ("sd15 640@32^2", 640, 32, 32, 2, 1e-5, False),
    ("sd15 1280@16^2", 1280, 16, 16, 2, 1e-5, True),
    ("sd15 1280@8^2", 1280, 8, 8, 2, 1e-5, False),
    ("sd15 2560@8^2 x8", 2560, 8, 8, 8, 1e-5, False),
    ("ragged 320@37x23", 320, 37, 23, 2, 1e-5, True),
    ("ragged 640@5x7", 640, 5, 7, 3, 1e-5, False),
]


def _gn_input(NB, HW, C, groups, chan_var, seed):
    g = _gen(seed)
    cpg = C // groups
    std = 0.5 + 1.5 * torch.rand(groups, generator=g, device="cuda")
    sign = torch.where(torch.rand(groups, generator=g, device="cuda") < 0.5, -1.0, 1.0)
    ratio = torch.tensor(RATIOS, device="cuda")[torch.arange(groups, device="cuda") % len(RATIOS)]
    mean_c = (sign * ratio * std).repeat_interleave(cpg)
    std_c = std.repeat_interleave(cpg)
    if chan_var:   # the mean also drifts across the channels of a group, by up to +-3 std
        mean_c = mean_c + torch.linspace(-3, 3, cpg, device="cuda").repeat(groups) * std_c
    x = torch.empty(NB, HW, C, dtype=torch.bfloat16, device="cuda")
    for b in range(NB):   # one image at a time keeps the fp32 temporaries small at 1024^2
        x[b] = (torch.randn(HW, C, generator=g, device="cuda") * std_c + mean_c).to(torch.bfloat16)
    w = (1 + 0.1 * torch.randn(C, generator=g, device="cuda")).to(torch.bfloat16)
    bias = (0.05 * torch.randn(C, generator=g, device="cuda")).to(torch.bfloat16)
    return x, w, bias


def _gn_errors(x, out, w, b, groups, eps, silu):
    """against fp64 F.group_norm, image by image: (engine error, torch CUDA bf16 group_norm error on the groups without an
    offset, torch's error on all groups)"""
    NB, HW, C = x.shape
    num_e, num_t, den = 0.0, torch.zeros(groups, dtype=torch.float64, device="cuda"), 0.0
    for i in range(NB):
        xi = x[i].t().reshape(1, C, HW)
        norm = F.group_norm(xi.double(), groups, w.double(), b.double(), eps)
        # torch's group_norm is checked on the norm itself (with SiLU its path would add a bf16 rounding of the SiLU output)
        tb = F.group_norm(xi.contiguous(), groups, w, b, eps)
        num_t = torch.maximum(num_t, (tb[0].double() - norm[0]).abs().view(groups, -1).amax(1) / norm.abs().max())
        # the documented rounding point of the SiLU variant: bf16 norm output, then SiLU
        ref = F.silu(norm.to(torch.bfloat16).double()) if silu else norm
        num_e = max(num_e, float((out[i].t().double() - ref[0]).abs().max()))
        den = max(den, float(ref.abs().max()))
        del norm, ref, tb
    zero_offset = torch.arange(groups, device="cuda") % len(RATIOS) == RATIOS.index(0.0)
    return num_e / den, float(num_t[zero_offset].max()), float(num_t.max())


@pytest.mark.parametrize("silu", [False, True], ids=["norm", "norm+silu"])
@pytest.mark.parametrize("name,C,H,W,NB,eps,chan_var", GN_CASES, ids=[c[0] for c in GN_CASES])
def test_groupnorm_matches_fp64(cuda, name, C, H, W, NB, eps, chan_var, silu):
    L = _lib()
    groups, HW = 32, H * W
    x, w, b = _gn_input(NB, HW, C, groups, chan_var, seed=C + HW + NB)
    out, tail = _guarded((NB, HW, C), torch.bfloat16)
    L.op_groupnorm(x, w, b, groups, eps, silu, out=out)
    torch.cuda.synchronize()
    _check_guard(out, tail)
    e_eng, e_torch0, e_torch = _gn_errors(x, out, w, b, groups, eps, silu)
    print("\n[groupnorm] %-24s %-9s engine %.2e | torch bf16: %.2e without offset, %.2e with"
          % (name, "silu" if silu else "", e_eng, e_torch0, e_torch))
    assert e_torch0 <= TOL_BF16, ("the bound is not one torch's own bf16 group_norm meets", name, e_torch0)
    assert e_eng <= TOL_BF16, (name, e_eng)
    again = L.op_groupnorm(x, w, b, groups, eps, silu)    # fixed summation order: the same bits every run
    assert torch.equal(_bits(again), _bits(out))


def test_groupnorm_2g_tensor(cuda):
    """the VAE's last level at max_images_per_batch 4: 4 x 1024^2 x 256 bf16 = 2^31 bytes, so any 32-bit byte or element
    offset (image base, pixel row) would wrap; every image is checked, the last one most of all"""
    L = _lib()
    NB, HW, C, groups = 4, 1024 * 1024, 256, 32
    x, w, b = _gn_input(NB, HW, C, groups, True, seed=2 ** 31 % 997)
    out, tail = _guarded((NB, HW, C), torch.bfloat16, guard=1 << 16)
    L.op_groupnorm(x, w, b, groups, 1e-6, True, out=out)
    torch.cuda.synchronize()
    _check_guard(out, tail)
    e_eng, e_torch0, e_torch = _gn_errors(x, out, w, b, groups, 1e-6, True)
    print("\n[groupnorm] 4 x 256@1024^2 silu engine %.2e | torch bf16: %.2e without offset, %.2e with"
          % (e_eng, e_torch0, e_torch))
    assert e_eng <= TOL_BF16 and e_torch0 <= TOL_BF16, (e_eng, e_torch0)


# ------------------------------------------------------------------------------------------------------------------------
# VAE mid-block attention
# ------------------------------------------------------------------------------------------------------------------------
def _attn_ref_rows(q, k, v, rows):
    """fp64 softmax(q k^T / sqrt(C)) v of the query rows `rows` of one image"""
    C = q.shape[-1]
    s = (q[rows].double() @ k.double().t()) * C ** -0.5
    return torch.softmax(s, -1) @ v.double()


@pytest.mark.parametrize("T,B,sigma", [(16384, 1, 1.0), (16384, 1, 3.0), (16384, 1, 6.0), (16384, 2, 3.0),
                                       (4096, 1, 6.0), (4096, 2, 1.0), (4096, 2, 6.0)])
def test_vae_attention_matches_fp64(cuda, T, B, sigma):
    """T = 16384 is the mid-block of 128^2 latents (a 1024^2 image), 4096 of 64^2; C = 512.  k is scaled so that the scaled
    logits q.k / sqrt(C) have standard deviation sigma.  The fp64 reference is formed for every 8th query row plus the rows on
    either side of each query-chunk boundary, in every image."""
    L = _lib()
    C = 512
    g = _gen(T + 10 * B + int(sigma))
    q = torch.randn(B, T, C, generator=g, device="cuda").to(torch.bfloat16)
    k = (torch.randn(B, T, C, generator=g, device="cuda") * sigma).to(torch.bfloat16)
    v = torch.randn(B, T, C, generator=g, device="cuda").to(torch.bfloat16)
    out, tail = _guarded((B, T, C), torch.bfloat16)
    L.op_vae_attention(q, k, v, out=out)
    sdpa = F.scaled_dot_product_attention(q[:, None], k[:, None], v[:, None])[:, 0]
    torch.cuda.synchronize()
    _check_guard(out, tail)
    chunk = (1 << 26) // T                                   # vae_attention_chunk_rows (vae.cu)
    edges = [r + d for r in range(chunk, T, chunk) for d in (-1, 0)]
    rows = torch.tensor(sorted(set(range(0, T, 8)) | set(edges) | {T - 1}), device="cuda")
    num_e = num_s = den = 0.0
    for b in range(B):
        ref = _attn_ref_rows(q[b], k[b], v[b], rows)
        num_e = max(num_e, float((out[b, rows].double() - ref).abs().max()))
        num_s = max(num_s, float((sdpa[b, rows].double() - ref).abs().max()))
        den = max(den, float(ref.abs().max()))
    e_eng, e_sdpa = num_e / den, num_s / den
    print("\n[vae attention] T %5d B %d logit std %.0f: engine %.2e | torch SDPA bf16 %.2e" % (T, B, sigma, e_eng, e_sdpa))
    assert e_eng <= max(TOL_BF16, 1.5 * e_sdpa), (T, B, sigma, e_eng, e_sdpa)


# ------------------------------------------------------------------------------------------------------------------------
# time embeddings
# ------------------------------------------------------------------------------------------------------------------------
def _emb_arg(t, dim):
    """the fp32 argument t * exp(-ln(1e4) j / half) as oracle.diffusion_oracle.timestep_embedding forms it (on the CPU)"""
    half = dim // 2
    exponent = -math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half
    return t.float().cpu()[:, None] * torch.exp(exponent)[None, :]


def _check_embedding(got, t, dim, what):
    """each element within one bf16 ulp of the fp64 value at the oracle's fp32 argument, widened by a few fp32 ulps of the
    argument: the kernel's expf (2 ulp) and the CPU's exp may round a frequency differently, which moves t * f by a few ulps
    of itself (2e-4 at t ~ 1000; it only shows where cos / sin cross zero).  Bit-equal to the bf16 oracle except for the
    few elements that such a shift carries across a bf16 rounding boundary."""
    from oracle import diffusion_oracle as D
    got = got.cpu()
    arg = _emb_arg(t, dim)
    oracle = D.timestep_embedding(t.cpu(), dim, torch.bfloat16)
    ref64 = torch.cat([torch.cos(arg.double()), torch.sin(arg.double())], -1)
    tol = _bf16_ulp(ref64) + torch.cat([arg, arg], -1).double().abs() * 2.0 ** -21
    err = (got.double() - ref64).abs()
    assert bool((err <= tol).all()), (what, float((err / tol).max()))
    diff = int((_bits(got) != _bits(oracle)).sum())
    print("\n[time embedding] %-28s %d of %d elements differ from the bf16 oracle by one rounding" % (what, diff, got.numel()))
    assert diff <= max(4, got.numel() // 100), (what, diff)


def test_timestep_embedding(cuda):
    L = _lib()
    euler = torch.linspace(999.0, 0.0, 50) * 0.987 + 0.3       # fractional (Euler-style) timesteps
    t = torch.cat([torch.tensor([0.0, 1.0, 999.0, 0.5, 981.0, 500.25]), euler]).float().cuda()
    for dim in (320, 256):                                      # SDXL / SD-1.5 timestep proj, SDXL time-id width
        out, tail = _guarded((t.numel(), dim), torch.bfloat16)
        L.op_timestep_embedding(t, out, dim)
        torch.cuda.synchronize()
        _check_guard(out, tail)
        _check_embedding(out, t, dim, "timesteps, dim %d" % dim)


def test_time_id_embedding_packs_after_the_text_embedding(cuda):
    """grp = 6 with col_off = cross-attention width: [text_embeds | emb(id_0) | ... | emb(id_5)] per row, SDXL add_embedding
    input (1792 + 6 x 256 = 3328 columns); the text columns stay as they were, bit for bit"""
    L = _lib()
    tid = torch.tensor([[1024, 1024, 0, 0, 1024, 1024], [4096, 4096, 0, 0, 4096, 4096], [512, 768, 17, 33, 1024, 1024],
                        [4096, 1, 4095, 2, 3000, 2048]], dtype=torch.float32, device="cuda")
    B, cd, dim = tid.shape[0], 1792, 256
    text = torch.randn(B, cd, generator=_gen(7), device="cuda").to(torch.bfloat16)
    out, tail = _guarded((B, cd + 6 * dim), torch.bfloat16)
    out[:, :cd] = text
    L.op_timestep_embedding(tid.reshape(-1).contiguous(), out, dim, col_off=cd, grp=6)
    torch.cuda.synchronize()
    _check_guard(out, tail)
    assert torch.equal(_bits(out[:, :cd]), _bits(text))
    _check_embedding(out[:, cd:].reshape(B * 6, dim), tid.reshape(-1), dim, "time ids up to 4096")


# ------------------------------------------------------------------------------------------------------------------------
# data movement: upsample, im2col, concat, NCHW <-> NHWC, VAE post-process
# ------------------------------------------------------------------------------------------------------------------------
def _rand_bf16(shape, seed):
    return torch.randn(*shape, generator=_gen(seed), device="cuda").to(torch.bfloat16)


# (C, H, W, NB): SDXL UNet up-samplers (CFG 2 and four slots 8), the VAE's (one image; and its last at four images), SD-1.5
UPSAMPLE_CASES = [(1280, 32, 32, 2), (640, 64, 64, 2), (1280, 32, 32, 8), (640, 64, 64, 8),
                  (512, 128, 128, 1), (512, 256, 256, 1), (256, 512, 512, 1), (256, 512, 512, 4),
                  (1280, 8, 8, 2), (1280, 16, 16, 2), (640, 32, 32, 2), (64, 5, 7, 3)]


@pytest.mark.parametrize("C,H,W,NB", UPSAMPLE_CASES, ids=["%dx%d@%dx%d" % (c[3], c[0], c[1], c[2]) for c in UPSAMPLE_CASES])
def test_upsample2x_bitwise(cuda, C, H, W, NB):
    L = _lib()
    x = _rand_bf16((NB, H, W, C), C + H + NB)
    out, tail = _guarded((NB, 2 * H, 2 * W, C), torch.bfloat16)
    L.op_upsample2x(x, out=out)
    torch.cuda.synchronize()
    _check_guard(out, tail)
    ref = x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    assert torch.equal(_bits(out), _bits(ref))


def _im2col_ref(x, stride):
    NB, H, W, C = x.shape
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    taps = [xp[:, r:r + stride * (Ho - 1) + 1:stride, s:s + stride * (Wo - 1) + 1:stride] for r in range(3) for s in range(3)]
    return torch.stack(taps, 3).reshape(NB, Ho, Wo, 9 * C)


# (C, H, W, NB, stride): the stride-2 downsamplers of SDXL and SD-1.5, stride 1 on the small maps conv3 cannot tile, odd planes
IM2COL_CASES = [(320, 128, 128, 2, 2), (640, 64, 64, 2, 2), (320, 128, 128, 8, 2), (320, 64, 64, 2, 2), (640, 32, 32, 2, 2),
                (1280, 16, 16, 2, 2), (1280, 8, 8, 2, 1), (2560, 8, 8, 2, 1), (64, 7, 5, 3, 1), (64, 7, 5, 3, 2),
                (320, 37, 23, 2, 2), (320, 37, 23, 2, 1), (16, 1, 1, 1, 2)]


@pytest.mark.parametrize("C,H,W,NB,stride", IM2COL_CASES, ids=["%dx%d@%dx%d/s%d" % (c[3], c[0], c[1], c[2], c[4])
                                                                for c in IM2COL_CASES])
def test_im2col3x3_bitwise(cuda, C, H, W, NB, stride):
    L = _lib()
    x = _rand_bf16((NB, H, W, C), C + H + W + stride)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    out, tail = _guarded((NB, Ho, Wo, 9 * C), torch.bfloat16)
    L.op_im2col3x3(x, stride, out=out)
    torch.cuda.synchronize()
    _check_guard(out, tail)
    assert torch.equal(_bits(out), _bits(_im2col_ref(x, stride)))


# (C_up, C_skip, H, W, NB): every skip concat of the SDXL up path (and SD-1.5's deepest)
CONCAT_CASES = [(1280, 1280, 32, 32, 2), (1280, 640, 32, 32, 2), (1280, 640, 64, 64, 2), (640, 640, 64, 64, 2),
                (640, 320, 64, 64, 2), (640, 320, 128, 128, 2), (320, 320, 128, 128, 2), (320, 320, 128, 128, 8),
                (1280, 1280, 8, 8, 2), (64, 32, 5, 7, 3)]


@pytest.mark.parametrize("C,S,H,W,NB", CONCAT_CASES, ids=["%dx(%d+%d)@%dx%d" % (c[4], c[0], c[1], c[2], c[3])
                                                          for c in CONCAT_CASES])
def test_concat_bitwise(cuda, C, S, H, W, NB):
    """the UNet's channel concat: copy_cols of the up-path activation, then of the skip, into one [M, C + S] buffer; after
    the first copy the skip's columns are still untouched"""
    L = _lib()
    M = NB * H * W
    a, s = _rand_bf16((M, C), C + M), _rand_bf16((M, S), S + M + 1)
    out, tail = _guarded((M, C + S), torch.bfloat16)
    L.op_copy_cols(a, out, 0)
    torch.cuda.synchronize()
    assert bool(torch.isnan(out[:, C:]).all()) and bool(torch.isnan(tail).all())
    L.op_copy_cols(s, out, C)
    torch.cuda.synchronize()
    _check_guard(out, tail)
    assert torch.equal(_bits(out), _bits(torch.cat([a, s], 1)))
    # a source narrower than its row stride (the first n of S columns) into the middle of a wider destination
    n = max(8, S // 16 * 8)
    wide, wtail = _guarded((M, C + S + 16), torch.bfloat16)
    L.op_copy_cols(s[:, :n], wide, 8)
    torch.cuda.synchronize()
    assert torch.equal(_bits(wide[:, 8:8 + n]), _bits(s[:, :n]))
    assert bool(torch.isnan(wide[:, :8]).all()) and bool(torch.isnan(wide[:, 8 + n:]).all()) and bool(torch.isnan(wtail).all())


# (C, Cp, H, W, NB): latents in (4 -> 8 channels) for the SDXL UNet (CFG 2, slots 8), the VAE (1 and 4 images), SD-1.5
LAYOUT_CASES = [(4, 8, 128, 128, 2), (4, 8, 128, 128, 8), (4, 8, 128, 128, 1), (4, 8, 128, 128, 4), (4, 8, 64, 64, 2),
                (4, 16, 5, 7, 3), (3, 8, 37, 23, 2)]


@pytest.mark.parametrize("C,Cp,H,W,NB", LAYOUT_CASES, ids=["%dx%d/%d@%dx%d" % (c[4], c[0], c[1], c[2], c[3])
                                                           for c in LAYOUT_CASES])
def test_nchw_nhwc_round_trip_bitwise(cuda, C, Cp, H, W, NB):
    L = _lib()
    x = _rand_bf16((NB, C, H, W), C + H + NB) * 4
    for scale in (1.0, 1 / 0.13025, float(torch.tensor(1 / 0.18215).to(torch.bfloat16))):
        nhwc, tail = _guarded((NB, H, W, Cp), torch.bfloat16)
        L.op_nchw_to_nhwc(x, Cp, scale, out=nhwc)
        torch.cuda.synchronize()
        _check_guard(nhwc, tail)
        want = torch.zeros(NB, H, W, Cp, dtype=torch.bfloat16, device="cuda")
        want[..., :C] = (x.float() * torch.tensor(scale, dtype=torch.float32)).to(torch.bfloat16).permute(0, 2, 3, 1)
        assert torch.equal(_bits(nhwc), _bits(want)), scale
    # back, from a row of ldx = Cp channels of which only the first C are read (the others hold NaN)
    src = torch.full((NB, H, W, Cp), NAN, dtype=torch.bfloat16, device="cuda")
    src[..., :C] = x.permute(0, 2, 3, 1)
    back, tail = _guarded((NB, C, H, W), torch.bfloat16)
    L.op_nhwc_to_nchw(src, C, out=back)
    torch.cuda.synchronize()
    _check_guard(back, tail)
    assert torch.equal(_bits(back), _bits(x))


@pytest.mark.parametrize("H,W,NB", [(1024, 1024, 1), (1024, 1024, 4), (512, 512, 2), (37, 23, 3)])
def test_vae_post_bitwise(cuda, H, W, NB):
    """(x / 2 + 0.5).clamp(0, 1) in bf16, as the reference post-processes the decoder output, read from the 8-channel padded
    rows conv_out writes (channels 3..7 hold NaN: they must not be read)"""
    L = _lib()
    x = torch.full((NB, H, W, 8), NAN, dtype=torch.bfloat16, device="cuda")
    x[..., :3] = _rand_bf16((NB, H, W, 3), H + NB) * 1.5
    x[0, 0, 0, :3] = torch.tensor([-1.0, 1.0, 3.0])    # the clamp edges
    out, tail = _guarded((NB, H, W, 3), torch.float32)
    L.op_vae_post(x, 3, out=out)
    torch.cuda.synchronize()
    _check_guard(out, tail)
    want = (x[..., :3] / 2 + 0.5).clamp(0, 1).float()
    assert torch.equal(_bits(out), _bits(want))


@pytest.mark.parametrize("B,L_,C", [(2, 64, 1792), (8, 64, 1792), (1, 77, 1792), (3, 5, 24), (2, 1, 1792)])
def test_mean_tokens(cuda, B, L_, C):
    """text_embeds = prompt_embeds.mean(1): the kernel sums in fp32 in its own order, so each element must be within one
    bf16 ulp of the fp64 mean plus the fp32 sum's own error bound (L x 2^-24 x the mean |x|, which only matters where the
    tokens cancel)"""
    L = _lib()
    x = _rand_bf16((B, L_, C), B + L_ + C) + 0.25
    out, tail = _guarded((B, C), torch.bfloat16)
    L.op_mean_tokens(x, out=out)
    torch.cuda.synchronize()
    _check_guard(out, tail)
    ref = x.double().mean(1)
    bound = _bf16_ulp(ref) + L_ * 2.0 ** -24 * x.double().abs().mean(1)
    assert bool(((out.double() - ref).abs() <= bound).all()), float(((out.double() - ref).abs() / bound).max())


# ------------------------------------------------------------------------------------------------------------------------
# PNDM glue (CFG combine + linear multistep update of the Emu1 pipeline)
# ------------------------------------------------------------------------------------------------------------------------
def _fma(a, b, c):
    """fp32 a * b + c with one rounding, as the kernel's fused multiply-adds (exact product in fp64)"""
    return (torch.as_tensor(a, dtype=torch.float64) * torch.as_tensor(b, dtype=torch.float64) + c.double()).float()


def _ref_multistep(lat, eps, hist, saved, p, cfg):
    B, C, h, w = lat.shape
    a, b, wc, w0, w1, w2, g, flags = [float(v) for v in p]
    flags = int(flags)
    bf = lambda v: v.to(torch.bfloat16).float()
    ec = eps[:B, :, :, :C].permute(0, 3, 1, 2).float()
    e = ec
    if cfg:
        eu = eps[B:2 * B, :, :, :C].permute(0, 3, 1, 2).float()
        e = bf(eu + bf(g * bf(ec - eu)))
    h0, h1, h2 = hist[0], hist[1], hist[2]
    # m = wc e + w0 h0 + w1 h1 + w2 h2 and lat = a x + b m as nvcc contracts them: fma(w2, h2, fma(w1, h1, fma(wc, e, w0 h0)))
    m = _fma(w2, h2, _fma(w1, h1, _fma(wc, e, h0 * torch.tensor(w0, dtype=torch.float32))))
    x = saved if flags & 2 else lat
    new_lat = _fma(b, m, x * torch.tensor(a, dtype=torch.float32))
    new_saved = lat.clone() if flags & 4 else saved.clone()
    new_hist = torch.stack([e, h0, h1]) if flags & 1 else hist.clone()
    return new_lat, new_hist, new_saved


@pytest.mark.parametrize("B", [1, 2, 3, 4])
@pytest.mark.parametrize("cfg", [0, 1], ids=["no-cfg", "cfg"])
def test_denoise_multistep_bitwise(cuda, B, cfg):
    """every flag combination (push the history, read the saved sample, store the incoming latent) on a ragged plane
    (HW = 35) and on Emu1's 64^2 latents; eps rows are NHWC with ld 8 (channels 4..7 hold NaN and must not be read), the
    unconditional rows hold NaN without CFG, and the saved sample holds NaN where it must not be read"""
    L = _lib()
    for (h, w) in ((5, 7), (64, 64)):
        C, ld = 4, 8
        g = torch.Generator().manual_seed(B * 10 + cfg + h)
        for flags in range(8):
            lat = torch.randn(B, C, h, w, generator=g) * 3
            hist = torch.randn(3, B, C, h, w, generator=g)
            saved = torch.randn(B, C, h, w, generator=g) if flags & 2 else torch.full((B, C, h, w), NAN)
            eps = torch.full((2 * B, h, w, ld), NAN).to(torch.bfloat16)
            eps[:(2 if cfg else 1) * B, :, :, :C] = torch.randn((2 if cfg else 1) * B, h, w, C, generator=g).to(torch.bfloat16)
            p = torch.cat([torch.randn(6, generator=g), torch.tensor([7.5, float(flags)])]).float()
            want = _ref_multistep(lat, eps, hist, saved, p, cfg)
            d_lat, d_hist, d_saved = lat.cuda(), hist.cuda(), saved.cuda()
            L.op_denoise_multistep(d_lat, eps.cuda(), d_hist, d_saved, p.cuda(), cfg)
            for got, ref, what in zip((d_lat, d_hist, d_saved), want, ("latents", "history", "saved")):
                assert torch.equal(_bits(got.cpu()), _bits(ref)), (B, cfg, flags, h, w, what)
