"""CPU: the diffusion operators of include/emu_b200_diffusion_ops.h are bound and exported, and refuse bad arguments before
any CUDA call (so also on a machine without a GPU).  Their numerics are in tests/test_diffusion_ops_gpu.py."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "emu_b200_diffusion_ops.h")


@pytest.fixture(scope="module")
def lib():
    from emu_b200 import build, _lib
    build.build()
    return _lib.load()


def test_diffusion_ops_header_symbols_are_bound_and_exported(lib):
    from emu_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(emu_[a-z0-9_]+)\s*\(", src)))
    assert sorted(_lib.DIFFUSION_OPS_SYMBOLS) == syms
    assert all(hasattr(lib, s) for s in syms)
    # the pinned symbol set of emu_b200.h and the other companion headers stay as they are
    others = set(_lib.SYMBOLS) | set(_lib.OPS_SYMBOLS) | set(_lib.GEN_SLOT_SYMBOLS)
    assert not set(_lib.DIFFUSION_OPS_SYMBOLS) & others


# addresses that are never dereferenced: every call below must be refused on its arguments alone
P = ctypes.c_void_p(0x10000000)
EPS = ctypes.c_float(1e-5)
ONE = ctypes.c_float(1.0)
I64 = ctypes.c_int64


def _good_args():
    """one valid argument list per entry point (never called as is: tests/test_diffusion_ops_gpu.py runs the real ones)"""
    N = None
    return {
        #                  x  w  b  y  NB HW    C    groups eps silu stream
        "emu_op_groupnorm": [P, P, P, P, 2, 4096, 320, 32, EPS, 1, N],
        #                           t  out rows dim  ld    col_off grp stream
        "emu_op_timestep_embedding": [P, P, 12, 256, 3328, 1792, 6, N],
        #                   x  y  NB H   W   C    stream
        "emu_op_upsample2x": [P, P, 2, 32, 32, 640, N],
        #                  x  out NB H   W   C    stride stream
        "emu_op_im2col3x3": [P, P, 2, 64, 64, 320, 2, N],
        #                  src dst rows       cols lds  ldd  col_off stream
        "emu_op_copy_cols": [P, P, I64(4096), 640, 640, 960, 320, N],
        #                     x  y  NB C  HW     Cp scale stream
        "emu_op_nchw_to_nhwc": [P, P, 2, 4, 16384, 8, ONE, N],
        #                     x  y  NB C  HW     ldx stream
        "emu_op_nhwc_to_nchw": [P, P, 2, 4, 16384, 8, N],
        #                    x  y  B  L   C     stream
        "emu_op_mean_tokens": [P, P, 2, 64, 1792, N],
        #                 x  y  n_pix         C  ldx stream
        "emu_op_vae_post": [P, P, I64(1 << 20), 3, 8, N],
        #                          lat eps hist saved B  C  HW    ld params cfg stream
        "emu_op_denoise_multistep": [P, P, P, P, 2, 4, 4096, 8, P, 1, N],
        #                      q  k  v  out B  T      C    stream
        "emu_op_vae_attention": [P, P, P, P, 1, 16384, 512, N],
    }


# (entry point, argument index, bad value, what it is)
BAD = [
    ("emu_op_groupnorm", 0, None, "x"), ("emu_op_groupnorm", 1, None, "w"), ("emu_op_groupnorm", 2, None, "b"),
    ("emu_op_groupnorm", 3, None, "y"), ("emu_op_groupnorm", 4, 0, "NB = 0"), ("emu_op_groupnorm", 5, 0, "HW = 0"),
    ("emu_op_groupnorm", 6, 0, "C = 0"), ("emu_op_groupnorm", 7, 0, "groups = 0"), ("emu_op_groupnorm", 6, 324, "C % 8"),
    ("emu_op_groupnorm", 7, 48, "C % groups"), ("emu_op_groupnorm", 6, 4352, "C > 4096"),
    ("emu_op_timestep_embedding", 0, None, "t"), ("emu_op_timestep_embedding", 1, None, "out"),
    ("emu_op_timestep_embedding", 2, 0, "rows = 0"), ("emu_op_timestep_embedding", 3, 0, "dim = 0"),
    ("emu_op_timestep_embedding", 3, 255, "odd dim"), ("emu_op_timestep_embedding", 6, 0, "grp = 0"),
    ("emu_op_timestep_embedding", 4, 3327, "ld < col_off + grp * dim"), ("emu_op_timestep_embedding", 5, -8, "col_off < 0"),
    ("emu_op_upsample2x", 0, None, "x"), ("emu_op_upsample2x", 1, None, "y"), ("emu_op_upsample2x", 2, 0, "NB = 0"),
    ("emu_op_upsample2x", 3, 0, "H = 0"), ("emu_op_upsample2x", 4, -1, "W < 0"), ("emu_op_upsample2x", 5, 0, "C = 0"),
    ("emu_op_upsample2x", 5, 644, "C % 8"),
    ("emu_op_im2col3x3", 0, None, "x"), ("emu_op_im2col3x3", 1, None, "out"), ("emu_op_im2col3x3", 2, 0, "NB = 0"),
    ("emu_op_im2col3x3", 3, 0, "H = 0"), ("emu_op_im2col3x3", 4, 0, "W = 0"), ("emu_op_im2col3x3", 5, 0, "C = 0"),
    ("emu_op_im2col3x3", 5, 4, "C % 8"), ("emu_op_im2col3x3", 6, 3, "stride = 3"), ("emu_op_im2col3x3", 6, 0, "stride = 0"),
    ("emu_op_copy_cols", 0, None, "src"), ("emu_op_copy_cols", 1, None, "dst"), ("emu_op_copy_cols", 2, I64(0), "rows = 0"),
    ("emu_op_copy_cols", 3, 0, "cols = 0"), ("emu_op_copy_cols", 3, 636, "cols % 8"), ("emu_op_copy_cols", 4, 644, "lds % 8"),
    ("emu_op_copy_cols", 5, 964, "ldd % 8"), ("emu_op_copy_cols", 6, 4, "col_off % 8"),
    ("emu_op_copy_cols", 4, 632, "lds < cols"), ("emu_op_copy_cols", 5, 952, "ldd < col_off + cols"),
    ("emu_op_copy_cols", 6, -8, "col_off < 0"),
    ("emu_op_nchw_to_nhwc", 0, None, "x"), ("emu_op_nchw_to_nhwc", 1, None, "y"), ("emu_op_nchw_to_nhwc", 2, 0, "NB = 0"),
    ("emu_op_nchw_to_nhwc", 3, 0, "C = 0"), ("emu_op_nchw_to_nhwc", 4, 0, "HW = 0"), ("emu_op_nchw_to_nhwc", 5, 3, "Cp < C"),
    ("emu_op_nhwc_to_nchw", 0, None, "x"), ("emu_op_nhwc_to_nchw", 1, None, "y"), ("emu_op_nhwc_to_nchw", 2, 0, "NB = 0"),
    ("emu_op_nhwc_to_nchw", 3, 0, "C = 0"), ("emu_op_nhwc_to_nchw", 4, 0, "HW = 0"), ("emu_op_nhwc_to_nchw", 5, 3, "ldx < C"),
    ("emu_op_mean_tokens", 0, None, "x"), ("emu_op_mean_tokens", 1, None, "y"), ("emu_op_mean_tokens", 2, 0, "B = 0"),
    ("emu_op_mean_tokens", 3, 0, "L = 0"), ("emu_op_mean_tokens", 4, 0, "C = 0"),
    ("emu_op_vae_post", 0, None, "x"), ("emu_op_vae_post", 1, None, "y"), ("emu_op_vae_post", 2, I64(0), "n_pix = 0"),
    ("emu_op_vae_post", 3, 0, "C = 0"), ("emu_op_vae_post", 4, 2, "ldx < C"),
    ("emu_op_denoise_multistep", 0, None, "latents"), ("emu_op_denoise_multistep", 1, None, "eps"),
    ("emu_op_denoise_multistep", 2, None, "hist"), ("emu_op_denoise_multistep", 3, None, "saved"),
    ("emu_op_denoise_multistep", 8, None, "params"), ("emu_op_denoise_multistep", 4, 0, "B = 0"),
    ("emu_op_denoise_multistep", 5, 0, "C = 0"), ("emu_op_denoise_multistep", 6, 0, "HW = 0"),
    ("emu_op_denoise_multistep", 7, 3, "ld < C"), ("emu_op_denoise_multistep", 9, 2, "cfg = 2"),
    ("emu_op_vae_attention", 0, None, "q"), ("emu_op_vae_attention", 1, None, "k"), ("emu_op_vae_attention", 2, None, "v"),
    ("emu_op_vae_attention", 3, None, "out"), ("emu_op_vae_attention", 4, 0, "B = 0"), ("emu_op_vae_attention", 5, 0, "T = 0"),
    ("emu_op_vae_attention", 6, 0, "C = 0"), ("emu_op_vae_attention", 6, 500, "C % 8"),
    ("emu_op_vae_attention", 5, 16383, "T % 8"),
]


def test_every_entry_point_is_exercised_by_the_refusals():
    assert {b[0] for b in BAD} == set(_good_args())


@pytest.mark.parametrize("name,i,bad,what", BAD, ids=["%s: %s" % (b[0], b[3]) for b in BAD])
def test_bad_arguments_are_refused_before_any_cuda_call(lib, name, i, bad, what):
    """NULL pointers, non-positive sizes, channel counts the vectorised kernels cannot take, a GroupNorm C that the groups do
    not divide or above 4096, an im2col stride outside {1, 2}, an odd embedding width and a padded width or row stride below
    the channel count come back as EMU_ERR_INVALID.  The pointers are fake: without a GPU a CUDA call made anyway would come
    back as a CUDA error, not EMU_ERR_INVALID.  With a GPU a missed check would launch on fake addresses, so the test runs
    only where there is none."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("fake device addresses: checked on a machine without a GPU")
    args = _good_args()[name]
    args[i] = bad
    fn = getattr(lib, name)
    fn.restype, fn.argtypes = ctypes.c_int, None
    assert fn(*args) == -1, (name, what)
