"""CPU: the decode-step operators of include/emu_b200_ops.h are bound and exported, and refuse bad arguments before any
CUDA call (so also on a machine without a GPU).  Their numerics are in tests/test_decode_ops_gpu.py."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "emu_b200_ops.h")


@pytest.fixture(scope="module")
def lib():
    from emu_b200 import build, _lib
    build.build()
    return _lib.load()


def test_ops_header_symbols_are_bound_and_exported(lib):
    from emu_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(emu_[a-z0-9_]+)\s*\(", src)))
    assert sorted(_lib.OPS_SYMBOLS) == syms
    assert all(hasattr(lib, s) for s in syms)
    # the pinned symbol set of emu_b200.h stays as it is: the operators live only in the companion header
    assert not set(_lib.OPS_SYMBOLS) & set(_lib.SYMBOLS)


# addresses that are never dereferenced: every call below must be refused on its arguments alone
P = ctypes.c_void_p(0x10000000)
F = ctypes.c_float(0.125)
ST12 = (ctypes.c_int64 * 12)(*([8] * 12))


def _good_args():
    """one valid argument list per entry point (never called as is: tests/test_decode_ops_gpu.py runs the real ones)"""
    N = None
    return {
        #                         q  k  v  B  H  D    T    pos start indir scale out hint stream
        "emu_op_attn_decode_rows": [P, P, P, 4, 2, 128, 256, P, N, N, F, P, 256, N],
        #                      qkv B  N  H  D    cos sin off pos0 pos_dev q_out kv_row kc vc T   stream
        "emu_op_rope_kv_write": [P, 4, 8, 2, 128, P, P, N, 0, N, N, N, P, P, 64, N],
        #                        indir src row_len B  T   n_tok stream
        "emu_op_kv_indir_update": [P, P, N, 4, 64, 10, N],
        #                   cache Bcap src B outer n_used H D   T  stream
        "emu_op_kv_reorder": [P, 8, P, 4, 2, 10, 2, 128, 64, N],
        #                    logits rows cols out stream
        "emu_op_argmax_rows": [P, 4, 1000, P, N],
        #                          q  k  v  out B  H  Nq  Nk  D    st12  scale causal kv_start kv_row kv_rows stream
        "emu_op_attn_prefill_rows": [P, P, P, P, 4, 2, 128, 128, 128, ST12, F, 1, N, P, 32, N],
    }


# (entry point, argument index, bad value, what it is)
BAD = [
    ("emu_op_attn_decode_rows", 0, None, "q"), ("emu_op_attn_decode_rows", 1, None, "k_cache"),
    ("emu_op_attn_decode_rows", 2, None, "v_cache"), ("emu_op_attn_decode_rows", 7, None, "pos"),
    ("emu_op_attn_decode_rows", 11, None, "out"), ("emu_op_attn_decode_rows", 3, 0, "B = 0"),
    ("emu_op_attn_decode_rows", 3, 33, "B = 33"), ("emu_op_attn_decode_rows", 5, 96, "D = 96"),
    ("emu_op_attn_decode_rows", 5, 0, "D = 0"), ("emu_op_attn_decode_rows", 4, 0, "H = 0"),
    ("emu_op_attn_decode_rows", 6, 0, "t_max = 0"), ("emu_op_attn_decode_rows", 12, 0, "max_len_hint = 0"),
    ("emu_op_attn_decode_rows", 12, 257, "max_len_hint > t_max"),
    ("emu_op_rope_kv_write", 0, None, "qkv"), ("emu_op_rope_kv_write", 5, None, "cos"),
    ("emu_op_rope_kv_write", 6, None, "sin"), ("emu_op_rope_kv_write", 12, None, "k_cache"),
    ("emu_op_rope_kv_write", 13, None, "v_cache"), ("emu_op_rope_kv_write", 1, 0, "B = 0"),
    ("emu_op_rope_kv_write", 1, 33, "B = 33"), ("emu_op_rope_kv_write", 4, 80, "D = 80"),
    ("emu_op_rope_kv_write", 2, 0, "N = 0"), ("emu_op_rope_kv_write", 3, 0, "H = 0"),
    ("emu_op_rope_kv_write", 14, 0, "t_max = 0"), ("emu_op_rope_kv_write", 8, 60, "pos0 + N > t_max"),
    ("emu_op_rope_kv_write", 8, -1, "pos0 < 0"),
    ("emu_op_kv_indir_update", 0, None, "indir"), ("emu_op_kv_indir_update", 1, None, "src_idx"),
    ("emu_op_kv_indir_update", 3, 0, "B = 0"), ("emu_op_kv_indir_update", 3, 33, "B = 33"),
    ("emu_op_kv_indir_update", 5, 0, "n_tok = 0"), ("emu_op_kv_indir_update", 5, 65, "n_tok > t_max"),
    ("emu_op_kv_indir_update", 4, 0, "t_max = 0"),
    ("emu_op_kv_reorder", 0, None, "cache"), ("emu_op_kv_reorder", 2, None, "src_idx"),
    ("emu_op_kv_reorder", 3, 0, "B = 0"), ("emu_op_kv_reorder", 3, 33, "B = 33"), ("emu_op_kv_reorder", 1, 3, "Bcap < B"),
    ("emu_op_kv_reorder", 7, 100, "D = 100"), ("emu_op_kv_reorder", 4, 0, "outer = 0"), ("emu_op_kv_reorder", 6, 0, "H = 0"),
    ("emu_op_kv_reorder", 5, 0, "n_used_tokens = 0"), ("emu_op_kv_reorder", 5, 65, "n_used_tokens > t_max"),
    ("emu_op_argmax_rows", 0, None, "logits"), ("emu_op_argmax_rows", 3, None, "out"), ("emu_op_argmax_rows", 1, 0, "rows = 0"),
    ("emu_op_argmax_rows", 2, 0, "cols = 0"), ("emu_op_argmax_rows", 2, -5, "cols < 0"),
    ("emu_op_attn_prefill_rows", 0, None, "q"), ("emu_op_attn_prefill_rows", 1, None, "k"),
    ("emu_op_attn_prefill_rows", 2, None, "v"), ("emu_op_attn_prefill_rows", 3, None, "out"),
    ("emu_op_attn_prefill_rows", 9, None, "st12"), ("emu_op_attn_prefill_rows", 4, 0, "B = 0"),
    ("emu_op_attn_prefill_rows", 4, 33, "B = 33"), ("emu_op_attn_prefill_rows", 8, 12, "D = 12"),
    ("emu_op_attn_prefill_rows", 8, 168, "D = 168"), ("emu_op_attn_prefill_rows", 6, 0, "Nq = 0"),
    ("emu_op_attn_prefill_rows", 7, 0, "Nk = 0"), ("emu_op_attn_prefill_rows", 5, 0, "H = 0"),
    ("emu_op_attn_prefill_rows", 14, 0, "kv_rows = 0 with kv_row"), ("emu_op_attn_prefill_rows", 14, 33, "kv_rows = 33"),
]


def test_every_entry_point_is_exercised_by_the_refusals():
    assert {b[0] for b in BAD} == set(_good_args())


@pytest.mark.parametrize("name,i,bad,what", BAD, ids=["%s: %s" % (b[0], b[3]) for b in BAD])
def test_bad_arguments_are_refused_before_any_cuda_call(lib, name, i, bad, what):
    """NULL pointers, a batch outside 1..32, an unsupported head width and non-positive sizes come back as EMU_ERR_INVALID.
    The pointers are fake: without a GPU a CUDA call made anyway would come back as a CUDA error, not EMU_ERR_INVALID.  With a
    GPU a missed check would launch on fake addresses, so the test runs only where there is none."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("fake device addresses: checked on a machine without a GPU")
    args = _good_args()[name]
    args[i] = bad
    fn = getattr(lib, name)
    fn.restype, fn.argtypes = ctypes.c_int, None
    assert fn(*args) == -1, (name, what)
