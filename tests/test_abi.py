"""CPU: the C-ABI library builds/loads and exports every symbol include/emu_b200.h declares; argument validation
that needs no GPU behaves (no compute calls here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "emu_b200.h")


def header_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(emu_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
    from emu_b200 import build, _lib
    build.build()
    return _lib.load()


def test_header_symbols_exported(lib):
    syms = header_symbols()
    assert len(syms) >= 25
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, missing


def test_python_binding_lists_every_symbol():
    from emu_b200 import _lib
    assert sorted(_lib.SYMBOLS) == header_symbols()


def test_version_and_counter(lib):
    assert b"sm_90a" in lib.emu_version()
    assert lib.emu_launch_count() >= 0


def test_config_struct_layout_matches_header():
    """EmuConfig in _lib.py must have the same field order/size as the C struct (all 4-byte fields)."""
    from emu_b200 import _lib
    src = open(HEADER).read()
    body = re.search(r"typedef struct EmuConfig \{(.*?)\} EmuConfig;", src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        decl = re.sub(r"^(int|float)\s+", "", decl)
        for n in decl.split(","):
            names.append(re.sub(r"\[.*\]", "", n.strip()))
    assert names == [f[0] for f in _lib.EmuConfig._fields_]
    assert ctypes.sizeof(_lib.EmuConfig) == 4 * (len(names) - 1) + 4 * 8


def test_no_cpu_fallback(lib):
    """Without a GPU the engine refuses to come up (EMU_ERR_CUDA) instead of computing on the host."""
    import torch
    from emu_b200 import _lib
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    cfg = _lib.EmuConfig()
    h = ctypes.c_void_p()
    assert lib.emu_engine_create(ctypes.byref(cfg), 0, 1, None, ctypes.byref(h)) == -2
    with pytest.raises(_lib.EmuError):
        _lib.Engine(cfg)


def test_product_never_imports_oracle():
    """The package must not route through oracle/ (test infrastructure only)."""
    pkg = os.path.join(ROOT, "emu_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt, f


def _struct_fields(name):
    src = open(HEADER).read()
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    out = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        decl = re.sub(r"^(int|float)\s+", "", decl)
        for n in decl.split(","):
            m = re.match(r"(\w+)(?:\[(\d+)\])?", n.strip())
            out.append((m.group(1), int(m.group(2) or 1)))
    return out


@pytest.mark.parametrize("name", ["EmuUNetConfig", "EmuVAEConfig"])
def test_diffusion_config_struct_layouts_match_header(name):
    """field order and array lengths of the ctypes mirrors == the C structs (every field is a 4-byte int / float)"""
    from emu_b200 import _lib
    cls = getattr(_lib, name)
    mine = [(f[0], ctypes.sizeof(f[1]) // 4) for f in cls._fields_]
    assert mine == _struct_fields(name)
    assert ctypes.sizeof(cls) == 4 * sum(n for _, n in mine)


def test_null_arguments_are_refused_not_dereferenced(lib):
    """Every entry point validates its handle / pointers before doing anything (header: "return value 0 = ok, negative = error
    ... nothing throws or aborts"): a NULL engine or NULL buffers come back as EMU_ERR_INVALID, also on a machine without a GPU."""
    N, F = None, ctypes.c_float
    calls = {
        "emu_engine_create": (N, 0, 1, N, N),
        "emu_engine_load_tensor": (N, b"k", N, 1, N, 0, N),
        "emu_vit_forward": (N, N, 1, N, 4, 1, N),
        "emu_llm_reset": (N, N),
        "emu_llm_embed": (N, N, 1, N, N),
        "emu_llm_prefill": (N, N, N, 1, 1, 1, N, N, N),
        "emu_llm_decode": (N, N, N, N, 1, N, N, N, -1, N),
        "emu_llm_expand": (N, N, 1, N),
        "emu_project": (N, 0, N, 1, N, N),
        "emu_cformer_forward": (N, N, 1, 1, N, N),
        "emu_unet_configure": (N, N),
        "emu_vae_configure": (N, N),
        "emu_vae_decode": (N, N, 1, 1, 1, N, N),
        "emu_beam_topk": (N, N, 1, 1, 10, 2, -1, N, 0, 0, ctypes.c_float(1.0), 0, 0, N, N, N, N),
        "emu_beam_step": (N, N, 1, 1, 10, 0, 4, 2, ctypes.c_float(1.0), ctypes.c_float(1.0), 0, N, N, N, N, N, N, N, N, N, N, N),
        "emu_sample_tokens": (N, 1, 1, F(1.0), 0, F(1.0), -1, ctypes.c_uint64(0), ctypes.c_uint64(0), N, N),
        "emu_unet_forward": (N, N, F(0.0), N, 1, N, N, 1, 1, 1, N, N),
        "emu_denoise_step": (N, N, F(1.0), F(0.5), F(1.0), F(3.0), N, 1, N, N, 1, 1, 1, N),
        "emu_denoise_step_multistep": (N, N, N, N, F(1.0), F(3.0), N, 1, 1, 1, 1, N),
        "emu_preprocess_image": (N, 1, 1, 1, 1, N, N, N, 0, N),
        "emu_image_to_uint8": (N, N, ctypes.c_int64(1), N),
        "emu_tp_head_range": (4, 2, 0, N, N),
        # the stand-alone operators take bare pointers: same rule
        "emu_op_gemm": (N, 0, N, 0, 1, 1, 1, N, N, 0, 0, N, 0, 0, 0, N),
        "emu_op_gemm_skinny": (N, 0, N, 0, 1, 1, 1, N, 0, 0, N, 0, 0, N),
        "emu_op_conv3x3": (N, 1, 1, 1, 1, N, 1, N, N, N, N),
        "emu_op_gemv": (N, 1, 1, N, 0, 1, N, F(1e-6), 0, N, N, 0, N, 0, 0, 0, N),
        "emu_op_gemv_rope_qkv": (N, 1, 1, 1, N, 0, 1, N, F(1e-6), N, N, N, N, N, N, N, 1, N),
        "emu_op_attn_prefill": (N, N, N, N, 1, 1, 1, 1, 1, N, F(1.0), 0, N, N, N),
        "emu_op_attn_decode": (N, N, N, 1, 1, 1, 1, N, N, F(1.0), N, 1, N),
        "emu_op_rmsnorm": (N, N, N, 1, 1, F(1e-6), N),
        "emu_op_layernorm": (N, N, N, N, N, 1, 1, F(1e-6), N),
        "emu_debug_gemm_phases": (N, 0, N, 0, 1, 1, 1, N, N, 0, 0, N, 0, 0, N, N),
        "emu_debug_gemv_phases": (N, 1, 1, N, 0, 1, N, F(1e-6), 0, N, 0, N, 0, 0, N, N),
    }
    skipped = set(header_symbols()) - set(calls)          # what is left takes no pointer that could be NULL-checked this way
    assert skipped == {"emu_engine_destroy", "emu_last_error", "emu_nccl_unique_id", "emu_llm_cur_len", "emu_launch_count",
                       "emu_version"}, skipped
    for name, args in calls.items():
        fn = getattr(lib, name)
        fn.restype = ctypes.c_int
        saved = fn.argtypes
        fn.argtypes = None                       # raw call: ctypes converts None -> NULL, ints -> int
        try:
            rc = fn(*args)
        finally:
            fn.argtypes = saved
        assert rc == -1, (name, rc)
    assert lib.emu_llm_cur_len(None) == -1


@pytest.mark.parametrize("w_off,x_off", [(8, 0), (0, 8), (2, 2)])
def test_gemv_refuses_misaligned_operands(lib, w_off, x_off):
    """W is read by TMA and x by bulk copies, so both must be 16-byte aligned: anything else is EMU_ERR_INVALID, decided before
    any pointer is dereferenced or any CUDA call is made (the addresses below are never touched)."""
    P = ctypes.c_void_p
    base = 0x10000000
    W, x, y = P(base + w_off), P(base + 0x100000 + x_off), P(base + 0x200000)
    N = K = 64
    rc = lib.emu_op_gemv(W, N, K, x, K, 1, None, ctypes.c_float(1e-6), 0, None, None, 0, y, N, 0, 0, None)
    assert rc == -1
