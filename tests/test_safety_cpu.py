"""CPU: the safety checker's oracle is pinned to transformers (pre-processing, tower), its head behaves as diffusers' does,
the published configuration adds up, and the new C entry points refuse bad arguments without a GPU."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import safety_oracle as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG_DIR = os.path.join(ROOT, "tests", "golden", "emu2_diffusion_config")
SHAPES = [(1024, 1024), (512, 768), (768, 512), (300, 301), (225, 1000)]   # (H, W)


def _image(h, w, seed):
    g = np.random.default_rng(seed)
    base = g.integers(0, 256, (h // 8 + 1, w // 8 + 1, 3), dtype=np.uint8)   # smooth-ish content, plus full-range noise
    img = np.repeat(np.repeat(base, 8, 0), 8, 1)[:h, :w].astype(np.int32) + g.integers(-40, 41, (h, w, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


@pytest.mark.parametrize("hw", SHAPES)
def test_preprocess_oracle_vs_clip_image_processor_pil(hw):
    from PIL import Image
    from transformers import CLIPImageProcessorPil
    proc = CLIPImageProcessorPil.from_pretrained(os.path.join(CFG_DIR, "feature_extractor"))
    img = _image(*hw, seed=hw[0] + hw[1])
    ref = proc(Image.fromarray(img), return_tensors="pt").pixel_values[0].numpy()
    got = S.preprocess(img)
    assert got.shape == ref.shape == (3, 224, 224)
    assert np.array_equal(got.view(np.uint32), ref.astype(np.float32).view(np.uint32))


def test_tower_oracle_fp32_vs_transformers_clip_vision_model():
    from transformers import CLIPVisionConfig, CLIPVisionModel
    cfg = dict(image_size=56, patch_size=14, width=128, layers=2, heads=2, mlp=512, proj_dim=64, n_special=3, n_concepts=17,
               ln_eps=1e-5)
    vc = CLIPVisionConfig(hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2, image_size=56,
                          patch_size=14, hidden_act="quick_gelu", layer_norm_eps=1e-5, attn_implementation="eager")
    model = CLIPVisionModel(vc).eval()
    sd = S.random_state_dict(cfg, seed=3)
    tower = {k[len("vision_model."):]: v for k, v in sd.items() if k.startswith(S.TOWER)}
    missing, unexpected = model.load_state_dict(tower, strict=False)
    assert not [m for m in missing if not m.endswith("position_ids")] and not unexpected
    px = torch.randn(2, 3, 56, 56, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        pooled = model(pixel_values=px).pooler_output
        ref = torch.nn.functional.linear(pooled, sd["visual_projection.weight"])
        got = S.tower(sd, px, cfg)
    assert (got - ref).abs().max().item() <= 1e-5


def test_published_checker_parameter_count():
    """303,179,776 in the tower + 786,432 projection + 20 x 768 embeddings + 20 thresholds"""
    shapes = S.param_shapes(S.VIT_L14)
    total = sum(int(np.prod(s)) for s in shapes.values())
    assert total == 303_981_588
    tower = sum(int(np.prod(s)) for k, s in shapes.items() if k.startswith(S.TOWER))
    assert tower == 303_179_776


def test_published_config_matches_fixture():
    import json
    from emu_b200.safety import SafetyChecker
    a = SafetyChecker()
    b = SafetyChecker(os.path.join(CFG_DIR, "safety_checker"), os.path.join(CFG_DIR, "feature_extractor"))
    for c in (a.scfg, b.scfg):
        assert (c.image_size, c.patch_size, c.width, c.layers, c.heads, c.mlp, c.proj_dim) == (224, 14, 1024, 24, 16, 4096, 768)
        assert (c.n_special, c.n_concepts, c.resize_shortest_edge, c.crop_size) == (3, 17, 224, 224)
    assert list(a.scfg.image_mean) == list(b.scfg.image_mean) and list(a.scfg.image_std) == list(b.scfg.image_std)
    assert json.load(open(os.path.join(CFG_DIR, "safety_checker", "config.json")))["vision_config"]["hidden_act"] == "quick_gelu"


def _head_sd(special_w, concept_w, proj=10):
    """unit embeddings along the axes: special-care j = axis j, concepts cycle over axes 3..7; axis 9 is free"""
    sd = {"special_care_embeds": torch.eye(3, proj), "concept_embeds": torch.eye(proj)[[3 + j % 5 for j in range(17)]],
          "special_care_embeds_weights": torch.tensor(special_w, dtype=torch.float32),
          "concept_embeds_weights": torch.tensor(concept_w, dtype=torch.float32)}
    return sd


def _unit(**axes):
    e = torch.zeros(1, 10)
    for k, v in axes.items():
        e[0, int(k[1:])] = v
    e[0, 9] = (1 - float((e ** 2).sum())) ** 0.5
    return e


def test_head_special_care_lifts_a_concept_just_below_its_threshold():
    """a concept whose raw score lies in (-0.01, 0) fires only when a special-care concept fired first"""
    sd = _head_sd([0.5, 0.9, 0.9], [0.605] + [0.9] * 16)
    emb = torch.cat([_unit(a0=0.7, a3=0.6), _unit(a0=0.3, a3=0.6)])   # concept 0: cos 0.6, raw score -0.005
    has, ss, cs, _, _ = S.head(sd, emb)
    assert ss[0, 0] > 0 and ss[1, 0] < 0
    assert -0.01 < cs[1, 0] < 0 and not has[1]
    assert 0 < cs[0, 0] < 0.01 and has[0]


def test_head_adjustment_carries_to_later_special_care_index():
    """special-care 0 fires, which lifts special-care 1 (raw score just below 0) over its threshold too"""
    sd = _head_sd([0.1, 0.605, 0.9], [2.0] * 17)
    emb = _unit(a0=0.8, a1=0.6)                      # special-care 1: raw -0.005, adjusted +0.005
    has, ss, cs, _, _ = S.head(sd, emb)
    assert ss[0, 0] > 0 and 0 < ss[0, 1] < 0.01
    assert not has[0]                                # no concept fires: the adjustment alone flags nothing


def test_blackout_zeros_flagged_images_only():
    g = np.random.default_rng(0)
    imgs = g.integers(1, 256, (3, 5, 7, 3), dtype=np.uint8)
    out = S.blackout(imgs, [False, True, False])
    assert out.dtype == np.uint8 and not out[1].any()
    assert np.array_equal(out[0], imgs[0]) and np.array_equal(out[2], imgs[2])


@pytest.fixture(scope="module")
def lib():
    from emu_b200 import _lib, build
    build.build()
    return _lib.load()


def test_safety_symbols_exported_and_listed(lib):
    import re
    from emu_b200 import _lib
    src = open(os.path.join(ROOT, "include", "emu_b200_safety.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    syms = sorted(set(re.findall(r"\b(emu_[a-z0-9_]+)\s*\(", src)))
    assert syms == sorted(_lib.SAFETY_SYMBOLS)
    assert all(hasattr(lib, s) for s in syms)


def test_safety_config_struct_layout_matches_header():
    import re
    from emu_b200 import _lib
    src = open(os.path.join(ROOT, "include", "emu_b200_safety.h")).read()
    body = re.search(r"typedef struct EmuSafetyConfig \{(.*?)\} EmuSafetyConfig;", src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        decl = re.sub(r"^(int|float)\s+", "", decl.strip())
        names += [re.sub(r"\[.*\]", "", n.strip()) for n in decl.split(",") if n.strip()]
    assert names == [f[0] for f in _lib.EmuSafetyConfig._fields_]
    assert ctypes.sizeof(_lib.EmuSafetyConfig) == 4 * (len(names) + 4)


def test_safety_entry_points_refuse_bad_arguments(lib):
    """NULL or out-of-range arguments are EMU_ERR_INVALID before any CUDA call (so also without a GPU)"""
    N, P = None, ctypes.c_void_p
    img, out, flags = P(0x10000000), P(0x20000000), P(0x30000000)
    m3 = (ctypes.c_float * 3)(0.5, 0.5, 0.5)
    calls = [
        ("emu_safety_configure", (N, N)),
        ("emu_safety_check", (N, img, 1, 64, 64, flags, N, N)),
        ("emu_safety_embed", (N, img, 1, out, N)),
        ("emu_preprocess_clip", (N, 1, 64, 64, 224, 224, m3, m3, out, 1, N)),
        ("emu_preprocess_clip", (img, 0, 64, 64, 224, 224, m3, m3, out, 1, N)),
        ("emu_preprocess_clip", (img, 1, 0, 64, 224, 224, m3, m3, out, 1, N)),
        ("emu_preprocess_clip", (img, 1, 64, 64, 224, 256, m3, m3, out, 1, N)),   # crop larger than the resized image
        ("emu_preprocess_clip", (img, 1, 64, 64, 224, 224, N, m3, out, 1, N)),
        ("emu_preprocess_clip", (img, 1, 64, 64, 224, 224, m3, m3, out, 7, N)),    # unknown dtype
        ("emu_preprocess_clip", (img, 1, 64, 64, 224, 224, m3, m3, N, 1, N)),
    ]
    for name, args in calls:
        fn = getattr(lib, name)
        fn.restype = ctypes.c_int
        assert fn(*args) == -1, (name, args)


def test_quick_gelu_mode_is_exported():
    from emu_b200 import _lib
    assert _lib.EPI_QUICK_GELU == 5
