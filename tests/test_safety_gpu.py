"""The safety checker on the GPU against oracle/safety_oracle.py: CLIP pre-processing bit for bit, the quick-GELU GEMM
epilogue, the tower's image_embeds (tiny and real ViT-L/14 width), the head's flags and black-out, and the two pipelines
routing their images through a built-in SafetyChecker."""
import numpy as np
import pytest
import torch

from helpers import assert_bf16_parity
from oracle import emu_oracle as O
from oracle import safety_oracle as S

pytestmark = pytest.mark.gpu

SHAPES = [(1024, 1024), (512, 768), (768, 512), (300, 301), (225, 1000)]
TINY = dict(image_size=224, patch_size=14, width=128, layers=2, heads=2, mlp=512, proj_dim=64, n_special=3, n_concepts=17,
            ln_eps=1e-5)


def _images(B, h, w, seed):
    g = np.random.default_rng(seed)
    return g.integers(0, 256, (B, h, w, 3), dtype=np.uint8)


def _scfg(cfg):
    from emu_b200 import _lib
    c = _lib.EmuSafetyConfig()
    for k in ("image_size", "patch_size", "width", "layers", "heads", "mlp", "proj_dim", "n_special", "n_concepts"):
        setattr(c, k, cfg[k])
    c.ln_eps, c.resize_shortest_edge, c.crop_size = cfg["ln_eps"], cfg["image_size"], cfg["image_size"]
    for i in range(3):
        c.image_mean[i], c.image_std[i] = S.CLIP_MEAN[i], S.CLIP_STD[i]
    return c


def _checker(cfg, sd):
    from emu_b200.safety import SafetyChecker
    ck = SafetyChecker()
    ck.scfg = _scfg(cfg)
    ck.load_state_dict(sd)
    return ck


@pytest.mark.parametrize("hw", SHAPES)
def test_preprocess_clip_bit_exact(cuda, hw):
    from emu_b200 import _lib
    imgs = _images(3, *hw, seed=hw[0] * 7 + hw[1])
    ref = np.stack([S.preprocess(im) for im in imgs])
    dev = torch.from_numpy(imgs).to(cuda)
    got32 = _lib.op_preprocess_clip(dev, dtype=torch.float32).cpu().numpy()
    got16 = _lib.op_preprocess_clip(dev, dtype=torch.bfloat16).cpu()
    assert np.array_equal(got32.view(np.uint32), ref.view(np.uint32))
    assert torch.equal(got16, torch.from_numpy(ref).to(torch.bfloat16))


def test_gemm_quick_gelu_epilogue(cuda):
    from emu_b200 import _lib
    g = torch.Generator().manual_seed(5)
    M, N, K = 257 * 2, 512, 256
    A = (torch.randn(M, K, generator=g)).to(torch.bfloat16)
    W = (torch.randn(N, K, generator=g) / 16).to(torch.bfloat16)
    b = (torch.randn(N, generator=g) * 0.1).to(torch.bfloat16)
    h32 = A.float() @ W.float().t() + b.float()
    ref32 = h32 * torch.sigmoid(1.702 * h32)
    got = _lib.op_gemm(A.to(cuda), W.to(cuda), bias=b.to(cuda), epi=_lib.EPI_QUICK_GELU).float().cpu()
    assert O.rel_err(got, ref32) <= 6e-3
    h = h32.to(torch.bfloat16)                               # the reference's bf16 rounding points
    ref16 = (h * torch.sigmoid(1.702 * h)).float()
    assert O.rel_err(got, ref16) <= 6e-3


@pytest.mark.parametrize("cfg,B", [(TINY, 1), (TINY, 4), (S.VIT_L14, 1), (S.VIT_L14, 4)],
                         ids=["tiny-B1", "tiny-B4", "vitl14-B1", "vitl14-B4"])
def test_tower_image_embeds_parity(cuda, cfg, B):
    sd = S.random_state_dict(cfg, seed=11)
    ck = _checker(cfg, sd)
    px = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(B)).to(torch.bfloat16).float()
    got = ck.embed(px.to(cuda)).float().cpu()
    sd_dev = {k: v.to(cuda) for k, v in sd.items()}
    with torch.no_grad():
        ref32 = S.tower(sd_dev, px.to(cuda), cfg, torch.float32).cpu()
        ref16 = S.tower(sd_dev, px.to(cuda), cfg, torch.bfloat16).float().cpu()
    assert_bf16_parity("safety tower %s B=%d" % (cfg["width"], B), got, ref32, ref16)


def _fire_setup(cuda):
    """tiny tower + four images; concept / special-care embeddings and thresholds placed on the engine's own cosines so that
    image 0 fires a concept outright, image 1 fires one only through the special-care adjustment, images 2 and 3 fire nothing"""
    sd = S.random_state_dict(TINY, seed=21)
    imgs = _images(4, 240, 300, seed=3)
    imgs[2] = 0
    imgs[3, :, :150] = 255
    ck = _checker(TINY, sd)
    dev = torch.from_numpy(imgs).to(cuda)
    from emu_b200 import _lib
    emb = ck.embed(_lib.op_preprocess_clip(dev)).cpu()             # bf16 [4, 64]
    e = emb.double()
    q = (torch.linalg.inv(e @ e.t()) @ e).float()                  # q_i . e_j = delta_ij: each q_i "sees" image i only
    sd["special_care_embeds"] = torch.stack([q[1], q[2] + q[3], -q[0]]).clone()
    sd["concept_embeds"] = torch.stack([q[0], q[1]] + [-q[0] - q[1]] * 15).clone()
    sp = S.cosine_distance(emb, sd["special_care_embeds"].to(torch.bfloat16)).double()
    co = S.cosine_distance(emb, sd["concept_embeds"].to(torch.bfloat16)).double()
    bf = lambda v: float(torch.tensor(float(v)).to(torch.bfloat16))
    sw = [bf(sp[1, 0] / 2), 2.0, 2.0]                                   # special-care 0: image 1 only
    c0 = bf(co[0, 0] / 2)                                               # concept 0: image 0 only
    c1 = bf(co[1, 1] + 0.005)                                           # concept 1: image 1 just below (+0.01 adjustment)
    assert 0.0025 < c1 - co[1, 1] < 0.0075, "concept 1 must sit in (-0.01, 0) for image 1"
    assert c0 < co[0, 0] - 0.01 and co[1:, 0].abs().max() < c0 - 0.01
    assert sp[1, 0] > sw[0] + 0.01 and sp[[0, 2, 3], 0].abs().max() < sw[0] - 0.01
    assert co[[0, 2, 3], 1].abs().max() < c1 - 0.02, "image 1 must be the only one near concept 1"
    sd["special_care_embeds_weights"] = torch.tensor(sw)
    sd["concept_embeds_weights"] = torch.tensor([c0, c1] + [2.0] * 15)
    return sd, imgs


def test_flags_blackout_and_oracle_agreement(cuda):
    sd, imgs = _fire_setup(cuda)
    ck = _checker(TINY, sd)
    dev = torch.from_numpy(imgs.copy()).to(cuda)
    flags, scores = ck.check_device(dev, scores=True)
    flags, scores, out = flags.cpu().tolist(), scores.cpu(), dev.cpu().numpy()
    assert flags == [1, 1, 0, 0]
    assert -0.01 < float(scores[1, 3 + 1]) - 0.01 < 0                    # concept 1 of image 1: raw score in (-0.01, 0)
    assert not out[0].any() and not out[1].any()
    assert np.array_equal(out[2], imgs[2]) and np.array_equal(out[3], imgs[3])
    # the head's flags from the engine's own embeddings (diffusers' code path, bf16 cosines)
    from emu_b200 import _lib
    emb = ck.embed(_lib.op_preprocess_clip(torch.from_numpy(imgs).to(cuda))).cpu()
    has, _, _, _, _ = S.head(sd, emb)
    assert [int(h) for h in has] == flags
    # ... and from the oracle's bf16 tower: equal wherever no score is within one bf16 ulp of cos from its boundary
    px = torch.from_numpy(np.stack([S.preprocess(im) for im in imgs])).to(cuda)
    sd_dev = {k: v.to(cuda) for k, v in sd.items()}
    with torch.no_grad():
        emb_o = S.tower(sd_dev, px, TINY, torch.bfloat16).cpu()
    has_o, ss, cs, scos, cos = S.head(sd, emb_o)
    allc = np.concatenate([scos, cos], 1)
    alls = np.concatenate([ss, cs], 1)
    ulp = np.abs(allc) * 2.0 ** -8 + 1e-30
    for i in range(4):
        if np.all(np.abs(alls[i]) > ulp[i]) and np.all(np.abs(alls[i] - 0.01) > ulp[i]):
            assert int(has_o[i]) == flags[i], (i, alls[i])


def test_check_reports_missing_weights(cuda):
    from emu_b200 import _lib
    from emu_b200.safety import SafetyChecker
    sd = S.random_state_dict(TINY, seed=1)
    sd.pop("concept_embeds")
    sd.pop(S.TOWER + "encoder.layers.1.self_attn.k_proj.bias")
    ck = _checker(TINY, sd)
    with pytest.raises(_lib.EmuError, match="concept_embeds"):
        ck.check_device(torch.zeros(1, 224, 224, 3, dtype=torch.uint8, device=cuda))
    ck.load_tensor("concept_embeds", torch.randn(17, 64))
    with pytest.raises(_lib.EmuError, match="layer 1 is missing self_attn.k_proj.bias"):
        ck.check_device(torch.zeros(1, 224, 224, 3, dtype=torch.uint8, device=cuda))
    with pytest.raises(_lib.EmuError, match="shape mismatch"):
        ck.load_tensor("concept_embeds", torch.randn(16, 64))
    assert isinstance(SafetyChecker(), SafetyChecker)


# ---- the pipelines: the decode is replaced by a fixed image, everything after it is the product path ----
def _fake_decode(engine, images01):
    engine.vae_decode = lambda z: images01[: z.shape[0]].clone()


def _emu2_pipeline(cuda, checker, images01):
    from emu_b200 import _lib
    from emu_b200.emu2.diffusion import EmuVisualGeneration
    g = EmuVisualGeneration.__new__(EmuVisualGeneration)
    g.engine = _lib.Engine(_lib.EmuConfig())
    g.safety_checker, g._warned_unfiltered, g.device_ = checker, False, cuda
    g.vae_scaling, g.vae_config = 0.13025, None
    if checker is not None and hasattr(checker, "bind"):
        checker.bind(g.engine)
    g._prepare_and_encode_inputs = lambda inputs, do_cfg: torch.zeros(2 if do_cfg else 1, 4, 8, device=cuda)
    g.denoise = lambda pe, B, *a, **k: torch.zeros(B, 4, 4, 4, device=cuda)
    _fake_decode(g.engine, images01)
    return g


def test_emu2_pipeline_with_builtin_checker(cuda):
    from emu_b200.safety import SafetyChecker
    sd, imgs = _fire_setup(cuda)
    images01 = torch.from_numpy(imgs).float().div(255).to(cuda)
    ck = SafetyChecker()
    ck.scfg = _scfg(TINY)
    g = _emu2_pipeline(cuda, ck, images01)
    g.load_state_dict({"safety_checker." + k: v for k, v in sd.items()})   # routed into the engine
    outs = g.forward_batch([["a"], ["b"], ["c"], ["d"]])
    assert [o.nsfw_content_detected for o in outs] == [True, True, False, False]
    assert not np.asarray(outs[0].image).any() and not np.asarray(outs[1].image).any()
    plain = _emu2_pipeline(cuda, None, images01)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = plain.forward_batch([["a"], ["b"], ["c"], ["d"]])
    assert all(r.nsfw_content_detected is None for r in ref)
    for i in (2, 3):
        assert np.array_equal(np.asarray(outs[i].image), np.asarray(ref[i].image))
    one = g.forward(["a"])                                  # forward: image 0 of the batch, which fires
    assert one.nsfw_content_detected is True and not np.asarray(one.image).any()
    _fake_decode(g.engine, images01[2:])
    one = g.forward(["c"])
    assert one.nsfw_content_detected is False and np.array_equal(np.asarray(one.image), np.asarray(ref[2].image))


def test_emu1_pipeline_with_builtin_checker(cuda):
    from emu_b200 import _lib
    from emu_b200.emu1.pipeline import EmuGenerationPipeline
    sd, imgs = _fire_setup(cuda)
    images01 = torch.from_numpy(imgs).float().div(255).to(cuda)
    for idx, want in ((1, True), (3, False)):
        ck = _checker(TINY, {})
        p = EmuGenerationPipeline.__new__(EmuGenerationPipeline)
        p.engine = _lib.Engine(_lib.EmuConfig())
        p.safety_checker, p._warned_unfiltered, p.device_ = ck, False, cuda
        p.vae_scaling, p.vae_config = 0.18215, None
        ck.bind(p.engine)
        p.load_state_dict({"safety_checker." + k: v for k, v in sd.items()})
        p._prepare_and_encode_inputs = lambda *a, **k: torch.zeros(2, 4, 8, device=cuda)
        p.denoise = lambda pe, B, *a, **k: torch.zeros(B, 4, 4, 4, device=cuda)
        _fake_decode(p.engine, images01[idx:idx + 1])
        img, flag = p.forward(["x"])
        assert flag is want
        assert np.array_equal(np.asarray(img), np.zeros_like(imgs[idx]) if want else imgs[idx])
