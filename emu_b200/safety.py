"""The pipelines' NSFW safety checker on the engine.

Drop-in for what the reference builds from ``safety_checker/`` and ``feature_extractor/`` and runs on every generated image
(Emu2/emu/diffusion.py:154-166, 236-249, 294-313; Emu1/models/pipeline.py:47-52, 132-141, 203-215): transformers'
CLIPImageProcessor + diffusers' StableDiffusionSafetyChecker (CLIP ViT-L/14 vision tower, visual_projection, cosine scores
against 3 special-care and 17 concept embeddings).  Here all of it runs on the device (emu_safety_check): flagged images are
blacked out in place and the flags stay on the GPU until the caller reads them.

    checker = SafetyChecker.from_pretrained("<Emu1 checkpoint>/safety_checker")     # config.json + weights
    checker = SafetyChecker()                   # published configuration; weights come with the Emu2-Gen checkpoint
    pipe = EmuVisualGeneration.from_pretrained(path, safety_checker=checker)

A pipeline given a SafetyChecker binds it to its own engine and routes the checkpoint's ``safety_checker.*`` weights into it.
Used on its own, the checker creates a small engine of its own at first use.  ``checker(images_uint8_numpy)`` keeps the
pipelines' hook contract: ``-> (images, [bool])``.
"""
import json
import os.path as osp
from typing import Optional

import numpy as np
import torch

from . import _lib, checkpoint
from .emu2.conf import EMU2_GEN_FEATURE_EXTRACTOR, EMU2_GEN_SAFETY_CHECKER

PREFIX = "safety_checker."


def _read_json(path_or_dict, name, default):
    if path_or_dict is None:
        return dict(default)
    if isinstance(path_or_dict, dict):
        return dict(path_or_dict)
    p = osp.join(path_or_dict, name) if osp.isdir(path_or_dict) else path_or_dict
    with open(p) as f:
        return json.load(f)


def safety_config(checker_cfg: dict, fe_cfg: dict, n_special: int = 3, n_concepts: int = 17) -> "_lib.EmuSafetyConfig":
    """safety_checker/config.json + feature_extractor/preprocessor_config.json -> EmuSafetyConfig"""
    v = checker_cfg.get("vision_config", checker_cfg)
    act = v.get("hidden_act", "quick_gelu")
    if act != "quick_gelu":
        raise NotImplementedError("safety checker tower activation %r (the engine runs quick_gelu)" % act)
    for flag in ("do_resize", "do_center_crop", "do_rescale", "do_normalize"):
        if not fe_cfg.get(flag, True):
            raise NotImplementedError("feature extractor with %s=False" % flag)
    if fe_cfg.get("resample", 3) != 3 or abs(fe_cfg.get("rescale_factor", 1 / 255) - 1 / 255) > 1e-12:
        raise NotImplementedError("feature extractor: only bicubic resampling and 1/255 rescaling are implemented")
    size, crop = fe_cfg.get("size", {"shortest_edge": 224}), fe_cfg.get("crop_size", {"height": 224, "width": 224})
    size = size["shortest_edge"] if isinstance(size, dict) else int(size)
    if isinstance(crop, dict):
        if crop["height"] != crop["width"]:
            raise NotImplementedError("non-square crop %r" % crop)
        crop = crop["height"]
    c = _lib.EmuSafetyConfig()
    c.image_size, c.patch_size = v.get("image_size", 224), v.get("patch_size", 32)
    c.width, c.layers = v["hidden_size"], v["num_hidden_layers"]
    c.heads, c.mlp = v["num_attention_heads"], v["intermediate_size"]
    c.proj_dim = checker_cfg.get("projection_dim", 768)
    c.n_special, c.n_concepts = n_special, n_concepts
    c.ln_eps = v.get("layer_norm_eps", 1e-5)
    c.resize_shortest_edge, c.crop_size = int(size), int(crop)
    for i in range(3):
        c.image_mean[i] = fe_cfg.get("image_mean", EMU2_GEN_FEATURE_EXTRACTOR["image_mean"])[i]
        c.image_std[i] = fe_cfg.get("image_std", EMU2_GEN_FEATURE_EXTRACTOR["image_std"])[i]
    return c


class SafetyChecker:
    """The built-in checker.  `config`: a safety_checker/ directory, its config.json, or a dict in that format (None = the
    published Emu2-Gen values); `feature_extractor`: a feature_extractor/ directory, its preprocessor_config.json or a dict
    (None = published values)."""

    def __init__(self, config=None, feature_extractor=None, engine: Optional["_lib.Engine"] = None, n_special: int = 3,
                 n_concepts: int = 17):
        self.config = _read_json(config, "config.json", EMU2_GEN_SAFETY_CHECKER)
        self.feature_extractor = _read_json(feature_extractor, "preprocessor_config.json", EMU2_GEN_FEATURE_EXTRACTOR)
        self.scfg = safety_config(self.config, self.feature_extractor, n_special, n_concepts)
        self.engine = None
        self._weights_path = None   # from_pretrained: streamed into the engine when it is bound
        self._pending = {}          # tensors handed over before an engine was bound
        if engine is not None:
            self.bind(engine)

    @classmethod
    def from_pretrained(cls, path: str, feature_extractor=None, engine=None, **kw):
        """A diffusers-format safety_checker/ directory (config.json + weights, keys without the pipeline prefix), as Emu1
        ships it.  The feature extractor defaults to the sibling feature_extractor/ directory when there is one."""
        if feature_extractor is None:
            sib = osp.join(osp.dirname(osp.normpath(path)), "feature_extractor")
            feature_extractor = sib if osp.exists(osp.join(sib, "preprocessor_config.json")) else None
        ins = cls(path, feature_extractor, **kw)
        ins._weights_path = path
        if engine is not None:
            ins.bind(engine)
        return ins

    # ---- engine ----
    def bind(self, engine: "_lib.Engine"):
        """Configure the checker on `engine` (a pipeline's engine) and load whatever weights are waiting."""
        engine.safety_configure(self.scfg)
        self.engine = engine
        if self._weights_path is not None:
            path, self._weights_path = self._weights_path, None
            checkpoint.load_into(engine, path, prefix=PREFIX)
        pending, self._pending = self._pending, {}
        for k, t in pending.items():
            self.load_tensor(k, t)
        return self

    def _ensure_engine(self):
        if self.engine is None:
            self.bind(_lib.Engine(_lib.EmuConfig()))
        return self.engine

    def load_tensor(self, key: str, t: torch.Tensor):
        """one checker weight, with or without the pipeline's `safety_checker.` prefix"""
        if not key.startswith(PREFIX):
            key = PREFIX + key
        if self.engine is None:
            self._pending[key] = t
            return
        self.engine.load_tensor(key, t)

    def load_state_dict(self, sd, strict=True):
        for k, v in sd.items():
            self.load_tensor(k, v)
        return self

    # ---- the check ----
    def check_device(self, images_u8: torch.Tensor, scores: bool = False):
        """images [B, H, W, 3] uint8 CUDA, contiguous; flagged images are zeroed IN PLACE.  -> flags int32 [B] on the device
        (and scores fp32 [B, n_special + n_concepts] with scores=True).  No host synchronisation."""
        return self._ensure_engine().safety_check(images_u8, scores=scores)

    def embed(self, pixel_values: torch.Tensor) -> torch.Tensor:
        """the tower alone: CLIP-normalised pixel_values [B, 3, 224, 224] -> image_embeds [B, 768] bf16"""
        return self._ensure_engine().safety_embed(pixel_values)

    def __call__(self, images_u8: np.ndarray):
        """The pipelines' hook contract: numpy uint8 [B, H, W, 3] -> (images with the flagged ones black, [bool] * B)."""
        dev = torch.from_numpy(np.ascontiguousarray(images_u8)).cuda()
        flags = self.check_device(dev)
        return dev.cpu().numpy(), [bool(f) for f in flags.tolist()]
