"""Drop-in for the reference's Emu1 image generation pipeline ``models.pipeline.EmuGenerationPipeline``
(Emu1/models/pipeline.py:20-262).

Same public surface: ``EmuGenerationPipeline.from_pretrained(path, args=...)`` over a checkpoint directory laid out as
``multimodal_encoder/pytorch_model.bin``, ``unet/``, ``vae/``, ``scheduler/`` (``feature_extractor/`` and ``safety_checker/`` feed
the optional post-filter), and ``forward(inputs, height=512, width=512, num_inference_steps=50, guidance_scale=7.5)`` returning
``(PIL.Image, nsfw flag | None)``.  ``inputs`` is the reference's interleaved list of strings and PIL images.

Arithmetic on the H100 engine: prompt -> ``Emu.generate_image`` (EVA-CLIP-g + Causal-Former + LLaMA-13B regression of 32 visual
embeddings, cached form) for [prompt, ""] -> Stable-Diffusion-1.5-topology UNet (1x1-conv projections, 8 heads per level = head
widths 40 / 80 / 160, no added conditioning) under classifier-free guidance with the PNDM / PLMS scheduler, one CUDA-graphed
fused iteration per timestep (emu_denoise_step_multistep) -> VAE decode -> uint8 on the device.

Safety stage: the reference runs diffusers' StableDiffusionSafetyChecker on the decoded image (:142-147, :218-232).
``safety_checker=emu_b200.safety.SafetyChecker.from_pretrained(f"{path}/safety_checker")`` runs it on the engine (bound to this
pipeline's engine, weights from that directory, the check on the device before the copy to the host); any other
``safety_checker=callable(images_uint8) -> (images, [bool])`` is called as a host hook.  Without one the image is returned
unfiltered, the flag is None (what the reference returns when built without a checker) and a UserWarning says so;
``requires_safety_checker=True`` turns a missing checker into an error.
"""
import json
import os.path as osp
import warnings
from typing import List, Optional, Tuple, Union

import numpy as np
import torch
from PIL import Image

from .. import _lib, checkpoint
from ..safety import SafetyChecker
from ..emu2.diffusion import image_transform, image_transform_cuda, unet_config_from_json, vae_config_from_json
from .modeling_emu import Emu
from .scheduler import PNDMScheduler

EVA_MEAN, EVA_STD = (0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)


class EmuGenerationPipeline:
    def __init__(self, multimodal_model=None, feature_extractor=None, safety_checker=None, scheduler=None, unet=None, vae=None,
                 eva_size=224, eva_mean=EVA_MEAN, eva_std=EVA_STD, *, emu_encoder: Optional[Emu] = None,
                 unet_config: Optional[dict] = None, vae_config: Optional[dict] = None,
                 requires_safety_checker: bool = False, **kwargs):
        """Reference-style construction takes PATHS (multimodal_model, scheduler, unet, vae: Emu1/models/pipeline.py:22-52);
        tests and synthetic runs may inject a ready `emu_encoder`, config dicts and a scheduler object instead."""
        hook = safety_checker if callable(safety_checker) else None
        if requires_safety_checker and hook is None:
            raise ValueError("requires_safety_checker=True but no safety_checker callable was given (the reference's "
                             "StableDiffusionSafetyChecker is third-party and not bundled with this engine)")
        self.safety_checker = hook
        self._warned_unfiltered = False
        if isinstance(safety_checker, str) and osp.exists(safety_checker):
            self._note_unfiltered("the checkpoint carries a safety_checker/ directory")
        self.emu_encoder = emu_encoder if emu_encoder is not None else self.prepare_emu("Emu-14B", multimodal_model, **kwargs)
        self.engine = self.emu_encoder.engine
        self.device_ = self.emu_encoder.device_
        if isinstance(self.safety_checker, SafetyChecker):
            self.safety_checker.bind(self.engine)
        if unet_config is None:
            unet_config = json.load(open(osp.join(unet, "config.json")))
        if vae_config is None and vae is not None:
            vae_config = json.load(open(osp.join(vae, "config.json")))
        self.unet_config, self.vae_config = unet_config, vae_config
        self.engine.unet_configure(unet_config_from_json(unet_config))
        if vae_config is not None:
            self.engine.vae_configure(vae_config_from_json(vae_config))
            self.vae_scale_factor = 2 ** (len(vae_config["block_out_channels"]) - 1)
            self.vae_scaling = vae_config.get("scaling_factor", 0.18215)
        else:
            self.vae_scale_factor, self.vae_scaling = 8, 0.18215
        if isinstance(scheduler, PNDMScheduler):
            self.scheduler = scheduler
        elif scheduler is not None and osp.exists(str(scheduler)):
            self.scheduler = PNDMScheduler.from_config(scheduler)
        else:
            self.scheduler = PNDMScheduler()
        if isinstance(unet, str) and osp.isdir(unet):
            checkpoint.load_into(self.engine, unet, prefix="unet.")
        if isinstance(vae, str) and osp.isdir(vae) and vae_config is not None:
            keep = lambda k: None if (".encoder." in k or k.startswith(("encoder.", "quant_conv"))) else k
            checkpoint.load_into(self.engine, vae, prefix="vae.", rename=keep)
        self.eva_size, self.eva_mean, self.eva_std = eva_size, eva_mean, eva_std

    # ---- plumbing the reference gets from nn.Module ----
    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    bfloat16 = cuda = to

    def transform(self, img, device=None):
        if device is not None and torch.device(device).type == "cuda":
            return image_transform_cuda(img, self.eva_size, self.eva_mean, self.eva_std, device=device)
        return image_transform(img, self.eva_size, self.eva_mean, self.eva_std)

    def load_state_dict(self, sd, strict=True):
        """unet.* / vae.* (decoder half) / emu_encoder.* keys in one dict (tests, synthetic weights)."""
        for k, v in sd.items():
            if k.startswith("safety_checker.") and not isinstance(self.safety_checker, SafetyChecker):
                self._note_unfiltered("the state dict carries safety_checker.* weights")
                continue
            if k.startswith("vae.") and (self.vae_config is None or ".encoder." in k or k.startswith("vae.quant_conv")):
                continue
            if k.startswith("emu_encoder."):
                k = k[len("emu_encoder."):]
            if k.endswith("rotary_emb.inv_freq"):
                continue
            self.engine.load_tensor(k, v)
        return self

    def _note_unfiltered(self, why):
        if self.safety_checker is None and not self._warned_unfiltered:
            warnings.warn("%s but this pipeline was built without a safety_checker hook: images are returned UNFILTERED "
                          "(pass safety_checker=callable to keep the reference's post-filter, Emu1/models/pipeline.py:218-232)"
                          % why, UserWarning, stacklevel=3)
            self._warned_unfiltered = True

    # ---- Emu1/models/pipeline.py:65-141 ----
    @torch.no_grad()
    def forward(self, inputs: List[Union[Image.Image, str]], height: int = 512, width: int = 512,
                num_inference_steps: int = 50, guidance_scale: float = 7.5, generator: Optional[torch.Generator] = None,
                latents: Optional[torch.Tensor] = None, output_type: str = "pil") -> Tuple[Image.Image, Optional[bool]]:
        do_cfg = guidance_scale > 1.0
        prompt_embeds = self._prepare_and_encode_inputs(inputs, self.device_, torch.bfloat16, do_cfg)
        latents = self.denoise(prompt_embeds.to(torch.bfloat16).contiguous(), 1, height, width, num_inference_steps,
                               guidance_scale, generator=generator, latents=latents)
        if output_type == "latent":
            return latents
        u8, flags = self.decode_and_check(latents)
        return Image.fromarray(u8[0]), (None if flags is None else flags[0])

    __call__ = forward

    @torch.no_grad()
    def denoise(self, prompt_embeds, batch_size, height=512, width=512, num_inference_steps=50, guidance_scale=7.5,
                generator=None, latents=None):
        """Steps 2-4 of the reference forward: timesteps, latents ~ N(0, 1) (init_noise_sigma = 1), the PLMS loop."""
        dev = self.device_
        self.scheduler.set_timesteps(num_inference_steps)
        h, w = height // self.vae_scale_factor, width // self.vae_scale_factor
        C = self.unet_config["in_channels"]
        if latents is None:
            latents = torch.randn((batch_size, C, h, w), generator=generator,
                                  device=dev if generator is None or generator.device.type == "cuda" else "cpu",
                                  dtype=torch.float32).to(dev)
        # the reference draws the latents in the model dtype (bf16 after pipeline.bfloat16()); the state is kept in fp32 here
        latents = latents.to(torch.bfloat16).float().contiguous()
        state = torch.zeros(4, *latents.shape, dtype=torch.float32, device=dev)
        for i, t in enumerate(self.scheduler.timesteps.tolist()):
            self.engine.denoise_step_multistep(latents, state, self.scheduler.step_coefficients(i), float(t), guidance_scale,
                                               prompt_embeds)
        return latents

    # ---- Emu1/models/pipeline.py:143-178 ----
    @torch.no_grad()
    def _prepare_and_encode_inputs(self, inputs, device="cpu", dtype=torch.float32, do_classifier_free_guidance=False,
                                   placeholder: str = "[<IMG_PLH>]"):
        pieces, images = [], []
        for x in inputs:
            if isinstance(x, str):
                pieces.append(x)
            else:
                pieces.append(placeholder)
                images.append(self.transform(x, self.device_))
        text_prompt = "".join(pieces)
        image_prompt = torch.stack(images).to(self.device_, torch.bfloat16) if images else None
        texts = [text_prompt, ""] if do_classifier_free_guidance else [text_prompt]   # [cond; uncond] in ONE padded batch
        return self.emu_encoder.generate_image(text=texts, image=image_prompt, placeholder=placeholder)

    # ---- Emu1/models/pipeline.py:180-200 ----
    def decode_latents_uint8(self, latents: torch.Tensor) -> np.ndarray:
        z = (latents.float() / self.vae_scaling).to(torch.bfloat16).contiguous()
        return _lib.op_image_to_uint8(self.engine.vae_decode(z)).cpu().numpy()

    def decode_and_check(self, latents: torch.Tensor):
        """decode -> uint8 -> safety stage; a built-in SafetyChecker runs on the device image before the copy to the host"""
        if isinstance(self.safety_checker, SafetyChecker):
            z = (latents.float() / self.vae_scaling).to(torch.bfloat16).contiguous()
            dev = _lib.op_image_to_uint8(self.engine.vae_decode(z))
            flags = self.safety_checker.check_device(dev)
            return dev.cpu().numpy(), [bool(f) for f in flags.tolist()]
        return self.run_safety_checker(self.decode_latents_uint8(latents))

    def decode_latents(self, latents: torch.Tensor) -> np.ndarray:
        z = (latents.float() / self.vae_scaling).to(torch.bfloat16).contiguous()
        return self.engine.vae_decode(z).cpu().numpy()

    def numpy_to_pil(self, images: np.ndarray):
        if images.ndim == 3:
            images = images[None, ...]
        images = (images * 255).round().astype("uint8")
        return [Image.fromarray(im.squeeze(), mode="L") if im.shape[-1] == 1 else Image.fromarray(im) for im in images]

    def run_safety_checker(self, images_u8: np.ndarray):
        if self.safety_checker is None:
            self._note_unfiltered("no safety_checker was given")
            return images_u8, None
        images_u8, flags = self.safety_checker(images_u8)
        return images_u8, [bool(f) for f in flags]

    # ---- Emu1/models/pipeline.py:234-262 ----
    def prepare_emu(self, model_name: str, model_path: str, args=None, **kwargs) -> Emu:
        cfg_path = osp.join("models", model_name + ".json")
        model_cfg = json.load(open(cfg_path)) if osp.exists(cfg_path) else {}
        model = Emu(**model_cfg, args=args, **kwargs)
        if model_path is not None:
            checkpoint.load_into(model.engine, model_path, rename=lambda k: None if k.startswith(
                ("visual.norm.", "visual.fc_norm.", "visual.head.", "visual.rope.")) else k)
        return model

    @classmethod
    def from_pretrained(cls, path: str, **kwargs):
        pick = lambda name, default: kwargs.pop(name, None) or default
        return cls(multimodal_model=pick("multimodal_model", f"{path}/multimodal_encoder/pytorch_model.bin"),
                   feature_extractor=pick("feature_extractor", f"{path}/feature_extractor"),
                   safety_checker=pick("safety_checker", f"{path}/safety_checker"),
                   scheduler=pick("scheduler", f"{path}/scheduler"), unet=pick("unet", f"{path}/unet"),
                   vae=pick("vae", f"{path}/vae"), **kwargs)
