"""Drop-in for the reference's ``emu.diffusion.EmuVisualGeneration`` (Emu2/emu/diffusion.py:31-383).

Same public surface — ``from_pretrained`` / ``from_config`` / ``forward(inputs, height, width,
num_inference_steps, guidance_scale, crop_info, original_size)`` returning an
``EmuVisualGenerationPipelineOutput(image, nsfw_content_detected)`` — with the arithmetic on the H100 engine:
prompt encoding through ``EmuModel.generate_image`` / ``encode_image``, the denoise loop as one CUDA-graphed
``emu_denoise_step`` per iteration (cat + scale_model_input + UNet + CFG + Euler fused), VAE decode on device.

Safety stage.  The reference runs diffusers' ``StableDiffusionSafetyChecker`` on the decoded image and blanks flagged ones
(Emu2/emu/diffusion.py:154-166, 236-249).  That CLIP classifier is third-party and not part of this engine, so it is NOT
silently dropped: pass ``safety_checker=callable(images_uint8 [B,H,W,3] numpy) -> (images, [bool])`` to keep the stage
(e.g. the diffusers module wrapped by the caller), or construct with the default ``safety_checker=None`` and get a
``UserWarning`` the first time an image is returned unfiltered (``nsfw_content_detected`` is then None, which is what the
reference reports for a pipeline built without a checker).  ``requires_safety_checker=True`` makes a missing hook an error.
"""
import json
import os
import os.path as osp
import warnings
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import torch
from PIL import Image

from .. import _lib
from .conf import CLIPVisionCfg, TextDecoderCfg
from .constants import DEFAULT_IMG_PLACEHOLDER, EVA_IMAGE_SIZE, OPENAI_DATASET_MEAN, OPENAI_DATASET_STD
from .emu import EmuModel
from .scheduler import EulerDiscreteScheduler


@dataclass
class EmuVisualGenerationPipelineOutput:
    image: Image.Image
    nsfw_content_detected: Optional[bool]


def image_transform(img: Image.Image, size=EVA_IMAGE_SIZE, mean=OPENAI_DATASET_MEAN, std=OPENAI_DATASET_STD):
    """TF.Resize((size,size), BICUBIC) -> ToTensor -> Normalize  (Emu2/emu/diffusion.py:59-63)."""
    img = img.convert("RGB").resize((size, size), resample=Image.BICUBIC)
    x = torch.from_numpy(np.asarray(img, dtype=np.uint8).copy()).permute(2, 0, 1).float().div(255.0)
    return (x - torch.tensor(mean)[:, None, None]) / torch.tensor(std)[:, None, None]


def image_transform_cuda(img: Image.Image, size=EVA_IMAGE_SIZE, mean=OPENAI_DATASET_MEAN, std=OPENAI_DATASET_STD,
                         dtype=torch.float32, device="cuda"):
    """Same transform on the GPU (emu_preprocess_image: Pillow-exact fixed-point bicubic + ToTensor + Normalize): only
    the raw uint8 pixels cross PCIe; the result is bit-identical to image_transform()."""
    raw = torch.from_numpy(np.asarray(img.convert("RGB"), dtype=np.uint8).copy())
    return _lib.op_preprocess_image(raw.to(device, non_blocking=True), size, size, mean, std, dtype=dtype)


def unet_config_from_json(cfg: dict) -> "_lib.EmuUNetConfig":
    u = _lib.EmuUNetConfig()
    u.in_channels, u.out_channels = cfg["in_channels"], cfg["out_channels"]
    boc = cfg["block_out_channels"]
    u.n_blocks = len(boc)
    tl = cfg.get("transformer_layers_per_block", 1)
    if isinstance(tl, int):
        tl = [tl] * len(boc)
    for i, c in enumerate(boc):
        u.block_out_channels[i] = c
        u.transformer_layers[i] = tl[i] if "CrossAttn" in cfg["down_block_types"][i] else 0
    u.layers_per_block = cfg["layers_per_block"]
    # the mid block (UNetMidBlock2DCrossAttn) takes transformer_layers_per_block[-1] whatever the last down block is
    u.mid_transformer_layers = tl[-1] if cfg.get("mid_block_type", "UNetMidBlock2DCrossAttn") == "UNetMidBlock2DCrossAttn" else 0
    ahd = cfg.get("num_attention_heads") or cfg["attention_head_dim"]
    # diffusers UNet2DConditionModel reads `attention_head_dim` as the NUMBER OF HEADS per level (a long-standing naming quirk):
    # SDXL [5, 10, 20] -> width 64 everywhere; SD-1.5 8 -> widths 40 / 80 / 160 / 160 (the Emu1 visual decoder)
    heads = list(ahd) if isinstance(ahd, (list, tuple)) else [ahd] * len(boc)
    has_attn = [u.transformer_layers[i] > 0 for i in range(len(boc))]
    has_attn[-1] = has_attn[-1] or u.mid_transformer_layers > 0
    widths = {c // h for c, h, t in zip(boc, heads, has_attn) if t}
    if len(widths) == 1:
        u.head_dim, u.num_heads = widths.pop(), 0
    elif len(set(heads)) == 1:
        u.head_dim, u.num_heads = 0, heads[0]
    else:
        raise NotImplementedError("attention heads %r over channels %r" % (heads, boc))
    u.cross_attention_dim = cfg["cross_attention_dim"]
    u.use_linear_projection = 1 if cfg.get("use_linear_projection") else 0
    u.addition_time_embed_dim = cfg.get("addition_time_embed_dim") or 0
    u.projection_class_embeddings_input_dim = cfg.get("projection_class_embeddings_input_dim") or 0
    u.norm_groups, u.norm_eps = cfg["norm_num_groups"], cfg["norm_eps"]
    # use_linear_projection=False (SD-1.5): proj_in / proj_out are 1x1 convolutions — on NHWC tokens that is the same
    # Linear, and the engine accepts their [C, C, 1, 1] weights as they are
    return u


def vae_config_from_json(cfg: dict) -> "_lib.EmuVAEConfig":
    v = _lib.EmuVAEConfig()
    v.latent_channels, v.out_channels = cfg["latent_channels"], cfg["out_channels"]
    v.n_blocks = len(cfg["block_out_channels"])
    for i, c in enumerate(cfg["block_out_channels"]):
        v.block_out_channels[i] = c
    v.layers_per_block, v.norm_groups = cfg["layers_per_block"], cfg["norm_num_groups"]
    return v


class EmuVisualGeneration:
    def __init__(self, multimodal_encoder: EmuModel, scheduler: EulerDiscreteScheduler, unet_config: dict,
                 vae_config: Optional[dict] = None, eva_size=EVA_IMAGE_SIZE, eva_mean=OPENAI_DATASET_MEAN,
                 eva_std=OPENAI_DATASET_STD, safety_checker=None, requires_safety_checker: bool = False, **kwargs):
        if requires_safety_checker and safety_checker is None:
            raise ValueError("requires_safety_checker=True but no safety_checker callable was given (the reference's "
                             "StableDiffusionSafetyChecker is third-party and not bundled with this engine)")
        self.safety_checker = safety_checker
        self._warned_unfiltered = False
        self.multimodal_encoder = multimodal_encoder
        self.engine = multimodal_encoder.engine
        self.scheduler = scheduler
        self.unet_config, self.vae_config = unet_config, vae_config
        self.engine.unet_configure(unet_config_from_json(unet_config))
        if vae_config is not None:
            self.engine.vae_configure(vae_config_from_json(vae_config))
            self.vae_scale_factor = 2 ** (len(vae_config["block_out_channels"]) - 1)
            self.vae_scaling = vae_config.get("scaling_factor", 0.13025)
        else:
            self.vae_scale_factor, self.vae_scaling = 8, 0.13025
        self.eva_size, self.eva_mean, self.eva_std = eva_size, eva_mean, eva_std
        self.negative_prompt = {}
        self.device_ = multimodal_encoder.device_

    def transform(self, img, device=None):
        if device is not None and torch.device(device).type == "cuda":
            return image_transform_cuda(img, self.eva_size, self.eva_mean, self.eva_std, device=device)
        return image_transform(img, self.eva_size, self.eva_mean, self.eva_std)

    def eval(self):
        return self

    def load_state_dict(self, sd, strict=True):
        """Keys as saved by the reference pipeline: multimodal_encoder.*, unet.*, vae.* (safety_checker.* ignored)."""
        for k, v in sd.items():
            if k.startswith("safety_checker."):
                self._note_checker_weights()
                continue
            if k.endswith("rotary_emb.inv_freq"):
                continue
            if k.startswith("vae.") and (self.vae_config is None or ".encoder." in k or k.startswith("vae.quant_conv")):
                continue  # only the decoder half is on the generate path
            self.engine.load_tensor(k, v)
        return self

    def _note_checker_weights(self):
        if self.safety_checker is None and not self._warned_unfiltered:
            warnings.warn("the checkpoint carries safety_checker.* weights but this pipeline was built without a "
                          "safety_checker hook: images are returned UNFILTERED (pass safety_checker=... to keep the "
                          "reference's post-filter, Emu2/emu/diffusion.py:236-249)", UserWarning, stacklevel=3)
            self._warned_unfiltered = True

    def run_safety_checker(self, images_u8: np.ndarray):
        """Emu2/emu/diffusion.py:236-249: returns (images, has_nsfw list) through the hook, or (images, None) without one."""
        if self.safety_checker is None:
            if not self._warned_unfiltered:
                warnings.warn("EmuVisualGeneration was built without a safety_checker: the image is returned unfiltered "
                              "and nsfw_content_detected is None", UserWarning, stacklevel=3)
                self._warned_unfiltered = True
            return images_u8, None
        images_u8, flags = self.safety_checker(images_u8)
        return images_u8, [bool(f) for f in flags]

    # ---- Emu2/emu/diffusion.py:77-166 ----
    @torch.no_grad()
    def forward(self, inputs, height: int = 1024, width: int = 1024, num_inference_steps: int = 50,
                guidance_scale: float = 3., crop_info: List[int] = [0, 0], original_size: List[int] = [1024, 1024],
                generator: Optional[torch.Generator] = None, latents: Optional[torch.Tensor] = None,
                output_type: str = "pil"):
        if not isinstance(inputs, list):
            inputs = [inputs]
        dev = self.device_
        do_cfg = guidance_scale > 1.0
        prompt_embeds = self._prepare_and_encode_inputs(inputs, do_cfg).to(torch.bfloat16).contiguous()
        batch_size = prompt_embeds.shape[0] // 2 if do_cfg else prompt_embeds.shape[0]
        latents = self.denoise(prompt_embeds, batch_size, height, width, num_inference_steps, guidance_scale, crop_info,
                               original_size, generator=generator, latents=latents)
        if output_type == "latent":
            return latents
        u8 = self.decode_latents_uint8(latents)
        u8, flags = self.run_safety_checker(u8)
        return EmuVisualGenerationPipelineOutput(image=Image.fromarray(u8[0]),
                                                 nsfw_content_detected=None if flags is None else flags[0])

    __call__ = forward

    @torch.no_grad()
    def forward_batch(self, batch_inputs, height: int = 1024, width: int = 1024, num_inference_steps: int = 50,
                      guidance_scale: float = 3., crop_info: List[int] = [0, 0], original_size: List[int] = [1024, 1024],
                      generator: Optional[torch.Generator] = None):
        """`forward` for several independent requests with the same sampler settings through ONE denoising loop (the serving
        shell's batch; BASELINE configs[4] is this with 32 prompts): every request is encoded as in `forward`, the conditional
        rows are stacked in front of the unconditional ones ([cond_1..cond_n; uncond_1..uncond_n], the layout `denoise` and
        emu_denoise_step take), one latent per request.  Returns one EmuVisualGenerationPipelineOutput per request."""
        assert isinstance(batch_inputs, list) and batch_inputs, "batch_inputs must be a non-empty list of `inputs` lists"
        do_cfg = guidance_scale > 1.0
        cond, uncond = [], []
        for inputs in batch_inputs:
            e = self._prepare_and_encode_inputs(inputs if isinstance(inputs, list) else [inputs], do_cfg)
            cond.append(e[:1])
            if do_cfg:
                uncond.append(e[1:2])
        prompt_embeds = torch.cat(cond + uncond, dim=0).to(torch.bfloat16).contiguous()
        latents = self.denoise(prompt_embeds, len(batch_inputs), height, width, num_inference_steps, guidance_scale,
                               crop_info, original_size, generator=generator)
        u8 = self.decode_latents_uint8(latents)
        u8, flags = self.run_safety_checker(u8)
        return [EmuVisualGenerationPipelineOutput(image=Image.fromarray(u8[i]),
                                                  nsfw_content_detected=None if flags is None else flags[i])
                for i in range(len(batch_inputs))]

    @torch.no_grad()
    def denoise(self, prompt_embeds, batch_size, height=1024, width=1024, num_inference_steps=50, guidance_scale=3.,
                crop_info=(0, 0), original_size=(1024, 1024), generator=None, latents=None):
        """Steps 2-4 of the reference forward (time ids, pooled text embedding, timesteps, latents, denoise loop)."""
        dev = self.device_
        do_cfg = guidance_scale > 1.0
        B2 = prompt_embeds.shape[0]
        time_ids = torch.tensor(list(original_size) + list(crop_info) + [height, width], dtype=torch.int32, device=dev)
        time_ids = time_ids[None].expand(B2, -1).contiguous()
        text_embeds = prompt_embeds.float().mean(dim=1).to(torch.bfloat16).contiguous()  # diffusion.py:113
        self.scheduler.set_timesteps(num_inference_steps)
        ts, sig = self.scheduler.timesteps, self.scheduler.sigmas
        h, w = height // self.vae_scale_factor, width // self.vae_scale_factor
        if latents is None:
            latents = torch.randn((batch_size, self.unet_config["in_channels"], h, w), generator=generator,
                                  device=dev if generator is None or generator.device.type == "cuda" else "cpu",
                                  dtype=torch.float32).to(dev)
        latents = (latents.to(torch.bfloat16).float() * self.scheduler.init_noise_sigma).contiguous()
        for i in range(num_inference_steps):
            self.engine.denoise_step(latents, float(sig[i]), float(sig[i + 1]), float(ts[i]), guidance_scale,
                                     prompt_embeds, text_embeds, time_ids)
        return latents

    # ---- boundary: Emu2/emu/diffusion.py:168-212 (same inputs, same two modes, same cache keys) ----
    def _split_prompt(self, inputs, placeholder):
        """interleaved [str | PIL.Image] -> (text with one placeholder per picture, stacked pictures or None, saw any text)"""
        pieces, pictures, saw_text = [], [], False
        for item in inputs:
            if isinstance(item, str):
                pieces.append(item)
                saw_text = True
            else:
                pieces.append(placeholder)
                pictures.append(self.transform(item, self.device_))
        stacked = torch.stack(pictures).to(self.device_, torch.bfloat16) if pictures else None
        return "".join(pieces), stacked, saw_text

    def _unconditional(self, key, make):
        """The classifier-free-guidance branch does not depend on the request: made once per mode, kept in
        `negative_prompt` under the reference's keys ("[NULL_IMAGE]" for autoencoding, "" for generation)."""
        if key not in self.negative_prompt:
            self.negative_prompt[key] = make()
        return self.negative_prompt[key]

    @torch.no_grad()
    def _prepare_and_encode_inputs(self, inputs, do_classifier_free_guidance=False,
                                   placeholder: str = DEFAULT_IMG_PLACEHOLDER):
        text, pictures, saw_text = self._split_prompt(inputs, placeholder)
        enc = self.multimodal_encoder
        if pictures is not None and not saw_text:
            # autoencoding mode (pictures only): the condition is the encoder's own image embedding
            key, cond = "[NULL_IMAGE]", enc.encode_image(image=pictures)
            make_uncond = lambda: enc.encode_image(image=torch.zeros_like(pictures))
        else:
            # generation mode: the decoder regresses the visual embeddings from the interleaved prompt
            key, cond = "", enc.generate_image(text=[text], image=pictures)
            make_uncond = lambda: enc.generate_image(text=[""])
        if not do_classifier_free_guidance:
            return cond
        return torch.cat([cond, self._unconditional(key, make_uncond)], dim=0)

    # ---- Emu2/emu/diffusion.py:214-234 ----
    def decode_latents(self, latents: torch.Tensor) -> np.ndarray:
        z = (latents.float() / self.vae_scaling).to(torch.bfloat16).contiguous()
        img = self.engine.vae_decode(z)  # [B, H, W, 3] fp32 in [0, 1]
        return img.cpu().numpy()

    def decode_latents_uint8(self, latents: torch.Tensor) -> np.ndarray:
        """decode_latents + numpy_to_pil's uint8 conversion on the device (emu_image_to_uint8): a quarter of the
        device->host bytes, bit-identical pixels.  [B, H, W, 3] uint8."""
        z = (latents.float() / self.vae_scaling).to(torch.bfloat16).contiguous()
        return _lib.op_image_to_uint8(self.engine.vae_decode(z)).cpu().numpy()

    def decode_latents_pil(self, latents: torch.Tensor):
        return [Image.fromarray(im) for im in self.decode_latents_uint8(latents)]

    def numpy_to_pil(self, images: np.ndarray):
        if images.ndim == 3:
            images = images[None, ...]
        images = (images * 255).round().astype("uint8")
        return [Image.fromarray(im) for im in images]

    # ---- Emu2/emu/diffusion.py:251-318 ----
    @classmethod
    def from_config(cls, path: Optional[str] = None, llama_config_path: Optional[str] = None, tokenizer=None,
                    safety_checker=None, requires_safety_checker: bool = False, **kwargs):
        """`path` (the reference's argument name, Emu2/emu/diffusion.py:270-273): a diffusers-style directory (unet/, vae/,
        scheduler/); None = the published Emu2-Gen configuration, which is what the reference's default (its own
        conf/diffusion_config) holds.  Sub-directory overrides as in the reference: unet= / vae= / scheduler= keyword paths."""
        from .conf import load_diffusion_config
        path = kwargs.pop("config_path", path)
        unet_cfg, vae_cfg, sched_cfg = load_diffusion_config(path)
        for part, rel in (("unet", "config.json"), ("vae", "config.json"), ("scheduler", "scheduler_config.json")):
            d = kwargs.pop(part, None)                       # reference: kwargs.pop("unet", None) etc., diffusion.py:275-279
            if d is not None:
                cfg = json.load(open(osp.join(d, rel)))
                if part == "unet":
                    unet_cfg = cfg
                elif part == "vae":
                    vae_cfg = cfg
                else:
                    sched_cfg = cfg
        kwargs.pop("feature_extractor", None)                # CLIP pre-processing of the third-party safety checker: see the hook
        if isinstance(safety_checker, str):                  # the reference passes a config DIRECTORY here; the hook is a callable
            safety_checker = None
        sched = EulerDiscreteScheduler(**{k: v for k, v in sched_cfg.items() if not k.startswith("_")})
        tcfg = TextDecoderCfg(llama_config_path=llama_config_path) if llama_config_path else TextDecoderCfg()
        enc = EmuModel(CLIPVisionCfg(), tcfg, tokenizer=tokenizer, **kwargs)
        return cls(multimodal_encoder=enc, scheduler=sched, unet_config=unet_cfg, vae_config=vae_cfg,
                   safety_checker=safety_checker, requires_safety_checker=requires_safety_checker)

    @classmethod
    def from_pretrained(cls, model_path: str, config_path: Optional[str] = None, dtype=torch.bfloat16,
                        use_safetensors: bool = True, **kwargs):
        # the reference takes the WEIGHTS FILE here and reads the configuration from its package (diffusion.py:251-267); a
        # directory that carries its own unet/ vae/ scheduler/ configs next to the weights is accepted as well
        if config_path is None and osp.isdir(model_path) and osp.exists(osp.join(model_path, "unet", "config.json")):
            config_path = model_path
        ins = cls.from_config(config_path, **kwargs)
        from .. import checkpoint

        def keep(k):  # same filter as load_state_dict: no safety checker, only the decoder half of the VAE
            if k.startswith("safety_checker."):
                ins._note_checker_weights()
                return None
            if k.startswith("vae.") and (ins.vae_config is None or ".encoder." in k or k.startswith("vae.quant_conv")):
                return None
            return k
        f = osp.join(model_path, "model.safetensors" if use_safetensors else "pytorch_model.bin")
        checkpoint.load_into(ins.engine, f if osp.exists(f) else model_path, rename=keep)
        return ins

    def device(self, module=None):
        return self.device_

    def dtype(self, module=None):
        return torch.bfloat16

    def multito(self, device_list):
        """The reference places layers on several GPUs of ONE process (Emu2/emu/mixin.py); this engine is one
        process per GPU with tensor parallelism instead — see bench.py / INTEGRATION.md."""
        return self

    multicuda = multito
