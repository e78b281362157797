"""Config dataclasses with the reference's field names and defaults (Emu2/emu/conf/emu_conf.py:7-40)."""
import json
import os.path as osp
from dataclasses import dataclass
from typing import Optional


@dataclass
class CLIPVisionCfg:
    """EVA-CLIP tower hyper-parameters: the reference's field names and defaults (Emu2/emu/conf/emu_conf.py:7-33) so that
    existing call sites and JSON configs keep working.  The engine reads image_size / patch_size / width / layers / head_width
    / mlp_ratio / postnorm / n_query / v_query; the training-only and variant switches are accepted and must keep their
    published values (checked in EmuModel.__init__)."""
    eva_model_name: str = "eva-clip-4b-14-x"
    image_size: int = 448
    patch_size: int = 14
    width: int = 1792
    layers: int = 64
    head_width: int = 112
    mlp_ratio: float = 8.571428571428571   # int(1792 * ratio) = 15360
    qkv_bias: bool = True                   # q / v bias, the k bias is zero
    drop_path_rate: float = 0.
    init_value: Optional[float] = None
    patch_dropout: float = 0.
    rope: bool = False
    global_average_pool: bool = False
    xattn: bool = False
    postnorm: bool = True                   # x + LN(f(x)) blocks, no final norm
    pt_hw_seq_len: int = 16
    intp_freq: bool = False
    naiveswiglu: bool = False
    subln: bool = False
    n_query: int = 64                       # pooled tokens per image
    v_query: int = 64                       # ... per video frame


@dataclass
class TextDecoderCfg:
    # directory holding config.json (+ tokenizer files when a tokenizer is not injected)
    llama_config_path: str = osp.join(osp.dirname(__file__), "llama_config")
    instruct: bool = False


# the published Emu2 decoder (Emu2/emu/conf/llama_config/config.json) — used when no config.json is given
EMU2_LLAMA_33B = dict(hidden_size=6656, num_hidden_layers=60, num_attention_heads=52, intermediate_size=17920,
                      rms_norm_eps=1e-6, max_position_embeddings=2048, vocab_size=32000, rope_theta=10000.0)


def load_llama_config(path_or_dict):
    if isinstance(path_or_dict, dict):
        cfg = dict(path_or_dict)
    else:
        p = path_or_dict
        if osp.isdir(p):
            p = osp.join(p, "config.json")
        cfg = json.load(open(p)) if osp.exists(p) else dict(EMU2_LLAMA_33B)
    cfg.setdefault("rope_theta", 10000.0)
    cfg.setdefault("rms_norm_eps", 1e-6)
    if cfg.get("num_key_value_heads", cfg["num_attention_heads"]) != cfg["num_attention_heads"]:
        raise ValueError("grouped-query attention is not part of the Emu decoder")
    return cfg


# The published Emu2-Gen diffusion configuration (the values of Emu2/emu/conf/diffusion_config/{unet,vae,scheduler}/*.json, the
# directory `EmuVisualGeneration.from_pretrained` / `from_config` default to in the reference, Emu2/emu/diffusion.py:254,272) —
# used when no configuration directory is given, so that `from_pretrained("<...>.safetensors")` works as it does there.
EMU2_GEN_UNET = dict(
    in_channels=4, out_channels=4, sample_size=128, block_out_channels=[320, 640, 1280], layers_per_block=2,
    down_block_types=["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"],
    up_block_types=["CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"], mid_block_type="UNetMidBlock2DCrossAttn",
    transformer_layers_per_block=[1, 2, 10], attention_head_dim=[5, 10, 20], cross_attention_dim=1792,
    use_linear_projection=True, addition_embed_type="text_time", addition_time_embed_dim=256,
    projection_class_embeddings_input_dim=3328, norm_num_groups=32, norm_eps=1e-5, act_fn="silu")
EMU2_GEN_VAE = dict(in_channels=3, out_channels=3, latent_channels=4, block_out_channels=[128, 256, 512, 512],
                    layers_per_block=2, norm_num_groups=32, sample_size=1024, scaling_factor=0.13025, act_fn="silu")
EMU2_GEN_SCHEDULER = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                          prediction_type="epsilon", interpolation_type="linear", timestep_spacing="leading", steps_offset=1,
                          use_karras_sigmas=False)

# The published safety checker (Emu2/emu/conf/diffusion_config/safety_checker/config.json, vision part + projection_dim: a CLIP
# ViT-L/14 tower) and its feature extractor (feature_extractor/preprocessor_config.json): what `SafetyChecker()` uses when no
# configuration directory is given.
EMU2_GEN_SAFETY_CHECKER = dict(
    projection_dim=768,
    vision_config=dict(hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16, patch_size=14,
                       image_size=224, num_channels=3, hidden_act="quick_gelu", layer_norm_eps=1e-5))
EMU2_GEN_FEATURE_EXTRACTOR = dict(
    do_resize=True, size={"shortest_edge": 224}, resample=3, do_center_crop=True, crop_size={"height": 224, "width": 224},
    do_rescale=True, rescale_factor=0.00392156862745098, do_normalize=True, do_convert_rgb=True,
    image_mean=[0.48145466, 0.4578275, 0.40821073], image_std=[0.26862954, 0.26130258, 0.27577711])


def load_diffusion_config(config_path=None):
    """-> (unet, vae, scheduler) config dicts from a diffusers-style directory (`unet/config.json`, `vae/config.json`,
    `scheduler/scheduler_config.json`); a part that is not on disk — or no directory at all — takes the published values"""
    def read(rel, default):
        p = osp.join(config_path, *rel) if config_path else None
        return json.load(open(p)) if p and osp.exists(p) else dict(default)
    return (read(("unet", "config.json"), EMU2_GEN_UNET), read(("vae", "config.json"), EMU2_GEN_VAE),
            read(("scheduler", "scheduler_config.json"), EMU2_GEN_SCHEDULER))
