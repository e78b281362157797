"""TEST INFRASTRUCTURE — CPU restatement of the pipelines' NSFW safety checker.

Only tests/ may import this module; the product path (emu_b200/csrc/safety.cu, preprocess.cu) never does.

Reference call sites: Emu2/emu/diffusion.py:154-166 and 236-249 (`run_safety_checker`: feature_extractor(numpy_to_pil(image))
-> safety_checker(images=image, clip_input=pixel_values.to(dtype))), Emu2/emu/diffusion.py:294-313 (CLIPImageProcessor from
feature_extractor/, StableDiffusionSafetyChecker(CLIPConfig) from safety_checker/, the whole pipeline cast to bf16), and
Emu1/models/pipeline.py:47-52, 132-141, 203-215 (the same two objects; bf16 through Emu1/image_inference.py:40).

  * preprocess   transformers CLIPImageProcessor with the reference's preprocessor_config.json: resize so the shortest edge
                 is 224 (long edge int(224 * long / short)), PIL bicubic on uint8; centre crop at top = (h' - 224) // 2,
                 left = (w' - 224) // 2; x / 255; (x - mean) / std in fp32.  PINNED: tests/test_safety_cpu.py compares it
                 bit for bit with transformers' CLIPImageProcessorPil.
  * tower        transformers CLIPVisionModel (vision_config of safety_checker/config.json) + visual_projection, in fp32 or
                 with the reference's bf16 rounding points (every module output in bf16; CLIPAttention scales q before the
                 scores, softmax output in bf16).  PINNED on a tiny config against CLIPVisionModel with eager attention.
  * head         diffusers 0.24.0 StableDiffusionSafetyChecker.forward + cosine_distance
                 (pipelines/stable_diffusion/safety_checker.py; diffusers is not installed: UNPINNED restatement).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import preprocess_oracle as PP

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)

# vision_config of the reference's safety_checker/config.json (Emu2/emu/conf/diffusion_config/safety_checker/config.json)
VIT_L14 = dict(image_size=224, patch_size=14, width=1024, layers=24, heads=16, mlp=4096, proj_dim=768, n_special=3,
               n_concepts=17, ln_eps=1e-5)
TOWER = "vision_model.vision_model."


# ---- (1) CLIPImageProcessor ----
def resized_size(h, w, size=224):
    """transformers get_resize_output_image_size(shortest_edge=size, default_to_square=False) -> (h', w')"""
    short, long = (w, h) if w <= h else (h, w)
    new_short, new_long = size, int(size * long / short)
    return (new_long, new_short) if w <= h else (new_short, new_long)


def preprocess(img_u8, size=224, crop=224, mean=CLIP_MEAN, std=CLIP_STD):
    """[H, W, 3] uint8 -> [3, crop, crop] float32"""
    h, w = img_u8.shape[:2]
    rh, rw = resized_size(h, w, size)
    r = PP.resize_bicubic_u8(img_u8, rh, rw)
    top, left = (rh - crop) // 2, (rw - crop) // 2
    return PP.to_tensor_normalize(r[top:top + crop, left:left + crop], mean, std)


# ---- (2) the tower ----
def param_shapes(cfg=VIT_L14):
    """name -> shape of every StableDiffusionSafetyChecker parameter the checker's forward uses (diffusers names)"""
    W, P, G, M = cfg["width"], cfg["patch_size"], cfg["image_size"] // cfg["patch_size"], cfg["mlp"]
    s = {TOWER + "embeddings.class_embedding": (W,), TOWER + "embeddings.patch_embedding.weight": (W, 3, P, P),
         TOWER + "embeddings.position_embedding.weight": (G * G + 1, W),
         TOWER + "pre_layrnorm.weight": (W,), TOWER + "pre_layrnorm.bias": (W,)}
    for l in range(cfg["layers"]):
        p = TOWER + "encoder.layers.%d." % l
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            s[p + "self_attn.%s.weight" % n] = (W, W)
            s[p + "self_attn.%s.bias" % n] = (W,)
        for n in ("layer_norm1", "layer_norm2"):
            s[p + n + ".weight"] = (W,)
            s[p + n + ".bias"] = (W,)
        s[p + "mlp.fc1.weight"], s[p + "mlp.fc1.bias"] = (M, W), (M,)
        s[p + "mlp.fc2.weight"], s[p + "mlp.fc2.bias"] = (W, M), (W,)
    s[TOWER + "post_layernorm.weight"] = s[TOWER + "post_layernorm.bias"] = (W,)
    s["visual_projection.weight"] = (cfg["proj_dim"], W)
    s["concept_embeds"] = (cfg["n_concepts"], cfg["proj_dim"])
    s["special_care_embeds"] = (cfg["n_special"], cfg["proj_dim"])
    s["concept_embeds_weights"] = (cfg["n_concepts"],)
    s["special_care_embeds_weights"] = (cfg["n_special"],)
    return s


def random_state_dict(cfg=VIT_L14, seed=0):
    """seeded weights under the diffusers key names (without the pipeline's `safety_checker.` prefix)"""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in param_shapes(cfg).items():
        if k.endswith(("layer_norm1.weight", "layer_norm2.weight", "layrnorm.weight", "layernorm.weight")):
            t = 1 + 0.1 * torch.randn(shp, generator=g)
        elif k.endswith("_weights"):
            t = 0.05 * torch.rand(shp, generator=g)
        elif k.endswith("embeds"):
            t = torch.randn(shp, generator=g)
        elif len(shp) == 1:
            t = 0.05 * torch.randn(shp, generator=g)
        else:
            t = torch.randn(shp, generator=g) / math.sqrt(int(np.prod(shp[1:])))
        sd[k] = t
    return sd


def tower(sd, pixel_values, cfg=VIT_L14, dtype=torch.float32):
    """pixel_values [B, 3, S, S] -> image_embeds [B, proj]; dtype float32, or bfloat16 for the reference's rounding points"""
    W, P, Hh = cfg["width"], cfg["patch_size"], cfg["heads"]
    D = W // Hh
    w = lambda k: sd[k].to(dtype)
    x = pixel_values.to(dtype)
    B = x.shape[0]
    pe = F.conv2d(x, w(TOWER + "embeddings.patch_embedding.weight"), stride=P).flatten(2).transpose(1, 2)
    cls = w(TOWER + "embeddings.class_embedding").expand(B, 1, -1)
    h = torch.cat([cls, pe], dim=1) + w(TOWER + "embeddings.position_embedding.weight")
    ln = lambda t, n: F.layer_norm(t, (W,), w(n + ".weight"), w(n + ".bias"), cfg["ln_eps"])
    h = ln(h, TOWER + "pre_layrnorm")
    N = h.shape[1]
    for l in range(cfg["layers"]):
        p = TOWER + "encoder.layers.%d." % l
        lin = lambda t, n: F.linear(t, w(p + n + ".weight"), w(p + n + ".bias"))
        r = h
        t = ln(h, p + "layer_norm1")
        q = lin(t, "self_attn.q_proj") * (D ** -0.5)
        k, v = lin(t, "self_attn.k_proj"), lin(t, "self_attn.v_proj")
        sh = lambda z: z.view(B, N, Hh, D).transpose(1, 2)
        a = torch.softmax(sh(q) @ sh(k).transpose(-1, -2), dim=-1)
        o = (a @ sh(v)).transpose(1, 2).reshape(B, N, W)
        h = r + lin(o, "self_attn.out_proj")
        r = h
        f = lin(ln(h, p + "layer_norm2"), "mlp.fc1")
        f = f * torch.sigmoid(1.702 * f)   # quick_gelu
        h = r + lin(f, "mlp.fc2")
    pooled = ln(h[:, 0], TOWER + "post_layernorm")
    return F.linear(pooled, w("visual_projection.weight"))


# ---- (3) the head: diffusers StableDiffusionSafetyChecker.forward ----
def cosine_distance(image_embeds, text_embeds):
    return torch.mm(F.normalize(image_embeds), F.normalize(text_embeds).t())


def head(sd, image_embeds):
    """-> (has_nsfw [B] bool, special_scores [B, S], concept_scores [B, C] (unrounded, float64), special_cos, cos) with the
    embeddings' dtype for the cosine products (bf16 in the pipelines), as diffusers computes them"""
    dt = image_embeds.dtype
    special_cos = cosine_distance(image_embeds, sd["special_care_embeds"].to(dt)).float().numpy()
    cos = cosine_distance(image_embeds, sd["concept_embeds"].to(dt)).float().numpy()
    sw, cw = sd["special_care_embeds_weights"].to(dt), sd["concept_embeds_weights"].to(dt)
    B = image_embeds.shape[0]
    has, ss, cs = [], np.zeros(special_cos.shape), np.zeros(cos.shape)
    for i in range(B):
        adjustment, bad = 0.0, []
        for j in range(special_cos.shape[1]):
            s = special_cos[i][j] - sw[j].item() + adjustment
            ss[i, j] = s
            if round(s, 3) > 0:
                adjustment = 0.01
        for j in range(cos.shape[1]):
            s = cos[i][j] - cw[j].item() + adjustment
            cs[i, j] = s
            if round(s, 3) > 0:
                bad.append(j)
        has.append(len(bad) > 0)
    return has, ss, cs, special_cos, cos


def blackout(images, has_nsfw):
    """flagged images -> zeros (black), the others untouched"""
    out = images.copy()
    for i, f in enumerate(has_nsfw):
        if f:
            out[i] = np.zeros(out[i].shape)
    return out
