"""TEST INFRASTRUCTURE — CPU oracle for the Emu2-Gen / Emu1 diffusion half of the generate path.

PARITY UNPINNED.  The arithmetic lives in `diffusers==0.24.0` (`Emu2/requirements.txt:13`; Emu1 pins 0.15.1),
which is neither vendored under /root/reference nor installed here (no network), so this file restates the
published diffusers algorithms — `UNet2DConditionModel` (SDXL topology as configured by
`Emu2/emu/conf/diffusion_config/unet/config.json`), `EulerDiscreteScheduler`
(`.../scheduler/scheduler_config.json`) and the `AutoencoderKL` decoder (`.../vae/config.json`) — and is anchored on
the reference's own call sites: `Emu2/emu/diffusion.py:107-149` (conditioning + denoise loop), `:214-219` (VAE).
Cross-checks available without diffusers: parameter count from the reference's JSON config (2.526 B expected,
SURVEY.md §8a row a14) and state-dict key layout (diffusers names).

Functional, state-dict driven, dtype-generic (fp32 = numerical oracle, bf16 = the reference's rounding points).
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this file.
"""
import math

import torch
import torch.nn.functional as F

# ------------------------------------------------------------------------------------------------
# configs (values from the reference's JSON files)
# ------------------------------------------------------------------------------------------------
EMU2_UNET = dict(in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280), layers_per_block=2,
                 transformer_layers_per_block=(0, 2, 10),  # block 0 is DownBlock2D: its "1" is unused
                 attention_head_dim=64, cross_attention_dim=1792, addition_time_embed_dim=256,
                 projection_class_embeddings_input_dim=3328, norm_num_groups=32, norm_eps=1e-5)
# Emu1 visual decoder: Stable-Diffusion-1.5 topology (the reference loads it from <ckpt>/unet/config.json,
# Emu1/models/pipeline.py:37-39): 1x1-conv proj_in / proj_out, 8 heads per level (widths 40 / 80 / 160), no added conditioning,
# cross-attention over the 32 regressed embeddings of width 5120
EMU1_UNET = dict(in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
                 transformer_layers_per_block=(1, 1, 1, 0), num_heads=8, cross_attention_dim=5120, use_linear_projection=False,
                 norm_num_groups=32, norm_eps=1e-5)
EMU1_SCHED = dict(beta_start=0.00085, beta_end=0.012, num_train_timesteps=1000, steps_offset=1)
EMU2_SCHED = dict(beta_start=0.00085, beta_end=0.012, num_train_timesteps=1000, steps_offset=1)
EMU2_VAE = dict(latent_channels=4, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                norm_num_groups=32, scaling_factor=0.13025)


# ------------------------------------------------------------------------------------------------
# building blocks
# ------------------------------------------------------------------------------------------------
def timestep_embedding(t, dim, dtype):
    """diffusers get_timestep_embedding(flip_sin_to_cos=True, downscale_freq_shift=0): [cos | sin]."""
    half = dim // 2
    exponent = -math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half
    emb = t.float()[:, None] * torch.exp(exponent)[None, :]
    return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1).to(dtype)


def linear(sd, p, x):
    w = sd[p + ".weight"]
    if w.dim() == 4:  # a 1x1 convolution applied to channel-last tokens (SD-1.5 proj_in / proj_out)
        w = w.reshape(w.shape[0], w.shape[1])
    return F.linear(x, w, sd.get(p + ".bias"))


def conv(sd, p, x, stride=1, padding=1):
    return F.conv2d(x, sd[p + ".weight"], sd.get(p + ".bias"), stride=stride, padding=padding)


def group_norm(sd, p, x, groups, eps):
    return F.group_norm(x, groups, sd[p + ".weight"], sd[p + ".bias"], eps)


def resnet_block(sd, p, x, emb, groups, eps):
    """ResnetBlock2D (time_embedding_norm="default", output_scale_factor=1)."""
    h = F.silu(group_norm(sd, p + "norm1", x, groups, eps))
    h = conv(sd, p + "conv1", h)
    h = h + linear(sd, p + "time_emb_proj", F.silu(emb))[:, :, None, None]
    h = F.silu(group_norm(sd, p + "norm2", h, groups, eps))
    h = conv(sd, p + "conv2", h)
    if (p + "conv_shortcut.weight") in sd:
        x = conv(sd, p + "conv_shortcut", x, padding=0)
    return x + h


def attention(sd, p, x, ctx, head_dim):
    """diffusers Attention (AttnProcessor): to_q/k/v without bias, to_out.0 with bias, scale = head_dim^-0.5."""
    B, N, C = x.shape
    heads = C // head_dim
    src = x if ctx is None else ctx
    q = F.linear(x, sd[p + "to_q.weight"]).view(B, N, heads, head_dim).transpose(1, 2)
    k = F.linear(src, sd[p + "to_k.weight"]).view(B, src.shape[1], heads, head_dim).transpose(1, 2)
    v = F.linear(src, sd[p + "to_v.weight"]).view(B, src.shape[1], heads, head_dim).transpose(1, 2)
    w = torch.softmax((q @ k.transpose(-1, -2)) * head_dim ** -0.5, dim=-1)
    o = (w @ v).transpose(1, 2).reshape(B, N, C)
    return linear(sd, p + "to_out.0", o)


def transformer_block(sd, p, x, ctx, head_dim):
    """BasicTransformerBlock: LN -> self-attn; LN -> cross-attn; LN -> GEGLU feed-forward (all residual)."""
    C = x.shape[-1]
    ln = lambda n, t: F.layer_norm(t, (C,), sd[p + n + ".weight"], sd[p + n + ".bias"], 1e-5)
    x = x + attention(sd, p + "attn1.", ln("norm1", x), None, head_dim)
    x = x + attention(sd, p + "attn2.", ln("norm2", x), ctx, head_dim)
    h = linear(sd, p + "ff.net.0.proj", ln("norm3", x))
    hidden, gate = h.chunk(2, dim=-1)
    return x + linear(sd, p + "ff.net.2", hidden * F.gelu(gate))


def transformer_2d(sd, p, x, ctx, n_layers, groups, head_dim):
    """Transformer2DModel with use_linear_projection=True (GroupNorm eps 1e-6, Linear proj_in/out)."""
    B, C, H, W = x.shape
    res = x
    h = group_norm(sd, p + "norm", x, groups, 1e-6)
    h = h.permute(0, 2, 3, 1).reshape(B, H * W, C)
    h = linear(sd, p + "proj_in", h)
    for k in range(n_layers):
        h = transformer_block(sd, f"{p}transformer_blocks.{k}.", h, ctx, head_dim)
    h = linear(sd, p + "proj_out", h)
    return h.reshape(B, H, W, C).permute(0, 3, 1, 2) + res


# ------------------------------------------------------------------------------------------------
# UNet2DConditionModel.forward
# ------------------------------------------------------------------------------------------------
def unet_forward(sd, cfg, sample, timestep, ctx, text_embeds=None, time_ids=None, prefix=""):
    """sample [B,4,h,w]; timestep scalar; ctx [B,L,cross_dim]; text_embeds [B,cross_dim]; time_ids [B,6].
    Returns the predicted noise [B,4,h,w].  Call site: Emu2/emu/diffusion.py:136-141."""
    g, eps = cfg["norm_num_groups"], cfg["norm_eps"]
    boc = cfg["block_out_channels"]
    # head width: fixed (SDXL, `attention_head_dim`) or channels / num_heads (SD-1.5: the same head COUNT at every level)
    hd_of = (lambda c: cfg["attention_head_dim"]) if cfg.get("attention_head_dim") else (lambda c: c // cfg["num_heads"])
    tl = cfg["transformer_layers_per_block"]
    lpb = cfg["layers_per_block"]
    nb = len(boc)
    B = sample.shape[0]
    dt = sample.dtype
    P = prefix
    t = torch.as_tensor(timestep, dtype=torch.float32).reshape(-1).expand(B)
    emb = timestep_embedding(t, boc[0], dt)
    emb = linear(sd, P + "time_embedding.linear_2", F.silu(linear(sd, P + "time_embedding.linear_1", emb)))
    if cfg.get("addition_time_embed_dim"):
        te = timestep_embedding(time_ids.flatten(), cfg["addition_time_embed_dim"], dt).reshape(B, -1)
        add = torch.cat([text_embeds.to(dt), te], dim=-1)
        emb = emb + linear(sd, P + "add_embedding.linear_2", F.silu(linear(sd, P + "add_embedding.linear_1", add)))
    h = conv(sd, P + "conv_in", sample)
    skips = [h]
    for i in range(nb):
        for j in range(lpb):
            h = resnet_block(sd, f"{P}down_blocks.{i}.resnets.{j}.", h, emb, g, eps)
            if tl[i] > 0:
                h = transformer_2d(sd, f"{P}down_blocks.{i}.attentions.{j}.", h, ctx, tl[i], g, hd_of(boc[i]))
            skips.append(h)
        if i < nb - 1:
            h = conv(sd, f"{P}down_blocks.{i}.downsamplers.0.conv", h, stride=2, padding=1)
            skips.append(h)
    h = resnet_block(sd, P + "mid_block.resnets.0.", h, emb, g, eps)
    if (P + "mid_block.attentions.0.norm.weight") in sd:
        h = transformer_2d(sd, P + "mid_block.attentions.0.", h, ctx, cfg.get("mid_block_layers", max(tl[-1], 1)), g,
                           hd_of(boc[-1]))
    elif tl[-1] > 0:
        h = transformer_2d(sd, P + "mid_block.attentions.0.", h, ctx, tl[-1], g, hd_of(boc[-1]))
    h = resnet_block(sd, P + "mid_block.resnets.1.", h, emb, g, eps)
    for i in range(nb):
        ri = nb - 1 - i  # reversed block index
        for j in range(lpb + 1):
            h = torch.cat([h, skips.pop()], dim=1)
            h = resnet_block(sd, f"{P}up_blocks.{i}.resnets.{j}.", h, emb, g, eps)
            if tl[ri] > 0:
                h = transformer_2d(sd, f"{P}up_blocks.{i}.attentions.{j}.", h, ctx, tl[ri], g, hd_of(boc[ri]))
        if i < nb - 1:
            h = F.interpolate(h, scale_factor=2.0, mode="nearest")
            h = conv(sd, f"{P}up_blocks.{i}.upsamplers.0.conv", h)
    h = F.silu(group_norm(sd, P + "conv_norm_out", h, g, eps))
    return conv(sd, P + "conv_out", h)


def unet_param_shapes(cfg):
    """Every parameter (diffusers key -> shape) of the UNet described by cfg; used to build random state dicts and
    to cross-check the parameter count against the reference's config (2.526 B for EMU2_UNET)."""
    boc, tl, lpb = cfg["block_out_channels"], cfg["transformer_layers_per_block"], cfg["layers_per_block"]
    cd, nb = cfg["cross_attention_dim"], len(cfg["block_out_channels"])
    temb = boc[0] * 4
    s = {}

    def lin(p, o, i, bias=True):
        s[p + ".weight"] = (o, i)
        if bias:
            s[p + ".bias"] = (o,)

    def cv(p, o, i, k=3):
        s[p + ".weight"] = (o, i, k, k)
        s[p + ".bias"] = (o,)

    def nrm(p, c):
        s[p + ".weight"] = (c,)
        s[p + ".bias"] = (c,)

    def resnet(p, cin, cout):
        nrm(p + "norm1", cin)
        cv(p + "conv1", cout, cin)
        lin(p + "time_emb_proj", cout, temb)
        nrm(p + "norm2", cout)
        cv(p + "conv2", cout, cout)
        if cin != cout:
            cv(p + "conv_shortcut", cout, cin, 1)

    conv_proj = cfg.get("use_linear_projection", True) is False

    def proj(p, c):
        if conv_proj:
            cv(p, c, c, 1)
        else:
            lin(p, c, c)

    def tfm(p, c, n):
        nrm(p + "norm", c)
        proj(p + "proj_in", c)
        for k in range(n):
            q = f"{p}transformer_blocks.{k}."
            for a, kd in (("attn1.", c), ("attn2.", cd)):
                lin(q + a + "to_q", c, c, False)
                lin(q + a + "to_k", c, kd, False)
                lin(q + a + "to_v", c, kd, False)
                lin(q + a + "to_out.0", c, c)
            for n_ in ("norm1", "norm2", "norm3"):
                nrm(q + n_, c)
            lin(q + "ff.net.0.proj", 8 * c, c)
            lin(q + "ff.net.2", c, 4 * c)
        proj(p + "proj_out", c)

    cv("conv_in", boc[0], cfg["in_channels"])
    lin("time_embedding.linear_1", temb, boc[0])
    lin("time_embedding.linear_2", temb, temb)
    if cfg.get("addition_time_embed_dim"):
        lin("add_embedding.linear_1", temb, cfg["projection_class_embeddings_input_dim"])
        lin("add_embedding.linear_2", temb, temb)
    cin = boc[0]
    skip_ch = [boc[0]]
    for i in range(nb):
        for j in range(lpb):
            resnet(f"down_blocks.{i}.resnets.{j}.", cin, boc[i])
            cin = boc[i]
            if tl[i] > 0:
                tfm(f"down_blocks.{i}.attentions.{j}.", cin, tl[i])
            skip_ch.append(cin)
        if i < nb - 1:
            cv(f"down_blocks.{i}.downsamplers.0.conv", cin, cin)
            skip_ch.append(cin)
    resnet("mid_block.resnets.0.", cin, cin)
    mid_layers = cfg.get("mid_block_layers", tl[-1])
    if mid_layers > 0:
        tfm("mid_block.attentions.0.", cin, mid_layers)
    resnet("mid_block.resnets.1.", cin, cin)
    for i in range(nb):
        ri = nb - 1 - i
        for j in range(lpb + 1):
            resnet(f"up_blocks.{i}.resnets.{j}.", cin + skip_ch.pop(), boc[ri])
            cin = boc[ri]
            if tl[ri] > 0:
                tfm(f"up_blocks.{i}.attentions.{j}.", cin, tl[ri])
        if i < nb - 1:
            cv(f"up_blocks.{i}.upsamplers.0.conv", cin, cin)
    nrm("conv_norm_out", boc[0])
    cv("conv_out", cfg["out_channels"], boc[0])
    return s


def random_state_dict(shapes, seed=0, dtype=torch.float32, prefix=""):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in shapes.items():
        if k.endswith(".weight") and len(shp) == 1:
            t = 1 + 0.1 * torch.randn(shp, generator=g)
        elif k.endswith(".bias"):
            t = 0.05 * torch.randn(shp, generator=g)
        else:
            fan_in = 1
            for d in shp[1:]:
                fan_in *= d
            t = torch.randn(shp, generator=g) / math.sqrt(fan_in)
        sd[prefix + k] = t.to(dtype)
    return sd


# ------------------------------------------------------------------------------------------------
# EulerDiscreteScheduler (timestep_spacing="leading", steps_offset=1, epsilon prediction, linear interpolation)
# ------------------------------------------------------------------------------------------------
def euler_tables(num_inference_steps, cfg=EMU2_SCHED):
    n = cfg["num_train_timesteps"]
    betas = torch.linspace(cfg["beta_start"] ** 0.5, cfg["beta_end"] ** 0.5, n, dtype=torch.float32) ** 2
    alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
    sig_all = ((1 - alphas_cumprod) / alphas_cumprod) ** 0.5
    step_ratio = n // num_inference_steps
    timesteps = (torch.arange(0, num_inference_steps) * step_ratio).round().flip(0).float() + cfg["steps_offset"]
    # np.interp(timesteps, arange(n), sigmas): timesteps are integers -> exact table values
    lo = timesteps.floor().long().clamp(max=n - 1)
    hi = (lo + 1).clamp(max=n - 1)
    frac = timesteps - lo.float()
    sigmas = sig_all[lo] * (1 - frac) + sig_all[hi] * frac
    sigmas = torch.cat([sigmas, torch.zeros(1)])
    init_noise_sigma = float((sigmas.max() ** 2 + 1) ** 0.5)  # "leading" spacing
    return timesteps, sigmas, init_noise_sigma


def denoise_loop(unet_fn, latents, ctx, text_embeds, time_ids, num_inference_steps, guidance_scale):
    """EmuVisualGeneration.forward steps 4 (Emu2/emu/diffusion.py:130-149) with CFG; ctx is [cond; uncond].
    `latents` must already be scaled by init_noise_sigma (:127)."""
    timesteps, sigmas, _ = euler_tables(num_inference_steps)
    for i, t in enumerate(timesteps):
        sigma, sigma_next = sigmas[i], sigmas[i + 1]
        x = torch.cat([latents] * 2)
        x = x / ((sigma ** 2 + 1) ** 0.5)                       # scale_model_input
        noise = unet_fn(x.to(latents.dtype), float(t), ctx, text_embeds, time_ids)
        cond, uncond = noise.chunk(2)                           # (cond, uncond) order, :145
        noise = uncond + guidance_scale * (cond - uncond)
        latents = latents + noise * (sigma_next - sigma)        # Euler step, epsilon prediction, s_churn = 0
    return latents


# ------------------------------------------------------------------------------------------------
# PNDMScheduler, skip_prk_steps=True (PLMS) — the scheduler of the Emu1 pipeline (Emu1/models/pipeline.py:43-45, 94-127)
# ------------------------------------------------------------------------------------------------
class PNDMOracle:
    """Literal restatement of diffusers PNDMScheduler.set_timesteps / step_plms / _get_prev_sample (Stable-Diffusion-1.5
    configuration: scaled-linear betas, set_alpha_to_one=False, steps_offset=1, epsilon prediction), list-of-tensors state
    like the original — deliberately NOT in the coefficient form the product uses (emu_b200/emu1/scheduler.py)."""

    def __init__(self, cfg=EMU1_SCHED):
        n = cfg["num_train_timesteps"]
        betas = torch.linspace(cfg["beta_start"] ** 0.5, cfg["beta_end"] ** 0.5, n, dtype=torch.float32) ** 2
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = self.alphas_cumprod[0]
        self.n, self.offset = n, cfg["steps_offset"]

    def set_timesteps(self, steps):
        self.steps = steps
        ratio = self.n // steps
        base = (torch.arange(0, steps) * ratio).round().long() + self.offset
        self.timesteps = torch.cat([base[:-1], base[-2:-1], base[-1:]]).flip(0)
        self.ets, self.counter, self.cur_sample = [], 0, None

    def _get_prev_sample(self, sample, timestep, prev_timestep, model_output):
        a_t = self.alphas_cumprod[timestep]
        a_p = self.alphas_cumprod[prev_timestep] if prev_timestep >= 0 else self.final_alpha_cumprod
        b_t, b_p = 1 - a_t, 1 - a_p
        sample_coeff = (a_p / a_t) ** 0.5
        denom = a_t * b_p ** 0.5 + (a_t * b_t * a_p) ** 0.5
        return sample_coeff * sample - (a_p - a_t) * model_output / denom

    def step(self, model_output, timestep, sample):
        ratio = self.n // self.steps
        prev_timestep = timestep - ratio
        if self.counter != 1:
            self.ets = self.ets[-3:]
            self.ets.append(model_output)
        else:
            prev_timestep = timestep
            timestep = timestep + ratio
        if len(self.ets) == 1 and self.counter == 0:
            self.cur_sample = sample
        elif len(self.ets) == 1 and self.counter == 1:
            model_output = (model_output + self.ets[-1]) / 2
            sample = self.cur_sample
            self.cur_sample = None
        elif len(self.ets) == 2:
            model_output = (3 * self.ets[-1] - self.ets[-2]) / 2
        elif len(self.ets) == 3:
            model_output = (23 * self.ets[-1] - 16 * self.ets[-2] + 5 * self.ets[-3]) / 12
        else:
            model_output = (1 / 24) * (55 * self.ets[-1] - 59 * self.ets[-2] + 37 * self.ets[-3] - 9 * self.ets[-4])
        self.counter += 1
        return self._get_prev_sample(sample, timestep, prev_timestep, model_output)


def pndm_denoise_loop(unet_fn, latents, ctx, num_inference_steps, guidance_scale):
    """EmuGenerationPipeline.forward step 4 (Emu1/models/pipeline.py:108-127); ctx is [cond; uncond], latents ~ N(0, 1)."""
    sch = PNDMOracle()
    sch.set_timesteps(num_inference_steps)
    for t in sch.timesteps.tolist():
        x = torch.cat([latents] * 2) if guidance_scale > 1.0 else latents   # scale_model_input is the identity for PNDM
        noise = unet_fn(x.to(latents.dtype), float(t), ctx)
        if guidance_scale > 1.0:
            cond, uncond = noise.chunk(2)
            noise = uncond + guidance_scale * (cond - uncond)
        latents = sch.step(noise, t, latents)
    return latents


# ------------------------------------------------------------------------------------------------
# AutoencoderKL.decode (post_quant_conv + Decoder: conv_in, mid(resnet, attn, resnet), 4 up blocks, norm, conv_out)
# ------------------------------------------------------------------------------------------------
def vae_resnet(sd, p, x, groups):
    h = F.silu(group_norm(sd, p + "norm1", x, groups, 1e-6))
    h = conv(sd, p + "conv1", h)
    h = F.silu(group_norm(sd, p + "norm2", h, groups, 1e-6))
    h = conv(sd, p + "conv2", h)
    if (p + "conv_shortcut.weight") in sd:
        x = conv(sd, p + "conv_shortcut", x, padding=0)
    return x + h


def vae_mid_attention(sd, p, x, groups):
    """diffusers Attention inside UNetMidBlock2D of the VAE: single head over C, GroupNorm, q/k/v/out WITH bias.  diffusers
    runs it through torch SDPA (AttnProcessor2_0), whose kernels keep the scores and the softmax in fp32 for bf16 inputs, so
    the bf16 policy here does the same: fp32 scores, probabilities rounded to the activation dtype before P V."""
    B, C, H, W = x.shape
    h = group_norm(sd, p + "group_norm", x, groups, 1e-6).view(B, C, H * W).transpose(1, 2)
    q, k, v = linear(sd, p + "to_q", h), linear(sd, p + "to_k", h), linear(sd, p + "to_v", h)
    w = torch.softmax((q.float() @ k.float().transpose(-1, -2)) * C ** -0.5, dim=-1).to(v.dtype)
    o = linear(sd, p + "to_out.0", w @ v)
    return o.transpose(1, 2).reshape(B, C, H, W) + x


def vae_decode(sd, cfg, z, prefix=""):
    """AutoencoderKL.decode(z).sample — call site Emu2/emu/diffusion.py:214-216 (z already divided by 0.13025)."""
    g, boc, lpb = cfg["norm_num_groups"], cfg["block_out_channels"], cfg["layers_per_block"]
    P = prefix
    z = conv(sd, P + "post_quant_conv", z, padding=0)
    h = conv(sd, P + "decoder.conv_in", z)
    h = vae_resnet(sd, P + "decoder.mid_block.resnets.0.", h, g)
    h = vae_mid_attention(sd, P + "decoder.mid_block.attentions.0.", h, g)
    h = vae_resnet(sd, P + "decoder.mid_block.resnets.1.", h, g)
    nb = len(boc)
    for i in range(nb):
        for j in range(lpb + 1):
            h = vae_resnet(sd, f"{P}decoder.up_blocks.{i}.resnets.{j}.", h, g)
        if i < nb - 1:
            h = F.interpolate(h, scale_factor=2.0, mode="nearest")
            h = conv(sd, f"{P}decoder.up_blocks.{i}.upsamplers.0.conv", h)
    h = F.silu(group_norm(sd, P + "decoder.conv_norm_out", h, g, 1e-6))
    return conv(sd, P + "decoder.conv_out", h)


def vae_decoder_param_shapes(cfg):
    boc, lpb, lc = cfg["block_out_channels"], cfg["layers_per_block"], cfg["latent_channels"]
    s = {}

    def cv(p, o, i, k=3):
        s[p + ".weight"] = (o, i, k, k)
        s[p + ".bias"] = (o,)

    def nrm(p, c):
        s[p + ".weight"] = (c,)
        s[p + ".bias"] = (c,)

    def resnet(p, cin, cout):
        nrm(p + "norm1", cin)
        cv(p + "conv1", cout, cin)
        nrm(p + "norm2", cout)
        cv(p + "conv2", cout, cout)
        if cin != cout:
            cv(p + "conv_shortcut", cout, cin, 1)

    cv("post_quant_conv", lc, lc, 1)
    top = boc[-1]
    cv("decoder.conv_in", top, lc)
    resnet("decoder.mid_block.resnets.0.", top, top)
    nrm("decoder.mid_block.attentions.0.group_norm", top)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        s[f"decoder.mid_block.attentions.0.{n}.weight"] = (top, top)
        s[f"decoder.mid_block.attentions.0.{n}.bias"] = (top,)
    resnet("decoder.mid_block.resnets.1.", top, top)
    rev = list(reversed(boc))
    cin = top
    for i, cout in enumerate(rev):
        for j in range(lpb + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}.", cin, cout)
            cin = cout
        if i < len(rev) - 1:
            cv(f"decoder.up_blocks.{i}.upsamplers.0.conv", cout, cout)
    nrm("decoder.conv_norm_out", boc[0])
    cv("decoder.conv_out", cfg["out_channels"], boc[0])
    return s
