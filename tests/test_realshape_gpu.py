"""Model-level parity at the BENCHMARKED shapes (VERDICT r01 item 1): one real-width unit of each model runs through the
ENGINE entry points (emu_llm_prefill / emu_llm_decode, emu_vit_forward, emu_unet_forward — not the stand-alone emu_op_*
operators) and is compared with the CPU oracle twice:

  * ref32 = the oracle in fp32 (the numerical truth of the reference arithmetic), and
  * ref16 = the oracle in the reference's own dtype policy (bf16 weights / activations, fp32 softmax and norm statistics).

The bound is relative to what bf16 storage costs the reference itself:
      err(engine, ref32)  <=  RATIO * err(ref16, ref32)          (RATIO = 1.5)
and the engine must sit within ULP_GATE of the bf16-policy oracle.  Both numbers are printed (run with -s) and quoted in
README.md.  Shapes: Emu2/emu/conf/llama_config/config.json:8-21 (6656 / 52 heads x 128 / 17920, vocab 32272),
Emu2/emu/conf/emu_conf.py:7-33 (1792 / 16 heads x 112 / 15360, 1025 tokens), Emu2/emu/conf/diffusion_config/unet/config.json
(C=640 at 64x64 with 2 transformer layers, C=1280 at 32x32 with 10, cross-attention over [2, 64, 1792]).
"""
import math

import pytest
import torch

from helpers import TINY_LLAMA, TINY_VISION, StubTokenizer, make_emu2_state_dict
from oracle import diffusion_oracle as D
from oracle import emu_oracle as O

pytestmark = pytest.mark.gpu

RATIO = 1.5       # engine error vs fp32 oracle, in units of the bf16-policy oracle's own error
ULP_GATE = 4e-3   # engine vs bf16-policy oracle: one bf16 ulp (2^-8) of the largest element


def report(name, out, ref32, ref16, ratio=RATIO, gate=ULP_GATE):
    e_eng, e_bf, e_pol = O.rel_err(out, ref32), O.rel_err(ref16, ref32), O.rel_err(out, ref16)
    print("\n[realshape] %-28s engine-vs-fp32 %.3e | bf16-oracle-vs-fp32 %.3e | ratio %.2f | engine-vs-bf16-oracle %.3e"
          % (name, e_eng, e_bf, e_eng / max(e_bf, 1e-12), e_pol))
    assert e_eng <= ratio * e_bf, (name, e_eng, e_bf)
    assert e_pol <= max(gate, ratio * e_bf), (name, e_pol, e_bf)
    return e_eng, e_bf, e_pol


def _bf16(sd):
    return {k: v.to(torch.bfloat16) for k, v in sd.items()}


# ------------------------------------------------------------------------------------------------------------------
# LLaMA-33B: ONE real decoder layer + final norm + lm_head; prefill 75 tokens (left pad on row 1) then 4 decode steps
# ------------------------------------------------------------------------------------------------------------------
LLAMA_33B_1L = dict(hidden_size=6656, num_hidden_layers=1, num_attention_heads=52, intermediate_size=17920,
                    rms_norm_eps=1e-6, max_position_embeddings=2048, vocab_size=32000, rope_theta=10000.0)


def _llama_sd(cfg, vocab, seed):
    g = torch.Generator().manual_seed(seed)
    H, F = cfg["hidden_size"], cfg["intermediate_size"]
    sd = {}
    p = "decoder.lm.model.layers.0."
    for n in ("q_proj", "k_proj", "v_proj", "o_proj"):
        sd[p + "self_attn.%s.weight" % n] = torch.randn(H, H, generator=g) / math.sqrt(H)
    sd[p + "mlp.gate_proj.weight"] = torch.randn(F, H, generator=g) / math.sqrt(H)
    sd[p + "mlp.up_proj.weight"] = torch.randn(F, H, generator=g) / math.sqrt(H)
    sd[p + "mlp.down_proj.weight"] = torch.randn(H, F, generator=g) / math.sqrt(F)
    sd[p + "input_layernorm.weight"] = 1 + 0.1 * torch.randn(H, generator=g)
    sd[p + "post_attention_layernorm.weight"] = 1 + 0.1 * torch.randn(H, generator=g)
    sd["decoder.lm.model.norm.weight"] = 1 + 0.1 * torch.randn(H, generator=g)
    sd["decoder.lm.model.embed_tokens.weight"] = torch.randn(vocab, H, generator=g)
    sd["decoder.lm.lm_head.weight"] = torch.randn(vocab, H, generator=g) / math.sqrt(H)
    return sd


def _oracle_llama_steps(sd, emb, mask, toks, heads):
    """prefill + teacher-forced decode steps -> list of [B, V] logits (fp32)"""
    cache = O.KVCache(1)
    m = mask.clone()
    h = O.llama_forward(sd, emb, m, layers=1, heads=heads, position_ids=O.hf_position_ids(m), cache=cache)
    outs = [O.lm_logits(sd, h[:, -1]).float()]
    for t in range(toks.shape[1]):
        m = torch.cat((m, torch.ones(m.shape[0], 1, dtype=m.dtype)), dim=1)
        e = torch.nn.functional.embedding(toks[:, t], sd["decoder.lm.model.embed_tokens.weight"]).unsqueeze(1)
        h = O.llama_forward(sd, e, m, layers=1, heads=heads, position_ids=m.long().sum(-1, keepdim=True) - 1, cache=cache)
        outs.append(O.lm_logits(sd, h[:, -1]).float())
    return outs


def test_llama33b_layer_prefill_and_decode(cuda):
    from helpers import VOCAB
    from emu_b200.emu2.conf import CLIPVisionCfg, TextDecoderCfg
    from emu_b200.emu2.emu import EmuModel
    cfg = LLAMA_33B_1L
    sd = _llama_sd(cfg, VOCAB, seed=21)
    vis = dict(TINY_VISION, layers=1)
    m = EmuModel(CLIPVisionCfg(**vis), TextDecoderCfg(), tokenizer=StubTokenizer(), llama_config=cfg, max_batch=2, max_seq=96)
    for k, v in sd.items():
        m.engine.load_tensor(k, v)
    g = torch.Generator().manual_seed(22)
    B, N = 2, 75
    emb = torch.randn(B, N, cfg["hidden_size"], generator=g).to(torch.bfloat16)
    mask = torch.ones(B, N, dtype=torch.long)
    mask[1, :7] = 0                                   # left padding, as the tokenizer produces (Emu2/emu/emu.py:58)
    toks = torch.randint(100, 31000, (B, 4), generator=g)
    with torch.no_grad():
        ref32 = _oracle_llama_steps(sd, emb.float(), mask, toks, cfg["num_attention_heads"])
        ref16 = _oracle_llama_steps(_bf16(sd), emb, mask, toks, cfg["num_attention_heads"])
    eng = m.engine
    eng.llm_reset()
    _, lg = eng.llm_prefill(emb.cuda(), mask.cuda(), hf_positions=True, want_logits=True)
    got = [lg.float().cpu()]
    buf = torch.empty_like(lg)
    for t in range(toks.shape[1]):
        eng.llm_decode(token_ids=toks[:, t].to(torch.int32).cuda().contiguous(), logits=buf, B=B)
        got.append(buf.float().cpu())
    for s, (a, r32, r16) in enumerate(zip(got, ref32, ref16)):
        report("llama33b layer %s" % ("prefill" if s == 0 else "decode step %d" % s), a, r32, r16)
    eng.close()


# ------------------------------------------------------------------------------------------------------------------
# EVA-CLIP-4B: ONE real post-norm block (1792 wide, 16 heads x 112, MLP 15360) over the 1025 tokens of a 448x448 image
# ------------------------------------------------------------------------------------------------------------------
EVA_1L = dict(image_size=448, patch_size=14, width=1792, layers=1, head_width=112, mlp_ratio=8.571428571428571,
              n_query=64, v_query=64)


def test_eva_clip_block_1025_tokens(cuda):
    from emu_b200.emu2.conf import CLIPVisionCfg, TextDecoderCfg
    from emu_b200.emu2.emu import EmuModel
    sd = make_emu2_state_dict(vision=EVA_1L, llama=TINY_LLAMA, seed=31)
    m = EmuModel(CLIPVisionCfg(**EVA_1L), TextDecoderCfg(), tokenizer=StubTokenizer(), llama_config=TINY_LLAMA, max_batch=1,
                 max_seq=32)
    m.load_state_dict(sd)
    g = torch.Generator().manual_seed(32)
    image = torch.randn(1, 3, 448, 448, generator=g).to(torch.bfloat16)
    vsd = {k: v for k, v in sd.items() if k.startswith("visual.")}
    with torch.no_grad():
        ref32 = O.vit_forward_features(vsd, image.float(), patch=14, num_heads=16, layers=1, postnorm=True)
        ref16 = O.vit_forward_features(_bf16(vsd), image, patch=14, num_heads=16, layers=1, postnorm=True).float()
        enc32 = O.encode_image(vsd, image.float(), patch=14, num_heads=16, layers=1, n_query=64)
        enc16 = O.encode_image(_bf16(vsd), image, patch=14, num_heads=16, layers=1, n_query=64).float()
    out = m.engine.vit_forward(image.cuda(), 0, pool=False).float().cpu()
    report("eva-clip block tokens", out, ref32, ref16)
    enc = m.encode_image(image.cuda()).float().cpu()
    report("eva-clip encode_image", enc, enc32, enc16)
    m.engine.close()


# ------------------------------------------------------------------------------------------------------------------
# SDXL-topology UNet stages at the benchmarked widths: C=640 on 64x64 (2 transformer layers, 4096 tokens) and C=1280 on
# 32x32 (10 layers, 1024 tokens), UNet batch 2 (CFG), 64 context tokens of width 1792, text_time conditioning
# ------------------------------------------------------------------------------------------------------------------
UNET_STAGES = dict(in_channels=4, out_channels=4, block_out_channels=(640, 1280), layers_per_block=1,
                   transformer_layers_per_block=(2, 10), attention_head_dim=64, cross_attention_dim=1792,
                   addition_time_embed_dim=256, projection_class_embeddings_input_dim=1792 + 6 * 256, norm_num_groups=32,
                   norm_eps=1e-5)


def test_unet_stages_c640_c1280(cuda):
    from test_unet_gpu import make_engine
    cfg = UNET_STAGES
    sd = D.random_state_dict(D.unet_param_shapes(cfg), seed=41)
    eng = make_engine(cfg, sd)
    g = torch.Generator().manual_seed(42)
    ctx = torch.randn(2, 64, 1792, generator=g).to(torch.bfloat16)
    te = ctx.float().mean(1).to(torch.bfloat16)
    tid = torch.tensor([[1024, 1024, 0, 0, 1024, 1024]] * 2)
    x = torch.randn(2, 4, 64, 64, generator=g).to(torch.bfloat16)
    with torch.no_grad():
        ref32 = D.unet_forward(sd, cfg, x.float(), 981.0, ctx.float(), te.float(), tid)
        ref16 = D.unet_forward(_bf16(sd), cfg, x, 981.0, ctx, te, tid).float()
    out = eng.unet_forward(x.cuda(), 981.0, ctx.cuda(), te.cuda(), tid.cuda()).float().cpu()
    report("unet stages C=640/1280", out, ref32, ref16)
    eng.close()


# ------------------------------------------------------------------------------------------------------------------
# SDXL VAE decoder at its published width (Emu2/emu/conf/diffusion_config/vae/config.json: 128/256/512/512, 2 layers per
# block, 32 groups) on 128x128 latents -> one 1024x1024 image: GroupNorm on planes up to 1024^2 and the mid-block attention
# over 16384 tokens of width 512.  The oracle runs on the GPU here (the CPU would take minutes at this size).
# ------------------------------------------------------------------------------------------------------------------
VAE_FULL = dict(latent_channels=4, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                norm_num_groups=32)


def test_vae_decoder_real_width_128_latents(cuda):
    from emu_b200 import _lib
    cfg = VAE_FULL
    sd = D.random_state_dict(D.vae_decoder_param_shapes(cfg), seed=51)
    eng = _lib.Engine(_lib.EmuConfig())
    v = _lib.EmuVAEConfig()
    v.latent_channels, v.out_channels, v.n_blocks = 4, 3, len(cfg["block_out_channels"])
    for i, c in enumerate(cfg["block_out_channels"]):
        v.block_out_channels[i] = c
    v.layers_per_block, v.norm_groups = cfg["layers_per_block"], cfg["norm_num_groups"]
    eng.vae_configure(v)
    eng.load_state_dict({"vae." + k: t for k, t in sd.items()})
    z = torch.randn(1, 4, 128, 128, generator=torch.Generator().manual_seed(52)).to(torch.bfloat16)
    post = lambda x: (x.float() / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1).cpu()
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    try:
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        with torch.no_grad():
            ref32 = post(D.vae_decode({k: t.cuda() for k, t in sd.items()}, cfg, z.float().cuda()))
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    with torch.no_grad():
        ref16 = post(D.vae_decode({k: t.to(torch.bfloat16).cuda() for k, t in sd.items()}, cfg, z.cuda()))
    torch.cuda.empty_cache()
    out = eng.vae_decode(z.cuda()).cpu()
    assert out.shape == ref32.shape == (1, 1024, 1024, 3)
    report("vae decoder 128^2 latents", out, ref32, ref16)
    eng.close()
