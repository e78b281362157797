"""GPU: latent slots (include/emu_b200_gen_slots.h) on the device.  The glue kernels against a torch restatement, bit for bit;
emu_denoise_step_slots with every slot on one schedule against emu_denoise_step; staggered traces through DenoiseSlotScheduler
on a tiny UNet and at the Emu2-Gen UNet widths, every request bitwise equal to its own solo loop, graphed and eager; and the
whole pipeline (tiny Emu2 encoder, tiny UNet, tiny VAE, the safety checker) against `forward` alone, byte for byte."""
import os

import numpy as np
import pytest
import torch

from oracle import diffusion_oracle as D
from test_gen_batching_cpu import make_plan, pipe_over, run_plan, solo

pytestmark = pytest.mark.gpu

TINY_UNET = dict(in_channels=4, out_channels=4, block_out_channels=(64, 128, 256), layers_per_block=2,
                 transformer_layers_per_block=(0, 1, 2), attention_head_dim=64, cross_attention_dim=128,
                 addition_time_embed_dim=32, projection_class_embeddings_input_dim=128 + 6 * 32, norm_num_groups=32,
                 norm_eps=1e-5)
# the same network in the diffusers JSON format EmuVisualGeneration reads (no mid-block attention, as TINY_UNET's engine)
TINY_UNET_JSON = dict(TINY_UNET, attention_head_dim=[1, 2, 4], use_linear_projection=True, mid_block_type="UNetMidBlock2D",
                      down_block_types=["DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"])
TINY_VAE = dict(latent_channels=4, out_channels=3, block_out_channels=(32, 64, 64), layers_per_block=1, norm_num_groups=32,
                scaling_factor=0.13025)


def _f64_inv(sig):
    return (1.0 / torch.sqrt((sig.double() ** 2 + 1).float())).float()


def ref_prepare(lat, params, Cp, copies, adjacent):
    B, C, h, w = lat.shape
    p = params.expand(B, 4) if params.dim() == 1 else params
    xin = torch.zeros(copies * B, h, w, Cp, dtype=torch.bfloat16)
    t = torch.full((copies * B,), float("nan"))
    for b in range(B):
        x = (lat[b].to(torch.bfloat16).float() * _f64_inv(p[b, 0])).to(torch.bfloat16).permute(1, 2, 0)
        for k in range(copies):
            row = 2 * b + k if adjacent else k * B + b
            xin[row, :, :, :C] = x
            t[row] = p[b, 2]
    return xin, t


def ref_euler(lat, eps, params, live, adjacent):
    B, C, h, w = lat.shape
    p = params.expand(B, 4) if params.dim() == 1 else params
    out = lat.clone()
    bf = lambda v: v.to(torch.bfloat16).float()
    for b in range(B):
        if live is not None and not live[b]:
            continue
        cr, ur = (2 * b, 2 * b + 1) if adjacent else (b, B + b)
        ec = eps[cr, :, :, :C].permute(2, 0, 1).float()
        e = ec
        if p[b, 3] > 1:
            eu = eps[ur, :, :, :C].permute(2, 0, 1).float()
            e = bf(eu + bf(p[b, 3] * bf(ec - eu)))
        # the kernel's lat += e * dt is one fused multiply-add: exact product, one rounding
        out[b] = (lat[b].double() + e.double() * (p[b, 1] - p[b, 0]).double()).float()
    return out


@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("adjacent", [False, True])
def test_glue_operators_match_torch_bitwise(cuda, B, adjacent):
    from emu_b200 import _lib
    g = torch.Generator().manual_seed(B * 2 + adjacent)
    h, w, C, Cp, ld = 5, 7, 4, 8, 8                       # HW = 35: no multiple of any grid stride
    lat = torch.randn(B, C, h, w, generator=g) * 10
    params = torch.stack([torch.rand(B, generator=g) * 10 + 0.1, torch.rand(B, generator=g) * 5,
                          torch.randint(1, 1000, (B,), generator=g).float(), torch.tensor([3.0, 1.0, 7.5, 0.5] * 8)[:B]], 1)
    for copies in ((2,) if adjacent else (1, 2)):      # adjacent rows: every slot owns two
        xin, t = _lib.op_denoise_prepare(lat.cuda(), params.cuda(), Cp, copies, adjacent)
        rx, rt = ref_prepare(lat, params, Cp, copies, adjacent)
        assert torch.equal(xin.cpu().view(torch.int16), rx.view(torch.int16)) and torch.equal(t.cpu(), rt)
    # one parameter set for every slot: the form emu_denoise_step uses
    xin, _ = _lib.op_denoise_prepare(lat.cuda(), params[0].contiguous().cuda(), Cp, 2, adjacent)
    assert torch.equal(xin.cpu().view(torch.int16), ref_prepare(lat, params[0], Cp, 2, adjacent)[0].view(torch.int16))
    eps = (torch.randn(2 * B, h, w, ld, generator=g)).to(torch.bfloat16)
    live = torch.tensor([1, 0, 1, 1, 0, 1, 1, 1][:B], dtype=torch.int32)
    for b in range(B):                                  # rows that must not be read hold NaN
        if not live[b]:
            eps[[2 * b, 2 * b + 1] if adjacent else [b, B + b]] = float("nan")
        elif params[b, 3] <= 1:
            eps[2 * b + 1 if adjacent else B + b] = float("nan")
    for lv in (live, None):
        if lv is None:
            eps = torch.nan_to_num(eps, nan=0.25)
        out = lat.clone().cuda()
        _lib.op_denoise_euler(out, eps.cuda(), params.cuda(), None if lv is None else lv.cuda(), adjacent)
        want = ref_euler(lat, eps, params, lv, adjacent)
        assert torch.equal(out.cpu().view(torch.int32), want.view(torch.int32))
        if lv is not None:
            dead = ~lv.bool()
            assert torch.equal(out.cpu()[dead].view(torch.int32), lat[dead].view(torch.int32))   # untouched, bit for bit


def _tiny_engine(cfg=TINY_UNET, seed=3):
    from test_unet_gpu import make_engine
    return make_engine(cfg, D.random_state_dict(D.unet_param_shapes(cfg), seed=seed))


@pytest.fixture(scope="module")
def tiny(cuda):
    return _tiny_engine()


def test_uniform_slots_equal_the_batched_step(tiny):
    """every slot on one schedule: emu_denoise_step_slots (rows 2b, 2b+1) == emu_denoise_step on the same B requests
    ([cond; uncond] rows), bitwise"""
    B, hw, steps = 3, 32, 3
    g = torch.Generator(device="cuda").manual_seed(5)
    cond, unc = torch.randn(B, 8, 128, generator=g, device="cuda"), torch.randn(1, 8, 128, generator=g, device="cuda")
    ctx = torch.cat([cond, unc.expand(B, -1, -1)]).to(torch.bfloat16).contiguous()
    te = ctx.float().mean(1).to(torch.bfloat16).contiguous()
    tid = torch.tensor([[1024, 768, 0, 16, 256, 256]] * (2 * B), dtype=torch.int32, device="cuda")
    lat0 = torch.randn(B, 4, hw, hw, generator=g, device="cuda") * 14.6
    il = torch.stack([torch.arange(B), torch.arange(B) + B], 1).reshape(-1).cuda()    # slot order: cond_b, uncond_b
    sctx, ste, stid = ctx[il].contiguous(), te[il].contiguous(), tid[il].contiguous()
    ts, sig, _ = D.euler_tables(steps)
    a, b = lat0.clone(), lat0.clone()
    live = torch.ones(B, dtype=torch.int32, device="cuda")
    params = torch.zeros(B, 4, device="cuda")
    for i in range(steps):
        tiny.denoise_step(a, float(sig[i]), float(sig[i + 1]), float(ts[i]), 3.0, ctx, te, tid)
        params.copy_(torch.tensor([float(sig[i]), float(sig[i + 1]), float(ts[i]), 3.0]).expand(B, 4))
        tiny.denoise_step_slots(b, params, live, sctx, ste, stid, B)
    assert torch.isfinite(a).all() and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _staggered(pipe, n_slots, hw, plan):
    from emu_b200.batching import DenoiseSlotScheduler
    f = pipe.vae_scale_factor
    sched = DenoiseSlotScheduler(pipe, n_slots=n_slots, height=hw * f, width=hw * f)
    reqs = run_plan(sched, plan, device="cuda")
    assert all(r.error is None for r in reqs), [r.error for r in reqs]
    return sched, [r.result for r in reqs]


def _check_trace(pipe, n_slots, hw, plan, Cc):
    sched, got = _staggered(pipe, n_slots, hw, plan)
    assert max(sched.batch_sizes) == n_slots
    f = pipe.vae_scale_factor
    for i, (r, (_, knobs)) in enumerate(zip(got, plan)):
        want = solo(pipe, hw * f, hw * f, knobs)
        assert torch.isfinite(want).all()
        assert torch.equal(r.view(torch.int32), want.view(torch.int32)), "request %d differs from its solo loop" % i
    return got


def test_staggered_trace_tiny_unet_graph_and_eager(tiny):
    """4 slots; joins at steps 0, 2 and 3; steps {2, 3, 5}, guidance {3, 1}, own time ids; every request equals its solo
    emu_denoise_step loop bitwise, and the graphed run equals the eager one"""
    pipe = pipe_over(tiny, TINY_UNET, 8, device="cuda")
    plan = make_plan(6, seed=2, L=8, Cc=128, hw=32, arrivals=[0, 0, 2, 2, 3, 3])
    graphed = _check_trace(pipe, 4, 32, plan, 128)
    os.environ["EMU_NO_GRAPH"] = "1"
    try:
        _, eager = _staggered(pipe, 4, 32, plan)
    finally:
        del os.environ["EMU_NO_GRAPH"]
    for a, b in zip(graphed, eager):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_staggered_trace_at_emu2_gen_widths(cuda):
    import bench
    eng, cfg = bench.make_unet_engine(seed=1)
    try:
        pipe = pipe_over(eng, cfg, 64, device="cuda")
        plan = make_plan(4, seed=3, L=64, Cc=cfg["cross_attention_dim"], hw=32, steps=(2, 3), arrivals=[0, 1, 1, 2])
        _check_trace(pipe, 3, 32, plan, cfg["cross_attention_dim"])
    finally:
        eng.close()


class TextTokenizer:
    """helpers.StubTokenizer plus text: one id per character, the special tokens as themselves, left padding"""

    def __new__(cls):
        import re
        from types import SimpleNamespace
        from helpers import StubTokenizer

        class T(StubTokenizer):
            def __call__(self, texts, padding="longest", return_tensors="pt"):
                pat = "(" + "|".join(re.escape(k) for k in self._special) + ")"
                rows = [[1] + [self._special[p] if p in self._special else 100 + ord(ch) % 1000
                               for p in re.split(pat, t) if p for ch in ([p] if p in self._special else p)] for t in texts]
                n = max(map(len, rows))
                ids = torch.tensor([[self.pad_token_id] * (n - len(r)) + r for r in rows])
                mask = torch.tensor([[0] * (n - len(r)) + [1] * len(r) for r in rows])
                return SimpleNamespace(input_ids=ids, attention_mask=mask)
        return T()


def test_scheduler_images_equal_forward_alone(cuda):
    """DenoiseSlotScheduler over an EmuVisualGeneration: the tiny Emu2 model encodes the prompts, the tiny UNet denoises,
    the tiny VAE decodes and the safety checker (a tiny tower) flags: every image and flag equals `forward` alone"""
    from helpers import TINY_LLAMA, TINY_VISION, make_emu2_state_dict
    from oracle import safety_oracle as S
    from test_safety_gpu import TINY as TINY_SAFETY, _checker
    from emu_b200.batching import DenoiseSlotScheduler, ImageRequest
    from emu_b200.emu2.conf import CLIPVisionCfg, TextDecoderCfg
    from emu_b200.emu2.diffusion import EmuVisualGeneration
    from emu_b200.emu2.emu import EmuModel
    from emu_b200.emu2.scheduler import EulerDiscreteScheduler
    m = EmuModel(CLIPVisionCfg(**TINY_VISION), TextDecoderCfg(), tokenizer=TextTokenizer(), llama_config=TINY_LLAMA,
                 max_batch=8, max_seq=128)
    m.load_state_dict(make_emu2_state_dict())
    ck = _checker(TINY_SAFETY, S.random_state_dict(TINY_SAFETY, seed=21))
    pipe = EmuVisualGeneration(m, EulerDiscreteScheduler(), TINY_UNET_JSON, TINY_VAE, safety_checker=ck)
    pipe.load_state_dict({"unet." + k: v for k, v in D.random_state_dict(D.unet_param_shapes(TINY_UNET), seed=3).items()})
    pipe.load_state_dict({"vae." + k: v for k, v in D.random_state_dict(D.vae_decoder_param_shapes(TINY_VAE), seed=5).items()})
    H = W = 128                                          # latent 32x32 (VAE factor 4)
    g = torch.Generator().manual_seed(9)
    knobs = [dict(inputs=["a cat"], num_inference_steps=3, guidance_scale=3.0),
             dict(inputs=["a red dog on grass"], num_inference_steps=2, guidance_scale=1.0, crop_info=[16, 0]),
             dict(inputs=["a bird"], num_inference_steps=4, guidance_scale=5.0, original_size=[768, 512])]
    for k in knobs:
        k["latents"] = torch.randn(1, 4, 32, 32, generator=g).cuda()
    sched = DenoiseSlotScheduler(pipe, n_slots=2, height=H, width=W)
    reqs = [sched.submit(ImageRequest(**knobs[0])), sched.submit(ImageRequest(**knobs[1]))]
    sched.step()
    reqs.append(sched.submit(ImageRequest(**knobs[2])))
    sched.run_until_idle()
    assert [r.error for r in reqs] == [None] * 3
    assert max(sched.batch_sizes) == 2
    for r, k in zip(reqs, knobs):
        alone = pipe.forward(height=H, width=W, **k)
        assert np.array_equal(np.asarray(r.result.image), np.asarray(alone.image))
        assert r.result.nsfw_content_detected == alone.nsfw_content_detected is not None
