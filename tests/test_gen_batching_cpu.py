"""CPU: continuous batching for image generation (emu_b200/batching.py's DenoiseSlotScheduler) gives every request the latents
`denoise` gives it alone, whatever joins and leaves around it; the serving shell's ContinuousWorker behind /v1/mmg answers what
the batching server answers; the C entry points of include/emu_b200_gen_slots.h are bound, exported and refuse bad arguments.
The engine here is a double that applies the oracle UNet row by row with the device glue's arithmetic; the device itself is in
tests/test_gen_batching_gpu.py."""
import ctypes
import json
import os
import re
import threading
import time
from types import SimpleNamespace as NS

import pytest
import torch

from oracle import diffusion_oracle as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "emu_b200_gen_slots.h")

CPU_UNET = dict(in_channels=4, out_channels=4, block_out_channels=(32, 64), layers_per_block=1,
                transformer_layers_per_block=(0, 1), attention_head_dim=32, cross_attention_dim=32,
                addition_time_embed_dim=8, projection_class_embeddings_input_dim=32 + 6 * 8, norm_num_groups=8, norm_eps=1e-5)
L_TOK = 4


class UNetDouble:
    """emu_denoise_step / emu_denoise_step_slots on the CPU: the glue with the kernels' fp32 / bf16 rounding points, the UNet
    (the fp32 oracle, output rounded to bf16) one row at a time, so a row's prediction cannot depend on its batch"""

    def __init__(self, sd, cfg):
        self.sd, self.cfg = sd, cfg
        self.slot_B = []
        self.fail_next = False

    def _eps(self, x, t, ctx, te, tid):
        return D.unet_forward(self.sd, self.cfg, x[None].float(), t, ctx[None].float(), te[None].float(),
                              tid[None]).to(torch.bfloat16)[0].float()

    def _slot(self, lat, p, ctx, te, tid, cond, uncond):
        sigma, sigma_next, t, g = [torch.tensor(v, dtype=torch.float32) for v in p]
        x = (lat.to(torch.bfloat16).float() * (1.0 / torch.sqrt(sigma * sigma + 1.0))).to(torch.bfloat16)
        ec = self._eps(x, float(t), ctx[cond], te[cond], tid[cond])
        e = ec
        if g > 1.0:
            eu = self._eps(x, float(t), ctx[uncond], te[uncond], tid[uncond])
            bf = lambda v: v.to(torch.bfloat16).float()
            e = bf(eu + bf(g * bf(ec - eu)))
        lat += e * (sigma_next - sigma)

    def denoise_step(self, lat, sigma, sigma_next, timestep, guidance, ctx, te, tid):
        B = lat.shape[0]
        for b in range(B):
            self._slot(lat[b], (sigma, sigma_next, timestep, guidance), ctx, te, tid, b, B + b)

    def denoise_step_slots(self, lat, params, live, ctx, te, tid, B):
        if self.fail_next:
            self.fail_next = False
            raise RuntimeError("engine failure")
        self.slot_B.append(B)
        for b in range(B):
            if int(live[b]):
                self._slot(lat[b], params[b].tolist(), ctx, te, tid, 2 * b, 2 * b + 1)


def pipe_over(engine, unet_cfg, L, device="cpu", vae_scale_factor=8):
    """an EmuVisualGeneration over `engine` without an encoder: requests carry prompt_embeds"""
    from emu_b200.emu2.diffusion import EmuVisualGeneration
    from emu_b200.emu2.scheduler import EulerDiscreteScheduler
    p = EmuVisualGeneration.__new__(EmuVisualGeneration)
    p.engine, p.unet_config, p.vae_scale_factor = engine, unet_cfg, vae_scale_factor
    p.scheduler = EulerDiscreteScheduler()
    p.multimodal_encoder = NS(n_query=L)
    p.device_ = device
    p.negative_prompt = {}
    return p


def make_plan(n, seed, L, Cc, hw, steps=(2, 3, 5), guidance=(3.0, 1.0), arrivals=None):
    """n requests: (arrival step, ImageRequest knobs) with staggered arrivals, mixed steps / guidance / time ids"""
    g = torch.Generator().manual_seed(seed)
    plan = []
    for i in range(n):
        gs = guidance[i % len(guidance)]
        plan.append((arrivals[i] if arrivals else i, dict(
            prompt_embeds=torch.randn(2 if gs > 1 else 1, L, Cc, generator=g).to(torch.bfloat16),
            latents=torch.randn(1, 4, hw, hw, generator=g), num_inference_steps=steps[i % len(steps)], guidance_scale=gs,
            crop_info=[8 * i, 4 * i], original_size=[512 + 64 * i, 1024 - 32 * i])))
    return plan


def run_plan(sched, plan, device="cpu"):
    """submit each request when the scheduler reaches its arrival step; run until idle -> requests in plan order"""
    from emu_b200.batching import ImageRequest
    reqs = []
    pending = sorted(range(len(plan)), key=lambda i: plan[i][0])
    out = [None] * len(plan)
    while pending or sched.busy():
        while pending and plan[pending[0]][0] <= sched.steps:
            i = pending.pop(0)
            k = dict(plan[i][1])
            k["prompt_embeds"] = k["prompt_embeds"].to(device)
            k["latents"] = k["latents"].to(device)
            out[i] = sched.submit(ImageRequest(height=sched.height, width=sched.width, output_type="latent", **k))
        sched.step()
    return out


def solo(pipe, height, width, knobs):
    k = dict(knobs)
    pe = k.pop("prompt_embeds").to(pipe.device_)
    lat = k.pop("latents").to(pipe.device_)
    return pipe.denoise(pe.to(torch.bfloat16), 1, height, width, k["num_inference_steps"], k["guidance_scale"],
                        k["crop_info"], k["original_size"], latents=lat)


@pytest.fixture(scope="module")
def unet_sd():
    return D.random_state_dict(D.unet_param_shapes(CPU_UNET), seed=7)


def test_every_request_gets_its_solo_latents_bitwise(unet_sd):
    from emu_b200.batching import DenoiseSlotScheduler
    eng = UNetDouble(unet_sd, CPU_UNET)
    pipe = pipe_over(eng, CPU_UNET, L_TOK)
    sched = DenoiseSlotScheduler(pipe, n_slots=3, height=64, width=64)
    plan = make_plan(5, seed=1, L=L_TOK, Cc=32, hw=8, arrivals=[0, 0, 2, 3, 3])
    reqs = run_plan(sched, plan)
    assert all(r.error is None for r in reqs), [r.error for r in reqs]
    for r, (_, knobs) in zip(reqs, plan):
        want = solo(pipe, 64, 64, knobs)
        assert torch.equal(r.result, want), r.slot
    # B = highest live slot + 1: 0 and 1 join at step 0 (2 and 3 steps); 2 joins at step 2 into slot 0, which 0 left; 3 and 4
    # join at step 3 into slots 1 and 2; 3 leaves after step 4, 4 after step 5, and 2 (5 steps) finishes alone in slot 0
    assert list(sched.batch_sizes) == [2, 2, 2, 3, 3, 3, 1]
    assert [r.slot for r in reqs] == [0, 1, 0, 1, 2]
    assert eng.slot_B[0] == 3                           # the warm-up at n_slots, every slot dead
    assert list(eng.slot_B[1:]) == list(sched.batch_sizes)


def test_slots_are_reused_and_a_failing_encode_fails_only_its_request(unet_sd):
    from emu_b200.batching import DenoiseSlotScheduler, ImageRequest
    eng = UNetDouble(unet_sd, CPU_UNET)
    pipe = pipe_over(eng, CPU_UNET, L_TOK)

    def encode(inputs, do_cfg):
        if inputs == ["bad"]:
            raise ValueError("cannot encode this prompt")
        g = torch.Generator().manual_seed(len(inputs[0]))
        return torch.randn(2 if do_cfg else 1, L_TOK, 32, generator=g)
    pipe._prepare_and_encode_inputs = encode
    sched = DenoiseSlotScheduler(pipe, n_slots=2, height=64, width=64)
    lat = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(3))
    mk = lambda text, steps: sched.submit(ImageRequest(inputs=[text], num_inference_steps=steps, height=64, width=64,
                                                       latents=lat, output_type="latent"))
    a, bad, b = mk("a cat", 2), mk("bad", 2), mk("a dog", 3)
    sched.step()
    assert a.slot == 0 and b.slot == 1 and bad.done.is_set() and "cannot encode" in str(bad.error)
    c = mk("a bird!", 2)
    sched.run_until_idle()
    assert c.slot == 0                                  # a's slot, free again after its two steps
    for r, text, steps in ((a, "a cat", 2), (b, "a dog", 3), (c, "a bird!", 2)):
        assert r.error is None
        want = pipe.denoise(encode([text], True).to(torch.bfloat16), 1, 64, 64, steps, 3.0, latents=lat)
        assert torch.equal(r.result, want)
    with pytest.raises(ValueError, match="512x512"):
        sched.submit(ImageRequest(inputs=["x"], height=512, width=512))


def test_an_engine_failure_fails_the_live_requests_and_the_scheduler_goes_on(unet_sd):
    from emu_b200.batching import DenoiseSlotScheduler
    eng = UNetDouble(unet_sd, CPU_UNET)
    pipe = pipe_over(eng, CPU_UNET, L_TOK)
    sched = DenoiseSlotScheduler(pipe, n_slots=2, height=64, width=64)
    plan = make_plan(2, seed=4, L=L_TOK, Cc=32, hw=8, steps=(2,), arrivals=[0, 0])
    eng.fail_next = True
    first = run_plan(sched, plan)
    assert all("engine failure" in str(r.error) for r in first) and not sched.busy()
    again = run_plan(sched, make_plan(1, seed=5, L=L_TOK, Cc=32, hw=8, steps=(2,)))
    assert again[0].error is None


# ---- the serving shell: /v1/mmg through --continuous-generation, posted as the demo front end posts it ----
class ServedPipe:
    """an EmuVisualGeneration over the engine double whose encoder and decoder are deterministic stand-ins"""

    def __new__(cls, sd, delay=0.0):
        eng = UNetDouble(sd, CPU_UNET)
        p = pipe_over(eng, CPU_UNET, L_TOK)

        def encode(inputs, do_cfg):
            g = torch.Generator().manual_seed(sum(map(ord, "".join(x for x in inputs if isinstance(x, str)))))
            return torch.randn(2 if do_cfg else 1, L_TOK, 32, generator=g)

        def decode(latents):
            time.sleep(delay)
            u8 = ((latents[:, :3].float().tanh() + 1) * 127.5).round().clamp(0, 255).to(torch.uint8)
            return u8.repeat_interleave(8, 2).repeat_interleave(8, 3).permute(0, 2, 3, 1).numpy(), None

        def initial(batch_size, height, width, init_noise_sigma, generator=None, latents=None):
            base = torch.linspace(-1, 1, 4 * 8 * 8).view(1, 4, 8, 8).repeat(batch_size, 1, 1, 1)
            return (base.to(torch.bfloat16).float() * init_noise_sigma).contiguous()
        p._prepare_and_encode_inputs, p.decode_and_check, p.initial_latents = encode, decode, initial
        return p


def test_generation_over_the_demo_form_matches_the_batching_server(unet_sd, monkeypatch):
    import requests
    from emu_b200 import serve
    import emu_b200.batching as batching
    monkeypatch.setattr(serve, "generate_scheduler_for",
                        lambda pipe, n: batching.DenoiseSlotScheduler(pipe, n, height=64, width=64))
    forms = [("a cat", "3.0", "2"), ("a dog", "3.0", "3"), ("a red bird", "1.0", "2"), ("a cat", "3.0", "3")]

    def post_all(url):
        out = [None] * len(forms)

        def one(i):
            p, g, s = forms[i]
            r = requests.post(url + "/v1/mmg", data=dict(log_id="g%d" % i, prompt=json.dumps([["TEXT", p]]),
                                                         classifier_free_guidance=g, steps=s), timeout=60)
            out[i] = r.json()
        ts = [threading.Thread(target=one, args=(i,)) for i in range(len(forms))]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        return out

    answers = {}
    for mode in ("batching", "continuous"):
        pipe = ServedPipe(unet_sd, delay=0.05)
        if mode == "batching":   # forward at 64x64 (the form cannot send a size; the continuous scheduler is built for it)
            fwd = pipe.forward
            pipe.forward = lambda inputs, **k: fwd(inputs, height=64, width=64, **k)
            fb = pipe.forward_batch
            pipe.forward_batch = lambda batch, **k: fb(batch, height=64, width=64, **k)
            pipe.__call__ = pipe.forward
        srv = serve.EmuServer(generate=_Callable(pipe), host="127.0.0.1", port=0, max_images_per_batch=3,
                              generate_scheduler=mode).start()
        try:
            answers[mode] = post_all("http://127.0.0.1:%d" % srv.port)
            if mode == "continuous":
                sched = srv.gen_workers[0].scheduler
                assert max(sched.batch_sizes) >= 2     # requests with 2 and 3 steps shared UNet steps
        finally:
            srv.shutdown()
    assert all(a["code"] == 0 for a in answers["continuous"]), answers["continuous"]
    assert answers["continuous"] == answers["batching"]
    with pytest.raises(ValueError, match="generate_scheduler"):
        serve.EmuServer(generate=ServedPipe(unet_sd), host="127.0.0.1", port=0, generate_scheduler="eager")


class _Callable:
    """the pipeline as BatchingWorker calls it (`pipeline(inputs=..., **knobs)`), every other attribute passed through"""

    def __init__(self, pipe):
        object.__setattr__(self, "_p", pipe)

    def __call__(self, inputs, **knobs):
        return self._p.forward(inputs, **knobs)

    def __getattr__(self, k):
        return getattr(self._p, k)


def test_continuous_generation_is_opt_in():
    from emu_b200 import serve
    from test_serve_cpu import FakeGen
    srv = serve.EmuServer(generate=FakeGen(), host="127.0.0.1", port=0)
    try:
        assert isinstance(srv.gen_workers[0], serve.BatchingWorker)
    finally:
        srv.httpd.server_close()
    ap_help = serve.main.__code__.co_consts
    assert any(isinstance(c, str) and "--continuous-generation" in c for c in ap_help)


# ---- the C entry points ----
@pytest.fixture(scope="module")
def lib():
    from emu_b200 import build, _lib
    build.build()
    return _lib.load()


def test_gen_slot_header_symbols_are_bound_and_exported(lib):
    from emu_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(emu_[a-z0-9_]+)\s*\(", src)))
    assert sorted(_lib.GEN_SLOT_SYMBOLS) == syms
    assert all(hasattr(lib, s) for s in syms)
    others = set(_lib.SYMBOLS) | set(_lib.SAFETY_SYMBOLS) | set(_lib.SLOT_SYMBOLS) | set(_lib.OPS_SYMBOLS)
    assert not set(_lib.GEN_SLOT_SYMBOLS) & others


P = ctypes.c_void_p(0x10000000)


def _good_args():
    N = None
    return {
        #                          e  lat params live ctx L  te tid B  h   w   stream
        "emu_denoise_step_slots": [P, P, P, P, P, 64, P, P, 4, 16, 16, N],
        #                          lat xin t  B  C  HW  Cp params ps copies cs ub stream
        "emu_op_denoise_prepare": [P, P, P, 4, 4, 35, 8, P, 4, 2, 2, 1, N],
        #                        lat eps live B  C  HW  ld params ps cs ub stream
        "emu_op_denoise_euler": [P, P, N, 4, 4, 35, 8, P, 4, 1, 4, N],
    }


BAD = [
    ("emu_denoise_step_slots", 0, None, "engine"), ("emu_denoise_step_slots", 1, None, "latents"),
    ("emu_denoise_step_slots", 2, None, "params"), ("emu_denoise_step_slots", 3, None, "live"),
    ("emu_denoise_step_slots", 4, None, "ctx"), ("emu_denoise_step_slots", 6, None, "text_embeds"),
    ("emu_denoise_step_slots", 7, None, "time_ids"), ("emu_denoise_step_slots", 8, 0, "B = 0"),
    ("emu_denoise_step_slots", 8, 33, "B = 33"), ("emu_denoise_step_slots", 5, 0, "L = 0"),
    ("emu_denoise_step_slots", 9, 0, "h = 0"), ("emu_denoise_step_slots", 10, -8, "w < 0"),
    ("emu_op_denoise_prepare", 0, None, "latents"), ("emu_op_denoise_prepare", 1, None, "xin"),
    ("emu_op_denoise_prepare", 2, None, "t_rows"), ("emu_op_denoise_prepare", 7, None, "params"),
    ("emu_op_denoise_prepare", 3, 0, "B = 0"), ("emu_op_denoise_prepare", 3, 33, "B = 33"),
    ("emu_op_denoise_prepare", 4, 0, "C = 0"), ("emu_op_denoise_prepare", 5, 0, "HW = 0"),
    ("emu_op_denoise_prepare", 6, 3, "Cp < C"), ("emu_op_denoise_prepare", 8, 3, "ps = 3"),
    ("emu_op_denoise_prepare", 9, 3, "copies = 3"), ("emu_op_denoise_prepare", 9, 1, "copies = 1 with adjacent rows"), ("emu_op_denoise_prepare", 11, 2, "cs = 2, ub = 2"),
    ("emu_op_denoise_euler", 0, None, "latents"), ("emu_op_denoise_euler", 1, None, "eps"),
    ("emu_op_denoise_euler", 7, None, "params"), ("emu_op_denoise_euler", 3, 0, "B = 0"),
    ("emu_op_denoise_euler", 3, 33, "B = 33"), ("emu_op_denoise_euler", 6, 3, "ld < C"),
    ("emu_op_denoise_euler", 5, -1, "HW < 0"), ("emu_op_denoise_euler", 10, 3, "cs = 1, ub != B"),
]


def test_every_entry_point_is_exercised_by_the_refusals():
    assert {b[0] for b in BAD} == set(_good_args())


@pytest.mark.parametrize("name,i,bad,what", BAD, ids=["%s: %s" % (b[0], b[3]) for b in BAD])
def test_bad_arguments_are_refused_before_any_cuda_call(lib, name, i, bad, what):
    """NULL pointers, B outside 1..32, non-positive sizes and a row layout other than the two are EMU_ERR_INVALID.  The
    pointers (the engine's included) are fake, so a missed check would crash or come back as another error; with a GPU it
    would launch on fake addresses, so the test runs only where there is none."""
    if torch.cuda.is_available():
        pytest.skip("fake device addresses: checked on a machine without a GPU")
    args = _good_args()[name]
    args[i] = bad
    fn = getattr(lib, name)
    fn.restype, fn.argtypes = ctypes.c_int, None
    assert fn(*args) == -1, (name, what)
