"""CPU: regression slots (include/emu_b200_regress.h) behind DenoiseSlotScheduler(encode_steps=R).  Over an oracle double of the
engine — slot-mode LLaMA with regression slots, the oracle UNet row by row — every pool request's L embeddings equal
`generate_image_cached` on its prompt alone, and its latents equal `denoise` on those embeddings alone, whatever joins and
leaves around it; a failing encode fails alone and gives both its slots back; without encode_steps the LLM never enters slot
mode; the serving flag needs continuous generation; the C entry points are bound, exported and refuse bad arguments."""
import ctypes
import os
import re
from types import SimpleNamespace as NS

import pytest
import torch
import torch.nn.functional as F
from PIL import Image

from helpers import StubTokenizer, make_emu2_state_dict
from oracle import diffusion_oracle as D
from oracle import emu_oracle as O
from test_batching_cpu import SlotOracleEngine
from test_gen_batching_cpu import CPU_UNET, UNetDouble, pipe_over
from test_generation_cpu import L, NH

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NQ, WIDTH, HIDDEN = 4, 128, 256                     # the tiny Emu2's n_query, ViT width and LLaMA width (tests/helpers.py)
UNET = dict(CPU_UNET, cross_attention_dim=WIDTH, projection_class_embeddings_input_dim=WIDTH + 6 * 8)


class RegressOracleEngine(SlotOracleEngine):
    """SlotOracleEngine + regression slots: each slot regresses as generate_image_cached does for its prompt alone (fp32
    feedback, bf16 output rows); the UNet entry points are UNetDouble's"""

    def __init__(self, sd, unet_sd, max_batch=8, max_seq=128):
        super().__init__(sd, max_batch, max_seq)
        self.unet = UNetDouble(unet_sd, UNET)
        self.denoise_step, self.denoise_step_slots = self.unet.denoise_step, self.unet.denoise_step_slots
        self.calls = []
        self.fail_join_len = None                   # a join with a prompt of this many tokens fails

    def slots_begin(self, n_slots):
        self.calls.append(("slots_begin", n_slots))
        super().slots_begin(n_slots)
        self.fb, self.k, self.regress = [None] * n_slots, [0] * n_slots, set()

    def regress_join(self, slots, new, embeds, out):
        self.calls.append(("regress_join", list(slots)))
        self._slots(slots, True)
        if self.fail_join_len in new:
            raise RuntimeError("join failed")
        off = 0
        for s, k in zip(slots, new):
            e, off = embeds[off:off + k][None].float(), off + k
            mm = torch.ones(1, k, dtype=torch.long)
            cache = O.KVCache(L)
            h = O.llama_forward(self.sd, e, mm, layers=L, heads=NH, cache=cache)
            r = F.linear(h[:, -1, :], self.sd["project_down.weight"])
            self.caches[s], self.masks[s], self.group[s], self.lens[s] = cache, mm, s, k
            self.fb[s], self.k[s] = r, 1
            out[s, 0] = r[0]
            self.regress.add(s)

    def regress_step(self, B, out):
        live = [s for s in range(self.n_slots) if self.group[s] >= 0]
        assert live and max(live) < B <= self.n_slots and all(s in self.regress for s in live)
        self.calls.append(("regress_step", B))
        for s in live:
            emb = F.linear(self.fb[s], self.sd["project_up.weight"]).unsqueeze(1)
            mask = torch.cat((self.masks[s], torch.ones(1, 1, dtype=self.masks[s].dtype)), dim=1)
            assert mask.shape[1] <= self.cfg.llm_max_seq, "KV cache full"
            h = O.llama_forward(self.sd, emb, mask, layers=L, heads=NH, cache=self.caches[s])
            r = F.linear(h[:, -1, :], self.sd["project_down.weight"])
            self.fb[s], self.masks[s], self.lens[s] = r, mask, self.lens[s] + 1
            if self.k[s] < out.shape[1]:
                out[s, self.k[s]] = r[0]
            self.k[s] = min(self.k[s] + 1, out.shape[1])

    def leave(self, slots):
        self.calls.append(("leave", list(slots)))
        super().leave(slots)
        self.regress -= set(slots)


class TextTokenizer(StubTokenizer):
    """StubTokenizer plus text: BOS, one id per character, the special tokens as themselves, left padding"""

    def __call__(self, texts, padding="longest", return_tensors="pt"):
        pat = "(" + "|".join(re.escape(k) for k in self._special) + ")"
        rows = [[1] + [self._special[p] if p in self._special else 100 + ord(ch) % 1000
                       for p in re.split(pat, t) if p for ch in ([p] if p in self._special else p)] for t in texts]
        n = max(map(len, rows))
        return NS(input_ids=torch.tensor([[self.pad_token_id] * (n - len(r)) + r for r in rows]),
                  attention_mask=torch.tensor([[0] * (n - len(r)) + [1] * len(r) for r in rows]))


def encoder(engine):
    """EmuModel's host code over the engine double, the ViT and projections by the oracle"""
    from emu_b200.emu2.emu import EmuModel
    sd = engine.sd
    m = EmuModel.__new__(EmuModel)
    engine.llm_embed = lambda ids: F.embedding(ids.long(), sd["decoder.lm.model.embed_tokens.weight"])
    m.engine, m.device_ = engine, torch.device("cpu")
    m.decoder, m.n_query, m.v_query, m.hidden = NS(tokenizer=TextTokenizer()), NQ, NQ, HIDDEN
    m.vision_cfg = NS(width=WIDTH)
    m.image_placeholder = "[IMG]" + "<image>" * NQ + "[/IMG]"

    def encode(image, n_query=None):
        if image.shape[-1] != 56:
            raise ValueError("picture of the wrong size")
        return O.encode_image(sd, image.float(), patch=14, num_heads=4, layers=2, n_query=n_query or NQ)
    m.encode_image = encode
    m._project_up = lambda x: F.linear(x.float(), sd["project_up.weight"])
    m._project_down = lambda x: F.linear(x.float(), sd["project_down.weight"])
    return m


def pipeline(sd, unet_sd, max_seq=128):
    from emu_b200.emu2.constants import OPENAI_DATASET_MEAN, OPENAI_DATASET_STD
    eng = RegressOracleEngine(sd, unet_sd, max_seq=max_seq)
    p = pipe_over(eng, UNET, NQ)
    p.multimodal_encoder = encoder(eng)
    p.eva_size, p.eva_mean, p.eva_std = 56, OPENAI_DATASET_MEAN, OPENAI_DATASET_STD
    return p, eng


@pytest.fixture(scope="module")
def sd():
    return make_emu2_state_dict()


@pytest.fixture(scope="module")
def unet_sd():
    return D.random_state_dict(D.unet_param_shapes(UNET), seed=7)


def picture(seed, size=56):
    g = torch.Generator().manual_seed(seed)
    return Image.fromarray(torch.randint(0, 256, (size, size, 3), generator=g, dtype=torch.uint8).numpy())


def plan(n_slots):
    """(arrival step, ImageRequest knobs): text prompts of different lengths, one picture + text prompt (both through the
    pool), one request with prompt_embeds and one pictures-only request (both encoded at admission), guidance 3 and 1"""
    g = torch.Generator().manual_seed(11)
    lat = lambda: torch.randn(1, 4, 8, 8, generator=g)
    items = [(0, dict(inputs=["a red cat"], guidance_scale=3.0, num_inference_steps=2)),
             (0, dict(inputs=["two dogs on a very long beach at dusk"], guidance_scale=1.0, num_inference_steps=3)),
             (0, dict(inputs=["x", picture(1), "in this style"], guidance_scale=3.0, num_inference_steps=2)),
             (1, dict(prompt_embeds=torch.randn(2, NQ, WIDTH, generator=g).to(torch.bfloat16), guidance_scale=3.0,
                      num_inference_steps=2)),
             (2, dict(inputs=["a bird"], guidance_scale=3.0, num_inference_steps=3, crop_info=[8, 4])),
             (2, dict(inputs=[picture(2)], guidance_scale=3.0, num_inference_steps=2)),
             (4, dict(inputs=["the sea"], guidance_scale=1.0, num_inference_steps=2, original_size=[768, 512]))]
    for _, k in items:
        k["latents"] = lat()
    return items


def run(sched, items):
    from emu_b200.batching import ImageRequest
    pending, out, calls = sorted(range(len(items)), key=lambda i: items[i][0]), [None] * len(items), 0
    while pending or sched.busy():
        while pending and items[pending[0]][0] <= calls:
            i = pending.pop(0)
            out[i] = sched.submit(ImageRequest(height=64, width=64, output_type="latent", **items[i][1]))
        sched.step()
        calls += 1
    return out


def solo_embeds(pipe, inputs):
    """the request's prompt embeddings regressed alone by the fp32 oracle (generate_image_cached), rounded to bf16"""
    from emu_b200.emu2.constants import DEFAULT_IMG_PLACEHOLDER
    enc = pipe.multimodal_encoder
    text, pictures, _ = pipe._split_prompt(inputs, DEFAULT_IMG_PLACEHOLDER)
    ids, mask, image_id = enc.image_prompt_ids([text])
    e = enc.image_prompt_embeds(ids, pictures, image_id)
    return O.generate_image_cached(enc.engine.sd, e, mask, NQ, layers=L, heads=NH).to(torch.bfloat16)


@pytest.mark.parametrize("R", [1, 5, 64])
def test_pool_requests_get_their_solo_embeddings_and_latents(sd, unet_sd, R):
    from emu_b200.batching import DenoiseSlotScheduler
    pipe, eng = pipeline(sd, unet_sd)
    sched = DenoiseSlotScheduler(pipe, n_slots=3, height=64, width=64, encode_steps=R)
    items = plan(3)
    reqs = run(sched, items)
    assert [r.error for r in reqs] == [None] * len(reqs)
    uncond = pipe.negative_prompt[""]
    for r, (_, k) in zip(reqs, items):
        if "prompt_embeds" in k:
            want = k["prompt_embeds"]
        elif all(not isinstance(x, str) for x in k["inputs"]):
            want = pipe._prepare_and_encode_inputs(k["inputs"], True).to(torch.bfloat16)
        else:
            cond = solo_embeds(pipe, k["inputs"])
            assert torch.equal(r.encoded[0], cond[0]), k["inputs"]
            want = torch.cat([cond, uncond.to(torch.bfloat16)]) if k["guidance_scale"] > 1 else cond
        assert torch.equal(r.encoded, want)
        alone = pipe.denoise(want, 1, 64, 64, k["num_inference_steps"], k["guidance_scale"],
                             k.get("crop_info", (0, 0)), k.get("original_size", (1024, 1024)), latents=k["latents"])
        assert torch.equal(r.result, alone)
    steps = [c[1] for c in eng.calls if c[0] == "regress_step"]
    assert steps and set(steps) == {3}                  # every regression step at B = n_slots
    assert sched.regress_steps == len(steps)
    assert max(sched.join_sizes) == 3                   # the three newcomers of step 0 joined in one call
    assert eng.calls[0] == ("slots_begin", 3) and not any(g >= 0 for g in eng.group)


def test_a_failing_encode_fails_alone_and_frees_its_slots(sd, unet_sd):
    from emu_b200.batching import DenoiseSlotScheduler, ImageRequest
    pipe, eng = pipeline(sd, unet_sd)
    sched = DenoiseSlotScheduler(pipe, n_slots=3, height=64, width=64, encode_steps=2)
    lat = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(3))
    mk = lambda inputs: sched.submit(ImageRequest(inputs=inputs, num_inference_steps=2, height=64, width=64, latents=lat,
                                                  output_type="latent"))
    eng.fail_join_len = len("bad join") + 2             # BOS + characters + [IMG]
    enc = pipe.multimodal_encoder
    vit = enc.encode_image

    def encode(image, n_query=None):                    # the ViT refuses a prompt with two pictures
        if image.shape[0] == 2:
            raise ValueError("cannot encode these pictures")
        return vit(image, n_query)
    enc.encode_image = encode
    a, bad_pic, bad_join = mk(["a cat"]), mk(["look", picture(3), picture(4)]), mk(["bad join"])
    sched.step()
    assert "cannot encode" in str(bad_pic.error) and "join failed" in str(bad_join.error)
    assert a.error is None and a.regressing
    assert sched.owner.count(None) == 2                 # both failed requests gave their latent slots back
    assert [g >= 0 for g in eng.group] == [True, False, False]
    b = mk(["a dog"])
    sched.run_until_idle()
    assert a.error is None and b.error is None and not sched.busy()
    assert b.slot == 1 and not any(g >= 0 for g in eng.group)
    cond = solo_embeds(pipe, ["a dog"])
    assert torch.equal(b.encoded[0], cond[0])


def test_a_failing_regression_step_fails_the_prompts_in_it(sd, unet_sd):
    from emu_b200.batching import DenoiseSlotScheduler, ImageRequest
    pipe, eng = pipeline(sd, unet_sd)
    sched = DenoiseSlotScheduler(pipe, n_slots=2, height=64, width=64, encode_steps=1)
    real = eng.regress_step

    def fail_once(B, out):
        eng.regress_step = real
        raise RuntimeError("engine failure")
    eng.regress_step = fail_once
    r = sched.submit(ImageRequest(inputs=["a cat"], num_inference_steps=2, height=64, width=64, output_type="latent"))
    sched.step()
    assert "engine failure" in str(r.error) and not sched.busy() and not any(g >= 0 for g in eng.group)
    again = sched.submit(ImageRequest(inputs=["a cat"], num_inference_steps=2, height=64, width=64, output_type="latent"))
    sched.run_until_idle()
    assert again.error is None


def test_without_encode_steps_the_llm_never_enters_slot_mode(sd, unet_sd):
    from emu_b200.batching import DenoiseSlotScheduler, ImageRequest
    pipe, eng = pipeline(sd, unet_sd)
    sched = DenoiseSlotScheduler(pipe, n_slots=2, height=64, width=64)
    reqs = [sched.submit(ImageRequest(inputs=[t], num_inference_steps=2, height=64, width=64, output_type="latent"))
            for t in ("a cat", "a dog")]
    sched.run_until_idle()
    assert all(r.error is None for r in reqs) and eng.n_slots == 0 and eng.calls == []
    assert sched.regress_steps == 0 and not sched.join_sizes


def test_a_prompt_that_overflows_llm_max_seq_is_refused_at_submit(sd, unet_sd):
    from emu_b200.batching import DenoiseSlotScheduler, ImageRequest
    pipe, _ = pipeline(sd, unet_sd, max_seq=16)
    sched = DenoiseSlotScheduler(pipe, n_slots=2, height=64, width=64, encode_steps=4)
    fits = "x" * (16 - 2 - (NQ - 1))                    # BOS + text + [IMG], then NQ - 1 regressed positions
    sched.submit(ImageRequest(inputs=[fits], num_inference_steps=1, height=64, width=64, output_type="latent"))
    with pytest.raises(ValueError, match="llm_max_seq"):
        sched.submit(ImageRequest(inputs=[fits + "x"], num_inference_steps=1, height=64, width=64))
    sched.run_until_idle()
    with pytest.raises(ValueError, match="encode_steps must be >= 1"):
        DenoiseSlotScheduler(pipeline(sd, unet_sd)[0], n_slots=2, height=64, width=64, encode_steps=0)
    with pytest.raises(ValueError, match="llm_max_batch"):
        DenoiseSlotScheduler(pipeline(sd, unet_sd)[0], n_slots=9, height=64, width=64, encode_steps=2)


def test_generate_encode_steps_needs_continuous_generation(sd, unet_sd):
    from emu_b200 import serve
    pipe, _ = pipeline(sd, unet_sd)
    with pytest.raises(ValueError, match="continuous"):
        serve.EmuServer(generate=pipe, host="127.0.0.1", port=0, generate_encode_steps=8)
    with pytest.raises(ValueError, match=">= 1"):
        serve.EmuServer(generate=pipe, host="127.0.0.1", port=0, generate_scheduler="continuous", generate_encode_steps=0)
    with pytest.raises(SystemExit):
        serve.main(["--generate-encode-steps", "8", "--disable-chat"])


# ---- the C entry points ----
HEADER = os.path.join(ROOT, "include", "emu_b200_regress.h")


@pytest.fixture(scope="module")
def lib():
    from emu_b200 import build, _lib
    build.build()
    return _lib.load()


def test_regress_header_symbols_are_bound_exported_and_disjoint(lib):
    from emu_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    syms = sorted(set(re.findall(r"\b(emu_[a-z0-9_]+)\s*\(", src)))
    assert sorted(_lib.REGRESS_SYMBOLS) == syms
    assert all(hasattr(lib, s) for s in syms)
    others = set(_lib.SYMBOLS + _lib.SAFETY_SYMBOLS + _lib.SLOT_SYMBOLS + _lib.OPS_SYMBOLS + _lib.PREFIX_SYMBOLS +
                 _lib.CHUNKED_SYMBOLS + _lib.GEN_SLOT_SYMBOLS + _lib.DIFFUSION_OPS_SYMBOLS)
    assert not others & set(syms)


P = ctypes.c_void_p(0x10000000)


def _i32(*v):
    return (ctypes.c_int32 * len(v))(*v)


def _good_args():
    N = None
    return {
        #                        e  slots     new       n  embeds out L  stream
        "emu_llm_regress_join": [P, _i32(0, 1), _i32(5, 7), 2, P, P, 64, N],
        #                        e  B  out L  stream
        "emu_llm_regress_step": [P, 4, P, 64, N],
    }


BAD = [
    ("emu_llm_regress_join", 0, None, "engine"), ("emu_llm_regress_join", 1, None, "slots"),
    ("emu_llm_regress_join", 2, None, "new"), ("emu_llm_regress_join", 4, None, "embeds"),
    ("emu_llm_regress_join", 5, None, "out"), ("emu_llm_regress_join", 3, 0, "n = 0"),
    ("emu_llm_regress_join", 3, 33, "n = 33"), ("emu_llm_regress_join", 6, 0, "L = 0"),
    ("emu_llm_regress_join", 6, -1, "L < 0"), ("emu_llm_regress_join", 1, _i32(0, -1), "slot -1"),
    ("emu_llm_regress_join", 1, _i32(32, 1), "slot 32"), ("emu_llm_regress_join", 2, _i32(5, 0), "no tokens"),
    ("emu_llm_regress_step", 0, None, "engine"), ("emu_llm_regress_step", 2, None, "out"),
    ("emu_llm_regress_step", 1, 0, "B = 0"), ("emu_llm_regress_step", 1, 33, "B = 33"),
    ("emu_llm_regress_step", 3, 0, "L = 0"),
]


def test_every_entry_point_is_exercised_by_the_refusals():
    assert {b[0] for b in BAD} == set(_good_args())


@pytest.mark.parametrize("name,i,bad,what", BAD, ids=["%s: %s" % (b[0], b[3]) for b in BAD])
def test_bad_arguments_are_refused_before_any_cuda_call(lib, name, i, bad, what):
    """NULL pointers, slot counts outside 1..32, slots outside 0..31, prompts without tokens, L <= 0 and B outside 1..32 are
    EMU_ERR_INVALID.  The engine pointer is fake, so a missed check would crash or come back as another error; with a GPU the
    call could reach fake addresses, so the test runs only where there is none.  The checks that need engine state (a slot
    beyond n_slots or occupied, B below the highest live slot, a live slot that is not a regression slot) are on the GPU, in
    tests/test_regress_slots_gpu.py."""
    if torch.cuda.is_available():
        pytest.skip("fake device addresses: checked on a machine without a GPU")
    args = _good_args()[name]
    args[i] = bad
    fn = getattr(lib, name)
    fn.restype, fn.argtypes = ctypes.c_int, None
    assert fn(*args) == -1, (name, what)
