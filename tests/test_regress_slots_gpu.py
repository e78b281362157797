"""GPU: regression slots (include/emu_b200_regress.h) on the tiny Emu2 model.  A prompt's embeddings are the same bits whatever
joins and leaves around it (joins of 1 and of 3, two pool sizes), they are within the bf16 bound of the fp32 oracle (tiny width
and one LLaMA-33B-width layer), the graphed step equals the eager one, the engine refuses what it cannot do, and
DenoiseSlotScheduler(encode_steps=2) gives every request the image and safety flag the same scheduler gives it alone."""
import math
import os

import numpy as np
import pytest
import torch

from helpers import TINY_LLAMA, TINY_VISION, StubTokenizer, assert_bf16_parity, make_emu2_state_dict
from oracle import emu_oracle as O
from test_gen_batching_gpu import TINY_UNET, TINY_UNET_JSON, TINY_VAE, TextTokenizer

pytestmark = pytest.mark.gpu
NQ, L = TINY_VISION["n_query"], 8


def _tiny_model(max_batch=8, max_seq=128):
    from emu_b200.emu2.conf import CLIPVisionCfg, TextDecoderCfg
    from emu_b200.emu2.emu import EmuModel
    m = EmuModel(CLIPVisionCfg(**TINY_VISION), TextDecoderCfg(), tokenizer=TextTokenizer(), llama_config=TINY_LLAMA,
                 max_batch=max_batch, max_seq=max_seq)
    m.load_state_dict(make_emu2_state_dict())
    return m


@pytest.fixture(scope="module")
def model(cuda):
    m = _tiny_model()
    yield m
    m.engine.close()


def _prompt(m, text):
    ids, _, image_id = m.image_prompt_ids([text])
    return m.image_prompt_embeds(ids, None, image_id)[0]


TEXTS = ["a red cat", "two dogs on a long beach", "x", "a bird in the sky at night", "the sea", "a cup of tea on a table"]


def _join(eng, m, slots, texts, out):
    es = [_prompt(m, t) for t in texts]
    eng.regress_join(slots, [e.shape[0] for e in es], torch.cat(es), out)


def _alone(m, n_slots, slot, text):
    """the prompt regressed alone in `slot` of a pool of n_slots: L embeddings"""
    eng = m.engine
    out = torch.zeros(n_slots, L, TINY_VISION["width"], dtype=torch.bfloat16, device="cuda")
    eng.slots_begin(n_slots)
    _join(eng, m, [slot], [text], out)
    for _ in range(L - 1):
        eng.regress_step(n_slots, out)
    return out[slot].clone()


def _busy(m, n_slots, target_slot, join_of_three):
    """the target prompt in target_slot while other prompts join (1 or 3 at a time) and leave around it"""
    eng = m.engine
    out = torch.zeros(n_slots, L, TINY_VISION["width"], dtype=torch.bfloat16, device="cuda")
    eng.slots_begin(n_slots)
    others = [s for s in range(n_slots) if s != target_slot]
    if join_of_three:                        # the target joins with two others in ONE join, then the neighbours churn
        _join(eng, m, [others[0], target_slot, others[1]], [TEXTS[1], TEXTS[0], TEXTS[2]], out)
        eng.regress_step(n_slots, out)
        eng.leave([others[0]])
        eng.regress_step(n_slots, out)
        _join(eng, m, [others[0]], [TEXTS[3]], out)
    else:                                    # the others regress first; the target joins alone, mid-way
        _join(eng, m, others[:2], TEXTS[3:5], out)
        eng.regress_step(n_slots, out)
        eng.regress_step(n_slots, out)
        _join(eng, m, [target_slot], [TEXTS[0]], out)
        eng.regress_step(n_slots, out)
        eng.leave([others[1]])
    while int(eng.slot_len(target_slot)) < _prompt(m, TEXTS[0]).shape[0] + L - 1:
        eng.regress_step(n_slots, out)
        live = [s for s in others if eng.slot_len(s) > 0]
        if len(live) < len(others):          # keep the pool churning: a free neighbour joins again
            free = [s for s in others if eng.slot_len(s) == 0][0]
            _join(eng, m, [free], [TEXTS[5]], out)
    got = out[target_slot].clone()
    eng.leave([s for s in range(n_slots) if eng.slot_len(s) > 0])
    return got


@pytest.mark.parametrize("n_slots,target", [(3, 1), (6, 4)])
def test_a_prompt_regresses_to_the_same_bits_whatever_joins_and_leaves(model, n_slots, target):
    alone = _alone(model, n_slots, target, TEXTS[0])
    assert torch.isfinite(alone.float()).all() and alone.float().abs().max() > 0
    for join_of_three in (True, False):
        got = _busy(model, n_slots, target, join_of_three)
        assert torch.equal(got.view(torch.int16), alone.view(torch.int16)), (n_slots, join_of_three)


def test_the_graphed_step_equals_eager(model):
    graphed = _busy(model, 3, 1, True)
    os.environ["EMU_NO_GRAPH"] = "1"
    try:
        eager = _busy(model, 3, 1, True)
    finally:
        del os.environ["EMU_NO_GRAPH"]
    assert torch.equal(graphed.view(torch.int16), eager.view(torch.int16))


def test_embedding_zero_against_generate_image(model):
    """embedding 0 regressed in a pool of 1 against generate_image alone (printed; DESIGN.md records the outcome)"""
    m = model
    ids, mask, image_id = m.image_prompt_ids([TEXTS[1]])
    ref = m.generate_image_from_ids(ids, mask, image_token_id=image_id)[0]
    pool = {}
    for n in (1, 4):
        pool[n] = _alone(m, n, 0, TEXTS[1])[:NQ]
        m.engine.leave([0])
    for n, got in pool.items():
        same0 = torch.equal(got[0].view(torch.int16), ref[0].view(torch.int16))
        same = torch.equal(got.view(torch.int16), ref.view(torch.int16))
        print("\n[regress] pool of %d: embedding 0 %s generate_image bitwise, all %d %s; max |diff| %.3e"
              % (n, "equals" if same0 else "differs from", NQ, "equal" if same else "do not",
                 float((got.float() - ref.float()).abs().max())))


def test_embeddings_are_within_the_bf16_bound_of_the_oracle(model):
    m = model
    sd = make_emu2_state_dict()
    bsd = {k: v.to(torch.bfloat16) for k, v in sd.items()}
    out = torch.zeros(3, L, TINY_VISION["width"], dtype=torch.bfloat16, device="cuda")
    m.engine.slots_begin(3)
    texts = [TEXTS[1], TEXTS[3]]
    _join(m.engine, m, [2, 0], texts, out)
    for _ in range(L - 1):
        m.engine.regress_step(3, out)
    for slot, t in zip([2, 0], texts):
        ids, mask, _ = m.image_prompt_ids([t])
        ids, mask = ids.cpu(), mask.cpu()
        emb32 = torch.nn.functional.embedding(ids, sd["decoder.lm.model.embed_tokens.weight"])
        emb16 = torch.nn.functional.embedding(ids, bsd["decoder.lm.model.embed_tokens.weight"])
        ref32 = O.generate_image_cached(sd, emb32, mask, L, layers=2, heads=2).float()
        ref16 = O.generate_image_cached(bsd, emb16, mask, L, layers=2, heads=2).float()
        assert_bf16_parity("regression slot %d (tiny)" % slot, out[slot:slot + 1].float().cpu(), ref32, ref16)
    m.engine.leave([0, 2])


def test_the_engine_refuses_what_it_cannot_do(model):
    from emu_b200._lib import EmuError
    m, eng = model, model.engine
    out = torch.zeros(4, L, TINY_VISION["width"], dtype=torch.bfloat16, device="cuda")
    e = _prompt(m, TEXTS[0])
    eng.llm_reset()
    with pytest.raises(EmuError, match="not in slot mode"):
        eng.regress_join([0], [e.shape[0]], e, out)
    eng.slots_begin(4)
    with pytest.raises(EmuError, match="no live slot"):
        eng.regress_step(4, out)
    eng.regress_join([2], [e.shape[0]], e, out)
    with pytest.raises(EmuError, match="slot 2 is occupied"):
        eng.regress_join([2], [e.shape[0]], e, out)
    with pytest.raises(EmuError, match="slot 5 out of range"):
        eng.regress_join([5], [e.shape[0]], e, torch.zeros(6, L, TINY_VISION["width"], dtype=torch.bfloat16, device="cuda"))
    with pytest.raises(EmuError, match="highest live slot 2"):
        eng.regress_step(2, out)
    eng.join([0], e[None])                    # a chat slot below B
    with pytest.raises(EmuError, match="slot 0 is live but did not join"):
        eng.regress_step(4, out)
    eng.leave([0])
    eng.regress_step(4, out)
    assert eng.slot_len(2) == e.shape[0] + 1
    eng.leave([2])


# ---- one LLaMA-33B-width layer (6656 / 52 heads x 128 / 17920) under the 1792-wide projections ----
def test_llama33b_width_layer_regression_is_within_the_bf16_bound(cuda):
    from helpers import VOCAB
    from test_realshape_gpu import LLAMA_33B_1L, _llama_sd
    from emu_b200.emu2.conf import CLIPVisionCfg, TextDecoderCfg
    from emu_b200.emu2.emu import EmuModel
    cfg, W = LLAMA_33B_1L, 1792
    sd = _llama_sd(cfg, VOCAB, seed=31)
    g = torch.Generator().manual_seed(32)
    H = cfg["hidden_size"]
    sd["project_up.weight"] = torch.randn(H, W, generator=g) / math.sqrt(W)
    sd["project_down.weight"] = torch.randn(W, H, generator=g) / math.sqrt(H)
    vis = dict(TINY_VISION, layers=1, width=W, head_width=112)
    m = EmuModel(CLIPVisionCfg(**vis), TextDecoderCfg(), tokenizer=StubTokenizer(), llama_config=cfg, max_batch=4, max_seq=64)
    for k, v in sd.items():
        m.engine.load_tensor(k, v)
    Lq, n_slots = 6, 4
    toks = [torch.randint(100, 31000, (1, n), generator=g) for n in (20, 13)]
    out = torch.zeros(n_slots, Lq, W, dtype=torch.bfloat16, device="cuda")
    eng = m.engine
    eng.slots_begin(n_slots)
    es = [eng.llm_embed(t.cuda())[0] for t in toks]
    eng.regress_join([1, 3], [e.shape[0] for e in es], torch.cat(es), out)
    for _ in range(Lq - 1):
        eng.regress_step(n_slots, out)
    bsd = {k: v.to(torch.bfloat16) for k, v in sd.items()}
    with torch.no_grad():
        for slot, t in zip([1, 3], toks):
            mask = torch.ones_like(t)
            ref32 = O.generate_image_cached(sd, torch.nn.functional.embedding(t, sd["decoder.lm.model.embed_tokens.weight"]),
                                            mask, Lq, layers=1, heads=cfg["num_attention_heads"]).float()
            ref16 = O.generate_image_cached(bsd, torch.nn.functional.embedding(t, bsd["decoder.lm.model.embed_tokens.weight"]),
                                            mask, Lq, layers=1, heads=cfg["num_attention_heads"]).float()
            assert_bf16_parity("regression slot %d (33B width)" % slot, out[slot:slot + 1].float().cpu(), ref32, ref16)
    eng.close()


# ---- the scheduler: images and flags equal each request through the same scheduler alone ----
def test_encode_steps_scheduler_images_equal_each_request_alone(cuda):
    from oracle import diffusion_oracle as D
    from oracle import safety_oracle as S
    from test_safety_gpu import TINY as TINY_SAFETY, _checker
    from emu_b200.batching import DenoiseSlotScheduler, ImageRequest
    from emu_b200.emu2.diffusion import EmuVisualGeneration
    from emu_b200.emu2.scheduler import EulerDiscreteScheduler
    m = _tiny_model()
    ck = _checker(TINY_SAFETY, S.random_state_dict(TINY_SAFETY, seed=21))
    pipe = EmuVisualGeneration(m, EulerDiscreteScheduler(), TINY_UNET_JSON, TINY_VAE, safety_checker=ck)
    pipe.load_state_dict({"unet." + k: v for k, v in D.random_state_dict(D.unet_param_shapes(TINY_UNET), seed=3).items()})
    pipe.load_state_dict({"vae." + k: v for k, v in D.random_state_dict(D.vae_decoder_param_shapes(TINY_VAE), seed=5).items()})
    H = W = 128
    g = torch.Generator().manual_seed(9)
    knobs = [dict(inputs=["a cat"], num_inference_steps=3, guidance_scale=3.0),
             dict(inputs=["a red dog on grass"], num_inference_steps=2, guidance_scale=1.0, crop_info=[16, 0]),
             dict(inputs=["a bird"], num_inference_steps=4, guidance_scale=5.0, original_size=[768, 512]),
             dict(inputs=["a tree by a lake"], num_inference_steps=2, guidance_scale=3.0)]
    for k in knobs:
        k["latents"] = torch.randn(1, 4, 32, 32, generator=g).cuda()
    sched = DenoiseSlotScheduler(pipe, n_slots=3, height=H, width=W, encode_steps=2)
    reqs = [sched.submit(ImageRequest(**knobs[0])), sched.submit(ImageRequest(**knobs[1]))]
    sched.step()
    reqs.append(sched.submit(ImageRequest(**knobs[2])))
    sched.step()
    sched.step()
    reqs.append(sched.submit(ImageRequest(**knobs[3])))
    sched.run_until_idle()
    assert [r.error for r in reqs] == [None] * 4
    assert max(sched.join_sizes) == 2 and max(sched.batch_sizes) >= 2 and sched.regress_steps > 0
    for r, k in zip(reqs, knobs):
        alone = sched.submit(ImageRequest(**k))
        sched.run_until_idle()
        assert alone.error is None and alone.slot == 0
        assert np.array_equal(np.asarray(r.result.image), np.asarray(alone.result.image))
        assert r.result.nsfw_content_detected == alone.result.nsfw_content_detected is not None
    m.engine.close()
