"""Generates tests/golden/live_reference.pt — what the UNMODIFIED reference (imported through oracle/ref_shim.py) returns
for the inputs of the tests that used to import it live:
  * Emu2 `EmuModel.encode_image` / `generate_image` of the tiny model (tests/helpers.py weights) and the tokenizer ids
    `generate_image` asked for at every iteration,
  * the Emu1 Causal-Former at the real t5-base dimensions and the Emu1 EVA ViT (head width 88), both with seeded weights
    that the tests regenerate (oracle.diffusion_oracle.random_state_dict; the weights are NOT stored),
  * Emu2 chat prompt assembly and Emu1 `utils.process_img` / `get_index`: strings and index arrays as they are, image
    tensors as SHA-256 digests of their bytes (bit-identical is the claim; the tensors themselves would be megabytes).

Run where the reference tree is available (EMU_REFERENCE_ROOT):  python tests/golden/gen_golden_live.py
"""
import hashlib
import importlib.util
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import diffusion_oracle as D, ref_shim, t5_oracle as T  # noqa: E402

T5_SEED, VIT_SEED = 21, 22


def digest(t):
    return None if t is None else hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def chat_inputs():
    """the inputs of the chat prompt-assembly test (tests/test_host_cpu.py)"""
    from PIL import Image
    from emu_b200.emu2.constants import DEFAULT_VIDEO_TOKEN, FAKE_VIDEO_END_TOKEN
    imgs = [Image.new("RGB", (64 + 10 * i, 48 + 7 * i), (10 * i, 200 - 20 * i, 30 + i)) for i in range(4)]
    plain = [
        [imgs[0], "describe"],
        ["before", imgs[1], "between", imgs[2], "after"],
        ["watch:", DEFAULT_VIDEO_TOKEN, imgs[0], imgs[1], FAKE_VIDEO_END_TOKEN, "what happens?", imgs[3]],
        ["text only"],
    ]
    chats = [
        ([[imgs[0], "what is this?"], ["a cat"], ["and this?", imgs[1]]], True),
        ([["hello"]], False),
        ([[imgs[2], imgs[3], "compare"], ["they differ"], ["how?"]], False),
    ]
    return plain, chats


def picture(seed, size):
    import numpy as np
    from PIL import Image
    rng = np.random.RandomState(seed)
    return Image.fromarray(rng.randint(0, 256, (size[1], size[0], 3), dtype=np.uint8))


PICTURES = ((1, (640, 480)), (2, (100, 333)), (3, (224, 224)))
FRAMES = ((300, 8), (9, 8), (17, 4), (1000, 8))


def main():
    from helpers import EMU1_VIS88, TINY_LLAMA, TINY_VISION, make_emu2_state_dict
    out = {}

    # ---- Emu2 encode_image / generate_image ----
    L, NH = TINY_LLAMA["num_hidden_layers"], TINY_LLAMA["num_attention_heads"]
    d = ref_shim.make_llama_config_dir(TINY_LLAMA["hidden_size"], L, NH, TINY_LLAMA["intermediate_size"])
    model = ref_shim.build_emu2_model(dict(TINY_VISION), d)
    model.load_state_dict(make_emu2_state_dict(), strict=True)
    img = torch.randn(1, 3, 56, 56, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        enc = model.encode_image(img)
        gi = model.generate_image(text=["two dogs"])
    tok = model.decoder.tokenizer
    ids = {}
    for k in range(5):
        i = tok(["two dogs[IMG]" + "<image>" * k], padding="longest", return_tensors="pt")
        ids[k] = (i.input_ids.clone(), i.attention_mask.clone())
    out["emu2"] = {"encode_image": enc.clone(), "generate_image": gi.clone(), "ids": ids}

    # ---- Emu1 Causal-Former at t5-base dimensions ----
    CF = ref_shim.import_emu1_causal_former()
    sd = D.random_state_dict(T.param_shapes(T.T5_BASE, 1408, 512, n_causal=32), seed=T5_SEED)
    for k in sd:
        if k.endswith("Attention.q.weight"):
            sd[k] = sd[k] * 0.125
    x = torch.randn(1, 257, 1408, generator=torch.Generator().manual_seed(T5_SEED + 1))
    t5 = {"seed": T5_SEED}
    for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        m = CF(None, n_causal=32, vision_width=1408, output_dim=512).eval().to(dt)
        missing, unexpected = m.load_state_dict({k[len("cformer."):]: v.to(dt) for k, v in sd.items()}, strict=False)
        assert not unexpected and all("embed_tokens" in k for k in missing), (missing, unexpected)
        with torch.no_grad():
            t5["out_" + name] = m(x.to(dt)).clone()
    out["t5_base"] = t5

    # ---- Emu1 EVA ViT, head width 88 ----
    vit = ref_shim.build_emu1_vit(EMU1_VIS88)
    shapes = {k: tuple(v.shape) for k, v in vit.state_dict().items()}
    vit.load_state_dict(D.random_state_dict(shapes, seed=VIT_SEED), strict=True)
    img = torch.randn(2, 3, 56, 56, generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        feats = vit.forward_features(img)
    out["emu1_vit"] = {"seed": VIT_SEED, "shapes": shapes, "features": feats.clone()}

    # ---- Emu2 chat prompt assembly ----
    ref_shim.import_emu2()
    import emu.chat as rchat
    ref = rchat.EmuChatGeneration.__new__(rchat.EmuChatGeneration)
    ref.transform = rchat.TF.Compose([
        rchat.TF.Resize((448, 448), interpolation=rchat.TF.InterpolationMode.BICUBIC), rchat.TF.ToTensor(),
        rchat.TF.Normalize(mean=rchat.OPENAI_DATASET_MEAN, std=rchat.OPENAI_DATASET_STD)])
    plain, chats = chat_inputs()
    out["chat_plain"] = []
    for inp in plain:
        b = ref._prepare_inputs(inp)
        out["chat_plain"].append({"prompt": b[0], "images": digest(b[1]), "videos": digest(b[2]), "rest": list(b[3:])})
    out["chat_multi"] = []
    for inp, grounding in chats:
        b = ref._prepare_chat_inputs(inp, is_grounding=grounding)
        out["chat_multi"].append({"prompt": b[0], "images": digest(b[1])})

    # ---- Emu1 utils.process_img / get_index ----
    if "decord" not in sys.modules:
        sys.modules["decord"] = types.ModuleType("decord")
        sys.modules["decord"].VideoReader = object  # imported at module level by the reference, unused here
    spec = importlib.util.spec_from_file_location("emu1_ref_utils", os.path.join(ref_shim.REFERENCE_ROOT, "Emu1", "utils.py"))
    ru = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ru)
    out["process_img"] = [digest(ru.process_img(img=picture(s, sz), device=torch.device("cpu"))) for s, sz in PICTURES]
    out["get_index"] = [torch.as_tensor(ru.get_index(f, s)) for f, s in FRAMES]

    path = os.path.join(HERE, "live_reference.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
