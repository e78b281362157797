"""The Emu1 example entry point on the H100 engine — what `python inference.py [--instruct] --ckpt-path ...` is in the reference
(Emu1/inference.py; BASELINE configs[0] is its captioning call on CPU).  Same command line, same helper names
(`prepare_model`, `Emu_inference`, `Emu_instruct_caption`, `pretrain_example`, `instruct_example`), same prompts and example files;
the model behind them is `emu_b200.emu1.modeling_emu.Emu` and the checkpoint — DeepSpeed `module` wrapper and the `--instruct`
LoRA adapters included — is streamed into the engine by emu_b200/checkpoint.py (adapters are folded into the base weights at
load, so there is no peft wrapper at run time).

Run from a directory that holds `models/Emu-14B.json`, `models/llama_config/` and `examples/` (the reference's own layout)."""
import argparse
import json

import torch

from .modeling_emu import Emu
from .utils import process_img, process_video

image_placeholder = "[IMG]" + "<image>" * 32 + "[/IMG]"
image_system_msg = ("You will be presented with an image: [IMG]ImageContent[/IMG]. You will be able to see the image after I "
                    "provide it to you. Please answer my questions based on the given image.")
video_system_msg = ("You are a helpful assistant and you will be presented with a video consisting of multiple chronological "
                    "images: [IMG]ImageContent[/IMG]. You will be able to see the video after I provide it to you. Please answer "
                    "my questions based on the given video.")
CAPTION_REQUEST = "Please provide an accurate and concise description of the given image."
CAPTION_LEAD_IN = "The image depicts a photo of"

emu_model = None          # set by main(); the helpers below use it like the reference's module-level global
args = None


def parse_args(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--instruct", action="store_true", default=False, help="Load Emu-I")
    p.add_argument("--ckpt-path", type=str, default="", help="Emu ckpt path")
    return p.parse_args(argv)


def prepare_model(model_name, args, **engine_kwargs):
    """inference.py:33-61: read models/<name>.json, build the model, load the checkpoint (non-strict, like the reference)."""
    with open("models/%s.json" % model_name, "r", encoding="utf8") as f:
        model_cfg = json.load(f)
    print("=====> model_cfg: %s" % model_cfg)
    model = Emu(**model_cfg, cast_dtype=torch.float, args=args, **engine_kwargs)
    print("=====> loading from ckpt_path %s" % args.ckpt_path)
    from .. import checkpoint
    # --instruct: the LoRA adapters (r = 16, alpha = 16 on q/k/v/o, inference.py:40-50) are merged while streaming
    checkpoint.load_into(model.engine, args.ckpt_path, lora=bool(args.instruct), rename=lambda k: None if k.startswith(
        ("visual.norm.", "visual.fc_norm.", "visual.head.", "visual.rope.")) else k)
    return model.eval()


def interleave(items):
    """[tensor | str, ...] -> (list of image tensors, the text with an image placeholder where every image stood)"""
    images = [x for x in items if not isinstance(x, str)]
    return images, "".join(x if isinstance(x, str) else image_placeholder for x in items)


def Emu_inference(image_list, text_sequence, system="", instruct=True, max_new_tokens=128, beam_size=5, length_penalty=0.0):
    prompt = ("%s [USER]: %s [ASSISTANT]:" % (system, text_sequence)).strip() if instruct else text_sequence
    print("===> prompt: %s" % prompt)
    samples = {"image": torch.cat(image_list, dim=0), "prompt": prompt}
    output_text = emu_model.generate(samples, max_new_tokens=max_new_tokens, num_beams=beam_size,
                                     length_penalty=length_penalty, repetition_penalty=1.0)[0].strip()
    print("===> output: %s\n" % output_text)
    return output_text


def Emu_instruct_caption(img):
    prompt = ("%s [USER]: %s%s [ASSISTANT]: %s" % (image_system_msg, image_placeholder, CAPTION_REQUEST, CAPTION_LEAD_IN)).strip()
    print("===> caption prompt: %s" % prompt)
    output_text = emu_model.generate({"image": img, "prompt": prompt}, max_new_tokens=512, num_beams=5, length_penalty=0.0,
                                     repetition_penalty=1.0)[0].strip()
    print("===> caption output: %s\n" % output_text)
    return output_text


def _img(path):
    return process_img(img_path=path, device=args.device)


def pretrain_example():
    """in-context learning with the pretrained model: two captioned pictures, then a third to caption"""
    images, text = interleave([_img("examples/dog.png"), "There are two dogs.", _img("examples/panda.png"),
                               "There are three pandas.", _img("examples/sunflower.png")])
    Emu_inference(images, text, instruct=False)


def instruct_example():
    """captioning, VQA, interleaved image-text input and video understanding with the instruction-tuned model"""
    image = _img("examples/iron_man.jpg")
    Emu_instruct_caption(image)
    Emu_inference([image], image_placeholder + "what is the man doing?", system=image_system_msg)
    books = []
    for n, name in enumerate(("first", "second", "third", "fourth"), start=1):
        books += [_img("examples/book%d.jpeg" % n), "This is the %s image." % name]
    Emu_inference(*interleave(books + ["Describe all images."]), system="")
    frames, text = process_video("examples/AppleVR.mp4", image_placeholder=image_placeholder, device=args.device)
    Emu_inference(frames, text + "What's the woman doing in the video?", system=video_system_msg, length_penalty=1.0)


def main(argv=None):
    global emu_model, args
    args = parse_args(argv)
    args.device = torch.device("cuda")            # the engine has no CPU path (the reference falls back to the CPU here)
    emu_model = prepare_model("Emu-14B", args)
    (instruct_example if args.instruct else pretrain_example)()


if __name__ == "__main__":
    main()
