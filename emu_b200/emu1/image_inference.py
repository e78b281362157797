"""The Emu1 image-generation example on the H100 engine (Emu1/image_inference.py): image blending, text-to-image and in-context
generation through `EmuGenerationPipeline`, 512 x 512, the reference's guidance scales and output file names."""
import argparse

from PIL import Image

from .pipeline import EmuGenerationPipeline

CASES = [
    # (inputs: str = text, ("img", path) = picture; guidance_scale; output file; label used in the safety message)
    ([("img", "examples/cat.jpg"), ("img", "examples/tiger.jpg")], 7.5, "image_blend_result.jpg", "ImageBlend"),
    (["An image of a dog wearing a pair of glasses."], 7.5, "text2image_result.jpg", "T2I"),
    (["This is the first image: ", ("img", "examples/dog.png"), "This is the second image: ", ("img", "examples/sunflower.png"),
      "The animal in the first image surrounded with the plant in the second image: "], 10.0, "incontext_result.jpg", "In-context"),
]


def parse_args(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--instruct", action="store_true", default=False, help="Load Emu-I")
    p.add_argument("--ckpt-path", type=str, default="", help="Emu Decoder ckpt path")
    return p.parse_args(argv)


def run_case(pipeline, inputs, guidance_scale, out_path, label):
    items = [Image.open(x[1]) if isinstance(x, tuple) else x for x in inputs]
    image, safety = pipeline(items, height=512, width=512, guidance_scale=guidance_scale)
    if safety is None or not safety:
        image.save(out_path)
    else:
        print("%s Generated Image Has Safety Concern!!!" % label)
    return image, safety


def main(argv=None):
    args = parse_args(argv)
    # the decoder pipeline was trained against the pretrained encoder only (image_inference.py:32-35)
    assert args.instruct is False, "Image Generation currently do not support instruct tuning model"
    pipeline = EmuGenerationPipeline.from_pretrained(path=args.ckpt_path, args=args)
    for case in CASES:
        run_case(pipeline, *case)


if __name__ == "__main__":
    main()
