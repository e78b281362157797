"""Drop-in for the reference's ``emu.chat.EmuChatGeneration`` (Emu2/emu/chat.py:20-286): image transform, prompt
assembly (plain / chat / grounding) and a call into ``EmuModel.generate`` — the host-side boundary of the
image->text path.  Method names, argument order and defaults follow the reference."""
import os.path as osp
from typing import List, Optional

import torch
from PIL import Image

from .conf import CLIPVisionCfg, TextDecoderCfg
from .constants import (ASSISTANT_TOKEN, DEFAULT_EOS_TOKEN, DEFAULT_IMG_PLACEHOLDER, DEFAULT_VID_PLACEHOLDER,
                        DEFAULT_VIDEO_TOKEN, EVA_IMAGE_SIZE, FAKE_VIDEO_END_TOKEN, GRD_SYMBOL, GROUND_SYSTEM_MESSAGE,
                        OPENAI_DATASET_MEAN, OPENAI_DATASET_STD, SYSTEM_MESSAGE, USER_TOKEN)
from .diffusion import image_transform, image_transform_cuda
from .emu import EmuModel


class EmuChatGeneration:
    def __init__(self, emu_model: EmuModel, eva_size=EVA_IMAGE_SIZE, eva_mean=OPENAI_DATASET_MEAN,
                 eva_std=OPENAI_DATASET_STD, **kwargs):
        self.emu_model = emu_model
        self.eva_size, self.eva_mean, self.eva_std = eva_size, eva_mean, eva_std

    def transform(self, img: Image.Image, device=None):
        """The reference's TF.Compose transform.  With a CUDA `device` the resize / ToTensor / Normalize run in the
        library (emu_preprocess_image, bit-identical output) and only the raw uint8 pixels are copied to the GPU."""
        if device is not None and torch.device(device).type == "cuda":
            return image_transform_cuda(img, self.eva_size, self.eva_mean, self.eva_std, device=device)
        return image_transform(img, self.eva_size, self.eva_mean, self.eva_std)

    # ---- Emu2/emu/chat.py:41-119 ----
    @torch.no_grad()
    def forward(self, inputs, is_grounding: bool = False, num_beams: int = 5, max_new_tokens: int = 10,
                min_len: int = 1, do_sample: bool = False, penalty_alpha: Optional[float] = None,
                top_p: Optional[float] = None, top_k: Optional[int] = None, temperature: Optional[float] = None,
                length_penalty: float = -1, repetition_penalty: float = 1.0, synced_gpus: bool = False,
                skip_special_tokens: bool = True, **kwargs):
        text_prompt, image_prompt, video_prompt, image_placeholder, video_placeholder = self.prepare(inputs, is_grounding)
        output = self.emu_model.generate(
            text=text_prompt, image=image_prompt, video=video_prompt, image_placeholder=image_placeholder,
            video_placeholder=video_placeholder, num_beams=num_beams, max_new_tokens=max_new_tokens, min_len=min_len,
            do_sample=do_sample, penalty_alpha=penalty_alpha, top_p=top_p, top_k=top_k, temperature=temperature,
            length_penalty=length_penalty, repetition_penalty=repetition_penalty, synced_gpus=synced_gpus,
            skip_special_tokens=skip_special_tokens, **kwargs)
        return output[0]

    __call__ = forward

    def prepare(self, inputs, is_grounding: bool = False):
        """one request's `inputs` (a plain list of strings and pictures, or chat turns) -> (prompt texts [1], image
        [n, 3, S, S] | None, video | None, image placeholder, video placeholder): what `forward` hands to
        EmuModel.generate, also used by the continuous-batching scheduler (emu_b200/batching.py)"""
        assert isinstance(inputs, list), "inputs must be a list"
        device, dtype = self.emu_model.device(), self.emu_model.dtype()
        if isinstance(inputs[0], list):
            assert len(inputs) % 2 == 1, "last message must be user input"
            return self._prepare_chat_inputs(inputs, is_grounding, device, dtype)
        assert all(isinstance(i, (str, Image.Image)) for i in inputs), "input can't be list of list for normal generation"
        return self._prepare_inputs(inputs, device, dtype)

    @torch.no_grad()
    def forward_batch(self, batch_inputs, is_grounding: bool = False, num_beams: int = 5, max_new_tokens: int = 10,
                      min_len: int = 1, do_sample: bool = False, penalty_alpha: Optional[float] = None,
                      top_p: Optional[float] = None, top_k: Optional[int] = None, temperature: Optional[float] = None,
                      length_penalty: float = -1, repetition_penalty: float = 1.0, skip_special_tokens: bool = True,
                      **kwargs):
        """`forward` for several independent requests with the same decoding knobs in ONE generate call (the serving shell's
        batch, emu_b200/serve.py): the prompts are left-padded to the longest (EmuModel.generate does that for a list of
        texts, Emu2/emu/emu.py:189), the pictures of all requests are concatenated in request order — which is the order in
        which the spliced <image> slots are filled (emu.py:199-203).  Returns one string per request."""
        assert isinstance(batch_inputs, list) and batch_inputs, "batch_inputs must be a non-empty list of `inputs` lists"
        device, dtype = self.emu_model.device(), self.emu_model.dtype()
        texts, images, videos = [], [], []
        for inputs in batch_inputs:
            assert isinstance(inputs, list), "inputs must be a list"
            if isinstance(inputs[0], list):
                assert len(inputs) % 2 == 1, "last message must be user input"
                text, image, video, iph, vph = self._prepare_chat_inputs(inputs, is_grounding, device, dtype)
            else:
                text, image, video, iph, vph = self._prepare_inputs(inputs, device, dtype)
            texts += text
            if image is not None:
                images.append(image)
            if video is not None:
                videos.append(video)
        return self.emu_model.generate(
            text=texts, image=torch.cat(images) if images else None, video=torch.cat(videos) if videos else None,
            image_placeholder=iph, video_placeholder=vph, num_beams=num_beams, max_new_tokens=max_new_tokens,
            min_len=min_len, do_sample=do_sample, penalty_alpha=penalty_alpha, top_p=top_p, top_k=top_k,
            temperature=temperature, length_penalty=length_penalty, repetition_penalty=repetition_penalty,
            skip_special_tokens=skip_special_tokens, **kwargs)

    def max_requests_per_batch(self, num_beams: int = 5) -> int:
        """how many requests one generate call can hold: every request takes num_beams KV-cache rows"""
        rows = int(self.emu_model.engine.cfg.llm_max_batch)
        return max(1, rows // max(1, int(num_beams)))

    # ---- prompt assembly (behaviour of Emu2/emu/chat.py:121-195, pinned by tests/test_host_cpu.py against the live
    #      reference).  A message is a flat list of strings and PIL images; "[VIDEO]" ... "[/VIDEO]" brackets frames. ----
    @staticmethod
    def _segments(items):
        """Yield ("text", str) | ("image", img) | ("video", img).  The closing video marker is consumed silently, the
        opening one is kept as text (that is what the tokenizer expects)."""
        in_video = False
        for it in items:
            if isinstance(it, str):
                if it == FAKE_VIDEO_END_TOKEN:
                    in_video = False
                    continue
                in_video = in_video or it == DEFAULT_VIDEO_TOKEN
                yield "text", it
            else:
                yield ("video" if in_video else "image"), it

    def _stack(self, pictures, device, dtype):
        if not pictures:
            return None
        return torch.stack([self.transform(p, device) for p in pictures]).to(device=device, dtype=dtype)

    def _prepare_inputs(self, inputs, device=torch.device("cpu"), dtype=torch.float32,
                        image_placeholder: str = DEFAULT_IMG_PLACEHOLDER, video_placeholder: str = DEFAULT_VID_PLACEHOLDER):
        pieces, pictures = [], {"image": [], "video": []}
        slot = {"image": image_placeholder, "video": video_placeholder}
        for kind, value in self._segments(inputs):
            if kind == "text":
                pieces.append(value)
            else:
                pieces.append(slot[kind])
                pictures[kind].append(value)
        return (["".join(pieces)], self._stack(pictures["image"], device, dtype),
                self._stack(pictures["video"], device, dtype), image_placeholder, video_placeholder)

    def _prepare_chat_inputs(self, inputs, is_grounding: bool = False, device=torch.device("cpu"), dtype=torch.float32,
                             image_placeholder: str = DEFAULT_IMG_PLACEHOLDER,
                             video_placeholder: str = DEFAULT_VID_PLACEHOLDER):
        """Turns alternate USER / ASSISTANT starting with USER; an assistant turn is closed with </s> before the next
        user turn; the prompt ends with an open assistant turn (plus <grounding> when asked for)."""
        parts = [GROUND_SYSTEM_MESSAGE if is_grounding else SYSTEM_MESSAGE]
        images, videos = [], []
        for turn, msg in enumerate(inputs):
            if turn % 2 == 1:
                parts.append(" %s: " % ASSISTANT_TOKEN)
            else:
                parts.append((" " if turn == 0 else DEFAULT_EOS_TOKEN) + "%s: " % USER_TOKEN)
            text, image, video, _, _ = self._prepare_inputs(msg, device, dtype, image_placeholder, video_placeholder)
            parts.append(text[0])
            if image is not None:
                images.append(image)
            if video is not None:
                videos.append(video)
        parts.append(" %s:" % ASSISTANT_TOKEN + (GRD_SYMBOL if is_grounding else ""))
        return (["".join(parts)], torch.cat(images) if images else None, torch.cat(videos) if videos else None,
                image_placeholder, video_placeholder)

    # ---- Emu2/emu/chat.py:197-232 ----
    @classmethod
    def from_config(cls, instruct: bool = False, llama_config_path: Optional[str] = None, tokenizer=None, **kwargs):
        vc = CLIPVisionCfg(n_query=256, v_query=64) if instruct else CLIPVisionCfg()  # chat.py:215-232
        tc = TextDecoderCfg(instruct=instruct) if llama_config_path is None else \
            TextDecoderCfg(llama_config_path=llama_config_path, instruct=instruct)
        return cls(emu_model=EmuModel(vc, tc, tokenizer=tokenizer, **kwargs))

    @classmethod
    def from_pretrained(cls, path: str, instruct: bool = False, dtype=torch.bfloat16, use_safetensors: bool = False,
                        **kwargs):
        ins = cls.from_config(instruct=instruct, **kwargs)
        # stream tensor by tensor into the packed / tensor-parallel device buffers (emu_b200/checkpoint.py); the
        # reference materialises the whole 74 GB state dict on the host first (Emu2/emu/chat.py:129-149)
        from .. import checkpoint
        checkpoint.load_into(ins.emu_model.engine, path)
        return ins

    def multito(self, device_list):
        """Layer-wise device placement of the reference (Emu2/emu/mixin.py) is replaced by one process per GPU with
        tensor parallelism (tp_rank / tp_size of EmuModel); within one process this is a no-op."""
        return self

    multicuda = multito
