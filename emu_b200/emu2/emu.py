"""Drop-in for the reference's ``emu.emu.EmuModel`` (Emu2/emu/emu.py:19-235) on the H100 engine.

Same constructor signature (vision_cfg, text_decoder_cfg), same public methods and argument meaning:
``encode_image``, ``generate``, ``generate_image``; weights enter through ``load_state_dict`` with the reference's
key names.  All arithmetic runs in libemu_b200.so (ViT, LLaMA prefill/decode, projections); this file only does
what the reference does on the host: placeholder replacement, tokenisation, index logic and detokenisation.
"""
from typing import List, Optional

import torch

from .. import _lib, generation
from .conf import CLIPVisionCfg, TextDecoderCfg, load_llama_config
from .constants import (DEFAULT_gIMG_TOKEN, DEFAULT_IMAGE_TOKEN, DEFAULT_IMG_END_TOKEN, DEFAULT_IMG_PLACEHOLDER,
                        DEFAULT_IMG_TOKEN, DEFAULT_PAD_TOKEN, DEFAULT_BOS_TOKEN, DEFAULT_EOS_TOKEN,
                        DEFAULT_VID_PLACEHOLDER, special_token_list)


def build_tokenizer(llama_config_path, instruct=False):
    """LlamaTokenizer + the Emu special tokens, exactly as Emu2/emu/lm.py:41-66 builds it."""
    import transformers
    tok = transformers.LlamaTokenizer.from_pretrained(llama_config_path)
    tok.add_special_tokens(dict(pad_token=DEFAULT_PAD_TOKEN, bos_token=DEFAULT_BOS_TOKEN, eos_token=DEFAULT_EOS_TOKEN,
                                additional_special_tokens=special_token_list(instruct)))
    return tok


def dp_image_slices(n_images: int, world: int):
    """Contiguous per-rank slices of a batch of images for the data-parallel ViT (SURVEY.md §8e: "EVA ViT — data-parallel over
    images, all-gather once"): rank r encodes images [lo_r, hi_r); every rank gets ceil(n / world) or fewer, in order."""
    per = (n_images + world - 1) // world
    return [(min(r * per, n_images), min((r + 1) * per, n_images)) for r in range(world)]


def encode_images_data_parallel(encode_local, image: torch.Tensor, rank: int, world: int, group=None):
    """Each tensor-parallel rank runs the (replicated) ViT on its slice of the image batch only; one all-gather of the pooled
    tokens puts the full [B, n_query, width] result on every rank, in the original order.  Bitwise identical to encoding the
    whole batch on one GPU (every image is independent of its batch neighbours in every kernel)."""
    import torch.distributed as dist
    B = image.shape[0]
    slices = dp_image_slices(B, world)
    per = slices[0][1] - slices[0][0]
    lo, hi = slices[rank]
    local = encode_local(image[lo:hi]) if hi > lo else None
    probe = local if local is not None else encode_local(image[:1])  # shape / dtype of one result row (rank without work)
    buf = torch.zeros(per, *probe.shape[1:], dtype=probe.dtype, device=probe.device)
    if local is not None:
        buf[: hi - lo] = local
    parts = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(parts, buf, group=group)
    return torch.cat([parts[r][: slices[r][1] - slices[r][0]] for r in range(world)], dim=0)


class _Decoder:
    """Mirror of the attribute surface callers touch on ``model.decoder`` (tokenizer, config, special ids)."""

    def __init__(self, tokenizer, llama_cfg, vocab):
        self.tokenizer = tokenizer
        self.config = llama_cfg
        self.vocab_size = vocab


class EmuModel:
    def __init__(self, vision_cfg: CLIPVisionCfg = None, text_decoder_cfg: TextDecoderCfg = None, *, tokenizer=None,
                 llama_config=None, max_batch: int = 8, max_seq: Optional[int] = None, tp_rank: int = 0,
                 tp_size: int = 1, nccl_uid: bytes = None, device="cuda"):
        vision_cfg = vision_cfg or CLIPVisionCfg()
        text_decoder_cfg = text_decoder_cfg or TextDecoderCfg()
        self.vision_cfg, self.text_decoder_cfg = vision_cfg, text_decoder_cfg
        lc = load_llama_config(llama_config if llama_config is not None else text_decoder_cfg.llama_config_path)
        self.llama_cfg = lc
        if tokenizer is None:
            tokenizer = build_tokenizer(text_decoder_cfg.llama_config_path, text_decoder_cfg.instruct)
        tokenizer.truncation_side = tokenizer.padding_side = "left"  # Emu2/emu/emu.py:58
        vocab = len(tokenizer)
        self.decoder = _Decoder(tokenizer, lc, vocab)
        self.device_ = torch.device(device)

        c = _lib.EmuConfig()
        c.llm_hidden, c.llm_layers = lc["hidden_size"], lc["num_hidden_layers"]
        c.llm_heads = lc["num_attention_heads"]
        c.llm_head_dim = lc["hidden_size"] // lc["num_attention_heads"]
        c.llm_ffn, c.llm_vocab = lc["intermediate_size"], vocab
        c.llm_rms_eps, c.llm_rope_theta = lc["rms_norm_eps"], lc["rope_theta"]
        c.llm_max_batch = max_batch
        c.llm_max_seq = max_seq or lc.get("max_position_embeddings", 2048)
        c.vit_image, c.vit_patch, c.vit_width = vision_cfg.image_size, vision_cfg.patch_size, vision_cfg.width
        c.vit_layers = vision_cfg.layers
        c.vit_heads = vision_cfg.width // vision_cfg.head_width
        c.vit_mlp = int(vision_cfg.width * vision_cfg.mlp_ratio)  # Emu2/emu/eva_vit.py:270
        c.vit_ln_eps = 1e-6                                       # Emu2/emu/emu.py:37
        c.vit_postnorm = 1 if vision_cfg.postnorm else 0
        c.vit_final_ln = 0
        c.vit_max_batch = 8
        if vision_cfg.rope or vision_cfg.naiveswiglu or vision_cfg.subln or vision_cfg.init_value:
            raise NotImplementedError("EVA variants with rope / swiglu / subln / layer-scale are not used by Emu2")
        self.engine = _lib.Engine(c, tp_rank=tp_rank, tp_size=tp_size, nccl_uid=nccl_uid)
        self.tp_rank, self.tp_size = tp_rank, tp_size
        self.hidden = c.llm_hidden

        self.n_query = vision_cfg.n_query
        self.v_query = vision_cfg.v_query
        self.image_placeholder = DEFAULT_IMG_TOKEN + DEFAULT_IMAGE_TOKEN * self.n_query + DEFAULT_IMG_END_TOKEN
        self.video_placeholder = DEFAULT_IMG_TOKEN + DEFAULT_gIMG_TOKEN * self.v_query + DEFAULT_IMG_END_TOKEN

    # ---- nn.Module-compatible plumbing ----
    def load_state_dict(self, state_dict, strict: bool = True):
        self.engine.load_state_dict(state_dict)
        return self

    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    def device(self, module=None):
        return self.device_

    def dtype(self, module=None):
        return torch.bfloat16

    # ---- Emu2/emu/emu.py:77-90 ----
    @torch.no_grad()
    def encode_image(self, image: torch.Tensor, *, n_query=None):
        n_query = n_query if n_query is not None else self.n_query
        image = image.to(self.device_)
        local = lambda x: self.engine.vit_forward(x, n_query, pool=True)
        if self.tp_size > 1 and image.shape[0] > 1 and self._dist_matches_tp():
            # several images under tensor parallelism (8-shot prompts, video frames): the ViT is replicated, so split the
            # IMAGES over the ranks instead of running all of them everywhere
            return encode_images_data_parallel(local, image, self.tp_rank, self.tp_size)
        return local(image)

    def _dist_matches_tp(self):
        import torch.distributed as dist
        return dist.is_available() and dist.is_initialized() and dist.get_world_size() == self.tp_size \
            and dist.get_rank() == self.tp_rank

    def _tokenize(self, text):
        inputs = self.decoder.tokenizer(text, padding="longest", return_tensors="pt")
        return inputs.input_ids.to(self.device_), inputs.attention_mask.to(self.device_)

    def _project_up(self, x):
        return self.engine.project(0, x, self.hidden)

    def _project_down(self, x):
        return self.engine.project(1, x, self.vision_cfg.width)

    # ---- Emu2/emu/emu.py:155-235 ----
    @torch.no_grad()
    def generate(self, text: List[str], image: Optional[torch.Tensor] = None, video: Optional[torch.Tensor] = None,
                 image_placeholder: str = DEFAULT_IMG_PLACEHOLDER, video_placeholder: str = DEFAULT_VID_PLACEHOLDER,
                 num_beams=5, max_new_tokens=10, min_len=1, do_sample=False, penalty_alpha=None, top_p=None,
                 top_k=None, temperature=None, length_penalty=-1, repetition_penalty=1.0, synced_gpus=False,
                 skip_special_tokens=True, **kwargs):
        tok = self.decoder.tokenizer
        IMAGE, VIDEO = tok.convert_tokens_to_ids([DEFAULT_IMAGE_TOKEN, DEFAULT_gIMG_TOKEN])
        text = [t.replace(image_placeholder, self.image_placeholder).replace(video_placeholder, self.video_placeholder)
                for t in text]
        input_ids, attention_mask = self._tokenize(text)
        outputs = self.generate_from_ids(input_ids, attention_mask, image=image, video=video, image_token_id=IMAGE,
                                         video_token_id=VIDEO, num_beams=num_beams, max_new_tokens=max_new_tokens,
                                         min_len=min_len, do_sample=do_sample, penalty_alpha=penalty_alpha, top_p=top_p,
                                         top_k=top_k, temperature=temperature, length_penalty=length_penalty,
                                         repetition_penalty=repetition_penalty, **kwargs)
        return tok.batch_decode(outputs, skip_special_tokens=skip_special_tokens)

    @torch.no_grad()
    def generate_from_ids(self, input_ids, attention_mask, image=None, video=None, image_token_id=32003,
                          video_token_id=32004, num_beams=5, max_new_tokens=10, min_len=1, do_sample=False,
                          penalty_alpha=None, top_p=None, top_k=None, temperature=None, length_penalty=-1,
                          repetition_penalty=1.0, eos_token_id=None, pad_token_id=None, **kwargs):
        """Token-id level entry (what `generate` does after tokenisation); returns new token ids [B, T]."""
        tok = self.decoder.tokenizer
        eos = eos_token_id if eos_token_id is not None else tok.eos_token_id
        pad = pad_token_id if pad_token_id is not None else tok.pad_token_id
        input_ids = input_ids.to(self.device_)
        attention_mask = attention_mask.to(self.device_)
        text_embeds = self.engine.llm_embed(input_ids)  # [B, N, H]
        if image is not None:
            e = self.encode_image(image, n_query=self.n_query)
            e = self._project_up(e.reshape(-1, e.shape[-1]))
            text_embeds[input_ids == image_token_id] = e
        if video is not None:
            e = self.encode_image(video, n_query=self.v_query)
            e = self._project_up(e.reshape(-1, e.shape[-1]))
            text_embeds[input_ids == video_token_id] = e
        # strategy selection as GenerationMixin does it from these knobs; the extra HF knobs the reference lets through its
        # **kwargs (no_repeat_ngram_size, prefix_allowed_tokens_fn, num_return_sequences, early_stopping) are honoured too
        return generation.generate(self.engine, text_embeds, attention_mask, max_new_tokens, eos, pad, do_sample=do_sample,
                                   num_beams=num_beams, min_length=min_len, length_penalty=length_penalty,
                                   repetition_penalty=repetition_penalty, penalty_alpha=penalty_alpha, top_k=top_k,
                                   top_p=top_p, temperature=temperature,
                                   no_repeat_ngram_size=kwargs.get("no_repeat_ngram_size", 0),
                                   prefix_allowed_tokens_fn=kwargs.get("prefix_allowed_tokens_fn"),
                                   num_return_sequences=kwargs.get("num_return_sequences", 1),
                                   early_stopping=kwargs.get("early_stopping", False), generator=kwargs.get("generator"),
                                   check_every=kwargs.get("check_every"))

    # ---- Emu2/emu/emu.py:92-153 ----
    @torch.no_grad()
    def generate_image(self, text: List[str], image: Optional[torch.Tensor] = None,
                       placeholder: str = DEFAULT_IMG_PLACEHOLDER):
        tok = self.decoder.tokenizer
        IMAGE = tok.convert_tokens_to_ids([DEFAULT_IMAGE_TOKEN])[0]
        text = [t.replace(placeholder, self.image_placeholder) for t in text]
        text = [f"{t}{DEFAULT_IMG_TOKEN}" for t in text]          # iteration 0 of the reference loop (:110-111)
        input_ids, attention_mask = self._tokenize(text)
        return self.generate_image_from_ids(input_ids, attention_mask, image=image, image_token_id=IMAGE)

    @torch.no_grad()
    def generate_image_from_ids(self, input_ids, attention_mask, image=None, image_token_id=32003):
        """The reference re-runs a full, cache-less forward for each of the n_query regressed embeddings
        (emu.py:109-147).  Causal masking makes that identical to one prefill of `text + [IMG]` followed by
        n_query-1 single-position steps fed with project_up(project_down(h_last)) (SURVEY.md §8a' item 2);
        positions are arange including pads (lm.model is called without position_ids, emu.py:133-138)."""
        input_ids = input_ids.to(self.device_)
        attention_mask = attention_mask.to(self.device_)
        B = input_ids.shape[0]
        embeds = self.engine.llm_embed(input_ids)
        if image is not None:
            e = self.encode_image(image)
            e = self._project_up(e.reshape(-1, e.shape[-1]))
            embeds[input_ids == image_token_id] = e  # every <image> in the prompt is a prompt slot at iteration 0
        self.engine.llm_reset()
        hidden, _ = self.engine.llm_prefill(embeds, attention_mask, hf_positions=False, want_hidden=True,
                                            want_logits=False)
        last = hidden[:, -1, :].contiguous()
        outs = torch.empty(B, self.n_query, self.vision_cfg.width, dtype=torch.bfloat16, device=self.device_)
        hbuf = torch.empty(B, self.hidden, dtype=torch.bfloat16, device=self.device_)
        for k in range(self.n_query):
            down = self._project_down(last)
            outs[:, k] = down
            if k == self.n_query - 1:
                break
            up = self._project_up(down).contiguous()
            self.engine.llm_decode(embeds=up, hidden=hbuf, B=B)
            last = hbuf
        return outs
