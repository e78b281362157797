"""Drop-in for the reference's Emu1 model ``models.modeling_emu.Emu`` (Emu1/models/modeling_emu.py:22-249).

Same public methods and argument meaning: ``generate(samples={"image","prompt"}, ...)`` (:100-185) and
``generate_image(text, image, placeholder)`` (:187-249).  Arithmetic on the H100 engine: EVA-CLIP-g ViT (pre-norm,
head_dim 88) + ``ln_visual`` -> Causal-Former (T5 decoder stack, 32 causal queries) -> LLaMA-13B prefill/decode;
the regression head is ``stu_regress_head`` and regressed embeddings are fed back directly (no project_up).
"""
import json
import os.path as osp
from typing import List, Optional

import torch

from .. import _lib, generation
from ..emu2.conf import load_llama_config

DEFAULT_IMG_PLACEHOLDER = "[<IMG_PLH>]"
EMU1_LLAMA_13B = dict(hidden_size=5120, num_hidden_layers=40, num_attention_heads=40, intermediate_size=13824,
                      rms_norm_eps=1e-6, max_position_embeddings=2048, vocab_size=32000, rope_theta=10000.0)
EMU1_VISION = dict(image_size=224, layers=40, width=1408, head_width=88, mlp_ratio=4.3637, patch_size=14)  # Emu-14B.json
T5_BASE = dict(layers=12, d_model=768, heads=12, d_ff=3072, buckets=32, max_distance=128)


def build_tokenizer(llama_config_path, instruct=False):
    """LlamaTokenizer + [PAD] and the three image tokens, as Emu1/models/modeling_llama.py:135-165 builds it."""
    import transformers
    tok = transformers.LlamaTokenizer.from_pretrained(llama_config_path, model_max_length=2048, padding_side="right",
                                                      use_fast=False)
    extra = ["[IMG]", "[/IMG]", "<image>"] + (["[USER]", "[ASSISTANT]"] if instruct else [])
    tok.add_special_tokens(dict(pad_token="[PAD]", bos_token="<s>", eos_token="</s>", unk_token="<unk>",
                                additional_special_tokens=extra))
    return tok


class _Decoder:
    def __init__(self, tokenizer, cfg):
        self.tokenizer = tokenizer
        self.config = cfg


class Emu:
    def __init__(self, embed_dim=1024, multimodal_cfg=None, vision_cfg=None, vladapter_cfg=None, *, tokenizer=None,
                 llama_config=None, llama_config_path="./models/llama_config", cformer_cfg=None, args=None, prompt=None,
                 max_batch: int = 8, max_seq: Optional[int] = None, device="cuda", **_ignored):
        # (_ignored: quick_gelu / cast_dtype / pad_id / apply_lemmatizer of the reference constructor — training / eval knobs
        # with no effect on generate; `prompt` is the default prompt `generate` falls back to, modeling_emu.py:128)
        vision_cfg = dict(EMU1_VISION, **(vision_cfg or {}))
        vladapter_cfg = vladapter_cfg or {"n_causal": 32}
        self.vision_cfg = vision_cfg
        self.n_causal = vladapter_cfg.get("n_causal", 32)
        lc = load_llama_config(llama_config if llama_config is not None else
                               (llama_config_path if osp.exists(llama_config_path) else EMU1_LLAMA_13B))
        self.llama_cfg = lc
        if tokenizer is None:
            tokenizer = build_tokenizer(llama_config_path, bool(getattr(args, "instruct", False)))
        self.decoder = _Decoder(tokenizer, lc)
        t5 = dict(T5_BASE, **(cformer_cfg or {}))
        self.device_ = torch.device(device)
        c = _lib.EmuConfig()
        c.llm_hidden, c.llm_layers, c.llm_heads = lc["hidden_size"], lc["num_hidden_layers"], lc["num_attention_heads"]
        c.llm_head_dim = lc["hidden_size"] // lc["num_attention_heads"]
        c.llm_ffn, c.llm_vocab = lc["intermediate_size"], len(tokenizer)
        c.llm_rms_eps, c.llm_rope_theta = lc["rms_norm_eps"], lc["rope_theta"]
        c.llm_max_batch, c.llm_max_seq = max_batch, max_seq or lc.get("max_position_embeddings", 2048)
        c.vit_image, c.vit_patch, c.vit_width = vision_cfg["image_size"], vision_cfg["patch_size"], vision_cfg["width"]
        c.vit_layers = vision_cfg["layers"]
        c.vit_heads = vision_cfg["width"] // vision_cfg["head_width"]
        c.vit_mlp = int(vision_cfg["width"] * vision_cfg["mlp_ratio"])
        c.vit_ln_eps, c.vit_postnorm, c.vit_final_ln, c.vit_max_batch = 1e-6, 0, 1, 8
        c.cf_layers, c.cf_dim, c.cf_heads, c.cf_ffn = t5["layers"], t5["d_model"], t5["heads"], t5["d_ff"]
        c.cf_queries, c.cf_enc_width, c.cf_out_dim = self.n_causal, vision_cfg["width"], lc["hidden_size"]
        c.cf_buckets, c.cf_max_distance = t5["buckets"], t5["max_distance"]
        self.engine = _lib.Engine(c)
        self.hidden = c.llm_hidden
        self.n_tokens = (vision_cfg["image_size"] // vision_cfg["patch_size"]) ** 2 + 1
        self.image_placeholder = "[IMG]" + "<image>" * self.n_causal + "[/IMG]"
        self.prompt = prompt

    @classmethod
    def from_json(cls, path, **kw):
        cfg = json.load(open(path))
        return cls(**cfg, **kw)

    def load_state_dict(self, state_dict, strict: bool = False):
        if "module" in state_dict and isinstance(state_dict["module"], dict):  # DeepSpeed-style ckpt (inference.py:54-57)
            state_dict = state_dict["module"]
        skip = ("visual.norm.", "visual.fc_norm.", "visual.head.", "visual.rope.")
        for k, v in state_dict.items():
            if k.endswith("rotary_emb.inv_freq") or k.startswith(skip):
                continue
            self.engine.load_tensor(k, v)
        return self

    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    # visual.forward_features -> ln_visual -> cformer  (modeling_emu.py:125-126)
    @torch.no_grad()
    def encode_image(self, image: torch.Tensor):
        feats = self.engine.vit_forward(image.to(self.device_), 0, pool=False)  # [B, 257, 1408] incl. ln_visual
        return self.engine.cformer_forward(feats, self.n_causal, self.hidden)   # [B, 32, 5120]

    def _tokenize_left(self, text):
        tok = self.decoder.tokenizer
        tok.padding_side = "left"
        inputs = tok(text, padding="longest", return_tensors="pt", add_special_tokens=True)
        tok.padding_side = "right"
        return inputs.input_ids.to(self.device_), inputs.attention_mask.to(self.device_)

    @torch.no_grad()
    def generate(self, samples, do_sample=False, num_beams=5, max_new_tokens=50, min_length=1, top_p=0.9,
                 repetition_penalty=1.0, length_penalty=0.0, num_captions=1, temperature=1, penalty_alpha=None,
                 top_k=None, no_repeat_ngram_size=None, **kwargs):
        prompt = samples["prompt"] if "prompt" in samples else self.prompt
        if isinstance(prompt, str):
            prompt = [prompt]
        input_ids, attention_mask = self._tokenize_left(prompt)
        out = self.generate_from_ids(input_ids, attention_mask, image=samples.get("image"), do_sample=do_sample,
                                     num_beams=num_beams, max_new_tokens=max_new_tokens, min_length=min_length,
                                     top_p=top_p, repetition_penalty=repetition_penalty, length_penalty=length_penalty,
                                     temperature=temperature, top_k=top_k, no_repeat_ngram_size=no_repeat_ngram_size,
                                     penalty_alpha=penalty_alpha, num_return_sequences=num_captions, **kwargs)
        return self.decoder.tokenizer.batch_decode(out, skip_special_tokens=True)

    @torch.no_grad()
    def generate_from_ids(self, input_ids, attention_mask, image=None, image_token_id=32003, do_sample=False,
                          num_beams=5, max_new_tokens=50, min_length=1, top_p=0.9, repetition_penalty=1.0,
                          length_penalty=0.0, temperature=1, top_k=None, eos_token_id=None, pad_token_id=None,
                          no_repeat_ngram_size=None, prefix_allowed_tokens_fn=None, penalty_alpha=None,
                          num_return_sequences=1, **kwargs):
        tok = self.decoder.tokenizer
        eos = eos_token_id if eos_token_id is not None else tok.eos_token_id
        pad = pad_token_id if pad_token_id is not None else tok.pad_token_id
        input_ids, attention_mask = input_ids.to(self.device_), attention_mask.to(self.device_)
        embeds = self.engine.llm_embed(input_ids)
        if image is not None:
            f = self.encode_image(image.to(torch.bfloat16))
            embeds[input_ids == image_token_id] = f.reshape(-1, f.shape[-1])
        # every knob modeling_emu.py:162-179 forwards to lm.generate; num_captions arrives as num_return_sequences
        return generation.generate(self.engine, embeds, attention_mask, max_new_tokens, eos, pad, do_sample=do_sample,
                                   num_beams=num_beams, min_length=min_length, length_penalty=length_penalty,
                                   repetition_penalty=repetition_penalty, penalty_alpha=penalty_alpha, top_k=top_k,
                                   top_p=top_p, temperature=temperature, no_repeat_ngram_size=no_repeat_ngram_size or 0,
                                   prefix_allowed_tokens_fn=prefix_allowed_tokens_fn,
                                   num_return_sequences=num_return_sequences,
                                   early_stopping=kwargs.get("early_stopping", False), generator=kwargs.get("generator"),
                                   check_every=kwargs.get("check_every"))

    @torch.no_grad()
    def generate_image(self, text: List[str], image: Optional[torch.Tensor] = None,
                       placeholder: str = DEFAULT_IMG_PLACEHOLDER) -> torch.Tensor:
        tok = self.decoder.tokenizer
        IMAGE = tok.convert_tokens_to_ids(["<image>"])[0]
        text = [t.replace(placeholder, self.image_placeholder) + "[IMG]" for t in text]
        inputs = tok(text, padding="longest", return_tensors="pt")   # right padding here (modeling_llama.py:139)
        return self.generate_image_from_ids(inputs.input_ids, inputs.attention_mask, image=image, image_token_id=IMAGE)

    @torch.no_grad()
    def generate_image_from_ids(self, input_ids, attention_mask, image=None, image_token_id=32003):
        """Cache-equivalent form of the reference's 32 full re-forwards (modeling_emu.py:205-243): prefill the
        prompt ending in [IMG], then feed stu_regress_head(h_last) back as the next input embedding."""
        input_ids, attention_mask = input_ids.to(self.device_), attention_mask.to(self.device_)
        ragged = bool((attention_mask[:, -1] == 0).any())
        if ragged:
            # The tokenizer pads on the RIGHT here (modeling_llama.py:139) and the reference appends the regressed
            # embeddings before the pads of each row (it re-tokenises the growing strings, modeling_emu.py:205-213), so every
            # row is an independent sequence at positions 0..len-1.  Same thing in cache form: rotate each row's pads to the
            # left and let the engine number positions from the first real token (hf_positions).
            n_pad = (attention_mask == 0).sum(1)
            idx = (torch.arange(input_ids.shape[1], device=self.device_)[None, :] - n_pad[:, None]) % input_ids.shape[1]
            input_ids, attention_mask = input_ids.gather(1, idx), attention_mask.gather(1, idx)
        B = input_ids.shape[0]
        embeds = self.engine.llm_embed(input_ids)
        if image is not None:
            f = self.encode_image(image.to(torch.bfloat16))
            embeds[input_ids == image_token_id] = f.reshape(-1, f.shape[-1])  # row-major order is kept by the rotation
        self.engine.llm_reset()
        hidden, _ = self.engine.llm_prefill(embeds, attention_mask, hf_positions=ragged, want_hidden=True,
                                            want_logits=False)
        last = hidden[:, -1, :].contiguous()
        outs = torch.empty(B, self.n_causal, self.hidden, dtype=torch.bfloat16, device=self.device_)
        hbuf = torch.empty(B, self.hidden, dtype=torch.bfloat16, device=self.device_)
        for k in range(self.n_causal):
            reg = self.engine.project(2, last, self.hidden).contiguous()   # stu_regress_head
            outs[:, k] = reg
            if k == self.n_causal - 1:
                break
            self.engine.llm_decode(embeds=reg, hidden=hbuf, B=B)
            last = hbuf
        return outs
