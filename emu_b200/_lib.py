"""ctypes binding of libemu_b200.so (the C ABI in include/emu_b200.h).

There is no CPU fallback: importing this module only loads the library; every compute entry point needs a
CUDA device and raises :class:`EmuError` otherwise.  If the shared library is missing the import fails loudly.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libemu_b200.so")

EMU_OK = 0
ERRORS = {-1: "EMU_ERR_INVALID", -2: "EMU_ERR_CUDA", -3: "EMU_ERR_NOMEM", -4: "EMU_ERR_STATE",
          -5: "EMU_ERR_UNSUPPORTED", -6: "EMU_ERR_NCCL"}
DTYPE_F32, DTYPE_BF16, DTYPE_F16 = 0, 1, 2
EPI_NONE, EPI_GELU, EPI_SWIGLU, EPI_GEGLU, EPI_RELU, EPI_QUICK_GELU = 0, 1, 2, 3, 4, 5


class EmuError(RuntimeError):
    pass


class EmuConfig(C.Structure):
    _fields_ = [
        ("llm_hidden", C.c_int), ("llm_layers", C.c_int), ("llm_heads", C.c_int), ("llm_head_dim", C.c_int),
        ("llm_ffn", C.c_int), ("llm_vocab", C.c_int),
        ("llm_rms_eps", C.c_float), ("llm_rope_theta", C.c_float),
        ("llm_max_batch", C.c_int), ("llm_max_seq", C.c_int),
        ("vit_image", C.c_int), ("vit_patch", C.c_int), ("vit_width", C.c_int), ("vit_layers", C.c_int),
        ("vit_heads", C.c_int), ("vit_mlp", C.c_int),
        ("vit_ln_eps", C.c_float), ("vit_postnorm", C.c_int), ("vit_final_ln", C.c_int), ("vit_max_batch", C.c_int),
        ("cf_layers", C.c_int), ("cf_dim", C.c_int), ("cf_heads", C.c_int), ("cf_ffn", C.c_int),
        ("cf_queries", C.c_int), ("cf_enc_width", C.c_int), ("cf_out_dim", C.c_int), ("cf_buckets", C.c_int),
        ("cf_max_distance", C.c_int),
        ("reserved", C.c_int * 8),
    ]


class EmuUNetConfig(C.Structure):
    _fields_ = [
        ("in_channels", C.c_int), ("out_channels", C.c_int), ("n_blocks", C.c_int),
        ("block_out_channels", C.c_int * 4), ("layers_per_block", C.c_int), ("transformer_layers", C.c_int * 4),
        ("head_dim", C.c_int), ("cross_attention_dim", C.c_int), ("use_linear_projection", C.c_int),
        ("addition_time_embed_dim", C.c_int), ("projection_class_embeddings_input_dim", C.c_int),
        ("norm_groups", C.c_int), ("norm_eps", C.c_float), ("mid_transformer_layers", C.c_int), ("num_heads", C.c_int),
    ]


class EmuVAEConfig(C.Structure):
    _fields_ = [
        ("latent_channels", C.c_int), ("out_channels", C.c_int), ("n_blocks", C.c_int),
        ("block_out_channels", C.c_int * 4), ("layers_per_block", C.c_int), ("norm_groups", C.c_int),
    ]


class EmuSafetyConfig(C.Structure):
    _fields_ = [
        ("image_size", C.c_int), ("patch_size", C.c_int), ("width", C.c_int), ("layers", C.c_int), ("heads", C.c_int),
        ("mlp", C.c_int), ("proj_dim", C.c_int), ("n_special", C.c_int), ("n_concepts", C.c_int), ("ln_eps", C.c_float),
        ("resize_shortest_edge", C.c_int), ("crop_size", C.c_int), ("image_mean", C.c_float * 3), ("image_std", C.c_float * 3),
    ]


# every symbol declared in include/emu_b200.h (tests/test_abi.py checks the header against this list)
SYMBOLS = [
    "emu_beam_topk", "emu_beam_step", "emu_sample_tokens", "emu_image_to_uint8", "emu_preprocess_image", "emu_engine_create", "emu_engine_destroy", "emu_last_error", "emu_nccl_unique_id", "emu_tp_head_range", "emu_engine_load_tensor",
    "emu_vit_forward", "emu_llm_reset", "emu_llm_embed", "emu_llm_prefill", "emu_llm_decode", "emu_llm_cur_len", "emu_llm_expand",
    "emu_project", "emu_cformer_forward", "emu_unet_configure", "emu_unet_forward", "emu_denoise_step",
    "emu_denoise_step_multistep", "emu_vae_configure", "emu_vae_decode", "emu_op_gemm", "emu_op_gemm_skinny", "emu_op_conv3x3", "emu_op_gemv", "emu_op_gemv_rope_qkv",
    "emu_op_attn_prefill", "emu_op_attn_decode", "emu_op_rmsnorm", "emu_op_layernorm", "emu_launch_count",
    "emu_debug_gemm_phases", "emu_debug_gemv_phases",
    "emu_version",
]
# ... and in include/emu_b200_safety.h (the safety checker)
SAFETY_SYMBOLS = ["emu_safety_configure", "emu_safety_check", "emu_safety_embed", "emu_preprocess_clip"]
# ... and in include/emu_b200_slots.h (slot mode: continuous batching)
SLOT_SYMBOLS = ["emu_llm_slots_begin", "emu_llm_join", "emu_llm_fork", "emu_llm_leave", "emu_llm_slot_len"]
# ... and in include/emu_b200_ops.h (the decode-step kernels as stand-alone operators)
OPS_SYMBOLS = ["emu_op_attn_decode_rows", "emu_op_rope_kv_write", "emu_op_kv_indir_update", "emu_op_kv_reorder",
               "emu_op_argmax_rows", "emu_op_attn_prefill_rows"]
# ... and in include/emu_b200_prefix.h (prefix caching: kept slots, per-slot continuation and the prefix copy kernel)
PREFIX_SYMBOLS = ["emu_llm_leave_keep", "emu_llm_slot_kept", "emu_llm_copy_prefix", "emu_llm_extend", "emu_llm_kv_cache",
                  "emu_op_kv_prefix_copy"]
# ... and in include/emu_b200_chunked.h (chunked prefill: the mixed decode + prefill step and its kernels)
CHUNKED_SYMBOLS = ["emu_llm_step", "emu_op_rope_kv_write_packed", "emu_op_attn_prefill_packed"]
# ... and in include/emu_b200_regress.h (regression slots: Emu2-Gen's prompt encoding for every slot at once)
REGRESS_SYMBOLS = ["emu_llm_regress_join", "emu_llm_regress_step"]
# ... and in include/emu_b200_spec.h (prompt-lookup speculative decoding: verify / commit, the draft and acceptance kernels)
SPEC_SYMBOLS = ["emu_llm_verify", "emu_llm_commit", "emu_spec_draft", "emu_spec_accept", "emu_op_attn_verify"]
# ... and in include/emu_b200_gen_slots.h (latent slots: continuous batching for image generation)
GEN_SLOT_SYMBOLS = ["emu_denoise_step_slots", "emu_op_denoise_prepare", "emu_op_denoise_euler"]
# ... and in include/emu_b200_diffusion_ops.h (the diffusion kernels as stand-alone operators)
DIFFUSION_OPS_SYMBOLS = ["emu_op_groupnorm", "emu_op_timestep_embedding", "emu_op_upsample2x", "emu_op_im2col3x3",
                         "emu_op_copy_cols", "emu_op_nchw_to_nhwc", "emu_op_nhwc_to_nchw", "emu_op_mean_tokens",
                         "emu_op_vae_post", "emu_op_denoise_multistep", "emu_op_vae_attention"]

_lib = None


def load():
    """Load libemu_b200.so; raise if it has not been built (no silent fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise EmuError("libemu_b200.so not found at %s — run `python -m emu_b200.build` (needs nvcc)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    lib.emu_last_error.restype = C.c_char_p
    lib.emu_last_error.argtypes = [C.c_void_p]
    lib.emu_version.restype = C.c_char_p
    lib.emu_launch_count.restype = C.c_uint64
    lib.emu_engine_destroy.restype = None
    lib.emu_engine_destroy.argtypes = [C.c_void_p]
    lib.emu_engine_create.argtypes = [C.POINTER(EmuConfig), C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]
    _lib = lib
    return lib


def _ptr(t):
    if t is None:
        return None
    if isinstance(t, int):
        return C.c_void_p(t)
    assert t.is_cuda, "engine arguments must be CUDA tensors"
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def check(rc, engine=None):
    if rc == EMU_OK:
        return
    msg = ERRORS.get(rc, str(rc))
    if engine is not None:
        detail = load().emu_last_error(engine)
        if detail:
            msg += ": " + detail.decode()
    raise EmuError(msg)


def require_cuda():
    if not torch.cuda.is_available():
        raise EmuError("emu_b200 needs a CUDA device (H100 / sm_90a); there is no CPU fallback")


_DT = {torch.float32: DTYPE_F32, torch.bfloat16: DTYPE_BF16, torch.float16: DTYPE_F16}


class Engine:
    """Thin RAII wrapper over EmuEngine*; methods map 1:1 to the C ABI."""

    def __init__(self, cfg: EmuConfig, tp_rank=0, tp_size=1, nccl_uid: bytes = None):
        require_cuda()
        self.lib = load()
        self.cfg = cfg
        self.h = C.c_void_p()
        uid = C.create_string_buffer(nccl_uid, 128) if nccl_uid is not None else None
        rc = self.lib.emu_engine_create(C.byref(cfg), tp_rank, tp_size, uid, C.byref(self.h))
        check(rc)
        self.tp_rank, self.tp_size = tp_rank, tp_size

    def close(self):
        if getattr(self, "h", None) is not None and self.h:
            self.lib.emu_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- weights ----
    def load_tensor(self, key: str, t: torch.Tensor):
        t = t.detach()
        if not t.is_contiguous():
            t = t.contiguous()
        if t.dtype not in _DT:
            t = t.float()
        shape = (C.c_int64 * max(t.dim(), 1))(*([int(s) for s in t.shape] or [1]))
        src = C.c_void_p(t.data_ptr())
        rc = self.lib.emu_engine_load_tensor(self.h, key.encode(), src, _DT[t.dtype], shape, max(t.dim(), 1), _stream())
        check(rc, self.h)

    def load_state_dict(self, sd, prefix=""):
        for k, v in sd.items():
            if k.endswith("rotary_emb.inv_freq"):
                continue
            self.load_tensor(prefix + k, v)

    # ---- ViT ----
    def vit_forward(self, image: torch.Tensor, n_query: int, pool=True):
        c = self.cfg
        B = image.shape[0]
        image = image.to(torch.bfloat16).contiguous()
        G = c.vit_image // c.vit_patch
        if pool:
            out = torch.empty(B, n_query, c.vit_width, dtype=torch.bfloat16, device=image.device)
        else:
            out = torch.empty(B, G * G + 1, c.vit_width, dtype=torch.bfloat16, device=image.device)
        check(self.lib.emu_vit_forward(self.h, _ptr(image), B, _ptr(out), n_query, 1 if pool else 0, _stream()), self.h)
        return out

    # ---- LLM ----
    def llm_reset(self):
        check(self.lib.emu_llm_reset(self.h, _stream()), self.h)

    def llm_embed(self, ids: torch.Tensor):
        ids32 = ids.to(torch.int32).contiguous()
        out = torch.empty(*ids.shape, self.cfg.llm_hidden, dtype=torch.bfloat16, device=ids.device)
        check(self.lib.emu_llm_embed(self.h, _ptr(ids32), ids32.numel(), _ptr(out), _stream()), self.h)
        return out

    def llm_prefill(self, embeds, attention_mask=None, hf_positions=True, want_hidden=False, want_logits=True):
        B, N, H = embeds.shape
        embeds = embeds.to(torch.bfloat16).contiguous()
        mask = attention_mask.to(torch.int32).contiguous() if attention_mask is not None else None
        hidden = torch.empty(B, N, H, dtype=torch.bfloat16, device=embeds.device) if want_hidden else None
        logits = torch.empty(B, self.cfg.llm_vocab, dtype=torch.float32, device=embeds.device) if want_logits else None
        check(self.lib.emu_llm_prefill(self.h, _ptr(embeds), _ptr(mask), B, N, 1 if hf_positions else 0, _ptr(hidden),
                                       _ptr(logits), _stream()), self.h)
        return hidden, logits

    def llm_decode(self, token_ids=None, embeds=None, beam_src=None, logits=None, hidden=None, next_ids=None,
                   ban_id=-1, B=None):
        if B is None:
            B = token_ids.shape[0] if token_ids is not None else embeds.shape[0]
        # the C entry point takes bare pointers: a short buffer would be written past its end
        c = self.cfg
        for name, t, need, dt in (("logits", logits, B * c.llm_vocab, torch.float32), ("hidden", hidden, B * c.llm_hidden, torch.bfloat16),
                                  ("next_ids", next_ids, B, torch.int32), ("token_ids", token_ids, B, torch.int32),
                                  ("beam_src", beam_src, B, torch.int32), ("embeds", embeds, B * c.llm_hidden, torch.bfloat16)):
            if t is not None and (t.dtype != dt or t.numel() < need or not t.is_contiguous()):
                raise ValueError(f"llm_decode: {name} must be a contiguous {dt} tensor of at least {need} elements, got "
                                 f"{tuple(t.shape)} {t.dtype}")
        check(self.lib.emu_llm_decode(self.h, _ptr(token_ids), _ptr(embeds), _ptr(beam_src), B, _ptr(logits),
                                      _ptr(hidden), _ptr(next_ids), ban_id, _stream()), self.h)

    def cur_len(self):
        return self.lib.emu_llm_cur_len(self.h)

    def llm_expand(self, src_idx, new_B):
        """cache row b <- row src_idx[b] for b < new_B (beam search: one prefill per prompt, then num_beams cache rows)"""
        src = src_idx.to(torch.int32).contiguous()
        check(self.lib.emu_llm_expand(self.h, _ptr(src), int(new_B), _stream()), self.h)

    # ---- slot mode (include/emu_b200_slots.h): continuous batching ----
    def slots_begin(self, n_slots):
        """forget the cache and enter slot mode with n_slots free slots (emu_llm_reset leaves it)"""
        check(self.lib.emu_llm_slots_begin(self.h, int(n_slots), _stream()), self.h)

    @staticmethod
    def _host_slots(slots):
        slots = [int(s) for s in slots]
        return (C.c_int32 * max(1, len(slots)))(*slots), len(slots)

    def join(self, slots, embeds, attention_mask=None, want_logits=True):
        """prefill len(slots) new sequences [n, N, hidden] (left-padded mask [n, N]) into the given free slots; returns the
        logits of every sequence's last position [n, vocab] fp32 (or None)"""
        n, N, H = embeds.shape
        if n != len(slots):
            raise ValueError("join: %d sequences for %d slots" % (n, len(slots)))
        embeds = embeds.to(torch.bfloat16).contiguous()
        mask = attention_mask.to(torch.int32).contiguous() if attention_mask is not None else None
        if mask is not None and tuple(mask.shape) != (n, N):
            raise ValueError("join: attention_mask must be [%d, %d], got %s" % (n, N, tuple(mask.shape)))
        logits = torch.empty(n, self.cfg.llm_vocab, dtype=torch.float32, device=embeds.device) if want_logits else None
        hs, cnt = self._host_slots(slots)
        check(self.lib.emu_llm_join(self.h, hs, cnt, _ptr(embeds), _ptr(mask), N, _ptr(logits), _stream()), self.h)
        return logits

    def fork(self, src_slot, dst_slots):
        """the free dst_slots continue the sequence of src_slot (beam expansion; no KV is moved)"""
        hs, cnt = self._host_slots(dst_slots)
        check(self.lib.emu_llm_fork(self.h, int(src_slot), hs, cnt, _stream()), self.h)

    def leave(self, slots):
        """free the given live slots (a beam group leaves together)"""
        hs, cnt = self._host_slots(slots)
        check(self.lib.emu_llm_leave(self.h, hs, cnt, _stream()), self.h)

    def slot_len(self, slot):
        return int(self.lib.emu_llm_slot_len(self.h, int(slot)))

    # ---- prefix caching (include/emu_b200_prefix.h) ----
    def kv_cache(self):
        """the engine's KV cache as a bf16 tensor view [layers, 2 (K, V), rows, heads, llm_max_seq, head_dim] (no copy)"""
        ptr, dims = C.c_void_p(), (C.c_int64 * 5)()
        check(self.lib.emu_llm_kv_cache(self.h, C.byref(ptr), dims), self.h)
        shape = tuple(int(d) for d in dims)

        class _View:
            __cuda_array_interface__ = dict(shape=shape, typestr="<i2", data=(ptr.value, False), version=3)
        t = torch.as_tensor(_View(), device="cuda").view(torch.bfloat16)
        return t.view(shape[0] // 2, 2, *shape[1:])

    def leave_keep(self, slots, keep):
        """free the given live slots, slot i keeping its first keep[i] cache positions (a beam group leaves together)"""
        if len(keep) != len(slots):
            raise ValueError("leave_keep: %d keep lengths for %d slots" % (len(keep), len(slots)))
        hs, cnt = self._host_slots(slots)
        hk, _ = self._host_slots(keep)
        check(self.lib.emu_llm_leave_keep(self.h, hs, hk, cnt, _stream()), self.h)

    def slot_kept(self, slot):
        return int(self.lib.emu_llm_slot_kept(self.h, int(slot)))

    def copy_prefix(self, src_slot, dst_slot, P):
        """positions [0, P) of src_slot's own row (live or kept) -> the free dst_slot, which becomes kept with length P"""
        check(self.lib.emu_llm_copy_prefix(self.h, int(src_slot), int(dst_slot), int(P), _stream()), self.h)

    def extend(self, slots, prefix, new, embeds, want_logits=True):
        """the free slots continue at length prefix[i] (<= their kept length) with new[i] tokens of embeds [n, N, hidden]
        (right-padded); returns the logits of every row's last real token [n, vocab] fp32 (or None)"""
        n, N, H = embeds.shape
        if not n == len(slots) == len(prefix) == len(new):
            raise ValueError("extend: %d rows for %d slots, %d prefixes, %d counts" % (n, len(slots), len(prefix), len(new)))
        embeds = embeds.to(torch.bfloat16).contiguous()
        logits = torch.empty(n, self.cfg.llm_vocab, dtype=torch.float32, device=embeds.device) if want_logits else None
        hs, cnt = self._host_slots(slots)
        hp, _ = self._host_slots(prefix)
        hn, _ = self._host_slots(new)
        check(self.lib.emu_llm_extend(self.h, hs, hp, hn, cnt, _ptr(embeds), N, _ptr(logits), _stream()), self.h)
        return logits

    # ---- chunked prefill (include/emu_b200_chunked.h) ----
    def step(self, slots, prefix, new, final, embeds, token_ids=None, B=0, beam_src=None, logits=None, want_logits=True):
        """one mixed step: the decode rows of slots [0, B) (token_ids [>= B] int32, beam_src [>= B] or None, logits
        [>= B, vocab] fp32 filled in place or None) and one packed prefill segment per free slot: slots[i] continues at
        prefix[i] with new[i] tokens of embeds [sum(new), hidden], live afterwards if final[i] else kept; returns the logits
        of every segment's last token [n, vocab] fp32 (or None)"""
        n = len(slots)
        if not n == len(prefix) == len(new) == len(final):
            raise ValueError("step: %d slots, %d prefixes, %d counts, %d final flags" % (n, len(prefix), len(new), len(final)))
        embeds = embeds.to(torch.bfloat16).contiguous()
        if embeds.dim() != 2 or embeds.shape[0] != sum(int(k) for k in new):
            raise ValueError("step: embeds must be [sum(new) = %d, hidden], got %s" % (sum(int(k) for k in new), tuple(embeds.shape)))
        c = self.cfg
        for name, t, need, dt in (("logits", logits, B * c.llm_vocab, torch.float32), ("token_ids", token_ids, B, torch.int32),
                                  ("beam_src", beam_src, B, torch.int32)):
            if t is not None and (t.dtype != dt or t.numel() < need or not t.is_contiguous()):
                raise ValueError(f"step: {name} must be a contiguous {dt} tensor of at least {need} elements, got "
                                 f"{tuple(t.shape)} {t.dtype}")
        last = torch.empty(n, c.llm_vocab, dtype=torch.float32, device=embeds.device) if want_logits else None
        hs, cnt = self._host_slots(slots)
        hp, _ = self._host_slots(prefix)
        hn, _ = self._host_slots(new)
        hf, _ = self._host_slots([1 if f else 0 for f in final])
        check(self.lib.emu_llm_step(self.h, _ptr(token_ids) if B else None, _ptr(beam_src) if B else None, int(B),
                                    _ptr(logits) if B else None, hs, hp, hn, hf, cnt, _ptr(embeds), _ptr(last), _stream()),
              self.h)
        return last

    # ---- regression slots (include/emu_b200_regress.h) ----
    def _regress_out(self, name, out, rows):
        # the C entry points take a bare pointer: a short buffer would be written past its end
        if out.dtype != torch.bfloat16 or out.dim() != 3 or not out.is_contiguous() or out.shape[0] < rows \
                or out.shape[2] != self.cfg.vit_width:
            raise ValueError("%s: out must be a contiguous bf16 [>= %d, L, %d] tensor, got %s %s"
                             % (name, rows, self.cfg.vit_width, tuple(out.shape), out.dtype))

    def regress_join(self, slots, new, embeds, out):
        """prefill len(slots) prompts into the free slots, packed back to back in embeds [sum(new), hidden] (prompt i has
        new[i] tokens, no padding); each slot becomes a live regression slot with its embedding 0 in out[slot][0]
        (out [n_slots, L, width] bf16, the other rows untouched)"""
        if len(new) != len(slots):
            raise ValueError("regress_join: %d token counts for %d slots" % (len(new), len(slots)))
        embeds = embeds.to(torch.bfloat16).contiguous()
        if embeds.dim() != 2 or embeds.shape[0] != sum(int(k) for k in new) or embeds.shape[1] != self.cfg.llm_hidden:
            raise ValueError("regress_join: embeds must be [sum(new) = %d, %d], got %s"
                             % (sum(int(k) for k in new), self.cfg.llm_hidden, tuple(embeds.shape)))
        self._regress_out("regress_join", out, max(int(s) for s in slots) + 1 if slots else 0)
        hs, cnt = self._host_slots(slots)
        hn, _ = self._host_slots(new)
        check(self.lib.emu_llm_regress_join(self.h, hs, hn, cnt, _ptr(embeds), _ptr(out), int(out.shape[1]), _stream()),
              self.h)

    def regress_step(self, B, out):
        """one regression step of every live slot below B: its next embedding goes to out[slot][k] (out as in regress_join;
        one CUDA graph per (B, out))"""
        self._regress_out("regress_step", out, int(B))
        check(self.lib.emu_llm_regress_step(self.h, int(B), _ptr(out), int(out.shape[1]), _stream()), self.h)

    # ---- speculative decoding (include/emu_b200_spec.h) ----
    def llm_verify(self, tokens, n, logits=None, next_ids=None, ban_id=-1, ban_rows=0):
        """one weight pass over tokens[:n] (int32, row 0 the last committed token, then the drafts) at positions L .. L + n - 1
        of the batch-1 cache: logits [n, vocab] fp32 and / or next_ids [n] int32 (rows < ban_rows without ban_id); the cache
        length stays L until llm_commit"""
        c = self.cfg
        for name, t, need, dt in (("tokens", tokens, n, torch.int32), ("logits", logits, n * c.llm_vocab, torch.float32),
                                  ("next_ids", next_ids, n, torch.int32)):
            if t is not None and (t.dtype != dt or t.numel() < need or not t.is_contiguous()):
                raise ValueError(f"llm_verify: {name} must be a contiguous {dt} tensor of at least {need} elements, got "
                                 f"{tuple(t.shape)} {t.dtype}")
        check(self.lib.emu_llm_verify(self.h, _ptr(tokens), int(n), _ptr(logits), _ptr(next_ids), int(ban_id), int(ban_rows),
                                      _stream()), self.h)

    def llm_commit(self, m):
        """keep the first m positions the last verify wrote"""
        check(self.lib.emu_llm_commit(self.h, int(m), _stream()), self.h)

    def spec_draft(self, hist, hist_len, k, max_ngram, max_length, eos_token_id, out, out_len):
        """the prompt-lookup draft of hist[:hist_len] (device int32 scalars / buffers): out[0] = the last token, out[1:1 + d]
        the draft, out_len = d"""
        if out.numel() < 1 + k or hist.dtype != torch.int32 or out.dtype != torch.int32:
            raise ValueError("spec_draft: int32 buffers, out of at least 1 + k = %d entries" % (1 + k))
        check(self.lib.emu_spec_draft(_ptr(hist), _ptr(hist_len), int(k), int(max_ngram), int(max_length), int(eos_token_id),
                                      _ptr(out), _ptr(out_len), _stream()))

    def spec_accept(self, hist, hist_len, tokens, next_ids, n, eos_token_id, max_len, stats):
        """append the accepted drafts of a verify over tokens[:n] and the token after them to hist; stats[:2] = (tokens
        appended, finished)"""
        if hist.numel() < max_len or hist.dtype != torch.int32:
            raise ValueError("spec_accept: hist must be int32 with room for max_len = %d tokens" % max_len)
        check(self.lib.emu_spec_accept(_ptr(hist), _ptr(hist_len), _ptr(tokens), _ptr(next_ids), int(n), int(eos_token_id),
                                       int(max_len), _ptr(stats), _stream()))

    def sample_tokens(self, logits, temperature=1.0, top_k=0, top_p=1.0, ban_id=-1, seed=0, offset=0):
        return op_sample_tokens(logits, temperature, top_k, top_p, -1 if ban_id is None else ban_id, seed, offset)

    def beam_topk(self, logits, running_scores, batch, beams, keep, ban_id=-1, prev_tokens=None, prev_len=0,
                  repetition_penalty=1.0, penalty_on_logits=False, no_repeat_ngram=0, allowed=None):
        if ban_id is None:
            ban_id = -1
        lg = logits if (logits.dtype == torch.float32 and logits.is_contiguous()) else logits.float().contiguous()
        return op_beam_topk(lg, running_scores, batch, beams, keep, ban_id=int(ban_id), prev_tokens=prev_tokens,
                            prev_len=prev_len, repetition_penalty=float(repetition_penalty),
                            penalty_on_logits=penalty_on_logits, no_repeat_ngram=int(no_repeat_ngram or 0), allowed=allowed)

    def beam_state(self, batch, beams, max_length, pad_token_id, device):
        return BeamState(batch, beams, max_length, pad_token_id, device)

    def beam_step(self, st, topk_lp, topk_idx, cur_len, eos_token_id, length_penalty, early_stopping):
        """emu_beam_step: hypothesis bookkeeping of one HF beam-search step on the device (no host synchronisation)."""
        best_len = st.max_length if (early_stopping == "never" and length_penalty > 0.0) else cur_len + 1
        es = 1 if early_stopping is True else (2 if early_stopping == "never" else 0)
        check(self.lib.emu_beam_step(_ptr(topk_lp), _ptr(topk_idx), st.batch, st.beams, self.cfg.llm_vocab, cur_len,
                                     st.max_length, int(eos_token_id), C.c_float(float((cur_len + 1) ** length_penalty)),
                                     C.c_float(float(best_len ** length_penalty)), es, _ptr(st.running_seq),
                                     _ptr(st.running_scores), _ptr(st.sequences), _ptr(st.beam_scores), _ptr(st.is_finished),
                                     _ptr(st.fin_len), _ptr(st.unsat), _ptr(st.done), _ptr(st.next_tokens), _ptr(st.beam_src),
                                     _stream()), self.h)
        st.done_calls.add_(st.done)   # device-side count of the calls that ended with `done` set (see BeamState.result)

    # ---- Emu1 Causal-Former ----
    def cformer_forward(self, vit_tokens, n_queries, out_dim):
        B, Nv, _ = vit_tokens.shape
        vit_tokens = vit_tokens.to(torch.bfloat16).contiguous()
        out = torch.empty(B, n_queries, out_dim, dtype=torch.bfloat16, device=vit_tokens.device)
        check(self.lib.emu_cformer_forward(self.h, _ptr(vit_tokens), B, Nv, _ptr(out), _stream()), self.h)
        return out

    def vae_configure(self, vcfg: "EmuVAEConfig"):
        self.vcfg = vcfg
        check(self.lib.emu_vae_configure(self.h, C.byref(vcfg)), self.h)

    def vae_decode(self, latents):
        """latents [B,4,h,w] bf16 (already divided by the scaling factor) -> images [B, 8h, 8w, 3] fp32 in [0,1]"""
        B, _, h, w = latents.shape
        latents = latents.to(torch.bfloat16).contiguous()
        f = 2 ** (self.vcfg.n_blocks - 1)
        out = torch.empty(B, h * f, w * f, self.vcfg.out_channels, dtype=torch.float32, device=latents.device)
        check(self.lib.emu_vae_decode(self.h, _ptr(latents), B, h, w, _ptr(out), _stream()), self.h)
        return out

    # ---- safety checker ----
    def safety_configure(self, scfg: "EmuSafetyConfig"):
        self.scfg = scfg
        check(self.lib.emu_safety_configure(self.h, C.byref(scfg)), self.h)

    def safety_check(self, images_u8, scores=False):
        """images [B, H, W, 3] uint8 CUDA (flagged ones are zeroed in place) -> flags int32 [B] (and the scores
        fp32 [B, n_special + n_concepts] with scores=True), all on the device"""
        assert images_u8.dtype == torch.uint8 and images_u8.dim() == 4 and images_u8.shape[3] == 3 and images_u8.is_cuda
        assert images_u8.is_contiguous(), "the check blacks out flagged images in place: pass a contiguous tensor"
        B, H, W, _ = images_u8.shape
        flags = torch.empty(B, dtype=torch.int32, device=images_u8.device)
        sc = (torch.empty(B, self.scfg.n_special + self.scfg.n_concepts, dtype=torch.float32, device=images_u8.device)
              if scores else None)
        check(self.lib.emu_safety_check(self.h, _ptr(images_u8), B, H, W, _ptr(flags), _ptr(sc), _stream()), self.h)
        return (flags, sc) if scores else flags

    def safety_embed(self, pixel_values):
        """pixel_values [B, 3, S, S] (CLIP-normalised) -> image_embeds [B, proj_dim] bf16"""
        pv = pixel_values.to(torch.bfloat16).contiguous()
        out = torch.empty(pv.shape[0], self.scfg.proj_dim, dtype=torch.bfloat16, device=pv.device)
        check(self.lib.emu_safety_embed(self.h, _ptr(pv), pv.shape[0], _ptr(out), _stream()), self.h)
        return out

    # ---- diffusion ----
    def unet_configure(self, ucfg: "EmuUNetConfig"):
        self.ucfg = ucfg
        check(self.lib.emu_unet_configure(self.h, C.byref(ucfg)), self.h)

    def unet_forward(self, latents, timestep, ctx, text_embeds=None, time_ids=None):
        """latents [B2,C,h,w] bf16 NCHW, ctx [B2,L,Cc], text_embeds [B2,Cc], time_ids [B2,6] int32 -> noise [B2,C,h,w]"""
        B2, Cc, h, w = latents.shape
        latents = latents.to(torch.bfloat16).contiguous()
        ctx = ctx.to(torch.bfloat16).contiguous()
        te = text_embeds.to(torch.bfloat16).contiguous() if text_embeds is not None else None
        ti = time_ids.to(torch.int32).contiguous() if time_ids is not None else None
        out = torch.empty(B2, self.ucfg.out_channels, h, w, dtype=torch.bfloat16, device=latents.device)
        check(self.lib.emu_unet_forward(self.h, _ptr(latents), C.c_float(float(timestep)), _ptr(ctx), ctx.shape[1],
                                        _ptr(te), _ptr(ti), B2, h, w, _ptr(out), _stream()), self.h)
        return out

    def denoise_step(self, latents_f32, sigma, sigma_next, timestep, guidance, ctx, text_embeds, time_ids):
        """One iteration of the denoise loop, latents [B,4,h,w] fp32 updated in place. ctx = [cond; uncond]."""
        B, _, h, w = latents_f32.shape
        assert latents_f32.dtype == torch.float32 and latents_f32.is_contiguous()
        check(self.lib.emu_denoise_step(self.h, _ptr(latents_f32), C.c_float(float(sigma)), C.c_float(float(sigma_next)),
                                        C.c_float(float(timestep)), C.c_float(float(guidance)), _ptr(ctx), ctx.shape[1],
                                        _ptr(text_embeds), _ptr(time_ids), B, h, w, _stream()), self.h)

    def denoise_step_slots(self, latents_f32, params, live, ctx, text_embeds, time_ids, B):
        """One iteration over latent slots 0..B-1 (include/emu_b200_gen_slots.h): latents [>=B,4,h,w] fp32 in place, params
        fp32 [>=B, 4] {sigma, sigma_next, timestep, guidance} and live int32 [>=B] on the device, read when the step runs.
        ctx [>=2B, L, Cc], text_embeds [>=2B, Cc], time_ids [>=2B, 6]: rows 2b / 2b+1 are slot b's cond / uncond."""
        _, _, h, w = latents_f32.shape
        for name, t, dt, rows in (("latents", latents_f32, torch.float32, B), ("params", params, torch.float32, B),
                                  ("live", live, torch.int32, B), ("ctx", ctx, torch.bfloat16, 2 * B),
                                  ("text_embeds", text_embeds, torch.bfloat16, 2 * B), ("time_ids", time_ids, torch.int32, 2 * B)):
            if t.dtype != dt or not t.is_contiguous() or t.shape[0] < rows:
                raise ValueError("denoise_step_slots: %s must be a contiguous %s tensor of at least %d rows, got %s %s"
                                 % (name, dt, rows, tuple(t.shape), t.dtype))
        if params.shape[1:] != (4,) or time_ids.shape[1:] != (6,):
            raise ValueError("denoise_step_slots: params must be [B, 4] and time_ids [2B, 6]")
        check(self.lib.emu_denoise_step_slots(self.h, _ptr(latents_f32), _ptr(params), _ptr(live), _ptr(ctx), ctx.shape[1],
                                              _ptr(text_embeds), _ptr(time_ids), int(B), h, w, _stream()), self.h)

    def denoise_step_multistep(self, latents_f32, state_f32, coef8, timestep, guidance, ctx):
        """One PNDM / PLMS iteration (emu_denoise_step_multistep): latents [B,4,h,w] fp32 in place, state [4,B,4,h,w] fp32."""
        B, _, h, w = latents_f32.shape
        assert latents_f32.dtype == torch.float32 and latents_f32.is_contiguous()
        assert state_f32.dtype == torch.float32 and state_f32.is_contiguous() and state_f32.numel() == 4 * latents_f32.numel()
        coef = (C.c_float * 8)(*[float(v) for v in coef8])
        check(self.lib.emu_denoise_step_multistep(self.h, _ptr(latents_f32), _ptr(state_f32), coef, C.c_float(float(timestep)),
                                                  C.c_float(float(guidance)), _ptr(ctx), ctx.shape[1], B, h, w, _stream()),
              self.h)

    def project(self, which: int, x: torch.Tensor, out_dim: int):
        x2 = x.reshape(-1, x.shape[-1]).to(torch.bfloat16).contiguous()
        y = torch.empty(x2.shape[0], out_dim, dtype=torch.bfloat16, device=x.device)
        check(self.lib.emu_project(self.h, which, _ptr(x2), x2.shape[0], _ptr(y), _stream()), self.h)
        return y.reshape(*x.shape[:-1], out_dim)


# ---- stand-alone operators (used by tests and micro-benchmarks) ----
def op_gemm(A, W, bias=None, residual=None, epi=EPI_NONE, out_fp32=False, force_bn=0):
    require_cuda()
    lib = load()
    M, K = A.shape
    N = W.shape[0]
    n_out = N // 2 if epi in (EPI_SWIGLU, EPI_GEGLU) else N
    Cm = torch.empty(M, n_out, dtype=torch.float32 if out_fp32 else torch.bfloat16, device=A.device)
    rc = lib.emu_op_gemm(_ptr(A), A.stride(0), _ptr(W), W.stride(0), M, N, K, _ptr(bias), _ptr(residual),
                         residual.stride(0) if residual is not None else 0, epi, _ptr(Cm), n_out,
                         1 if out_fp32 else 0, force_bn, _stream())
    check(rc)
    return Cm


def op_gemm_skinny(X, W, residual=None, epi=EPI_NONE, out_fp32=False):
    """X [B <= 32, K] . W [N, K]^T through the wide-decode projection kernel (gemm_skinny.cu)"""
    require_cuda()
    lib = load()
    B, K = X.shape
    N = W.shape[0]
    n_out = N // 2 if epi == EPI_SWIGLU else N
    Cm = torch.empty(B, n_out, dtype=torch.float32 if out_fp32 else torch.bfloat16, device=X.device)
    check(lib.emu_op_gemm_skinny(_ptr(X), X.stride(0), _ptr(W), W.stride(0), B, N, K, _ptr(residual),
                                 residual.stride(0) if residual is not None else 0, epi, _ptr(Cm), n_out, 1 if out_fp32 else 0,
                                 _stream()))
    return Cm


def debug_gemm_phases(A, W, bias=None, residual=None, epi=EPI_NONE, force_bn=0):
    """emu_op_gemm + per-CTA phase stamps -> (C, stamps [148, 8] int64 on the host)"""
    require_cuda()
    lib = load()
    M, K = A.shape
    N = W.shape[0]
    n_out = N // 2 if epi in (EPI_SWIGLU, EPI_GEGLU) else N
    Cm = torch.empty(M, n_out, dtype=torch.bfloat16, device=A.device)
    stamps = torch.zeros(148, 8, dtype=torch.int64, device=A.device)
    check(lib.emu_debug_gemm_phases(_ptr(A), A.stride(0), _ptr(W), W.stride(0), M, N, K, _ptr(bias), _ptr(residual),
                                    residual.stride(0) if residual is not None else 0, epi, _ptr(Cm), n_out, force_bn,
                                    _ptr(stamps), _stream()))
    return Cm, stamps.cpu()


def op_conv3x3(x_nhwc, w_k, bias=None, residual=None):
    require_cuda()
    lib = load()
    NB, H, W_, Cin = x_nhwc.shape
    Cout = w_k.shape[0]
    y = torch.empty(NB, H, W_, Cout, dtype=torch.bfloat16, device=x_nhwc.device)
    check(lib.emu_op_conv3x3(_ptr(x_nhwc), NB, H, W_, Cin, _ptr(w_k), Cout, _ptr(bias), _ptr(residual), _ptr(y),
                             _stream()))
    return y


def op_gemv(W, x, norm_w=None, eps=1e-6, mode=EPI_NONE, bias=None, residual=None, out_fp32=False, pdl=False):
    require_cuda()
    lib = load()
    N, K = W.shape
    B = x.shape[0]
    n_out = N // 2 if mode == EPI_SWIGLU else N
    y = torch.empty(B, n_out, dtype=torch.float32 if out_fp32 else torch.bfloat16, device=x.device)
    rc = lib.emu_op_gemv(_ptr(W), N, K, _ptr(x), x.stride(0), B, _ptr(norm_w), C.c_float(eps), mode, _ptr(bias),
                         _ptr(residual), residual.stride(0) if residual is not None else 0, _ptr(y), n_out,
                         1 if out_fp32 else 0, 1 if pdl else 0, _stream())
    check(rc)
    return y


def op_gemv_rope_qkv(W, n_heads, head_dim, x, norm_w, eps, rope_cos, rope_sin, pos, pos_off, k_cache, v_cache, t_max):
    require_cuda()
    lib = load()
    B = x.shape[0]
    q = torch.empty(B, n_heads * head_dim, dtype=torch.bfloat16, device=x.device)
    rc = lib.emu_op_gemv_rope_qkv(_ptr(W), n_heads, head_dim, W.shape[1], _ptr(x), x.stride(0), B, _ptr(norm_w),
                                  C.c_float(eps), _ptr(rope_cos), _ptr(rope_sin), _ptr(pos), _ptr(pos_off), _ptr(q),
                                  _ptr(k_cache), _ptr(v_cache), t_max, _stream())
    check(rc)
    return q


def op_attn_prefill(q, k, v, scale, causal=False, kv_start=None, bias=None):
    """q [B,Nq,H,D], k/v [B,Nk,H,D] (any strides with contiguous D) -> [B,Nq,H,D]"""
    require_cuda()
    lib = load()
    B, Nq, H, D = q.shape
    Nk = k.shape[1]
    out = torch.empty(B, Nq, H, D, dtype=torch.bfloat16, device=q.device)
    st = []
    for t in (q, k, v, out):
        assert t.stride(3) == 1
        st += [t.stride(0), t.stride(1), t.stride(2)]
    st12 = (C.c_int64 * 12)(*st)
    rc = lib.emu_op_attn_prefill(_ptr(q), _ptr(k), _ptr(v), _ptr(out), B, H, Nq, Nk, D, st12, C.c_float(scale),
                                 1 if causal else 0, _ptr(kv_start), _ptr(bias), _stream())
    check(rc)
    return out


def op_preprocess_image(img_u8_hwc, out_h, out_w, mean, std, dtype=torch.float32):
    """[H, W, 3] uint8 CUDA tensor -> [3, out_h, out_w] fp32/bf16: Resize(BICUBIC) + ToTensor + Normalize, bit-exact with the
    reference's torchvision + Pillow transform."""
    require_cuda()
    lib = load()
    assert img_u8_hwc.dtype == torch.uint8 and img_u8_hwc.dim() == 3 and img_u8_hwc.shape[2] == 3 and img_u8_hwc.is_cuda
    img = img_u8_hwc.contiguous()
    H, W, _ = img.shape
    out = torch.empty(3, out_h, out_w, dtype=dtype, device=img.device)
    m3 = (C.c_float * 3)(*[float(v) for v in mean])
    s3 = (C.c_float * 3)(*[float(v) for v in std])
    code = {torch.float32: DTYPE_F32, torch.bfloat16: DTYPE_BF16}[dtype]
    check(lib.emu_preprocess_image(_ptr(img), H, W, out_h, out_w, m3, s3, _ptr(out), code, _stream()))
    return out


def op_preprocess_clip(images_u8_bhwc, size=224, crop=224, mean=(0.48145466, 0.4578275, 0.40821073),
                       std=(0.26862954, 0.26130258, 0.27577711), dtype=torch.bfloat16):
    """[B, H, W, 3] uint8 CUDA -> [B, 3, crop, crop]: CLIPImageProcessor (shortest-edge bicubic resize, centre crop, rescale,
    normalise), bit-exact with transformers' CLIPImageProcessorPil."""
    require_cuda()
    x = images_u8_bhwc
    assert x.dtype == torch.uint8 and x.dim() == 4 and x.shape[3] == 3 and x.is_cuda
    x = x.contiguous()
    B, H, W, _ = x.shape
    out = torch.empty(B, 3, crop, crop, dtype=dtype, device=x.device)
    m3 = (C.c_float * 3)(*[float(v) for v in mean])
    s3 = (C.c_float * 3)(*[float(v) for v in std])
    code = {torch.float32: DTYPE_F32, torch.bfloat16: DTYPE_BF16}[dtype]
    check(load().emu_preprocess_clip(_ptr(x), B, H, W, int(size), int(crop), m3, s3, _ptr(out), code, _stream()))
    return out


def op_image_to_uint8(image01):
    """fp32 [0,1] CUDA tensor -> uint8 (x * 255, round half to even) — numpy_to_pil's conversion on the device."""
    require_cuda()
    x = image01.contiguous()
    assert x.dtype == torch.float32 and x.is_cuda
    out = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    check(load().emu_image_to_uint8(_ptr(x), _ptr(out), C.c_int64(x.numel()), _stream()))
    return out


def op_sample_tokens(logits, temperature=1.0, top_k=0, top_p=1.0, ban_id=-1, seed=0, offset=0):
    """logits [R, V] fp32 CUDA -> int32 [R]: temperature -> top-k -> top-p -> multinomial on the device."""
    require_cuda()
    lg = logits if (logits.dtype == torch.float32 and logits.is_contiguous()) else logits.float().contiguous()
    out = torch.empty(lg.shape[0], dtype=torch.int32, device=lg.device)
    check(load().emu_sample_tokens(_ptr(lg), lg.shape[0], lg.shape[1], C.c_float(temperature or 1.0), int(top_k or 0),
                                   C.c_float(1.0 if top_p is None else top_p), int(ban_id), C.c_uint64(seed & (2 ** 64 - 1)),
                                   C.c_uint64(offset), _ptr(out), _stream()))
    return out


class BeamState:
    """Device-resident state of one beam search (layout documented at emu_beam_step in include/emu_b200.h)."""

    def __init__(self, batch, beams, max_length, pad_token_id, device):
        self.batch, self.beams, self.max_length = batch, beams, max_length
        i32 = dict(dtype=torch.int32, device=device)
        self.running_seq = torch.full((2, batch, beams, max_length), pad_token_id, **i32)
        self.sequences = torch.full((2, batch, beams, max_length), pad_token_id, **i32)
        self.running_scores = torch.zeros(batch, beams, dtype=torch.float32, device=device)
        self.running_scores[:, 1:] = -1e9
        self.beam_scores = torch.full((batch, beams), -1e9, dtype=torch.float32, device=device)
        self.is_finished = torch.zeros(batch, beams, **i32)
        self.fin_len = torch.zeros(batch, beams, **i32)
        self.unsat = torch.ones(batch, **i32)
        self.done = torch.zeros(1, **i32)
        self.done_calls = torch.zeros(1, **i32)
        self.next_tokens = torch.zeros(batch * beams, **i32)
        self.beam_src = torch.zeros(batch * beams, **i32)

    def live(self, cur_len):
        """the plane holding the sequences after `cur_len` tokens"""
        return cur_len & 1

    def is_done(self):
        return bool(self.done.item())   # the only device->host synchronisation of the loop

    def final_len(self, cur_len):
        """The step count at which the search finished.  The host polls `done` only every few steps and the steps launched
        in between are no-ops on this state — they do not flip the sequence planes either — so the plane that holds the
        final hypotheses is the one of the step that SET `done`, not of the step at which the host noticed:
        calls made = cur_len, of which done_calls ended with `done` set  =>  finished after cur_len + 1 - done_calls steps."""
        late = int(self.done_calls.item())
        return cur_len + 1 - late if late > 0 else cur_len

    def result(self, cur_len, n=1):
        """the n best finished hypotheses of every batch row, best first: [batch * n, longest of them] (HF
        num_return_sequences; the reference's default and Emu1's num_captions=1 take n = 1)"""
        cur_len = self.final_len(cur_len)
        best = self.sequences[self.live(cur_len), :, :n, :].reshape(self.batch * n, self.max_length)
        gen_len = int(self.fin_len[:, :n].max())
        return best[:, :gen_len].to(torch.int64)


def op_beam_topk(logits, running_scores, batch, beams, keep, ban_id=-1, prev_tokens=None, prev_len=0, repetition_penalty=1.0,
                 penalty_on_logits=False, no_repeat_ngram=0, allowed=None):
    """logits [batch*beams, V] fp32 (overwritten), running_scores [batch, beams] fp32 -> (scores [batch, keep] fp32,
    flat indices [batch, keep] int32 = beam*V + token), HF _beam_search step semantics.  prev_tokens: int32 [batch*beams, L]
    (any row stride), prev_len valid tokens per row."""
    require_cuda()
    lib = load()
    V = logits.shape[-1]
    assert logits.dtype == torch.float32 and logits.is_contiguous()
    rs = running_scores.to(torch.float32).contiguous().view(-1) if running_scores is not None else None
    stride = 0
    if prev_tokens is not None and prev_len > 0:
        assert prev_tokens.dtype == torch.int32 and prev_tokens.stride(-1) == 1
        prev_tokens = prev_tokens.reshape(batch * beams, -1) if prev_tokens.dim() != 2 else prev_tokens
        stride = prev_tokens.stride(0)
    else:
        prev_tokens, prev_len = None, 0
    if allowed is not None:
        allowed = allowed.to(torch.uint8).contiguous()
    out_lp = torch.empty(batch, keep, dtype=torch.float32, device=logits.device)
    out_idx = torch.empty(batch, keep, dtype=torch.int32, device=logits.device)
    check(lib.emu_beam_topk(_ptr(logits), _ptr(rs), batch, beams, V, keep, ban_id, _ptr(prev_tokens), int(prev_len), int(stride),
                            C.c_float(repetition_penalty), 1 if penalty_on_logits else 0, int(no_repeat_ngram), _ptr(allowed),
                            _ptr(out_lp), _ptr(out_idx), _stream()))
    return out_lp, out_idx


def op_attn_decode(q, k_cache, v_cache, pos, start, scale, max_len):
    """q [B,H*D]; caches [B,H,T,D]; pos/start int32 [B] -> [B,H*D]"""
    require_cuda()
    lib = load()
    B, H, T, D = k_cache.shape
    out = torch.empty(B, H * D, dtype=torch.bfloat16, device=q.device)
    rc = lib.emu_op_attn_decode(_ptr(q), _ptr(k_cache), _ptr(v_cache), B, H, D, T, _ptr(pos), _ptr(start),
                                C.c_float(scale), _ptr(out), max_len, _stream())
    check(rc)
    return out


# ---- the decode-step kernels (include/emu_b200_ops.h) ----
def _i32(t, name):
    if t is not None and (t.dtype != torch.int32 or not t.is_contiguous()):
        raise ValueError("%s must be a contiguous int32 tensor" % name)
    return _ptr(t)


def op_attn_decode_rows(q, k_cache, v_cache, pos, start, scale, max_len_hint, indir=None):
    """q [B, H*D] (B <= 32); caches [rows, H, T, D]; pos / start int32 [B] (start may be None); indir int32 [rows, T] or None
    (row b) -> [B, H*D]"""
    require_cuda()
    _, H, T, D = k_cache.shape
    B = q.shape[0]
    out = torch.empty(B, H * D, dtype=torch.bfloat16, device=q.device)
    check(load().emu_op_attn_decode_rows(_ptr(q), _ptr(k_cache), _ptr(v_cache), B, H, D, T, _i32(pos, "pos"),
                                         _i32(start, "start"), _i32(indir, "indir"), C.c_float(scale), _ptr(out),
                                         int(max_len_hint), _stream()))
    return out


def op_rope_kv_write(qkv, H, D, rope_cos, rope_sin, k_cache, v_cache, pos_off=None, pos0=0, pos_dev=None, q_out=None,
                     kv_row=None):
    """qkv [B, N, 3*H*D] (q rotated in place unless q_out [B*N, H*D] is given); caches [rows, H, T, D] written in place"""
    require_cuda()
    B, N, _ = qkv.shape
    assert qkv.is_contiguous() and k_cache.is_contiguous() and v_cache.is_contiguous()
    check(load().emu_op_rope_kv_write(_ptr(qkv), B, N, H, D, _ptr(rope_cos), _ptr(rope_sin), _i32(pos_off, "pos_off"),
                                      int(pos0), _i32(pos_dev, "pos_dev"), _ptr(q_out), _i32(kv_row, "kv_row"), _ptr(k_cache),
                                      _ptr(v_cache), k_cache.shape[2], _stream()))


def op_kv_indir_update(indir, src_idx, n_tok, row_len=None):
    """indir int32 [rows, T] in place: indir[b, t] <- indir[src_idx[b], t] for b < len(src_idx), t < n_tok (and < row_len[b])"""
    require_cuda()
    check(load().emu_op_kv_indir_update(_i32(indir, "indir"), _i32(src_idx, "src_idx"), _i32(row_len, "row_len"),
                                        src_idx.numel(), indir.shape[1], int(n_tok), _stream()))


def op_kv_reorder(cache, src_idx, n_used_tokens, B=None):
    """cache [outer, Bcap, H, T, D] in place: row b <- row src_idx[b] for b < B, slots t < n_used_tokens"""
    require_cuda()
    outer, Bcap, H, T, D = cache.shape
    assert cache.is_contiguous()
    B = src_idx.numel() if B is None else B
    check(load().emu_op_kv_reorder(_ptr(cache), Bcap, _i32(src_idx, "src_idx"), int(B), outer, int(n_used_tokens), H, D, T,
                                   _stream()))


def op_argmax_rows(logits):
    """logits fp32 [rows, cols] (contiguous, any base alignment) -> int32 [rows], first index of the maximum"""
    require_cuda()
    assert logits.dtype == torch.float32 and logits.is_contiguous()
    out = torch.empty(logits.shape[0], dtype=torch.int32, device=logits.device)
    check(load().emu_op_argmax_rows(_ptr(logits), logits.shape[0], logits.shape[1], _ptr(out), _stream()))
    return out


def op_attn_prefill_rows(q, k, v, scale, causal=False, kv_start=None, kv_row=None):
    """q [B,Nq,H,D]; k/v [rows,Nk,H,D] views (any strides with contiguous D) of which query batch b reads batch kv_row[b]
    (kv_row None: k/v have B entries and b reads b) -> [B,Nq,H,D]"""
    require_cuda()
    B, Nq, H, D = q.shape
    Nk = k.shape[1]
    out = torch.empty(B, Nq, H, D, dtype=torch.bfloat16, device=q.device)
    st = []
    for t in (q, k, v, out):
        assert t.stride(3) == 1
        st += [t.stride(0), t.stride(1), t.stride(2)]
    st12 = (C.c_int64 * 12)(*st)
    check(load().emu_op_attn_prefill_rows(_ptr(q), _ptr(k), _ptr(v), _ptr(out), B, H, Nq, Nk, D, st12, C.c_float(scale),
                                          1 if causal else 0, _i32(kv_start, "kv_start"), _i32(kv_row, "kv_row"),
                                          k.shape[0] if kv_row is not None else 0, _stream()))
    return out


# ---- chunked prefill kernels (include/emu_b200_chunked.h) ----
def op_attn_verify(q, k_cache, v_cache, pos, scale, row=0, start=None, indir=None, n=None):
    """the verify attention: q [n, >= H*D] bf16 (head h of row j at [j, h*D:(h+1)*D]), one layer's cache [rows, H, t_max, D];
    query j sees positions start[0] .. pos[0] + j of cache row `row` (through indir [t_max] if given) -> [n, H*D] bf16"""
    _, H, t_max, D = k_cache.shape
    n = q.shape[0] if n is None else n
    out = torch.empty(n, H * D, dtype=torch.bfloat16, device=q.device)
    check(load().emu_op_attn_verify(_ptr(q), C.c_long(q.stride(0)), _ptr(k_cache), _ptr(v_cache), int(n), int(H), int(D),
                                    int(t_max), int(row), _i32(pos, "pos"), _i32(start, "start"), _i32(indir, "indir"),
                                    C.c_float(scale), _ptr(out), _stream()))
    return out


def op_rope_kv_write_packed(qkv, H, D, rope_cos, rope_sin, k_cache, v_cache, B=0, pos=None, pos_off=None, active=None,
                            q_out=None, seg_row=None, seg_q0=None, seg_new=None, seg_posoff=None):
    """qkv [M, 3*H*D] packed: rows [0, B) decode rows (q -> q_out [B, H*D], k / v at slot pos[b] of row b if active[b]), then
    the segments (seg_new[i] rows each, q in place, k / v at slots seg_q0[i] + j of row seg_row[i]); caches [rows, H, T, D]"""
    require_cuda()
    M = qkv.shape[0]
    n = 0 if seg_new is None else seg_new.numel()
    assert qkv.is_contiguous() and k_cache.is_contiguous() and v_cache.is_contiguous()
    check(load().emu_op_rope_kv_write_packed(_ptr(qkv), M, int(B), n, H, D, _ptr(rope_cos), _ptr(rope_sin), _i32(pos, "pos"),
                                             _i32(pos_off, "pos_off"), _i32(active, "active"), _ptr(q_out),
                                             _i32(seg_row, "seg_row"), _i32(seg_q0, "seg_q0"), _i32(seg_new, "seg_new"),
                                             _i32(seg_posoff, "seg_posoff"), _ptr(k_cache), _ptr(v_cache), k_cache.shape[2],
                                             _stream()))


def op_attn_prefill_packed(q, k, v, scale, q_row0, q_len, q_off, kv_start=None, kv_row=None, Nq=None, out=None):
    """causal attention over packed queries: q [rows, H, D], batch b's q_len[b] queries start at row q_row0[b] and sit at key
    positions q_off[b] + i; k / v [kv_rows, Nk, H, D] views read at batch kv_row[b] (None: b).  Writes those rows of out
    [rows, H, D] (a new zero tensor if None) and returns it; Nq = the longest q_len (read back if None)"""
    require_cuda()
    rows, H, D = q.shape
    Nk = k.shape[1]
    if out is None:
        out = torch.zeros(rows, H, D, dtype=torch.bfloat16, device=q.device)
    if Nq is None:
        Nq = int(q_len.max())
    for t in (q, k, v, out):
        assert t.stride(-1) == 1
    st10 = (C.c_int64 * 10)(q.stride(0), q.stride(1), k.stride(0), k.stride(1), k.stride(2), v.stride(0), v.stride(1),
                            v.stride(2), out.stride(0), out.stride(1))
    check(load().emu_op_attn_prefill_packed(_ptr(q), _ptr(k), _ptr(v), _ptr(out), rows, q_len.numel(), H, int(Nq), Nk, D, st10,
                                            C.c_float(scale), _i32(q_row0, "q_row0"), _i32(q_len, "q_len"), _i32(q_off, "q_off"),
                                            _i32(kv_start, "kv_start"), _i32(kv_row, "kv_row"),
                                            k.shape[0] if kv_row is not None else 0, _stream()))
    return out


def op_kv_prefix_copy(cache, src, dst, P):
    """cache [outer, rows, H, T, D] bf16 in place: positions [0, P) of row src -> row dst"""
    require_cuda()
    outer, rows, H, T, D = cache.shape
    assert cache.is_contiguous() and cache.dtype == torch.bfloat16
    check(load().emu_op_kv_prefix_copy(_ptr(cache), outer, rows, H, D, T, int(src), int(dst), int(P), _stream()))


# ---- the denoise-step glue (include/emu_b200_gen_slots.h) ----
def _rows_layout(B, slots_adjacent):
    return (2, 1) if slots_adjacent else (1, B)


def op_denoise_prepare(latents, params, Cp, copies=2, slots_adjacent=False):
    """latents [B, C, h, w] fp32, params fp32 [B, 4] (or [4]: one set for every slot) -> (UNet input NHWC bf16
    [copies*B, h, w, Cp], per-row timesteps fp32 [copies*B]); slot b's rows are b and B + b, or 2b and 2b + 1 (copies = 2)"""
    require_cuda()
    B, Cc, h, w = latents.shape
    assert latents.dtype == torch.float32 and latents.is_contiguous()
    assert params.dtype == torch.float32 and params.is_contiguous()
    cs, ub = _rows_layout(B, slots_adjacent)
    xin = torch.empty(copies * B, h, w, Cp, dtype=torch.bfloat16, device=latents.device)
    t_rows = torch.empty(copies * B, dtype=torch.float32, device=latents.device)
    check(load().emu_op_denoise_prepare(_ptr(latents), _ptr(xin), _ptr(t_rows), B, Cc, h * w, int(Cp), _ptr(params),
                                        4 if params.dim() == 2 else 0, int(copies), cs, ub, _stream()))
    return xin, t_rows


def op_denoise_euler(latents, eps_nhwc, params, live=None, slots_adjacent=False):
    """latents [B, C, h, w] fp32 updated in place from the noise prediction eps NHWC bf16 [rows, h, w, ld] (rows as
    op_denoise_prepare's); params fp32 [B, 4] or [4]; live int32 [B] or None"""
    require_cuda()
    B, Cc, h, w = latents.shape
    assert latents.dtype == torch.float32 and latents.is_contiguous()
    assert eps_nhwc.dtype == torch.bfloat16 and eps_nhwc.is_contiguous()
    assert params.dtype == torch.float32 and params.is_contiguous()
    cs, ub = _rows_layout(B, slots_adjacent)
    check(load().emu_op_denoise_euler(_ptr(latents), _ptr(eps_nhwc), _i32(live, "live"), B, Cc, h * w, eps_nhwc.shape[-1],
                                      _ptr(params), 4 if params.dim() == 2 else 0, cs, ub, _stream()))


# ---- the diffusion kernels (include/emu_b200_diffusion_ops.h) ----
def _c_float(v):
    return C.c_float(float(v))


def _bf16c(t, name):
    if t.dtype != torch.bfloat16 or not t.is_contiguous():
        raise ValueError("%s must be a contiguous bf16 tensor" % name)
    return _ptr(t)


def op_groupnorm(x, w, b, groups, eps, silu=False, out=None):
    """x [NB, HW, C] (or [NB, H, W, C]) NHWC bf16; w, b [C] bf16 -> GroupNorm (+SiLU), same shape (written into out if given)"""
    require_cuda()
    NB, Cc = x.shape[0], x.shape[-1]
    HW = x.numel() // (NB * Cc)
    y = torch.empty_like(x) if out is None else out
    check(load().emu_op_groupnorm(_bf16c(x, "x"), _bf16c(w, "w"), _bf16c(b, "b"), _bf16c(y, "out"), NB, HW, Cc, int(groups),
                                  _c_float(eps), 1 if silu else 0, _stream()))
    return y


def op_timestep_embedding(t, out, dim, col_off=0, grp=1):
    """t fp32 [rows] -> [cos | sin] embeddings of width dim written into out bf16 [rows / grp, ld] at columns
    col_off + (r % grp) * dim of output row r / grp"""
    require_cuda()
    assert t.dtype == torch.float32 and t.is_contiguous()
    check(load().emu_op_timestep_embedding(_ptr(t), _bf16c(out, "out"), t.numel(), int(dim), out.stride(0), int(col_off),
                                           int(grp), _stream()))
    return out


def op_upsample2x(x, out=None):
    """x [NB, H, W, C] bf16 -> [NB, 2H, 2W, C], nearest"""
    require_cuda()
    NB, H, W, Cc = x.shape
    y = torch.empty(NB, 2 * H, 2 * W, Cc, dtype=x.dtype, device=x.device) if out is None else out
    check(load().emu_op_upsample2x(_bf16c(x, "x"), _ptr(y), NB, H, W, Cc, _stream()))
    return y


def op_im2col3x3(x, stride, out=None):
    """x [NB, H, W, C] bf16 -> [NB, Ho, Wo, 9 C] (3x3 taps, pad 1)"""
    require_cuda()
    NB, H, W, Cc = x.shape
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    y = torch.empty(NB, Ho, Wo, 9 * Cc, dtype=x.dtype, device=x.device) if out is None else out
    check(load().emu_op_im2col3x3(_bf16c(x, "x"), _ptr(y), NB, H, W, Cc, int(stride), _stream()))
    return y


def op_copy_cols(src, dst, col_off):
    """dst[:, col_off:col_off + src.shape[1]] = src (2-D bf16 views with unit column stride) in place"""
    require_cuda()
    assert src.dtype == dst.dtype == torch.bfloat16 and src.stride(1) == 1 and dst.stride(1) == 1
    check(load().emu_op_copy_cols(_ptr(src), _ptr(dst), C.c_int64(src.shape[0]), src.shape[1], src.stride(0), dst.stride(0),
                                  int(col_off), _stream()))


def op_nchw_to_nhwc(x, Cp, scale=1.0, out=None):
    """x [NB, C, H, W] bf16 -> [NB, H, W, Cp] bf16(x * scale), zero channels past C"""
    require_cuda()
    NB, Cc, H, W = x.shape
    y = torch.empty(NB, H, W, Cp, dtype=x.dtype, device=x.device) if out is None else out
    check(load().emu_op_nchw_to_nhwc(_bf16c(x, "x"), _ptr(y), NB, Cc, H * W, int(Cp), _c_float(scale), _stream()))
    return y


def op_nhwc_to_nchw(x, Cc, out=None):
    """x [NB, H, W, ld] bf16 -> its first Cc channels as [NB, Cc, H, W]"""
    require_cuda()
    NB, H, W, ld = x.shape
    y = torch.empty(NB, Cc, H, W, dtype=x.dtype, device=x.device) if out is None else out
    check(load().emu_op_nhwc_to_nchw(_bf16c(x, "x"), _ptr(y), NB, int(Cc), H * W, ld, _stream()))
    return y


def op_mean_tokens(x, out=None):
    """x [B, L, C] bf16 -> [B, C], the mean over L"""
    require_cuda()
    B, L, Cc = x.shape
    y = torch.empty(B, Cc, dtype=x.dtype, device=x.device) if out is None else out
    check(load().emu_op_mean_tokens(_bf16c(x, "x"), _ptr(y), B, L, Cc, _stream()))
    return y


def op_vae_post(x, Cc, out=None):
    """x [..., ld] bf16 -> fp32 [..., Cc] = clamp(x / 2 + 0.5, 0, 1) of the first Cc channels"""
    require_cuda()
    ld = x.shape[-1]
    n_pix = x.numel() // ld
    y = torch.empty(*x.shape[:-1], Cc, dtype=torch.float32, device=x.device) if out is None else out
    check(load().emu_op_vae_post(_bf16c(x, "x"), _ptr(y), C.c_int64(n_pix), int(Cc), ld, _stream()))
    return y


def op_denoise_multistep(latents, eps_nhwc, hist, saved, params, cfg):
    """latents, saved [B, C, h, w] fp32 and hist [3, B, C, h, w] fp32 updated in place from eps NHWC bf16 [B or 2B, h, w, ld];
    params fp32 [8] on the device (layout at emu_op_denoise_multistep)"""
    require_cuda()
    B, Cc, h, w = latents.shape
    for t, n in ((latents, "latents"), (hist, "hist"), (saved, "saved"), (params, "params")):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError("%s must be a contiguous fp32 tensor" % n)
    check(load().emu_op_denoise_multistep(_ptr(latents), _bf16c(eps_nhwc, "eps"), _ptr(hist), _ptr(saved), B, Cc, h * w,
                                          eps_nhwc.shape[-1], _ptr(params), 1 if cfg else 0, _stream()))


def op_vae_attention(q, k, v, out=None):
    """q, k, v [B, T, C] bf16 -> softmax(q k^T / sqrt(C)) v, [B, T, C]"""
    require_cuda()
    B, T, Cc = q.shape
    assert k.shape == v.shape == q.shape
    out = torch.empty_like(q) if out is None else out
    check(load().emu_op_vae_attention(_bf16c(q, "q"), _bf16c(k, "k"), _bf16c(v, "v"), _ptr(out), B, T, Cc, _stream()))
    return out


def op_rmsnorm(x, w, eps):
    require_cuda()
    y = torch.empty_like(x)
    check(load().emu_op_rmsnorm(_ptr(x), _ptr(w), _ptr(y), x.shape[0], x.shape[1], C.c_float(eps), _stream()))
    return y


def op_layernorm(x, w, b, eps, residual=None):
    require_cuda()
    y = torch.empty_like(x)
    check(load().emu_op_layernorm(_ptr(x), _ptr(w), _ptr(b), _ptr(residual), _ptr(y), x.shape[0], x.shape[1],
                                  C.c_float(eps), _stream()))
    return y


def launch_count():
    return int(load().emu_launch_count())
