"""Tensor-parallel parity check: run under torchrun with N GPUs.

Every rank builds the tiny Emu2 LLM with tp_size = WORLD_SIZE (NCCL communicator created inside libemu_b200.so from a
unique id broadcast over torch.distributed), runs prefill + 4 teacher-forced decode steps at 2 cache rows (skinny-GEMV path)
and at 11 rows (wide path), and every rank checks the logits against the fp32 CPU oracle with the bf16-noise-relative bound of the
GPU tests (error <= 1.5 x the bf16-policy oracle's own error) and bitwise equality across ranks.  The head count never divides the rank count (3 heads on 2 ranks = 2/1, 5 on 4 = 2/1/1/1, 13 on 8 =
2/2/2/2/2/1/1/1 — the same uneven split as Emu2's 52 heads on 8 GPUs = 7/7/7/7/6/6/6/6) to exercise the zero-weight head
slot, and the vocabulary is the Emu2-Chat one (32274: not divisible by 4 or 8) to exercise the padded lm_head shard.
"""
import ctypes
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from helpers import StubTokenizer, make_emu2_state_dict  # noqa: E402
from emu_b200 import _lib  # noqa: E402
from oracle import emu_oracle as O  # noqa: E402

VIS = dict(image_size=56, patch_size=14, width=128, layers=1, head_width=32, mlp_ratio=4.0, n_query=4, v_query=4)
HEADS = {1: 3, 2: 3, 4: 5, 8: 13}
VOCAB_CHAT = 32274   # 32000 + [PAD] + 271 specials + [USER] + [ASSISTANT]  (Emu2/emu/lm.py:63-65, instruct=True)


def llama_cfg(world):
    h = HEADS.get(world, 3)
    return dict(hidden_size=128 * h, num_hidden_layers=2, num_attention_heads=h, intermediate_size=1024, rms_norm_eps=1e-6,
                max_position_embeddings=256, vocab_size=32000, rope_theta=10000.0)


class ChatTokenizer(StubTokenizer):
    def __len__(self):
        return VOCAB_CHAT


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    buf = torch.zeros(128, dtype=torch.uint8, device="cuda")
    if rank == 0:
        raw = ctypes.create_string_buffer(128)
        _lib.check(_lib.load().emu_nccl_unique_id(raw))
        buf.copy_(torch.frombuffer(bytearray(raw.raw), dtype=torch.uint8))
    dist.broadcast(buf, 0)
    uid = bytes(buf.cpu().numpy().tobytes())

    from emu_b200.emu2.conf import CLIPVisionCfg, TextDecoderCfg
    from emu_b200.emu2.emu import EmuModel
    LLAMA = llama_cfg(world)
    sd = make_emu2_state_dict(vision=VIS, llama=LLAMA, vocab=VOCAB_CHAT)
    m = EmuModel(CLIPVisionCfg(**VIS), TextDecoderCfg(), tokenizer=ChatTokenizer(), llama_config=LLAMA, max_batch=12,
                 max_seq=64, tp_rank=rank, tp_size=world, nccl_uid=uid)
    m.load_state_dict(sd)
    bf16_sd = {k: (v.to(torch.bfloat16) if v.is_floating_point() else v) for k, v in sd.items()}
    nh = LLAMA["num_attention_heads"]

    def oracle(sdx, ids, mask, toks):
        """prefill + teacher-forced decode steps -> list of last-position logits (fp32)"""
        B = ids.shape[0]
        emb = torch.nn.functional.embedding(ids, sdx["decoder.lm.model.embed_tokens.weight"])
        cache = O.KVCache(2)
        mm = mask.clone()
        h = O.llama_forward(sdx, emb, mm, layers=2, heads=nh, position_ids=O.hf_position_ids(mm), cache=cache)
        outs = [O.lm_logits(sdx, h[:, -1]).float()]
        for t in range(toks.shape[1]):
            mm = torch.cat((mm, torch.ones(B, 1, dtype=mm.dtype)), dim=1)
            e = torch.nn.functional.embedding(toks[:, t], sdx["decoder.lm.model.embed_tokens.weight"]).unsqueeze(1)
            h = O.llama_forward(sdx, e, mm, layers=2, heads=nh, position_ids=mm.long().sum(-1, keepdim=True) - 1, cache=cache)
            outs.append(O.lm_logits(sdx, h[:, -1]).float())
        return outs

    errs, ratios = [], []
    # B = 2: the skinny-GEMV decode path (exchange fused into the GEMV epilogue); B = 11: the wide path (> 8 cache rows:
    # wgmma skinny GEMM + peer-memory reduce kernel), both with left padding
    for B in (2, 11):
        g = torch.Generator().manual_seed(5 + B)
        ids = torch.randint(100, 30000, (B, 9), generator=g)
        mask = torch.ones_like(ids)
        for r in range(B):
            mask[r, : r % 4] = 0
        toks = torch.randint(100, 30000, (B, 4), generator=g)
        ref32, ref16 = oracle(sd, ids, mask, toks), oracle(bf16_sd, ids, mask, toks)
        m.engine.llm_reset()
        _, lg = m.engine.llm_prefill(m.engine.llm_embed(ids.cuda()), mask.cuda(), hf_positions=True, want_logits=True)
        got = [lg.clone()]
        out = torch.empty_like(lg)
        for t in range(toks.shape[1]):
            m.engine.llm_decode(token_ids=toks[:, t].to(torch.int32).cuda().contiguous(), logits=out, B=B)
            got.append(out.clone())
        for x, r32, r16 in zip(got, ref32, ref16):
            e_eng, e_bf = O.rel_err(x.float().cpu(), r32), O.rel_err(r16, r32)
            errs.append(e_eng)
            ratios.append(e_eng / max(e_bf, 1e-12))
            bad = e_eng > max(1.5 * e_bf, 2e-3)   # the bound the GPU tests use: 1.5 x the bf16-policy oracle's own error
            # every rank must hold bitwise identical logits (fixed-order reduction), or greedy tokens could diverge
            ref0 = x.clone()
            dist.broadcast(ref0, 0)
            if bad or not torch.equal(ref0, x):
                errs.append(1e9)
    worst = torch.tensor([max(errs)], device="cuda")
    dist.all_reduce(worst, op=dist.ReduceOp.MAX)
    if rank == 0:
        print("TP%d logits rel err vs fp32 oracle per step (2 rows then 11 rows): %s" % (world, ["%.2e" % e for e in errs]), flush=True)
        print("TP%d ratio to the bf16-policy oracle's own error (bound 1.5): %s" % (world, ["%.2f" % r for r in ratios]), flush=True)
    ok = float(worst) < 1e8
    dist.barrier()
    dist.destroy_process_group()
    if not ok:
        sys.exit(1)
    if rank == 0:
        print("TP_CHECK_OK", flush=True)


if __name__ == "__main__":
    main()
