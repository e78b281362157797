"""Tensor-parallel host logic.

CPU (gloo, world_size 2): head-range partition exported by the C ABI (emu_tp_head_range) tiles the head set for
divisible and non-divisible head counts, and the rendezvous plumbing bench.py uses (a 128-byte id broadcast from
rank 0) works across processes.  GPU (>= 2 devices): tools/tp_check.py under torchrun compares TP-N logits with the
CPU oracle."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _head_ranges(n_heads, tp):
    from emu_b200 import _lib
    lib = _lib.load()
    out = []
    for r in range(tp):
        s, c = ctypes.c_int(), ctypes.c_int()
        assert lib.emu_tp_head_range(n_heads, tp, r, ctypes.byref(s), ctypes.byref(c)) == 0
        out.append((s.value, c.value))
    return out


@pytest.mark.parametrize("n_heads,tp", [(52, 8), (52, 4), (52, 2), (40, 8), (3, 2), (16, 8), (5, 1)])
def test_head_ranges_tile_the_heads(n_heads, tp):
    rs = _head_ranges(n_heads, tp)
    pos = 0
    for s, c in rs:
        assert s == pos and c >= n_heads // tp and c <= (n_heads + tp - 1) // tp
        pos += c
    assert pos == n_heads


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    # the same 128-byte id broadcast bench.py / tools/tp_check.py do (ncclUniqueId stand-in: no GPU here)
    buf = torch.zeros(128, dtype=torch.uint8)
    if rank == 0:
        buf.copy_(torch.arange(128, dtype=torch.uint8))
    dist.broadcast(buf, 0)
    mine = _head_ranges(52, world)[rank]
    gathered = [None] * world
    dist.all_gather_object(gathered, mine)
    ok = bool((buf == torch.arange(128, dtype=torch.uint8)).all()) and sum(c for _, c in gathered) == 52
    # row-parallel partial sums + all-reduce == the full projection (what the engine does with NCCL on the GPU)
    g = torch.Generator().manual_seed(0)
    x, w = torch.randn(2, 64, generator=g), torch.randn(16, 64, generator=g)
    cols = slice(rank * 64 // world, (rank + 1) * 64 // world)
    part = x[:, cols] @ w[:, cols].t()
    dist.all_reduce(part)
    ok = ok and torch.allclose(part, x @ w.t(), atol=1e-4)
    q.put((rank, ok))
    dist.destroy_process_group()


def _dp_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from emu_b200.emu2.emu import encode_images_data_parallel
    ok = True
    for B in (1, 2, 3, 5, 8):      # fewer images than ranks, ragged, even
        imgs = torch.arange(B, dtype=torch.float32).view(B, 1, 1, 1).expand(B, 3, 4, 4).contiguous()
        seen = []

        def encode_local(x):       # stand-in for the ViT: one "token" row per image that names the image
            seen.append(x[:, 0, 0, 0].tolist())
            return x[:, 0, :2, :2].reshape(x.shape[0], 4, 1) * 10.0
        out = encode_images_data_parallel(encode_local, imgs, rank, world)
        ok = ok and out.shape == (B, 4, 1) and torch.equal(out[:, 0, 0], torch.arange(B, dtype=torch.float32) * 10.0)
    q.put((rank, ok))
    dist.destroy_process_group()


def test_vit_data_parallel_sharding_gloo_world2():
    """Data-parallel ViT under tensor parallelism (SURVEY.md §8e row 2): slices tile the batch in order, the gathered result
    is the batch in its original order on every rank — also when a rank has no image."""
    from emu_b200.emu2.emu import dp_image_slices
    for n, w in [(32, 8), (4, 8), (1, 2), (5, 4), (9, 2)]:
        sl = dp_image_slices(n, w)
        assert len(sl) == w and sl[0][0] == 0 and sl[-1][1] == n and all(a[1] == b[0] for a, b in zip(sl, sl[1:]))
    assert dp_image_slices(32, 8) == [(4 * r, 4 * r + 4) for r in range(8)]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + os.getpid() % 1000
    ps = [ctx.Process(target=_dp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = [q.get(timeout=120) for _ in ps]
    for p in ps:
        p.join(timeout=60)
    assert sorted(res) == [(0, True), (1, True)]


def test_gloo_world2_rendezvous_and_sharding():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 1000
    ps = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = [q.get(timeout=120) for _ in ps]
    for p in ps:
        p.join(timeout=60)
    assert sorted(res) == [(0, True), (1, True)]


@pytest.mark.gpu
def test_tp2_logits_match_oracle():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29611", os.path.join(ROOT, "tools", "tp_check.py")],
                       capture_output=True, text=True, timeout=600)
    assert "TP_CHECK_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


@pytest.mark.gpu
def test_cfg_parallel_pair_matches_single_gpu():
    """UNet denoising split over a CFG-parallel pair: latents bitwise equal on both ranks and to the single-GPU loop."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29613",
                        os.path.join(ROOT, "tools", "cfg_parallel_check.py")], capture_output=True, text=True, timeout=600)
    assert "CFG_PARALLEL_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
