"""GPU: the decode-step kernels through their stand-alone entry points (include/emu_b200_ops.h), each against a plain
reference of the same operation at the shapes the served model runs: up to 32 cache rows, 52 heads (26 per tensor-parallel
rank) of 128, caches of thousands of slots.

* attention (decode through the beam row table, prefill into chosen cache rows): an fp64 torch reference over the same bf16
  inputs, held to TOL_BF16 per row (relative max-abs error; one bf16 rounding of the largest element is 2^-9 = 2e-3).
* RoPE + KV append: bit-exact against the HF formulation in bf16 (q * cos + rotate_half(q) * sin, every op rounded).
* row-table update, cache reorder, argmax: they only move or select data, so they must match a Python loop exactly.

Sentinels: every cache slot a kernel must not read holds bf16 NaN, so a read out of range reaches an output and fails the
test without any fault.  Slots a kernel may load but must weight by zero (left padding before kv_start inside a loaded
block) hold 1e4 instead, because 0 x NaN would be NaN.
"""
import numpy as np
import pytest
import torch

from oracle import emu_oracle as O

pytestmark = pytest.mark.gpu

TOL_BF16 = 6e-3
ROWS = 32          # KV-cache rows the engine holds at most (kLlmMaxRows)
NUM_SMS = 132      # H100 SXM
NAN = float("nan")


def _randn(shape, seed, dev, scale=1.0, dtype=torch.bfloat16):
    g = torch.Generator(device=dev).manual_seed(seed)
    return (torch.randn(shape, generator=g, device=dev) * scale).to(dtype)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _rel_err(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


# ------------------------------------------------------------------------------------------------------------------------
# attn_decode through the row table
# ------------------------------------------------------------------------------------------------------------------------
def _decode_splits(B, H, hint):
    """the split-KV count attn_decode picks (attention.cu), used here only to place row lengths on and around split edges"""
    ns = min(-(-2 * NUM_SMS // (H * B)), -(-hint // 64))
    ns = max(ns, min(-(-8 * NUM_SMS // (H * B)), hint // 512))
    return max(1, min(ns, 16))


def _decode_cases(T, ns):
    """(start, pos) per row: the attended tokens are [start, pos]"""
    per = -(-T // ns)
    k = max(1, min(3, (T - 1) // ns))
    return [
        (0, 0),                                  # length 1
        (0, max(0, ns - 2)),                     # shorter than the split count: empty splits
        (0, ns * k - 1),                         # exactly k tokens per split
        (0, ns * k),                             # one past a split boundary
        (0, T - 1),                              # the last slot of the cache
        (min(per + 3, T - 2), T - 1),            # start past the first split of a full-length row
        (T // 2, T // 2),                        # start == pos
        (5, min(T - 1, 3 * per + 17)),           # left padding, several splits
        (1, min(T - 1, per)),                    # one split's worth, shifted by one
    ]


def _ancestor(b):
    a = (7 * b + 3) % ROWS
    return a if a != b else (a + 1) % ROWS


def _decode_reference(q, K, V, table, start, pos, scale):
    """fp64 softmax(q K^T scale) V per row over the slots the table names -> [B, H, D]"""
    B = q.shape[0]
    _, H, _, D = K.shape
    outs = []
    for b in range(B):
        t = torch.arange(int(start[b]), int(pos[b]) + 1, device=K.device)
        rows = table[b, t].long()
        kb, vb = K[rows, :, t].double(), V[rows, :, t].double()          # [n, H, D]
        s = torch.einsum("hd,nhd->hn", q[b].view(H, D).double(), kb) * scale
        outs.append(torch.einsum("hn,nhd->hd", torch.softmax(s, dim=-1), vb))
    return torch.stack(outs)


@pytest.mark.parametrize("T", [128, 2048, 4096])
@pytest.mark.parametrize("H,D", [(52, 128), (26, 128), (8, 64)])
@pytest.mark.parametrize("B", [1, 9, 20, 32])
def test_attn_decode_rows(cuda, B, H, D, T):
    """Per-row lengths and starts at the length hint the engine passes (t_max), through no table, the identity table
    (bitwise equal to none) and a beam-tree table (prefix from an ancestor row, suffix from the row itself).  Every call
    runs twice: the split combine counters must reset themselves."""
    from emu_b200 import _lib
    ns = _decode_splits(B, H, T)
    cases = _decode_cases(T, ns)
    scale = D ** -0.5
    q = _randn((B, H * D), 1, cuda)
    n_launch = -(-len(cases) // B)
    for shift in range(n_launch):
        sp = [cases[(b + shift * B) % len(cases)] for b in range(B)]
        start = torch.tensor([s for s, _ in sp], dtype=torch.int32, device=cuda)
        pos = torch.tensor([p for _, p in sp], dtype=torch.int32, device=cuda)
        own = torch.arange(ROWS, dtype=torch.int32, device=cuda)[:, None].expand(ROWS, T).contiguous()
        tree = own.clone()
        for b in range(B):
            s, p = sp[b]
            cut = s + (p - s + 1) // 2 + 1 if p > s else s   # tokens [start, cut) come from the ancestor (empty for length 1)
            tree[b, :cut] = _ancestor(b)
        for name, table in (("none", None), ("identity", own), ("beam tree", tree)):
            tab = own if table is None else table
            # NaN everywhere no row reads
            read = torch.zeros(ROWS, T, dtype=torch.bool, device=cuda)
            for b in range(B):
                t = torch.arange(sp[b][0], sp[b][1] + 1, device=cuda)
                read[tab[b, t].long(), t] = True
            K = _randn((ROWS, H, T, D), 10 + shift, cuda)
            V = _randn((ROWS, H, T, D), 20 + shift, cuda)
            K.masked_fill_(~read[:, None, :, None], NAN)
            V.masked_fill_(~read[:, None, :, None], NAN)
            out = _lib.op_attn_decode_rows(q, K, V, pos, start, scale, T, indir=table)
            again = _lib.op_attn_decode_rows(q, K, V, pos, start, scale, T, indir=table)
            assert torch.equal(_bits(out), _bits(again)), (name, "second launch differs: combine counters not reset")
            assert torch.isfinite(out.float()).all(), (name, "read a slot outside the attended range")
            ref = _decode_reference(q, K, V, tab, start, pos, scale)
            got = out.view(B, H, D)
            for b in range(B):
                err = _rel_err(got[b], ref[b])
                assert err < TOL_BF16, (name, b, sp[b], ns, err)
            if name == "none":
                plain = out
            elif name == "identity":
                assert torch.equal(_bits(out), _bits(plain)), "identity table differs from no table"
            del K, V


def test_attn_decode_rows_refuses_a_hint_past_the_cache_and_33_rows(cuda):
    from emu_b200 import _lib
    q = torch.zeros(1, 128, dtype=torch.bfloat16, device=cuda)
    K = torch.zeros(1, 1, 64, 128, dtype=torch.bfloat16, device=cuda)
    pos = torch.zeros(1, dtype=torch.int32, device=cuda)
    with pytest.raises(_lib.EmuError, match="EMU_ERR_INVALID"):
        _lib.op_attn_decode_rows(q, K, K, pos, None, 1.0, 65)
    with pytest.raises(_lib.EmuError, match="EMU_ERR_INVALID"):
        _lib.op_attn_decode_rows(torch.zeros(33, 128, dtype=torch.bfloat16, device=cuda), K, K, pos, None, 1.0, 64)


# ------------------------------------------------------------------------------------------------------------------------
# rope_kv_write: prefill, join into chosen rows, decode
# ------------------------------------------------------------------------------------------------------------------------
def _rope_tables(D, n_pos, dev):
    cos, sin = O.rope_cos_sin(torch.arange(n_pos)[None], D, 10000.0, torch.bfloat16)
    return cos[0, :, :D // 2].contiguous().to(dev), sin[0, :, :D // 2].contiguous().to(dev)


def _deinterleave(t):
    return torch.cat((t[..., 0::2], t[..., 1::2]), dim=-1)


def _interleave(t):
    d = t.shape[-1] // 2
    return torch.stack((t[..., :d], t[..., d:]), dim=-1).flatten(-2)


def _hf_rope(x_il, positions, cos_t, sin_t):
    """x [..., H, D] pair-interleaved bf16, positions [...] -> the HF rotation in bf16, pair-interleaved again.  cos / sin
    are HF's [.., D] rows (both halves equal), taken from the same bf16 tables the kernel reads."""
    x = _deinterleave(x_il.cpu())
    p = positions.cpu().long()
    cos = torch.cat((cos_t.cpu(), cos_t.cpu()), dim=-1)[p].unsqueeze(-2)
    sin = torch.cat((sin_t.cpu(), sin_t.cpu()), dim=-1)[p].unsqueeze(-2)
    return _interleave(x * cos + O.rotate_half(x) * sin)


ROPE_SHAPES = [(52, 128, 32), (52, 128, 5), (2, 64, 32), (2, 64, 3)]


@pytest.mark.parametrize("H,D,B", ROPE_SHAPES)
def test_rope_kv_write_prefill(cuda, H, D, B):
    """N = 75 tokens from slot 0 with per-row left padding (pos_off): from each row's first real token the rotated q (in
    place), k and v in the cache are bit-exact; pad slots are finite; slots past the prompt keep their NaN."""
    from emu_b200 import _lib
    N, T = 75, 128
    qkv = _randn((B, N, 3 * H * D), 30, cuda)
    before = qkv.clone()
    pad = torch.tensor([(7 * b) % 40 for b in range(B)], dtype=torch.int32, device=cuda)
    cos, sin = _rope_tables(D, T, cuda)
    kc = torch.full((B, H, T, D), NAN, dtype=torch.bfloat16, device=cuda)
    vc = kc.clone()
    _lib.op_rope_kv_write(qkv, H, D, cos, sin, kc, vc, pos_off=pad, pos0=0)
    x = before.view(B, N, 3, H, D)
    posn = (torch.arange(N)[None] - pad.cpu()[:, None].long()).clamp_min(0)          # [B, N]
    q_ref, k_ref = _hf_rope(x[:, :, 0], posn, cos, sin), _hf_rope(x[:, :, 1], posn, cos, sin)
    got = qkv.view(B, N, 3, H, D).cpu()
    assert torch.equal(_bits(got[:, :, 1:]), _bits(x[:, :, 1:].cpu())), "k / v part of qkv must stay as it was"
    kcc, vcc = kc.cpu(), vc.cpu()
    for b in range(B):
        p = int(pad[b])
        assert torch.equal(_bits(got[b, p:, 0]), _bits(q_ref[b, p:])), b
        assert torch.equal(_bits(kcc[b, :, p:N]), _bits(k_ref[b, p:].transpose(0, 1))), b
        assert torch.equal(_bits(vcc[b, :, p:N]), _bits(x[b, p:, 2].cpu().transpose(0, 1))), b
        assert torch.isfinite(kcc[b, :, :N].float()).all() and torch.isfinite(got[b, :, 0].float()).all()
    assert torch.isnan(kcc[:, :, N:].float()).all() and torch.isnan(vcc[:, :, N:].float()).all()


@pytest.mark.parametrize("H,D", [(52, 128), (2, 64)])
def test_rope_kv_write_join_into_chosen_rows(cuda, H, D):
    """A join prefills B = 3 sequences into rows {9, 2, 30} of a 32-row cache: those rows get the rotated k / v at slots
    [0, N), every other row and slot stays bitwise as it was."""
    from emu_b200 import _lib
    B, N, T = 3, 75, 96
    rows = torch.tensor([9, 2, 30], dtype=torch.int32, device=cuda)
    pad = torch.tensor([0, 11, 4], dtype=torch.int32, device=cuda)
    qkv = _randn((B, N, 3 * H * D), 31, cuda)
    x = qkv.clone().view(B, N, 3, H, D)
    cos, sin = _rope_tables(D, T, cuda)
    kc, vc = _randn((ROWS, H, T, D), 32, cuda), _randn((ROWS, H, T, D), 33, cuda)
    k0, v0 = kc.clone(), vc.clone()
    _lib.op_rope_kv_write(qkv, H, D, cos, sin, kc, vc, pos_off=pad, pos0=0, kv_row=rows)
    posn = (torch.arange(N)[None] - pad.cpu()[:, None].long()).clamp_min(0)
    k_ref = _hf_rope(x[:, :, 1], posn, cos, sin)
    written = torch.zeros(ROWS, T, dtype=torch.bool)
    for b in range(B):
        r, p = int(rows[b]), int(pad[b])
        assert torch.equal(_bits(kc[r, :, p:N].cpu()), _bits(k_ref[b, p:].transpose(0, 1))), b
        assert torch.equal(_bits(vc[r, :, p:N].cpu()), _bits(x[b, p:, 2].cpu().transpose(0, 1))), b
        written[r, :N] = True
    keep = ~written.to(cuda)[:, None, :, None].expand_as(kc)
    assert torch.equal(_bits(kc)[keep], _bits(k0)[keep]), "a row or slot outside the join was written"
    assert torch.equal(_bits(vc)[keep], _bits(v0)[keep]), "a row or slot outside the join was written"
    q_ref = _hf_rope(x[:, :, 0], posn, cos, sin)
    got = qkv.view(B, N, 3, H, D).cpu()
    for b in range(B):
        p = int(pad[b])
        assert torch.equal(_bits(got[b, p:, 0]), _bits(q_ref[b, p:])), b


@pytest.mark.parametrize("H,D,B", ROPE_SHAPES)
def test_rope_kv_write_decode(cuda, H, D, B):
    """N = 1 with a different device slot per row (slot mode): k / v land at slot pos_dev[b] of row b, rotated at
    pos_dev[b] - pos_off[b]; the rotated q goes compact to q_out and qkv stays unchanged; nothing else in the cache moves."""
    from emu_b200 import _lib
    T = 2048
    qkv = _randn((B, 1, 3 * H * D), 34, cuda)
    before = qkv.clone()
    slot = torch.tensor([(613 * b + 5) % T for b in range(B)], dtype=torch.int32)
    slot[0] = T - 1
    pad = torch.tensor([min(int(slot[b]), (3 * b) % 17) for b in range(B)], dtype=torch.int32)
    cos, sin = _rope_tables(D, T, cuda)
    kc, vc = _randn((B, H, T, D), 35, cuda), _randn((B, H, T, D), 36, cuda)
    k0, v0 = kc.clone(), vc.clone()
    q_out = torch.full((B, H * D), NAN, dtype=torch.bfloat16, device=cuda)
    _lib.op_rope_kv_write(qkv, H, D, cos, sin, kc, vc, pos_off=pad.to(cuda), pos0=0, pos_dev=slot.to(cuda), q_out=q_out)
    assert torch.equal(_bits(qkv), _bits(before)), "the decode form writes q to q_out, not in place"
    x = before.view(B, 3, H, D)
    posn = (slot - pad).long()
    q_ref, k_ref = _hf_rope(x[:, 0], posn, cos, sin), _hf_rope(x[:, 1], posn, cos, sin)
    assert torch.equal(_bits(q_out.view(B, H, D).cpu()), _bits(q_ref))
    written = torch.zeros(B, T, dtype=torch.bool)
    for b in range(B):
        s = int(slot[b])
        assert torch.equal(_bits(kc[b, :, s].cpu()), _bits(k_ref[b])), b
        assert torch.equal(_bits(vc[b, :, s].cpu()), _bits(x[b, 2].cpu())), b
        written[b, s] = True
    keep = ~written.to(cuda)[:, None, :, None].expand_as(kc)
    assert torch.equal(_bits(kc)[keep], _bits(k0)[keep]) and torch.equal(_bits(vc)[keep], _bits(v0)[keep])


# ------------------------------------------------------------------------------------------------------------------------
# beam re-parenting: row table and cache reorder
# ------------------------------------------------------------------------------------------------------------------------
def _beam_src(B):
    """cycles in both directions plus many-to-one"""
    src = list(range(B))
    third = max(1, B // 3)
    a = list(range(0, third))
    b = list(range(third, min(B, 2 * third)))
    for i, r in enumerate(a):                 # forward cycle
        src[r] = a[(i + 1) % len(a)]
    for i, r in enumerate(b):                 # backward cycle
        src[r] = b[(i - 1) % len(b)]
    for r in range(2 * third, B):             # many to one
        src[r] = B - 1 if r % 2 else third
    return src


@pytest.mark.parametrize("n_tok", [1, 1000, 4096])
@pytest.mark.parametrize("B", [5, 20, 32])
@pytest.mark.parametrize("with_len", [False, True])
def test_kv_indir_update(cuda, B, n_tok, with_len):
    from emu_b200 import _lib
    T = 4096
    g = torch.Generator().manual_seed(B * 7 + n_tok)
    table = torch.randint(0, ROWS, (ROWS, T), generator=g, dtype=torch.int32)
    src = _beam_src(B)
    row_len = None
    if with_len:
        lens = torch.randint(0, n_tok + 1, (B,), generator=g, dtype=torch.int32)
        lens[0], lens[-1] = 0, n_tok
        if B > 2:
            lens[1] = n_tok + 5 if n_tok + 5 <= T else n_tok
        row_len = lens
    want = table.clone()
    for b in range(B):
        n = n_tok if row_len is None else min(n_tok, int(row_len[b]))
        want[b, :n] = table[src[b], :n]
    dev = table.to(cuda)
    _lib.op_kv_indir_update(dev, torch.tensor(src, dtype=torch.int32, device=cuda), n_tok,
                            row_len=None if row_len is None else row_len.to(cuda))
    assert torch.equal(dev.cpu(), want)


@pytest.mark.parametrize("B,D", [(3, 128), (8, 64), (9, 128), (20, 128), (32, 64)])
def test_kv_reorder(cuda, B, D):
    """HF _reorder_cache in place over [outer = 2 x layers][Bcap][H][t_max][D], only the first B rows and the slots
    t < n_used_tokens; B <= 8 and B > 8 take different kernel instantiations."""
    from emu_b200 import _lib
    outer, Bcap, H, T, n_used = 2 * 3, B + 3, 4, 256, 201
    cache = _randn((outer, Bcap, H, T, D), 40, cuda)
    old = cache.clone()
    src = torch.tensor(_beam_src(B), dtype=torch.int32)
    _lib.op_kv_reorder(cache, src.to(cuda), n_used)
    want = old.clone()
    want[:, :B, :, :n_used] = old[:, :, :, :n_used].index_select(1, src.to(cuda).long())
    assert torch.equal(_bits(cache), _bits(want))


def test_kv_reorder_refuses_33_rows(cuda):
    from emu_b200 import _lib
    cache = torch.zeros(2, 33, 1, 16, 64, dtype=torch.bfloat16, device=cuda)
    with pytest.raises(_lib.EmuError, match="EMU_ERR_INVALID"):
        _lib.op_kv_reorder(cache, torch.arange(33, dtype=torch.int32, device=cuda), 8)


# ------------------------------------------------------------------------------------------------------------------------
# argmax_rows: first index of the maximum
# ------------------------------------------------------------------------------------------------------------------------
def _plant(x, kind):
    """x: one fp32 row (numpy, modified in place) with a planted maximum of the given kind"""
    cols = x.shape[0]
    top = float(np.abs(x).max()) + 1.0
    if kind == "float4 tie":            # two lanes of one 16-byte load
        i = min(4 * (cols // 8) + 1, cols - 2)
        x[i] = x[i + 1] = top
    elif kind == "warps tie":           # elements owned by different warps (and, for small rows, different threads)
        i, j = min(4 * 40 + 3, cols - 2), min(4 * 900, cols - 1)
        x[i] = x[j] = top
    elif kind == "same thread tie":     # one thread, successive trips of its loop
        i, j = min(4 * 5 + 2, cols - 2), min(4 * (5 + 1024) + 2, cols - 1)
        x[i] = x[j] = top
    elif kind == "ends tie":
        x[0] = x[cols - 1] = top
    elif kind == "last only":
        x[cols - 1] = top
    elif kind == "all -inf":
        x[:] = -np.inf
    elif kind == "+inf":
        x[cols // 3] = top
        x[min(cols // 2 + 1, cols - 1)] = np.inf
        x[cols - 1] = np.inf
    return x


ARGMAX_KINDS = ["float4 tie", "warps tie", "same thread tie", "ends tie", "last only", "all -inf", "+inf", "random"]


@pytest.mark.parametrize("cols", [32272, 16136, 1001, 5])
@pytest.mark.parametrize("rows", [1, 20, 32])
def test_argmax_rows_first_maximum(cuda, rows, cols):
    """Against numpy.argmax (documented to return the first occurrence), with the base aligned (float4 loads where cols
    allows) and offset by one float (the scalar loop)."""
    from emu_b200 import _lib
    rng = np.random.default_rng(rows * 100003 + cols)
    for shift in range(-(-len(ARGMAX_KINDS) // rows)):
        x = rng.standard_normal((rows, cols)).astype(np.float32)
        for r in range(rows):
            _plant(x[r], ARGMAX_KINDS[(r + shift * rows) % len(ARGMAX_KINDS)])
        want = np.argmax(x, axis=1)
        for off in (0, 1):
            buf = torch.empty(rows * cols + 4, dtype=torch.float32, device=cuda)
            view = buf[off:off + rows * cols].view(rows, cols)
            view.copy_(torch.from_numpy(x))
            got = _lib.op_argmax_rows(view).cpu().numpy()
            assert np.array_equal(got, want), (off, np.nonzero(got != want), got[got != want], want[got != want])


# ------------------------------------------------------------------------------------------------------------------------
# attn_prefill reading chosen cache rows (a join)
# ------------------------------------------------------------------------------------------------------------------------
def _prefill_reference(q, k, v, scale, causal, kv_start):
    """fp64 masked softmax attention, q [Nq,H,D], k/v [Nk,H,D] -> [Nq,H,D]"""
    Nq, Nk = q.shape[0], k.shape[0]
    s = torch.einsum("qhd,khd->hqk", q.double(), k.double()) * scale
    kj = torch.arange(Nk, device=q.device)[None, :]
    mask = kj < kv_start
    if causal:
        mask = mask | (kj > torch.arange(Nq, device=q.device)[:, None] + (Nk - Nq))
    s = s.masked_fill(mask[None], float("-inf"))
    return torch.einsum("hqk,khd->qhd", torch.softmax(s, dim=-1), v.double())


@pytest.mark.parametrize("Nq,extra,causal", [(128, 0, True), (128, 37, True), (300, 0, True), (300, 45, True),
                                             (300, 45, False), (40, 0, True), (40, 29, True), (40, 29, False)])
@pytest.mark.parametrize("H,D", [(52, 128), (2, 128)])
def test_attn_prefill_rows(cuda, H, D, Nq, extra, causal):
    """Query batch b reads K / V of cache row kv_row[b]; the K / V views span all 32 rows (kv_rows = 32, as the engine
    passes llm_max_batch).  Nq >= 128 runs the wgmma kernel, Nq = 40 the mma.sync kernel.  Every other row and the slots
    past Nk hold NaN; left padding before kv_start holds 1e4."""
    from emu_b200 import _lib
    B, T = 3, 384
    Nk = Nq + extra
    rows = torch.tensor([9, 2, 30], dtype=torch.int32, device=cuda)
    kv_start = torch.tensor([0, 5, min(70, Nk // 2)], dtype=torch.int32, device=cuda)
    scale = D ** -0.5
    q = _randn((B, Nq, H, D), 50, cuda)
    kc = torch.full((ROWS, H, T, D), NAN, dtype=torch.bfloat16, device=cuda)
    vc = kc.clone()
    for b in range(B):
        r, s = int(rows[b]), int(kv_start[b])
        kc[r, :, :Nk] = _randn((H, Nk, D), 51 + b, cuda)
        vc[r, :, :Nk] = _randn((H, Nk, D), 61 + b, cuda)
        kc[r, :, :s] = 1e4
        vc[r, :, :s] = 1e4
    kview, vview = kc.permute(0, 2, 1, 3)[:, :Nk], vc.permute(0, 2, 1, 3)[:, :Nk]      # [32, Nk, H, D] strided
    out = _lib.op_attn_prefill_rows(q, kview, vview, scale, causal=causal, kv_start=kv_start, kv_row=rows)
    assert torch.isfinite(out.float()).all(), "read a NaN slot: another row, or past Nk"
    for b in range(B):
        r, s = int(rows[b]), int(kv_start[b])
        ref = _prefill_reference(q[b], kview[r], vview[r], scale, causal, s)
        first = max(0, s - (Nk - Nq)) if causal else 0       # query rows that see at least one key
        err = _rel_err(out[b, first:], ref[first:])
        assert err < TOL_BF16, (b, err)
