"""
The routing and dispatch kernels of csrc/moe.cu, one by one, against exact or fp64 host references: gate top-k with slot
ranking and failure injection, layout_exchange, scatter_rows, combine_rows and gate_bwd.  They run at world size 1, where
the rank's own symmetric heap is its only peer.  Two whole-layer cases cover the configurations nothing else compares with
an oracle: the benchmark's default emulator gate (bf16 logits, so ties are common) and failure injection.

The CPU tests check the host references themselves.
"""
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lah_b200  # noqa: F401
from lah_b200.ops import kernels as K
from routing_support import F64, rel, slots
from routing_support import rt, world1  # noqa: F401 (fixtures)

GAMMA = 0x9E3779B97F4A7C15
LAYOUT_MAX_E = 4096
BF16 = torch.bfloat16


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_splitmix64_ref_matches_the_published_sequence():
    """the first outputs of a splitmix64 generator seeded with 0 are hash(0), hash(gamma), hash(2 gamma)"""
    x = np.array([0, GAMMA, (2 * GAMMA) % 2 ** 64], dtype=np.uint64)
    assert [int(v) for v in K.splitmix64_ref(x)] == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]


@pytest.mark.parametrize("rate", [0.1, 0.5, 0.9])
def test_gate_fail_mask_ref_rate_and_key(rate):
    B, E, seed = 4096, 64, 1337 * 7919 + 3
    m = K.gate_fail_mask_ref(B, E, rate, seed, 2 ** 33 + 5)
    assert m.shape == (B, E) and m.dtype == torch.bool
    n = B * E
    assert abs(m.float().mean().item() - rate) <= 5 * (rate * (1 - rate) / n) ** 0.5
    # a row depends on token_offset + b only, and the seed changes it
    assert torch.equal(K.gate_fail_mask_ref(B - 1, E, rate, seed, 2 ** 33 + 6), m[1:])
    assert not torch.equal(K.gate_fail_mask_ref(B, E, rate, seed + 1, 2 ** 33 + 5), m)
    # one draw by hand: key = seed ^ (token * FNV prime + expert), 24 high bits of the hash against the float32 rate
    b, e = 17, 40
    key = (seed ^ (((2 ** 33 + 5 + b) * 0x100000001B3 + e) % 2 ** 64)) % 2 ** 64
    u = (int(K.splitmix64_ref(np.array([key], dtype=np.uint64))[0]) >> 40) / 2 ** 24
    assert bool(m[b, e]) == (u < float(np.float32(rate)))


def test_gate_topk_ref_breaks_ties_toward_the_smaller_expert_id():
    logits = torch.tensor([[1.0, 3.0, 3.0, 2.0, 3.0, 3.0]])
    idx, w = K.gate_topk_ref(logits, (6,), 3)
    assert idx.tolist() == [[1, 2, 4]] and torch.allclose(w, torch.full((1, 3), 1 / 3))
    alive = torch.tensor([1, 1, 0, 1, 1, 1], dtype=torch.uint8)
    assert K.gate_topk_ref(logits, (6,), 3, alive=alive)[0].tolist() == [[1, 4, 5]]
    # a 2-d grid: scores [[1, 1, 0], [2, 2, 1]] flattened row-major
    idx, _ = K.gate_topk_ref(torch.tensor([[0.0, 1.0, 1.0, 1.0, 0.0]]), (2, 3), 3)
    assert idx.tolist() == [[3, 4, 0]]
    # every score tied: the k smallest ids, in order
    assert K.gate_topk_ref(torch.zeros(2, 7), (7,), 4)[0].tolist() == [[0, 1, 2, 3]] * 2
    # fewer alive experts than k (and k larger than the grid): missing slots are -1 with weight 0
    idx, w = K.gate_topk_ref(torch.tensor([[5.0, 5.0]]), (2,), 4, alive=torch.tensor([0, 1]))
    assert idx.tolist() == [[1, -1, -1, -1]] and w.tolist() == [[1.0, 0.0, 0.0, 0.0]]


# ---------------------------------------------------------------------------------------------------------------- GPU
def rows_view(w, rows, H):
    """[rows, H] bf16 at the start of the receive region, and its byte offset in the heap"""
    return w.region[: rows * H * 2].view(BF16).view(rows, H), w.region_off


def set_token_base(w, base):
    w.step_ctr[2:4].view(torch.int64).fill_(base)


def emulator_logits(B, E, gen):
    """the arithmetic of FusedDMoE.gate_logits on CUDA: bf16 LayerNorm, bf16 GEMM with normalised keys -> bf16 values"""
    x = torch.randn(B, 512, generator=gen).to(BF16).cuda()
    keys = F.normalize(torch.randn(512, E, generator=gen), dim=-1).to(BF16).cuda()
    xn = F.layer_norm(x, (512,), torch.ones(512, dtype=BF16, device="cuda"), torch.zeros(512, dtype=BF16, device="cuda"))
    return (xn @ keys).float()


def make_logits(kind, B, grid, gen):
    total = sum(grid)
    if kind == "emulator":
        return emulator_logits(B, total, gen)
    if kind == "bf16":   # 1-d and 2-d grids: the kernel's and the oracle's score sums agree exactly
        return torch.randn(B, total, generator=gen).to(BF16).float().cuda()
    # 3-d and 4-d grids sum in a different order; quarter integers are exact in any order (and tie often)
    return (torch.randint(-12, 13, (B, total), generator=gen).float() / 4).cuda()


def make_alive(kind, E, k, gen):
    if kind == "all":
        return None
    if kind == "dead30":
        return (torch.rand(E, generator=gen) > 0.3).to(torch.uint8).cuda()
    a = torch.zeros(E, dtype=torch.uint8)
    if kind == "fewer_than_k":
        a[torch.randperm(E, generator=gen)[: k - 1]] = 1
    return a.cuda()


def run_gate(logits, grid, k, counts0, **kw):
    B = logits.shape[0]
    idx = torch.full((B * k,), 12345, dtype=torch.int32, device="cuda")
    pos = torch.full_like(idx, 12345)
    w = torch.full((B * k,), 7.0, device="cuda")
    counts = counts0.clone()
    K.gate_topk(logits, grid, k, idx=idx, w=w, pos=pos, counts=counts, **kw)
    torch.cuda.synchronize()
    return idx.view(B, k).long(), w.view(B, k), pos.view(B, k).long(), counts.long()


def check_gate_against_ref(logits, grid, k, alive, fail_mask, out, counts0):
    """idx, counts and pos exact; missing slots -1 / 0 / 0; w within 1e-6 of the fp64 softmax of the selected scores"""
    idx, w, pos, counts = out
    E = int(np.prod(grid))
    ridx, _ = K.gate_topk_ref(logits, grid, k, alive=alive, fail_mask=fail_mask)
    assert torch.equal(idx, ridx), int((idx != ridx).any(1).sum())
    valid = ridx >= 0
    exp_counts = counts0.long() + torch.bincount(ridx[valid], minlength=E)
    assert torch.equal(counts, exp_counts)
    assert torch.equal(pos.cpu(), slots(ridx).cpu())
    scores = K.product_key_scores(logits, grid).double()
    sel = torch.gather(scores, 1, ridx.clamp(min=0)).masked_fill(~valid, float("-inf"))
    w_ref = torch.where(valid, torch.softmax(sel, dim=-1), torch.zeros_like(sel)).nan_to_num(0.0)
    assert bool((w[~valid] == 0).all()) and bool((pos[~valid] == 0).all())
    werr = (w.double() - w_ref).abs().max().item() if w.numel() else 0.0
    assert werr < 1e-6, werr
    return ridx, werr


GATE_GRIDS = [((64,), 4, "emulator"), ((1024,), 4, "bf16"), ((2048,), 4, "bf16"), ((4096,), 4, "bf16"),
              ((16,), 8, "bf16"), ((2, 32), 8, "bf16"), ((3, 5, 7), 4, "dyadic"), ((2, 3, 4, 5), 6, "dyadic")]


@pytest.mark.gpu
@pytest.mark.parametrize("alive_kind", ["all", "dead30", "fewer_than_k", "none"])
@pytest.mark.parametrize("B", [1, 7, 1001, 4096])
@pytest.mark.parametrize("grid,k,kind", GATE_GRIDS, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else str(v))
def test_gate_topk_is_exact(rt, record_property, grid, k, kind, B, alive_kind):
    """exact top-k with equal scores taking the smaller expert id, per-expert slots in token-major order (B * k > 1024 makes
    rank_slots_kernel loop), accumulating counts, and the softmax weights.  Dense gates over 2048 and 4096 experts need
    more than 48 KB of shared memory per CTA"""
    gen = torch.Generator().manual_seed(zlib.crc32(repr((grid, k, B, alive_kind)).encode()))
    E = int(np.prod(grid))
    logits = make_logits(kind, B, grid, gen)
    alive = make_alive(alive_kind, E, k, gen)
    counts0 = torch.randint(0, 50, (E,), generator=gen, dtype=torch.int32).cuda()
    out = run_gate(logits, grid, k, counts0, alive=alive)
    ridx, werr = check_gate_against_ref(logits, grid, k, alive, None, out, counts0)
    record_property("w_max_abs_err", werr)
    n_alive = E if alive is None else int(alive.sum())
    assert bool(((ridx >= 0).sum(1) == min(k, n_alive)).all())


@pytest.mark.gpu
def test_gate_topk_rejects_bad_arguments(rt):
    logits = torch.zeros(4, 16, device="cuda")
    i = torch.zeros(4 * 9, dtype=torch.int32, device="cuda")
    with pytest.raises(rt.native.NativeError):
        K.gate_topk(logits, (16,), 9, idx=i, w=i.float(), pos=i, counts=torch.zeros(16, dtype=torch.int32, device="cuda"))
    big = torch.zeros(1, LAYOUT_MAX_E + 1, device="cuda")
    with pytest.raises(rt.native.NativeError):
        K.gate_topk(big, (LAYOUT_MAX_E + 1,), 4, idx=i, w=i.float(), pos=i,
                    counts=torch.zeros(LAYOUT_MAX_E + 1, dtype=torch.int32, device="cuda"))


@pytest.mark.gpu
@pytest.mark.parametrize("grid,k,rate,B,token_offset,base", [
    ((64,), 4, 0.1, 1001, 0, 0),
    ((64,), 4, 0.1, 4096, 2 ** 32 + 17, 0),
    ((16,), 4, 0.9, 1001, 5, 2 ** 33 + 3),        # fewer than k survivors for most tokens
    ((4, 4), 4, 0.5, 512, 2 ** 40, 2 ** 35),
    ((2, 32), 8, 0.3, 7, 123, 456),
], ids=["e64_r0.1", "e64_r0.1_offset2^32", "e16_r0.9_base", "4x4_r0.5_offset_base", "2x32_k8_r0.3"])
def test_gate_failure_injection_is_exact(rt, grid, k, rate, B, token_offset, base):
    """the dropped (token, expert) pairs are exactly gate_fail_mask_ref's, keyed on token_offset + the device token base"""
    gen = torch.Generator().manual_seed(B + k)
    E = int(np.prod(grid))
    seed = 0xDEADBEEFCAFEF00D
    logits = make_logits("bf16", B, grid, gen)
    alive = make_alive("dead30", E, k, gen)
    counts0 = torch.zeros(E, dtype=torch.int32, device="cuda")
    set_token_base(rt, base)
    out = run_gate(logits, grid, k, counts0, alive=alive, failure_rate=rate, seed=seed, token_offset=token_offset)
    fail = K.gate_fail_mask_ref(B, E, rate, seed, token_offset + base).cuda()
    ridx, _ = check_gate_against_ref(logits, grid, k, alive, fail, out, counts0)
    assert not torch.equal(ridx, K.gate_topk_ref(logits, grid, k, alive=alive)[0])   # the failures changed the routing


@pytest.mark.gpu
def test_gate_token_base_counts_like_token_offset(rt):
    """the device token base (what a captured CUDA graph advances between replays) and the token_offset argument add up"""
    gen = torch.Generator().manual_seed(5)
    logits = make_logits("bf16", 300, (64,), gen)
    zeros = torch.zeros(64, dtype=torch.int32, device="cuda")
    kw = dict(failure_rate=0.3, seed=99)
    T = 2 ** 34 + 77
    set_token_base(rt, 0)
    a = run_gate(logits, (64,), 4, zeros, token_offset=T, **kw)
    set_token_base(rt, T)
    b = run_gate(logits, (64,), 4, zeros, token_offset=0, **kw)
    set_token_base(rt, T - 1000)
    c = run_gate(logits, (64,), 4, zeros, token_offset=1000, **kw)
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, z)


# ------------------------------------------------------------------------------------------------ layout_exchange
def layout_oracle(counts, align, tile_rows, max_rows):
    """world-1 layout: groups in expert order, each padded to `align` rows; tiles of `tile_rows` rows name their group"""
    c = counts.long().cpu()
    padded = (c + align - 1) // align * align
    off = torch.cumsum(padded, 0) - padded
    total = int(padded.sum())
    max_tiles = max_rows // tile_rows
    tile_group = torch.full((max_tiles,), -1, dtype=torch.long)
    tiles = torch.repeat_interleave(torch.arange(len(c)), padded // tile_rows)[:max_tiles]
    tile_group[: len(tiles)] = tiles
    return dict(dst_row=off, group_off=torch.cat([off, torch.tensor([total])]), group_rows=c, tile_group=tile_group,
                total_rows=torch.tensor([total]), step_rows=c, route_owner=torch.zeros_like(c), overflow=total > max_rows)


def layout_counts(kind, gen):
    if kind == "sparse":
        c = torch.randint(0, 40, (64,), generator=gen) * (torch.rand(64, generator=gen) > 0.5)
    elif kind == "hot":
        c = torch.zeros(16, dtype=torch.long)
        c[5], c[0], c[15] = 1000, 3, 17
    elif kind == "e4096":
        c = torch.randint(0, 3, (LAYOUT_MAX_E,), generator=gen)
    else:
        c = torch.zeros(32, dtype=torch.long)
    return c.to(torch.int32)


CANARY = -777


def canaried(n, fill):
    """int32 output array of n entries followed by 8 canary entries"""
    t = torch.full((n + 8,), CANARY, dtype=torch.int32, device="cuda")
    t[:n] = fill
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("overflow", [False, True])
@pytest.mark.parametrize("kind", ["sparse", "hot", "e4096", "empty"])
@pytest.mark.parametrize("align,tile_rows", [(16, 16), (128, 128), (256, 128)])
def test_layout_exchange_matches_oracle(rt, align, tile_rows, kind, overflow):
    """every table exact against the Python layout (tiles outside the groups -1), nothing written past any table, the slot
    counters zeroed, the counts published with the epoch flag, and STATUS_OVERFLOW when the groups exceed max_rows"""
    gen = torch.Generator().manual_seed(align + len(kind))
    counts = layout_counts(kind, gen)
    E = counts.numel()
    total = int(((counts.long() + align - 1) // align * align).sum())
    if overflow and total < 2 * align:
        pytest.skip("nothing to overflow")
    max_rows = total - align if overflow else total + 3 * align
    ref = layout_oracle(counts, align, tile_rows, max_rows)
    max_tiles = max_rows // tile_rows
    cnt = counts.cuda()
    out = dict(dst_row=canaried(E, 4242), group_off=canaried(E + 1, 4242), group_rows=canaried(E, 4242),
               tile_group=canaried(max_tiles, 4242), total_rows=canaried(1, 4242), step_rows=canaried(E, 4242),
               route_owner=canaried(E, 4242), owned_shadow=canaried(2 * E, 4242))
    rt.step_ctr[0] = 1 << 20
    K.layout_exchange(rt.cnt_all_off, rt.flags_off, K.SLOT_COUNTS, 3, E, E, max_rows, align=align, tile_rows=tile_rows,
                      counts=cnt, status=rt.status, shadow_slots=0, **out)
    torch.cuda.synchronize()
    for name, t in out.items():
        n = t.numel() - 8
        assert bool((t[n:] == CANARY).all()), f"{name}: canary overwritten"
        if name == "owned_shadow":
            assert torch.equal(t[:n].view(E, 2).cpu(), torch.tensor([[-1, 0]] * E, dtype=torch.int32)), name
        else:
            assert torch.equal(t[:n].long().cpu(), ref[name]), name
    assert bool((cnt == 0).all()), "the slot counters must be left zeroed"
    assert torch.equal(rt.cnt_all[0, :E].cpu(), counts), "published counts"
    assert int(rt.flags[K.SLOT_COUNTS, 0]) == (1 << 20) + 3
    assert int(rt.status[0]) == (K.STATUS_OVERFLOW if ref["overflow"] else 0)


# ------------------------------------------------------------------------------------------------ scatter_rows
def routed_pairs(B, k, E, gen, drop=0.1):
    """distinct experts per token, ~drop of the slots without an expert"""
    idx = torch.argsort(torch.rand(B, E, generator=gen), dim=1)[:, :k]
    idx[torch.rand(B, k, generator=gen) < drop] = -1
    return idx


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fits", "overflow"])
@pytest.mark.parametrize("mode", ["forward", "backward"])
@pytest.mark.parametrize("H,align", [(256, 16), (512, 128), (1024, 256)])
def test_scatter_rows(rt, H, align, mode, case):
    """every routed row lands bit-exact at dst_row[e] + pos (backward: the gradient row times the gate weight, rounded to
    bf16); padding rows are zeroed; rows after the groups, and the canary rows after the buffer, keep their contents"""
    gen = torch.Generator().manual_seed(H + align + len(mode) + len(case))
    B, k, E = 301, 4, 16
    idx = routed_pairs(B, k, E, gen)
    pos = slots(idx).flatten()
    counts = torch.bincount(idx[idx >= 0], minlength=E).to(torch.int32)
    total = int(((counts.long() + align - 1) // align * align).sum())
    max_rows = total - 2 * align if case == "overflow" else total + 2 * align
    lay = layout_oracle(counts, align, align, max_rows)
    row = torch.where(idx.flatten() >= 0, lay["dst_row"][idx.flatten().clamp(min=0)] + pos, torch.full_like(pos, -1))
    row = torch.where(row < max_rows, row, torch.full_like(row, -1))
    canary_rows = 64
    buf, off = rows_view(rt, max_rows + canary_rows, H)
    buf.copy_(torch.randn(max_rows + canary_rows, H, generator=gen).to(BF16))
    before = buf.clone()
    src = torch.randn(B, H, generator=gen).to(BF16).cuda()
    w = torch.rand(B * k, generator=gen).cuda()
    d = lambda t: t.to(torch.int32).cuda()   # noqa: E731
    idx_d, pos_d = d(idx.flatten()), d(pos)
    rt.step_ctr[0] = 5000
    if mode == "forward":
        pair_row = torch.full((B * k,), 999999, dtype=torch.int32, device="cuda")
        K.scatter_rows(src, None, idx_d, pos_d, d(lay["dst_row"]), pair_row, off, rt.flags_off, K.SLOT_DISPATCH, 7, k, E,
                       max_rows, d(lay["group_off"]), d(lay["group_rows"]), rt.done_counter, rt.status, align=align,
                       route_owner=torch.zeros(E, dtype=torch.int32, device="cuda"), num_groups=E)
        slot = K.SLOT_DISPATCH
    else:
        pair_row = d(row)
        K.scatter_rows(src, w, idx_d, pos_d, None, pair_row, off, rt.flags_off, K.SLOT_GRAD, 7, k, E, max_rows,
                       d(lay["group_off"]), d(lay["group_rows"]), rt.done_counter, rt.status, align=align, num_groups=E)
        slot = K.SLOT_GRAD
    torch.cuda.synchronize()
    assert torch.equal(pair_row.long().cpu(), row)
    got = buf.cpu()
    exp = before.cpu().clone()
    p = torch.nonzero(row >= 0).squeeze(1)
    sent = src.cpu()[p // k]
    if mode == "backward":
        sent = (sent.float() * w.cpu()[p].unsqueeze(1)).to(BF16)
    exp[row[p]] = sent
    for e in range(E):
        r0 = int(lay["group_off"][e] + counts[e])
        r1 = min(max_rows, int(lay["group_off"][e] + (counts[e] + align - 1) // align * align))
        if r1 > r0:
            exp[r0:r1] = 0
    bad = (got.view(torch.int16) != exp.view(torch.int16)).any(1).nonzero().squeeze(1)
    assert bad.numel() == 0, f"{bad.numel()} rows differ, first {bad[:8].tolist()} (max_rows {max_rows}, total {total})"
    assert int(rt.flags[slot, 0]) == 5007
    assert int(rt.done_counter) == 0
    assert int(rt.status[0]) == (K.STATUS_OVERFLOW if case == "overflow" and mode == "forward" else 0)


@pytest.mark.gpu
def test_scatter_rows_rejects_unsupported_width(rt):
    src = torch.zeros(8, 768, dtype=BF16, device="cuda")
    i = torch.zeros(8, dtype=torch.int32, device="cuda")
    with pytest.raises(rt.native.NativeError):
        K.scatter_rows(src, None, i, i, i, i, rt.region_off, rt.flags_off, K.SLOT_DISPATCH, 1, 1, 1, 64, i, i,
                       rt.done_counter, rt.status)


# ------------------------------------------------------------------------------------------------ combine_rows
def bf16_ulp(x):
    """spacing of bf16 numbers at |x| (x float64)"""
    _, e = torch.frexp(x.abs().clamp(min=2.0 ** -126))
    return torch.pow(2.0, (e - 8).to(x.dtype))


def pairs_with_rows(B, k, E, R, gen):
    """routed pairs with distinct receive rows; some slots without an expert, some routed pairs without a row (dropped by
    scatter_rows), and token 0 with no pair at all"""
    idx = routed_pairs(B, k, E, gen, drop=0.15)
    pair_row = torch.randperm(R, generator=gen)[: B * k].view(B, k)
    pair_row[torch.rand(B, k, generator=gen) < 0.05] = -1
    idx[0] = -1
    pair_row = torch.where(idx >= 0, pair_row, torch.full_like(pair_row, -1))
    return idx, pair_row


@pytest.mark.gpu
@pytest.mark.parametrize("weighted", [True, False])
@pytest.mark.parametrize("H", [256, 512, 1024])
@pytest.mark.parametrize("k", [1, 4, 8])
def test_combine_rows(rt, record_property, k, H, weighted):
    """out[b] = sum_j w_j src[pair_row[b, j]] within one bf16 ulp of the fp64 sum, plus the bound of fp32 accumulation
    (which only matters where the terms cancel)"""
    gen = torch.Generator().manual_seed(k * H + weighted)
    B, E = 333, 16
    R = B * k + 100
    idx, pair_row = pairs_with_rows(B, k, E, R, gen)
    src, off = rows_view(rt, R, H)
    src.copy_(torch.randn(R, H, generator=gen).to(BF16))
    w = torch.rand(B, k, generator=gen) if weighted else None
    out = torch.full((B, H), 3.0, dtype=BF16, device="cuda")
    K.combine_rows(off, idx.flatten().to(torch.int32).cuda(), pair_row.flatten().to(torch.int32).cuda(),
                   w.flatten().cuda() if weighted else None, out, k, E)
    torch.cuda.synchronize()
    present = (pair_row >= 0).double()
    terms = src.cpu().double()[pair_row.clamp(min=0)] * (present * (w.double() if weighted else 1.0)).unsqueeze(-1)
    ref = terms.sum(1)
    tol = bf16_ulp(ref) + k * 2.0 ** -23 * terms.abs().sum(1)
    err = (out.cpu().double() - ref.to(BF16).double()).abs()
    record_property("max_err_ulp", (err / bf16_ulp(ref)).max().item())
    assert bool((err <= tol).all()), f"max error {(err / bf16_ulp(ref)).max().item():.2f} ulp"
    assert bool((out[0] == 0).all()) and not bool(torch.signbit(out[0].float()).any()), "a token with no pair"


# ------------------------------------------------------------------------------------------------ gate_bwd
@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 4, 8])
@pytest.mark.parametrize("grid,H", [((64,), 256), ((4, 4), 512), ((2, 32), 1024), ((3, 5, 7), 512)])
def test_gate_bwd(rt, record_property, grid, H, k):
    """dlogits against fp64 autograd of sum_j w_j <g, y_j>, w = softmax over the selected scores.  Missing slots (no
    expert) have no weight; a selected pair dropped by scatter_rows (no row) keeps its weight with y_j = 0.  Experts of a
    grid share coordinates, so several slots add into one logit"""
    gen = torch.Generator().manual_seed(k * H + len(grid))
    B = 257
    E = int(np.prod(grid))
    logits = torch.randn(B, sum(grid), generator=gen, dtype=torch.float64)
    idx = K.gate_topk_ref(logits.float(), grid, k)[0]
    idx[torch.rand(B, k, generator=gen) < 0.15] = -1
    R = B * k + 50
    pair_row = torch.randperm(R, generator=gen)[: B * k].view(B, k)
    pair_row[torch.rand(B, k, generator=gen) < 0.05] = -1
    pair_row = torch.where(idx >= 0, pair_row, torch.full_like(pair_row, -1))
    yo, off = rows_view(rt, R, H)
    yo.copy_(torch.randn(R, H, generator=gen).to(BF16))
    g = torch.randn(B, H, generator=gen).to(BF16)
    # fp64 oracle
    lg = logits.clone().requires_grad_(True)
    valid = idx >= 0
    sel = torch.gather(K.product_key_scores(lg, grid), 1, idx.clamp(min=0)).masked_fill(~valid, float("-inf"))
    wts = torch.where(valid, torch.softmax(sel, dim=-1), torch.zeros_like(sel)).nan_to_num(0.0)
    y = yo.cpu().double()[pair_row.clamp(min=0)] * (pair_row >= 0).double().unsqueeze(-1)
    (wts * (g.double().unsqueeze(1) * y).sum(-1)).sum().backward()
    dl = torch.full((B, sum(grid)), 5.0, device="cuda")
    K.gate_bwd(off, g.cuda(), idx.flatten().to(torch.int32).cuda(), pair_row.flatten().to(torch.int32).cuda(),
               wts.detach().float().flatten().cuda(), dl, k, E, grid)
    torch.cuda.synchronize()
    if k == 1:
        assert bool((dl == 0).all())
    else:
        err = rel(dl.cpu(), lg.grad, *F64)
        record_property("rel_l2_err", err)
        assert err < 1e-4, err


# ------------------------------------------------------------------------------------------------ whole layer
def gate_ties(logits, k):
    """(tokens whose k-th and (k+1)-th best scores are equal, tokens with equal scores among their k + 1 best)"""
    top = torch.sort(logits, dim=-1, descending=True).values[:, : k + 1]
    return int((top[:, k - 1] == top[:, k]).sum()), int((top[:, 1:] == top[:, :-1]).any(1).sum())


@pytest.mark.gpu
def test_bench_default_layer_matches_oracle_on_tied_bf16_logits(record_property):
    """the configuration bench.py reports (emulator gate over 64 experts, k = 4, hidden 512, small expert path): the fused
    layer's routing equals the oracle's exactly on the same bf16-valued logits, ties included; y, dx and dlogits within
    check_layer_small's tolerances"""
    from lah_b200.parallel import engine as E
    cfg = E.DMoEConfig(hidden=512, grid_size=(64,), k=4, num_layers=1, tokens_per_rank=256, gate_mode="emulator",
                       expert_path="small", lr=1e-3)
    torch.manual_seed(0)
    ctx = E.EngineContext(cfg)
    try:
        layer = E.FusedDMoE(cfg, ctx).cuda()
        B = 256
        gen = torch.Generator().manual_seed(11)
        x = torch.randn(B, 512, generator=gen).to(BF16).cuda()
        gy = torch.randn(B, 512, generator=gen).to(BF16).cuda()
        logits = layer.gate_logits(x).detach()
        assert torch.equal(logits, logits.to(BF16).float())
        boundary, any_tie = gate_ties(logits, cfg.k)
        print(f"\nemulator gate, {B} tokens: {boundary} tie(s) between the 4th and 5th score, {any_tie} token(s) with a tie "
              f"in their top 5")
        record_property("ties", dict(boundary=boundary, top5=any_tie))
        assert any_tie > 0, "the case must exercise ties"
        ridx = K.gate_topk_ref(logits, cfg.grid_size, cfg.k, alive=ctx.alive)[0]
        # oracle first: the fused backward updates the experts in place
        xr, lr_ = x.float().requires_grad_(True), logits.clone().requires_grad_(True)
        yr = layer._forward_ref(xr, lr_)
        yr.backward(gy.float())
        xf, lf = x.clone().requires_grad_(True), logits.clone().requires_grad_(True)
        y = E._FusedDMoEFunction.apply(xf, lf, layer)
        idx = layer.ws.idx[: B * cfg.k].view(B, cfg.k).long().clone()
        y.backward(gy)
        torch.cuda.synchronize()
        ctx.check_status()
        assert torch.equal(idx, ridx), int((idx != ridx).any(1).sum())
        errs = dict(y=rel(y, yr, *F64), dx=rel(xf.grad, xr.grad, *F64), dlogits=rel(lf.grad, lr_.grad, *F64))
        record_property("errors", errs)
        assert errs["y"] < 2e-2 and errs["dx"] < 3e-2 and errs["dlogits"] < 5e-2, errs
    finally:
        ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rate", [0.1, 0.5])
def test_failure_injected_layer_matches_oracle(record_property, rate):
    """product-key gate (4, 4) with failure injection in training mode: the fused layer drops exactly the pairs of
    gate_fail_mask_ref (seed cfg.seed * 7919 + layer index, token offset = device token base + ctx.token_counter), and y,
    dx and the proj gradient meet check_layer's tolerances.  In eval mode nothing fails."""
    from lah_b200.parallel import engine as E
    cfg = E.DMoEConfig(hidden=512, grid_size=(4, 4), k=4, num_layers=2, tokens_per_rank=512, lr=1e-3, failure_rate=rate,
                       expert_path="big")
    torch.manual_seed(3)
    ctx = E.EngineContext(cfg)
    try:
        layer = E.FusedDMoE(cfg, ctx, layer_index=1).cuda()
        B, Ex = 512, cfg.num_experts
        gen = torch.Generator().manual_seed(int(rate * 100))
        x = torch.randn(B, 512, generator=gen).to(BF16).cuda()
        gy = torch.randn(B, 512, generator=gen).to(BF16).cuda()
        ctx.begin_step()                       # a non-zero device token base
        layer.eval()
        with torch.no_grad():
            layer(x)                           # eval: no failures, and ctx.token_counter moves on
            torch.cuda.synchronize()
            logits = layer.gate_logits(x, layer.proj)
        assert torch.equal(layer.ws.idx[: B * cfg.k].view(B, cfg.k).long(),
                           K.gate_topk_ref(logits, cfg.grid_size, cfg.k, alive=ctx.alive)[0])
        layer.train()
        base = int(ctx.step_ctr[2:4].view(torch.int64).item())
        assert base > 0 and ctx.token_counter == B
        fail = K.gate_fail_mask_ref(B, Ex, rate, cfg.seed * 7919 + layer.layer_index, base + ctx.token_counter).cuda()
        layer.ref_fail_mask = fail
        ridx = K.gate_topk_ref(logits, cfg.grid_size, cfg.k, alive=ctx.alive, fail_mask=fail)[0]
        # oracle first: the fused backward updates the experts in place
        xr = x.float().requires_grad_(True)
        lr_ = F.linear(xr, layer.proj.weight.detach(), layer.proj.bias.detach())
        lr_.retain_grad()
        assert torch.equal(lr_.detach(), logits)
        yr = layer._forward_ref(xr, lr_)
        yr.backward(gy.float())
        dproj_ref = lr_.grad.t() @ xr.detach()
        xf = x.clone().requires_grad_(True)
        y = layer(xf)
        idx = layer.ws.idx[: B * cfg.k].view(B, cfg.k).long().clone()
        y.backward(gy)
        torch.cuda.synchronize()
        ctx.check_status()
        assert torch.equal(idx, ridx), int((idx != ridx).any(1).sum())
        assert int((ridx < 0).sum()) > 0 or rate < 0.5
        errs = dict(y=rel(y, yr, *F64), dx=rel(xf.grad, xr.grad, *F64),
                    dproj=rel(layer.proj.weight.grad, dproj_ref, *F64))
        record_property("errors", errs)
        assert errs["y"] < 2e-2 and errs["dx"] < 3e-2 and errs["dproj"] < 5e-2, errs
    finally:
        ctx.close()
