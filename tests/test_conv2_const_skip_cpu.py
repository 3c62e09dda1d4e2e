"""Class-valued blocks of the second 3x3x3 convolution of a PVConv (k_conv2_flags, conv_tc.cu: Params::cls_flag), without
a GPU: a restatement of k_conv2_flags -- per 64-row block of the row tiles' span, a test of the 27 neighbours of every
interior row in the sparse first convolution's activity mask -- checked against a numpy dilation of the occupancy grid
by two voxels, and a simulation of k_conv_tc's producer / consumer protocol when class-valued blocks leave tiles or
whole items without copies and a warpgroup without MMAs: it cannot deadlock on the rings conv_tc_run allows."""
import random

import numpy as np
import pytest
from scipy import ndimage

from tests.test_conv_weight_parts_cpu import layout


def activity_mask(occ):
    """k_sparse_conv_gather's mask: [r^3] bits (x-major, z fastest) of voxels with an occupied neighbour"""
    return ndimage.binary_dilation(occ, np.ones((3, 3, 3), bool)).reshape(-1)


def kernel_flags(mask, r):
    """k_conv2_flags, restated: flags of the 2 * ceil(r rp^2 / 128) blocks of rows rp^2 + 64 k .. + 63"""
    rp = r + 2
    p_end = (rp - 1) * rp * rp
    nblk = 2 * -(-(r * rp * rp) // 128)
    out = np.zeros(nblk, np.uint8)
    for k in range(nblk):
        hit = False
        for p in range(rp * rp + 64 * k, rp * rp + 64 * k + 64):
            x, y, z = p // (rp * rp), (p // rp) % rp, p % rp
            if p >= p_end or not (1 <= y <= r and 1 <= z <= r):
                continue
            for dx in (-1, 0, 1):
                for dy in (-1, 0, 1):
                    for dz in (-1, 0, 1):
                        xx, yy, zz = x + dx, y + dy, z + dz
                        if 1 <= xx <= r and 1 <= yy <= r and 1 <= zz <= r:
                            hit |= bool(mask[((xx - 1) * r + (yy - 1)) * r + (zz - 1)])
        out[k] = 0 if hit else 1
    return out


def dilation_flags(occ, r):
    """the same from the occupancy: no interior row within two voxels (Chebyshev) of an occupied one"""
    rp = r + 2
    near = np.zeros((rp, rp, rp), bool)
    near[1:-1, 1:-1, 1:-1] = ndimage.binary_dilation(occ, np.ones((5, 5, 5), bool))
    span = near.reshape(-1)[rp * rp:(rp - 1) * rp * rp]
    nblk = 2 * -(-span.size // 128)
    pad = np.zeros(nblk * 64, bool)
    pad[:span.size] = span
    return (~pad.reshape(nblk, 64).any(1)).astype(np.uint8)


def cloud(kind, r, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "gauss":
        c = rng.standard_normal((n, 3))
    elif kind == "surface":
        c = rng.standard_normal((n, 3))
        c /= np.linalg.norm(c, axis=1, keepdims=True)
    else:                                                     # one voxel and the six face centres
        c = np.zeros((n, 3))
        for i, (a, s) in enumerate([(a, s) for a in range(3) for s in (1.0, -1.0)]):
            c[i, a] = s
    c = c - c.mean(0)
    c = c / (2 * np.linalg.norm(c, axis=1).max()) + 0.5
    v = np.clip(np.rint(c * (r - 1)), 0, r - 1).astype(int)
    occ = np.zeros((r, r, r), bool)
    occ[v[:, 0], v[:, 1], v[:, 2]] = True
    return occ


@pytest.mark.parametrize("kind", ["gauss", "surface", "faces"])
@pytest.mark.parametrize("r,n", [(32, 2048), (16, 1024), (13, 500), (8, 64)])
def test_flags_match_dilation(kind, r, n):
    occ = cloud(kind, r, n, r * 7 + n)
    got = kernel_flags(activity_mask(occ), r)
    want = dilation_flags(occ, r)
    assert np.array_equal(got, want)
    assert got.sum() < got.size


def simulate(items, nchunk, ntg, a_depth, b_depth, drain=True):
    """k_conv_tc's row-tile protocol with class-valued blocks.  items: per item, per tile the pair of flags (block of
    warpgroup 0, of warpgroup 1).  The producer copies the weights of an item with a live tile (not both blocks
    flagged) and the A stages of its live tiles; each warpgroup waits for those stages, issues on the tiles whose own
    block is computed (one group in flight after wgmma.wait_group 1, released one group late), releases the others at
    once, and retires its MMAs at the end of every slab when it has a class-valued block in the item.  A ring slot is
    free once both warpgroups released it.  Returns False on a deadlock."""
    a_rel, b_rel = [{}, {}], [{}, {}]
    a_done, b_done = [0], [0]

    def freed(rel, n):
        return n in rel[0] and n in rel[1]

    def producer():
        na = nb = 0
        for tiles in items:
            live = [not (f0 and f1) for f0, f1 in tiles]
            if not any(live):
                continue
            for _ in range(nchunk * ntg):
                while nb - b_depth >= 0 and not freed(b_rel, nb - b_depth):
                    yield
                nb += 1
                b_done[0] = nb
                for j in range(len(tiles)):
                    if not live[j]:
                        continue
                    while na - a_depth >= 0 and not freed(a_rel, na - a_depth):
                        yield
                    na += 1
                    a_done[0] = na

    def consumer(wg):
        na = nb = 0
        ar, br = a_rel[wg], b_rel[wg]
        for tiles in items:
            live = [not (f0 and f1) for f0, f1 in tiles]
            mine = [not t[wg] for t in tiles]
            if not any(live):
                continue
            partial = drain and any(l and not m for l, m in zip(live, mine))
            pend_a = pend_b = None
            for _ in range(nchunk * ntg):
                while b_done[0] <= nb:
                    yield
                issued = False
                for j in range(len(tiles)):
                    if not live[j]:
                        continue
                    while a_done[0] <= na:
                        yield
                    if not mine[j]:
                        ar[na] = 1
                    else:
                        for x, rel in ((pend_a, ar), (pend_b, br)):
                            if x is not None:
                                rel[x] = 1
                        pend_a = na
                        pend_b = None
                        issued = True
                    na += 1
                if pend_b is not None:
                    for x, rel in ((pend_a, ar), (pend_b, br)):
                        if x is not None:
                            rel[x] = 1
                    pend_a = pend_b = None
                if issued:
                    pend_b = nb
                else:
                    br[nb] = 1
                if partial and pend_b is not None:
                    for x, rel in ((pend_a, ar), (pend_b, br)):
                        if x is not None:
                            rel[x] = 1
                    pend_a = pend_b = None
                nb += 1
            for x, rel in ((pend_a, ar), (pend_b, br)):
                if x is not None:
                    rel[x] = 1

    progs = [producer(), consumer(0), consumer(1)]
    done = [False] * 3
    while not all(done):
        moved = False
        for i, g in enumerate(progs):
            if done[i]:
                continue
            before = (a_done[0], b_done[0], sum(map(len, a_rel)), sum(map(len, b_rel)))
            try:
                next(g)
            except StopIteration:
                done[i] = True
                moved = True
            if (a_done[0], b_done[0], sum(map(len, a_rel)), sum(map(len, b_rel))) != before:
                moved = True
        if not moved:
            return False
    return True


# the row-tile second convolutions (cin = cout) at B = 32, also with the level-0 shared-memory cap beside the side stream,
# with TF32 operands and with FP16 ones (autocast: 8 channels per 16-byte group, so the tiling of cin / 2 TF32 channels)
@pytest.mark.parametrize("f16", [False, True])
@pytest.mark.parametrize("cap", [0, 196 * 1024])
@pytest.mark.parametrize("c,r", [(32, 32), (64, 32), (64, 16), (64, 13)])
def test_protocol_cannot_deadlock(c, r, cap, f16):
    cpg = 8 if f16 else 4
    L = layout(c * 4 // cpg, c, r, 32, cap=cap)
    assert L["ib"] == 0 and L["tps"] == 9 and L["a_stages"] >= L["G"]   # conv_tc_run's condition for the flags
    assert L["kg"] == ({32: 4, 64: 8}[c] if f16 else 8)                  # conv_tc_prepare_f16's KG
    nchunk = -(-(c // cpg) // L["kg"])
    rng = random.Random(c * 100 + r + cap + f16)
    for p_flag in (0.0, 0.2, 0.5, 0.8, 1.0):
        for _ in range(4):
            items = [[(rng.random() < p_flag, rng.random() < p_flag) for _ in range(rng.randint(1, L["G"]))] for _ in range(6)]
            assert simulate(items, nchunk, 3, L["a_stages"], L["b_stages"]), (L, items)
    # the worst case: one computed block per item and warpgroup, in its first or its last tile
    G = L["G"]
    for j in (0, G - 1):
        t = [(True, True)] * G
        t[j] = (False, True)
        t[G - 1 - j] = (t[G - 1 - j][0], False)
        assert simulate([t] * 4, nchunk, 3, L["a_stages"], L["b_stages"]), (L, t)


def test_protocol_needs_the_slab_drain():
    """without the per-slab retirement, a warpgroup that computes only the first of four live tiles holds that tile's A
    stage until the next slab's copy of it, which a ring of four stages cannot hold: the simulation finds the deadlock"""
    items = [[(False, False), (True, False), (True, False), (True, False)]] * 2
    assert simulate(items, 1, 3, 4, 2)
    assert not simulate(items, 1, 3, 4, 2, drain=False)
    assert simulate(items, 1, 3, 5, 2, drain=False)
