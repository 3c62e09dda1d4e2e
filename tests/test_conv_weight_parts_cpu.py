"""3x3x3 weight slabs streamed in 3-tap parts (csrc/conv_tc.cu): a restatement of conv_tc_run's choice between whole
weight slabs and 3-tap parts (block groups only) and of the shared-memory layout it leads to, for every 3x3x3 shape of
the prior's step, and checks of the pipeline it runs -- every accumulator takes its taps in the same order in both
modes, and the producer / consumer protocol of the two rings cannot deadlock, with or without occupancy skips, also
for row tiles in parts (which conv_tc_run does not take).  No GPU needed."""
import random

import pytest

from tests.test_conv_interior_cpu import block_row

SMEM = 227 * 1024
CAP_BESIDE_AUX = 196 * 1024        # net.cu: what a level-0 convolution may claim while the side stream runs
SMS = 132                          # H100 SXM


def tiling(cin, cout, r, B, sms=SMS):
    """conv_tc_prepare / conv_tc_run: (NT, KG, items' tiles G, blocks per group ib or 0, A stage bytes, fixed bytes)"""
    nt = cout if cout < 128 else 128
    g = cin // 4
    kg = 4 if nt > 64 else 8
    if g < kg:
        kg = 2 if g <= 2 else (4 if g <= 4 else 8)
    fixed = 128 * 4 + 8 * 2 * nt * 4 + 64 * 8 + 128 + 1024
    slab = 9 * kg * nt * 16
    if nt == 128:                                     # interior blocks
        rp, nzb = r + 2, -(-r // 8)
        npl = nzb * nzb
        nblk = r * npl

        def window(ib):
            return max(block_row(min(f + ib, nblk) - 1, rp, nzb, npl) - block_row(f, rp, nzb, npl) + 9 * rp + 10
                       for f in range(0, nblk, ib))
        four = (cout // nt) * B * -(-nblk // 4) >= sms and (SMEM - fixed - 2 * slab) // (kg * window(4) * 16) >= 3
        ib = 4 if four else 2
        return nt, kg, 1, ib, kg * window(ib) * 16, fixed
    G = 4 if nt <= 32 else 2
    return nt, kg, G, 0, kg * (128 + 2 * (r + 3)) * 16, fixed


def ring(tps, nt, kg, blk, a_stage, fixed, cap=0):
    """conv_tc_run's ring(): (weight stages, A stages) beside weight stages of tps taps"""
    stage = tps * kg * nt * 16
    b = 2 if tps == 9 else 4
    if blk and tps == 9:
        limit = (cap or SMEM) - fixed
        while b < 4 and (limit - (b + 1) * stage) // a_stage >= max(4, b + 1):
            b += 1
    a = (SMEM - fixed - b * stage) // a_stage
    if cap and a >= 5:
        capped = (cap - fixed - b * stage) // a_stage
        if 4 <= capped < a:
            a = capped
    a = min(a, 16)
    return b, (a if a >= 2 else 0)


def layout(cin, cout, r, B, cap=0, whole=False, sms=SMS, row_parts=False):
    """row_parts: also consider 3-tap parts for row tiles (2 G A stages), which conv_tc_run does not"""
    nt, kg, G, ib, a_stage, fixed = tiling(cin, cout, r, B, sms)
    blk = ib > 0
    b9, a9 = ring(9, nt, kg, blk, a_stage, fixed, cap)
    b3, a3 = ring(3, nt, kg, blk, a_stage, fixed, cap) if (blk or row_parts) and not whole else (0, 0)
    parts = a3 > a9 and a3 >= (G + 1 if blk else 2 * G)
    tps, b, a = (3, b3, a3) if parts else (9, b9, a9)
    assert a >= 2
    smem = a * a_stage + b * tps * kg * nt * 16 + fixed
    return dict(tps=tps, b_stages=b, a_stages=a, a_whole=a9, G=G, ib=ib, smem=smem, kg=kg, nt=nt)


def expected_taps(cin, cout, r, B, sms=SMS):
    return layout(cin, cout, r, B, sms=sms)["tps"]


# every 3x3x3 convolution of the prior's step: (cin, cout, r) -> (taps per weight stage, A stages) at B = 32
STEP = {
    (4, 32, 32): (9, 16), (32, 32, 32): (9, 6),   # row tiles keep whole slabs
    (128, 64, 16): (9, 3), (64, 64, 16): (9, 3), (64, 64, 32): (9, 3),
    (192, 128, 8): (3, 9), (128, 128, 8): (3, 9),  # 2-block groups: 5 A stages with whole slabs
    (128, 128, 16): (3, 5),                       # 4-block groups: 3 A stages with whole slabs
}
# what parts would give the row tiles (see the comment in conv_tc_run for why they are not taken)
ROW_PARTS = {(4, 32, 32): (9, 16), (32, 32, 32): (9, 6), (128, 64, 16): (3, 6), (64, 64, 16): (3, 6), (64, 64, 32): (3, 5)}


@pytest.mark.parametrize("shape", sorted(STEP))
def test_step_shapes_choose_the_deeper_ring(shape):
    L = layout(*shape, 32)
    assert (L["tps"], L["a_stages"]) == STEP[shape]
    assert L["smem"] <= SMEM
    if L["tps"] == 3:
        assert L["a_stages"] > L["a_whole"]


@pytest.mark.parametrize("shape", sorted(ROW_PARTS))
def test_row_tile_parts_restated(shape):
    L = layout(*shape, 32, row_parts=True)
    assert (L["tps"], L["a_stages"]) == ROW_PARTS[shape] and L["smem"] <= SMEM


def test_block_groups_gain_a_stages():
    assert layout(128, 128, 8, 32)["a_whole"] == 5 and layout(128, 128, 8, 32)["a_stages"] == 9
    assert layout(128, 128, 16, 32)["a_whole"] == 3 and layout(128, 128, 16, 32)["a_stages"] == 5
    assert layout(128, 128, 16, 32)["ib"] == 4


@pytest.mark.parametrize("cin,cout", [(4, 32), (32, 32)])
def test_level0_shapes_fit_beside_the_side_stream(cin, cout):
    L = layout(cin, cout, 32, 32, cap=CAP_BESIDE_AUX)
    assert L["smem"] <= CAP_BESIDE_AUX and L["tps"] == 9


@pytest.mark.parametrize("cin,cout,r,B", [(c, o, r, B) for (c, o, _) in STEP for r in (13, 16, 32, 5) for B in (1, 3, 32)])
@pytest.mark.parametrize("cap", [0, CAP_BESIDE_AUX])
def test_layout_fits_and_ring_invariants(cin, cout, r, B, cap):
    L = layout(cin, cout, r, B, cap=cap)
    assert L["smem"] <= SMEM
    if L["tps"] == 3:
        assert L["b_stages"] >= 3 + 1                   # the 3 parts of the slab in use and one being copied
        assert L["a_stages"] >= (L["G"] + 1 if L["ib"] else 2 * L["G"])
        assert L["a_stages"] > L["a_whole"]
        if cap and layout(cin, cout, r, B, cap=cap, whole=True)["smem"] <= cap:
            # where whole slabs honour the cap, parts do too unless the ring would drop below 4
            assert L["smem"] <= cap or L["a_stages"] <= 4 or L["a_whole"] < 4
    assert layout(cin, cout, r, B, cap=cap, whole=True)["tps"] == 9


def issue_order(nchunk, ntg, ntile, tps, kg):
    """the consumer's wgmma sequence of one item: (tile, chunk, x-plane, tap, k-step) in issue order"""
    seq = []
    for cc in range(nchunk):
        for tg in range(ntg):
            for s in range(9 // tps):
                for j in range(ntile):
                    for u in range(tps // 3):
                        for t in range(3):
                            for ks in range(kg // 2):
                                seq.append((j, cc, tg, s * tps + u * 3 + t, ks))
    return seq


@pytest.mark.parametrize("G,kg,nchunk", [(2, 8, 2), (4, 8, 1), (1, 4, 4), (2, 8, 16)])
def test_every_accumulator_takes_taps_in_order_in_both_modes(G, kg, nchunk):
    per_acc = {}
    for tps in (9, 3):
        seq = issue_order(nchunk, 3, G, tps, kg)
        for j in range(G):
            mine = [x[1:] for x in seq if x[0] == j]
            # chunks, x-planes, taps 0 .. 8 and k-steps in lexicographic order
            assert mine == sorted(mine)
            assert [x[2] for x in mine[:9 * (kg // 2)]] == [t for t in range(9) for _ in range(kg // 2)]
            per_acc.setdefault(j, []).append(mine)
    for j, (a, b) in per_acc.items():
        assert a == b


def simulate(items, nchunk, ntg, nparts, a_depth, b_depth, skip_of):
    """Runs k_conv_tc's producer and consumer protocol (one group in flight after wgmma.wait_group 1, releases one
    group late, the skip path) as two interleaved sequential programs; returns False on a deadlock."""
    a_rel, b_rel = set(), set()                       # released ring uses
    a_done, b_done = [0], [0]                         # uses the producer has filled

    def producer():
        na = nb = 0
        for ntile in items:
            for k in range(nchunk * ntg):
                for s in range(nparts):
                    if s == 1:
                        for j in range(ntile):
                            while na - a_depth >= 0 and na - a_depth not in a_rel:
                                yield
                            na += 1
                            a_done[0] = na
                    while nb - b_depth >= 0 and nb - b_depth not in b_rel:
                        yield
                    nb += 1
                    b_done[0] = nb
                if nparts == 1:
                    for j in range(ntile):
                        while na - a_depth >= 0 and na - a_depth not in a_rel:
                            yield
                        na += 1
                        a_done[0] = na

    def consumer():
        na = nb = 0
        for ntile in items:
            pend_a = pend_b = None
            for k in range(nchunk * ntg):
                last_slab = k == nchunk * ntg - 1
                skip = [False] * ntile
                for s in range(nparts):
                    while b_done[0] <= nb:
                        yield
                    issued = False
                    for j in range(ntile):
                        if s == 0:
                            while a_done[0] <= na + j:
                                yield
                            skip[j] = skip_of(na + j) and not last_slab
                            if skip[j]:
                                a_rel.add(na + j)
                        if not skip[j]:
                            for x, rel in ((pend_a, a_rel), (pend_b, b_rel)):
                                if x is not None:
                                    rel.add(x)
                            pend_a = pend_b = None
                            if s == nparts - 1:
                                pend_a = na + j
                            issued = True
                    if pend_b is not None:
                        for x, rel in ((pend_a, a_rel), (pend_b, b_rel)):
                            if x is not None:
                                rel.add(x)
                        pend_a = pend_b = None
                    if issued:
                        pend_b = nb
                    else:
                        b_rel.add(nb)
                    nb += 1
                na += ntile
            for x, rel in ((pend_a, a_rel), (pend_b, b_rel)):
                if x is not None:
                    rel.add(x)

    p, c = producer(), consumer()
    p_end = c_end = False
    while not (p_end and c_end):
        moved = False
        for which in (0, 1):
            g = p if which == 0 else c
            if (p_end, c_end)[which]:
                continue
            before = (a_done[0], b_done[0], len(a_rel), len(b_rel))
            try:
                next(g)
            except StopIteration:
                if which == 0:
                    p_end = True
                else:
                    c_end = True
                moved = True
            if (a_done[0], b_done[0], len(a_rel), len(b_rel)) != before:
                moved = True
        if not moved:
            return False
    return True


# the layouts above with the (producer-side) occupancy skip of sparse first convolutions
CASES = [(cin, cout, r, B) for (cin, cout, _) in STEP for r in (13, 16, 32) for B in (1, 32)]


@pytest.mark.parametrize("row_parts", [False, True])
@pytest.mark.parametrize("cin,cout,r,B", CASES)
def test_pipeline_protocol_cannot_deadlock(cin, cout, r, B, row_parts):
    L = layout(cin, cout, r, B, row_parts=row_parts)
    occ = L["ib"] > 0 or L["a_stages"] >= 2 * L["G"]   # conv_tc_run drops the row tiles' flags on shallower rings
    rng = random.Random(cin * 1000 + cout * 10 + r + B)
    nchunk = -(-(cin // 4) // L["kg"])
    for trial in range(6):
        items = [rng.randint(1, L["G"]) for _ in range(5)]
        p_skip = (0.0, 0.3, 0.7, 1.0, 0.5, 0.9)[trial]
        flags = {}

        def skip_of(n):
            if not occ:
                return False
            if n not in flags:
                flags[n] = rng.random() < p_skip
            return flags[n]
        nparts = 9 // L["tps"]
        assert simulate(items, nchunk, 3, nparts, L["a_stages"], L["b_stages"], skip_of), (L, items, p_skip)


def test_protocol_needs_the_ring_invariants():
    """the simulation does find a deadlock: 3-tap parts on an A ring shallower than an item's tiles"""
    assert not simulate([4, 4], 1, 3, 3, 3, 4, lambda n: False)
    assert simulate([4, 4], 1, 3, 3, 4, 4, lambda n: False)
    assert simulate([4, 4], 1, 3, 3, 8, 4, lambda n: n % 3 == 0)
