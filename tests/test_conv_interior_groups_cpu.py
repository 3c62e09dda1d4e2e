"""4-block groups of the 128-channel 3x3x3 convolution (csrc/conv_tc.cu, conv_tc_run): the restatement of the block
groups and operand windows in test_conv_interior_cpu.py, for groups of ib = 4 consecutive blocks (two per consumer
warpgroup), and the rule that chooses them.  Checked without a GPU."""
import pytest

from tests.test_conv_interior_cpu import block_row, block_voxels

NT, KG = 128, 4                                       # N = 128 runs 16-channel chunks
FIXED = 128 * 4 + 8 * 2 * NT * 4 + 64 * 8 + 128 + 1024  # bias, statistics, barriers, occupancy flags
B_STAGE = 9 * KG * NT * 16                            # one 9-tap weight slab, 72 KB
SMEM = 227 * 1024


def geometry(r, ib):
    rp, nzb = r + 2, -(-r // 8)
    npl = nzb * nzb
    nblk = r * npl
    wrows = max(block_row(min(f + ib, nblk) - 1, rp, nzb, npl) - block_row(f, rp, nzb, npl) + 9 * rp + 10
                for f in range(0, nblk, ib))
    return rp, nzb, npl, nblk, wrows


def a_stages(r, ib):
    return (SMEM - FIXED - 2 * B_STAGE) // (KG * geometry(r, ib)[4] * 16)


def blocks_per_group(r, B, n_tiles=1, sms=132):
    """conv_tc_run: 4-block groups while there are as many groups as SMs and the window leaves 3 A stages"""
    nblk = geometry(r, 4)[3]
    return 4 if n_tiles * B * -(-nblk // 4) >= sms and a_stages(r, 4) >= 3 else 2


@pytest.mark.parametrize("r", [16, 13, 8, 32, 5, 12])
def test_four_block_groups_cover_interior_once_and_windows_hold_every_tap(r):
    rp, nzb, npl, nblk, wrows = geometry(r, 4)
    rows = rp ** 3
    interior = {((x + 1) * rp + y + 1) * rp + z + 1 for x in range(r) for y in range(r) for z in range(r)}
    stored = []
    for g in range(-(-nblk // 4)):
        f = 4 * g
        nb = min(4, nblk - f)
        for wg in range(2):                               # warpgroup wg takes blocks wg and wg + 2 of the group
            nbw = (nb - wg + 1) // 2
            assert nbw == len([j for j in range(2) if 2 * j + wg < nb])
            for j in range(nbw):
                k = f + 2 * j + wg
                vox = block_voxels(k, r, rp, nzb, npl)
                stored += [row for row, ok in vox if ok]
                for dx in range(3):
                    w0 = block_row(f, rp, nzb, npl) - rp - 1 + (dx - 1) * rp * rp
                    assert w0 >= 0
                    for dy in range(3):
                        for dz in range(3):
                            for row, ok in vox:
                                src = row + (dx - 1) * rp * rp + (dy - 1) * rp + dz - 1
                                assert 0 <= src - w0 < wrows          # inside the copied window
                                if ok:
                                    assert src < rows             # a stored row reads no row past the shape
    assert sorted(stored) == sorted(interior)                          # every interior voxel exactly once, no halo row


def test_window_and_ring_of_four_block_groups():
    assert geometry(16, 4)[4] == 18 * 18                  # one whole haloed x-plane
    assert geometry(13, 4)[4] == 273
    assert KG * geometry(16, 4)[4] * 16 == 20736          # bytes of one A stage
    assert a_stages(16, 4) == 3                           # beside 2 weight slabs: one A stage more than slabs
    assert SMEM - FIXED - 2 * B_STAGE - 3 * 20736 >= 0


def test_group_size_choice():
    # B = 32 on 132 SMs: r = 16 has 512 groups of 4, r = 8 would have 64 (half the SMs idle)
    assert blocks_per_group(16, 32) == 4
    assert blocks_per_group(13, 32) == 4
    assert blocks_per_group(8, 32) == 2
    assert blocks_per_group(16, 1) == 2 and blocks_per_group(13, 1) == 2
    # many shapes at r = 8: a 4-block window (four x-planes) leaves only 2 A stages, 2-block groups stay
    assert a_stages(8, 4) == 2 and blocks_per_group(8, 1000) == 2
    # the 3x3x3 grids of the project (r <= 32) always leave room for the ring of the group size they take
    for r in range(3, 33):
        for B in (1, 3, 32, 256):
            assert a_stages(r, blocks_per_group(r, B)) >= 2, (r, B)
