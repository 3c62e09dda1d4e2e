"""The 3x3x3 tensor-core convolution with 128 output channels computes interior voxels only (csrc/conv_tc.cu): a
restatement of its block groups and operand windows, checked without a GPU.

A block is 8 y-lines x 8 z of one x plane (64 wgmma rows, 8-row groups rp apart); blocks are ordered z fastest, then y,
then x; a group is ib = 2 * tiles_per_item(N) consecutive blocks of one shape, and its operand window under tap group
dx runs from (x+dx-1, y0-1, z0-1) of its first block for stage_rows rows."""
import pytest

from tests.test_host_tables_cpu import _conv_items_sched1


def tiles_per_item(nt):
    return 4 if nt <= 32 else (2 if nt <= 64 else 1)


def block_row(k, rp, nzb, npl):
    x, rem = divmod(k, npl)
    yb, zb = divmod(rem, nzb)
    return ((x + 1) * rp + 1 + 8 * yb) * rp + 1 + 8 * zb


def geometry(r, nt):
    rp, nzb = r + 2, -(-r // 8)
    npl = nzb * nzb
    nblk, ib = r * npl, 2 * tiles_per_item(nt)
    wrows = max(block_row(min(f + ib, nblk) - 1, rp, nzb, npl) - block_row(f, rp, nzb, npl) + 9 * rp + 10
                for f in range(0, nblk, ib))
    return rp, nzb, npl, nblk, ib, wrows


def block_voxels(k, r, rp, nzb, npl):
    """(row, stored) for the block's 64 fragment rows: row i is (y0 + i // 8, z0 + i % 8)"""
    s, rem = block_row(k, rp, nzb, npl), k % npl
    y0, z0 = 1 + 8 * (rem // nzb), 1 + 8 * (rem % nzb)
    return [(s + (i // 8) * rp + i % 8, y0 + i // 8 <= r and z0 + i % 8 <= r) for i in range(64)]


@pytest.mark.parametrize("r", [8, 16, 32, 5, 12])
@pytest.mark.parametrize("nt", [128])
def test_groups_cover_interior_once_and_windows_hold_every_tap(r, nt):
    rp, nzb, npl, nblk, ib, wrows = geometry(r, nt)
    rows = rp ** 3
    interior = {((x + 1) * rp + y + 1) * rp + z + 1 for x in range(r) for y in range(r) for z in range(r)}
    stored = []
    for g in range(-(-nblk // ib)):
        f = g * ib
        blocks = range(f, min(f + ib, nblk))
        for k in blocks:
            vox = block_voxels(k, r, rp, nzb, npl)
            stored += [row for row, ok in vox if ok]
            for dx in range(3):
                w0 = block_row(f, rp, nzb, npl) - rp - 1 + (dx - 1) * rp * rp
                assert w0 >= 0
                for dy in range(3):
                    for dz in range(3):
                        for row, ok in vox:
                            src = row + (dx - 1) * rp * rp + (dy - 1) * rp + dz - 1
                            assert 0 <= src - w0 < wrows                  # inside the copied window
                            if ok:
                                assert src < rows                     # a stored row reads no row past the shape
    assert sorted(stored) == sorted(interior)                              # every interior voxel exactly once, no halo row


def test_window_sizes_of_the_step():
    # (r, N) -> rows per channel group of one stage
    assert geometry(8, 128)[5] == 2 * 10 * 10  # two whole x planes
    assert geometry(16, 128)[5] == 10 * 18     # 8 y-lines x 16 z
    assert geometry(32, 128)[5] == 9 * 34 + 18


def test_ring_depth_of_the_step():
    # conv_tc_run at N = 128: 16-channel chunks (KG = 4), 9-tap weight slabs of 72 KB, fixed tail (bias, statistics,
    # barriers, occupancy flags); at least 4 A stages beside 2 weight slabs
    nt, kg = 128, 4
    fixed = 128 * 4 + 8 * 2 * nt * 4 + 64 * 8 + 128 + 1024
    b_stage = 9 * kg * nt * 16
    for r in (8, 16):
        assert (227 * 1024 - fixed - 2 * b_stage) // (kg * geometry(r, nt)[5] * 16) >= 4, r


@pytest.mark.parametrize("r,nt,B", [(r, nt, B) for r in (8, 16, 32) for nt in (128,) for B in (1, 3, 32)])
def test_both_schedules_deal_every_group_once(r, nt, B):
    _, _, _, nblk, ib, _ = geometry(r, nt)
    ntile, n_nt, sms = -(-nblk // ib), 1, 132
    U = n_nt * B * ntile
    per_cta = -(-U // sms)
    grid = -(-U // per_cta)
    # sched 0: contiguous ranges, one group per item
    seen0 = [u for i in range(grid) for u in range(U * i // grid, U * (i + 1) // grid)]
    assert sorted(seen0) == list(range(U))
    # sched 1: rounds of adjacent groups
    seen1 = []
    for items in _conv_items_sched1(U, B * ntile, grid, 1):
        for _, v0, n in items:
            assert n == 1
            seen1.append(v0)
    assert sorted(seen1) == list(range(U))
