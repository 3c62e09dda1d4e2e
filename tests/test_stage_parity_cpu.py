"""CPU side of the stage tests (tests/test_stage_parity_gpu.py): the clouds reach the occupancies they are built for
(the oracle's voxel indices), and the TF32 operand models are the bit-level operations they claim to be."""
import numpy as np
import pytest
import torch

from tests import stage_ref as SR


@pytest.mark.parametrize("K,N,r", [(127, 2048, 32), (128, 2048, 32), (129, 2048, 32), (256, 2048, 32), (127, 1024, 16),
                                   (128, 1024, 16), (129, 1024, 16), (256, 1024, 16), (129, 700, 32), (256, 4096, 32)])
def test_sites_cloud_occupancy(K, N, r):
    c = SR.sites_cloud(K, N, r, seed=K + N + r)
    assert c.shape == (3, N)
    assert SR.occupancy(c[None], r) == [K]


@pytest.mark.parametrize("N,r", [(2048, 32), (4096, 32), (1024, 16), (500, 13), (64, 8)])
def test_clustered_cloud_occupancy(N, r):
    c = SR.clustered_cloud(N)
    ids = SR.voxel_ids(c[None], r)[0]
    vals, counts = torch.unique(ids, return_counts=True)
    assert len(vals) == 7 and int(counts.max()) == N - 6
    xyz = torch.stack([ids[-6:] // (r * r), ids[-6:] // r % r, ids[-6:] % r], 1)
    for k in range(6):                                        # each extreme point sits on a face of the grid
        assert int(xyz[k, k // 2]) == (r - 1 if k % 2 == 0 else 0)


def test_gaussian_cloud_is_spread():
    occ = SR.occupancy(SR.gaussian_cloud(3, 2048)[None], 32)[0]
    assert 1000 < occ <= 2048


def _tf32_bits_reference(x, mode):
    """Rounding of float32 values to 10 mantissa bits, computed from frexp in float64."""
    x = x.numpy().astype(np.float64)
    m, e = np.frexp(np.abs(x))                  # |x| = m * 2^e, m in [0.5, 1)
    q = m * 2.0 ** 11                           # 11 significant bits: 1 implicit + 10
    q = np.floor(q) if mode == "trunc" else np.floor(q + 0.5)
    return torch.from_numpy((np.sign(x) * np.ldexp(q / 2.0 ** 11, e)).astype(np.float32))


def test_tf32_operand_models_match_their_definitions():
    g = torch.Generator().manual_seed(5)
    x = torch.cat([torch.randn(100000, generator=g) * 10 ** torch.randint(-6, 6, (100000,), generator=g).float(),
                   torch.tensor([1.0, -1.0, 1.0 + 2 ** -11, -(1.0 + 2 ** -11), 1.0 + 3 * 2 ** -11, 1.5 - 2 ** -23, 0.0])])
    assert torch.equal(SR.tf32_trunc(x), _tf32_bits_reference(x, "trunc"))
    assert torch.equal(SR.tf32_rna(x), _tf32_bits_reference(x, "rna"))
    # ties go away from zero; truncation goes toward zero
    assert SR.tf32_rna(torch.tensor([1.0 + 2 ** -11, -(1.0 + 2 ** -11)])).tolist() == [1.0 + 2 ** -10, -(1.0 + 2 ** -10)]
    assert SR.tf32_trunc(torch.tensor([1.0 + 2 ** -10 - 2 ** -23])).tolist() == [1.0]


def test_scatter_grid_model_is_the_fused_multiply_add_chain():
    """scatter_grid = f0 * (1/n), then fma(f_k, 1/n, acc) over the voxel's points in ascending order."""
    g = torch.Generator().manual_seed(6)
    feats = torch.randn(1, 3, 50, generator=g)
    ids = torch.randint(0, 4, (1, 50), generator=g)
    grid = SR.scatter_grid(feats, ids, 2).view(3, 8)
    for v in range(8):
        pts = (ids[0] == v).nonzero().flatten().tolist()
        for c in range(3):
            if not pts:
                assert grid[c, v] == 0
                continue
            inv = np.float32(1.0) / np.float32(len(pts))
            acc = np.float32(feats[0, c, pts[0]].item()) * inv
            for k in pts[1:]:
                acc = np.float32(np.float64(feats[0, c, k].item()) * np.float64(inv) + np.float64(acc))
            assert grid[c, v].item() == acc
