"""Float64 brute-force restatement of the JSD occupancy grid, and the seeded inputs of the score goldens
(tests/golden/make_golden_eval_metrics.py records the reference's outputs on them into ref_eval_metrics.npz).

TEST INFRASTRUCTURE ONLY: the library never imports this.

  occupancy   utils/evaluation_metrics_fast.py:604-647 (entropy_of_occupancy_grid): for every point the nearest
              cell by exact float64 squared distance (dx*dx + dy*dy) + dz*dz of the float32 inputs, lowest cell
              index on a tie; point_counts = the reference's grid_counters, cloud_counts = grid_bernoulli_rvars.
"""
import numpy as np
import torch

# occupancy cases: name -> (resolution, seed, clouds, points per cloud, kind)
OCC_CASES = {
    'r28_cube': (28, 11, 6, 1024, 'cube'),          # the unit cube, corners outside the sphere included
    'r28_far': (28, 12, 3, 500, 'far'),             # points up to ~2 away from the grid
    'r28_centres': (28, 13, 4, 300, 'centres'),     # half the points exactly on cell centres
    'r28_single': (28, 14, 1, 777, 'cube'),         # one cloud, ragged point count
    'r9': (9, 15, 5, 400, 'cube'),
    'r48': (48, 16, 3, 600, 'cube'),                # 54088 cells: 53 shared-memory chunks of the cell table
}
GRID_RESOLUTIONS = (9, 28, 48)
JSD_SEEDS = (21, 22)                                # sample set, reference set: 10 clouds of 512 points each
SCORE_SHAPES = (24, 20, 256)                        # samples, references, points per cloud


def grid_cells(resolution):
    """The in-sphere cell table, built independently of the library: float64 i / (r - 1) - 0.5 stored as float32,
    kept where the float32 norm is <= 0.5."""
    v = (np.arange(resolution) * (1.0 / float(resolution - 1)) - 0.5).astype(np.float32)
    g = np.stack(np.meshgrid(v, v, v, indexing='ij'), -1).reshape(-1, 3)
    return g[np.linalg.norm(g, axis=1) <= 0.5]


def occ_clouds(name):
    """float32 [S,N,3] clouds of an occupancy case."""
    res, seed, s, n, kind = OCC_CASES[name]
    rng = np.random.default_rng(seed)
    if kind == 'cube':
        return rng.uniform(-0.5, 0.5, (s, n, 3)).astype(np.float32)
    if kind == 'far':
        return (rng.standard_normal((s, n, 3)) * 0.8).astype(np.float32)
    x = rng.uniform(-0.45, 0.45, (s, n, 3)).astype(np.float32)
    cells = grid_cells(res)
    x[:, ::2] = cells[rng.integers(0, len(cells), (s, (n + 1) // 2))]
    return x


def jsd_sets():
    """(samples, references) float32 [10,512,3]: a ball of radius 0.45 against a flattened ellipsoid."""
    out = []
    for seed, squash in zip(JSD_SEEDS, (1.0, 0.5)):
        rng = np.random.default_rng(seed)
        d = rng.standard_normal((10, 512, 3))
        d /= np.linalg.norm(d, axis=2, keepdims=True)
        x = d * 0.45 * rng.uniform(0, 1, (10, 512, 1)) ** (1 / 3)
        x[..., 2] *= squash
        out.append(x.astype(np.float32))
    return out[0], out[1]


def score_sets():
    """(samples [24,256,3], references [20,256,3]) float32 torch tensors whose CD and EMD nearest neighbours are
    well separated: every cloud is its own random blob, scaled and shifted by a per-cloud amount, and the first
    twelve samples are noisy copies of references."""
    ns, nr, n = SCORE_SHAPES
    g = torch.Generator().manual_seed(31)
    blob = lambda k: torch.randn(k, n, 3, generator=g) * (0.05 + 0.25 * torch.rand(k, 1, 1, generator=g)) \
        + (torch.rand(k, 1, 3, generator=g) - 0.5) * 0.6
    refs = blob(nr)
    samples = blob(ns)
    samples[:12] = refs[torch.arange(12) * 3 % nr][:, torch.randperm(n, generator=g)] \
        + 0.03 * torch.randn(12, n, 3, generator=g)
    return samples, refs


def occupancy(clouds, cells):
    """clouds [S,N,3], cells [K,3] (float32) -> (point_counts [K], cloud_counts [K]) int64."""
    clouds = np.asarray(clouds, np.float32)
    c = np.asarray(cells, np.float32).astype(np.float64)
    k = len(c)
    point_counts = np.zeros(k, np.int64)
    cloud_counts = np.zeros(k, np.int64)
    for pc in clouds:
        p = pc.astype(np.float64)
        nearest = np.empty(len(p), np.int64)
        for a in range(0, len(p), 256):
            q = p[a:a + 256]
            dx = q[:, None, 0] - c[None, :, 0]
            dy = q[:, None, 1] - c[None, :, 1]
            dz = q[:, None, 2] - c[None, :, 2]
            nearest[a:a + 256] = np.argmin((dx * dx + dy * dy) + dz * dz, axis=1)    # first minimum
        point_counts += np.bincount(nearest, minlength=k)
        cloud_counts[np.unique(nearest)] += 1
    return point_counts, cloud_counts
