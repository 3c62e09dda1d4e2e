"""Record the reference's score outputs (utils/evaluation_metrics_fast.py) into tests/golden/ref_eval_metrics.npz.

Runs on the CPU against an unmodified reference checkout (tests/golden/ref_import.py).  The reference's Chamfer
extension would JIT-build into its own tree at import, so third_party.ChamferDistancePytorch.* is stubbed; the
recorded functions do not call it.  Inputs are rebuilt from the seeds in tests/eval_metrics_oracle.py; only outputs
are stored:
  grid/<r>/...        shape and SHA-256 of unit_cube_grid_point_cloud(r, clip_sphere=True)[0]
  occ/<case>/...      entropy_of_occupancy_grid's grid counts (point_counts), its per-cloud occupancy
                      (cloud_counts, from the same NearestNeighbors query) and entropy
  jsd/...             jsd_between_point_cloud_sets and both sets' grid counters at resolution 28
  knn/k<k>/<key>      knn(Mxx, Mxy, Myy, k) on seeded matrices without ties; mmd_cov/<key>: lgan_mmd_cov
  all/<key>           compute_all_metrics on score_sets(), its _pairwise_EMD_CD_ patched to the float64 CPU
                      restatements in oracle/metrics.py

    python tests/golden/make_golden_eval_metrics.py [out.npz]
"""
import hashlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests.golden import ref_import  # noqa: E402
from tests import eval_metrics_oracle as EO  # noqa: E402

OUT = os.path.join(HERE, "ref_eval_metrics.npz")


def import_reference():
    ref_import.install()
    for name in ("third_party.ChamferDistancePytorch", "third_party.ChamferDistancePytorch.chamfer3D",
                 "third_party.ChamferDistancePytorch.chamfer3D.dist_chamfer_3D"):
        if name not in sys.modules:
            ref_import._stub(name)
    import utils.evaluation_metrics_fast as ref
    return ref


def knn_matrices():
    g = torch.Generator().manual_seed(41)
    return torch.rand(7, 7, generator=g), torch.rand(7, 9, generator=g), torch.rand(9, 9, generator=g)


def mmd_cov_matrix():
    return torch.rand(11, 8, generator=torch.Generator().manual_seed(42))


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def occupancy_reference(ref, clouds, resolution):
    """The reference's entropy_of_occupancy_grid, plus grid_bernoulli_rvars (its per-cloud counts) obtained from the
    same NearestNeighbors query the function makes."""
    from sklearn.neighbors import NearestNeighbors
    ent, point_counts = ref.entropy_of_occupancy_grid(clouds, resolution, True)
    cells, _ = ref.unit_cube_grid_point_cloud(resolution, True)
    nn = NearestNeighbors(n_neighbors=1).fit(cells.reshape(-1, 3))
    cloud_counts = np.zeros(len(cells))
    for pc in clouds:
        cloud_counts[np.unique(nn.kneighbors(pc)[1])] += 1
    return ent, point_counts, cloud_counts


def pairwise_oracle(metric, a, b, batch_size, **kw):
    from oracle import metrics as OM
    a, b = a.numpy(), b.numpy()
    if metric == 'CD':
        m = OM.pairwise_cd(a, b)
    else:
        m = np.array([OM.emd_approx(np.repeat(a[i:i + 1], len(b), 0), b) for i in range(len(a))]) / a.shape[1]
    m = torch.from_numpy(m).float()
    return m, m


def record():
    ref = import_reference()
    out = {}
    for r in EO.GRID_RESOLUTIONS:
        cells, spacing = ref.unit_cube_grid_point_cloud(r, True)
        out["grid/%d/shape" % r] = np.array(cells.shape)
        out["grid/%d/sha256" % r] = np.array(digest(cells))
    for name, (res, *_rest) in EO.OCC_CASES.items():
        ent, pc, cc = occupancy_reference(ref, EO.occ_clouds(name), res)
        out["occ/%s/point_counts" % name] = pc.astype(np.int64)
        out["occ/%s/cloud_counts" % name] = cc.astype(np.int64)
        out["occ/%s/entropy" % name] = np.array(ent)
    s, r = EO.jsd_sets()
    out["jsd/value"] = np.array(ref.jsd_between_point_cloud_sets(s, r, resolution=28))
    out["jsd/sample_counts"] = ref.entropy_of_occupancy_grid(s, 28, True)[1].astype(np.int64)
    out["jsd/ref_counts"] = ref.entropy_of_occupancy_grid(r, 28, True)[1].astype(np.int64)
    for k in (1, 3):
        for key, v in ref.knn(*knn_matrices(), k).items():
            out["knn/k%d/%s" % (k, key)] = v.numpy()
    for key, v in ref.lgan_mmd_cov(mmd_cov_matrix()).items():
        out["mmd_cov/%s" % key] = v.numpy()
    ref._pairwise_EMD_CD_ = pairwise_oracle
    samples, refs = EO.score_sets()
    for key, v in ref.compute_all_metrics(samples, refs, 8, verbose=False).items():
        out["all/%s" % key] = np.array(v)
    return out


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else OUT
    np.savez_compressed(path, **record())
    print("wrote", path)
