"""The score port's host side against the reference's outputs recorded in tests/golden/ref_eval_metrics.npz
(tests/golden/make_golden_eval_metrics.py): the JSD grid table, the float64 occupancy restatement, the entropy and
divergence, and knn / lgan_mmd_cov on CPU tensors."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from lion_b200.utils import evaluation_metrics_fast as E
from lion_b200.utils.data_helper import normalize_point_clouds
from lion_b200.utils.eval_helper import get_ref_num
from tests import eval_metrics_oracle as EO
from tests.golden import ref_import

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_eval_metrics.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.mark.parametrize("res", EO.GRID_RESOLUTIONS)
def test_grid_table_matches_reference_digest(golden, res):
    cells, spacing = E.unit_cube_grid_point_cloud(res, clip_sphere=True)
    assert cells.dtype == np.float32 and spacing == 1.0 / (res - 1)
    assert tuple(cells.shape) == tuple(golden["grid/%d/shape" % res])
    assert hashlib.sha256(cells.tobytes()).hexdigest() == str(golden["grid/%d/sha256" % res])
    assert np.array_equal(cells, EO.grid_cells(res))
    full, _ = E.unit_cube_grid_point_cloud(res)
    assert full.shape == (res, res, res, 3)


@pytest.mark.parametrize("name", list(EO.OCC_CASES))
def test_occupancy_oracle_equals_reference_counts(golden, name):
    res, _, s, _, _ = EO.OCC_CASES[name]
    pc, cc = EO.occupancy(EO.occ_clouds(name), EO.grid_cells(res))
    assert np.array_equal(pc, golden["occ/%s/point_counts" % name])
    assert np.array_equal(cc, golden["occ/%s/cloud_counts" % name])
    assert abs(E.occupancy_entropy(cc, s) - float(golden["occ/%s/entropy" % name])) <= 1e-12


def test_jsd_of_oracle_counts_matches_reference(golden):
    s, r = EO.jsd_sets()
    cells = EO.grid_cells(28)
    ps, pr = EO.occupancy(s, cells)[0], EO.occupancy(r, cells)[0]
    assert np.array_equal(ps, golden["jsd/sample_counts"]) and np.array_equal(pr, golden["jsd/ref_counts"])
    jsd = E.jensen_shannon_divergence(ps.astype(np.float64), pr.astype(np.float64))
    assert abs(jsd - float(golden["jsd/value"])) <= 1e-12


def test_jensen_shannon_divergence_errors():
    with pytest.raises(ValueError, match="Negative"):
        E.jensen_shannon_divergence(np.array([1.0, -1.0]), np.array([1.0, 1.0]))
    with pytest.raises(ValueError, match="Non equal"):
        E.jensen_shannon_divergence(np.array([1.0, 1.0]), np.array([1.0, 1.0, 1.0]))
    assert E.jensen_shannon_divergence(np.array([1.0, 3.0]), np.array([1.0, 3.0])) == 0.0


def _knn_inputs():
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_golden_eval_metrics as M
    return M


@pytest.mark.parametrize("k", [1, 3])
def test_knn_equals_reference(golden, k):
    out = E.knn(*_knn_inputs().knn_matrices(), k)
    keys = {key.split("/")[2] for key in golden if key.startswith("knn/k%d/" % k)}
    assert set(out) == keys
    for key, v in out.items():
        assert np.array_equal(v.numpy(), golden["knn/k%d/%s" % (k, key)]), key


def test_lgan_mmd_cov_equals_reference(golden):
    out = E.lgan_mmd_cov(_knn_inputs().mmd_cov_matrix())
    assert set(out) == {"lgan_mmd", "lgan_cov", "lgan_mmd_smp"}
    for key, v in out.items():
        assert np.array_equal(v.numpy(), golden["mmd_cov/%s" % key]), key


def test_result_line_columns(tmp_path):
    res = {'lgan_mmd-CD': 0.0012345, 'lgan_cov-CD': 0.5, '1-NN-CD-acc': 0.55, 'jsd': 0.0123}
    head, line = E.formulate_results(res, 'airplane', '-', '', 3)
    assert head == ['Dataset', 'reported', 'MMD-CDx0.001↓', 'MMD-EMDx0.01↓', 'COV-CD%↑', 'COV-EMD%↑',
                    '1-NNA-CD%↓', '1-NNA-EMD%↓', 'JSD↓']
    assert line == ['airplane', 'SE3', '1.2345', '0.0000', '50.00', '0.00', '55.00', '0.00', '0.01']
    out = tmp_path / "eval_out.csv"
    E.write_results(str(out), res, dataset='airplane')
    E.write_results(str(out), res, dataset='airplane')
    rows = [[c.strip() for c in r.split('\t')] for r in out.read_text().splitlines()]
    assert len(rows) == 4 and rows[0][:3] == ['Dataset', 'Model', 'MMD-CDx0.001↓'] and rows[2] == rows[0]
    assert rows[1][0] == 'airplane' and float(rows[1][2]) == 1.2345 and float(rows[1][4]) == 50.0
    assert 'MMD-CDx0.001' in E.print_results(res)


def test_normalize_point_clouds_and_ref_num():
    x = torch.rand(3, 50, 6) * torch.tensor([1.0, 2.0, 3.0, 1.0, 1.0, 1.0]) + 0.3
    out = torch.stack(normalize_point_clouds(x))
    assert torch.equal(out[..., 3:], x[..., 3:])
    lo, hi = out[..., :3].amin(1), out[..., :3].amax(1)
    assert torch.allclose((lo + hi) / 2, torch.zeros(3, 3), atol=1e-6)
    assert torch.allclose((hi - lo).amax(1), torch.full((3,), 2.0), atol=1e-6)
    assert get_ref_num('airplane') == 405 and get_ref_num('all') == 1000 and get_ref_num('car', luo_split=True) == 528
    with pytest.raises(AssertionError):
        get_ref_num('boat')


@pytest.mark.skipif(not ref_import.available(), reason="needs the reference checkout")
def test_golden_script_reproduces_the_npz(tmp_path):
    pytest.importorskip("sklearn")
    out = tmp_path / "again.npz"
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tests", "golden", "make_golden_eval_metrics.py"), str(out)])
    a, b = dict(np.load(GOLDEN)), dict(np.load(out))
    assert set(a) == set(b)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
