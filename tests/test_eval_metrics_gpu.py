"""Generation scores on the GPU: lion_occupancy_grid and the JSD against the reference's recorded outputs
(tests/golden/ref_eval_metrics.npz) and the float64 restatement (tests/eval_metrics_oracle.py); the matrix blocks of
compute_all_metrics against separate pairwise calls; MMD / COV / 1-NNA against the reference's compute_all_metrics on
the CPU oracle's matrices; compute_score end to end."""
import numpy as np
import pytest
import torch

from lion_b200 import _lib as L
from lion_b200.utils import evaluation_metrics_fast as E
from lion_b200.utils.data_helper import normalize_point_clouds
from lion_b200.utils.eval_helper import compute_score
from tests import eval_metrics_oracle as EO
from tests.test_eval_metrics_cpu import GOLDEN
from tests.util import gen

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.mark.parametrize("name", list(EO.OCC_CASES))
def test_occupancy_kernel_equals_reference_counts(golden, name):
    res, _, s, n, _ = EO.OCC_CASES[name]
    clouds = EO.occ_clouds(name)
    cells, _ = E.unit_cube_grid_point_cloud(res, clip_sphere=True)
    pc, cc = E.occupancy_counts(clouds, cells)
    assert pc.dtype == np.int32 and pc.shape == (len(cells),)
    assert np.array_equal(pc, golden["occ/%s/point_counts" % name]) and pc.sum() == s * n
    assert np.array_equal(cc, golden["occ/%s/cloud_counts" % name]) and cc.max() <= s
    again = E.occupancy_counts(torch.from_numpy(clouds).cuda(), cells)
    assert np.array_equal(again[0], pc) and np.array_equal(again[1], cc), "occupancy counts are not reproducible"
    ent, counts = E.entropy_of_occupancy_grid(clouds, res, in_sphere=True)
    assert abs(ent - float(golden["occ/%s/entropy" % name])) <= 1e-12 and np.array_equal(counts, pc)


def test_occupancy_kernel_ties_and_oracle():
    """Exact ties go to the lowest cell index, also against a duplicate cell in a later shared-memory chunk; and a
    larger seeded case against the float64 restatement."""
    cells = np.zeros((2500, 3), np.float32)
    cells[:, 0] = np.arange(2500, dtype=np.float32) + 10.0        # far away, never nearest
    cells[3] = (0, 0, 0)
    cells[7] = (1, 0, 0)
    cells[2100] = (0, 0, 0)                                        # duplicate of cell 3 in the third chunk
    pts = np.array([[[0.5, 0, 0], [0, 0, 0], [1, 0, 0], [0.5, 0.25, 0]]], np.float32)
    pc, cc = E.occupancy_counts(pts, cells)
    assert pc[3] == 3 and pc[7] == 1 and pc.sum() == 4 and cc[3] == 1 and cc[7] == 1 and cc.sum() == 2
    x = np.random.default_rng(5).uniform(-0.6, 0.6, (7, 1500, 3)).astype(np.float32)
    cells = EO.grid_cells(20)
    got, want = E.occupancy_counts(x, cells), EO.occupancy(x, cells)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def test_occupancy_rejects_bad_arguments():
    lib = L.lib()
    buf = torch.zeros(64, dtype=torch.int32, device="cuda")
    p = L.ptr(buf)
    assert lib.lion_occupancy_grid(None, p, 1, 1, 1, p, p, L.stream()) != 0
    assert lib.lion_occupancy_grid(p, p, 1, 0, 1, p, p, L.stream()) != 0
    assert lib.lion_occupancy_grid(p, p, 65536, 65536, 1, p, p, L.stream()) != 0       # S * N > INT_MAX
    assert b"INT_MAX" in lib.lion_last_error()
    assert lib.lion_occupancy_grid(p, p, 1, 1, 2_000_000, p, p, L.stream()) != 0       # bitmap beyond shared memory
    torch.cuda.synchronize()
    assert torch.count_nonzero(buf) == 0


def test_jsd_equals_reference(golden):
    s, r = EO.jsd_sets()
    jsd = E.jsd_between_point_cloud_sets(s, r, resolution=28)
    assert abs(jsd - float(golden["jsd/value"])) <= 1e-12
    assert E.jsd_between_point_cloud_sets(torch.from_numpy(s).cuda(), torch.from_numpy(r)) == jsd


def test_matrix_blocks_equal_separate_calls(monkeypatch):
    s, r = gen(61, 5, 700, 3) * 0.3, gen(62, 4, 700, 3) * 0.3
    s, r = s.cuda(), r.cuda()
    s2 = gen(63, 5, 500, 3).cuda() * 0.3                             # another point count
    for metric, fn in (('CD', E.pairwise_CD), ('EMD', E.pairwise_EMD)):
        for smp in (s, s2):
            whole = E._score_matrices(metric, r, smp)
            assert whole[0].shape == (4, 5) and whole[1].shape == (4, 4) and whole[2].shape == (5, 5)
            assert all(torch.equal(a, b) for a, b in zip(whole, (fn(r, smp), fn(r, r), fn(smp, smp))))
            monkeypatch.setitem(E.LAUNCH_WORK, metric, 2 * 5 * 700 * 700)     # two rows per launch
            chunked = E._score_matrices(metric, r, smp)
            monkeypatch.undo()
            assert all(torch.equal(a, b) for a, b in zip(whole, chunked)), metric
    with pytest.raises(NotImplementedError):
        E._score_matrices('JSD', r, s)


def test_scores_equal_reference(golden):
    samples, refs = EO.score_sets()
    res = E.compute_all_metrics(samples.cuda(), refs.cuda(), 8, verbose=False)
    want = {k[len("all/"):]: float(v) for k, v in golden.items() if k.startswith("all/")}
    assert set(res) == set(want)
    for k, v in want.items():
        if k.startswith("lgan_mmd"):
            tol = 1e-5 if k.endswith("-CD") else 2e-3
            assert abs(res[k] - v) <= tol * abs(v), (k, res[k], v)
        else:
            assert res[k] == v, (k, res[k], v)
    cd_only = E.compute_all_metrics(samples.cuda(), refs.cuda(), 8, verbose=True, metric2=None)
    assert set(cd_only) == {k for k in want if k.endswith("-CD") or "-CD-" in k}
    assert all(cd_only[k] == res[k] for k in cd_only)
    with pytest.raises(L.LionError):
        E.compute_all_metrics(samples, refs, 8, verbose=False)


def test_emd_cd_against_per_pair_ops():
    s, r = gen(64, 6, 512, 3) * 0.3, gen(65, 6, 512, 3) * 0.35
    out = E.EMD_CD(s.cuda(), r.cuda(), 4, reduced=False)
    dl, dr = E.distChamferCUDAnograd(s.cuda(), r.cuda())
    assert torch.equal(out['MMD-CD'], dl.mean(1) + dr.mean(1))
    assert torch.equal(out['MMD-EMD'], E.emd_approx(s.cuda(), r.cuda(), require_grad=False))
    red = E.EMD_CD(s.cuda(), r.cuda(), 4)
    assert torch.equal(red['MMD-CD'], out['MMD-CD'].mean()) and torch.equal(red['MMD-EMD'], out['MMD-EMD'].mean())
    g = E.EMD_CD(s.cuda().requires_grad_(True), r.cuda(), 6, require_grad=True)
    (g['MMD-CD'] + g['MMD-EMD']).backward()


def _files(tmp_path, n_smp_points, channels):
    g = torch.Generator().manual_seed(71)
    ref = torch.randn(6, 256, channels, generator=g) * 0.3
    mean = torch.randn(6, 1, 3, generator=g) * 0.1
    std = torch.rand(6, 1, 1, generator=g) + 0.5
    smp = torch.randn(8, n_smp_points, channels, generator=g) * 0.3        # two more samples than references
    torch.save({'ref': ref, 'mean': mean, 'std': std}, tmp_path / "ref.pt")
    torch.save(smp, tmp_path / "smp.pt")
    return str(tmp_path / "smp.pt"), str(tmp_path / "ref.pt"), smp, ref, mean, std


@pytest.mark.parametrize("norm_box,n_smp_points,channels,cd_only", [
    (False, 256, 3, False), (True, 256, 3, False), (False, 300, 3, True), (True, 256, 6, True)])
def test_compute_score_end_to_end(tmp_path, monkeypatch, norm_box, n_smp_points, channels, cd_only):
    out, ref_name, smp, ref, mean, std = _files(tmp_path, n_smp_points, channels)
    monkeypatch.chdir(tmp_path)
    np.random.seed(5)
    res = compute_score(out, ref_name, norm_box=norm_box, cd_only=cd_only, dataset='t')
    np.random.seed(5)
    if n_smp_points > 256:
        smp = smp[:, np.random.permutation(np.arange(n_smp_points))[:256]]
    smp, ref = smp[:6, :, :3], ref[:, :, :3]
    if norm_box:
        smp, ref = 0.5 * torch.stack(normalize_point_clouds(smp)), 0.5 * torch.stack(normalize_point_clouds(ref))
    else:
        smp, ref = smp * std + mean, ref * std + mean
    want = E.compute_all_metrics(smp.cuda(), ref.cuda(), 256, verbose=False, metric2=None if cd_only else 'EMD')
    want['jsd'] = E.jsd_between_point_cloud_sets(smp.numpy(), ref.numpy())
    assert res == want
    rows = (tmp_path / "results" / "eval_out.csv").read_text().splitlines()
    assert len(rows) == 2 and rows[1].split('\t')[0].strip() == ('t-normbox' if norm_box else 't')
