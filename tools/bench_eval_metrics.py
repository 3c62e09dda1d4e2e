"""Wall time of compute_score (MMD / COV / 1-NNA for CD and EMD, and JSD) on synthetic 2048-point sets, split into its
phases, with the card's name and power limit from the same run.

python tools/bench_eval_metrics.py [--sizes 405 1000] [--probe]   -> JSON lines

For every size n (n samples against n references; 405 = the airplane test split, 1000 = 'all'):
  total_s          compute_score wall time (the sample / reference files are written to a temporary directory
                   first, outside the timed region; skip_write=True)
  cd_s, emd_s      the three CD matrices, the three EMD matrices (host clock around each phase, synchronised)
  jsd_s            jsd_between_point_cloud_sets (both occupancy-grid launches, entropy, divergence)
  bookkeeping_s    the rest: loading, de-normalising, lgan_mmd_cov, knn, printing
  longest_launch_ms  the longest single pairwise CD / EMD launch (CUDA events around each)
  jsd_host_s       the reference's host route for the same JSD (sklearn NearestNeighbors on the grid and per-point
                   Python loops), where sklearn is installed; otherwise "not available"
--probe: per-pair time of lion_emd_pairwise at 2048 points (the basis of evaluation_metrics_fast.LAUNCH_WORK).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from lion_b200.utils import eval_helper as H  # noqa: E402
from lion_b200.utils import evaluation_metrics_fast as E  # noqa: E402

N = 2048


def card():
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return {"card": torch.cuda.get_device_name(), "power_limit": pl or "unknown"}


def synth(n, seed):
    """n clouds of N points: per-cloud blobs inside the unit sphere, stored normalised with a mean and std."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, N, 3, generator=g) * (0.08 + 0.1 * torch.rand(n, 1, 1, generator=g))
    x += (torch.rand(n, 1, 3, generator=g) - 0.5) * 0.3
    mean = torch.zeros(n, 1, 3)
    std = torch.ones(n, 1, 1)
    return x, mean, std


def jsd_host(sample, ref, resolution=28):
    """The reference's JSD route on the host: a NearestNeighbors query per cloud, counts by Python loops."""
    from sklearn.neighbors import NearestNeighbors
    cells, _ = E.unit_cube_grid_point_cloud(resolution, clip_sphere=True)
    nn = NearestNeighbors(n_neighbors=1).fit(cells)

    def counters(pcs):
        counts = np.zeros(len(cells))
        for pc in pcs:
            _, idx = nn.kneighbors(pc)
            for i in np.squeeze(idx):
                counts[i] += 1
        return counts
    return E.jensen_shannon_divergence(counters(sample), counters(ref))


class Phases:
    """Host-clock time of each patched phase and CUDA-event time of every pairwise launch."""

    def __init__(self):
        self.t = {"CD": 0.0, "EMD": 0.0, "JSD": 0.0}
        self.launches = []
        self._orig = (E._score_matrices, E.pairwise_CD, E.pairwise_EMD, H.jsd_between_point_cloud_sets)

    def __enter__(self):
        score, pcd, pemd, jsd = self._orig

        def phase(name, fn):
            def w(*a, **k):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = fn(*a, **k)
                torch.cuda.synchronize()
                self.t[name if name != "score" else a[0]] += time.perf_counter() - t0
                return out
            return w

        def launch(what, fn):
            def w(*a, **k):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = fn(*a, **k)
                e1.record()
                self.launches.append((what, e0, e1))
                return out
            return w
        E._score_matrices = phase("score", score)
        E.pairwise_CD, E.pairwise_EMD = launch("CD", pcd), launch("EMD", pemd)
        H.jsd_between_point_cloud_sets = phase("JSD", jsd)
        return self

    def __exit__(self, *exc):
        E._score_matrices, E.pairwise_CD, E.pairwise_EMD, H.jsd_between_point_cloud_sets = self._orig
        torch.cuda.synchronize()
        return False

    def longest(self):
        ms = [(e0.elapsed_time(e1), what) for what, e0, e1 in self.launches]
        return max(ms) if ms else (0.0, "-")


def run_size(n, tmp):
    smp, _, _ = synth(n, 1)
    ref, mean, std = synth(n, 2)
    smp_name, ref_name = os.path.join(tmp, "smp_%d.pt" % n), os.path.join(tmp, "ref_%d.pt" % n)
    torch.save(smp, smp_name)
    torch.save({"ref": ref, "mean": mean, "std": std}, ref_name)
    with Phases() as ph:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = H.compute_score(smp_name, ref_name, skip_write=True, dataset="synthetic")
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
    ms, what = ph.longest()
    rec = dict(card(), n_sample=n, n_ref=n, points=N, total_s=round(total, 3), cd_s=round(ph.t["CD"], 3),
               emd_s=round(ph.t["EMD"], 3), jsd_s=round(ph.t["JSD"], 3),
               bookkeeping_s=round(total - sum(ph.t.values()), 3), longest_launch_ms=round(ms, 1), longest_launch=what,
               launches=len(ph.launches), scores={k: round(v, 6) for k, v in res.items()})
    try:
        import sklearn  # noqa: F401
        t0 = time.perf_counter()
        jsd_ref = jsd_host(smp.numpy(), ref.numpy())
        rec["jsd_host_s"] = round(time.perf_counter() - t0, 3)
        rec["jsd_host_minus_ours"] = float(jsd_ref - res["jsd"])
    except ImportError:
        rec["jsd_host_s"] = "not available"
    print(json.dumps(rec), flush=True)


def probe():
    s, _, _ = synth(4, 3)
    r, _, _ = synth(405, 4)
    s, r = s.cuda(), r.cuda()
    E.pairwise_EMD(s[:1], r[:8])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    E.pairwise_EMD(s, r)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    print(json.dumps(dict(card(), what="lion_emd_pairwise per-pair time", pairs=4 * 405, points=N, ms=round(ms, 2),
                          us_per_pair=round(1e3 * ms / (4 * 405), 2))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="*", default=[405, 1000])
    ap.add_argument("--probe", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval_metrics needs a CUDA device")
    if a.probe:
        probe()
    with tempfile.TemporaryDirectory() as tmp:
        smp, mean, std = synth(6, 5)             # warm-up: module loads and kernel attributes, outside the timings
        torch.save(smp, os.path.join(tmp, "w.pt"))
        torch.save({"ref": smp, "mean": mean, "std": std}, os.path.join(tmp, "wr.pt"))
        H.compute_score(os.path.join(tmp, "w.pt"), os.path.join(tmp, "wr.pt"), skip_write=True)
        for n in a.sizes:
            run_size(n, tmp)


if __name__ == "__main__":
    main()
