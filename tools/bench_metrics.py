"""Time the Chamfer metric kernels (CUDA events): the fused pairwise CD matrix and the drop-in
nearest-neighbour op driven the reference's way (one sample cloud expanded against all references).
python tools/bench_metrics.py [n_sample n_ref]   -> JSON lines

python tools/bench_metrics.py --backward [B]      -> JSON lines: the differentiable losses at B pairs of 2048-point
clouds (default 32): EMD forward + backward and Chamfer backward, time and peak torch.cuda.max_memory_allocated,
against the reference's emd_ext / chamfer_3D extensions in oracle/_ref/ when they are built, with the card's name and
power limit."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lion_b200.utils.evaluation_metrics_fast import pairwise_CD, pairwise_EMD, distChamferCUDAnograd


def timed(fn, iters=3):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def peak_mib(fn):
    """Peak allocation above what was live before fn ran, MiB."""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)


def card():
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return {"card": torch.cuda.get_device_name(), "power_limit": pl or "unknown"}


def err(got, want):
    """max-abs error / max-abs reference, and the share of bit-equal elements."""
    return {"max_rel_err": float((got - want).abs().max() / want.abs().max().clamp_min(1e-30)),
            "bit_equal": round(float((got == want).float().mean()), 6)}


def backward_leg(B):
    from oracle import build_ref
    from lion_b200.third_party.ChamferDistancePytorch.chamfer3D.dist_chamfer_3D import chamfer_3DDist, _backward
    from lion_b200.third_party.PyTorchEMD.emd import earth_mover_distance
    N = 2048
    g = torch.Generator().manual_seed(0)
    a = (torch.randn(B, N, 3, generator=g) * 0.4).cuda()
    b = (torch.randn(B, N, 3, generator=g) * 0.4 + 0.05).cuda()
    gw = torch.randn(B, generator=g).cuda()
    info = dict(card(), B=B, points=N)
    ref_emd, ref_cd = build_ref.load_emd(), build_ref.load_chamfer()

    def emd_ours():
        x1, x2 = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
        (earth_mover_distance(x1, x2, transpose=False) * gw).sum().backward()
        return x1.grad, x2.grad

    def emd_ref():
        match = ref_emd.approxmatch_forward(a, b)
        ref_emd.matchcost_forward(a, b, match)
        return ref_emd.matchcost_backward((gw / float(N)).contiguous(), a, b, match)

    legs = [("EMD forward+backward", "lion_emd_approx_saved + lion_emd_backward", emd_ours,
             "emd_ext approxmatch + matchcost + matchcost_backward", emd_ref if ref_emd else None)]

    x1, x2 = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    d1, d2, i1, i2 = chamfer_3DDist()(x1, x2)
    gd1, gd2 = torch.randn(B, N, generator=g).cuda(), torch.randn(B, N, generator=g).cuda()
    rg1, rg2 = torch.zeros(B, N, 3, device="cuda"), torch.zeros(B, N, 3, device="cuda")

    def cd_ours():
        return _backward(a, b, i1, i2, gd1, gd2)

    def cd_ref():
        rg1.zero_(); rg2.zero_()                  # the reference accumulates into zeroed gradients
        ref_cd.backward(a, b, rg1, rg2, gd1, gd2, i1, i2)
        return rg1, rg2

    legs.append(("Chamfer backward", "lion_chamfer_backward", cd_ours, "chamfer_3D.backward", cd_ref if ref_cd else None))

    def cd_fb_ours():
        y1, y2 = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
        e1, e2, _, _ = chamfer_3DDist()(y1, y2)
        torch.autograd.backward([e1, e2], [gd1, gd2])

    def cd_fb_ref():
        dd1, dd2 = torch.zeros(B, N, device="cuda"), torch.zeros(B, N, device="cuda")
        j1, j2 = torch.zeros(B, N, dtype=torch.int32, device="cuda"), torch.zeros(B, N, dtype=torch.int32, device="cuda")
        ref_cd.forward(a, b, dd1, dd2, j1, j2)
        ref_cd.backward(a, b, torch.zeros(B, N, 3, device="cuda"), torch.zeros(B, N, 3, device="cuda"), gd1, gd2, j1, j2)

    for what, ours_name, ours, ref_name, ref in legs:
        rec = dict(info, what=what, ours=ours_name, ours_ms=round(timed(ours, iters=10), 3))
        rec["reference"] = ref_name
        if ref is None:
            rec["reference_ms"] = "not available (oracle/_ref not built)"
        else:
            rec["reference_ms"] = round(timed(ref, iters=10), 3)
            o, r = ours(), ref()
            rec["grad1_vs_reference"], rec["grad2_vs_reference"] = err(o[0], r[0]), err(o[1], r[1])
        print(json.dumps(rec))
    # peak memory of one differentiable evaluation of each loss (forward + backward)
    mem = dict(info, what="peak max_memory_allocated above the inputs, MiB", emd_ours=peak_mib(emd_ours),
               chamfer_ours=peak_mib(cd_fb_ours))
    mem["emd_reference"] = peak_mib(emd_ref) if ref_emd else "not available"
    mem["chamfer_reference"] = peak_mib(cd_fb_ref) if ref_cd else "not available"
    print(json.dumps(mem))


if "--backward" in sys.argv:
    rest = [v for v in sys.argv[1:] if v != "--backward"]
    backward_leg(int(rest[0]) if rest else 32)
    sys.exit(0)

ns = int(sys.argv[1]) if len(sys.argv) > 1 else 64
nr = int(sys.argv[2]) if len(sys.argv) > 2 else 405
N = 2048
g = torch.Generator().manual_seed(0)
s = torch.randn(ns, N, 3, generator=g).cuda()
r = torch.randn(nr, N, 3, generator=g).cuda()


def composed():
    rows = []
    for i in range(ns):
        dl, dr = distChamferCUDAnograd(s[i:i + 1].expand(nr, -1, -1).contiguous(), r)
        rows.append(dl.mean(1) + dr.mean(1))
    return torch.stack(rows)


pair_evals = 2.0 * ns * nr * N * N          # both directions
for name, fn in (("fused lion_chamfer_pairwise", lambda: pairwise_CD(s, r)), ("drop-in op, reference-style loop", composed)):
    ms = timed(fn)
    print(json.dumps({"what": name, "n_sample": ns, "n_ref": nr, "points": N, "ms": round(ms, 3),
                      "cloud_pairs_per_s": round(ns * nr / (ms * 1e-3)), "gflops_8_per_point_pair": round(8 * pair_evals / (ms * 1e-3) / 1e9)}))
assert torch.allclose(pairwise_CD(s, r), composed(), rtol=1e-5, atol=0)
# approximate EMD: 30 exp-weighted N x M passes per pair (MUFU-bound); a smaller block of the matrix
ne = max(1, ns // 8)
ms = timed(lambda: pairwise_EMD(s[:ne], r), iters=1)
print(json.dumps({"what": "fused lion_emd_pairwise", "n_sample": ne, "n_ref": nr, "points": N, "ms": round(ms, 3),
                  "cloud_pairs_per_s": round(ne * nr / (ms * 1e-3)), "gexp_per_s": round(30.0 * ne * nr * N * N / (ms * 1e-3) / 1e9)}))
