"""Backward passes of the differentiable Chamfer (chamfer_3DDist) and approximate EMD (earth_mover_distance) through
torch.autograd, against the outputs of the reference's own backward kernels (chamfer3D.cu:155-195 NmDistanceGradKernel,
emd_kernel.cu:280-353 matchcostgrad1/2) stored in tests/golden/ref_metrics_backward.npz (tests/refvec_backward.py),
torch autograd, and the float64 restatements of tests/metrics_backward_oracle.py."""
import numpy as np
import pytest
import torch

from oracle import build_ref
from tests import metrics_backward_oracle as OB
from tests import refvec as R
from tests import refvec_backward as RB
from tests.util import assert_close, gen

pytestmark = pytest.mark.gpu


def _chamfer_mod():
    mod = build_ref.load_chamfer()
    assert mod is not None, "oracle/_ref/chamfer_3D.so is missing (python oracle/build_ref.py)"
    return mod


def _emd_mod():
    mod = build_ref.load_emd()
    assert mod is not None, "oracle/_ref/emd_ext.so is missing (python oracle/build_ref.py)"
    return mod


def _Dist():
    from lion_b200.third_party.ChamferDistancePytorch.chamfer3D.dist_chamfer_3D import chamfer_3DDist
    return chamfer_3DDist()


def _clouds(B, N, M):
    a, b = gen(101, B, N, 3), gen(102, B, M, 3)
    if N > 4 and M > 4:
        a[:, : max(2, N // 8)] = a[:, :1]          # duplicated points: many share one nearest neighbour
        b[:, : max(2, M // 8)] = b[:, :1]
        b[:, 3] = b[:, 1]
    return a, b


def _chamfer_grads(a, b, gd1, gd2):
    x1 = a.cuda().requires_grad_(True)
    x2 = b.cuda().requires_grad_(True)
    d1, d2, i1, i2 = _Dist()(x1, x2)
    torch.autograd.backward([d1, d2], [gd1.cuda(), gd2.cuda()])
    return x1.grad, x2.grad, i1, i2


def _ref_chamfer_backward(a, b, gd1, gd2):
    mod = _chamfer_mod()
    B, n, m = a.shape[0], a.shape[1], b.shape[1]
    a, b = a.cuda(), b.cuda()
    d1 = torch.zeros(B, n, device="cuda"); d2 = torch.zeros(B, m, device="cuda")
    i1 = torch.zeros(B, n, dtype=torch.int32, device="cuda"); i2 = torch.zeros(B, m, dtype=torch.int32, device="cuda")
    mod.forward(a, b, d1, d2, i1, i2)
    g1 = torch.zeros(B, n, 3, device="cuda"); g2 = torch.zeros(B, m, 3, device="cuda")
    mod.backward(a, b, g1, g2, gd1.cuda().contiguous(), gd2.cuda().contiguous(), i1, i2)
    return g1, g2


def _exact_where_single(got, st, scattered, what):
    """Elements of points with at most one scattered term equal the reference bit for bit (on the stored elements)."""
    a = got.detach().cpu().numpy()
    one = np.repeat((scattered <= 1).ravel(), 3)
    if st.full is not None:
        sel = np.nonzero(one)[0]
        want = st.full.ravel()[sel]
    else:
        keep = one[st.idx]
        sel, want = st.idx[keep], st.vals[keep]
    assert np.array_equal(a.ravel()[sel], want), "%s: %d elements with <= 1 scattered term differ" % (
        what, int((a.ravel()[sel] != want).sum()))
    return sel.size


def _chamfer_close(got, want, amax, bound, what, sel=None):
    """|got - want| <= max(1e-6 max|want|, bound) elementwise (on the elements `sel` when given).

    bound is the fp32 summation error allowance of each element: where hundreds of points share one nearest neighbour,
    an fp32 sum of their terms -- the reference's atomics in whatever order they land, or this library's ascending
    order -- is only within gamma_n * sum |t_i| of the exact gradient, which can exceed 1e-6 of the largest element."""
    g = got.detach().cpu().double().numpy().ravel()
    b = bound.ravel()
    if sel is not None:
        g, b = g[sel], b[sel]
    assert np.isfinite(g).all(), "%s: non-finite values" % what
    err = np.abs(g - np.asarray(want, np.float64).ravel())
    ok = err <= np.maximum(1e-6 * amax, b)
    assert ok.all(), "%s: %d elements exceed max(1e-6 max-abs, fp32 sum bound); max-abs error / max-abs = %.3e" % (
        what, int((~ok).sum()), err.max() / amax)
    return err.max() / amax


@pytest.mark.parametrize("B,N,M", [(3, 2048, 2048), (2, 1000, 777), (1, 5, 3000), (2, 4100, 513)])
def test_chamfer_backward_matches_reference_kernel(B, N, M):
    a, b = _clouds(B, N, M)
    gd1, gd2 = gen(103, B, N), gen(104, B, M)
    g1, g2, i1, i2 = _chamfer_grads(a, b, gd1, gd2)
    r1, r2 = RB.ref_out("chamfer_backward/%d-%d-%d" % (B, N, M), lambda: _ref_chamfer_backward(a, b, gd1, gd2))
    (_, s1, n1), (_, s2, n2) = OB.chamfer_backward(a.numpy(), b.numpy(), i1.cpu().numpy(), i2.cpu().numpy(), gd1.numpy(),
                                                   gd2.numpy(), magnitude=True)
    for got, st, bound, what in ((g1, r1, 2 * OB.fp32_sum_bound(s1, n1), "Chamfer grad1 vs reference kernel"),
                                 (g2, r2, 2 * OB.fp32_sum_bound(s2, n2), "Chamfer grad2 vs reference kernel")):
        assert tuple(got.shape) == st.shape
        if st.full is not None:
            _chamfer_close(got, st.full, st.amax, bound, what)
        else:
            _chamfer_close(got, st.vals, st.amax, bound, what, sel=st.idx)
    i1, i2 = i1.cpu().numpy(), i2.cpu().numpy()
    cnt1 = np.stack([np.bincount(i2[k], minlength=N) for k in range(B)])     # scattered terms of each xyz1 point
    cnt2 = np.stack([np.bincount(i1[k], minlength=M) for k in range(B)])
    _exact_where_single(g1, r1, cnt1, "Chamfer grad1")
    _exact_where_single(g2, r2, cnt2, "Chamfer grad2")
    h1, h2, _, _ = _chamfer_grads(a, b, gd1, gd2)
    assert torch.equal(g1, h1) and torch.equal(g2, h2), "Chamfer backward is not bit-reproducible"


@pytest.mark.parametrize("B,N,M", [(3, 2048, 2048), (2, 1000, 777), (1, 5, 3000), (2, 4100, 513)])
def test_chamfer_backward_matches_autograd(B, N, M):
    a, b = _clouds(B, N, M)
    gd1, gd2 = gen(105, B, N), gen(106, B, M)
    g1, g2, i1, i2 = _chamfer_grads(a, b, gd1, gd2)
    x1 = a.cuda().double().requires_grad_(True)
    x2 = b.cuda().double().requires_grad_(True)
    bi = torch.arange(B, device="cuda")[:, None]
    d1 = ((x1 - x2[bi, i1.long()]) ** 2).sum(-1)
    d2 = ((x2 - x1[bi, i2.long()]) ** 2).sum(-1)
    torch.autograd.backward([d1, d2], [gd1.cuda().double(), gd2.cuda().double()])
    (o1, s1, n1), (o2, s2, n2) = OB.chamfer_backward(a.numpy(), b.numpy(), i1.cpu().numpy(), i2.cpu().numpy(), gd1.numpy(),
                                                     gd2.numpy(), magnitude=True)
    for got, want, o, bound, what in ((g1, x1.grad, o1, OB.fp32_sum_bound(s1, n1), "Chamfer grad1"),
                                      (g2, x2.grad, o2, OB.fp32_sum_bound(s2, n2), "Chamfer grad2")):
        want = want.cpu().numpy()
        amax = np.abs(want).max()
        _chamfer_close(got, want, amax, bound, what + " vs autograd")
        _chamfer_close(got, o, amax, bound, what + " vs float64 oracle")


def _emd_grads(a, b, gw, transpose):
    from lion_b200.third_party.PyTorchEMD.emd import earth_mover_distance
    x1 = (a.transpose(1, 2) if transpose else a).contiguous().cuda().requires_grad_(True)
    x2 = (b.transpose(1, 2) if transpose else b).contiguous().cuda().requires_grad_(True)
    cost = earth_mover_distance(x1, x2, transpose=transpose)
    (cost * gw.cuda()).sum().backward()
    g1, g2 = x1.grad, x2.grad
    if transpose:
        g1, g2 = g1.transpose(1, 2), g2.transpose(1, 2)
    return cost.detach(), g1, g2


def _ref_emd_backward(a, b, grad_cost):
    mod = _emd_mod()
    a, b = a.cuda(), b.cuda()
    match = mod.approxmatch_forward(a, b)
    g1, g2 = mod.matchcost_backward(grad_cost.cuda().contiguous(), a, b, match)
    return g1, g2


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("B,N,M", [(3, 2048, 2048), (2, 512, 512), (2, 1024, 256), (2, 300, 1200), (1, 7, 5)])
def test_emd_backward_matches_reference_kernels_and_oracle(B, N, M, transpose):
    from lion_b200.third_party.PyTorchEMD.emd_nograd import earth_mover_distance_nograd
    a, b = gen(91, B, N, 3) * 0.4, gen(92, B, M, 3) * 0.4 + 0.1          # the forward test's clouds
    gw = gen(107, B)
    cost, g1, g2 = _emd_grads(a, b, gw, transpose)
    assert torch.equal(cost, earth_mover_distance_nograd(a.cuda(), b.cuda(), transpose=False)), \
        "the saving forward must give the no-grad cost bit for bit"
    grad_cost = gw / float(N)                      # what autograd hands the Function through `/ N`
    r1, r2 = RB.ref_out("emd_backward/%d-%d-%d" % (B, N, M), lambda: _ref_emd_backward(a, b, grad_cost))
    R.close(g1, r1, 2e-5, "EMD grad1 vs reference kernels")
    R.close(g2, r2, 2e-5, "EMD grad2 vs reference kernels")
    if N * M <= 1024 * 1024:
        o1, o2 = OB.emd_backward(a.numpy(), b.numpy(), grad_cost.numpy())
        assert_close(g1, torch.from_numpy(o1), 2e-3, "EMD grad1 vs float64 oracle")
        assert_close(g2, torch.from_numpy(o2), 2e-3, "EMD grad2 vs float64 oracle")
    _, h1, h2 = _emd_grads(a, b, gw, transpose)
    assert torch.equal(g1, h1) and torch.equal(g2, h2), "EMD backward is not bit-reproducible"


def test_no_grad_path_builds_no_graph():
    from lion_b200.third_party.ChamferDistancePytorch.chamfer3D.dist_chamfer_3D import chamfer_3DDist_nograd
    from lion_b200.third_party.PyTorchEMD.emd import earth_mover_distance
    from lion_b200.third_party.PyTorchEMD.emd_nograd import earth_mover_distance_nograd
    a = gen(111, 2, 600, 3).cuda().requires_grad_(True)
    b = gen(112, 2, 500, 3).cuda().requires_grad_(True)
    want = chamfer_3DDist_nograd()(a.detach(), b.detach())
    with torch.no_grad():
        got = _Dist()(a, b)
        cost = earth_mover_distance(a, b, transpose=False)
    for g, w in zip(got, want):
        assert g.grad_fn is None and not g.requires_grad and torch.equal(g, w)
    assert cost.grad_fn is None and torch.equal(cost, earth_mover_distance_nograd(a.detach(), b.detach(), transpose=False))
    # inputs that do not require grad take the plain call as well
    got = _Dist()(a.detach(), b.detach())
    assert all(g.grad_fn is None for g in got)
    # with grad, the indices are constants and the distances are the no-grad ones
    d1, d2, i1, i2 = _Dist()(a, b)
    assert d1.grad_fn is not None and not i1.requires_grad and not i2.requires_grad
    assert torch.equal(d1, want[0]) and torch.equal(d2, want[1]) and torch.equal(i1, want[2]) and torch.equal(i2, want[3])


def test_autocast_runs_fp32_and_returns_input_dtype():
    from lion_b200.third_party.PyTorchEMD.emd import earth_mover_distance
    a16 = (gen(113, 2, 512, 3) * 0.4).half().cuda().requires_grad_(True)
    b16 = (gen(114, 2, 400, 3) * 0.4 + 0.1).half().cuda().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.float16):
        d1, d2, _, _ = _Dist()(a16, b16)
        cost = earth_mover_distance(a16, b16, transpose=False)
    assert d1.dtype == torch.float32 and d2.dtype == torch.float32 and cost.dtype == torch.float32
    cd16 = torch.autograd.grad(d1.sum() + d2.sum(), [a16, b16])
    emd16 = torch.autograd.grad(cost.sum(), [a16, b16])
    assert all(g.dtype == torch.float16 for g in cd16 + emd16)
    # the fp32 computation on the fp16 values, its gradients rounded to fp16
    a32 = a16.detach().float().requires_grad_(True)
    b32 = b16.detach().float().requires_grad_(True)
    e1, e2, _, _ = _Dist()(a32, b32)
    cd32 = torch.autograd.grad(e1.sum() + e2.sum(), [a32, b32])
    emd32 = torch.autograd.grad(earth_mover_distance(a32, b32, transpose=False).sum(), [a32, b32])
    for g16, g32 in zip(cd16 + emd16, cd32 + emd32):
        assert torch.equal(g16, g32.half())


def test_loss_composition_gives_finite_gradients():
    from lion_b200.utils.evaluation_metrics_fast import distChamferCUDA, emd_approx
    B, N = 32, 2048
    x = (gen(115, B, N, 3) * 0.4).cuda().requires_grad_(True)
    y = (gen(116, B, N, 3) * 0.4 + 0.05).cuda()
    dl, dr = distChamferCUDA(x, y)
    loss_cd = dl.mean(1) + dr.mean(1)                 # utils/model_helper.py loss_fn: Chamfer term
    loss_emd = emd_approx(x, y) * N                   # ... and its EMD term
    (loss_cd.sum() + loss_emd.sum()).backward()
    assert torch.isfinite(x.grad).all() and x.grad.abs().max() > 0
    assert loss_cd.grad_fn is not None and loss_emd.grad_fn is not None
