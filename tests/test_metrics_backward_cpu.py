"""The float64 Chamfer and EMD backward restatements (tests/metrics_backward_oracle.py) against torch float64 autograd
through the same formulations: a gather on fixed nearest-neighbour indices, and sum |x1 - x2|^2 * match with the match
detached."""
import numpy as np
import torch

from oracle import metrics as OM
from tests import metrics_backward_oracle as OB
from tests.util import gen


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def test_chamfer_backward_oracle_matches_autograd():
    a, b = gen(1, 2, 70, 3), gen(2, 2, 45, 3)
    a[:, 1:20] = a[:, :1]                               # many points share one nearest neighbour
    b[:, 3] = b[:, 1]
    _, _, i1, i2 = OM.chamfer_forward(a.numpy(), b.numpy())
    gd1, gd2 = gen(3, 2, 70), gen(4, 2, 45)
    x1 = a.double().requires_grad_(True)
    x2 = b.double().requires_grad_(True)
    bi = torch.arange(2)[:, None]
    d1 = ((x1 - x2[bi, torch.from_numpy(i1).long()]) ** 2).sum(-1)
    d2 = ((x2 - x1[bi, torch.from_numpy(i2).long()]) ** 2).sum(-1)
    ((d1 * gd1.double()).sum() + (d2 * gd2.double()).sum()).backward()
    g1, g2 = OB.chamfer_backward(a.numpy(), b.numpy(), i1, i2, gd1.numpy(), gd2.numpy())
    assert _rel(g1, x1.grad.numpy()) < 1e-12 and _rel(g2, x2.grad.numpy()) < 1e-12


def test_emd_backward_oracle_matches_autograd():
    for n, m in ((40, 40), (48, 16), (9, 30)):
        a, b = gen(5, 2, n, 3) * 0.4, gen(6, 2, m, 3) * 0.4 + 0.1
        match = OB.emd_match(a.numpy(), b.numpy())
        # the restated match gives the forward oracle's cost
        d2 = ((a.double()[:, :, None, :] - b.double()[:, None, :, :]) ** 2).sum(-1).numpy()
        assert _rel((d2 * match).sum((1, 2)), OM.emd_approx(a.numpy(), b.numpy())) < 1e-12
        gc = gen(7, 2).double()
        x1 = a.double().requires_grad_(True)
        x2 = b.double().requires_grad_(True)
        w = torch.from_numpy(match).detach()
        cost = (((x1[:, :, None, :] - x2[:, None, :, :]) ** 2).sum(-1) * w).sum((1, 2))
        (cost * gc).sum().backward()
        g1, g2 = OB.emd_backward(a.numpy(), b.numpy(), gc.numpy(), match)
        assert _rel(g1, x1.grad.numpy()) < 1e-12 and _rel(g2, x2.grad.numpy()) < 1e-12
