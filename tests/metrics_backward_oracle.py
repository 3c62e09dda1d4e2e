"""Float64 restatements of the Chamfer and approximate-EMD backward passes (TEST INFRASTRUCTURE ONLY).

  chamfer_backward  third_party/ChamferDistancePytorch/chamfer3D/chamfer3D.cu:155-195 (NmDistanceGradKernel, launched
                    once per direction): the direct term of every point plus the scattered terms of the points of the
                    other cloud whose nearest neighbour it is.
  emd_match         the soft assignment of third_party/PyTorchEMD/cuda/emd_kernel.cu:23-170 (approxmatch), as in
                    oracle/metrics.py emd_approx, returned as match [B, N, M] (match[b][k][l] = the reference's
                    match[b][l][k]).
  emd_backward      emd_kernel.cu:280-353 (matchcostgrad1 / matchcostgrad2) with the match held constant.
"""
import numpy as np


def chamfer_backward(xyz1, xyz2, idx1, idx2, graddist1, graddist2, magnitude=False):
    """xyz1 [B,N,3], xyz2 [B,M,3], idx1 [B,N], idx2 [B,M], graddist1 [B,N], graddist2 [B,M] -> grad1, grad2 (float64).

    With magnitude=True, each gradient comes with the sum of the absolute values of its terms and the number of
    terms: an fp32 sum of n terms t_i is within gamma_n * sum |t_i| (gamma_n = n u / (1 - n u), u = 2^-24) of exact."""
    x1 = np.asarray(xyz1, np.float64)
    x2 = np.asarray(xyz2, np.float64)
    g1 = 2.0 * np.asarray(graddist1, np.float64)[..., None]
    g2 = 2.0 * np.asarray(graddist2, np.float64)[..., None]
    grad1, grad2 = np.zeros_like(x1), np.zeros_like(x2)
    abs1, abs2 = np.zeros_like(x1), np.zeros_like(x2)
    n1, n2 = np.ones(x1.shape[:2]), np.ones(x2.shape[:2])
    for b in range(x1.shape[0]):
        t1 = g1[b] * (x1[b] - x2[b][idx1[b]])            # d dist1[i] / d xyz1[i], times graddist1
        t2 = g2[b] * (x2[b] - x1[b][idx2[b]])
        grad1[b] += t1
        np.add.at(grad2[b], idx1[b], -t1)
        grad2[b] += t2
        np.add.at(grad1[b], idx2[b], -t2)
        abs1[b] += np.abs(t1)
        np.add.at(abs2[b], idx1[b], np.abs(t1))
        abs2[b] += np.abs(t2)
        np.add.at(abs1[b], idx2[b], np.abs(t2))
        np.add.at(n1[b], idx2[b], 1)
        np.add.at(n2[b], idx1[b], 1)
    if magnitude:
        return (grad1, abs1, n1), (grad2, abs2, n2)
    return grad1, grad2


def fp32_sum_bound(abs_sum, n_terms):
    """gamma_n * sum |t_i| per element (n_terms per point, broadcast over xyz)."""
    nu = n_terms[..., None] * 2.0 ** -24
    return nu / (1.0 - nu) * abs_sum


def emd_match(xyz1, xyz2):
    """xyz1 [B,N,3], xyz2 [B,M,3] -> match [B,N,M] (float64, exact exp)."""
    xyz1 = np.asarray(xyz1, np.float64)
    xyz2 = np.asarray(xyz2, np.float64)
    B, n, m = xyz1.shape[0], xyz1.shape[1], xyz2.shape[1]
    out = np.zeros((B, n, m))
    for b in range(B):
        d2 = ((xyz2[b][None, :, :] - xyz1[b][:, None, :]) ** 2).sum(-1)
        multiL, multiR = (1.0, float(n // m)) if n >= m else (float(m // n), 1.0)
        remainL = np.full(n, multiL)
        remainR = np.full(m, multiR)
        for j in range(7, -3, -1):
            level = -(4.0 ** j) if j != -2 else 0.0
            e = np.exp(level * d2)
            ratioL = remainL / (1e-9 + e @ remainR)
            sumr = (e.T @ ratioL) * remainR
            ratioR = np.minimum(remainR / (sumr + 1e-9), 1.0) * remainR
            remainR = np.maximum(0.0, remainR - sumr)
            w = e * ratioL[:, None] * ratioR[None, :]
            out[b] += w
            remainL = np.maximum(0.0, remainL - w.sum(1))
    return out


def emd_backward(xyz1, xyz2, grad_cost, match=None):
    """d/dxyz of sum_b grad_cost[b] * sum_{k,l} |xyz1_k - xyz2_l|^2 match[k][l], match constant -> grad1, grad2."""
    x1 = np.asarray(xyz1, np.float64)
    x2 = np.asarray(xyz2, np.float64)
    w = emd_match(x1, x2) if match is None else match
    gc = np.asarray(grad_cost, np.float64)[:, None, None]
    diff = x1[:, :, None, :] - x2[:, None, :, :]           # [B,N,M,3]
    grad1 = gc * 2.0 * np.einsum("bkl,bklc->bkc", w, diff)
    grad2 = -gc * 2.0 * np.einsum("bkl,bklc->blc", w, diff)
    return grad1, grad2
