"""Chamfer part of the generation metrics -- mirror of the reference's
utils/evaluation_metrics_fast.py: `distChamferCUDAnograd` (:83-88 region) and the pairwise CD matrix of
`_pairwise_EMD_CD_` (:272-340), which `compute_all_metrics` feeds to MMD / COV / 1-NNA.

`_pairwise_EMD_CD_(metric='CD', ...)` is ONE kernel launch per <= 65535 sample clouds
(lion_chamfer_pairwise: a CTA per (sample, reference) pair, both directions, means reduced on
chip) instead of the reference's Python double loop with an expanded copy of the sample cloud
per reference batch; metric='EMD' likewise (lion_emd_pairwise: the fused approxmatch + matchcost
kernel per pair, no [Nr, M, N] match matrices).

The reconstruction losses of utils/model_helper.py:17-74 are differentiable: `distChamferCUDA` (reference :99-109)
and `emd_approx(require_grad=True)` (reference :122-147) backpropagate through the library's Chamfer and EMD
backward kernels.  `distChamferCUDA_l1` (reference :31-57) is not provided: it imports `models.pvcnn.functional`,
which does not exist in the reference tree."""
import torch

from .. import _lib as L
from ..third_party.ChamferDistancePytorch.chamfer3D.dist_chamfer_3D import chamfer_3DDist, chamfer_3DDist_nograd
from ..third_party.PyTorchEMD.emd import earth_mover_distance
from ..third_party.PyTorchEMD.emd_nograd import earth_mover_distance_nograd


def distChamferCUDAnograd(x, y, points_dim=3):
    """x, y [B,N,3] -> (dl [B,N], dr [B,M]) squared nearest-neighbour distances both ways."""
    assert x.dim() == 3 and y.dim() == 3 and x.shape[2] == points_dim and y.shape[2] == points_dim
    dl, dr, _, _ = chamfer_3DDist_nograd()(x, y)
    return dl, dr


@torch.no_grad()
def pairwise_CD(sample_pcs, ref_pcs):
    """[Ns,N,3], [Nr,M,3] -> [Ns,Nr] Chamfer matrix (dl.mean(1) + dr.mean(1) of every pair)."""
    if not sample_pcs.is_cuda or not ref_pcs.is_cuda:
        raise L.LionError("lion_b200 needs CUDA tensors; there is no CPU path")
    s = sample_pcs.detach().to(torch.float32).contiguous()
    r = ref_pcs.detach().to(torch.float32).contiguous()
    assert s.dim() == 3 and r.dim() == 3 and s.shape[2] == 3 and r.shape[2] == 3
    ns, n = s.shape[0], s.shape[1]
    nr, m = r.shape[0], r.shape[1]
    out = torch.empty(ns, nr, device=s.device)
    with torch.cuda.device(s.device):
        for a in range(0, ns, 65535):
            e = min(ns, a + 65535)
            L.check(L.lib().lion_chamfer_pairwise(L.ptr(s[a:e]), L.ptr(r), L.ptr(out[a:e]), e - a, nr, n, m, L.stream()),
                    "chamfer_pairwise")
    return out


def distChamferCUDA(x, y):
    """x [B,N,3], y [B,M,3] -> (dist1 [B,N], dist2 [B,M]), differentiable (reference :99-109)."""
    assert x.dim() == 3 and y.dim() == 3 and x.shape[2] == 3 and y.shape[2] == 3, f'get {x.shape} and {y.shape}'
    dist1, dist2, _, _ = chamfer_3DDist()(x.cuda(), y.cuda())
    return dist1, dist2


def emd_approx(sample, ref, require_grad=True):
    """[B,N,3] x [B,M,3] -> [B] approximate EMD / N (reference :122-147); differentiable when require_grad."""
    if not require_grad:
        return earth_mover_distance_nograd(sample.cuda(), ref.cuda(), transpose=False)
    return earth_mover_distance(sample.cuda(), ref.cuda(), transpose=False)


@torch.no_grad()
def pairwise_EMD(sample_pcs, ref_pcs):
    """[Ns,N,3], [Nr,M,3] -> [Ns,Nr] approximate-EMD matrix (each entry = emd_approx of the pair)."""
    if not sample_pcs.is_cuda or not ref_pcs.is_cuda:
        raise L.LionError("lion_b200 needs CUDA tensors; there is no CPU path")
    s = sample_pcs.detach().to(torch.float32).contiguous()
    r = ref_pcs.detach().to(torch.float32).contiguous()
    assert s.dim() == 3 and r.dim() == 3 and s.shape[2] == 3 and r.shape[2] == 3
    out = torch.empty(s.shape[0], r.shape[0], device=s.device)
    with torch.cuda.device(s.device):
        L.check(L.lib().lion_emd_pairwise(L.ptr(s), L.ptr(r), L.ptr(out), s.shape[0], r.shape[0], s.shape[1], r.shape[1],
                                          L.stream()), "emd_pairwise")
    return out / float(s.shape[1])


def _pairwise_EMD_CD_(metric, sample_pcs, ref_pcs, batch_size, require_grad=True, accelerated_cd=True, verbose=True):
    """Same signature and return convention as the reference: (all_cd, all_emd), both the CD matrix
    when metric == 'CD' (reference :311-314 returns the same list twice)."""
    if metric == 'CD':
        cd = pairwise_CD(sample_pcs, ref_pcs)
        return cd, cd
    if metric == 'EMD':
        emd = pairwise_EMD(sample_pcs, ref_pcs)
        return emd, emd
    raise NotImplementedError(metric)
