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
which does not exist in the reference tree.

The scores (reference :184-687): `compute_all_metrics` (MMD / COV / 1-NNA for CD and EMD) builds each of the three
matrices it needs once, where the reference builds M_rs twice; `knn` / `lgan_mmd_cov` run as torch ops on the device
of the matrices, as in the reference; `jsd_between_point_cloud_sets` finds every point's nearest grid cell with
lion_occupancy_grid instead of sklearn's NearestNeighbors and per-point Python loops, and keeps the entropy and
divergence in float64 numpy / scipy.  `EMD_CD`, `print_results` and `write_results` keep the reference's
signatures and column text."""
import warnings

import numpy as np
import torch
from loguru import logger
from scipy.stats import entropy
from tabulate import tabulate

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


def _require_cuda(*tensors):
    for t in tensors:
        if not (torch.is_tensor(t) and t.is_cuda):
            raise L.LionError("lion_b200 needs CUDA tensors; there is no CPU path")


def EMD_CD(sample_pcs, ref_pcs, batch_size, accelerated_cd=False, reduced=True, require_grad=False):
    """Paired CD and EMD of sample i against reference i, in batches of batch_size (reference :184-226).  The Chamfer
    distances always come from the library's kernel (accelerated_cd is accepted for the reference's signature)."""
    n_sample, n_ref = sample_pcs.shape[0], ref_pcs.shape[0]
    assert n_sample == n_ref, "REF:%d SMP:%d" % (n_ref, n_sample)
    cd, emd = [], []
    for a in range(0, n_sample, batch_size):
        s, r = sample_pcs[a:a + batch_size], ref_pcs[a:a + batch_size]
        dl, dr = distChamferCUDA(s, r) if require_grad else distChamferCUDAnograd(s, r)
        cd.append(dl.mean(dim=1) + dr.mean(dim=1))
        emd.append(emd_approx(s, r, require_grad=require_grad))
    cd, emd = torch.cat(cd), torch.cat(emd)
    if reduced:
        cd, emd = cd.mean(), emd.mean()
    return {'MMD-CD': cd, 'MMD-EMD': emd}


def formulate_results(results, dataset, hash, step, epoch):
    """(header words, value words) of one score line (reference :229-250)."""
    reported = '' if step == '' and epoch == '' else f'S{step}E{epoch}'
    head, line = [], []
    if dataset != '-':
        head.append('Dataset')
        line.append(f'{dataset}')
    if hash != '-':
        head.append('Model')
        line.append(f'{hash}')
    if step != '' or epoch != '':
        head.append('reported')
        line.append(reported)
    g = lambda k: results.get(k, 0)
    head += ['MMD-CDx0.001↓', 'MMD-EMDx0.01↓', 'COV-CD%↑', 'COV-EMD%↑', '1-NNA-CD%↓',
             '1-NNA-EMD%↓', 'JSD↓']
    line += [f"{g('lgan_mmd-CD') * 1000:.4f}", f"{g('lgan_mmd-EMD') * 100:.4f}", f"{g('lgan_cov-CD') * 100:.2f}",
             f"{g('lgan_cov-EMD') * 100:.2f}", f"{g('1-NN-CD-acc') * 100:.2f}", f"{g('1-NN-EMD-acc') * 100:.2f}",
             f"{g('jsd'):.2f}"]
    if results.get('url', None) is not None:
        head.append('url')
        line.append(f"{results.get('url', '-')}")
    # the reference joins the words with single spaces and splits them again: a value containing a space is split too
    return ' '.join(head).split(' '), ' '.join(line).split(' ')


def write_results(out_file, results, dataset='', hash='', step='', epoch=''):
    """Append the score line, tab-separated with its header, to out_file (reference :253-260)."""
    head, line = formulate_results(results, dataset, hash, step, epoch)
    text = tabulate([line], head, tablefmt="tsv")
    with open(out_file, "a") as f:
        f.write(text + '\n')
    return text


def print_results(results, dataset='-', hash='-', step='', epoch=''):
    """Log the score line as a plain table (reference :263-269)."""
    head, line = formulate_results(results, dataset, hash, step, epoch)
    msg = tabulate([line], head, tablefmt="plain")
    logger.info('\n{}', msg)
    return msg


def knn(Mxx, Mxy, Myy, k, sqrt=False):
    """k-nearest-neighbour two-sample test on the block matrix [[Mxx, Mxy], [Mxy^T, Myy]] (reference :406-445).
    The x set (refs in compute_all_metrics) is labelled 1, the y set 0; every element is classified by the majority
    label of its k nearest others (topk along dim 0, ties resolved by torch on the matrices' device)."""
    n0, n1 = Mxx.size(0), Myy.size(0)
    label = torch.cat((torch.ones(n0), torch.zeros(n1))).to(Mxx)
    M = torch.cat((torch.cat((Mxx, Mxy), 1), torch.cat((Mxy.transpose(0, 1), Myy), 1)), 0)
    if sqrt:
        M = M.abs().sqrt()
    M = M + torch.diag(torch.full((n0 + n1,), float('inf'), dtype=Mxx.dtype, device=Mxx.device))   # not one's own neighbour
    _, idx = M.topk(k, 0, False)
    count = torch.zeros(n0 + n1).to(Mxx)
    for i in range(k):
        count = count + label.index_select(0, idx[i])
    pred = torch.ge(count, (float(k) / 2) * torch.ones(n0 + n1).to(Mxx)).float()
    s = {'tp': (pred * label).sum(), 'fp': (pred * (1 - label)).sum(),
         'fn': ((1 - pred) * label).sum(), 'tn': ((1 - pred) * (1 - label)).sum()}
    s['precision'] = s['tp'] / (s['tp'] + s['fp'] + 1e-10)
    s['recall'] = s['tp'] / (s['tp'] + s['fn'] + 1e-10)
    s['acc_t'] = s['tp'] / (s['tp'] + s['fn'] + 1e-10)
    s['acc_f'] = s['tn'] / (s['tn'] + s['fp'] + 1e-10)
    s['acc'] = torch.eq(label, pred).float().mean()
    return s


def lgan_mmd_cov(all_dist):
    """all_dist [N_sample, N_ref] -> MMD (mean over refs of the distance to the closest sample), COV (share of refs
    that are some sample's closest ref) and MMD from the sample side (reference :448-460)."""
    n_ref = all_dist.size(1)
    min_from_smp, min_idx = torch.min(all_dist, dim=1)
    min_from_ref, _ = torch.min(all_dist, dim=0)
    cov = float(min_idx.unique().view(-1).size(0)) / float(n_ref)
    return {'lgan_mmd': min_from_ref.mean(), 'lgan_cov': torch.tensor(cov).to(all_dist),
            'lgan_mmd_smp': min_from_smp.mean()}


# Every score matrix is issued in row chunks of at most LAUNCH_WORK[metric] point pairs (cloud pairs x N x M) per
# launch, so that no single launch holds a shared GPU for much more than a second.  Measured on an H100 80GB HBM3 at a
# 700 W power limit with 2048-point clouds: lion_chamfer_pairwise 2.4 us and lion_emd_pairwise 65.8 us per cloud pair.
LAUNCH_WORK = {'CD': 400000 * 2048 * 2048, 'EMD': 15000 * 2048 * 2048}


def _rows(metric, a, b):
    """pairwise_CD / pairwise_EMD(a, b) in row chunks; every entry is computed as in one call, bit for bit."""
    if metric not in LAUNCH_WORK:
        raise NotImplementedError(metric)
    fn = pairwise_CD if metric == 'CD' else pairwise_EMD
    rows = max(1, LAUNCH_WORK[metric] // (b.shape[0] * a.shape[1] * b.shape[1]))
    return torch.cat([fn(a[i:i + rows], b) for i in range(0, a.shape[0], rows)])


def _score_matrices(metric, ref_pcs, sample_pcs):
    """(M_rs, M_rr, M_ss) of one metric, refs as the rows of M_rs, each matrix computed once."""
    return _rows(metric, ref_pcs, sample_pcs), _rows(metric, ref_pcs, ref_pcs), _rows(metric, sample_pcs, sample_pcs)


@torch.no_grad()
def compute_all_metrics(sample_pcs, ref_pcs, batch_size, verbose=True, accelerated_cd=False, metric1='CD',
                        metric2='EMD', **print_kwargs):
    """MMD, COV and 1-NNA of sample_pcs [Ns,N,3] against ref_pcs [Nr,M,3] (CUDA tensors) under metric1 and, unless it
    is None, metric2 (reference :463-560): keys lgan_mmd-*, lgan_cov-*, lgan_mmd_smp-*, 1-NN-*-acc_t, 1-NN-*-acc_f,
    1-NN-*-acc.  batch_size and accelerated_cd are accepted for the reference's signature; the matrix kernels need
    neither."""
    _require_cuda(sample_pcs, ref_pcs)
    results = {}
    for metric in (metric1, metric2):
        if metric is None:
            continue
        if verbose:
            logger.info('eval metric: {}; device: {}, {}', metric, ref_pcs.device, sample_pcs.device)
        M_rs, M_rr, M_ss = _score_matrices(metric, ref_pcs, sample_pcs)
        results.update({'%s-%s' % (k, metric): v.item() for k, v in lgan_mmd_cov(M_rs.t()).items()})
        if verbose:
            print_results(results, **print_kwargs)
        one_nn = knn(M_rr, M_rs, M_ss, 1, sqrt=False)
        results.update({'1-NN-%s-%s' % (metric, k): v.item() for k, v in one_nn.items() if 'acc' in k})
        if verbose:
            print_results(results, **print_kwargs)
    return results


# ---- JSD (reference :566-687, after github.com/optas/latent_3d_points) ------------------------------------------------
def unit_cube_grid_point_cloud(resolution, clip_sphere=False):
    """Centres of a resolution^3 grid spanning the unit cube, (cells [r,r,r,3] or, with clip_sphere, [K,3] of the
    cells whose float32 norm is <= 0.5; spacing).  Each coordinate is the float64 value i * spacing - 0.5 stored as
    float32, as the reference's element-wise assignments store it."""
    spacing = 1.0 / float(resolution - 1)
    axis = np.arange(resolution) * spacing - 0.5
    grid = np.empty((resolution, resolution, resolution, 3), np.float32)
    grid[..., 0] = axis[:, None, None]
    grid[..., 1] = axis[None, :, None]
    grid[..., 2] = axis[None, None, :]
    if clip_sphere:
        grid = grid.reshape(-1, 3)
        grid = grid[np.linalg.norm(grid, axis=1) <= 0.5]
    return grid, spacing


def _to_cuda(x):
    """numpy array or tensor -> contiguous float32 CUDA tensor (its own device, or the current one)."""
    if not torch.cuda.is_available():
        raise L.LionError("lion_b200 needs a CUDA device; there is no CPU path")
    t = torch.as_tensor(x)
    dev = t.device if t.is_cuda else torch.device('cuda', torch.cuda.current_device())
    return t.detach().to(dev, torch.float32).contiguous()


def occupancy_counts(pclouds, cells):
    """pclouds [S,N,3], cells [K,3] -> (point_counts [K], cloud_counts [K]) int32 numpy arrays: how many points, and
    how many clouds, have each cell as their nearest (exact float64 distance, lowest index on a tie)."""
    x = _to_cuda(pclouds)
    c = torch.as_tensor(cells, dtype=torch.float32).to(x.device).contiguous()
    assert x.dim() == 3 and x.shape[2] == 3 and c.dim() == 2 and c.shape[1] == 3
    k = c.shape[0]
    point_counts = torch.empty(k, dtype=torch.int32, device=x.device)
    cloud_counts = torch.empty(k, dtype=torch.int32, device=x.device)
    with torch.cuda.device(x.device):
        L.check(L.lib().lion_occupancy_grid(L.ptr(x), L.ptr(c), x.shape[0], x.shape[1], k, L.ptr(point_counts),
                                            L.ptr(cloud_counts), L.stream()), "occupancy_grid")
    return point_counts.cpu().numpy(), cloud_counts.cpu().numpy()


def entropy_of_occupancy_grid(pclouds, grid_resolution, in_sphere=False, verbose=False):
    """(mean over cells of the entropy of "the cell is occupied by a cloud", point count of every cell [K] float64)
    for a set of clouds [S,N,3] (numpy or torch), the cells being those of unit_cube_grid_point_cloud."""
    x = _to_cuda(pclouds)
    bound = 0.5 + 10e-4
    if verbose and (abs(x.max().item()) > bound or abs(x.min().item()) > bound):
        warnings.warn('Point-clouds are not in unit cube.')
    if verbose and in_sphere and x.norm(dim=2).max().item() > bound:
        warnings.warn('Point-clouds are not in unit sphere.')
    cells, _ = unit_cube_grid_point_cloud(grid_resolution, in_sphere)
    cells = cells.reshape(-1, 3)
    point_counts, cloud_counts = occupancy_counts(x, cells)
    return occupancy_entropy(cloud_counts, x.shape[0]), point_counts.astype(np.float64)


def occupancy_entropy(cloud_counts, n_clouds):
    """Mean over all cells of the entropy (nats) of the Bernoulli variable "a cloud occupies the cell", estimated
    from how many of n_clouds clouds occupy each cell."""
    p = cloud_counts[cloud_counts > 0] / float(n_clouds)
    acc = float(entropy(np.stack((p, 1.0 - p)), axis=0).sum()) if p.size else 0.0
    return acc / len(cloud_counts)


def jsd_between_point_cloud_sets(sample_pcs, ref_pcs, resolution=28):
    """Jensen-Shannon divergence between the occupancy distributions of two sets of clouds (numpy or torch, [S,N,3])
    over the in-sphere cells of a resolution^3 grid."""
    sample_grid_var = entropy_of_occupancy_grid(sample_pcs, resolution, True)[1]
    ref_grid_var = entropy_of_occupancy_grid(ref_pcs, resolution, True)[1]
    return jensen_shannon_divergence(sample_grid_var, ref_grid_var)


def jensen_shannon_divergence(P, Q):
    if np.any(P < 0) or np.any(Q < 0):
        raise ValueError('Negative values.')
    if len(P) != len(Q):
        raise ValueError('Non equal size.')
    P_, Q_ = P / np.sum(P), Q / np.sum(Q)
    res = entropy((P_ + Q_) / 2.0, base=2) - (entropy(P_, base=2) + entropy(Q_, base=2)) / 2.0
    if not np.allclose(res, _jsdiv(P_, Q_), atol=10e-5, rtol=0):
        warnings.warn('Numerical values of two JSD methods don\'t agree.')
    return res


def _jsdiv(P, Q):
    """The same divergence as the mean of the two KL divergences to the midpoint distribution."""
    def kl(a, b):
        keep = np.logical_and(a > 0, b > 0)
        a, b = a[keep], b[keep]
        return np.sum(a * np.log2(a / b))
    P_, Q_ = P / np.sum(P), Q / np.sum(Q)
    M = 0.5 * (P_ + Q_)
    return 0.5 * (kl(P_, M) + kl(Q_, M))
