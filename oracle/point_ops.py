"""CPU restatement of the reference's point<->voxel and neighbourhood operators.

TEST INFRASTRUCTURE ONLY.  Nothing in the product path (lion_b200/) may import this file;
only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs do.

Every function restates one CUDA kernel of the reference's third_party/pvcnn extension
(paths below are relative to third_party/pvcnn/functional/ in the reference) in vectorised
torch-CPU / numpy, fp32, keeping the reference's tie-breaking, padding and clamping rules.

Parity status: PINNED ON THE GPU BOX ONLY.  The reference ships no golden vectors or tests
for these kernels (SURVEY.md section 4) and its kernels cannot execute in the CPU container;
tests/test_point_ops_gpu.py checks this file and the product kernels against the reference's
own kernels compiled into oracle/_ref/ (oracle/build_ref.py).  Distances are evaluated with
the FMA contraction nvcc applies to the reference sources (see `_sqdist`), emulated in
float64; a double-rounding mismatch is possible in principle (never observed).
"""
import numpy as np
import torch


# --------------------------------------------------------------------------------------
# helpers
# --------------------------------------------------------------------------------------
def _f32(x):
    return np.asarray(x, dtype=np.float32)


def _fma32(a, b, c):
    """fmaf(a,b,c) for float32 arrays, via float64 (a*b is exact in float64)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def _sqdist(dx, dy, dz):
    """dx*dx + dy*dy + dz*dz as nvcc -O3 compiles it in the reference kernels
    (sampling.cu:134-135, ball_query.cu:34-38, neighbor_interpolate.cu:42):
    FMUL t=dy*dy ; FFMA t=dx*dx+t ; FFMA t=dz*dz+t  (read off `cuobjdump -sass
    oracle/_ref/_pvcnn_backend.so`: the first product of the left-most add is the one that
    gets fused)."""
    dx, dy, dz = _f32(dx), _f32(dy), _f32(dz)
    t = (dy * dy).astype(np.float32)
    t = _fma32(dx, dx, t)
    return _fma32(dz, dz, t)


# --------------------------------------------------------------------------------------
# Voxelization.forward  (models/pvcnn2_ada.py:173-188)
# --------------------------------------------------------------------------------------
def voxel_coords(coords, r, normalize=True, eps=0.0):
    """coords [B,3,N] fp32 -> (norm_coords [B,3,N] fp32 in [0,r-1], vox [B,3,N] int32).

    centre by the mean over points; scale by 2*max_n ||c||_2 (+eps); shift .5; times r;
    clamp [0,r-1]; round half-to-even (pvcnn2_ada.py:177-185)."""
    coords = torch.as_tensor(coords, dtype=torch.float32)
    nc = coords - coords.mean(2, keepdim=True)
    if normalize:
        nc = nc / (nc.norm(dim=1, keepdim=True).max(dim=2, keepdim=True).values * 2.0 + eps) + 0.5
    else:
        nc = (nc + 1) / 2.0
    nc = torch.clamp(nc * r, 0, r - 1)
    vox = torch.round(nc).to(torch.int32)
    return nc, vox


def _last_pow2(n):
    p = 1
    while p * 2 <= n:
        p *= 2
    return p


def cuda_mean_lastdim(x):
    """`x.mean(2)` of a contiguous fp32 [B,3,N] tensor with the BITS torch's CUDA reduction produces
    (third-party arithmetic: PyTorch ATen/native/cuda/Reduce.cuh -- `reduce_kernel<512, 1, ReduceOp<float,
    MeanOps<...>>>`, vt0 = 4 -- restated from its published algorithm; pinned on the GPU box against
    torch itself by tests/test_point_ops_gpu.py::test_cuda_mean_emulation_matches_torch).

    The summation order depends on the number of outputs (3B) as well as on N:
      * reduction over the contiguous dimension; vectorised by 4 when N >= 128;
      * block = (W lanes along the reduction) x (H outputs): W0 = min(last_pow2(dim0), 32),
        H = min(last_pow2(3B), 512 / W0), W = min(last_pow2(dim0), 512 / H), dim0 = N/4 (vectorised) or N;
      * lane x keeps 4 accumulators: vectorised -> accumulator j sums elements 4*(x + k*W) + j, k = 0, 1, ...;
        otherwise accumulator (k mod 4) sums element x + k*W; leftovers (N % 4) go to accumulator 0 of lane
        (element - tail_start); the accumulators are folded ((a0 + a1) + a2) + a3;
      * lanes are folded by a shared-memory tree for offsets W/2 ... 32 (x += x[+offset]) and then a
        shuffle-down tree with offsets 16, 8, 4, 2, 1; the result is multiplied by float(3B) / float(3B*N).
    Rows whose start is not 16-byte aligned (N % 4 != 0) go through Reduce.cuh's head-alignment path; that case
    is restated too (shift = row offset mod 4)."""
    x = np.ascontiguousarray(np.asarray(x, dtype=np.float32))
    B, C, N = x.shape
    n_out = B * C
    vec = N >= 128
    dim0 = N // 4 if vec else N
    d0p = _last_pow2(dim0) if dim0 < 512 else 512
    d1p = _last_pow2(n_out) if n_out < 512 else 512
    W = min(d0p, 32)
    H = min(d1p, 512 // W)
    W = min(d0p, 512 // H)
    factor = np.float32(n_out) / np.float32(n_out * N)
    out = np.zeros((B, C), np.float32)
    f32 = np.float32
    for o in range(n_out):
        row = x.reshape(n_out, N)[o]
        acc = np.zeros((W, 4), np.float32)
        if vec:
            data, end = row, N
            shift = (o * N) % 4                      # elements past the previous 16-byte boundary (base is aligned)
            if shift > 0:
                # head: lanes shift..3 take one element each of the first (partial) vector
                for lane in range(shift, 4):
                    if lane < W and lane - shift < N:
                        acc[lane, 0] = f32(acc[lane, 0] + row[lane - shift])
                data = row[4 - shift:]
                end = N + shift - 4
            nvec = max(end, 0) // 4
            for idx in range(nvec):
                lane = idx % W
                v = data[4 * idx:4 * idx + 4]
                acc[lane] = (acc[lane] + v).astype(np.float32)
            tail_start = end - end % 4 if end > 0 else 0
            for i in range(tail_start, max(end, 0)):
                lane = i - tail_start
                acc[lane, 0] = f32(acc[lane, 0] + data[i])
        else:
            for lane in range(min(W, N)):
                k = 0
                idx = lane
                while idx + 3 * W < N:               # unrolled by vt0 = 4: accumulator i takes element idx + i*W
                    for i in range(4):
                        acc[lane, i] = f32(acc[lane, i] + row[idx + i * W])
                    idx += 4 * W
                i = 0
                while idx < N and i < 4:
                    acc[lane, i] = f32(acc[lane, i] + row[idx])
                    idx += W
                    i += 1
        v = acc[:, 0].copy()
        for j in range(1, 4):
            v = (v + acc[:, j]).astype(np.float32)
        off = W // 2
        while off >= 32:                             # shared-memory tree
            v[:off] = (v[:off] + v[off:2 * off]).astype(np.float32)
            off //= 2
        w = v[:min(W, 32)].copy()
        if len(w) < 32:
            w = np.concatenate([w, np.zeros(32 - len(w), np.float32)])   # lanes >= W hold the identity
        off = min(W, 32) // 2
        while off > 0:                               # shuffle-down tree, offsets DEcreasing (lane i += lane i+off)
            sh = np.concatenate([w[off:], w[-off:]])
            w = (w + sh).astype(np.float32)
            off //= 2
        out[o // C, o % C] = f32(w[0] * factor)
    return out


def voxel_coords_cuda_order(coords, r, normalize=True, eps=0.0):
    """Voxelization.forward (models/pvcnn2_ada.py:173-188) with the bits torch produces ON CUDA: only the mean
    depends on the device (summation order); the 3-term norm, max, division, scale, clamp and round are
    order-free.  coords [B,3,N] -> (norm_coords, vox int32)."""
    c = np.ascontiguousarray(np.asarray(coords, dtype=np.float32))
    mean = cuda_mean_lastdim(c)[:, :, None]
    nc = (c - mean).astype(np.float32)
    if normalize:
        sq = (nc * nc).astype(np.float32)
        nrm = np.sqrt(((sq[:, 0] + sq[:, 1]).astype(np.float32) + sq[:, 2]).astype(np.float32)).astype(np.float32)
        den = (nrm.max(axis=1) * np.float32(2.0) + np.float32(eps)).astype(np.float32)[:, None, None]
        nc = ((nc / den).astype(np.float32) + np.float32(0.5)).astype(np.float32)
    else:
        nc = ((nc + np.float32(1.0)) / np.float32(2.0)).astype(np.float32)
    nc = np.clip((nc * np.float32(r)).astype(np.float32), np.float32(0), np.float32(r - 1))
    t = torch.from_numpy(nc)
    return t, torch.round(t).to(torch.int32)


def round_to_voxel(norm_coords):
    """The integer part only: round-half-even of already normalised coordinates."""
    return torch.round(torch.as_tensor(norm_coords, dtype=torch.float32)).to(torch.int32)


# --------------------------------------------------------------------------------------
# avg_voxelize  (src/voxelization/vox.cu:18-34 grid_stats, :48-72 avg_voxelize; vox.cpp:17-43)
# --------------------------------------------------------------------------------------
def avg_voxelize(features, vox, r):
    """features [B,C,N] fp32, vox [B,3,N] int -> (out [B,C,r,r,r], ind [B,N] int32, cnt [B,r^3] int32).

    ind = x*r^2 + y*r + z (vox.cu:31); out[b,c,ind] = sum_i feat[b,c,i] * (1/cnt) (vox.cu:66-68).
    The reference accumulates with float atomics in arbitrary order; here the sum runs in
    ascending point index (one admissible order)."""
    features = torch.as_tensor(features, dtype=torch.float32)
    vox = torch.as_tensor(vox).to(torch.int64)
    B, C, N = features.shape
    r3 = r * r * r
    ind = vox[:, 0] * (r * r) + vox[:, 1] * r + vox[:, 2]                 # [B,N]
    cnt = torch.zeros(B, r3, dtype=torch.int32)
    cnt.scatter_add_(1, ind, torch.ones_like(ind, dtype=torch.int32))
    inv = (1.0 / cnt.to(torch.float32).gather(1, ind)).to(torch.float32)  # 1.0/float(cnt) (vox.cu:65)
    out = torch.zeros(B, C, r3, dtype=torch.float32)
    out.scatter_add_(2, ind[:, None, :].expand(B, C, N), features * inv[:, None, :])
    return out.view(B, C, r, r, r), ind.to(torch.int32), cnt


# --------------------------------------------------------------------------------------
# trilinear_devoxelize  (src/interpolate/trilinear_devox.cu:21-105)
# --------------------------------------------------------------------------------------
def trilinear_corners(coords, r):
    """coords [B,3,N] fp32 (already in voxel units, clamped to [0,r-1]) ->
    (idx [B,8,N] int64, wgt [B,8,N] fp32) in the reference's corner order 000,001,...,111
    (x major, z minor).  The hi-corner offset is 0 when the fractional part is 0
    (trilinear_devox.cu:64-66), so indices stay inside the grid."""
    c = torch.as_tensor(coords, dtype=torch.float32)
    lo = torch.floor(c)
    d1 = c - lo
    d0 = 1.0 - d1
    x0, y0, z0 = d0[:, 0], d0[:, 1], d0[:, 2]
    x1, y1, z1 = d1[:, 0], d1[:, 1], d1[:, 2]
    # weights: ((x*y)*z) left-to-right as written in the kernel (:53-60)
    w = torch.stack([x0 * y0 * z0, x0 * y0 * z1, x0 * y1 * z0, x0 * y1 * z1,
                     x1 * y0 * z0, x1 * y0 * z1, x1 * y1 * z0, x1 * y1 * z1], dim=1)
    lo_i = lo.to(torch.int64)
    hx = (d1[:, 0] > 0).to(torch.int64) * (r * r)
    hy = (d1[:, 1] > 0).to(torch.int64) * r
    hz = (d1[:, 2] > 0).to(torch.int64)
    i000 = lo_i[:, 0] * (r * r) + lo_i[:, 1] * r + lo_i[:, 2]
    idx = torch.stack([i000, i000 + hz, i000 + hy, i000 + hy + hz,
                       i000 + hx, i000 + hx + hz, i000 + hx + hy, i000 + hx + hy + hz], dim=1)
    return idx, w


def trilinear_devoxelize(features, coords, r):
    """features [B,C,r,r,r] (or [B,C,r^3]), coords [B,3,N] -> [B,C,N]:
    sum over the 8 corners in the kernel's order (:97-102)."""
    features = torch.as_tensor(features, dtype=torch.float32)
    B, C = features.shape[:2]
    f = features.reshape(B, C, -1)
    idx, w = trilinear_corners(coords, r)
    N = idx.shape[-1]
    out = None
    for k in range(8):
        g = f.gather(2, idx[:, k][:, None, :].expand(B, C, N)) * w[:, k][:, None, :]
        out = g if out is None else out + g
    return out


# --------------------------------------------------------------------------------------
# furthest_point_sample / gather  (src/sampling/sampling.cu:86-167, :17-31; sampling.cpp:43-58)
# --------------------------------------------------------------------------------------
FPS_BLOCK = 512  # the reference launches <<<b, 512>>> unconditionally (sampling.cu:171)


def furthest_point_sample_idx(coords, m):
    """coords [B,3,N] fp32 -> idx [B,m] int32.

    First pick is point 0; running min-distance starts at 1e38 (sampling.cpp:54); each round
    picks argmax of the updated min-distance.  Ties: thread t scans k=t,t+512,... with strict
    '>' (keeps its smallest k), then the tree reduction keeps the lower slot unless the upper
    is strictly larger (sampling.cu:141-157) => winner = max distance, then smallest k%512,
    then smallest k."""
    c = _f32(torch.as_tensor(coords).numpy() if isinstance(coords, torch.Tensor) else coords)
    B, _, N = c.shape
    idx = np.zeros((B, m), dtype=np.int32)
    dist = np.full((B, N), 1e38, dtype=np.float32)
    k = np.arange(N)
    # rank used to break ties exactly like the block reduction
    order_key = (k % FPS_BLOCK).astype(np.int64) * N + k
    tie_order = np.argsort(order_key, kind="stable")      # positions sorted by preference
    old = np.zeros(B, dtype=np.int64)
    ar = np.arange(B)
    for j in range(1, m):
        p = c[ar, :, old]                                  # [B,3]
        d = _sqdist(c[:, 0] - p[:, 0:1], c[:, 1] - p[:, 1:2], c[:, 2] - p[:, 2:3])
        dist = np.minimum(d, dist)
        # note: threads beyond N contribute best=-1 and never win (distances are >= 0)
        dd = dist[:, tie_order]
        win = tie_order[np.argmax(dd, axis=1)]             # first max in preference order
        old = win
        idx[:, j] = win
    return torch.from_numpy(idx)


def gather(features, idx):
    """features [B,C,N], idx [B,M] -> [B,C,M]  (sampling.cu:28-30)."""
    features = torch.as_tensor(features)
    idx = torch.as_tensor(idx).to(torch.int64)
    B, C, _ = features.shape
    return features.gather(2, idx[:, None, :].expand(B, C, idx.shape[1]))


def furthest_point_sample(coords, m):
    """sampling.py:39-54: centres' coordinates [B,3,m]."""
    return gather(torch.as_tensor(coords, dtype=torch.float32), furthest_point_sample_idx(coords, m))


# --------------------------------------------------------------------------------------
# ball_query  (src/ball_query/ball_query.cu:19-50; ball_query.cpp:20-22 zero-init)
# --------------------------------------------------------------------------------------
def ball_query(centers, points, radius, k):
    """centers [B,3,M], points [B,3,N] -> int32 [B,M,k]: the first k point indices (ascending)
    with d^2 < r^2 (strict, float r2 = radius*radius computed in float, ball_query.cpp),
    padded with the first hit; no hit -> zeros."""
    ce = _f32(torch.as_tensor(centers).numpy())
    pt = _f32(torch.as_tensor(points).numpy())
    B, _, M = ce.shape
    N = pt.shape[2]
    r2 = np.float32(np.float32(radius) * np.float32(radius))
    out = np.zeros((B, M, k), dtype=np.int32)
    for b in range(B):
        d2 = _sqdist(ce[b, 0][:, None] - pt[b, 0][None, :],
                     ce[b, 1][:, None] - pt[b, 1][None, :],
                     ce[b, 2][:, None] - pt[b, 2][None, :])          # [M,N]
        hit = d2 < r2
        rank = np.cumsum(hit, axis=1) - 1                            # position among hits
        nhit = hit.sum(axis=1)
        first = np.argmax(hit, axis=1)                               # 0 if none (zeros anyway)
        row = np.where(nhit[:, None] > 0, first[:, None], 0) * np.ones((1, k), dtype=np.int64)
        mm, nn = np.nonzero(hit & (rank < k))
        row[mm, rank[mm, nn]] = nn
        out[b] = row.astype(np.int32)
    return torch.from_numpy(out)


# --------------------------------------------------------------------------------------
# grouping  (src/grouping/grouping.cu:18-36)
# --------------------------------------------------------------------------------------
def grouping(features, idx):
    """features [B,C,N], idx [B,M,U] -> [B,C,M,U]."""
    features = torch.as_tensor(features)
    idx = torch.as_tensor(idx).to(torch.int64)
    B, C, _ = features.shape
    M, U = idx.shape[1:]
    return features.gather(2, idx.reshape(B, 1, M * U).expand(B, C, M * U)).view(B, C, M, U)


# --------------------------------------------------------------------------------------
# nearest_neighbor_interpolate  (src/interpolate/neighbor_interpolate.cu:20-75, :90-116)
# --------------------------------------------------------------------------------------
def three_nn(points, centers):
    """points [B,3,N], centers [B,3,M] -> (idx [B,3,N] int32, wgt [B,3,N] fp32).

    Brute-force 3 smallest squared distances with the kernel's strict '<' cascade (a later
    centre never displaces an equal earlier one), clamp to [1e-10,1e10], weights
    d1d2/(d0d1+d0d2+d1d2) etc. (:61-73).  With fewer than three centres the missing slots keep
    the kernel's initial index 0 and distance 1e40 (:37-38), which the clamp turns into 1e10."""
    pt = _f32(torch.as_tensor(points).numpy())
    ce = _f32(torch.as_tensor(centers).numpy())
    B, _, N = pt.shape
    M = ce.shape[2]
    idx = np.zeros((B, 3, N), dtype=np.int32)
    wgt = np.zeros((B, 3, N), dtype=np.float32)
    for b in range(B):
        d = _sqdist(pt[b, 0][:, None] - ce[b, 0][None, :],
                    pt[b, 1][:, None] - ce[b, 1][None, :],
                    pt[b, 2][:, None] - ce[b, 2][None, :])           # [N,M]
        order = np.argsort(d, axis=1, kind="stable")[:, :3]          # stable == strict '<' cascade
        best = np.take_along_axis(d, order, axis=1).astype(np.float32)
        if M < 3:  # unreachable in LION (M >= 16): the slots no centre filled keep index 0 and 1e40
            order = np.concatenate([order, np.zeros((N, 3 - M), dtype=order.dtype)], axis=1)
            best = np.concatenate([best, np.full((N, 3 - M), np.inf, dtype=np.float32)], axis=1)
        best = np.maximum(np.minimum(np.float32(1e10), best), np.float32(1e-10))
        d0, d1, d2 = best[:, 0], best[:, 1], best[:, 2]
        d0d1 = (d0 * d1).astype(np.float32)
        d0d2 = (d0 * d2).astype(np.float32)
        d1d2 = (d1 * d2).astype(np.float32)
        inv = (np.float32(1.0) / ((d0d1 + d0d2).astype(np.float32) + d1d2).astype(np.float32)).astype(np.float32)
        wgt[b, 0] = d1d2 * inv
        wgt[b, 1] = d0d2 * inv
        wgt[b, 2] = d0d1 * inv
        idx[b] = order.T.astype(np.int32)
    return torch.from_numpy(idx), torch.from_numpy(wgt)


def nearest_neighbor_interpolate(points, centers, centers_features):
    """-> [B,C,N] = cf[.,i0]*w0 + cf[.,i1]*w1 + cf[.,i2]*w2 (:112-114)."""
    cf = torch.as_tensor(centers_features, dtype=torch.float32)
    idx, wgt = three_nn(points, centers)
    B, C, _ = cf.shape
    N = idx.shape[2]
    out = None
    for j in range(3):
        g = cf.gather(2, idx[:, j].to(torch.int64)[:, None, :].expand(B, C, N)) * wgt[:, j][:, None, :]
        out = g if out is None else out + g
    return out
