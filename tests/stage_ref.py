"""Float64 references of the stages of a PVConv (first convolution, AdaGN-1 + Swish grid, second convolution, SE fold,
point branch, devoxelisation), of the linear attention and of the SA module's MLP -- with their operands modelled the
way the kernels hand them to the tensor cores -- and the point clouds the stage tests run them on.

Operand model (TF32 = 10 explicit mantissa bits):
  * packed weights are rounded to nearest, ties away from zero (cvt.rna, csrc/conv_tc.cu), like every operand a kernel
    rounds itself (k_act_rows with flag 1, the fused SA pass 2);
  * an fp32 operand that no kernel rounds (the scatter grid, the compact voxel list, the gathered SA rows) is read by
    the tensor core with its low 13 mantissa bits ignored: truncation toward zero.
"""
import numpy as np
import torch

from oracle import point_ops as OP


def tf32_rna(x):
    """cvt.rna.tf32.f32: round the magnitude to 10 mantissa bits, ties away from zero."""
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1fff).view(torch.float32)


def tf32_trunc(x):
    """An fp32 operand as the tensor core reads it in TF32 mode: the low 13 mantissa bits dropped."""
    i = x.contiguous().view(torch.int32)
    return (i & ~0x1fff).view(torch.float32)


# ---------------------------------------------------------------------------------------------------------------------
# point clouds [3, N]
# ---------------------------------------------------------------------------------------------------------------------
def gaussian_cloud(seed, N, scale=0.4):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(3, N, generator=g) * scale


def clustered_cloud(N):
    """Every point but six at the origin, one voxel; the six on the axes at distance 1 land on the grid's faces
    (voxel coordinate 0 or r - 1).  Occupancy 7 at every resolution; one voxel list of N - 6 points."""
    c = torch.zeros(3, N)
    for k, (a, s) in enumerate([(0, 1.0), (0, -1.0), (1, 1.0), (1, -1.0), (2, 1.0), (2, -1.0)]):
        c[a, N - 6 + k] = s
    return c


def sites_cloud(K, N, r, seed):
    """K well-separated sites, each repeated, occupying exactly K voxels at (even) resolution r.

    In voxel units u, two anchors at (+-r/2, 0, 0) fix the largest centred norm at r/2, so a site u with |u| < r/2
    lands on voxel u + r/2 exactly (normalisation: (c - mean) / (2 max |c - mean|) + 1/2, times r).  Sites come in
    pairs +-u with equal repeat counts (plus the origin when K is odd), so the mean stays 0 and no site drifts."""
    assert r % 2 == 0 and 2 <= K <= N
    h = r // 2
    rng = np.random.default_rng(seed)
    ax = np.arange(-(h - 1), h)
    u = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    pos = (u[:, 0] > 0) | ((u[:, 0] == 0) & ((u[:, 1] > 0) | ((u[:, 1] == 0) & (u[:, 2] > 0))))   # one of each +-u
    u = u[pos & ((u * u).sum(1) < (h - 0.5) ** 2) & ~((u[:, 0] == h - 1) & (u[:, 1] == 0) & (u[:, 2] == 0))]
    npairs = (K - 2) // 2
    assert npairs <= len(u), (K, r)
    pick = u[rng.permutation(len(u))[:npairs]]
    sites = [np.array([h, 0, 0]), np.array([-h, 0, 0])]
    for p in pick:
        sites += [p, -p]
    if K % 2:
        sites.append(np.zeros(3, dtype=np.int64))
    sites = np.stack(sites).astype(np.float64)
    cnt = np.full(K, N // K)
    left = N - cnt.sum()
    i = 0
    while left >= 2:                                   # extra points go to whole pairs
        cnt[i] += 1; cnt[i + 1] += 1
        left -= 2; i = (i + 2) % (K - K % 2)
    if left:
        cnt[K - 1] += 1                                # K odd: the origin
    pts = np.repeat(sites, cnt, axis=0)[rng.permutation(N)]
    return torch.from_numpy((pts * 0.03).T.astype(np.float32)).contiguous()


def voxel_ids(coords, r):
    """[B,3,N] -> the kernels' voxel index x r^2 + y r + z of every point (oracle, CUDA summation order)."""
    _, vox = OP.voxel_coords_cuda_order(coords, r)
    v = vox.to(torch.int64)
    return v[:, 0] * r * r + v[:, 1] * r + v[:, 2]


def occupancy(coords, r):
    ids = voxel_ids(coords, r)
    return [int(torch.unique(ids[b]).numel()) for b in range(ids.shape[0])]


# ---------------------------------------------------------------------------------------------------------------------
# first convolution of a PVConv
# ---------------------------------------------------------------------------------------------------------------------
def scatter_grid(features, ids, r):
    """The grid k_scatter / k_scatter_compact build: per voxel, its points in ascending order, acc = f0 * (1/n), then
    acc = fma(f_k, 1/n, acc) (the compiler contracts the kernel's multiply-add).  features [B,C,N] fp32 on the device,
    ids [B,N] -> [B,C,r,r,r] fp32."""
    B, C, N = features.shape
    dev = features.device
    V = r ** 3
    gid = (ids.to(dev) + torch.arange(B, device=dev)[:, None] * V).reshape(-1)          # [B*N] voxel of the batch
    cnt = torch.zeros(B * V, dtype=torch.int64, device=dev).scatter_add_(0, gid, torch.ones_like(gid))
    inv = (1.0 / cnt[gid].to(torch.float32)).double()
    order = torch.argsort(gid * N + torch.arange(B * N, device=dev) % N)              # by voxel, then point
    sg = gid[order]
    first = torch.ones_like(sg, dtype=torch.bool)
    first[1:] = sg[1:] != sg[:-1]
    start = torch.cummax(torch.where(first, torch.arange(B * N, device=dev), torch.zeros_like(sg)), 0).values
    rank = torch.empty_like(sg)
    rank[order] = torch.arange(B * N, device=dev) - start
    f = features.permute(0, 2, 1).reshape(B * N, C).double()
    acc = torch.zeros(B * V, C, dtype=torch.float32, device=dev)
    for k in range(int(rank.max()) + 1):
        sel = rank == k
        v = gid[sel]
        t = f[sel] * inv[sel, None]
        acc[v] = (t if k == 0 else acc[v].double() + t).float()
    return acc.view(B, V, C).permute(0, 2, 1).reshape(B, C, r, r, r).contiguous()


def conv3x3x3_f64(x, w, b):
    """27 shifted float64 matmuls + bias: x [B,Ci,r,r,r], w [Co,Ci,3,3,3] -> [B,Co,r,r,r] (zero padding 1)."""
    B, _, r = x.shape[0], x.shape[1], x.shape[2]
    xp = torch.nn.functional.pad(x, (1, 1, 1, 1, 1, 1))
    out = b.view(1, -1, 1, 1, 1).repeat(B, 1, r, r, r)
    for kx in range(3):
        for ky in range(3):
            for kz in range(3):
                out += torch.einsum("oc,bcxyz->boxyz", w[:, :, kx, ky, kz], xp[:, :, kx:kx + r, ky:ky + r, kz:kz + r])
    return out


def conv1_reference(features, coords, w, b, r, tc=True):
    """float64 reference of a PVConv's first convolution on the device of `features`."""
    rna, trunc = operand_models(tc)
    ids = voxel_ids(coords, r)
    g = scatter_grid(features, ids, r)
    return conv3x3x3_f64(trunc(g).double(), rna(w.to(features.device)).double(), b.to(features.device).double())


# ---------------------------------------------------------------------------------------------------------------------
# SA MLP
# ---------------------------------------------------------------------------------------------------------------------
def sa_rows(features, coords, centers, nidx):
    """Layer-1 operand [B, M, 32, 4 + Cf]: [p - c in fp32, 0 | features], as k_group_gather / the fused gather build it."""
    B, Cf, N = features.shape
    M, U = nidx.shape[1:]
    idx = nidx.reshape(B, 1, M * U).long()
    p = coords.gather(2, idx.expand(B, 3, M * U)).view(B, 3, M, U)
    d = p - centers[:, :, :, None]
    f = features.gather(2, idx.expand(B, Cf, M * U)).view(B, Cf, M, U)
    z = torch.zeros(B, 1, M, U, dtype=features.dtype, device=features.device)
    return torch.cat([d, z, f], 1).permute(0, 2, 3, 1).contiguous()


def fold_affine(ssum, ssq, gamma, beta, fb, count):
    """k_affine_prep in float64: GroupNorm(8) statistics from the per-channel sums, then AdaGN's factor / bias."""
    B, C = ssum.shape
    cpg = C // 8
    n = count * cpg
    mean = ssum.view(B, 8, cpg).sum(-1) / n
    var = (ssq.view(B, 8, cpg).sum(-1) / n - mean * mean).clamp_min(0)
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    mean, rstd = mean.repeat_interleave(cpg, 1), rstd.repeat_interleave(cpg, 1)
    f, bb = fb[:, :C], fb[:, C:]
    return rstd * gamma * f, (beta - mean * rstd * gamma) * f + bb


def swish_act(v32, scale, shift):
    """The next layer's operand: rna(swish(fma(v, scale, shift))), v fp32 [B,M,U,C], scale / shift fp32 [B,C]."""
    a = (v32.double() * scale[:, None, None, :].double() + shift[:, None, None, :].double()).float().double()
    return tf32_rna((a * torch.sigmoid(a)).float())


# ---------------------------------------------------------------------------------------------------------------------
# second half of a PVConv: AdaGN-1 + Swish grid, second convolution, SE fold, point branch, devoxelisation
#
# `tc` selects the operand model: True for layers the tensor-core kernels run (output widths that are multiples of
# 32), False for the SIMT kernels (and for comparisons with the fp32 oracle), which read every operand unrounded.
# ---------------------------------------------------------------------------------------------------------------------
def _ident(x):
    return x


def operand_models(tc):
    """(weight model, model of an fp32 operand no kernel rounds) for a tensor-core (tc) or SIMT layer."""
    return (tf32_rna, tf32_trunc) if tc else (_ident, _ident)


def act_grid(raw1, scale, shift, rna=True):
    """k_act_grid: rna(swish(fma(raw1, scale, shift))) on the interior, exactly 0 on the one-voxel halo.
    raw1 fp32 [B,C,r,r,r], scale / shift fp32 [B,C] -> fp32 [B,C,r+2,r+2,r+2]."""
    a = (raw1.double() * scale[:, :, None, None, None].double() + shift[:, :, None, None, None].double()).float().double()
    y = (a * torch.sigmoid(a)).float()
    if rna:
        y = tf32_rna(y)
    return torch.nn.functional.pad(y, (1, 1, 1, 1, 1, 1))


def fold_se(ssum, ssq, gamma, beta, fb, count, w1, w2):
    """k_affine_prep with the SE gate, in float64: fold AdaGN-2 from the sums, then SE3d's gate from the per-channel
    mean of its output, mean(scale x + shift) = scale mean(x) + shift; the gate multiplies scale and shift."""
    rs, rt = fold_affine(ssum, ssq, gamma, beta, fb, count)
    m = rs * (ssum / count) + rt
    gate = torch.sigmoid(torch.relu(m @ w1.double().T) @ w2.double().T)
    return rs * gate, rt * gate


def point_conv(features, w, b, tc=True):
    """The point branch's raw 1x1 convolution in float64: features fp32 [B,Ci,N], w [Co,Ci,1] -> [B,Co,N]."""
    rna, trunc = operand_models(tc)
    w = rna(w.reshape(w.shape[0], -1).contiguous()).double()
    return torch.einsum("oc,bcn->bon", w, trunc(features).double()) + b.double()[None, :, None]


def trilinear_f64(grid, nc, r):
    """Trilinear devoxelisation in float64: grid [B,C,r,r,r], nc [B,3,N] normalised coordinates in [0, r-1] ->
    [B,C,N].  A corner whose weight is 0 (fractional part 0) is not read."""
    B, C = grid.shape[:2]
    f = grid.reshape(B, C, -1)
    c = nc.to(grid.device).double()
    lo = torch.floor(c)
    d1 = c - lo
    lo = lo.long()
    hi = torch.minimum(lo + 1, torch.full_like(lo, r - 1))
    out = 0
    for kx in (0, 1):
        for ky in (0, 1):
            for kz in (0, 1):
                ix, iy, iz = [(hi if k else lo)[:, a] for a, k in enumerate((kx, ky, kz))]
                w = 1.0
                for a, k in enumerate((kx, ky, kz)):
                    w = w * (d1[:, a] if k else 1.0 - d1[:, a])
                idx = (ix * r + iy) * r + iz
                out = out + f.gather(2, idx[:, None, :].expand(B, C, idx.shape[-1])) * w[:, None, :]
    return out


def devox_fuse(raw2, s2, t2, nc, rawp, sp, tp):
    """k_devox_fuse in float64: trilinear(raw2 * s2 + t2) at nc, plus swish(rawp * sp + tp).  raw2 [B,C,r,r,r],
    rawp [B,C,N], scale / shift [B,C]."""
    r = raw2.shape[-1]
    g = raw2.double() * s2.double()[:, :, None, None, None] + t2.double()[:, :, None, None, None]
    a = rawp.double() * sp.double()[:, :, None] + tp.double()[:, :, None]
    return trilinear_f64(g, nc, r) + a * torch.sigmoid(a)


# ---------------------------------------------------------------------------------------------------------------------
# linear attention
# ---------------------------------------------------------------------------------------------------------------------
def attn_qkv(x, wqkv, tc=True):
    """to_qkv in float64: x fp32 [B,C,N], wqkv [3 H 32, C, 1, 1] -> [B, 3 H 32, N]."""
    rna, trunc = operand_models(tc)
    w = rna(wqkv.reshape(wqkv.shape[0], -1).contiguous()).double()
    return torch.einsum("oc,bcn->bon", w, trunc(x).double())


def attn_core(qkv, heads):
    """k_attn_ctx + k_attn_apply in float64: softmax over the points of k, ctx = k v^T, o = ctx^T q.
    qkv [B, 3 H 32, N] (channels ordered qkv, head, c) -> o [B, H 32, N]."""
    B, _, N = qkv.shape
    q, k, v = qkv.double().view(B, 3, heads, 32, N).unbind(1)
    k = torch.softmax(k, dim=-1)
    ctx = torch.einsum("bhdn,bhen->bhde", k, v)
    return torch.einsum("bhde,bhdn->bhen", ctx, q).reshape(B, heads * 32, N)


def attn_out(o, wo, bo, tc=True):
    """to_out in float64: o fp32 [B, H 32, N], wo [C, H 32, 1, 1] -> [B,C,N]."""
    rna, trunc = operand_models(tc)
    w = rna(wo.reshape(wo.shape[0], -1).contiguous()).double()
    return torch.einsum("oc,bcn->bon", w, trunc(o).double()) + bo.double()[None, :, None]


# ---------------------------------------------------------------------------------------------------------------------
# FP module: 3-NN interpolation, [interpolated | skip] concatenation, unpooled MLP; the U-Net's glue
# ---------------------------------------------------------------------------------------------------------------------
def interp_fma(cf, idx, wgt):
    """k_interp_rows in fp32: f0 * w0, then fma(f1, w1, .), then fma(f2, w2, .).  cf [B,C,M] fp32, idx [B,3,N], wgt
    [B,3,N] fp32 -> [B,C,N] fp32 (each fma through float64, where a * b is exact)."""
    B, C, _ = cf.shape
    N = idx.shape[-1]
    g = [cf.gather(2, idx[:, k].long()[:, None, :].expand(B, C, N)).double() for k in range(3)]
    w = [wgt[:, k][:, None, :].double() for k in range(3)]
    a = (g[0] * w[0]).float()
    a = (g[1] * w[1] + a.double()).float()
    return (g[2] * w[2] + a.double()).float()


def act_rows(raw, scale, shift, rna):
    """k_act_rows<1>: swish(fma(raw, scale, shift)), rounded to TF32 (rna) where the next layer reads it.
    raw fp32 [B,C,N], scale / shift fp32 [B,C] -> fp32 [B,C,N] (the swish in float64)."""
    a = (raw.double() * scale[:, :, None].double() + shift[:, :, None].double()).float().double()
    y = (a * torch.sigmoid(a)).float()
    return tf32_rna(y) if rna else y


def mlp_fold(sums, sqs, sd, p, style, count):
    """fold_affine of the AdaGN at state-dict prefix p (norm.*, emd.*) from per-channel sums."""
    fb = style.double() @ sd[p + "emd.weight"].double().T + sd[p + "emd.bias"].double()
    return fold_affine(sums, sqs, sd[p + "norm.weight"].double(), sd[p + "norm.bias"].double(), fb, count)


def sinusoid(t, E):
    """k_time_sinusoid in float64 of the kernel's fp32 argument e = fl(t * freq), freq = fl(exp(float64)) as build_unet
    computes it.  t fp32 [B] -> float64 [B, E] (sin | cos)."""
    half = E // 2
    fr = torch.from_numpy(np.exp(np.arange(half, dtype=np.float64) * -(np.log(10000.0) / (half - 1))).astype(np.float32))
    e = (t.float()[:, None].cpu() * fr[None, :]).double()
    return torch.cat([torch.sin(e), torch.cos(e)], 1)


def linear_f64(x, w, b, leaky=False):
    y = x.double() @ w.double().T + b.double()
    return torch.where(y > 0, y, 0.1 * y) if leaky else y


# ---------------------------------------------------------------------------------------------------------------------
# global prior (csrc/global_prior.cu): positional embedding, split-K Linears on the tensor cores, SE cells
#
# Operand model of k_gp_partial: the activation slice is rounded by the kernel, cvt.rna of fl32(x + add); the weights
# are staged by cp.async unrounded and handed to mma.sync as fp32 bits, so the tensor core reads them truncated.
# ---------------------------------------------------------------------------------------------------------------------
def gp_operand_models(tc=True):
    """(activation model, weight model) of a global-prior Linear; identities for comparisons with the fp32 oracle."""
    return (tf32_rna, tf32_trunc) if tc else (_ident, _ident)


def gp_freqs(half):
    """The frequency table global_prior_build computes on the host: expf(fl32(i) * fl32(-log(1e4) / (half - 1))), here
    as float64 exp of the fp32 argument rounded to fp32 (the correctly rounded expf).  At half = 64 this is the
    reference's torch.exp table bit for bit; torch's CPU exp (its AVX-512 path) differs from it in 3 of 128 entries at
    half = 128 and in 1 at half = 32, which depends on the host's instruction set and is not modelled."""
    step = np.float32(np.log(10000.0) / (half - 1))
    arg = np.arange(half, dtype=np.float32) * -step
    return torch.from_numpy(np.exp(arg.astype(np.float64)).astype(np.float32))


def gp_posemb(t, emb, scale):
    """k_gp_posemb in float64 of the kernel's fp32 argument fl32(fl32(t * scale) * freq).  t [B] -> float64 [B, emb]."""
    tf = t.float().cpu() * torch.tensor(scale, dtype=torch.float32)
    e = (tf[:, None] * gp_freqs(emb // 2)[None, :]).double()
    return torch.cat([torch.sin(e), torch.cos(e)], 1)


def gp_linear_f64(x, w, b, add=None, tc=True):
    """One k_gp_partial + k_gp_reduce Linear in float64 on modelled operands: W~ x~ + b with x~ = act(fl32(x + add)) and
    W~ = wmodel(w).  x, add [B, K] (rounded to fp32 first), w [O, K, ...], b [O] or None.  Returns (y, bound) float64
    [B, O], bound = |W~| |x~| + |b|: the scale of the sum's rounding error, which no cancellation can hide."""
    act, wm = gp_operand_models(tc)
    xs = x.float() if add is None else x.float() + add.float()
    xt = act(xs).double()
    wt = wm(w.reshape(w.shape[0], -1).float().contiguous()).double().to(xt.device)
    y, bound = xt @ wt.T, xt.abs() @ wt.abs().T
    if b is not None:
        y, bound = y + b.double().to(xt.device), bound + b.abs().double().to(xt.device)
    return y, bound


def gp_conv1_f64(h, temb, cmap, w, b, tc=True):
    """A cell's conv1 as the kernel reads it: act(fl32(h + temb)), and for CLIP cells [act(fl32(h + temb)) | act(cmap)]
    (the cmap half meets the zero half of [temb | 0])."""
    if cmap is None:
        return gp_linear_f64(h, w, b, add=temb, tc=tc)
    return gp_linear_f64(torch.cat([h.float(), cmap.float()], 1), w, b,
                         add=torch.cat([temb.float(), torch.zeros_like(cmap, dtype=torch.float32)], 1), tc=tc)


def gp_cell_out(s, w2, bb, h, tc=True):
    """k_gp_reduce of SE fc2: sigmoid(W~2 s~) * bb + h, the gate in float64.  Returns (y, bound = |gate bb| + |h|)."""
    z, _ = gp_linear_f64(s, w2, None, tc=tc)
    gb = torch.sigmoid(z) * bb.double()
    return gb + h.double(), gb.abs() + h.double().abs()


def gp_forward_f64(sd, x, t, clip=None, emb=128, scale=1.0, tc=True):
    """The global prior (Prior.forward with SE cells) in float64, the operand model applied to its own activations.
    Returns {stage: float64 [B, width]} with the probe's tap names (cells as lists) and 'out'."""
    relu = torch.relu
    S = {"pe": gp_posemb(t, emb, scale).to(x.device)}
    S["t0"] = gp_linear_f64(S["pe"], sd["temb_layer.0.weight"], sd["temb_layer.0.bias"], tc=tc)[0]
    S["temb"] = gp_linear_f64(S["t0"], sd["temb_layer.1.weight"], sd["temb_layer.1.bias"], tc=tc)[0]
    S["cmap"] = None
    if clip is not None:
        S["cmap"] = gp_linear_f64(clip, sd["clip_feat_mapping.weight"], sd["clip_feat_mapping.bias"], tc=tc)[0]
    h = S["h0"] = gp_linear_f64(x, sd["input_layer.weight"], sd["input_layer.bias"], tc=tc)[0]
    for n in ("a", "bb", "s", "h"):
        S[n] = []
    k = 0
    while "all_modules.%d.conv1.weight" % k in sd:
        p = "all_modules.%d." % k
        a = relu(gp_conv1_f64(h, S["temb"], S["cmap"], sd[p + "conv1.weight"], sd[p + "conv1.bias"], tc=tc)[0])
        bb = relu(gp_linear_f64(a, sd[p + "conv2.weight"], sd[p + "conv2.bias"], tc=tc)[0])
        s = relu(gp_linear_f64(bb, sd[p + "SE.fc.0.weight"], None, tc=tc)[0])
        h = gp_cell_out(s, sd[p + "SE.fc.2.weight"], bb.float(), h.float(), tc=tc)[0]
        for n, v in zip(("a", "bb", "s", "h"), (a, bb, s, h)):
            S[n].append(v)
        k += 1
    S["out"] = gp_linear_f64(h, sd["output_layer.weight"], sd["output_layer.bias"], tc=tc)[0]
    return S
