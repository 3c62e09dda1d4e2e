"""CPU side of the stage tests (tests/test_stage_parity_gpu.py): the clouds reach the occupancies they are built for
(the oracle's voxel indices), and the TF32 operand models are the bit-level operations they claim to be."""
import numpy as np
import pytest
import torch

from oracle import point_ops as OP
from tests import stage_ref as SR


@pytest.mark.parametrize("K,N,r", [(127, 2048, 32), (128, 2048, 32), (129, 2048, 32), (256, 2048, 32), (127, 1024, 16),
                                   (128, 1024, 16), (129, 1024, 16), (256, 1024, 16), (129, 700, 32), (256, 4096, 32),
                                   (127, 256, 8), (129, 256, 8)])
def test_sites_cloud_occupancy(K, N, r):
    c = SR.sites_cloud(K, N, r, seed=K + N + r)
    assert c.shape == (3, N)
    assert SR.occupancy(c[None], r) == [K]


@pytest.mark.parametrize("N,r", [(2048, 32), (4096, 32), (1024, 16), (500, 13), (64, 8)])
def test_clustered_cloud_occupancy(N, r):
    c = SR.clustered_cloud(N)
    ids = SR.voxel_ids(c[None], r)[0]
    vals, counts = torch.unique(ids, return_counts=True)
    assert len(vals) == 7 and int(counts.max()) == N - 6
    xyz = torch.stack([ids[-6:] // (r * r), ids[-6:] // r % r, ids[-6:] % r], 1)
    for k in range(6):                                        # each extreme point sits on a face of the grid
        assert int(xyz[k, k // 2]) == (r - 1 if k % 2 == 0 else 0)


def test_gaussian_cloud_is_spread():
    occ = SR.occupancy(SR.gaussian_cloud(3, 2048)[None], 32)[0]
    assert 1000 < occ <= 2048


def _tf32_bits_reference(x, mode):
    """Rounding of float32 values to 10 mantissa bits, computed from frexp in float64."""
    x = x.numpy().astype(np.float64)
    m, e = np.frexp(np.abs(x))                  # |x| = m * 2^e, m in [0.5, 1)
    q = m * 2.0 ** 11                           # 11 significant bits: 1 implicit + 10
    q = np.floor(q) if mode == "trunc" else np.floor(q + 0.5)
    return torch.from_numpy((np.sign(x) * np.ldexp(q / 2.0 ** 11, e)).astype(np.float32))


def test_tf32_operand_models_match_their_definitions():
    g = torch.Generator().manual_seed(5)
    x = torch.cat([torch.randn(100000, generator=g) * 10 ** torch.randint(-6, 6, (100000,), generator=g).float(),
                   torch.tensor([1.0, -1.0, 1.0 + 2 ** -11, -(1.0 + 2 ** -11), 1.0 + 3 * 2 ** -11, 1.5 - 2 ** -23, 0.0])])
    assert torch.equal(SR.tf32_trunc(x), _tf32_bits_reference(x, "trunc"))
    assert torch.equal(SR.tf32_rna(x), _tf32_bits_reference(x, "rna"))
    # ties go away from zero; truncation goes toward zero
    assert SR.tf32_rna(torch.tensor([1.0 + 2 ** -11, -(1.0 + 2 ** -11)])).tolist() == [1.0 + 2 ** -10, -(1.0 + 2 ** -10)]
    assert SR.tf32_trunc(torch.tensor([1.0 + 2 ** -10 - 2 ** -23])).tolist() == [1.0]


def test_scatter_grid_model_is_the_fused_multiply_add_chain():
    """scatter_grid = f0 * (1/n), then fma(f_k, 1/n, acc) over the voxel's points in ascending order."""
    g = torch.Generator().manual_seed(6)
    feats = torch.randn(1, 3, 50, generator=g)
    ids = torch.randint(0, 4, (1, 50), generator=g)
    grid = SR.scatter_grid(feats, ids, 2).view(3, 8)
    for v in range(8):
        pts = (ids[0] == v).nonzero().flatten().tolist()
        for c in range(3):
            if not pts:
                assert grid[c, v] == 0
                continue
            inv = np.float32(1.0) / np.float32(len(pts))
            acc = np.float32(feats[0, c, pts[0]].item()) * inv
            for k in pts[1:]:
                acc = np.float32(np.float64(feats[0, c, k].item()) * np.float64(inv) + np.float64(acc))
            assert grid[c, v].item() == acc


# ---------------------------------------------------------------------------------------------------------------------
# second half of a PVConv and the linear attention (tests/test_pvconv_tail_stage_gpu.py, test_attention_stage_gpu.py):
# the float64 references, chained with the TF32 models switched off, restate the fp32 oracle
# ---------------------------------------------------------------------------------------------------------------------
def _cfg():
    from lion_b200.config import default_prior_cfg
    return default_prior_cfg()


def _sd(mod, seed):
    from tests.synth import synth_state_dict
    return synth_state_dict({k: list(v.shape) for k, v in mod.state_dict().items()}, seed)


def _gn(sd, p, style):
    fb = style.double() @ sd[p + "emd.weight"].double().T + sd[p + "emd.bias"].double()
    return sd[p + "norm.weight"].double(), sd[p + "norm.bias"].double(), fb


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


@pytest.mark.parametrize("cin,cout,r,N,attn", [(4, 32, 6, 150, False), (16, 32, 5, 90, True), (20, 40, 5, 100, False)])
def test_pvconv_stage_references_restate_the_oracle(cin, cout, r, N, attn):
    from lion_b200.models.pvcnn2_ada import PVConv
    from oracle import net as ON
    from oracle import point_ops as OP
    sd = _sd(PVConv(cin, cout, 3, r, with_se=True, attention=attn, cfg=_cfg()), 7)
    B = 2
    feats, style = torch.randn(B, cin, N, generator=torch.Generator().manual_seed(1)), torch.randn(B, 128)
    coords = torch.randn(B, 3, N, generator=torch.Generator().manual_seed(2)) * 0.4
    V = float(r ** 3)
    raw1 = SR.conv1_reference(feats, coords, sd["voxel_layers.0.weight"], sd["voxel_layers.0.bias"], r, tc=False)
    s1, t1 = SR.fold_affine(raw1.sum((2, 3, 4)), (raw1 * raw1).sum((2, 3, 4)), *_gn(sd, "voxel_layers.1.", style), V)
    act = SR.act_grid(raw1.float(), s1.float(), t1.float(), rna=False)[:, :, 1:-1, 1:-1, 1:-1]
    raw2 = SR.conv3x3x3_f64(act.double(), sd["voxel_layers.4.weight"].double(), sd["voxel_layers.4.bias"].double())
    s2, t2 = SR.fold_se(raw2.sum((2, 3, 4)), (raw2 * raw2).sum((2, 3, 4)), *_gn(sd, "voxel_layers.5.", style), V,
                        sd["voxel_layers.6.fc.0.weight"], sd["voxel_layers.6.fc.2.weight"])
    rawp = SR.point_conv(feats, sd["point_features.layers.0.weight"], sd["point_features.layers.0.bias"], tc=False)
    sp, tp = SR.fold_affine(rawp.sum(2), (rawp * rawp).sum(2), *_gn(sd, "point_features.layers.1.", style), float(N))
    nc, _ = OP.voxel_coords_cuda_order(coords, r)
    out = SR.devox_fuse(raw2, s2, t2, nc, rawp, sp, tp)
    if attn:
        qkv = SR.attn_qkv(out.float(), sd["attn.to_qkv.weight"], tc=False)
        out = SR.attn_out(SR.attn_core(qkv, 4).float(), sd["attn.to_out.weight"], sd["attn.to_out.bias"], tc=False)
    ref = ON.pvconv(sd, "", dict(kind="pvconv", cin=cin, cout=cout, r=r, attn=attn), feats, coords, style)
    assert _rel(out, ref) < 2e-5


@pytest.mark.parametrize("C,heads,N", [(64, 4, 129), (128, 8, 300)])
def test_attention_references_restate_the_oracle(C, heads, N):
    from lion_b200.models.pvcnn2_ada import LinearAttention
    from oracle import net as ON
    sd = _sd(LinearAttention(C, heads), 8)
    x = torch.randn(2, C, N, generator=torch.Generator().manual_seed(3))
    qkv = SR.attn_qkv(x, sd["to_qkv.weight"], tc=False)
    out = SR.attn_out(SR.attn_core(qkv, heads).float(), sd["to_out.weight"], sd["to_out.bias"], tc=False)
    assert _rel(out, ON.linear_attention(sd, "", x, heads)) < 1e-5


def test_trilinear_reference_restates_the_oracle():
    """Including points on the grid's faces and at integer coordinates, where the high corners weigh 0."""
    from oracle import point_ops as OP
    r, N = 6, 400
    g = torch.Generator().manual_seed(4)
    grid = torch.randn(2, 5, r, r, r, generator=g)
    nc = torch.rand(2, 3, N, generator=g) * (r - 1)
    nc[:, :, :50] = torch.randint(0, r, (2, 3, 50), generator=g).float()
    nc[:, 0, 50:60] = r - 1
    got = SR.trilinear_f64(grid.double(), nc, r)
    assert _rel(got, OP.trilinear_devoxelize(grid, nc, r)) < 1e-6
    assert torch.equal(got[:, :, :50], grid.double().reshape(2, 5, -1).gather(
        2, ((nc[:, 0, :50] * r + nc[:, 1, :50]) * r + nc[:, 2, :50]).long()[:, None].expand(2, 5, 50)))


def test_act_grid_model_matches_its_definition():
    """act_grid = rna(float32(swish(float32(x * scale + shift)))) inside, 0 on every halo position."""
    g = torch.Generator().manual_seed(9)
    B, C, r = 2, 3, 3
    raw = torch.randn(B, C, r, r, r, generator=g) * 4
    s, t = torch.randn(B, C, generator=g), torch.randn(B, C, generator=g)
    got = SR.act_grid(raw, s, t)
    assert got.shape == (B, C, r + 2, r + 2, r + 2) and got.dtype == torch.float32
    inner = got[:, :, 1:-1, 1:-1, 1:-1]
    halo = got.clone()
    halo[:, :, 1:-1, 1:-1, 1:-1] = 0
    assert (halo == 0).all()
    for b in range(B):
        for c in range(C):
            for i, v in enumerate(raw[b, c].flatten().tolist()):
                a = np.float32(np.float64(v) * np.float64(s[b, c].item()) + np.float64(t[b, c].item()))
                y = np.float32(np.float64(a) / (1.0 + np.exp(-np.float64(a))))
                want = _tf32_bits_reference(torch.tensor([y]), "rna")[0].item()
                assert inner[b, c].flatten()[i].item() == want


# ---------------------------------------------------------------------------------------------------------------------
# FP module and the U-Net's glue (tests/test_fp_stage_gpu.py, test_unet_glue_stage_gpu.py)
# ---------------------------------------------------------------------------------------------------------------------
def _three_nn_scalar(pt, ce):
    """neighbor_interpolate.cu:36-73 transcribed literally for one shape: double best distances starting at 1e40, the
    strict '<' cascade, the clamp to [1e-10, 1e10] in double, products rounded to float, fp32 sum and reciprocal."""
    f32 = np.float32
    N, M = pt.shape[1], ce.shape[1]
    idx, wgt = np.zeros((3, N), np.int32), np.zeros((3, N), np.float32)
    for j in range(N):
        best, bi = [1e40, 1e40, 1e40], [0, 0, 0]
        for k in range(M):
            dx, dy, dz = (f32(pt[a, j]) - f32(ce[a, k]) for a in range(3))
            d = float(OP._sqdist(dx, dy, dz))
            if d < best[2]:
                best[2], bi[2] = d, k
                if d < best[1]:
                    best[2], bi[2], best[1], bi[1] = best[1], bi[1], d, k
                    if d < best[0]:
                        best[1], bi[1], best[0], bi[0] = best[0], bi[0], d, k
        b = [max(min(float(f32(1e10)), v), float(f32(1e-10))) for v in best]
        d0d1, d0d2, d1d2 = f32(b[0] * b[1]), f32(b[0] * b[2]), f32(b[1] * b[2])
        inv = f32(f32(1.0) / f32(f32(d0d1 + d0d2) + d1d2))
        wgt[:, j] = [f32(d1d2 * inv), f32(d0d2 * inv), f32(d0d1 * inv)]
        idx[:, j] = bi
    return idx, wgt


@pytest.mark.parametrize("M,kind", [(1, "gauss"), (2, "gauss"), (3, "gauss"), (40, "gauss"), (30, "ties"), (20, "dup")])
def test_three_nn_oracle_matches_the_reference_cascade(M, kind):
    """The oracle's 3-NN against a scalar transcription of the reference kernel, including fewer than three centres
    (the missing slots keep index 0 and distance 1e40) and exact distance ties (the lower index stays first)."""
    g = torch.Generator().manual_seed(M)
    if kind == "ties":
        pts = torch.randint(-4, 4, (2, 3, 60), generator=g).float() / 4
        ce = torch.randint(-2, 2, (2, 3, M), generator=g).float() / 2
    else:
        pts, ce = torch.randn(2, 3, 60, generator=g) * 0.3, torch.randn(2, 3, M, generator=g) * 0.3
        if kind == "dup":
            ce = torch.cat([ce[:, :, :M // 2]] * 2, 2)
    idx, wgt = OP.three_nn(pts, ce)
    for b in range(2):
        ri, rw = _three_nn_scalar(pts[b].numpy(), ce[b].numpy())
        assert np.array_equal(idx[b].numpy(), ri) and np.array_equal(wgt[b].numpy(), rw)
    if M < 3:                                             # a missing slot (distance clamped to 1e10) weighs next to nothing
        assert (idx[:, M:] == 0).all() and (wgt[:, M:] < 1e-9).all()


def test_fp_references_restate_the_oracle():
    from lion_b200.models.pvcnn2_ada import PointNetFPModule
    from oracle import net as ON
    from oracle import point_ops as OP
    cc, cp, outs, N, M, B = 24, 5, [32, 16], 90, 20, 2
    sd = _sd(PointNetFPModule(cc + cp, outs, cfg=_cfg()), 10)
    g = torch.Generator().manual_seed(11)
    pc, ce = torch.randn(B, 3, N, generator=g) * 0.3, torch.randn(B, 3, M, generator=g) * 0.3
    cf, pf, style = torch.randn(B, cc, M, generator=g), torch.randn(B, cp, N, generator=g), torch.randn(B, 128, generator=g)
    idx, wgt = OP.three_nn(pc, ce)
    x = torch.cat([SR.interp_fma(cf, idx, wgt), pf], 1)
    for l, c in enumerate(outs):
        raw = SR.point_conv(x, sd["mlp.layers.%d.weight" % (3 * l)], sd["mlp.layers.%d.bias" % (3 * l)], tc=False)
        s, t = SR.mlp_fold(raw.sum(2), (raw * raw).sum(2), sd, "mlp.layers.%d." % (3 * l + 1), style, float(N))
        x = SR.act_rows(raw.float(), s.float(), t.float(), rna=False)
    ref, _ = ON.fp_module(sd, "", dict(kind="fp", cin=cc + cp, mlp=outs), pc, ce, cf, pf, None, style)
    assert _rel(x, ref) < 2e-5
    # the interpolation is the oracle's up to the fused multiply-adds
    assert _rel(SR.interp_fma(cf, idx, wgt), OP.nearest_neighbor_interpolate(pc, ce, cf)) < 1e-6


def test_time_embedding_reference_restates_the_oracle():
    import torch.nn.functional as TF
    from oracle import net as ON
    E = 64
    t = torch.tensor([0.0, 1.0, 500.0, 999.0, 1000.0])
    sinu = SR.sinusoid(t, E)
    assert (sinu - ON.timestep_embedding(t, E).double()).abs().max() < 2e-6
    g = torch.Generator().manual_seed(12)
    w0, b0, w2, b2 = (torch.randn(E, E, generator=g) * 0.2, torch.randn(E, generator=g) * 0.1,
                      torch.randn(E, E, generator=g) * 0.2, torch.randn(E, generator=g) * 0.1)
    got = SR.linear_f64(SR.linear_f64(sinu, w0, b0, leaky=True), w2, b2)
    ref = TF.linear(TF.leaky_relu(TF.linear(ON.timestep_embedding(t, E), w0, b0), 0.1), w2, b2)
    assert _rel(got, ref) < 1e-5


def test_classifier_reference_restates_the_oracle():
    from oracle import net as ON
    from tests.synth import synth_state_dict
    C, N, B, nc = 64, 80, 2, 3
    shapes = {"classifier.0.layers.0.weight": [128, C, 1], "classifier.0.layers.0.bias": [128],
              "classifier.0.layers.1.norm.weight": [128], "classifier.0.layers.1.norm.bias": [128],
              "classifier.0.layers.1.emd.weight": [256, 128], "classifier.0.layers.1.emd.bias": [256],
              "classifier.2.weight": [nc, 128, 1], "classifier.2.bias": [nc]}
    sd = synth_state_dict(shapes, 13)
    g = torch.Generator().manual_seed(14)
    feat, style = torch.randn(B, C, N, generator=g), torch.randn(B, 128, generator=g)
    raw = SR.point_conv(feat, sd["classifier.0.layers.0.weight"], sd["classifier.0.layers.0.bias"], tc=False)
    s, t = SR.mlp_fold(raw.sum(2), (raw * raw).sum(2), sd, "classifier.0.layers.1.", style, float(N))
    hc = SR.act_rows(raw.float(), s.float(), t.float(), rna=False)
    out = torch.einsum("oc,bcn->bon", sd["classifier.2.weight"].reshape(nc, 128).double(), hc.double()) + sd["classifier.2.bias"].double()[None, :, None]
    h = ON.shared_mlp(sd, "classifier.0.", feat, style, 1)
    ref = torch.einsum("oc,bcn->bon", sd["classifier.2.weight"].reshape(nc, 128), h) + sd["classifier.2.bias"][None, :, None]
    assert _rel(out, ref) < 2e-5


# ---------------------------------------------------------------------------------------------------------------------
# global prior (tests/test_global_prior_stage_gpu.py)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["default", "clip", "ragged", "ragged_clip"])
def test_global_prior_reference_restates_the_oracle(which):
    """The float64 chain with identity operand models (fp32 activations between layers) is the fp32 oracle's
    Prior.forward, up to fp32 rounding: max-abs error / max-abs reference measured 3.9e-7 on the CPU (the CLIP model)."""
    from oracle import net as ON
    from tests import test_global_prior_stage_gpu as GS
    spec = {"default": GS.DEFAULT, "clip": GS.CLIP, "ragged": GS.RAGGED, "ragged_clip": GS.RAGGED_CLIP}[which]
    _, sd = GS.gp_net(*spec)
    x, t, clip = GS.gp_inputs(spec, 5, 21)
    got = SR.gp_forward_f64(sd, x, t, clip, spec[2], spec[5], tc=False)["out"]
    with torch.no_grad():
        ref = ON.global_prior_forward(sd, x, t, clip_feat=clip, embedding_dim=spec[2], embedding_scale=spec[5])
    assert _rel(got, ref) < 1.2e-6


@pytest.mark.parametrize("half", [20, 32, 64, 128])
def test_global_prior_frequencies_are_the_host_expf_table(half):
    """SR.gp_freqs is the table global_prior_build uploads: expf((float)i * -(float)(log(1e4) / (half - 1)))."""
    import ctypes
    import ctypes.util
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    libm.expf.restype, libm.expf.argtypes = ctypes.c_float, [ctypes.c_float]
    step = np.float32(np.log(10000.0) / (half - 1))
    host = [libm.expf(float(np.float32(np.float32(i) * -step))) for i in range(half)]
    assert torch.equal(SR.gp_freqs(half), torch.tensor(host, dtype=torch.float32))
