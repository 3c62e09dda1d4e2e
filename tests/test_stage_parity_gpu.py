"""Stage-level float64 parity of two tensor-core GEMM paths of the sampling step that the module tests see only through
a 2e-3 tolerance: the first convolution of a PVConv (dense tensor-core or sparse k_ygemm + gather) and the SA module's
MLP (fused sa_fused.cu passes or the unfused pooled epilogue).  lion_pvconv_conv1_probe / lion_sa_mlp_probe run the
product code and return what a module's output hides: raw outputs, fused GroupNorm sums, folded AdaGN affines and the
pooled extremes.  References are float64 on the device with the TF32 operand model of tests/stage_ref.py.

Maximum errors measured on one H100 80GB HBM3 (SXM, 700 W power limit) are listed next to each tolerance below."""
import ctypes as C

import pytest
import torch

from lion_b200 import _lib as L
from oracle import point_ops as OP
from tests import stage_ref as SR
from tests.synth import synth_state_dict
from tests.util import gen

pytestmark = pytest.mark.gpu

TOL_CONV = 3e-5        # raw first-convolution output, max-abs error / max-abs reference, per shape (measured 9.4e-6)
TOL_SUM_OWN = 1e-6     # fused GroupNorm sums against float64 sums of the same output, relative to sum |v|, sum v^2 (2.6e-7)
TOL_SUM_L1 = 4e-6      # SA layer-1 sums against the reference: operands modelled exactly (1.2e-6)
TOL_SUM_REF = 3e-5     # first-convolution sums against the reference (7.4e-6)
# SA layers after the first: their operands are rna(swish(...)) of the reference's own previous layer, whose TF32 ties
# fall differently from the kernel's wherever the two previous layers differ in the last bit (2.2e-5 for two layers,
# 9.2e-5 for the third layer of the 3-layer shape at B = 32)
TOL_SUM_NEXT = 2e-4
TOL_FOLD = 1e-6        # folded AdaGN scale / shift against a float64 fold of the probe's own sums (1.5e-7)
TOL_POOL = 1.3e-4      # pooled minimum / maximum: rms error over the rms of V, per shape (4.3e-5)


def _cfg():
    from lion_b200.config import default_prior_cfg
    return default_prior_cfg()


def _load(mod, seed):
    sd = synth_state_dict({k: list(v.shape) for k, v in mod.state_dict().items()}, seed)
    mod.load_state_dict(sd)
    return mod.cuda().eval(), {k: v.cuda() for k, v in sd.items()}


def _sum_err(got, v, dims):
    """max over (shape, channel) of |sum - ref| / sum |v| and |sqsum - ref| / sum v^2 (v float64)."""
    s, q = got
    e1 = ((s - v.sum(dims)).abs() / v.abs().sum(dims).clamp_min(1e-300)).max().item()
    e2 = ((q - (v * v).sum(dims)).abs() / (v * v).sum(dims).clamp_min(1e-300)).max().item()
    return max(e1, e2)


# ---------------------------------------------------------------------------------------------------------------------
# first convolution of a PVConv
# ---------------------------------------------------------------------------------------------------------------------
def _clouds(B, N, r, seed):
    """Gaussian, clustered and (at even r) 'sites' clouds with 127 / 128 / 129 / 256 occupied voxels -- k_ygemm's
    128-row block boundaries -- mixed in one batch, so that the occupancy differs from shape to shape."""
    if B >= 6:
        # (at most r^3 / 2 sites: the r = 8 grid holds the 127 - 129 sites clouds, not the 256 one)
        kinds = ["gauss", "cluster"] + [("sites", k) for k in (127, 128, 129, 256) if k <= N and k < r ** 3 // 2 and r % 2 == 0]
    else:
        kinds = ["gauss", "cluster"] + ([("sites", 129 if N < 2048 else 256)] if r % 2 == 0 and N >= 256 else [])
    kinds = (kinds + ["gauss"] * B)[:B]
    out = []
    for b, k in enumerate(kinds):
        if k == "gauss":
            out.append(SR.gaussian_cloud(seed + b, N, scale=0.2 + 0.05 * (b % 5)))
        elif k == "cluster":
            out.append(SR.clustered_cloud(N))
        else:
            out.append(SR.sites_cloud(k[1], N, r, seed + b))
    return torch.stack(out).contiguous()


def _conv1_probe(m, feats, coords, path, r, cout):
    B, _, N = feats.shape
    out = torch.empty(B, cout, r, r, r, device="cuda")
    s = torch.empty(B, cout, dtype=torch.float64, device="cuda")
    q = torch.empty_like(s)
    taken = C.c_int(0)
    L.check(L.lib().lion_pvconv_conv1_probe(m.h, L.ptr(feats), L.ptr(coords), path, L.ptr(out), L.ptr(s), L.ptr(q),
                                            C.byref(taken), B, N, L.stream()), "pvconv_conv1_probe")
    torch.cuda.synchronize()
    return out, s, q, taken.value


CONV1_CASES = [(32, 32, 32, 2048, 32), (64, 64, 32, 2048, 32),      # shapes of the step
               (128, 64, 16, 1024, 32),                              # sparse at the threshold N * 4 = r^3
               (128, 64, 16, 1025, 2),                               # dense just past it
               (16, 32, 32, 4096, 3),                                # smallest cin of the wide packing, largest N
               (64, 64, 32, 700, 3),                                 # ragged N
               (64, 64, 13, 500, 2),                                 # V = 2197: the gather's last warp is partial
               (36, 32, 32, 2048, 2),                                # sparse wanted, k_ygemm unusable (cin % 8) -> dense
               (4, 32, 32, 2048, 2), (128, 128, 8, 64, 2)]           # no wide packing -> dense


@pytest.mark.parametrize("cin,cout,r,N,B", CONV1_CASES)
def test_pvconv_conv1_stage(cin, cout, r, N, B):
    from lion_b200.models.pvcnn2_ada import PVConv
    mod, sd = _load(PVConv(cin, cout, 3, r, with_se=True, attention=False, cfg=_cfg()), 31)
    m = L.model_for(mod, L.KIND_PVCONV, mod.lion_desc(), mod.lion_params())
    feats = gen(40 + cin, B, cin, N).cuda()
    coords = _clouds(B, N, r, 100 * r + N).cuda()
    wide = cin >= 16 and cin % 8 == 0 and cout in (32, 64)            # k_ygemm's wide packing serves the layer
    auto_sparse = N * 4 <= r ** 3 and wide
    ref = SR.conv1_reference(feats, coords.cpu(), sd["voxel_layers.0.weight"], sd["voxel_layers.0.bias"], r)
    style = gen(41, B, 128).cuda()
    before = mod((feats, coords, None, style))[0].clone()

    paths = [0, 1] + ([2] if N * 4 <= r ** 3 and wide else [])
    for path in paths:
        out, s, q, taken = _conv1_probe(m, feats, coords, path, r, cout)
        assert taken == ({0: 2 if auto_sparse else 1, 1: 1, 2: 2}[path]), (path, taken)
        v = out.double().view(B, cout, -1)
        rv = ref.view(B, cout, -1)
        err = ((v - rv).abs().amax((1, 2)) / rv.abs().amax((1, 2))).max().item()
        e_own = _sum_err((s, q), v, 2)
        e_ref = _sum_err((s, q), rv, 2)
        print("conv1 %s path %d: raw %.2e, sums vs own %.2e, vs reference %.2e" % ((cin, cout, r, N, B), taken, err, e_own, e_ref))
        assert err <= TOL_CONV, "raw output (path %d): %.3e > %.1e" % (taken, err, TOL_CONV)
        assert e_own <= TOL_SUM_OWN, "sums against the probe's own output: %.3e > %.1e" % (e_own, TOL_SUM_OWN)
        assert e_ref <= TOL_SUM_REF, "sums against the reference: %.3e > %.1e" % (e_ref, TOL_SUM_REF)
        again = _conv1_probe(m, feats, coords, path, r, cout)[0]
        assert torch.equal(again, out), "path %d is not bit-reproducible" % taken
        if B > 1:                                                  # every shape alone: the same bits
            for b in range(B):
                alone = _conv1_probe(m, feats[b:b + 1].contiguous(), coords[b:b + 1].contiguous(), path, r, cout)[0]
                assert torch.equal(alone[0], out[b]), "path %d, shape %d: B = %d differs from B = 1" % (taken, b, B)
    # a product call after the probes (the dense one scatters into the context's zero grid) gives the same bits
    assert torch.equal(mod((feats, coords, None, style))[0], before)


def test_pvconv_conv1_forced_path_that_cannot_run_is_an_error():
    from lion_b200.models.pvcnn2_ada import PVConv
    for cin, cout, r, N in [(128, 64, 16, 1025), (36, 32, 32, 2048), (4, 32, 32, 2048), (128, 128, 8, 64)]:
        mod, _ = _load(PVConv(cin, cout, 3, r, with_se=True, attention=False, cfg=_cfg()), 31)
        m = L.model_for(mod, L.KIND_PVCONV, mod.lion_desc(), mod.lion_params())
        feats, coords = gen(1, 2, cin, N).cuda(), gen(2, 2, 3, N, scale=0.4).cuda()
        out = torch.full((2, cout, r, r, r), 7.0, device="cuda")
        s = torch.full((2, cout), 7.0, dtype=torch.float64, device="cuda")
        rc = L.lib().lion_pvconv_conv1_probe(m.h, L.ptr(feats), L.ptr(coords), 2, L.ptr(out), L.ptr(s), L.ptr(s), None, 2, N,
                                             L.stream())
        torch.cuda.synchronize()
        assert rc != 0 and b"sparse" in L.lib().lion_last_error()
        assert (out == 7.0).all() and (s == 7.0).all(), "a refused probe wrote its outputs"


# ---------------------------------------------------------------------------------------------------------------------
# SA MLP
# ---------------------------------------------------------------------------------------------------------------------
def _sa_probe(m, feats, coords, style, path, outs, M):
    B, _, N = feats.shape
    dev = "cuda"
    tot = sum(outs)
    centers = torch.empty(B, 3, M, device=dev)
    s = torch.empty(B * tot, dtype=torch.float64, device=dev)
    q = torch.empty_like(s)
    sc = torch.empty(B * tot, device=dev)
    sh = torch.empty_like(sc)
    mm = torch.empty(B, outs[-1] // 4, M, 2, 4, device=dev)
    taken = C.c_int(0)
    L.check(L.lib().lion_sa_mlp_probe(m.h, L.ptr(feats), L.ptr(coords), L.ptr(style), path, L.ptr(centers), L.ptr(s), L.ptr(q),
                                      L.ptr(sc), L.ptr(sh), L.ptr(mm), C.byref(taken), B, N, L.stream()), "sa_mlp_probe")
    torch.cuda.synchronize()
    per, off = [], 0
    for c in outs:
        n = B * c
        per.append(tuple(t[off:off + n].view(B, c) for t in (s, q, sc, sh)))
        off += n
    pool = mm.permute(0, 3, 1, 4, 2).reshape(B, 2, outs[-1], M)         # [B][min|max][C][M]
    return centers, per, pool, taken.value


LEVEL0 = (32, 1024, 0.1, (32, 64), 2048)
SA_SHAPES = [LEVEL0, (64, 256, 0.2, (64, 128), 1024), (128, 64, 0.4, (128, 128), 256), (192, 16, 0.8, (128, 128, 128), 64)]
SA_CASES = ([(*s, B) for s in SA_SHAPES for B in (2, 32)] + [(*LEVEL0, 1), (*LEVEL0, 5),
            (32, 1020, 0.1, (32, 64), 2048, 32),        # 255 tiles: a short last CTA range of the fused kernel
            (32, 1024, 0.02, (32, 64), 2048, 32)])      # most centres have fewer than 32 neighbours


@pytest.mark.parametrize("cfeat,M,radius,outs,N,B", SA_CASES)
def test_sa_mlp_stage(cfeat, M, radius, outs, N, B):
    from lion_b200.models.pvcnn2_ada import PointNetSAModule
    mod, sd = _load(PointNetSAModule(M, radius, 32, cfeat, list(outs), cfg=_cfg()), 32)
    m = L.model_for(mod, L.KIND_SA, mod.lion_desc(), mod.lion_params())
    feats = gen(50 + cfeat, B, cfeat, N).cuda()
    coords = gen(51 + B, B, 3, N, scale=0.3).cuda()
    style = gen(52, B, 128).cuda()
    fidx = OP.furthest_point_sample_idx(coords.cpu(), M)
    centers_ref = OP.gather(coords.cpu(), fidx).cuda()
    nidx = OP.ball_query(centers_ref.cpu(), coords.cpu(), radius, 32).cuda()
    rows = SR.sa_rows(feats, coords, centers_ref, nidx)                 # [B, M, 32, 4 + cfeat] fp32
    fused_ok = (cfeat, tuple(outs)) == (32, (32, 64))
    p = "mlps.0.layers.%d."
    for path in ([0, 1] if fused_ok else [0]):
        centers, per, pool, taken = _sa_probe(m, feats, coords, style, path, list(outs), M)
        assert taken == (2 if fused_ok and path == 0 else 1)
        assert torch.equal(centers, centers_ref), "probe centres differ from the oracle's FPS"
        a = SR.tf32_trunc(rows).double()                                  # gathered rows: read as TF32 by truncation
        errs = []
        for l, c in enumerate(outs):
            w = sd[p % (3 * l) + "weight"].reshape(c, -1)
            if l == 0:                                                    # [rel-xyz(3) | features] -> packed [xyz, 0 | f]
                w = torch.cat([w[:, :3], torch.zeros(c, 1, device="cuda"), w[:, 3:]], 1)
            v = a @ SR.tf32_rna(w.contiguous()).double().T + sd[p % (3 * l) + "bias"].double()
            s, q, sc, sh = per[l]
            errs.append(_sum_err((s, q), v, (1, 2)))
            g = p % (3 * l + 1)
            fb = style.double() @ sd[g + "emd.weight"].double().T + sd[g + "emd.bias"].double()
            rs, rt = SR.fold_affine(s, q, sd[g + "norm.weight"].double(), sd[g + "norm.bias"].double(), fb, float(M * 32))
            ef = max(((sc.double() - rs).abs().max() / rs.abs().max()).item(), ((sh.double() - rt).abs().max() / rt.abs().max()).item())
            errs.append(ef)
            tol = TOL_SUM_L1 if l == 0 else TOL_SUM_NEXT
            assert errs[-2] <= tol, "layer %d sums: %.3e > %.1e" % (l, errs[-2], tol)
            assert ef <= TOL_FOLD, "layer %d folded affine: %.3e > %.1e" % (l, ef, TOL_FOLD)
            if l + 1 < len(outs):
                a = SR.swish_act(v.float(), sc, sh).double()
        refp = torch.stack([v.amin(2), v.amax(2)], 1).permute(0, 1, 3, 2)  # [B, 2, C, M]
        d = pool.double() - refp
        # (a layer-1 output one ulp off the reference flips the TF32 rounding of a few layer-2 operands: single extremes
        # then move by up to ~5e-4 of max |V| while the kernel is right, so the extremes are bounded in rms)
        ep = (d.pow(2).mean((1, 2, 3)).sqrt() / v.pow(2).mean((1, 2, 3)).sqrt()).max().item()
        em = (d.abs().amax((1, 3)) / v.abs().amax((1, 2))).max().item()
        print("sa %s path %d: sums/fold per layer %s, pool rms %.2e (max %.2e)" % ((cfeat, M, radius, outs, N, B), taken,
                                                                              " ".join("%.2e" % e for e in errs), ep, em))
        assert ep <= TOL_POOL, "pooled extremes: %.3e > %.1e" % (ep, TOL_POOL)


def test_sa_mlp_forced_fused_that_cannot_run_is_an_error():
    from lion_b200.models.pvcnn2_ada import PointNetSAModule
    mod, _ = _load(PointNetSAModule(256, 0.2, 32, 64, [64, 128], cfg=_cfg()), 32)
    m = L.model_for(mod, L.KIND_SA, mod.lion_desc(), mod.lion_params())
    feats, coords, style = gen(1, 2, 64, 1024).cuda(), gen(2, 2, 3, 1024, scale=0.3).cuda(), gen(3, 2, 128).cuda()
    z = torch.zeros(2 * 256 * 256, device="cuda")
    zd = torch.zeros(2 * 192, dtype=torch.float64, device="cuda")
    rc = L.lib().lion_sa_mlp_probe(m.h, L.ptr(feats), L.ptr(coords), L.ptr(style), 2, L.ptr(z), L.ptr(zd), L.ptr(zd), L.ptr(z),
                                   L.ptr(z), L.ptr(z), None, 2, 1024, L.stream())
    torch.cuda.synchronize()
    assert rc != 0 and b"fused" in L.lib().lion_last_error()
    assert (z == 0).all() and (zd == 0).all()
