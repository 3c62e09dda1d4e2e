"""Stage-level float64 parity of the second half of a PVConv, which the module tests see only through a 2e-3 tolerance:
the AdaGN-1 + Swish grid (k_act_grid), the second 3x3x3 convolution (SIMT, tensor-core row tiles or 2- / 4-block
interior groups) with its GroupNorm sums, the AdaGN-2 fold with the SE gate (k_affine_prep), the point branch and the
devoxelisation that adds them (k_devox_fuse).  lion_pvconv_probe runs the product code, NaN-fills the grids of raw1,
act1 and raw2 before their producers run (so that a read of an unwritten halo row shows up), and returns each stage's
input and output; every reference below is built from the probe's own previous stage, so each tolerance covers one
kernel.  References are float64 on the device with the TF32 operand model of tests/stage_ref.py.

Maximum errors measured on one H100 80GB HBM3 (SXM, 700 W power limit) are listed next to each tolerance below."""
import ctypes as C

import pytest
import torch

from lion_b200 import _lib as L
from oracle import point_ops as OP
from tests import stage_ref as SR
from tests.test_stage_parity_gpu import _cfg, _clouds, _load, _sum_err
from tests.util import gen

pytestmark = pytest.mark.gpu

TOL_FOLD1 = 1.3e-6     # AdaGN-1 scale / shift against a float64 fold of float64 sums of the probe's raw1 (measured 4.4e-7)
TOL_CONV2 = 3.3e-5     # raw second-convolution output, max-abs error / max-abs reference, per shape (1.2e-5)
TOL_SUM_OWN = 5e-7     # GroupNorm sums against float64 sums of the probe's own output, relative to sum |v|, sum v^2 (1.5e-7)
# second-convolution sums against the reference (3.2e-5 at 128 channels): the fp32 accumulation of the tensor cores
# leaves a small bias of one sign in every output, and the sum over r^3 voxels adds it up
TOL_SUM_REF = 1e-4
TOL_FOLD = 6e-7        # folded affines against a float64 fold of the probe's own sums, SE gate included (2.0e-7)
TOL_POINT = 2.5e-6     # point branch raw output and its sums against the reference (1.0e-6)
TOL_FUSED = 7e-7       # devoxelised + point branch, max-abs error / max-abs reference, per shape (2.3e-7)
# A shape run alone against the same shape in a batch (see the end of test_pvconv_tail_stage): GroupNorm sums relative
# to the largest |sum| of the shape (9.2e-8), folded affines (2.0e-7), the grids and outputs after them (9.1e-5: an act1
# value whose TF32 rounding flipped moves by 2^-11 of itself), and the output of the attention shape (1.5e-4: a changed
# truncation of one of its TF32 inputs moves that input by 2^-10 of itself)
TOL_ALONE_SUM = 3e-7
TOL_ALONE_AFF = 6e-7
TOL_ALONE = 3e-4
TOL_ALONE_ATTN = 5e-4

# (cin, cout, r, N, B, attn)
STEP_SHAPES = [(4, 32, 32, 2048), (32, 32, 32, 2048), (64, 64, 32, 2048), (128, 64, 16, 1024), (128, 128, 16, 1024),
               (192, 128, 8, 256), (128, 128, 8, 256), (128, 128, 8, 64)]
PV_CASES = ([(ci, co, r, N, 32, (ci, co, r) == (128, 64, 16)) for ci, co, r, N in STEP_SHAPES] +
            [(128, 128, 16, 1024, 2, False),        # 2-block interior groups (4-block at B = 32)
             (64, 128, 13, 500, 3, False),          # ragged r: interior blocks masked past r
             (64, 64, 32, 700, 3, False),           # ragged N
             (20, 40, 5, 100, 2, False)])           # C not a multiple of 32: SIMT convolutions, k_affine_prep's non-warp SE


def _conv2_kernel(cout, r, B):
    """The kernel conv_tc_run picks: row tiles below 128 output channels, 4-block groups while there are as many of them
    as SMs (r = 16 at B = 32), 2-block groups otherwise; SIMT for widths that are not a multiple of 32."""
    if cout % 32:
        return 0
    if cout < 128:
        return 1
    return 4 if (r, B) == (16, 32) else 2


def _probe(m, feats, coords, style, cout, r):
    B, _, N = feats.shape
    rp, d = r + 2, "cuda"
    o = dict(raw1=torch.empty(B, cout, r, r, r, device=d), act1=torch.empty(B, cout, rp, rp, rp, device=d),
             raw2=torch.empty(B, cout, r, r, r, device=d), rawp=torch.empty(B, cout, N, device=d),
             sums=torch.empty(4, B, cout, dtype=torch.float64, device=d), affine=torch.empty(6, B, cout, device=d),
             fused=torch.empty(B, cout, N, device=d), out=torch.empty(B, cout, N, device=d))
    kern = C.c_int(-1)
    L.check(L.lib().lion_pvconv_probe(m.h, L.ptr(feats), L.ptr(coords), L.ptr(style), L.ptr(o["raw1"]), L.ptr(o["act1"]),
                                      L.ptr(o["raw2"]), L.ptr(o["rawp"]), L.ptr(o["sums"]), L.ptr(o["affine"]), L.ptr(o["fused"]),
                                      L.ptr(o["out"]), C.byref(kern), B, N, L.stream()), "pvconv_probe")
    torch.cuda.synchronize()
    o["kernel"] = kern.value
    return o


def _rel(got, ref, dims):
    """max over shapes of max |got - ref| / max |ref| (float64)."""
    return ((got.double() - ref).abs().amax(dims) / ref.abs().amax(dims).clamp_min(1e-300)).max().item()


def _fold_err(sc, sh, rs, rt):
    return max(((sc.double() - rs).abs().max() / rs.abs().max()).item(), ((sh.double() - rt).abs().max() / rt.abs().max()).item())


def _tf32_ulps(got, ref):
    """|got - ref| in units of the TF32 ulp of ref (10 explicit mantissa bits)."""
    _, e = torch.frexp(ref.abs())
    ulp = torch.ldexp(torch.ones_like(ref, dtype=torch.float64), (e - 11).to(torch.int32))
    return ((got.double() - ref.double()).abs() / ulp).max().item()


def _gn(sd, i, style):
    p = "voxel_layers.%d." % i
    fb = style.double() @ sd[p + "emd.weight"].double().T + sd[p + "emd.bias"].double()
    return sd[p + "norm.weight"].double(), sd[p + "norm.bias"].double(), fb


@pytest.mark.parametrize("cin,cout,r,N,B,attn", PV_CASES)
def test_pvconv_tail_stage(cin, cout, r, N, B, attn):
    from lion_b200.models.pvcnn2_ada import LinearAttention, PVConv
    mod, sd = _load(PVConv(cin, cout, 3, r, with_se=True, attention=attn, cfg=_cfg()), 33)
    m = L.model_for(mod, L.KIND_PVCONV, mod.lion_desc(), mod.lion_params())
    feats = gen(60 + cin, B, cin, N).cuda()
    coords = _clouds(B, N, r, 7 * r + N).cuda()
    style = gen(61, B, 128).cuda()
    tc = cout % 32 == 0                                            # tensor-core convolutions (else SIMT)
    V = float(r ** 3)
    P = _probe(m, feats, coords, style, cout, r)
    assert P["kernel"] == _conv2_kernel(cout, r, B), "second convolution ran kernel %d" % P["kernel"]
    s1, t1, sp, tp, s2, t2 = P["affine"].unbind(0)
    sum2, sq2, sump, sqp = P["sums"].unbind(0)

    # AdaGN-1 fold from float64 sums of the probe's raw1 (the conv1 stage test checks raw1 and its fused sums)
    v1 = P["raw1"].double().view(B, cout, -1)
    rs1, rt1 = SR.fold_affine(v1.sum(2), (v1 * v1).sum(2), *_gn(sd, 1, style), V)
    e_fold1 = _fold_err(s1, t1, rs1, rt1)

    # k_act_grid: within 1 TF32 ulp inside, exactly 0 on every halo position (x = 0 and x = r + 1 planes included)
    act = P["act1"]
    ref_act = SR.act_grid(P["raw1"], s1, t1)
    inner = (slice(None), slice(None), slice(1, -1), slice(1, -1), slice(1, -1))
    e_act = _tf32_ulps(act[inner], ref_act[inner])
    halo = torch.ones_like(act, dtype=torch.bool)
    halo[inner] = False
    assert torch.isfinite(act).all(), "act1 grid has NaNs: a position k_act_grid did not write"
    assert (act[halo] == 0).all(), "act1 halo is not zero"
    assert torch.equal(act[inner], SR.tf32_rna(act[inner])), "act1 is not rounded to TF32"

    # second convolution on the probe's act1, and its GroupNorm sums
    rna, _ = SR.operand_models(tc)
    ref2 = SR.conv3x3x3_f64(act[inner].double(), rna(sd["voxel_layers.4.weight"]).double(), sd["voxel_layers.4.bias"].double())
    v2, rv2 = P["raw2"].double().view(B, cout, -1), ref2.view(B, cout, -1)
    e_conv2 = _rel(v2, rv2, (1, 2))
    e2_own, e2_ref = _sum_err((sum2, sq2), v2, 2), _sum_err((sum2, sq2), rv2, 2)

    # AdaGN-2 + SE fold of the probe's own sums
    rs2, rt2 = SR.fold_se(sum2, sq2, *_gn(sd, 5, style), V, sd["voxel_layers.6.fc.0.weight"], sd["voxel_layers.6.fc.2.weight"])
    e_fold2 = _fold_err(s2, t2, rs2, rt2)

    # point branch: 1x1 convolution of the features, its sums and fold
    refp = SR.point_conv(feats, sd["point_features.layers.0.weight"], sd["point_features.layers.0.bias"], tc)
    vp = P["rawp"].double()
    e_point = max(_rel(vp, refp, (1, 2)), _sum_err((sump, sqp), refp, 2))
    ep_own = _sum_err((sump, sqp), vp, 2)
    g = "point_features.layers.1."
    fbp = style.double() @ sd[g + "emd.weight"].double().T + sd[g + "emd.bias"].double()
    rsp, rtp = SR.fold_affine(sump, sqp, sd[g + "norm.weight"].double(), sd[g + "norm.bias"].double(), fbp, float(N))
    e_foldp = _fold_err(sp, tp, rsp, rtp)

    # devoxelisation + point branch at the oracle's normalised coordinates (bit-exact to the kernels')
    nc, _ = OP.voxel_coords_cuda_order(coords.cpu(), r)
    ref_f = SR.devox_fuse(P["raw2"], s2, t2, nc, P["rawp"], sp, tp)
    e_fused = _rel(P["fused"], ref_f, (1, 2))

    print("pvconv tail %s kernel %d: fold1 %.2e, act1 %.2f ulp, conv2 %.2e, sums vs own %.2e / ref %.2e, fold2+SE %.2e, "
          "point %.2e (own sums %.2e), point fold %.2e, fused %.2e" % ((cin, cout, r, N, B, attn), P["kernel"], e_fold1, e_act,
                                                                      e_conv2, e2_own, e2_ref, e_fold2, e_point, ep_own, e_foldp,
                                                                      e_fused))
    assert e_fold1 <= TOL_FOLD1, "AdaGN-1 fold: %.3e > %.1e" % (e_fold1, TOL_FOLD1)
    assert e_act <= 1.0, "act1: %.2f TF32 ulps" % e_act
    assert e_conv2 <= TOL_CONV2, "conv2 raw output: %.3e > %.1e" % (e_conv2, TOL_CONV2)
    assert e2_own <= TOL_SUM_OWN, "conv2 sums against its own output: %.3e > %.1e" % (e2_own, TOL_SUM_OWN)
    assert e2_ref <= TOL_SUM_REF, "conv2 sums against the reference: %.3e > %.1e" % (e2_ref, TOL_SUM_REF)
    assert e_fold2 <= TOL_FOLD, "AdaGN-2 + SE fold: %.3e > %.1e" % (e_fold2, TOL_FOLD)
    assert e_point <= TOL_POINT, "point branch: %.3e > %.1e" % (e_point, TOL_POINT)
    assert ep_own <= TOL_SUM_OWN, "point sums against its own output: %.3e > %.1e" % (ep_own, TOL_SUM_OWN)
    assert e_foldp <= TOL_FOLD, "point-branch fold: %.3e > %.1e" % (e_foldp, TOL_FOLD)
    assert e_fused <= TOL_FUSED, "devoxelised + point branch: %.3e > %.1e" % (e_fused, TOL_FUSED)

    # the module output: lion_pvconv_fwd gives the same bits; with attention, so does a stand-alone attention of the
    # same weights applied to the probe's fused input
    assert torch.equal(mod((feats, coords, None, style))[0], P["out"]), "probe output differs from lion_pvconv_fwd"
    if attn:
        att = LinearAttention(cout).cuda().eval()
        att.load_state_dict({k[len("attn."):]: v for k, v in sd.items() if k.startswith("attn.")})
        assert torch.equal(att(P["fused"]), P["out"]), "attention of the probe's fused input differs from its output"
    else:
        assert torch.equal(P["fused"], P["out"])

    # the same bits run after run, and for every shape alone
    again = _probe(m, feats, coords, style, cout, r)
    for k in ("raw1", "act1", "raw2", "rawp", "sums", "affine", "fused", "out"):
        assert torch.equal(again[k], P[k]), "%s is not bit-reproducible" % k
    # Every shape alone.  The raw outputs of the first convolution and of the point branch do not depend on the batch:
    # the same bits.  The GroupNorm sums of the tensor-core row tiles (32 and 64 channels, and k_conv_stats for 128) are
    # fp32 sums over the tiles of one work item, flushed with one fp64 atomic per channel, and the items are equal
    # ranges of the batch's flat tile space: which tiles share an fp32 partial depends on B, so the sums may differ in
    # their last fp32 bits (the interior-block and SIMT shapes here happen to match bit for bit).  A fold of such sums
    # can round to a neighbouring float; a TF32 rounding of act1 or a truncation of the attention's input then flips here
    # and there, and the grids and outputs after it move by that much.
    if B > 1:
        e_sum = e_aff = e_grid = e_out = 0.0
        for b in range(B):
            one = _probe(m, feats[b:b + 1].contiguous(), coords[b:b + 1].contiguous(), style[b:b + 1].contiguous(), cout, r)
            for k in ("raw1", "rawp"):
                assert torch.equal(one[k][0], P[k][b]), "%s of shape %d: B = %d differs from B = 1" % (k, b, B)
            e_sum = max(e_sum, ((one["sums"][:, 0] - P["sums"][:, b]).abs().amax(1) / P["sums"][:, b].abs().amax(1)).max().item())
            e_aff = max(e_aff, _rel(one["affine"][:, 0], P["affine"][:, b].double(), 1))
            e_grid = max(e_grid, *[_rel(one[k], P[k][b:b + 1].double(), tuple(range(1, P[k].dim()))) for k in ("act1", "raw2", "fused")])
            e_out = max(e_out, _rel(one["out"], P["out"][b:b + 1].double(), (1, 2)))
        print("  alone vs batch: sums %.2e, affine %.2e, act1 / raw2 / fused %.2e, out %.2e" % (e_sum, e_aff, e_grid, e_out))
        assert e_sum <= TOL_ALONE_SUM, "GroupNorm sums, alone vs batch: %.3e > %.1e" % (e_sum, TOL_ALONE_SUM)
        assert e_aff <= TOL_ALONE_AFF, "folded affines, alone vs batch: %.3e > %.1e" % (e_aff, TOL_ALONE_AFF)
        assert e_grid <= TOL_ALONE, "act1 / raw2 / fused, alone vs batch: %.3e > %.1e" % (e_grid, TOL_ALONE)
        tol_out = TOL_ALONE_ATTN if attn else TOL_ALONE
        assert e_out <= tol_out, "output, alone vs batch: %.3e > %.1e" % (e_out, tol_out)


def test_pvconv_scatter_grid_is_restored():
    """The dense first convolution scatters into a persistent all-zero grid that k_act_grid's extra blocks zero again:
    cloud A, then cloud B, then cloud A again gives A's bits."""
    from lion_b200.models.pvcnn2_ada import PVConv
    cin, cout, r, N, B = 4, 32, 32, 2048, 2
    mod, _ = _load(PVConv(cin, cout, 3, r, with_se=True, attention=False, cfg=_cfg()), 34)
    m = L.model_for(mod, L.KIND_PVCONV, mod.lion_desc(), mod.lion_params())
    style = gen(62, B, 128).cuda()
    fa, ca = gen(63, B, cin, N).cuda(), gen(64, B, 3, N, scale=0.3).cuda()
    fb, cb = gen(65, B, cin, N).cuda(), gen(66, B, 3, N, scale=0.5).cuda()
    first = _probe(m, fa, ca, style, cout, r)
    other = _probe(m, fb, cb, style, cout, r)
    assert not torch.equal(other["raw1"], first["raw1"])
    again = _probe(m, fa, ca, style, cout, r)
    for k in ("raw1", "act1", "out"):
        assert torch.equal(again[k], first[k]), "%s of cloud A changed after cloud B: the scatter grid was not restored" % k
