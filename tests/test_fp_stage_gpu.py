"""Stage-level float64 parity of the FP module, which the module test sees only through a 2e-3 tolerance: the 3-NN search
of k_three_nn_c4 (centres tiled through shared memory, 1024 at a time), the interpolation k_interp_rows and the skip copy
k_copy_groups that build the MLP input [interpolated | skip], and the unpooled SharedMLP (1x1 convolutions on the tensor
cores, GroupNorm sums, AdaGN fold, k_act_rows<1>).  lion_fp_probe runs the product code, NaN-fills the MLP input before
its producers run (so that a row or channel nobody writes shows up), and returns each stage's input and output; every
reference below is built from the probe's own previous stage, so each tolerance covers one kernel.  References are
float64 on the device with the TF32 operand model of tests/stage_ref.py.

Maximum errors measured on one H100 80GB HBM3 (SXM, 700 W power limit) are listed next to each tolerance below."""
import ctypes as C

import pytest
import torch

from lion_b200 import _lib as L
from oracle import point_ops as OP
from tests import stage_ref as SR
from tests.test_pvconv_tail_stage_gpu import _fold_err, _rel, _tf32_ulps
from tests.test_stage_parity_gpu import _cfg, _load, _sum_err
from tests.util import gen

pytestmark = pytest.mark.gpu

TOL_RAW = 3.5e-6       # raw 1x1 output, max-abs error / max-abs reference, per shape (measured 1.2e-6)
TOL_SUM_OWN = 5e-7     # GroupNorm sums against float64 sums of the probe's own raw output (1.6e-7)
TOL_SUM_REF = 5.5e-6   # GroupNorm sums against float64 sums of the reference (1.8e-6)
TOL_FOLD = 4e-7        # folded scale / shift against a float64 fold of the probe's own sums (1.3e-7)
TOL_ACT_LAST = 4e-7    # last layer's (unrounded) activation, max-abs error / max-abs reference, per shape (1.4e-7)
TOL_ALONE_SUM = 1.5e-7  # a shape alone against the same shape in a batch: sums relative to the shape's largest |sum| (5.1e-8)
# The interpolation measured 0 ulps (the fma chain exactly) and is held to 1 ulp; the non-last activations measured
# 1 TF32 ulp and are held to it.
# (cc, cp, mlp, N, M): the four FP stages of a sampling step
STEP = [(192, 128, (128, 128), 64, 16), (192, 128, (128, 128), 256, 64), (192, 64, (128, 128), 1024, 256),
        (192, 1, (128, 128, 64), 2048, 1024)]
# (cc, cp, mlp, N, M, B, cloud)
CASES = ([(*s, B, "subset") for s in STEP for B in (2, 32)] +
         [(192, 1, (128, 128, 64), 2048, 1025, 2, "gauss"),      # the centre tile loop past 1024 ...
          (64, 1, (64, 64), 2048, 2048, 2, "gauss"),              # ... and two full tiles
          (64, 4, (64,), 300, 1, 2, "gauss"),                     # fewer than three centres
          (64, 4, (64,), 300, 2, 3, "gauss"),
          (128, 64, (128, 128), 700, 256, 3, "gauss"),            # ragged N
          (128, 64, (128, 64), 100, 64, 2, "gauss"),              # N < blockDim
          (128, 0, (128, 128), 256, 64, 2, "gauss"),              # no skip
          (128, 6, (128, 128), 256, 64, 2, "gauss"),              # skip padded 6 -> 8
          (128, 64, (128, 128), 512, 128, 2, "dup"),              # every centre twice
          (128, 64, (128, 128), 1024, 300, 2, "lattice")])        # exact distance ties


def _cloud(kind, B, N, M, seed):
    """(points [B,3,N], centres [B,3,M]).  subset: the centres are the first M points (d = 0, clamped to 1e-10); dup:
    M / 2 points each listed twice; lattice: points and centres on a grid of spacing 1/8 (exact squared distances,
    many ties), centres in shuffled order so that the tie-break is by index, not by position."""
    pc = gen(seed, B, 3, N, scale=0.3)
    if kind == "subset":
        return pc, pc[:, :, :M].contiguous()
    if kind == "gauss":
        return pc, gen(seed + 1, B, 3, M, scale=0.3)
    if kind == "dup":
        c = gen(seed + 1, B, 3, M // 2, scale=0.3)
        return pc, torch.cat([c, c], 2)[:, :, torch.randperm(M, generator=torch.Generator().manual_seed(seed))].contiguous()
    g = torch.Generator().manual_seed(seed)
    pts = torch.randint(-8, 8, (B, 3, N), generator=g).float() / 8
    ce = torch.randint(-4, 4, (B, 3, M), generator=g).float() / 4        # the even sites of the same grid
    return pts, ce


def _fp_probe(m, pc, cc, cf, pf, style, outs, ccat):
    B, N, M = pc.shape[0], pc.shape[2], cc.shape[2]
    d, tot = "cuda", sum(outs)
    o = dict(idx=torch.empty(B, 3, N, dtype=torch.int32, device=d), wgt=torch.empty(B, 3, N, device=d),
             cat=torch.empty(B, ccat, N, device=d), raw=torch.empty(B * N * tot, device=d), act=torch.empty(B * N * tot, device=d),
             s=torch.empty(B * tot, dtype=torch.float64, device=d), q=torch.empty(B * tot, dtype=torch.float64, device=d),
             sc=torch.empty(B * tot, device=d), sh=torch.empty(B * tot, device=d))
    L.check(L.lib().lion_fp_probe(m.h, L.ptr(pc), L.ptr(cc), L.ptr(cf), L.ptr(pf), L.ptr(style), L.ptr(o["idx"]), L.ptr(o["wgt"]),
                                  L.ptr(o["cat"]), L.ptr(o["raw"]), L.ptr(o["act"]), L.ptr(o["s"]), L.ptr(o["q"]), L.ptr(o["sc"]),
                                  L.ptr(o["sh"]), B, N, M, L.stream()), "fp_probe")
    torch.cuda.synchronize()
    layers, off = [], 0
    for c in outs:
        layers.append(dict(raw=o["raw"][off * N:(off + B * c) * N].view(B, c, N), act=o["act"][off * N:(off + B * c) * N].view(B, c, N),
                           **{k: o[k][off:off + B * c].view(B, c) for k in ("s", "q", "sc", "sh")}))
        off += B * c
    o["layers"] = layers
    return o


def _ulps32(got, ref):
    """|got - ref| in units of the fp32 ulp of ref."""
    _, e = torch.frexp(ref.double().abs())
    return ((got.double() - ref.double()).abs() / torch.ldexp(torch.ones_like(ref, dtype=torch.float64), (e - 24).to(torch.int32))).max().item()


@pytest.mark.parametrize("cc,cp,outs,N,M,B,cloud", CASES)
def test_fp_stage(cc, cp, outs, N, M, B, cloud):
    from lion_b200.models.pvcnn2_ada import PointNetFPModule
    outs = list(outs)
    mod, sd = _load(PointNetFPModule(cc + cp, outs, cfg=_cfg()), 35)
    m = L.model_for(mod, L.KIND_FP, [cc, cp, 128, len(outs)] + outs, mod.mlp.lion_params())
    pc, ctr = _cloud(cloud, B, N, M, 70 + N + M)
    cf, style = gen(71, B, cc, M).cuda(), gen(72, B, 128).cuda()
    pf = gen(73, B, cp, N).cuda() if cp else None
    pc, ctr = pc.cuda(), ctr.cuda()
    cp4 = -(-cp // 4) * 4
    ccat = cc + cp4
    P = _fp_probe(m, pc, ctr, cf, pf, style, outs, ccat)

    # 3-NN: the oracle's indices and its fp32 weights, bit for bit
    ridx, rwgt = OP.three_nn(pc.cpu(), ctr.cpu())
    assert torch.equal(P["idx"].cpu(), ridx), "3-NN indices differ from the oracle (%d points)" % int((P["idx"].cpu() != ridx).sum())
    assert torch.equal(P["wgt"].cpu(), rwgt), "3-NN weights differ from the oracle"

    # MLP input: interpolation within 1 fp32 ulp of the fma chain, the skip bitwise, the padding exactly 0
    cat = P["cat"]
    assert torch.isfinite(cat).all(), "the MLP input has NaNs: a row or channel nobody wrote"
    e_interp = _ulps32(cat[:, :cc], SR.interp_fma(cf, P["idx"], P["wgt"]))
    if cp:
        assert torch.equal(cat[:, cc:cc + cp], pf), "skip channels differ from the input"
    assert (cat[:, cc + cp:] == 0).all(), "skip padding channels are not zero"

    # MLP: each layer from the probe's own input to it
    x = cat
    errs = []
    for l, c in enumerate(outs):
        Lr = P["layers"][l]
        w = sd["mlp.layers.%d.weight" % (3 * l)].reshape(c, -1)
        if l == 0:
            w = torch.cat([w, torch.zeros(c, ccat - cc - cp, device="cuda")], 1)
        ref = SR.point_conv(x, w.contiguous(), sd["mlp.layers.%d.bias" % (3 * l)])
        v = Lr["raw"].double()
        e_raw = _rel(v, ref, (1, 2))
        e_own, e_ref = _sum_err((Lr["s"], Lr["q"]), v, 2), _sum_err((Lr["s"], Lr["q"]), ref, 2)
        rs, rt = SR.mlp_fold(Lr["s"], Lr["q"], sd, "mlp.layers.%d." % (3 * l + 1), style, float(N))
        e_fold = _fold_err(Lr["sc"], Lr["sh"], rs, rt)
        last = l == len(outs) - 1
        ra = SR.act_rows(Lr["raw"], Lr["sc"], Lr["sh"], rna=not last)
        if last:
            e_act = _rel(Lr["act"], ra.double(), (1, 2))
            assert e_act <= TOL_ACT_LAST, "layer %d activation: %.3e > %.1e" % (l, e_act, TOL_ACT_LAST)
        else:
            e_act = _tf32_ulps(Lr["act"], ra)
            assert torch.equal(Lr["act"], SR.tf32_rna(Lr["act"])), "layer %d activation is not rounded to TF32" % l
            assert e_act <= 1.0, "layer %d activation: %.2f TF32 ulps" % (l, e_act)
        errs.append((e_raw, e_own, e_ref, e_fold, e_act))
        assert e_raw <= TOL_RAW, "layer %d raw output: %.3e > %.1e" % (l, e_raw, TOL_RAW)
        assert e_own <= TOL_SUM_OWN, "layer %d sums against its own output: %.3e > %.1e" % (l, e_own, TOL_SUM_OWN)
        assert e_ref <= TOL_SUM_REF, "layer %d sums against the reference: %.3e > %.1e" % (l, e_ref, TOL_SUM_REF)
        assert e_fold <= TOL_FOLD, "layer %d fold: %.3e > %.1e" % (l, e_fold, TOL_FOLD)
        x = Lr["act"]
    print("fp %s: interp %.2f ulp; per layer raw / sums own / sums ref / fold / act: %s" % (
        (cc, cp, outs, N, M, B, cloud), e_interp, "; ".join(" ".join("%.2e" % e for e in t) for t in errs)))
    assert e_interp <= 1.0, "interpolation: %.2f fp32 ulps" % e_interp

    # the module output: lion_fp_module_fwd gives the same bits
    args = (pc, ctr, cf) + ((pf,) if cp else ()) + (None, style)
    assert torch.equal(mod(args)[0], P["layers"][-1]["act"]), "probe output differs from lion_fp_module_fwd"

    # the same bits run after run; every shape alone: the same 3-NN and MLP input, sums within a tolerance (the tensor-core
    # GroupNorm sums depend on the batch in their last fp32 bits, see tests/test_pvconv_tail_stage_gpu.py)
    again = _fp_probe(m, pc, ctr, cf, pf, style, outs, ccat)
    for k in ("idx", "wgt", "cat", "raw", "act", "s", "q", "sc", "sh"):
        assert torch.equal(again[k], P[k]), "%s is not bit-reproducible" % k
    if B > 1:
        e_sum = 0.0
        for b in range(B):
            sl = slice(b, b + 1)
            one = _fp_probe(m, pc[sl].contiguous(), ctr[sl].contiguous(), cf[sl].contiguous(),
                            pf[sl].contiguous() if cp else None, style[sl].contiguous(), outs, ccat)
            for k in ("idx", "wgt", "cat"):
                assert torch.equal(one[k][0], P[k][b]), "%s of shape %d: B = %d differs from B = 1" % (k, b, B)
            for l in range(len(outs)):
                for k in ("s", "q"):
                    a, r = one["layers"][l][k][0], P["layers"][l][k][b]
                    e_sum = max(e_sum, ((a - r).abs().max() / r.abs().max()).item())
        print("  alone vs batch: sums %.2e" % e_sum)
        assert e_sum <= TOL_ALONE_SUM, "GroupNorm sums, alone vs batch: %.3e > %.1e" % (e_sum, TOL_ALONE_SUM)
