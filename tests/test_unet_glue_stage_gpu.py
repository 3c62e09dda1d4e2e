"""Stage-level parity of the U-Net's glue, which the network tests see only through whole-network tolerances: the time
embedding (k_time_sinusoid, two k_small_linear), the CLIP mixing and the 61 AdaGN style Linears of k_style_linear (and
their cached copy from lion_unet_cache_style, which sampling uses), the FP stages' inputs (the time-embedding concat
k_copy_groups + k_fill_groups, the level's 3-NN from the side stream, the skip features, the interpolated MLP input)
and the classifier head (cls0 on the tensor cores, cls2 on the SIMT kernel, k_pf_to_pm when num_classes != 4).
lion_unet_probe runs lion_unet_forward and copies each of these out on the main stream where it is computed; a
side-stream result only after the main stream's wait for its event.  References are float64 on the device, built from
the probe's own previous stage; the 3-NN and the copies are compared bit for bit.

Maximum errors measured on one H100 80GB HBM3 (SXM, 700 W power limit) are listed next to each tolerance below."""
import ctypes as C

import pytest
import torch

from lion_b200 import _lib as L
from oracle import net as ON
from oracle import point_ops as OP
from tests import stage_ref as SR
from tests.synth import synth_state_dict
from tests.test_fp_stage_gpu import _ulps32
from tests.test_pvconv_tail_stage_gpu import _fold_err, _rel
from tests.test_stage_parity_gpu import _sum_err
from tests.util import gen

pytestmark = pytest.mark.gpu

N = 2048
TOL_SINU = 2e-7        # sinusoid, max-abs error (sin / cos of arguments up to ~1000 rad) (measured 5.7e-8)
TOL_LINEAR = 3.5e-7    # time-embedding Linears and style affines, max-abs error / max-abs reference (1.2e-7)
TOL_RAW = 1.3e-6       # cls0 raw output, max-abs error / max-abs reference (4.2e-7)
TOL_SUM_OWN = 1.5e-7   # cls0 sums against float64 sums of its own raw output (4.9e-8)
TOL_SUM_REF = 2.3e-6   # cls0 sums against float64 sums of the reference (7.6e-7)
TOL_FOLD = 4e-7        # cls0 fold against a float64 fold of its own sums (1.3e-7)
TOL_ACT = 4.2e-7       # cls0 output (unrounded swish), max-abs error / max-abs reference (1.4e-7)
TOL_OUT = 1.8e-6       # cls2 output against a float64 einsum of the probe's cls0 output (5.9e-7)
# each FP stage's output against the fp32 CPU oracle run of the whole network, B <= 3 (2.6e-3): TF32 operands through
# up to ~50 layers; the interpolation measured 0 fp32 ulps and is held to 1
TOL_STAGE = 8e-3
TIMES = [0.0, 1.0, 500.0, 999.0, 1000.0]


def _net(kind, E=64):
    """kind: prior, prior_clip or decoder; E: the prior's time-embedding width (cfg.ddpm.time_dim)."""
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.latent_points_ada import PVCNN2Unet
    clip = kind == "prior_clip"
    cfg = default_prior_cfg(clip=clip)
    if kind == "decoder":
        spec = ON.decoder_spec()
        net = PVCNN2Unet(3, 0, True, extra_feature_channels=1, input_dim=3, cfg=cfg, sa_blocks=ON.DEC_SA_BLOCKS,
                         fp_blocks=ON.FP_BLOCKS)
    else:
        spec = ON.prior_spec(time_dim=E, clip=clip)
        net = PVCNN2Unet(4, E, True, extra_feature_channels=1, input_dim=3, cfg=cfg, sa_blocks=ON.PRIOR_SA_BLOCKS,
                         fp_blocks=ON.FP_BLOCKS, clip_forge_enable=clip, clip_forge_dim=cfg.clipforge.feat_dim)
    sd = synth_state_dict({k: list(v.shape) for k, v in net.state_dict().items()}, 41)
    net.load_state_dict(sd)
    return net.cuda().eval(), {k: v.cuda() for k, v in sd.items()}, spec, cfg


def _stages(spec):
    """Per FP stage: (C_prev, cp, level points n, centres M, stage output channels, state-dict prefix of its last block)."""
    plan = ON.build_plan(spec)
    E = spec.embed_dim
    n = [N] + [blocks[-1]["m"] for blocks in plan["sa"]]
    out = []
    for j, blocks in enumerate(plan["fp"]):
        l = len(plan["sa"]) - 1 - j
        cp = spec.extra_feature_channels if l == 0 else plan["sa"][l - 1][-1]["mlp"][-1]
        cprev = blocks[0]["cin"] - cp - E
        cout = blocks[-1]["cout"] if blocks[-1]["kind"] == "pvconv" else blocks[-1]["mlp"][-1]
        out.append((cprev, cp, n[l], n[l + 1], cout, ON._prefix("fp", j, len(blocks) - 1, len(blocks))))
    return out, plan["ch_fp"]


def _pf(B, C, R):
    return torch.empty(B, -(-C // 4), R, 4, device="cuda")


def _cm(pf, C):
    """packed [B][G][R][4] -> [B,C,R]"""
    B, G, R, _ = pf.shape
    return pf.permute(0, 1, 3, 2).reshape(B, 4 * G, R)[:, :C]


def _probe(m, spec, x, t, style, clip, n_style, style_total):
    B = x.shape[0]
    E, d = spec.embed_dim, "cuda"
    st, ch = _stages(spec)
    T = dict(sinu=torch.empty(B, max(E, 1), device=d), h=torch.empty(B, max(E, 1), device=d), temb=torch.empty(B, max(E, 1), device=d),
             aff=torch.empty(B, style_total, device=d))
    taps = [T["sinu"], T["h"], T["temb"], T["aff"]]
    T["fp"] = []
    for cprev, cp, n, M, cout, _ in st:
        s = dict(cf=_pf(B, cprev + E, M), idx=torch.empty(B, n, 3, dtype=torch.int32, device=d), wgt=torch.empty(B, n, 3, device=d),
                 skip=_pf(B, cp, n), cat=_pf(B, cprev + E + -(-cp // 4) * 4, n), out=_pf(B, cout, n))
        T["fp"].append(s)
        taps += [s[k] for k in ("cf", "idx", "wgt", "skip", "cat", "out")]
    T.update(feat=_pf(B, ch, N), cls_raw=_pf(B, 128, N), cls_sums=torch.empty(2, B, 128, dtype=torch.float64, device=d),
             cls_aff=torch.empty(2, B, 128, device=d), hc=_pf(B, 128, N), out=torch.empty(B, N, spec.num_classes, device=d))
    taps += [T[k] for k in ("feat", "cls_raw", "cls_sums", "cls_aff", "hc")]
    arr = (C.c_void_p * len(taps))(*[p.data_ptr() for p in taps])
    table = (C.c_int * (2 * n_style))()
    L.check(L.lib().lion_unet_probe(m.h, L.ptr(x), L.ptr(t), L.ptr(style), L.ptr(clip), L.ptr(T["out"]), arr, len(taps), table,
                                    n_style, B, N, L.stream()), "unet_probe")
    torch.cuda.synchronize()
    T["table"] = [(table[2 * i], table[2 * i + 1]) for i in range(n_style)]
    return T, st


def _emd_layers(sd):
    """The AdaGN style Linears in module order: (prefix, channels)."""
    return [(k[:-len("emd.weight")], sd[k[:-len("emd.weight")] + "norm.weight"].numel()) for k in sd if k.endswith("emd.weight")]


@pytest.mark.parametrize("kind,B", [("prior", 1), ("prior", 3), ("prior", 32), ("prior_clip", 3), ("decoder", 3)])
def test_unet_glue_stages(kind, B):
    net, sd, spec, cfg = _net(kind)
    m = L.model_for(net, L.KIND_UNET, net.lion_desc(), net.lion_params())
    E = spec.embed_dim
    x = gen(80 + B, B, N, 4, scale=0.4).cuda()
    t = torch.tensor([TIMES[b % len(TIMES)] for b in range(B)], device="cuda") if E else None
    style = gen(81, B, cfg.latent_pts.style_dim).cuda()
    clip = gen(82, B, cfg.clipforge.feat_dim).cuda() if spec.clip else None
    layers = _emd_layers(sd)
    total = sum(2 * c for _, c in layers)
    P, st = _probe(m, spec, x, t, style, clip, len(layers), total)
    e = {}

    # time embedding, each stage from the probe's previous one
    if E:
        e["sinu"] = (P["sinu"].double() - SR.sinusoid(t, E).cuda()).abs().max().item()
        h = SR.linear_f64(P["sinu"], sd["embedf.0.weight"], sd["embedf.0.bias"], leaky=True)
        e["h"] = _rel(P["h"], h, (0, 1))
        e["temb"] = _rel(P["temb"], SR.linear_f64(P["h"], sd["embedf.2.weight"], sd["embedf.2.bias"]), (0, 1))
        assert e["sinu"] <= TOL_SINU and max(e["h"], e["temb"]) <= TOL_LINEAR, e

    # style affines: every layer at its recorded offset, against style @ W^T + b (after the CLIP mixing)
    s = style.double()
    if spec.clip:
        cf = SR.linear_f64(clip, sd["clip_forge_mapping.weight"], sd["clip_forge_mapping.bias"])
        s = SR.linear_f64(torch.cat([style.double(), cf], 1), sd["style_clip.weight"], sd["style_clip.bias"])
    e["aff"] = 0.0
    off = 0
    for (p, c), (o, n) in zip(layers, P["table"]):
        assert (o, n) == (off, 2 * c), "style layer %s: (offset, width) (%d, %d), expected (%d, %d)" % (p, o, n, off, 2 * c)
        ref = SR.linear_f64(s, sd[p + "emd.weight"], sd[p + "emd.bias"])
        e["aff"] = max(e["aff"], _rel(P["aff"][:, o:o + n], ref, (0, 1)))
        off += n
    assert e["aff"] <= TOL_LINEAR, "style affines: %.3e > %.1e" % (e["aff"], TOL_LINEAR)

    # FP stages: the 3-NN of each level on the oracle's FPS chain, the concat, the skip and the MLP input
    coords = [x[..., :3].permute(0, 2, 1).cpu().contiguous()]
    for _, (_, sa) in enumerate(spec.sa_blocks):
        coords.append(OP.furthest_point_sample(coords[-1], sa[0]))
    n_sa = len(spec.sa_blocks)
    tap = {}
    if B <= 3:
        with torch.no_grad():
            ON.unet_forward({k: v.cpu() for k, v in sd.items()}, spec, x.permute(0, 2, 1).cpu(), t=None if t is None else t.cpu(),
                            style=style.cpu(), clip_feat=None if clip is None else clip.cpu(), tap=tap)
    e["interp"] = e["stage"] = 0.0
    prev = None
    for j, ((cprev, cp, n, M, cout, pre), S) in enumerate(zip(st, P["fp"])):
        l = n_sa - 1 - j
        ridx, rwgt = OP.three_nn(coords[l], coords[l + 1])
        assert torch.equal(S["idx"].permute(0, 2, 1).cpu(), ridx), "stage %d: 3-NN indices differ from the oracle" % j
        assert torch.equal(S["wgt"].permute(0, 2, 1).cpu(), rwgt), "stage %d: 3-NN weights differ from the oracle" % j
        cfm = _cm(S["cf"], cprev + E)
        if prev is not None:
            assert torch.equal(cfm[:, :cprev], prev), "stage %d: centre features differ from the previous stage's output" % j
        if E:
            assert torch.equal(cfm[:, cprev:], P["temb"][:, :, None].expand(B, E, M)), "stage %d: temb concat is not temb" % j
        skip = _cm(S["skip"], -(-cp // 4) * 4)
        if l == 0:
            assert torch.equal(skip[:, 0], x[..., 3]) and (skip[:, 1:] == 0).all(), "level-0 skip is not [x[..., 3], 0, 0, 0]"
        cat = _cm(S["cat"], cprev + E + skip.shape[1])
        assert torch.isfinite(cat).all(), "stage %d: MLP input has NaNs" % j
        assert torch.equal(cat[:, cprev + E:], skip), "stage %d: skip part of the MLP input differs" % j
        e["interp"] = max(e["interp"], _ulps32(cat[:, :cprev + E], SR.interp_fma(cfm, S["idx"].permute(0, 2, 1), S["wgt"].permute(0, 2, 1))))
        prev = _cm(S["out"], cout)
        if tap:
            e["stage"] = max(e["stage"], _rel(prev, tap[pre].cuda().double(), (1, 2)))
    assert e["interp"] <= 1.0, "interpolation: %.2f fp32 ulps" % e["interp"]
    assert e["stage"] <= TOL_STAGE, "FP stage outputs against the oracle: %.3e > %.1e" % (e["stage"], TOL_STAGE)

    # head: cls0 from the probe's own input, cls2 from the probe's own cls0 output
    _, ch = _stages(spec)
    feat = _cm(P["feat"], ch)
    assert torch.equal(feat, prev), "head input differs from the last FP stage's output"
    raw, hc = _cm(P["cls_raw"], 128), _cm(P["hc"], 128)
    ref = SR.point_conv(feat, sd["classifier.0.layers.0.weight"], sd["classifier.0.layers.0.bias"])
    e["raw"] = _rel(raw, ref, (1, 2))
    e["sum_own"] = _sum_err(P["cls_sums"].unbind(0), raw.double(), 2)
    e["sum_ref"] = _sum_err(P["cls_sums"].unbind(0), ref, 2)
    rs, rt = SR.mlp_fold(*P["cls_sums"].unbind(0), sd, "classifier.0.layers.1.", s, float(N))
    e["fold"] = _fold_err(*P["cls_aff"].unbind(0), rs, rt)
    e["act"] = _rel(hc, SR.act_rows(raw, *P["cls_aff"].unbind(0), rna=False).double(), (1, 2))
    w2 = sd["classifier.2.weight"].reshape(spec.num_classes, 128).double()
    out_ref = torch.einsum("oc,bcn->bno", w2, hc.double()) + sd["classifier.2.bias"].double()
    e["out"] = _rel(P["out"], out_ref, (1, 2))
    print("unet %s B=%d: %s" % (kind, B, ", ".join("%s %.2e" % kv for kv in e.items())))
    assert e["raw"] <= TOL_RAW, "cls0 raw output: %.3e > %.1e" % (e["raw"], TOL_RAW)
    assert e["sum_own"] <= TOL_SUM_OWN and e["sum_ref"] <= TOL_SUM_REF, "cls0 sums: %.3e / %.3e" % (e["sum_own"], e["sum_ref"])
    assert e["fold"] <= TOL_FOLD, "cls0 fold: %.3e > %.1e" % (e["fold"], TOL_FOLD)
    assert e["act"] <= TOL_ACT, "cls0 output: %.3e > %.1e" % (e["act"], TOL_ACT)
    assert e["out"] <= TOL_OUT, "cls2 output: %.3e > %.1e" % (e["out"], TOL_OUT)

    # the probe computes what lion_unet_forward computes; the cached style vectors are the inline ones, bit for bit
    inline = net.forward_point_major(x, t=t, style=style, clip_feat=clip)
    assert torch.equal(inline, P["out"]), "probe output differs from lion_unet_forward"
    L.check(L.lib().lion_unet_cache_style(m.h, L.ptr(style), L.ptr(clip), B, L.stream()), "unet_cache_style")
    cached, _ = _probe(m, spec, x, t, None, None, len(layers), total)
    assert torch.equal(cached["aff"], P["aff"]), "cached style affines differ from the inline ones"
    assert torch.equal(cached["out"], P["out"]), "output with the cached style differs from the inline style"


@pytest.mark.parametrize("E", [256])
def test_unet_time_embedding_wide(E):
    """A prior U-Net with time_dim = 256: 128 frequencies, more than the 64 threads k_time_sinusoid is launched with.
    The sinusoid and the two time-embedding Linears against float64, each from the probe's previous stage."""
    net, sd, spec, cfg = _net("prior", E)
    m = L.model_for(net, L.KIND_UNET, net.lion_desc(), net.lion_params())
    B = 2
    x = gen(90, B, N, 4, scale=0.4).cuda()
    t = torch.tensor([999.0, 1000.0], device="cuda")
    style = gen(91, B, cfg.latent_pts.style_dim).cuda()
    layers = _emd_layers(sd)
    P, _ = _probe(m, spec, x, t, style, None, len(layers), sum(2 * c for _, c in layers))
    e = {"sinu": (P["sinu"].double() - SR.sinusoid(t, E).cuda()).abs().max().item()}
    e["h"] = _rel(P["h"], SR.linear_f64(P["sinu"], sd["embedf.0.weight"], sd["embedf.0.bias"], leaky=True), (0, 1))
    e["temb"] = _rel(P["temb"], SR.linear_f64(P["h"], sd["embedf.2.weight"], sd["embedf.2.bias"]), (0, 1))
    print("unet time embedding E=%d: %s" % (E, ", ".join("%s %.2e" % kv for kv in e.items())), flush=True)
    assert e["sinu"] <= TOL_SINU and max(e["h"], e["temb"]) <= TOL_LINEAR, e
    assert torch.equal(net.forward_point_major(x, t=t, style=style), P["out"]), "probe output differs from lion_unet_forward"
