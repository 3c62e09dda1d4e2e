"""Sampling under torch.autocast("cuda", float16): the FP16-operand second 3x3x3 convolution of every PVConv.

The FP16 route (LION_FWD_CONV_FP16) changes two kernels: the AdaGN-1 + Swish pass writes its grid as FP16 (rounded to
nearest even) and the second convolution multiplies FP16 activations by FP16 weights with fp32 accumulation.  These
tests check the convolution alone (Conv3d), the PVConv stage around it (lion_pvconv_probe_flags, float64 references
with the FP16 operand model), one network step against the fp32 oracle, and the samplers' enable_autocast flag.

Maximum errors measured on one H100 80GB HBM3 (SXM, 700 W power limit) are listed next to each tolerance below."""
import ctypes as C

import numpy as np
import pytest
import torch

from lion_b200 import _lib as L
from tests import stage_ref as SR
from tests.synth import synth_state_dict
from tests.test_pvconv_tail_stage_gpu import PV_CASES, TOL_FOLD, TOL_SUM_OWN, _conv2_kernel, _fold_err, _gn
from tests.test_stage_parity_gpu import _cfg, _clouds, _load, _sum_err
from tests.util import gen, rel_err, rms_err

pytestmark = pytest.mark.gpu

TOL_CONV_F64 = 2e-5     # Conv3d against float64 conv3d of FP16-rounded operands, per shape: fp32 accumulation order only (6.4e-6)
TOL_CONV_CUDNN = 2e-3   # Conv3d against cuDNN under autocast (fp16 output), per shape (8.0e-4)
TOL_CONV_SUMS = 1e-5    # fused GroupNorm sums against float64 sums of the kernel's own output (7.9e-8)
TOL_CONV2 = 3.3e-5      # stage: raw second-convolution output against float64 of the probe's act1 and FP16 weights (8.6e-6)
# stage: act1 within 1 FP16 ulp of the float64 model (0.50 ulp); conv2 sums against its own output TOL_SUM_OWN (9.7e-8);
# AdaGN-2 + SE fold TOL_FOLD (2.1e-7)
# network, B = 32, against the oracle's eager port on the GPU (the reference's point kernels, TF32 off):
TOL_NET_RATIO = 1.5     # err(FP16) <= 1.5 x err(TF32): the operand mantissas are equal (2.62e-3 vs 2.43e-3: 1.08)
# and err(FP16) <= err(the same oracle under torch.autocast(float16), point operators in fp32) (2.62e-3 vs 4.76e-3)
TOL_LOOP_RMS = 5e-2     # 10 DDPM steps, FP16 against TF32 (relative RMS, 2.8e-2)

CONV_CASES = [(32, 32, 32, 32), (64, 64, 32, 32), (64, 64, 16, 32), (128, 128, 16, 32), (128, 128, 8, 32),
              (32, 32, 13, 1), (64, 64, 13, 2), (128, 128, 13, 3)]


def _conv(cin, cout, seed):
    from lion_b200.models.pvcnn2_ada import Conv3d
    m = Conv3d(cin, cout).cuda()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        m.weight.copy_(torch.randn(m.weight.shape, generator=g) * (1.0 / (27 * cin) ** 0.5))
        m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
    return m


def _per_shape(got, ref):
    B = got.shape[0]
    return ((got.double() - ref.double()).view(B, -1).abs().amax(1) / ref.double().view(B, -1).abs().amax(1)).max().item()


@pytest.mark.parametrize("cin,cout,r,B", CONV_CASES)
def test_conv3d_fp16(cin, cout, r, B):
    m = _conv(cin, cout, 3 + cin + r)
    x = gen(40 + r + B, B, cin, r, r, r).cuda()
    with torch.autocast("cuda", dtype=torch.float16):
        y, s, q = m(x, return_gn_stats=True)
        y2, s2, q2 = m(x, return_gn_stats=True)
        ref_cudnn = torch.nn.functional.conv3d(x, m.weight, m.bias, padding=1)
    torch.cuda.synchronize()
    assert y.dtype == torch.float32 and ref_cudnn.dtype == torch.float16
    # the FP16 kernel ran: TF32 and FP16 operands differ only at rounding ties and below 2^-14, which this input has
    assert not torch.equal(y, m(x)), "the call under autocast gave the bits of the TF32 route"
    assert torch.equal(y, y2) and torch.equal(s, s2) and torch.equal(q, q2), "not bit-reproducible run to run"
    ref = SR.conv3x3x3_f64(x.half().double(), m.weight.detach().half().double(), m.bias.detach().double())
    e64 = _per_shape(y, ref)
    ecu = _per_shape(y, ref_cudnn.float())
    v = y.double().view(B, cout, -1)
    esum = _sum_err((s, q), v, 2)
    print("conv3d fp16 (%d,%d,%d,B=%d): vs f64 %.2e, vs cuDNN autocast %.2e, sums %.2e" % (cin, cout, r, B, e64, ecu, esum))
    assert e64 <= TOL_CONV_F64, e64
    assert ecu <= TOL_CONV_CUDNN, ecu
    assert esum <= TOL_CONV_SUMS, esum


@pytest.mark.parametrize("cin,cout,r,B", [(4, 32, 8, 2), (32, 40, 8, 2), (64, 32, 8, 2)])
def test_conv3d_fp16_unserved_shapes_run_as_tf32(cin, cout, r, B):
    """Shapes the FP16 kernel does not serve give the bits of the same call outside autocast."""
    m = _conv(cin, cout, 5 + cin)
    x = gen(41, B, cin, r, r, r).cuda()
    y32, s32, q32 = m(x, return_gn_stats=True)
    with torch.autocast("cuda", dtype=torch.float16):
        y16, s16, q16 = m(x, return_gn_stats=True)
    assert torch.equal(y32, y16) and torch.equal(s32, s16) and torch.equal(q32, q16)
    with torch.autocast("cuda", dtype=torch.bfloat16):      # bf16 autocast is not the FP16 route: fp32 / TF32 as today
        yb = m(x)
    assert torch.equal(y32, yb)


def _probe16(m, feats, coords, style, cout, r):
    B, _, N = feats.shape
    rp, d = r + 2, "cuda"
    o = dict(raw1=torch.empty(B, cout, r, r, r, device=d), act1=torch.empty(B, cout, rp, rp, rp, device=d),
             raw2=torch.empty(B, cout, r, r, r, device=d), rawp=torch.empty(B, cout, N, device=d),
             sums=torch.empty(4, B, cout, dtype=torch.float64, device=d), affine=torch.empty(6, B, cout, device=d),
             fused=torch.empty(B, cout, N, device=d), out=torch.empty(B, cout, N, device=d))
    kern = C.c_int(-1)
    L.check(L.lib().lion_pvconv_probe_flags(m.h, L.ptr(feats), L.ptr(coords), L.ptr(style), L.ptr(o["raw1"]), L.ptr(o["act1"]),
                                            L.ptr(o["raw2"]), L.ptr(o["rawp"]), L.ptr(o["sums"]), L.ptr(o["affine"]),
                                            L.ptr(o["fused"]), L.ptr(o["out"]), C.byref(kern), B, N, L.FWD_CONV_FP16, L.stream()),
            "pvconv_probe_flags")
    torch.cuda.synchronize()
    o["kernel"] = kern.value
    return o


def _fp16_ulp(ref):
    """the FP16 ulp at |ref| (10 explicit mantissa bits; subnormal spacing 2^-24 below 2^-14)"""
    _, e = torch.frexp(ref.abs())
    return torch.ldexp(torch.ones_like(ref, dtype=torch.float64), (e - 11).clamp_min(-24).to(torch.int32))


@pytest.mark.parametrize("cin,cout,r,N,B,attn", [c for c in PV_CASES if c[1] in (32, 64, 128)])
def test_pvconv_fp16_stage(cin, cout, r, N, B, attn):
    from lion_b200.models.pvcnn2_ada import PVConv
    mod, sd = _load(PVConv(cin, cout, 3, r, with_se=True, attention=attn, cfg=_cfg()), 33)
    m = L.model_for(mod, L.KIND_PVCONV, mod.lion_desc(), mod.lion_params())
    feats = gen(60 + cin, B, cin, N).cuda()
    coords = _clouds(B, N, r, 7 * r + N).cuda()
    style = gen(61, B, 128).cuda()
    V = float(r ** 3)
    P = _probe16(m, feats, coords, style, cout, r)
    assert P["kernel"] == _conv2_kernel(cout, r, B), "second convolution ran kernel %d" % P["kernel"]
    s1, t1, sp, tp, s2, t2 = P["affine"].unbind(0)
    sum2, sq2, _, _ = P["sums"].unbind(0)

    # FP16 act1: exactly FP16-representable, within 1 FP16 ulp of the float64 model, 0 on every halo position
    act = P["act1"]
    inner = (slice(None), slice(None), slice(1, -1), slice(1, -1), slice(1, -1))
    halo = torch.ones_like(act, dtype=torch.bool)
    halo[inner] = False
    assert torch.isfinite(act).all(), "act1 grid has NaNs: a position the FP16 activation pass did not write"
    assert (act[halo] == 0).all(), "act1 halo is not zero"
    assert torch.equal(act, act.half().float()), "act1 is not FP16"
    a = P["raw1"].double() * s1[:, :, None, None, None].double() + t1[:, :, None, None, None].double()
    ref_act = a * torch.sigmoid(a)
    e_act = ((act[inner].double() - ref_act).abs() / _fp16_ulp(ref_act)).max().item()
    assert e_act <= 1.0, "act1 is %.2f FP16 ulps from the float64 model" % e_act

    # second convolution on the probe's own act1 with FP16 weights, and its sums
    ref2 = SR.conv3x3x3_f64(act[inner].double(), sd["voxel_layers.4.weight"].half().double(), sd["voxel_layers.4.bias"].double())
    v2, rv2 = P["raw2"].double().view(B, cout, -1), ref2.view(B, cout, -1)
    e_conv2 = ((v2 - rv2).abs().amax(2) / rv2.abs().amax(2)).max().item()
    e2_own = _sum_err((sum2, sq2), v2, 2)
    rs2, rt2 = SR.fold_se(sum2, sq2, *_gn(sd, 5, style), V, sd["voxel_layers.6.fc.0.weight"], sd["voxel_layers.6.fc.2.weight"])
    e_fold2 = _fold_err(s2, t2, rs2, rt2)
    print("pvconv fp16 stage (%d,%d,%d,N=%d,B=%d): act1 %.2f ulp, conv2 %.2e, sums %.2e, fold %.2e"
          % (cin, cout, r, N, B, e_act, e_conv2, e2_own, e_fold2))
    assert e_conv2 <= TOL_CONV2, e_conv2
    assert e2_own <= TOL_SUM_OWN, e2_own
    assert e_fold2 <= TOL_FOLD, e_fold2


def _prior(seed=11, steps=None):
    import json
    import os
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.latent_points_ada_localprior import PVCNN2Prior
    keys = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "keys.json")))
    cfg = default_prior_cfg(num_steps=steps)
    m = PVCNN2Prior(cfg.sde, 1, cfg)
    sd = synth_state_dict(keys["prior"], seed)
    m.load_state_dict(sd)
    return m.cuda().eval(), sd, cfg


class _PointOpsFp32:
    """A point-operator backend of oracle/net.py as the reference runs it under autocast: its autograd Functions are
    custom_fwd(cast_inputs=torch.float32), so every floating-point input is cast to fp32 and the operator runs with
    autocast off.  `log` collects the index-like results (voxel indices, FPS centres, ball-query neighbours)."""

    def __init__(self, ops, log):
        self.ops, self.log = ops, log

    def __getattr__(self, name):
        fn = getattr(self.ops, name)

        def call(*a, **k):
            a = [v.float() if torch.is_tensor(v) and v.is_floating_point() else v for v in a]
            with torch.autocast("cuda", enabled=False):
                out = fn(*a, **k)
            if name == "voxel_coords":
                self.log.append((name, out[1]))
            elif name in ("furthest_point_sample", "ball_query"):
                self.log.append((name, out))
            return out
        return call


def test_prior_step_b32_fp16_against_oracle_and_oracle_autocast():
    """One PVCNN2Prior step at B = 32.  y32 = the oracle's eager port on the GPU (oracle/net.py with the reference's
    own point kernels, oracle/_ref) with TF32 disabled; err(y) = max|y - y32| / max|y32|.  The FP16 route is no further
    from y32 than 1.5x the TF32 route and no further than the same oracle run under torch.autocast(float16) -- the
    reference's autocast route -- and the voxel / FPS / ball-query indices of that route equal the fp32 ones."""
    from oracle import build_ref
    from oracle import net as ON
    from oracle import point_ops, ref_cuda_ops
    if build_ref.load_ref() is None:
        pytest.skip("oracle/_ref/_pvcnn_backend.so was not built (the reference sources were not available to build())")
    m, sd, _ = _prior()
    B, dev = 32, torch.device("cuda")
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, 8192, 1, 1, generator=g).cuda()
    style = torch.randn(B, 128, 1, 1, generator=g).cuda()
    t = torch.randint(1, 1001, (B,), generator=g).float().cuda()
    e32 = m(x=x, t=t, condition_input=style)
    with torch.autocast("cuda", dtype=torch.float16):
        e16 = m(x=x, t=t, condition_input=style)
        again = m(x=x, t=t, condition_input=style)
    assert e16.dtype == torch.float32 and torch.isfinite(e16).all()
    assert torch.equal(e16, again), "the FP16 forward is not bit-reproducible run to run"
    assert not torch.equal(e16, e32), "autocast did not change the route"
    # outside autocast the TF32 route is unchanged by an FP16 call in between
    assert torch.equal(m(x=x, t=t, condition_input=style), e32)

    sdd = {k: v.to(dev) for k, v in sd.items()}
    logs = {}
    flags = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    try:
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        for mode in ("fp32", "autocast"):
            logs[mode] = []
            ON.set_point_ops(_PointOpsFp32(ref_cuda_ops, logs[mode]))
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16, enabled=mode == "autocast"):
                logs[mode + "_out"] = ON.prior_forward(sdd, ON.prior_spec(), x, t, style)
    finally:
        ON.set_point_ops(point_ops)
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = flags
    y32, yac = logs["fp32_out"], logs["autocast_out"]
    assert len(logs["fp32"]) == len(logs["autocast"]) > 0
    for (n0, a), (n1, b) in zip(logs["fp32"], logs["autocast"]):
        assert n0 == n1 and torch.equal(a, b), "%s differs between the fp32 and the autocast route" % n0
    err16, err32, errac = rel_err(e16, y32), rel_err(e32, y32), rel_err(yac.float(), y32)
    print("prior step B=32 vs the fp32 oracle: FP16 %.3e, TF32 %.3e, oracle under autocast %.3e" % (err16, err32, errac))
    assert err16 <= TOL_NET_RATIO * err32, (err16, err32)
    assert err16 <= errac, (err16, errac)


def test_ddpm_loop_autocast_graph_equals_eager():
    from lion_b200.utils.diffusion_pvd import DiffusionDiscretized
    m, _, cfg = _prior(steps=10)
    diff = DiffusionDiscretized(cfg.sde, None, cfg)
    g = torch.Generator(device="cuda").manual_seed(3)
    x_T = torch.randn(1, 8192, 1, 1, device="cuda", generator=g)
    zs = list(torch.randn(10, 1, 8192, 1, 1, device="cuda", generator=g))
    style = torch.randn(1, 128, 1, 1, device="cuda", generator=g)
    outs = {}
    for use_graph in (False, True):
        diff.use_cuda_graph = use_graph
        outs[use_graph], _ = diff.run_denoising_diffusion(m, 1, [8192, 1, 1], condition_input=style, given_noise=(x_T, zs),
                                                          enable_autocast=True)
    assert torch.isfinite(outs[True]).all()
    assert torch.equal(outs[False], outs[True]), "graph-replayed FP16 loop differs from the eager one"
    diff.use_cuda_graph = True
    tf32, _ = diff.run_denoising_diffusion(m, 1, [8192, 1, 1], condition_input=style, given_noise=(x_T, zs))
    e = rms_err(outs[True], tf32)
    print("10 DDPM steps, FP16 vs TF32: relative RMS %.3e" % e)
    assert e < TOL_LOOP_RMS, e


def test_samplers_accept_enable_autocast():
    from lion_b200.models.score_sde.resnet import PriorSEDrop
    from lion_b200.models.vae_adain import Model
    from lion_b200.trainers.train_2prior import generate_samples_vada_2prior
    from lion_b200.utils.diffusion_continuous import make_diffusion
    from lion_b200.utils.diffusion_pvd import DiffusionDiscretized
    import json
    import os
    keys = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "keys.json")))
    lp, _, cfg = _prior(steps=6)
    gp = PriorSEDrop(cfg.sde, 128, cfg)
    gp.load_state_dict(synth_state_dict(keys["global"], 14))
    gp = gp.cuda().eval()
    vae = Model(cfg)
    vae.decoder.load_state_dict(synth_state_dict(keys["decoder"], 13))
    vae = vae.cuda().eval()
    diff = DiffusionDiscretized(cfg.sde, None, cfg)
    style = torch.randn(2, 128, 1, 1, device="cuda")
    res = {}
    for ac in (True, False):                          # same seeds and noise with the flag on and off
        torch.manual_seed(9)
        res["ddim", ac] = diff.run_ddim(lp, 2, [8192, 1, 1], 1.0, ac, is_image=False, ddim_step=4, condition_input=style)
        torch.manual_seed(9)
        res["ddpm", ac] = generate_samples_vada_2prior(vae.latent_shape(), torch.nn.ModuleList([gp, lp]), diff, vae, 2, ac)[0]
        ode = make_diffusion(cfg.sde)
        noise = torch.randn(1, 8192, 1, 1, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
        res["ode", ac] = ode.sample_model_ode(lp, 1, [8192, 1, 1], 1e-5, 1e-2, ac, 1.0, noise=noise, condition_input=style[:1],
                                              init_t=0.05)
    out, hist = res["ddim", True]
    assert out.shape == (2, 8192, 1, 1) and torch.isfinite(out).all() and len(hist) == 4
    img = res["ddpm", True]
    assert img.shape == (2, 2048, 3) and torch.isfinite(img).all()
    y, nfe, _ = res["ode", True]
    assert y.shape == (1, 8192, 1, 1) and torch.isfinite(y).all() and nfe > 0
    # the flag reached the model call: each sampler's result differs from the same seeded call without it
    assert not torch.equal(out, res["ddim", False][0]), "run_ddim ignored enable_autocast"
    assert not torch.equal(img, res["ddpm", False]), "generate_samples_vada_2prior ignored enable_autocast"
    assert not torch.equal(y, res["ode", False][0]), "sample_model_ode ignored enable_autocast"


def test_trainer_sample_forwards_autocast_train():
    from lion_b200.trainers.train_2prior import generate_samples_vada_2prior
    from lion_b200.trainers.train_prior import Trainer
    from lion_b200.config import default_prior_cfg
    cfg = default_prior_cfg(num_steps=6)
    assert cfg.sde.autocast_train is False
    cfg.sde.autocast_train = True
    tr = Trainer(cfg)
    shp = lambda m: {k: list(v.shape) for k, v in m.state_dict().items()}
    tr.dae[0].load_state_dict(synth_state_dict(shp(tr.dae[0]), 14))
    tr.dae[1].load_state_dict(synth_state_dict(shp(tr.dae[1]), 11))
    tr.model.decoder.load_state_dict(synth_state_dict(shp(tr.model.decoder), 13))
    seen = []
    real = tr.fun_generate_samples_vada

    def spy(*a, **k):
        seen.append(k.get("enable_autocast"))
        return real(*a, **k)

    tr.fun_generate_samples_vada = spy
    torch.manual_seed(5)
    traj = tr.sample(num_shapes=2)
    assert seen == [True]
    torch.manual_seed(5)
    img, *_ = generate_samples_vada_2prior(tr.model.latent_shape(), tr.dae, tr.diffusion_disc, tr.model, 2, True)
    assert torch.equal(traj, img.permute(0, 2, 1).contiguous())
    assert np.isfinite(traj.cpu().numpy()).all()
