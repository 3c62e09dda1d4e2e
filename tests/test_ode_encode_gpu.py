"""The probability-flow ODE's encoding direction and the interpolation routes on the GPU:
  * the device-resident RK45 (lion_b200/csrc/ode.cu) against scipy's solve_ivp driving the same GPU forward -- same nfe,
    accepted / rejected steps and final t, states within 1e-6 of max|y| -- in both directions, for both priors;
  * compute_ode_nll against tests/golden/ode_encode.npz (the unmodified reference on CPU, make_golden_ode_encode.py);
  * encode-then-sample round trip, the autocast route, graph replay vs the all-eager driver;
  * sde.embedding_scale in the point prior's U-Net;
  * interpolate_latent.generate_samples / Trainer.vis_sample and encode_interp_interp.Trainer.eval_nll end to end.
Spans are short: with random weights the full span is a diverging ODE (see tests/test_ode_gpu.py)."""
import json
import os

import numpy as np
import pytest
import torch

from tests.synth import synth_state_dict
from tests.util import assert_close

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
KEYS = json.load(open(os.path.join(G, "keys.json")))
EKEYS = json.load(open(os.path.join(G, "keys_encoder.json")))


def _cfg():
    from lion_b200.config import default_prior_cfg
    cfg = default_prior_cfg()
    cfg.sde.merge_from_list(["ode_sample", 1, "beta_end", 20.0, "embedding_scale", 1000.0])   # script/interpolate*.sh
    return cfg


def _priors(cfg):
    from lion_b200.models.latent_points_ada_localprior import PVCNN2Prior
    from lion_b200.models.score_sde.resnet import PriorSEDrop
    gp = PriorSEDrop(cfg.sde, 128, cfg)
    gp.load_state_dict(synth_state_dict(KEYS["global"], 14))
    lp = PVCNN2Prior(cfg.sde, 1, cfg)
    lp.load_state_dict(synth_state_dict(KEYS["prior"], 11))
    return gp.cuda().eval(), lp.cuda().eval()


def _diffusion(cfg):
    from lion_b200.utils.diffusion_continuous import make_diffusion
    return make_diffusion(cfg.sde)


def _host_solve(d, dae, y0, t0, t_bound, tol, negate, condition_input=None):
    """scipy's solve_ivp around the same GPU forward, as the reference's torchdiffeq wrapper drives it"""
    from scipy.integrate import solve_ivp
    shape = y0.shape

    def fun(s, y):
        t = torch.tensor(-s if negate else s).to("cuda", torch.float32)
        x = torch.tensor(y).to("cuda", torch.float32).reshape(shape)
        eps = dae(x=x, t=t, condition_input=condition_input)
        dx = d.f(t=t) * x + 0.5 * d.g2(t=t) * eps / torch.sqrt(d.var(t=t))
        return (-dx if negate else dx).cpu().numpy().reshape(-1)

    t_eval = np.array([t0, t_bound])
    sol = solve_ivp(fun, t_span=[t0, t_bound], y0=y0.cpu().numpy().reshape(-1).astype(np.float64), t_eval=t_eval,
                    method="RK45", rtol=tol, atol=tol, dense_output=True)
    assert sol.status == 0, sol.message
    accepted = len(sol.sol.ts) - 1
    rejected = (sol.nfev - 2 - 6 * accepted) // 6
    return sol.y[:, -1], {"nfe": sol.nfev, "n_accepted": accepted, "n_rejected": rejected, "t": float(sol.t[-1])}


@pytest.mark.parametrize("prior,negate", [("global", False), ("global", True), ("point", False), ("point", True)])
def test_device_integrator_is_scipys_rk45(prior, negate):
    cfg = _cfg()
    gp, lp = _priors(cfg)
    d = _diffusion(cfg)
    g = torch.Generator().manual_seed(41)
    if prior == "global":
        dae, y0, cond, tol = gp, torch.randn(2, 128, 1, 1, generator=g), None, 1e-3
    else:
        dae, y0, tol = lp, torch.randn(1, 8192, 1, 1, generator=g), 1e-2
        cond = torch.randn(1, 128, 1, 1, generator=g).cuda()
    # encoding: t = 0.85 -> 1 forward in time; sampling: t = 0.15 -> 0.05 as s = -t increasing with the RHS negated
    t0, t1 = (-0.15, -0.05) if negate else (0.85, 1.0)
    y0 = y0.cuda()
    out, st = d.ode_solve_device(dae, y0, t0, t1, tol, condition_input=cond, negate=negate)
    ref, st_ref = _host_solve(d, dae, y0, t0, t1, tol, negate, condition_input=cond)
    assert st == st_ref, (st, st_ref)
    ref = torch.from_numpy(ref)
    err = (out.double().cpu().reshape(-1) - ref).abs().max().item()
    assert err <= 1e-6 * ref.abs().max().item(), (err, ref.abs().max().item())


def test_compute_ode_nll_global_prior_golden():
    z = np.load(os.path.join(G, "ode_encode.npz"))
    cfg = _cfg()
    gp, _ = _priors(cfg)
    d = _diffusion(cfg)
    out, st = d.ode_solve_device(gp, torch.from_numpy(z["g_eps"]).cuda(), float(np.float32(z["g_ode_eps"])), 1.0, float(z["g_tol"]))
    assert abs(st["nfe"] - int(z["g_nfe"])) <= max(12, int(z["g_nfe"]) // 4), (st["nfe"], int(z["g_nfe"]))
    x = d.compute_ode_nll(gp, torch.from_numpy(z["g_eps"]).cuda(), float(z["g_ode_eps"]), float(z["g_tol"]))
    assert torch.equal(x, out)
    assert_close(x, torch.from_numpy(z["g_out"]), 2e-2, "compute_ode_nll of the global prior vs the reference's solver")


def test_compute_ode_nll_point_prior_golden():
    z = np.load(os.path.join(G, "ode_encode.npz"))
    cfg = _cfg()
    _, lp = _priors(cfg)
    d = _diffusion(cfg)
    style = torch.from_numpy(z["l_style"]).cuda()
    out, st = d.ode_solve_device(lp, torch.from_numpy(z["l_eps"]).cuda(), float(np.float32(z["l_ode_eps"])), 1.0,
                                 float(z["l_tol"]), condition_input=style)
    assert abs(st["nfe"] - int(z["l_nfe"])) <= max(12, int(z["l_nfe"]) // 2), (st["nfe"], int(z["l_nfe"]))
    # a TF32 network against an fp32 CPU run, amplified by the ODE near t = 1 (make_golden_ode_encode.py): ~10x the tolerance
    assert_close(out, torch.from_numpy(z["l_out"]), 1e-1, "compute_ode_nll of the latent-point prior vs the reference's solver")


def test_encode_then_sample_recovers_the_input():
    """compute_ode_nll over [a, 1], then sample_model_ode from 1 back to a.  The network's TF32 rounding makes the vector
    field non-smooth at the 1e-4 level, so the round trip cannot reach the solver tolerance itself; it must recover the
    input as well as scipy's own encoding does (host solve_ivp around the same forward, then the same sampler)."""
    cfg = _cfg()
    gp, _ = _priors(cfg)
    d = _diffusion(cfg)
    a, tol = 0.85, 1e-5
    x0 = torch.randn(2, 128, 1, 1, generator=torch.Generator().manual_seed(43)).cuda()
    xT = d.compute_ode_nll(gp, x0, a, tol)
    back, _, _ = d.sample_model_ode(gp, 2, [128, 1, 1], a, tol, False, 1.0, noise=xT.clone(), init_t=1.0)
    err = ((back - x0).abs().max() / x0.abs().max()).item()
    xT_host, _ = _host_solve(d, gp, x0, float(np.float32(a)), 1.0, tol, False)
    back_host, _, _ = d.sample_model_ode(gp, 2, [128, 1, 1], a, tol, False, 1.0,
                                         noise=torch.from_numpy(xT_host).float().cuda().view_as(x0), init_t=1.0)
    err_host = ((back_host - x0).abs().max() / x0.abs().max()).item()
    assert err < 2e-2 and err <= 1.5 * err_host + 1e-4, (err, err_host)


def test_compute_ode_nll_autocast_runs_finite():
    cfg = _cfg()
    _, lp = _priors(cfg)
    d = _diffusion(cfg)
    g = torch.Generator().manual_seed(44)
    x0, style = torch.randn(2, 8192, 1, 1, generator=g).cuda(), torch.randn(2, 128, 1, 1, generator=g).cuda()
    x = d.compute_ode_nll(lp, x0, 0.9, 1e-2, enable_autocast=True, condition_input=style)
    assert x.shape == x0.shape and x.dtype == torch.float32 and torch.isfinite(x).all()


@pytest.mark.parametrize("prior", ["global", "point"])
def test_graph_replay_equals_the_eager_driver(prior):
    cfg = _cfg()
    gp, lp = _priors(cfg)
    d = _diffusion(cfg)
    g = torch.Generator().manual_seed(45)
    if prior == "global":
        dae, x0, cond, a, tol = gp, torch.randn(4, 128, 1, 1, generator=g).cuda(), None, 0.85, 1e-3
    else:
        dae, x0, a, tol = lp, torch.randn(2, 8192, 1, 1, generator=g).cuda(), 0.9, 1e-2
        cond = torch.randn(2, 128, 1, 1, generator=g).cuda()
    replayed, st = d.ode_solve_device(dae, x0, a, 1.0, tol, condition_input=cond)
    assert st["n_accepted"] >= 2, st          # more than the eager first attempt
    d.use_cuda_graph = False
    eager, st_eager = d.ode_solve_device(dae, x0, a, 1.0, tol, condition_input=cond)
    assert st == st_eager and torch.equal(replayed, eager)


def test_point_prior_embedding_scale():
    """At embedding_scale 1000 the U-Net matches the reference (prior_fwd tolerances); the scale enters as fl(t * scale),
    so the network at scale 1000 fed t equals, bit for bit, the network at scale 1 fed fl(t * 1000)."""
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.latent_points_ada_localprior import PVCNN2Prior
    from tests.util import rms_err
    z = np.load(os.path.join(G, "ode_encode.npz"))
    _, lp = _priors(_cfg())
    x, t, style = (torch.from_numpy(z[k]).cuda() for k in ("s_x", "s_t", "s_style"))
    eps = lp(x=x, t=t, condition_input=style)
    assert rms_err(eps, z["s_eps"]) < 4e-3
    assert_close(eps, torch.from_numpy(z["s_eps"]), 5e-3, "PVCNN2Prior at embedding_scale 1000 vs the reference")
    cfg1 = default_prior_cfg()
    lp1 = PVCNN2Prior(cfg1.sde, 1, cfg1)
    lp1.load_state_dict(synth_state_dict(KEYS["prior"], 11))
    lp1 = lp1.cuda().eval()
    eps1 = lp1(x=x, t=t * 1000.0, condition_input=style)
    assert torch.equal(eps, eps1)


def _vae(cfg):
    from lion_b200.models.vae_adain import Model
    vae = Model(cfg)
    sd = {}
    for pre, shapes, seed in (("style_encoder.", EKEYS["style_encoder"], 21), ("encoder.", EKEYS["point_encoder"], 22),
                              ("decoder.", KEYS["decoder"], 13)):
        sd.update({pre + k: v for k, v in synth_state_dict(shapes, seed).items()})
    vae.load_state_dict(sd)
    return vae


def _trainer(module, cfg, tmp_path):
    cfg.save_dir = str(tmp_path)
    tr = module.Trainer(cfg)
    tr.model.load_state_dict(_vae(cfg).state_dict())
    tr.dae[0].load_state_dict(synth_state_dict(KEYS["global"], 14))
    tr.dae[1].load_state_dict(synth_state_dict(KEYS["prior"], 11))
    return tr


@pytest.mark.parametrize("modes", [("interpolate", "freeze"), ("linear_interpolate", "interpolate"),
                                   ("subtract", "subtract"), ("freeze", "linear_interpolate")])
def test_generate_samples_modes(modes):
    from lion_b200.trainers.interpolate_latent import generate_samples
    from lion_b200.utils.diffusion_continuous import DiffusionVPSDE
    cfg = _cfg()
    gp, lp = _priors(cfg)
    vae = _vae(cfg).cuda().eval()
    noises = []

    class Recording(DiffusionVPSDE):
        def sample_model_ode(self, *a, **k):
            noises.append(a[7].clone())
            return super().sample_model_ode(*a, **k)

    torch.manual_seed(5)
    B = 16                                      # subtract_noise reads shapes 9 .. 15
    img, nfe, t_ode, t_all, out = generate_samples(vae.latent_shape(), torch.nn.ModuleList([gp, lp]), Recording(cfg.sde), vae, B,
                                                   False, ode_eps=0.9, ode_solver_tol=1e-2, ode_sample=1,
                                                   generate_mode_global=modes[0], generate_mode_local=modes[1])
    assert img.shape == (B, 2048, 3) and torch.isfinite(img).all() and torch.equal(out["gen_x"], img) and float(nfe) > 0
    assert out["sampled_eps"].shape == (B, 8192, 1, 1)
    for noise, mode in zip(noises, modes):
        if mode == "freeze":
            assert torch.equal(noise, noise[:1].expand_as(noise))
        elif mode == "interpolate":
            p = 1.0 / B
            assert torch.allclose(noise[1], np.sqrt(p) * noise[-1] + np.sqrt(1 - p) * noise[0])
        elif mode == "subtract":
            assert not torch.equal(noise[0], noise[1])


def test_interpolate_latent_vis_sample_writes_the_reference_layout(tmp_path):
    from lion_b200.trainers import interpolate_latent
    cfg = _cfg()
    cfg.sde.ode_eps = 0.9
    tr = _trainer(interpolate_latent, cfg, tmp_path)
    tr.num_interp, tr.num_val_samples = 2, 3
    tr.vis_sample(None)
    for idx in range(2):
        d = tmp_path / "interp" / "mode_interpolate_interpolate_2048" / ("%04d" % idx)
        files = sorted(os.listdir(d))
        assert files == ["%04d.pt" % i for i in range(3)], files
        x = torch.load(d / "0000.pt")
        assert x.shape == (2048, 3) and torch.isfinite(x).all()


def test_encode_interp_interp_eval_nll(tmp_path):
    from lion_b200.trainers import encode_interp_interp
    cfg = _cfg()
    cfg.sde.ode_eps = 0.9
    tr = _trainer(encode_interp_interp, cfg, tmp_path)
    g = torch.Generator().manual_seed(46)
    batch = {"tr_points": 0.3 * torch.randn(3, 2048, 3, generator=g)}
    assert tr.eval_nll(0, data_loader=[batch]) == 0
    d = tmp_path / "enc60_interpolate_interpolate" / "sph_B4_0000"
    assert sorted(os.listdir(d)) == ["%04d" % i for i in range(4)]
    clouds = [torch.load(d / ("%04d" % i)) for i in range(4)]
    assert all(c.shape == (2048, 3) and torch.isfinite(c).all() for c in clouds)
