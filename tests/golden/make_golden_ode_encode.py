"""Generate tests/golden/ode_encode.npz from the UNMODIFIED reference (container only):

    python tests/golden/make_golden_ode_encode.py

With the configuration script/interpolate.sh and script/interpolate_posterior.sh run under (sde.beta_end 20.0,
sde.embedding_scale 1000.0) and key-seeded synthetic weights, on CPU:
  * `DiffusionBase.compute_ode_nll` (utils/diffusion_continuous.py:90-176, scipy RK45 through the reference's vendored
    torchdiffeq wrapper, data latents at t = ode_eps to noise at t = 1) of the global prior (PriorSEDrop, 2 latents,
    ode_eps 0.85, tolerance 1e-3) and of the latent-point prior (PVCNN2Prior, 1 latent, ode_eps 0.99, tolerance 1e-2).
    Short spans: with random weights the full span is a diverging ODE (see make_golden_ode.py), and near t = 1
    (beta_end 20) the point prior's ODE amplifies errors of the network output: in this reference run, noise of 2e-3
    of max|eps| added to every evaluation moves x(1) by 0.46 of max|x(1)| over [0.9, 1], 0.20 over [0.97, 1] and 0.04
    over [0.99, 1].  A TF32 network differs from this fp32 run by that much, so only the shortest span is a pin.
    Stored: inputs, x at t = 1 and the number of network evaluations;
  * `interpolate_noise`, `linear_interpolate_noise` and `subtract_noise` (trainers/interpolate_latent.py:23-57) of one
    seeded [20, 16, 1, 1] noise block each;
  * a PVCNN2Prior forward at embedding_scale 1000 (B = 2, t in [0, 1])."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.golden import ref_import as R  # noqa: E402

R.install()
import numpy as np  # noqa: E402
import torch  # noqa: E402

from tests.golden.make_golden import load_synth, gen  # noqa: E402

torch.set_num_threads(8)


def noise_edits():
    """The three noise edits, imported from the reference trainer (its rendering imports are stubbed)."""
    for n in ["torchvision", "torchvision.utils", "utils.vis_helper"]:
        if n not in sys.modules:
            R._stub(n)
    import trainers.interpolate_latent as IL
    return IL.interpolate_noise, IL.linear_interpolate_noise, IL.subtract_noise


def main():
    cfg = R.load_cfg(overrides=["sde.beta_end", 20.0, "sde.embedding_scale", 1000.0])
    from models.latent_points_ada_localprior import PVCNN2Prior
    from models.score_sde.resnet import PriorSEDrop
    import utils.diffusion_continuous as DC
    diff = DC.make_diffusion(cfg.sde)
    out = {}
    with torch.no_grad():
        gp = PriorSEDrop(cfg.sde, cfg.latent_pts.style_dim, cfg)
        load_synth(gp, 14)
        eps = gen(601, 2, 128, 1, 1)
        z = diff.compute_ode_nll(gp, eps, 0.85, 1e-3)
        out.update(g_eps=eps.numpy(), g_out=z.numpy(), g_nfe=np.int32(DC.nfe_counter), g_tol=np.float32(1e-3),
                   g_ode_eps=np.float32(0.85))
        print("global: nfe", DC.nfe_counter, float(z.abs().mean()))
        lp = PVCNN2Prior(cfg.sde, 1, cfg)
        load_synth(lp, 11)
        eps_l = gen(602, 1, 8192, 1, 1)
        style = gen(603, 1, 128, 1, 1)
        zl = diff.compute_ode_nll(lp, eps_l, 0.99, 1e-2, condition_input=style)
        out.update(l_eps=eps_l.numpy(), l_style=style.numpy(), l_out=zl.numpy(), l_nfe=np.int32(DC.nfe_counter),
                   l_tol=np.float32(1e-2), l_ode_eps=np.float32(0.99))
        print("local: nfe", DC.nfe_counter, float(zl.abs().mean()))

        x = gen(605, 2, 8192, 1, 1)
        t = torch.tensor([0.981, 0.012])
        style2 = gen(606, 2, 128, 1, 1)
        e = lp(x=x, t=t, condition_input=style2, clip_feat=None)
        out.update(s_x=x.numpy(), s_t=t.numpy(), s_style=style2.numpy(), s_eps=e.numpy())
        print("prior forward at embedding_scale 1000:", float(e.abs().mean()))

    interp, linear, subtract = noise_edits()
    noise = gen(604, 20, 16, 1, 1)
    out.update(n_in=noise.numpy(), n_interpolate=interp(noise.clone()).numpy(), n_linear=linear(noise.clone()).numpy(),
               n_subtract=subtract(noise.clone()).numpy())
    np.savez_compressed(os.path.join(HERE, "ode_encode.npz"), **out)


if __name__ == "__main__":
    main()
