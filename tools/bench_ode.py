"""The probability-flow ODE's encoding direction on the device against the host route's mechanics.

    python tools/bench_ode.py [--batches 4 32] [--rounds 3] > ode.jsonl

For both priors (synthetic key-seeded weights, the sde.embedding_scale 1000 configuration of script/interpolate*.sh) and
batches of 4 and 32 latents, the same span is integrated two ways, alternated over `--rounds` rounds:
  device  DiffusionBase.compute_ode_nll: scipy's RK45 restated in lion_b200/csrc/ode.cu, one step attempt captured as a
          CUDA graph and replayed, a few bytes of status read per attempt;
  host    scipy.integrate.solve_ivp(RK45, t_eval=[ode_eps, 1]) around the same GPU forward, as the reference's torchdiffeq
          wrapper and sample_model_ode's host route drive it: per evaluation the state goes to the GPU, the network runs
          eagerly, the derivative comes back, the host synchronises.
Wall time is a host clock around each whole integration (which ends in a device synchronise); NFE and ms per NFE are
printed for both, with the speed-up, the largest deviation between the two results relative to max|x|, and whether the
two agree on NFE.  Spans are short (global prior t = 0.85 -> 1, point prior t = 0.9 -> 1) because with random weights
the full span is a diverging ODE; the tolerance is the scripts' 1e-5.  The card's name and power limit are read in the
same call and printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def host_route(d, dae, y0, t0, t1, tol, condition_input):
    """solve_ivp around the GPU forward; -> (x at t1, nfe)"""
    from scipy.integrate import solve_ivp
    shape = y0.shape
    nfe = [0]

    def fun(s, y):
        nfe[0] += 1
        t = torch.tensor(s).to("cuda", torch.float32)
        x = torch.reshape(torch.tensor(y).to("cuda", torch.float32), shape)
        eps = dae(x=x, t=t, condition_input=condition_input)
        return (d.f(t=t) * x + 0.5 * d.g2(t=t) * eps / torch.sqrt(d.var(t=t))).detach().cpu().numpy().reshape(-1)

    t_eval = np.array([t0, t1], dtype=np.float32)
    sol = solve_ivp(fun, t_span=[t_eval.min(), t_eval.max()], y0=y0.cpu().numpy().reshape(-1), t_eval=t_eval,
                    method="RK45", rtol=tol, atol=tol)
    return torch.tensor(sol.y).T.to("cuda", torch.float32).reshape(-1, *shape)[-1], nfe[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[4, 32])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--tol", type=float, default=1e-5)
    a = ap.parse_args()
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.latent_points_ada_localprior import PVCNN2Prior
    from lion_b200.models.score_sde.resnet import PriorSEDrop
    from lion_b200.utils.diffusion_continuous import make_diffusion
    from tests.synth import synth_state_dict
    keys = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "keys.json")))
    torch.cuda.set_device(0)
    cfg = default_prior_cfg()
    cfg.sde.merge_from_list(["beta_end", 20.0, "embedding_scale", 1000.0])
    gp = PriorSEDrop(cfg.sde, 128, cfg)
    gp.load_state_dict(synth_state_dict(keys["global"], 14))
    lp = PVCNN2Prior(cfg.sde, 1, cfg)
    lp.load_state_dict(synth_state_dict(keys["prior"], 11))
    gp, lp = gp.cuda().eval(), lp.cuda().eval()
    d = make_diffusion(cfg.sde)
    print(json.dumps({"card": card()}), flush=True)
    for name, dae, dim, ode_eps in (("global", gp, 128, 0.85), ("point", lp, 8192, 0.9)):
        for B in a.batches:
            g = torch.Generator().manual_seed(7)
            x0 = torch.randn(B, dim, 1, 1, generator=g).cuda()
            cond = torch.randn(B, 128, 1, 1, generator=g).cuda() if name == "point" else None
            t0 = float(np.float32(ode_eps))
            d.ode_solve_device(dae, x0, t0, 1.0, a.tol, condition_input=cond)       # warm-up: builds, packs, sizes the arena
            dev_s, host_s = [], []
            for _ in range(a.rounds):
                torch.cuda.synchronize()
                s = time.perf_counter()
                xd, st = d.ode_solve_device(dae, x0, t0, 1.0, a.tol, condition_input=cond)
                torch.cuda.synchronize()
                dev_s.append(time.perf_counter() - s)
                s = time.perf_counter()
                xh, nfe_h = host_route(d, dae, x0, ode_eps, 1.0, a.tol, cond)
                torch.cuda.synchronize()
                host_s.append(time.perf_counter() - s)
            dev, host = min(dev_s), min(host_s)
            rec = {"prior": name, "B": B, "span": [t0, 1.0], "tol": a.tol,
                   "device": {"s": round(dev, 4), "nfe": st["nfe"], "ms_per_nfe": round(1e3 * dev / st["nfe"], 3),
                              "accepted": st["n_accepted"], "rejected": st["n_rejected"], "all_s": [round(v, 4) for v in dev_s]},
                   "host": {"s": round(host, 4), "nfe": nfe_h, "ms_per_nfe": round(1e3 * host / nfe_h, 3),
                            "all_s": [round(v, 4) for v in host_s]},
                   "speedup": round(host / dev, 3), "same_nfe": st["nfe"] == nfe_h,
                   "max_dev_rel": float((xd - xh).abs().max() / xh.abs().max())}
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
