"""Continuous-time VPSDE and the probability-flow ODE sampler -- host-side mirror of the reference's
utils/diffusion_continuous.py (`make_diffusion` :21-36, `DiffusionBase` :39-88, `sample_model_ode` :178-249,
`DiffusionVPSDE` :571-621), the route `generate_samples_vada_2prior(ode_sample=1)` takes
(trainers/train_2prior.py:64-80).  SURVEY.md 8f rank 4.

The ODE dx/dt = f(t) x + 0.5 g^2(t) eps_theta(x, t) / sqrt(var(t)) is integrated from t = init_t (1.0) down to the
cutoff ode_eps with scipy's adaptive RK45 ON THE HOST, exactly as the reference does through its vendored torchdiffeq
`scipy_solver` wrapper (third_party/torchdiffeq/torchdiffeq/_impl/scipy_wrapper.py: state as a float64 numpy vector,
time reversed by negation, one model call per right-hand-side evaluation with t as a 0-dim tensor).  The model call is
the same C-ABI network forward the DDPM loop uses; the step count (NFE) is adaptive, so nothing is graph-captured.
Only `sde_type == 'vpsde'` is provided (every shipped config, default_config.py:121)."""
import gc
from timeit import default_timer as timer

import numpy as np
import torch
from loguru import logger


def make_diffusion(args):
    if args.sde_type == 'vpsde':
        return DiffusionVPSDE(args)
    raise ValueError("lion_b200: only sde_type 'vpsde' is provided (got %r)" % (args.sde_type,))


class DiffusionBase(object):
    def __init__(self, args):
        self.sigma2_0 = args.sigma2_0
        self.sde_type = args.sde_type

    def sample_q(self, x_init, noise, var_t, m_t):
        return m_t * x_init + torch.sqrt(var_t) * noise

    @torch.no_grad()
    def sample_model_ode(self, dae, num_samples, shape, ode_eps, ode_solver_tol, enable_autocast, temp, noise=None,
                         condition_input=None, mixing_logit=None, use_cust_ode_func=0, init_t=1.0, return_all_sample=False,
                         clip_feat=None):
        """-> (samples [num_samples, *shape], nfe, seconds)  [+ all evaluated time points when return_all_sample]"""
        assert not use_cust_ode_func, "lion_b200: standard ODE function only"
        assert not getattr(dae, 'mixed_prediction', False), "lion_b200: mixed_prediction is off in every shipped prior config"
        gc.collect()
        dae.eval()
        device = torch.device('cuda', torch.cuda.current_device())
        if noise is None:
            noise = torch.randn(size=[num_samples] + list(shape), device=device)
        y0 = (temp * noise).to(torch.float32)
        yshape = y0.shape
        nfe = [0]

        def ode_func(t, x):
            """dx/dt at time t (0-dim tensor), reference :212-229"""
            nfe[0] += 1
            if nfe[0] % 100 == 0:
                logger.info('nfe_counter={}', nfe[0])
            with torch.autocast("cuda", dtype=torch.float16, enabled=bool(enable_autocast)):
                variance = self.var(t=t)
                params = dae(x=x, t=t, condition_input=condition_input, clip_feat=clip_feat)
                return self.f(t=t) * x + 0.5 * self.g2(t=t) * params / torch.sqrt(variance)

        # torchdiffeq's odeint integrates decreasing time spans by negating time: s = -t, dy/ds = -f(-s, y)
        def np_func(s, y):
            t = (-torch.tensor(s)).to(device, torch.float32)
            x = torch.reshape(torch.tensor(y).to(device, torch.float32), yshape)
            return (-ode_func(t, x)).detach().cpu().numpy().reshape(-1)

        from scipy.integrate import solve_ivp
        t_eval = np.array([-init_t, -ode_eps], dtype=np.float32)          # torch.tensor([init_t, ode_eps]) is fp32
        start = timer()
        sol = solve_ivp(np_func, t_span=[t_eval.min(), t_eval.max()], y0=y0.detach().cpu().numpy().reshape(-1), t_eval=t_eval,
                        method='RK45', rtol=ode_solver_tol, atol=ode_solver_tol)
        samples_out = torch.tensor(sol.y).T.to(device, torch.float32).reshape(-1, *yshape)
        ode_solve_time = timer() - start
        if return_all_sample:
            return samples_out[-1], samples_out, nfe[0], ode_solve_time
        return samples_out[-1], nfe[0], ode_solve_time


class DiffusionVPSDE(DiffusionBase):
    """VPSDE with linear beta(t) on t in [0, 1] (reference :571-621; beta_start / beta_end are the DDPM values x 1000)."""

    def __init__(self, args):
        super().__init__(args)
        self.beta_start = args.beta_start
        self.beta_end = args.beta_end
        self.time_eps = args.time_eps

    def f(self, t):
        return -0.5 * self.g2(t)

    def g2(self, t):
        return self.beta_start + (self.beta_end - self.beta_start) * t

    def var(self, t):
        return 1.0 - (1.0 - self.sigma2_0) * torch.exp(-self.beta_start * t - 0.5 * (self.beta_end - self.beta_start) * t * t)

    def e2int_f(self, t):
        return torch.exp(-0.5 * self.beta_start * t - 0.25 * (self.beta_end - self.beta_start) * t * t)

    def inv_var(self, var):
        c = torch.log((1 - var) / (1 - self.sigma2_0))
        a = self.beta_end - self.beta_start
        return (-self.beta_start + torch.sqrt(np.square(self.beta_start) - 2 * a * c)) / a

    def mixing_component(self, x_noisy, var_t, t, enabled):
        return torch.sqrt(var_t) * x_noisy if enabled else None
