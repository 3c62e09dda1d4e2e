"""Continuous-time VPSDE and the probability-flow ODE sampler -- host-side mirror of the reference's
utils/diffusion_continuous.py (`make_diffusion` :21-36, `DiffusionBase` :39-88, `sample_model_ode` :178-249,
`DiffusionVPSDE` :571-621), the route `generate_samples_vada_2prior(ode_sample=1)` takes
(trainers/train_2prior.py:64-80).  SURVEY.md 8f rank 4.

The ODE dx/dt = f(t) x + 0.5 g^2(t) eps_theta(x, t) / sqrt(var(t)) is integrated from t = init_t (1.0) down to the
cutoff ode_eps with scipy's adaptive RK45 ON THE HOST, exactly as the reference does through its vendored torchdiffeq
`scipy_solver` wrapper (third_party/torchdiffeq/torchdiffeq/_impl/scipy_wrapper.py: state as a float64 numpy vector,
time reversed by negation, one model call per right-hand-side evaluation with t as a 0-dim tensor).  The model call is
the same C-ABI network forward the DDPM loop uses; the step count (NFE) is adaptive, so nothing is graph-captured.

The encoding direction, `compute_ode_nll` (reference :90-176: data latents at t = ode_eps to noise at t = 1, used by
trainers/encode_interp_interp.py), runs the same scipy algorithm ON THE DEVICE instead (`ode_solve_device`, kernels in
lion_b200/csrc/ode.cu): the float64 state, the stages and the step-size controller never leave the GPU, and one step
attempt (six network forwards and the integrator kernels) is captured once as a CUDA graph and replayed; the host reads
a few bytes of integrator status per attempt.
Only `sde_type == 'vpsde'` is provided (every shipped config, default_config.py:121)."""
import ctypes
import gc
import os
from timeit import default_timer as timer

import numpy as np
import torch
from loguru import logger

from .. import _lib as L


def make_diffusion(args):
    if args.sde_type == 'vpsde':
        return DiffusionVPSDE(args)
    raise ValueError("lion_b200: only sde_type 'vpsde' is provided (got %r)" % (args.sde_type,))


class DiffusionBase(object):
    def __init__(self, args):
        self.sigma2_0 = args.sigma2_0
        self.sde_type = args.sde_type
        self.use_cuda_graph = os.environ.get('LION_NO_GRAPH', '0') != '1'   # eager step attempts for profilers

    def sample_q(self, x_init, noise, var_t, m_t):
        return m_t * x_init + torch.sqrt(var_t) * noise

    @torch.no_grad()
    def compute_ode_nll(self, dae, eps, ode_eps, ode_solver_tol, enable_autocast=False, no_autograd=False, num_samples=1,
                        report_std=False, condition_input=None, clip_feat=None):
        """Carry `eps` from t = ode_eps to t = 1 along the probability-flow ODE; returns x at t = 1 shaped like eps (the
        reference's return value; its log-likelihood terms are commented out there as well).

        The span is the reference's torch.tensor([ode_eps, 1.0]) in fp32, integrated forward in time by scipy's RK45
        algorithm restated on the device (`ode_solve_device`) with rtol = atol = ode_solver_tol.  The reference repeats
        the identical deterministic integration `num_samples` times and keeps the last; it is integrated once here.
        no_autograd and report_std do not change the result there either.  enable_autocast runs the network as the
        other routes do under autocast (FP16 operands in the second convolution of every PVConv, fp32 outputs)."""
        assert not getattr(dae, 'mixed_prediction', False), "lion_b200: mixed_prediction is off in every shipped prior config"
        gc.collect()
        dae.eval()
        t0 = float(np.float32(ode_eps))
        x, stats = self.ode_solve_device(dae, eps, t0, 1.0, ode_solver_tol, enable_autocast=enable_autocast,
                                         condition_input=condition_input, clip_feat=clip_feat)
        logger.info('nfe_counter: {}', stats['nfe'])
        return x

    @torch.no_grad()
    def ode_solve_device(self, dae, y0, t0, t_bound, tol, enable_autocast=False, condition_input=None, clip_feat=None,
                         negate=False):
        """Integrate dy/ds = +-(f(t) y + 0.5 g2(t) dae(y, t) / sqrt(var(t))) from s = t0 to s = t_bound with scipy's RK45
        (rtol = atol = tol), all on the device.  t = s, or t = -s with the right-hand side negated when `negate`
        (torchdiffeq's treatment of a decreasing span, as sample_model_ode's host route integrates).  Returns (the
        dense-output value at t_bound shaped like y0, {nfe, n_accepted, n_rejected, t}).

        The first step attempt runs eagerly (it builds the networks and sizes their scratch arena); the next is captured
        with capture_graph and every later attempt replays it.  The integrator's state is read by the host once per
        attempt.  Raises RuntimeError when the step size falls below scipy's minimum."""
        dev = y0.device if y0.is_cuda else torch.device('cuda', torch.cuda.current_device())
        y0 = y0.detach().to(dev, torch.float32).contiguous()
        shape, n, B = y0.shape, y0.numel(), y0.shape[0]
        rtol = max(float(tol), 100 * np.finfo(float).eps)          # scipy's validate_tol
        if t0 == t_bound:
            return y0.clone(), {'nfe': 0, 'n_accepted': 0, 'n_rejected': 0, 't': t_bound}
        lib = L.lib()
        f64 = dict(device=dev, dtype=torch.float64)
        y, y_new, K = torch.empty(n, **f64), torch.empty(n, **f64), torch.empty(7, n, **f64)
        partials = torch.zeros(L.ODE_PARTIALS, **f64)
        x = torch.empty(shape, device=dev, dtype=torch.float32)
        tm = torch.empty(B, device=dev, dtype=torch.float32)
        out = torch.empty(shape, device=dev, dtype=torch.float32)
        nbytes = lib.lion_ode_state_bytes()
        assert nbytes == ctypes.sizeof(L.OdeState), "lion_b200: LionOdeState layout differs from the library's"
        st = torch.zeros(nbytes, device=dev, dtype=torch.uint8)
        st_host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        P = L.ptr
        sde = (float(self.beta_start), float(self.beta_end), float(self.sigma2_0))

        def evaluate(stage):
            L.check(lib.lion_ode_stage(P(st), P(y), P(y_new), P(K), n, stage, P(x), P(tm), B, L.stream()), "ode_stage")
            with torch.autocast("cuda", dtype=torch.float16, enabled=bool(enable_autocast)):
                eps = dae(x=x, t=tm, condition_input=condition_input, clip_feat=clip_feat)
            eps = eps.to(torch.float32).contiguous()
            L.check(lib.lion_ode_rhs(P(st), P(x), P(eps), P(K), n, stage, *sde, P(tm), L.stream()), "ode_rhs")

        def control(what):
            L.check(lib.lion_ode_norms(P(st), P(y), P(y_new), P(K), n, what, P(partials), L.stream()), "ode_norms")
            L.check(lib.lion_ode_control(P(st), P(partials), n, what, L.stream()), "ode_control")

        def attempt():
            L.check(lib.lion_ode_control(P(st), P(partials), n, L.ODE_BEGIN, L.stream()), "ode_control")
            for stage in range(1, 7):
                evaluate(stage)
            control(L.ODE_END)
            L.check(lib.lion_ode_commit(P(st), P(y), P(y_new), P(K), n, L.stream()), "ode_commit")

        def status():
            st_host.copy_(st, non_blocking=True)
            torch.cuda.current_stream().synchronize()
            return L.OdeState.from_buffer_copy(st_host.numpy().tobytes())

        with torch.cuda.device(dev):
            L.check(lib.lion_ode_init(P(st), P(y0), P(y), n, float(t0), float(t_bound), rtol, float(tol), int(bool(negate)),
                                      L.stream()), "ode_init")
            evaluate(0)                                             # f0 = fun(t0, y0)
            control(L.ODE_INIT_H0)
            evaluate(L.ODE_STAGE_PROBE)                             # f1 of select_initial_step
            control(L.ODE_INIT_H1)
            attempt()
            s = status()
            graph = None
            if s.status == L.ODE_RUNNING and self.use_cuda_graph and getattr(dae, 'lion_graph_safe', True):
                with L.capture_graph() as graph:
                    attempt()
            while s.status == L.ODE_RUNNING:
                if graph is not None:
                    graph.replay()
                else:
                    attempt()
                s = status()
            if s.status == L.ODE_TOO_SMALL:
                raise RuntimeError("lion_b200: RK45 step size fell below the minimum at t = %r (nfe = %d, %d steps accepted)"
                                   % (-s.t if negate else s.t, s.nfe, s.n_accepted))
            L.check(lib.lion_ode_dense_end(P(st), P(y), P(K), n, P(out), L.stream()), "ode_dense_end")
        return out, {'nfe': s.nfe, 'n_accepted': s.n_accepted, 'n_rejected': s.n_rejected, 't': s.t}

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
