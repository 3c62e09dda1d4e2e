"""Discrete DDPM / DDIM samplers -- mirror of the reference's utils/diffusion_pvd.py
(DiffusionDiscretized :17-563; only the sampling methods and their constants).

`run_denoising_diffusion` keeps the reference's signature and return values.  With one of this
package's networks as `model`, one denoising step = [network forward, noise draw, fused
update kernel, step-counter kernel] is captured ONCE into a CUDA graph and replayed T-1
times: per-step scalars live in a device table indexed by a device-side step counter, so
there is no host work inside the loop (the reference issues ~10^3 launches and ~5*10^3 ATen
calls per step from Python).  The per-step update replays the reference's fp32 operation
order (SURVEY.md Appendix B 13a); noise is drawn with torch.randn on the same generator in
the same order (1 + T draws per prior, the t=0 draw included).
"""
import os

import numpy as np
import torch
from loguru import logger

from .. import _lib as L
from .diffusion import make_beta_schedule


class DiffusionDiscretized(object):
    def __init__(self, args, var_fun, cfg):
        self.cfg = cfg
        self._diffusion_steps = cfg.ddpm.num_steps
        self._denoising_stddevs = 'beta'
        self.p2_gamma = cfg.ddpm.p2_gamma
        self.p2_k = cfg.ddpm.p2_k
        self.use_p2_weight = cfg.ddpm.use_p2_weight
        self.betas = make_beta_schedule(cfg.ddpm.sched_mode, cfg.ddpm.beta_1, cfg.ddpm.beta_T, cfg.ddpm.num_steps).numpy()
        self._device = torch.device('cuda', torch.cuda.current_device()) if torch.cuda.is_available() else torch.device('cpu')
        self._betas_init, self._alphas, self._alpha_bars, self._betas_post_init, self.snr = \
            self._generate_base_constants(diffusion_steps=self._diffusion_steps)
        self._tables = None
        self.use_cuda_graph = os.environ.get('LION_NO_GRAPH', '0') != '1'   # eager loop for profilers
        self.last_gpu_launches = 0
        self.total_gpu_launches = 0      # kernels of this library launched by all sampling loops so far

    def _generate_base_constants(self, diffusion_steps):
        """float64 numpy -> fp32 tensors (diffusion_pvd.py:118-142)"""
        betas_np = self.betas
        alphas_np = 1.0 - betas_np
        alpha_bars_np = np.cumprod(alphas_np)
        snr = 1.0 / (1 - alpha_bars_np) - 1
        betas_post_np = betas_np[1:] * (1.0 - alpha_bars_np[:-1]) / (1.0 - alpha_bars_np[1:])
        betas_post_init_np = np.append(betas_post_np[0], betas_post_np)
        f = lambda a: torch.from_numpy(a).float().to(self._device)
        return f(betas_np), f(alphas_np), f(alpha_bars_np), f(betas_post_init_np), f(snr)

    def get_p_log_scales(self, timestep, stddev_type):
        if stddev_type == 'beta':
            return 0.5 * torch.log(torch.gather(self._betas_init, 0, timestep - 1))
        elif stddev_type == 'beta_post':
            return 0.5 * torch.log(torch.gather(self._betas_post_init, 0, timestep - 1))
        elif stddev_type == 'learn':
            return None
        raise ValueError('Unknown stddev_type: {}'.format(stddev_type))

    def get_q_posterior_mean(self, x_noisy, prediction, t):
        if t == 0:
            return 1.0 / torch.sqrt(self._alpha_bars[0]) * (x_noisy - torch.sqrt(1.0 - self._alpha_bars[0]) * prediction)
        return 1.0 / torch.sqrt(self._alphas[t]) * (
            x_noisy - self._betas_init[t] * prediction / torch.sqrt(1.0 - self._alpha_bars[t]))

    def get_mixing_component(self, x_noisy, timestep, enabled):
        if enabled:
            raise NotImplementedError("lion_b200: mixed prediction is disabled in every shipped prior config")
        return None

    # ------------------------------------------------------------------------------------
    # training objective (diffusion_pvd.py:44-113): the quantities train_2prior.train_iter draws for its prior losses
    def _iw_at(self, B, timestep):
        """timestep int64 [B] in [1, T] -> (timestep, var_t [B,1,1,1] = 1 - alpha_bar, m_t [B,1,1,1] = sqrt(alpha_bar),
        loss weight (the p2 weight 1 / (p2_k + snr)^p2_gamma [B] with ddpm.use_p2_weight, 1.0 otherwise), None, None)"""
        alpha_bars = torch.gather(self._alpha_bars, 0, timestep - 1)
        var_t = (1.0 - alpha_bars)[:, None, None, None]
        m_t = torch.sqrt(alpha_bars)[:, None, None, None]
        loss_weight = 1.0
        if self.use_p2_weight:
            loss_weight = torch.gather(1 / (self.p2_k + self.snr) ** self.p2_gamma, 0, timestep - 1).view(B)
        return timestep, var_t, m_t, loss_weight, None, None

    def iw_quantities(self, B, *args):
        """Diffusion quantities at B timesteps drawn uniformly from {1, .., T}: floor(U[0, 1) * T) + 1 with U from
        torch.rand on this object's device (the reference draws on 'cuda').  Extra arguments (time_eps, iw_sample_p,
        iw_subvp_like_vp_sde in the reference's call) are ignored, as there."""
        rho = torch.rand(size=[B], device=self._alpha_bars.device) * self._diffusion_steps
        timestep = rho.type(torch.int64)
        assert timestep.max() <= self._diffusion_steps - 1, 'get max at %d' % timestep.max()
        return self._iw_at(B, timestep + 1)

    def iw_quantities_t(self, B, timestep, *args):
        """iw_quantities at given 0-based timesteps [B] (int64, in [0, T-1])."""
        return self._iw_at(B, timestep.view(B) + 1)

    def sample_q(self, x_init, noise, var_t, m_t):
        """A draw of the forward process at t: m_t * x_init + sqrt(var_t) * noise, all 4-D ([B, C, 1, 1], var_t and m_t
        [B, 1, 1, 1] as iw_quantities returns them)."""
        assert len(x_init.shape) == 4 and len(var_t.shape) == 4 and len(m_t.shape) == 4
        assert x_init.shape[0] == m_t.shape[0]
        return m_t * x_init + torch.sqrt(var_t) * noise

    # ------------------------------------------------------------------------------------
    def _step_tables(self, device):
        """[T][4] fp32 rows consumed by lion_ddpm_update, built with the reference's own fp32
        expressions (diffusion_pvd.py:161, :475-486)."""
        if self._tables is None or self._tables.device != device:
            a, ab, b = self._alphas.to(device), self._alpha_bars.to(device), self._betas_init.to(device)
            tab = torch.stack([1.0 / torch.sqrt(a), b, torch.sqrt(1.0 - ab), torch.exp(0.5 * torch.log(b))], dim=1)
            tab[0, 0] = 1.0 / torch.sqrt(ab[0])
            tab[0, 1] = torch.sqrt(1.0 - ab[0])
            tab[0, 2] = 1.0
            tab[0, 3] = 0.0
            self._tables = tab.contiguous()
        return self._tables

    @torch.no_grad()
    def run_denoising_diffusion(self, model, num_samples, shape, temp=1.0, enable_autocast=False, is_image=False,
                                prior_var=1.0, condition_input=None, given_noise=None, clip_feat=None, cls_emb=None,
                                grid_emb=None):
        """Run the full denoising sampling loop (reference: diffusion_pvd.py:223-303).  enable_autocast runs the model
        call under torch.autocast("cuda", float16) as the reference does, the captured step included (the mode is
        baked into the graph); this package's networks return fp32 there."""
        if is_image or cls_emb is not None or grid_emb is not None:
            raise NotImplementedError("lion_b200: is_image / cls_emb / grid_emb are not used by LION's sampling path")
        if getattr(model, 'mixed_prediction', False):
            raise NotImplementedError("lion_b200: mixed prediction is disabled in every shipped prior config")
        model.eval()
        T = self._diffusion_steps
        size = [num_samples] + list(shape)
        if given_noise is None:
            x0 = torch.randn(size=size, device='cuda')
        else:
            x0 = given_noise[0].to('cuda', torch.float32)
        dev = x0.device
        n = x0.numel()
        tables = self._step_tables(dev)
        x = x0.clone().contiguous()                 # updated in place every step
        hist = torch.empty([T] + size, device=dev, dtype=torch.float32)
        noise = torch.empty(size, device=dev, dtype=torch.float32)
        step = torch.zeros(1, device=dev, dtype=torch.int32)
        tfl = torch.zeros(num_samples, device=dev, dtype=torch.float32)
        lib = L.lib()
        launches = 0

        # given_noise[1] may be a device-resident block: an object with `device_block` (contiguous fp32 CUDA tensor
        # [T, *size], row t = the noise of timestep t) and optionally `ensure(t)` (called on the host before step t is
        # enqueued, e.g. to make the stream wait for an upload still in flight).  The step then fetches its row inside the
        # captured graph (lion_ddpm_fetch_noise, indexed by the device-side step counter) instead of one host-issued copy
        # per step between graph replays.
        block = getattr(given_noise[1], 'device_block', None) if given_noise is not None else None
        if block is not None:
            if not (block.is_cuda and block.dtype == torch.float32 and block.is_contiguous() and block.shape[0] >= T
                    and block[0].numel() == n and n % 4 == 0 and block.data_ptr() % 16 == 0):
                raise ValueError("lion_b200: given_noise device_block must be a contiguous fp32 CUDA tensor [T, *size]")
        ensure = getattr(given_noise[1], 'ensure', None) if block is not None else None

        def draw_noise(t):
            if given_noise is None:
                torch.randn(size, device=dev, out=noise)
            elif block is not None:
                if ensure is not None:
                    ensure(t)
            else:
                noise.copy_(given_noise[1][t].to(dev, torch.float32))

        def body(draw):
            with torch.autocast("cuda", dtype=torch.float16, enabled=enable_autocast):
                pred = model(x=x, t=tfl, condition_input=condition_input, clip_feat=clip_feat)
            if draw:
                torch.randn(size, device=dev, out=noise)
            elif block is not None:
                L.check(lib.lion_ddpm_fetch_noise(L.ptr(noise), L.ptr(block), L.ptr(step), n, L.stream()), "ddpm_fetch_noise")
            L.check(lib.lion_ddpm_update(L.ptr(x), L.ptr(pred.contiguous()), L.ptr(noise), L.ptr(x), L.ptr(tables),
                                         L.ptr(step), float(temp), n, L.ptr(hist), T, L.stream()), "ddpm_update")
            L.check(lib.lion_ddpm_next_step(L.ptr(step), L.ptr(tfl), num_samples, L.stream()), "ddpm_next_step")
            return pred

        with torch.cuda.device(dev):
            L.check(lib.lion_ddpm_set_step(L.ptr(step), L.ptr(tfl), num_samples, T - 1, L.stream()), "ddpm_set_step")
            graph_ok = self.use_cuda_graph and getattr(model, 'lion_graph_safe', True) and T > 2
            # step T-1 runs eagerly: it builds/packs the model and sizes the scratch arena
            if given_noise is not None:
                draw_noise(T - 1)
            body(given_noise is None)
            per_step = L.last_launches(dev) + 2 + (1 if block is not None else 0)
            launches += per_step
            graph = None
            if graph_ok:
                if given_noise is not None:
                    draw_noise(T - 2)
                with L.capture_graph() as graph:
                    body(given_noise is None)
            for t in reversed(range(0, T - 1)):
                if t % 500 == 0:
                    logger.info('t={}; shape={}, num_samples={}, sample shape: {}', t, shape, num_samples, x.shape)
                if given_noise is not None:
                    draw_noise(t)
                if graph is not None:
                    graph.replay()
                else:
                    body(given_noise is None)
                launches += per_step
        self.last_gpu_launches = launches
        self.total_gpu_launches += launches
        # the reference appends x_noisy after every step, and at t == 0 x_noisy is not updated
        # (diffusion_pvd.py:292-298), so the last entry repeats the one before it
        pred_x = [hist[k] for k in range(T - 1)] + [hist[T - 2] if T > 1 else x0]
        x_image = hist[T - 1]
        model.train()
        return x_image, {'pred_x': pred_x}

    def _ddim_tables(self, steps, kappa, device):
        """[S][4] fp32 rows {a, c, sigma, t+1} consumed by lion_ddim_update, built with the
        reference's own fp32 scalar expressions (diffusion_pvd.py:437-451)."""
        Alpha_bar = self._alpha_bars.cpu()
        rows = []
        for i, t in enumerate(steps):
            if i == len(steps) - 1:
                assert t == 0
                alpha_next = torch.tensor(1.0)
                sigma = torch.tensor(0.0)
            else:
                alpha_next = Alpha_bar[steps[i + 1]]
                sigma = kappa * torch.sqrt((1 - alpha_next) / (1 - Alpha_bar[t]) * (1 - Alpha_bar[t] / alpha_next))
            a = torch.sqrt(alpha_next / Alpha_bar[t])
            c = torch.sqrt(1 - alpha_next - sigma ** 2) - torch.sqrt(1 - Alpha_bar[t]) * torch.sqrt(alpha_next / Alpha_bar[t])
            rows.append(torch.stack([a, c, sigma.to(torch.float32), torch.tensor(float(t + 1))]))
        return torch.stack(rows).to(torch.float32).contiguous().to(device)

    @torch.no_grad()
    def run_ddim(self, model, num_samples, shape, temp=1.0, enable_autocast=False, is_image=True, prior_var=1.0,
                 condition_input=None, ddim_step=100, skip_type='uniform', kappa=1.0, clip_feat=None, grid_emb=None,
                 x_noisy=None, dae_index=-1, given_noise=None):
        """DDIM sampler on the same networks (reference: diffusion_pvd.py:389-473): S = ddim_step model
        calls instead of T.  Like the DDPM loop, the step (model forward + update + step counter)
        is captured in a CUDA graph and replayed; the per-step scalars come from a device table.

        Noise: the reference draws `torch.randn(size)` on the CPU generator once per step and
        copies it to the device (:464-465); the S draws are made up front, in the same order,
        from the same generator (nothing else consumes it inside the loop), so a seeded run sees
        the same values.  given_noise (extension, [S, *size]) replaces them.  enable_autocast: as in
        run_denoising_diffusion."""
        if grid_emb is not None:
            raise NotImplementedError("lion_b200: grid_emb is not used by LION's sampling path")
        if getattr(model, 'mixed_prediction', False):
            raise NotImplementedError("lion_b200: mixed prediction is disabled in every shipped prior config")
        model.eval()
        size = [num_samples] + list(shape)
        x_noisy = torch.randn(size=size, device='cuda') if x_noisy is None else x_noisy.cuda()
        dev = x_noisy.device
        S = ddim_step
        if skip_type == 'uniform':
            c = (self._diffusion_steps - 1.0) / (S - 1.0)
            list_tau = [int(np.floor(i * c)) for i in range(S)]
        elif skip_type == 'quad':
            seq = np.linspace(0, np.sqrt(self._diffusion_steps * 0.8), S) ** 2
            list_tau = [int(s) for s in list(seq)]
        else:
            raise NotImplementedError(skip_type)
        steps = sorted(list(list_tau), reverse=True)
        tables = self._ddim_tables(steps, kappa, dev)
        if given_noise is None:
            noise = torch.stack([torch.randn(size) for _ in range(S)]).to(dev)
        else:
            noise = torch.as_tensor(given_noise, dtype=torch.float32).reshape([S] + size).to(dev)
        noise = noise.contiguous()
        x = x_noisy.to(torch.float32).clone().contiguous()
        n = x.numel()
        hist = torch.empty([S] + size, device=dev, dtype=torch.float32)
        step = torch.zeros(1, device=dev, dtype=torch.int32)
        tfl = torch.zeros(num_samples, device=dev, dtype=torch.float32)
        lib = L.lib()

        def body():
            with torch.autocast("cuda", dtype=torch.float16, enabled=enable_autocast):
                pred = model(x=x, t=tfl, condition_input=condition_input, clip_feat=clip_feat)
            L.check(lib.lion_ddim_update(L.ptr(x), L.ptr(pred.contiguous()), L.ptr(noise), L.ptr(x), L.ptr(tables),
                                         L.ptr(step), n, L.ptr(hist), L.stream()), "ddim_update")
            L.check(lib.lion_ddim_next_step(L.ptr(step), L.ptr(tfl), L.ptr(tables), num_samples, S, L.stream()), "ddim_next_step")

        launches = 0
        with torch.cuda.device(dev):
            L.check(lib.lion_ddim_set_step(L.ptr(step), L.ptr(tfl), L.ptr(tables), num_samples, S, 0, L.stream()), "ddim_set_step")
            body()                      # eager first step: builds/packs the model, sizes the arena
            per_step = L.last_launches(dev) + 2
            launches += per_step
            graph = None
            if self.use_cuda_graph and getattr(model, 'lion_graph_safe', True) and S > 2:
                with L.capture_graph() as graph:
                    body()
            for _ in range(1, S):
                if graph is not None:
                    graph.replay()
                else:
                    body()
                launches += per_step
        self.last_gpu_launches = launches
        self.total_gpu_launches += launches
        model.train()
        return hist[S - 1], [hist[k] for k in range(S)]
