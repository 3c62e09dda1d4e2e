"""Latent interpolation by ODE sampling -- host-side mirror of the reference's trainers/interpolate_latent.py, the trainer
`script/interpolate.sh` selects (trainer.type trainers.interpolate_latent, sde.ode_sample 1, sde.embedding_scale 1000):
the noise edits `linear_interpolate_noise` / `interpolate_noise` / `subtract_noise` (:23-57), `generate_samples` (:125-177,
the probability-flow ODE route of both priors with a per-prior noise edit) and `Trainer.vis_sample` (:188-255: 40 seeded
batches of 20 shapes saved as %04d.pt files).

The noise edits keep the reference's quirks: they edit their argument in place and return it, the mixing weight is
p = k / len(noise) (so the last shape is never reached by the blend), and `subtract_noise` uses the fixed indices
12 / 15 / 9 / 10 (it needs at least 16 shapes).  Not kept: the rendered images (`validate_inspect` draws them) and the
EMA parameter swap; the modules hold whatever weights were loaded."""
import os
from timeit import default_timer as timer

import numpy as np
import torch
from loguru import logger

from ..utils.diffusion_continuous import DiffusionBase, make_diffusion
from .train_prior import Trainer as PriorTrainer


def linear_interpolate_noise(noise):
    noise_a = noise[0].contiguous()
    noise_b = noise[-1].contiguous()
    for k in range(1, noise.shape[0] - 1):
        p = float(k) / len(noise)
        noise[k] = p * noise_b + (1 - p) * noise_a
    return noise


def interpolate_noise(noise):
    noise_a = noise[0].contiguous()
    noise_b = noise[-1].contiguous()
    for k in range(1, noise.shape[0] - 1):
        p = float(k) / len(noise)
        noise[k] = np.sqrt(p) * noise_b + np.sqrt(1 - p) * noise_a
    return noise


def subtract_noise(noise):
    noise_a = noise[12].contiguous()
    noise_b = noise[15].contiguous()
    diff = noise_a - noise_b
    add_target_1 = noise[9]
    add_target_2 = noise[10]
    noise_list = [noise_a, noise_b, add_target_1, add_target_2, add_target_1 + diff, add_target_2 + diff]
    noise[:6] = torch.stack(noise_list)
    return noise


_NOISE_EDITS = {'subtract': subtract_noise, 'interpolate': interpolate_noise, 'linear_interpolate': linear_interpolate_noise}


@torch.no_grad()
def generate_samples(shape, dae, diffusion, vae, num_samples, enable_autocast, ode_eps=0.00001, ode_solver_tol=1e-5,
                     ode_sample=False, prior_var=1.0, temp=1.0, vae_temp=1.0, noise=None, need_denoise=False,
                     ddim_step=0, writer=None, generate_mode_global='interpolate', generate_mode_local='freeze'):
    """-> (gen_x [num_samples, N, 3], nfe, ode time, sampling time, output) as the reference's; output['gen_x'] = gen_x.
    Per prior level i (0: global, 1: latent points) fresh noise is drawn, edited by the level's mode ('interpolate',
    'linear_interpolate', 'subtract', or 'freeze': every shape takes shape 0's noise) and integrated by the ODE sampler,
    conditioned on the previous level's sample."""
    output = {}
    if not ode_sample:
        raise NotImplementedError("interpolate_latent.generate_samples: only the ODE route (sde.ode_sample 1) is provided, "
                                  "as in the reference")
    assert isinstance(diffusion, DiffusionBase), 'ODE-based sampling requires cont. diffusion!'
    assert ode_eps is not None, 'ODE-based sampling requires integration cutoff ode_eps!'
    assert ode_solver_tol is not None, 'ODE-based sampling requires ode solver tolerance!'
    start = timer()
    condition_input = None
    eps_list = []
    for i in range(len(dae)):
        noise = torch.randn(size=[num_samples] + shape[i], device='cuda')
        generate_mode = generate_mode_global if i == 0 else generate_mode_local
        logger.info('level: {}, generate_mode: {}', i, generate_mode)
        if generate_mode in _NOISE_EDITS:
            noise = _NOISE_EDITS[generate_mode](noise)
        elif generate_mode == 'freeze':
            for k in range(1, noise.shape[0]):
                noise[k] = noise[0]
        eps, nfe, time_ode_solve = diffusion.sample_model_ode(dae[i], num_samples, shape[i], ode_eps, ode_solver_tol,
                                                              enable_autocast, temp, noise, condition_input=condition_input)
        condition_input = eps
        eps_list.append(eps)
        output['sampled_eps'] = eps
    eps = vae.compose_eps(eps_list)
    output['print/sample_mean_global'] = eps.view(num_samples, -1).mean(-1).mean()
    output['print/sample_var_global'] = eps.view(num_samples, -1).var(-1).mean()
    decomposed_eps = vae.decompose_eps(eps)
    image = vae.sample(num_samples=num_samples, decomposed_eps=decomposed_eps)
    output['gen_x'] = image
    sampling_time = timer() - start
    nfe_torch = torch.tensor(nfe * 1.0, device='cuda')
    sampling_time_torch = torch.tensor(sampling_time * 1.0, device='cuda')
    time_ode_solve_torch = torch.tensor(time_ode_solve * 1.0, device='cuda')
    return image, nfe_torch, time_ode_solve_torch, sampling_time_torch, output


class Trainer(PriorTrainer):
    is_diffusion = 0
    generate_mode_global = 'interpolate'
    generate_mode_local = 'interpolate'
    num_val_samples = 20          # the reference's __init__ sets cfg.num_val_samples = 20
    num_interp = 40               # batches written by vis_sample

    def __init__(self, cfg, args=None):
        super().__init__(cfg, args)
        self.diffusion_cont = make_diffusion(cfg.sde)

    @torch.no_grad()
    def vis_sample(self, writer=None, num_vis=None, step=0, include_pred_x0=True, save_file=None):
        """Seed 0, then `num_interp` batches of `num_val_samples` shapes from generate_samples (the ODE route when
        cfg.sde.ode_sample); batch idx goes to save_dir/interp/mode_<global>_<local>_<points>/<idx %04d>/<shape %04d>.pt.
        Returns the last batch's output dict."""
        shape = self.model.latent_shape()
        ode_sample = self.cfg.sde.ode_sample
        diffusion = self.diffusion_cont if ode_sample else self.diffusion_disc
        rank, seed = 0, 0
        torch.manual_seed(rank + seed)
        np.random.seed(rank + seed)
        torch.cuda.manual_seed(rank + seed)
        torch.cuda.manual_seed_all(rank + seed)
        self.model.eval()
        self.dae.eval()
        output = {}
        for idx in range(self.num_interp):
            output_dir = os.path.join(self.cfg.save_dir, 'interp', 'mode_%s_%s_%d' % (
                self.generate_mode_global, self.generate_mode_local, self.sample_num_points), '%04d' % idx)
            logger.info('will save to {}', output_dir)
            os.makedirs(output_dir, exist_ok=True)
            gen_x, nstep, ode_time, sample_time, output = generate_samples(
                shape, self.dae, diffusion, self.model, self.num_val_samples, enable_autocast=self.cfg.sde.autocast_train,
                ode_eps=self.cfg.sde.ode_eps, ode_sample=ode_sample, generate_mode_global=self.generate_mode_global,
                generate_mode_local=self.generate_mode_local)
            logger.info('cast={}, sample step={}, ode_time={}, sample_time={}', self.cfg.sde.autocast_train, nstep,
                        ode_time, sample_time)
            for idxx in range(len(gen_x)):
                torch.save(gen_x[idxx], output_dir + '/%04d.pt' % idxx)
        return output

    def eval_sample(self, step=0):
        logger.info('skip eval-sample')
        return 0
