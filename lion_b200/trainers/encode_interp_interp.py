"""Interpolation between two encoded shapes -- host-side mirror of the reference's trainers/encode_interp_interp.py, the
trainer `script/interpolate_posterior.sh` selects (trainer.type trainers.encode_interp_interp, sde.ode_sample 1,
sde.embedding_scale 1000).  `Trainer.eval_nll` (:121-322): the first two shapes of every batch are encoded (global
latent, then latent points conditioned on it), carried to noise along the probability-flow ODE (`compute_ode_nll`, on the
device), blended by `interpolate_noise` into four noises, brought back by the ODE sampler and decoded.

There are no data loaders in this package: eval_nll takes the batches ({'tr_points': [B0, N, 3]}, B0 >= 2) as an
iterable.  Not kept: rendered images, the VAE loss of the batch (`get_loss`, training side) and the EMA swap."""
import os

import torch
from loguru import logger

from ..utils.diffusion_continuous import make_diffusion
from .interpolate_latent import interpolate_noise
from .train_prior import Trainer as BaseTrainer


class Trainer(BaseTrainer):
    is_diffusion = 0
    generate_mode_global = 'interpolate'
    generate_mode_local = 'interpolate'

    def __init__(self, cfg, args=None):
        super().__init__(cfg, args)
        self.diffusion_cont = make_diffusion(cfg.sde)
        self.draw_sample_when_vis = 0

    @torch.no_grad()
    def eval_sample(self, step=0):
        pass

    @torch.no_grad()
    def eval_nll(self, step, ntest=None, save_file=False, data_loader=None):
        """For batch vid of data_loader: shapes (a, b) -> B = 4 inputs (a, b, a, b) -> 4 interpolated clouds [N, 3] saved
        as save_dir/enc60_<global>_<local>/sph_B4_<vid %04d>/<i %04d>.  Returns 0."""
        if data_loader is None:
            raise ValueError("lion_b200: eval_nll needs the batches (an iterable of {'tr_points': [B0, N, 3]})")
        cfg = self.cfg
        diffusion = self.diffusion_cont if cfg.sde.ode_sample else self.diffusion_disc
        num_selected = 60
        output_dir_template = cfg.save_dir + '/enc%d_%s_%s/' % (num_selected, self.generate_mode_global, self.generate_mode_local)
        ode_eps = cfg.sde.ode_eps
        ode_solver_tol = 1e-5
        enable_autocast = False
        temp = 1.0
        clip_feat = None
        self.model.eval()
        self.dae.eval()
        dae = self.dae
        B = 4
        for vid, val_batch in enumerate(data_loader):
            output_dir = output_dir_template + '/sph_B%d_%04d' % (B, vid)
            os.makedirs(output_dir, exist_ok=True)
            pt_cur = val_batch['tr_points'][:2]
            B0, N, C = pt_cur.shape
            inputs = pt_cur[None].expand(B // B0, -1, -1, -1).contiguous().view(B, N, C).contiguous().cuda().float()
            file_name = ['%04d' % i for i in range(B)]
            # -- global latent --
            dist = self.model.encode_global(inputs)
            shape = self.model.latent_shape()[0]
            eps = dist.sample()[0]
            eps_shape_global = eps.shape
            eps_global = eps.view([B] + shape).contiguous()
            # -- latent points, conditioned on the encoded global latent --
            style = self.model.global2style(eps_global.view(eps_shape_global))
            dist_local = self.model.encode_local(inputs, style)
            shape = self.model.latent_shape()[1]
            eps = dist_local.sample()[0]
            eps_shape_local = eps.shape
            eps = eps.view([B] + shape)
            # -- to noise, interpolate, back --  (the reference passes the latent-point shape to both samplers; with the
            # noise given, the shape is not used)
            eps_T_global_interp = diffusion.compute_ode_nll(dae[0], eps_global, ode_eps, ode_solver_tol, condition_input=None)
            eps_T_global_interp = interpolate_noise(eps_T_global_interp.contiguous())
            eps_0_global_interp, _, _ = diffusion.sample_model_ode(dae[0], B, shape, ode_eps, ode_solver_tol, enable_autocast,
                                                                   temp, noise=eps_T_global_interp, condition_input=None,
                                                                   clip_feat=clip_feat)
            eps_T_local_interp = diffusion.compute_ode_nll(dae[1], eps, ode_eps, ode_solver_tol, condition_input=eps_global)
            eps_T_local_interp = interpolate_noise(eps_T_local_interp.contiguous())
            eps_0_local_interp, _, _ = diffusion.sample_model_ode(dae[1], B, shape, ode_eps, ode_solver_tol, enable_autocast,
                                                                  temp, noise=eps_T_local_interp,
                                                                  condition_input=eps_0_global_interp, clip_feat=clip_feat)
            style = self.model.global2style(eps_0_global_interp.view(eps_shape_global))
            eps_local = eps_0_local_interp.view(eps_shape_local)
            gen_x = self.model.decoder(None, beta=None, context=eps_local, style=style)
            for i, file_name_i in enumerate(file_name):
                torch.save(gen_x[i], os.path.join(output_dir, file_name_i))
            logger.info('save output at : {}', output_dir)
        return 0
