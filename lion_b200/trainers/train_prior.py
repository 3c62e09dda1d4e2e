"""Sampling-side `Trainer` -- host-side mirror of the three sampling entry points SURVEY.md section 2 row 11 stars:
`Trainer.sample` (reference trainers/train_prior.py:645-701), `Trainer.eval_sample`'s generation half
(trainers/base_trainer.py:446-487) and, through them, `generate_samples_vada_2prior` (trainers/train_2prior.py:49-127).

What is kept: the constructor's model half (`build_model` VAE, `build_prior` = ModuleList([style prior, point prior]) +
`DiffusionDiscretized`, trainers/train_2prior.py:415-451), `resume(ckpt)` for the reference's checkpoint keys
(`dae_state_dict`, `vae_state_dict`; train_prior.py:294-326), and the two sampling methods with their signatures, return
layouts ([B,3,N] from `sample`, [num,N,3] from `eval_sample`), iteration count and seeding scheme.
What is not: data loaders, optimisers / EMA swaps (the modules hold whatever weights were loaded), training iterations,
visualisation, metric bookkeeping -- none of it is on the sampling path (SURVEY.md section 2: OUT OF SCOPE).

Multi-GPU (`torch.distributed` initialised): every rank generates its own batches and the finished clouds are
all_gathered once, device to device (lion_b200/utils/dist_sampling.py); ranks draw distinct noise unless
`reference_seeding=True` reproduces the reference's same-seed-on-every-rank behaviour (base_trainer.py:459-463)."""
import os

import numpy as np
import torch
import torch.distributed as dist
from loguru import logger

from ..models.lion import import_model
from ..models.vae_adain import Model as VAE
from ..third_party.pvcnn import functional as pvcnn_fn
from ..utils import dist_sampling
from ..utils.diffusion_pvd import DiffusionDiscretized
from .train_2prior import generate_samples_vada_2prior


class Trainer(object):
    def __init__(self, cfg, args=None):
        self.cfg, self.args = cfg, args
        self.device_str = 'cuda'
        device = torch.device('cuda', torch.cuda.current_device())
        self.model = VAE(cfg).to(device)                                           # build_model
        self.dae = torch.nn.ModuleList([                                           # build_prior (train_2prior.py:415-451)
            import_model(cfg.latent_pts.style_prior)(cfg.sde, cfg.latent_pts.style_dim, cfg),
            import_model(cfg.sde.prior_model)(cfg.sde, cfg.shapelatent.latent_dim, cfg)]).to(device)
        self.dae.num_points = self.dae[1].num_points
        self.dae.num_classes = self.dae[1].num_classes
        self.diffusion_disc = DiffusionDiscretized(cfg.sde, None, cfg)
        self.num_steps = self.diffusion_disc._diffusion_steps
        self.sample_num_points = cfg.data.tr_max_sample_points
        self.fun_generate_samples_vada = generate_samples_vada_2prior

    def resume(self, path, **kwargs):
        """dae / vae weights from a reference checkpoint (optimizer / EMA state is ignored: sampling consumes the weights
        that sit in the modules)."""
        ckpt = torch.load(path, map_location='cpu', weights_only=False)
        self.dae.load_state_dict(ckpt['dae_state_dict'])
        self.model.load_state_dict(ckpt['vae_state_dict'])
        return ckpt.get('epoch', 0)

    @torch.no_grad()
    def sample(self, num_shapes=2, num_points=2048, device_str='cuda', for_vis=True, use_ddim=False, save_file=None,
               ddim_step=0, clip_feat=None):
        """returns the final samples in shape [B,3,N]"""
        assert not self.cfg.clipforge.enable, 'not support yet (the reference asserts the same; pass clip_feat to ' \
                                              'generate_samples_vada_2prior or LION.sample for text2shape)'
        assert self.cfg.sde.ode_sample == 0, "lion_b200: sde.ode_sample must be 0 (DDPM / DDIM sampling)"
        self.model.eval()
        self.dae.eval()
        latent_shape = self.model.latent_shape()
        gen_x, nstep, ode_time, sample_time, output_fsample = self.fun_generate_samples_vada(
            latent_shape, self.dae, self.diffusion_disc, self.model, num_shapes, enable_autocast=self.cfg.sde.autocast_train,
            ode_sample=0,
            need_denoise=self.cfg.eval.need_denoise, ddim_step=ddim_step, clip_feat=clip_feat)
        assert gen_x.shape[2] == self.cfg.ddpm.input_dim
        if gen_x.shape[1] > self.sample_num_points:
            gen_x = pvcnn_fn.furthest_point_sample(gen_x.permute(0, 2, 1).contiguous(), self.sample_num_points).permute(0, 2, 1).contiguous()
        traj = gen_x.permute(0, 2, 1).contiguous()          # BN3 -> B3N
        if save_file:
            os.makedirs(os.path.dirname(save_file) or '.', exist_ok=True)
            torch.save(traj.permute(0, 2, 1), save_file)
        return traj

    @torch.no_grad()
    def eval_sample(self, step=0, num_ref=None, batch_size_test=None, ddim_step=0, output_name=None, reference_seeding=False):
        """Generation half of base_trainer.eval_sample (:446-492): num_gen_iter batches of batch_size_test shapes per rank,
        re-seeded per batch, gathered over ranks; returns gen_pcs [num, N, 3] on the host (rank order) and saves them on
        rank 0 when output_name is given.  The scores that follow in the reference (MMD / COV / 1-NNA, JSD) come from
        lion_b200.utils.eval_helper.compute_score(output_name, ref_name)."""
        world = dist.get_world_size() if (dist.is_available() and dist.is_initialized()) else 1
        rank = dist.get_rank() if world > 1 else 0
        batch_size_test = batch_size_test or self.cfg.data.batch_size_test
        num_ref = num_ref or self.cfg.num_ref
        len_test_loader = num_ref // batch_size_test + 1
        if world > 1:
            num_gen_iter = max(1, len_test_loader // world)
            if num_gen_iter * batch_size_test * world < num_ref:
                num_gen_iter += 1
        else:
            num_gen_iter = len_test_loader
        seed = self.cfg.trainer.seed
        gen_pcs = []
        for i in range(num_gen_iter):
            s = dist_sampling.rank_seed(seed + i, rank, reference_behaviour=reference_seeding)
            torch.manual_seed(s)
            np.random.seed(s % (2 ** 32))
            torch.cuda.manual_seed_all(s)
            logger.info('#%d/%d; BS=%d' % (i, num_gen_iter, batch_size_test))
            x = self.sample(num_shapes=batch_size_test, num_points=self.sample_num_points, for_vis=False,
                            ddim_step=ddim_step).permute(0, 2, 1).contiguous()          # B,3,N -> B,N,3
            gen_pcs.append(x)
        gen_pcs = torch.cat(gen_pcs, dim=0)
        gen_pcs = dist_sampling.gather_samples(gen_pcs).cpu()                          # one device-to-device all_gather
        if output_name and rank == 0:
            os.makedirs(os.path.dirname(output_name) or '.', exist_ok=True)
            torch.save(gen_pcs, output_name)
        return gen_pcs
