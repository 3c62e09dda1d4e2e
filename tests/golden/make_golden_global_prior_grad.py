"""Generate tests/golden/global_prior_grad.npz from the UNMODIFIED reference (container only):

    python tests/golden/make_golden_global_prior_grad.py

On CPU, in float64, at a reduced width (nf 32, 2 cells, D 16, embedding_dim 16; CLIP feature width 16) with
key-seeded synthetic weights:
  * the style prior's term of train_2prior.train_iter (trainers/train_2prior.py:276-313, pvd_mse_loss 1): timesteps,
    var_t and m_t from DiffusionDiscretized.iw_quantities, eps_t = sample_q(eps, noise, var_t, m_t), the prior's output
    and F.mse_loss against the noise, then its backward -- for PriorSEDrop in train() mode with nn.Dropout multiplying
    by stored scaled masks, and for PriorSEClip.  Stored: the inputs (eps_t fp32, t, the positional embedding the
    reference computed, clip features, masks, noise), the loss, dL/d eps_t and every parameter gradient by state-dict
    name ("<net>/g/<key>");
  * one DiffusionDiscretized.iw_quantities draw (B = 16, torch.manual_seed(5)) without and with ddpm.use_p2_weight, and
    sample_q of seeded inputs at it."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.golden import ref_import as R  # noqa: E402

R.install()
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tests.golden.make_golden import load_synth, gen  # noqa: E402

B, D, NF, CELLS, EMB, CLIP_DIM, P_DROP = 6, 16, 32, 2, 16, 16, 0.2


class _Mask(torch.nn.Module):
    """nn.Dropout replaced by a multiplication with a stored scaled mask [B, nf]."""

    def __init__(self, mask):
        super().__init__()
        self.mask = mask

    def forward(self, x):
        return x * self.mask[:, :, None, None]


class _Const(torch.nn.Module):
    """The positional embedding, computed in fp32 by the reference, handed to the float64 network."""

    def __init__(self, v):
        super().__init__()
        self.v = v

    def forward(self, t):
        return self.v


def prior_term(net, diff, tag, seed, clip_feat=None, masks=None):
    """The style prior's loss and gradients (train_2prior.py:284-313 for latent_id 0), float64."""
    torch.manual_seed(seed)
    t_p, var_t_p, m_t_p, _, _, _ = diff.iw_quantities(B)
    eps = gen(seed + 1, B, D, 1, 1)
    noise_p = gen(seed + 2, B, D, 1, 1)
    eps_t_p = diff.sample_q(eps, noise_p, var_t_p, m_t_p)          # fp32, as the reference computes it
    temb_fun = net.temb_fun
    pe = temb_fun(t_p)                                              # fp32 positional embedding
    net.temb_fun = _Const(pe.double())
    net.double()
    if masks is not None:
        net.train()
        for k, blk in enumerate(net.all_modules):
            blk.dropout = _Mask(masks[k])
    x = eps_t_p.double().requires_grad_(True)
    clip = None if clip_feat is None else clip_feat.double()
    pred = net(x, t_p, clip_feat=clip)
    loss = F.mse_loss(pred.contiguous().view(B, -1), noise_p.double().view(B, -1), reduction='mean')
    loss.backward()
    out = {tag + "/x": eps_t_p.view(B, D).numpy(), tag + "/t": t_p.float().numpy(), tag + "/pe": pe.numpy(),
           tag + "/noise": noise_p.view(B, D).numpy(), tag + "/loss": np.float64(loss.item()),
           tag + "/dx": x.grad.view(B, D).numpy()}
    for k, p in net.named_parameters():
        out[tag + "/g/" + k] = p.grad.numpy()
    if clip_feat is not None:
        out[tag + "/clip"] = clip_feat.numpy()
    if masks is not None:
        out[tag + "/mask"] = masks.numpy()
    print(tag, "loss", loss.item(), "|dx|", x.grad.norm().item())
    return out


def main():
    torch.set_num_threads(8)
    small = ["sde.num_channels_dae", NF, "sde.num_cell_per_scale_dae", CELLS, "sde.embedding_dim", EMB,
             "sde.dropout", P_DROP]
    cfg = R.load_cfg(overrides=small)
    cfg_clip = R.load_cfg(overrides=small + ["clipforge.enable", 1, "clipforge.feat_dim", CLIP_DIM])
    from models.score_sde.resnet import PriorSEClip, PriorSEDrop
    from utils.diffusion_pvd import DiffusionDiscretized
    diff = DiffusionDiscretized(None, None, cfg)
    out = {}

    net = PriorSEDrop(cfg.sde, D, cfg)
    load_synth(net, 21)
    g = torch.Generator().manual_seed(22)
    masks = (torch.rand(CELLS, B, NF, generator=g) >= P_DROP).double() / (1 - P_DROP)
    out.update(prior_term(net, diff, "drop", 23, masks=masks))

    net = PriorSEClip(cfg_clip.sde, D, cfg_clip)
    load_synth(net, 24)
    out.update(prior_term(net, diff, "clip", 25, clip_feat=gen(26, B, CLIP_DIM)))

    for p2 in (0, 1):
        c = R.load_cfg(overrides=["ddpm.use_p2_weight", p2])
        d = DiffusionDiscretized(None, None, c)
        torch.manual_seed(5)
        t, var_t, m_t, w, _, _ = d.iw_quantities(16)
        x0, nz = gen(27, 16, 4, 1, 1), gen(28, 16, 4, 1, 1)
        out.update({"iw%d/t" % p2: t.numpy(), "iw%d/var_t" % p2: var_t.numpy(), "iw%d/m_t" % p2: m_t.numpy(),
                    "iw%d/weight" % p2: np.asarray(w, dtype=np.float32),
                    "iw%d/x0" % p2: x0.numpy(), "iw%d/noise" % p2: nz.numpy(),
                    "iw%d/sample_q" % p2: d.sample_q(x0, nz, var_t, m_t).numpy()})
        tt = torch.tensor([0, 1, 499, 998, 999])
        r = d.iw_quantities_t(5, tt)
        out.update({"iwt%d/t" % p2: tt.numpy(), "iwt%d/var_t" % p2: r[1].numpy(), "iwt%d/m_t" % p2: r[2].numpy(),
                    "iwt%d/weight" % p2: np.asarray(r[3], dtype=np.float32)})
    np.savez_compressed(os.path.join(HERE, "global_prior_grad.npz"), **out)


if __name__ == "__main__":
    main()
