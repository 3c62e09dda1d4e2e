"""CPU checks of the style prior's training side against tests/golden/global_prior_grad.npz (made from the unmodified
reference by make_golden_global_prior_grad.py): the float64 restatement the GPU gradient tests compare with
(tests/gp_grad_ref.py) reproduces the reference's loss and gradients; DiffusionDiscretized.iw_quantities,
iw_quantities_t and sample_q reproduce the reference's draws; the training entry points of the C ABI are exported
with the argument counts include/lion_b200.h declares."""
import os
import re

import numpy as np
import pytest
import torch

from tests import gp_grad_ref as GR
from tests.synth import synth_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "global_prior_grad.npz")
# (D, nf, emb, cells, clip_dim, dropout) of the golden's networks, and their weight seeds
SMALL = (16, 32, 16, 2, 16, 0.2)
SEEDS = {"drop": 21, "clip": 24}


def small_net(clip):
    """The golden's reduced-width PriorSEDrop / PriorSEClip (on the CPU; its weights are not loaded)."""
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.score_sde.resnet import PriorSEClip, PriorSEDrop
    D, nf, emb, cells, clip_dim, p = SMALL
    cfg = default_prior_cfg(clip=clip)
    cfg.sde.num_channels_dae, cfg.sde.embedding_dim, cfg.sde.num_cell_per_scale_dae, cfg.sde.dropout = nf, emb, cells, p
    cfg.clipforge.feat_dim = clip_dim
    return (PriorSEClip if clip else PriorSEDrop)(cfg.sde, D, cfg)


def small_sd(tag):
    net = small_net(tag == "clip")
    return synth_state_dict({k: list(v.shape) for k, v in net.state_dict().items()}, SEEDS[tag])


@pytest.mark.parametrize("tag", ["drop", "clip"])
def test_restatement_matches_reference_gradients(tag):
    z = np.load(GOLDEN)
    G = GR.golden(tag, z)
    sd = small_sd(tag)
    assert set(sd) == set(G["grads"])
    loss, dx, grads = GR.mse_grads(sd, G["x"], G["pe"], G["noise"], G["clip"], G["mask"])
    assert abs(loss.item() - G["loss"]) <= 1e-13 * abs(G["loss"])
    errs = {"dx": ((dx - G["dx"]).norm() / G["dx"].norm()).item()}
    for k, g in grads.items():
        ref = G["grads"][k]
        errs[k] = ((g.view(ref.shape) - ref).norm() / ref.norm().clamp_min(1e-300)).item()
    worst = max(errs, key=errs.get)
    assert errs[worst] <= 1e-12, "%s: relative Frobenius error %.3e" % (worst, errs[worst])


def _diffusion(p2):
    from lion_b200.config import default_prior_cfg
    from lion_b200.utils.diffusion_pvd import DiffusionDiscretized
    cfg = default_prior_cfg()
    cfg.ddpm.use_p2_weight = p2
    d = DiffusionDiscretized(None, None, cfg)
    # the golden was drawn on the CPU; draw on it here as well
    d._alpha_bars, d.snr = d._alpha_bars.cpu(), d.snr.cpu()
    return d


@pytest.mark.parametrize("p2", [0, 1])
def test_iw_quantities_and_sample_q_match_reference(p2):
    z = np.load(GOLDEN)
    d = _diffusion(p2)
    torch.manual_seed(5)
    t, var_t, m_t, w, a, b = d.iw_quantities(16)
    assert a is None and b is None
    assert torch.equal(t, torch.from_numpy(z["iw%d/t" % p2]))
    assert torch.equal(var_t, torch.from_numpy(z["iw%d/var_t" % p2]))
    assert torch.equal(m_t, torch.from_numpy(z["iw%d/m_t" % p2]))
    if p2:
        assert torch.equal(w, torch.from_numpy(z["iw1/weight"]))
    else:
        assert w == 1.0
    q = d.sample_q(torch.from_numpy(z["iw%d/x0" % p2]), torch.from_numpy(z["iw%d/noise" % p2]), var_t, m_t)
    assert torch.equal(q, torch.from_numpy(z["iw%d/sample_q" % p2]))
    r = d.iw_quantities_t(5, torch.from_numpy(z["iwt%d/t" % p2]))
    assert torch.equal(r[0], torch.from_numpy(z["iwt%d/t" % p2]) + 1)
    assert torch.equal(r[1], torch.from_numpy(z["iwt%d/var_t" % p2]))
    assert torch.equal(r[2], torch.from_numpy(z["iwt%d/m_t" % p2]))
    if p2:
        assert torch.equal(r[3], torch.from_numpy(z["iwt1/weight"]))


def _declared_arity():
    src = open(os.path.join(ROOT, "include", "lion_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for name, args in re.findall(r"\b(lion_global_prior_[a-z_]+)\s*\(([^)]*)\)", src):
        out[name] = len([a for a in args.split(",") if a.strip() and a.strip() != "void"])
    return out


def test_training_entry_points_exported_with_declared_arity():
    from lion_b200 import _lib
    lib = _lib.lib()
    arity = _declared_arity()
    new = ["lion_global_prior_saved_floats", "lion_global_prior_forward_train", "lion_global_prior_backward",
           "lion_global_prior_backward_probe"]
    for n in new:
        assert n in arity, "%s is not declared" % n
        fn = getattr(lib, n)
        assert len(fn.argtypes) == arity[n], "%s: %d ctypes arguments, %d declared" % (n, len(fn.argtypes), arity[n])
    import ctypes as C
    assert lib.lion_global_prior_saved_floats.restype == C.c_size_t
