"""In-place parameter updates (an optimizer or EMA step) reach the library's packed weights: the next forward re-runs
every re-pack step of the model (lion_model_refresh).  The shipped prior has all of them: the SIMT packing (the 128->4
classifier), padded biases and a bias-free convolution (the attention qkv), the wide-tap layout of the sparse first
convolution (the r = 32 PVConvs), and the tensor-core packings, including the ones k_sa_fused and k_ygemm read."""
import json
import os

import pytest
import torch

from tests.synth import synth_state_dict
from tests.util import gen

pytestmark = pytest.mark.gpu
KEYS = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "keys.json")))


def _prior(sd):
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.latent_points_ada_localprior import PVCNN2Prior
    cfg = default_prior_cfg()
    m = PVCNN2Prior(cfg.sde, 1, cfg)
    m.load_state_dict(sd)
    return m.cuda().eval()


def test_in_place_update_matches_rebuilt_model():
    m = _prior(synth_state_dict(KEYS["prior"], 11))
    x, style = gen(81, 2, 8192, 1, 1).cuda(), gen(82, 2, 128, 1, 1).cuda()
    t = torch.tensor([600.0, 40.0]).cuda()
    before = m(x=x, t=t, condition_input=style)
    g = torch.Generator().manual_seed(83)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.02 * torch.randn(p.shape, generator=g).to(p.device))
    after = m(x=x, t=t, condition_input=style)
    rebuilt = _prior({k: v.detach().cpu().clone() for k, v in m.state_dict().items()})(x=x, t=t, condition_input=style)
    assert not torch.equal(after, before), "the update did not change the output"
    assert torch.equal(after, rebuilt), "the re-packed model differs from one built from the updated parameters"
