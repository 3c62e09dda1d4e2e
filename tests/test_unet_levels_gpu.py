"""U-Nets deeper than the shipped four levels.  Every level's FPS, ball query, voxel preps and 3-NN search run on the
library's side stream and reach the main stream through per-level events, so the depth of a network is bounded by
nothing but its point counts.  Small PVCNN2Unets built from custom sa_blocks / fp_blocks, against the CPU oracle, and
graph-replayed against eager."""
import pytest
import torch

from oracle import net as ON
from tests.synth import synth_state_dict
from tests.util import assert_close, gen

pytestmark = pytest.mark.gpu
TOL = 5e-3      # the prior's tolerance (tests/test_net_gpu.py)
N = 2048


def _blocks(n_sa):
    """n_sa SA levels, the centres halving from N / 2, PVConvs on the first two levels; the mirrored FP stages, with
    PVConvs on the two stages that return to those levels.  Level 1's points are voxelised at two resolutions: 8 for
    its SA level, 16 for its FP stage."""
    sa = [((32, 2, 16) if i == 0 else (64, 1, 8) if i == 1 else None, (N >> (i + 1), 0.1 * 1.5 ** i, 32, (64, 64)))
          for i in range(n_sa)]
    fp = [((64, 64), (64, 1, 16) if j == n_sa - 2 else (32, 1, 16) if j == n_sa - 1 else None) for j in range(n_sa)]
    return sa, fp


@pytest.mark.parametrize("n_sa", [5, 9])
def test_deep_unet_matches_oracle_and_graph_replay(n_sa):
    from lion_b200 import _lib as L
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.latent_points_ada import PVCNN2Unet
    cfg = default_prior_cfg()
    sa, fp = _blocks(n_sa)
    net = PVCNN2Unet(4, 64, True, extra_feature_channels=1, input_dim=3, cfg=cfg, sa_blocks=sa, fp_blocks=fp)
    sd = synth_state_dict({k: list(v.shape) for k, v in net.state_dict().items()}, 21)
    net.load_state_dict(sd)
    net = net.cuda().eval()
    B = 2
    x, style = gen(61, B, 4, N), gen(62, B, cfg.latent_pts.style_dim)
    t = torch.tensor([700.0, 20.0])
    xc, tc, sc = x.cuda(), t.cuda(), style.cuda()
    eager = net(xc, t=tc, style=sc)
    with torch.no_grad():
        ref = ON.unet_forward(sd, ON.UnetSpec(4, 64, 1, sa, fp, input_dim=3), x, t=t, style=style)
    assert_close(eager, ref, TOL, "%d-level U-Net vs oracle" % n_sa)
    with L.capture_graph() as g:
        graphed = net(xc, t=tc, style=sc)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(graphed, eager), "graph replay differs from the eager forward"
