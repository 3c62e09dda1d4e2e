"""The sparse first convolution's activity mask (k_sparse_conv_gather): the gather stores only voxels with an occupied
neighbour and k_act_grid substitutes the bias-only value for the rest.  Every result must be bitwise the one of the
whole-grid route that lion_ctx_set_sparse_conv1_dense restores: the probe's grids and GroupNorm sums (the probe stores
raw1 whole but k_act_grid still substitutes), PVConv and PVCNN2Prior outputs (store skipping on) and graph-replayed
denoising steps.  The mask itself is checked against a host dilation of the occupancy grid the gather read.

Clouds: a Gaussian latent-point blob; all but a few points in one voxel with the rest in voxels on all six faces of the
grid (next to the halo); and the same plus eight points on the diagonals, as close to the corners as the normalisation
(the farthest point lands at radius r / 2) lets a point go."""
import math

import pytest
import torch
import torch.nn.functional as F

from lion_b200 import _lib as L
from tests import stage_ref as SR
from tests.test_pvconv_tail_stage_gpu import _probe
from tests.test_stage_parity_gpu import _cfg, _load
from tests.util import gen

pytestmark = pytest.mark.gpu


def _dense(on):
    L.check(L.lib().lion_ctx_set_sparse_conv1_dense(L.ctx(), 1 if on else 0), "sparse conv1 dense")


def _both(fn):
    """fn() with the activity mask (default) and with the whole-grid route"""
    try:
        _dense(True)
        ref = fn()
        _dense(False)
        got = fn()
    finally:
        _dense(False)
    return got, ref


def _faces_cloud(N, corners):
    c = torch.zeros(3, N)
    k = N - 1
    for a in range(3):
        for s in (1.0, -1.0):
            c[a, k] = s
            k -= 1
    if corners:
        d = 1.0 / math.sqrt(3.0)
        for sx in (d, -d):
            for sy in (d, -d):
                for sz in (d, -d):
                    c[:, k] = torch.tensor([sx, sy, sz])
                    k -= 1
    return c


def _clouds(B, N, seed):
    kinds = (["gauss", "faces", "corners"] * B)[:B]
    out = []
    for b, k in enumerate(kinds):
        if k == "gauss":
            out.append(SR.gaussian_cloud(seed + b, N, scale=0.2 + 0.05 * (b % 5)))
        else:
            out.append(_faces_cloud(N, k == "corners"))
    return torch.stack(out).contiguous()


def _pvconv(cin, cout, r, attn, seed=33):
    from lion_b200.models.pvcnn2_ada import PVConv
    mod, _ = _load(PVConv(cin, cout, 3, r, with_se=True, attention=attn, cfg=_cfg()), seed)
    return mod


# (cin, cout, r, N, B, attn): the first-convolution classes of a step at B = 32 (4 -> 32 is dense: its mask is null and
# nothing may change), the r = 16 one also at B = 2, an r = 32 one at B = 1, and a ragged r = 13 grid whose last mask
# word is partial
CASES = [(4, 32, 32, 2048, 32, False), (32, 32, 32, 2048, 32, False), (64, 64, 32, 2048, 32, False),
         (128, 64, 16, 1024, 32, True), (128, 64, 16, 1024, 2, True), (64, 64, 32, 2048, 1, False),
         (64, 64, 13, 500, 3, False)]


@pytest.mark.parametrize("cin,cout,r,N,B,attn", [c for c in CASES if c[0] != 4])
def test_mask_matches_occupancy(cin, cout, r, N, B, attn):
    mod = _pvconv(cin, cout, r, attn)
    m = L.model_for(mod, L.KIND_PVCONV, mod.lion_desc(), mod.lion_params())
    feats, coords = gen(70 + cin, B, cin, N).cuda(), _clouds(B, N, 5 * r).cuda()
    rp, W = r + 2, (r ** 3 + 31) // 32
    vgrid = torch.empty(B, rp, rp, rp, dtype=torch.int32, device="cuda")
    mask = torch.empty(B, W, dtype=torch.int32, device="cuda")
    L.check(L.lib().lion_pvconv_conv1_mask_probe(m.h, L.ptr(feats), L.ptr(coords), L.ptr(vgrid), L.ptr(mask), B, N, L.stream()),
            "conv1 mask probe")
    torch.cuda.synchronize()
    occ = (vgrid >= 0).float()
    assert occ[:, 0].sum() == 0 and occ[:, -1].sum() == 0 and occ[:, :, 0].sum() == 0 and occ[:, :, :, -1].sum() == 0
    act = F.max_pool3d(occ[:, None], 3, stride=1)[:, 0].reshape(B, -1) > 0      # [B, r^3], x-major, z fastest
    bits = torch.zeros(B, W * 32, dtype=torch.int64, device="cuda")
    bits[:, :r ** 3] = act.long()
    ref = (bits.view(B, W, 32) << torch.arange(32, device="cuda")).sum(-1)
    assert torch.equal(mask.long() & 0xffffffff, ref), "activity mask differs from the dilated occupancy"
    a = act.float().mean().item()
    assert 0 < a < 1, a


@pytest.mark.parametrize("cin,cout,r,N,B,attn", CASES)
def test_probe_equal(cin, cout, r, N, B, attn):
    mod = _pvconv(cin, cout, r, attn)
    m = L.model_for(mod, L.KIND_PVCONV, mod.lion_desc(), mod.lion_params())
    feats, coords, style = gen(60 + cin, B, cin, N).cuda(), _clouds(B, N, 7 * r).cuda(), gen(61, B, 128).cuda()
    got, ref = _both(lambda: _probe(m, feats, coords, style, cout, r))
    for k in ("raw1", "act1", "raw2", "rawp", "sums", "affine", "fused", "out"):
        assert torch.equal(got[k], ref[k]), "%s differs between the masked and the whole-grid route" % k


def test_probe_equal_fp16():
    """The FP16 activation grid (autocast route) substitutes h8_pack of the same bias-only value"""
    cin, cout, r, N, B = 64, 64, 32, 2048, 4
    mod = _pvconv(cin, cout, r, False)
    m = L.model_for(mod, L.KIND_PVCONV, mod.lion_desc(), mod.lion_params())
    feats, coords, style = gen(62, B, cin, N).cuda(), _clouds(B, N, 3).cuda(), gen(63, B, 128).cuda()
    rp, d = r + 2, "cuda"

    def run():
        o = [torch.empty(B, cout, r, r, r, device=d), torch.empty(B, cout, rp, rp, rp, device=d),
             torch.empty(B, cout, r, r, r, device=d), torch.empty(B, cout, N, device=d),
             torch.empty(4, B, cout, dtype=torch.float64, device=d), torch.empty(6, B, cout, device=d),
             torch.empty(B, cout, N, device=d), torch.empty(B, cout, N, device=d)]
        L.check(L.lib().lion_pvconv_probe_flags(m.h, L.ptr(feats), L.ptr(coords), L.ptr(style), *[L.ptr(t) for t in o], None,
                                                B, N, L.FWD_CONV_FP16, L.stream()), "pvconv_probe_flags")
        torch.cuda.synchronize()
        return o

    got, ref = _both(run)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a, b), "probe output %d differs under FP16" % i


@pytest.mark.parametrize("cin,cout,r,N,B,attn", [c for c in CASES if c[4] > 1])
def test_pvconv_output_equal(cin, cout, r, N, B, attn):
    """Outside probe mode the gather skips the stores of inactive voxels"""
    mod = _pvconv(cin, cout, r, attn)
    feats, coords, style = gen(64 + cin, B, cin, N).cuda(), _clouds(B, N, 11 * r).cuda(), gen(65, B, 128).cuda()
    got, ref = _both(lambda: mod((feats, coords, None, style))[0].clone())
    assert torch.equal(got, ref), "PVConv output differs between the masked and the whole-grid route"


def _prior():
    from tests.test_net_gpu import _prior as prior
    return prior()


@pytest.mark.parametrize("B", [32, 2, 1])
def test_prior_forward_equal(B):
    m = _prior()
    g = torch.Generator().manual_seed(B)
    x = (torch.randn(B, 8192, 1, 1, generator=g) * 0.5).cuda()
    style = torch.randn(B, 128, 1, 1, generator=g).cuda()
    t = torch.full((B,), 321.0).cuda()
    got, ref = _both(lambda: m(x=x, t=t, condition_input=style).clone())
    assert torch.equal(got, ref), "PVCNN2Prior output differs between the masked and the whole-grid route"


def test_graph_replayed_steps_equal():
    """10 DDPM steps of the point prior, the later ones replayed from a captured graph"""
    from lion_b200.config import default_prior_cfg
    from lion_b200.utils.diffusion_pvd import DiffusionDiscretized
    cfg = default_prior_cfg(num_steps=10)
    diff = DiffusionDiscretized(cfg.sde, None, cfg)
    diff.use_cuda_graph = True
    m, B = _prior(), 4
    style = gen(66, B, 128).view(B, 128, 1, 1).cuda()

    def run():
        torch.manual_seed(123)
        z, lst = diff.run_denoising_diffusion(m, B, [8192, 1, 1], condition_input=style)
        torch.cuda.synchronize()
        return z.clone(), [p.clone() for p in lst["pred_x"]]

    (z1, h1), (z0, h0) = _both(run)
    assert len(h1) == 10
    assert all(torch.equal(a, b) for a, b in zip(h1, h0)), "a step's latent differs between the two routes"
    assert torch.equal(z1, z0)
