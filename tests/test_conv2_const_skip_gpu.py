"""Class-valued blocks of the second 3x3x3 convolution of a PVConv (k_conv2_flags, conv_tc.cu: Params::cls_flag).  After a
sparse first convolution the activation grid holds one value per (shape, channel) at every inactive voxel, and the row
tiles' 64-row blocks none of whose rows has an active neighbour take their outputs and GroupNorm sums from the 27
border-class values instead of being computed.  Every result must be bitwise the one of lion_ctx_set_conv2_class_mode(1),
which computes every block: the probe's grids (the probe stores the skipped rows) and GroupNorm sums, the FP16 route,
PVConv and PVCNN2Prior outputs and graph-replayed denoising steps.  Outside probe mode the skipped rows are not stored:
mode 2 fills the output grid with NaNs first, and the result must not change.  The flagged-block count is checked
against a dilation of the occupancy grid.

Clouds (tests/test_sparse_conv1_mask_gpu.py): a Gaussian latent-point blob; all but a few points in one voxel with the
rest on all six faces of the grid; the same plus points towards the eight corners.  Grids: r = 32 (32 and 64 channels),
an r = 16 layer and a ragged r = 13 one."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from lion_b200 import _lib as L
from tests.test_pvconv_tail_stage_gpu import _probe
from tests.test_sparse_conv1_mask_gpu import _clouds, _pvconv
from tests.util import gen

pytestmark = pytest.mark.gpu


def _mode(m):
    L.check(L.lib().lion_ctx_set_conv2_class_mode(L.ctx(), m), "conv2 class mode")


def _both(fn, mode=0):
    """fn() with class-valued blocks skipped (mode 0, or 2: output grid poisoned first) and with every block computed"""
    try:
        _mode(1)
        ref = fn()
        _mode(mode)
        got = fn()
    finally:
        _mode(0)
    return got, ref


def _counts():
    n, t = C.c_longlong(-1), C.c_longlong(-1)
    L.check(L.lib().lion_ctx_last_conv2_class_blocks(L.ctx(), C.byref(n), C.byref(t)), "conv2 class blocks")
    return n.value, t.value


# (cin, cout, r, N, B, attn): the second convolutions after a sparse first one at B = 32, the r = 16 one also at B = 2,
# an r = 32 one at B = 1, and a ragged r = 13 grid
CASES = [(32, 32, 32, 2048, 32, False), (64, 64, 32, 2048, 32, False), (128, 64, 16, 1024, 32, True),
         (128, 64, 16, 1024, 2, True), (64, 64, 32, 2048, 1, False), (64, 64, 13, 500, 3, False)]


@pytest.mark.parametrize("cin,cout,r,N,B,attn", CASES)
def test_probe_equal(cin, cout, r, N, B, attn):
    mod = _pvconv(cin, cout, r, attn)
    m = L.model_for(mod, L.KIND_PVCONV, mod.lion_desc(), mod.lion_params())
    feats, coords, style = gen(80 + cin, B, cin, N).cuda(), _clouds(B, N, 13 * r).cuda(), gen(81, B, 128).cuda()
    got, ref = _both(lambda: _probe(m, feats, coords, style, cout, r))
    n, t = _counts()
    assert 0 < n < t, (n, t)
    for k in ("raw1", "act1", "raw2", "rawp", "sums", "affine", "fused", "out"):
        assert torch.equal(got[k], ref[k]), "%s differs between skipped and computed class-valued blocks" % k
    assert not torch.isnan(got["raw2"]).any()


@pytest.mark.parametrize("cin,cout,r,N,B,attn", CASES)
def test_flag_count_matches_dilation(cin, cout, r, N, B, attn):
    """flagged blocks = 64-row blocks of the row tiles' span with no interior row within two voxels of an occupied one"""
    mod = _pvconv(cin, cout, r, attn)
    m = L.model_for(mod, L.KIND_PVCONV, mod.lion_desc(), mod.lion_params())
    feats, coords = gen(82 + cin, B, cin, N).cuda(), _clouds(B, N, 17 * r).cuda()
    rp = r + 2
    vgrid = torch.empty(B, rp, rp, rp, dtype=torch.int32, device="cuda")
    mask = torch.empty(B, (r ** 3 + 31) // 32, dtype=torch.int32, device="cuda")
    L.check(L.lib().lion_pvconv_conv1_mask_probe(m.h, L.ptr(feats), L.ptr(coords), L.ptr(vgrid), L.ptr(mask), B, N, L.stream()),
            "conv1 mask probe")
    style = gen(83, B, 128).cuda()
    mod((feats, coords, None, style))
    n, t = _counts()
    occ = (vgrid >= 0).float()[:, None]
    near = F.max_pool3d(occ, 5, stride=1, padding=2)[:, 0] > 0               # within two voxels of an occupied one
    inner = torch.zeros(rp, rp, rp, dtype=torch.bool, device="cuda")
    inner[1:-1, 1:-1, 1:-1] = True
    busy = (near & inner).reshape(B, -1)[:, rp * rp:(rp - 1) * rp * rp]      # the row tiles' span, x-major rows
    nblk = 2 * -(-busy.shape[1] // 128)
    pad = torch.zeros(B, nblk * 64, dtype=torch.bool, device="cuda")
    pad[:, :busy.shape[1]] = busy
    want = int((~pad.view(B, nblk, 64).any(-1)).sum().item())
    assert t == B * nblk and n == want, (n, want, t)


def test_probe_equal_fp16():
    """FP16 activation grid (autocast route): the class grid takes h8_pack of the same inactive value"""
    cin, cout, r, N, B = 64, 64, 32, 2048, 4
    mod = _pvconv(cin, cout, r, False)
    m = L.model_for(mod, L.KIND_PVCONV, mod.lion_desc(), mod.lion_params())
    feats, coords, style = gen(84, B, cin, N).cuda(), _clouds(B, N, 9).cuda(), gen(85, B, 128).cuda()
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
    assert _counts()[0] > 0
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a, b), "probe output %d differs under FP16" % i


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("cin,cout,r,N,B,attn", [c for c in CASES if c[4] > 1])
def test_pvconv_output_equal(cin, cout, r, N, B, attn, mode):
    """Outside probe mode the skipped rows are not stored; mode 2 leaves them NaN, and no reader may see one"""
    mod = _pvconv(cin, cout, r, attn)
    feats, coords, style = gen(86 + cin, B, cin, N).cuda(), _clouds(B, N, 19 * r).cuda(), gen(87, B, 128).cuda()
    got, ref = _both(lambda: mod((feats, coords, None, style))[0].clone(), mode)
    assert torch.equal(got, ref), "PVConv output differs between skipped and computed class-valued blocks"


def _prior():
    from tests.test_net_gpu import _prior as prior
    return prior()


@pytest.mark.parametrize("B", [32, 2, 1])
def test_prior_forward_equal(B):
    m = _prior()
    g = torch.Generator().manual_seed(100 + B)
    x = torch.randn(B, 8192, 1, 1, generator=g).cuda()
    style = torch.randn(B, 128, 1, 1, generator=g).cuda()
    t = torch.full((B,), 999.0).cuda()
    got, ref = _both(lambda: m(x=x, t=t, condition_input=style).clone(), 2)
    assert torch.equal(got, ref), "PVCNN2Prior output differs between skipped and computed class-valued blocks"


def test_graph_replayed_steps_equal():
    """10 DDPM steps of the point prior, the later ones replayed from a captured graph"""
    from lion_b200.config import default_prior_cfg
    from lion_b200.utils.diffusion_pvd import DiffusionDiscretized
    cfg = default_prior_cfg(num_steps=10)
    diff = DiffusionDiscretized(cfg.sde, None, cfg)
    diff.use_cuda_graph = True
    m, B = _prior(), 4
    style = gen(88, B, 128).view(B, 128, 1, 1).cuda()

    def run():
        torch.manual_seed(321)
        z, lst = diff.run_denoising_diffusion(m, B, [8192, 1, 1], condition_input=style)
        torch.cuda.synchronize()
        return z.clone(), [p.clone() for p in lst["pred_x"]]

    (z1, h1), (z0, h0) = _both(run)
    assert len(h1) == 10
    assert all(torch.equal(a, b) for a, b in zip(h1, h0)), "a step's latent differs between the two routes"
    assert torch.equal(z1, z0)
