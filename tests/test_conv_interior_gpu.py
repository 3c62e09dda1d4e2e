"""The 3x3x3 tensor-core convolution on interior 8x8 voxel blocks (csrc/conv_tc.cu): every shape class of the prior
step at B = 32 and ragged ones, against cuDNN; GroupNorm sums; bit-reproducibility; the occupancy skip of a dense first
convolution on a sparse scatter grid."""
import pytest
import torch

from oracle import net as ON
from tests.synth import synth_state_dict
from tests.util import assert_close, gen

pytestmark = pytest.mark.gpu

SHAPES = [  # (cin, cout, r, B)
    (4, 32, 32, 32), (32, 32, 32, 32), (64, 64, 32, 32), (128, 64, 16, 32), (64, 64, 16, 32), (128, 128, 16, 32),
    (192, 128, 8, 32), (128, 128, 8, 32),
    (4, 32, 16, 1), (36, 64, 8, 3), (192, 128, 16, 3), (64, 256, 8, 3), (36, 32, 32, 1),
    (36, 32, 12, 3), (4, 64, 5, 1), (64, 128, 13, 2),      # r not a multiple of 8: partial last blocks
]


def _tf32_rna(x):
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1fff).view(torch.float32)


@pytest.mark.parametrize("cin,cout,r,B", SHAPES)
def test_interior_conv_vs_cudnn(cin, cout, r, B):
    from lion_b200.models.pvcnn2_ada import Conv3d
    m = Conv3d(cin, cout, 3, stride=1, padding=1)
    w, b = gen(71, cout, cin, 3, 3, 3, scale=(27 * cin) ** -0.5), gen(72, cout, scale=0.1)
    m.load_state_dict({"weight": w, "bias": b})
    m = m.cuda().eval()
    x = gen(73, B, cin, r, r, r).cuda()
    out, ssum, ssq = m(x, return_gn_stats=True)
    old_cudnn, old_mm = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cudnn.allow_tf32 = False
        ref_t = torch.nn.functional.conv3d(_tf32_rna(x.cpu()).cuda(), _tf32_rna(w).cuda(), b.cuda(), padding=1)
        ref = torch.nn.functional.conv3d(x, w.cuda(), b.cuda(), padding=1)
    finally:
        torch.backends.cudnn.allow_tf32 = old_cudnn
        torch.backends.cuda.matmul.allow_tf32 = old_mm
    assert_close(out, ref_t, 2e-5, "conv3d vs fp32 cuDNN on TF32-rounded operands")
    assert_close(out, ref, 2e-3, "conv3d vs fp32 conv3d")
    o64 = out.double().view(B, cout, -1)
    assert_close(ssum, o64.sum(-1), 1e-5, "fused GroupNorm sum")
    assert_close(ssq, (o64 * o64).sum(-1), 1e-5, "fused GroupNorm sum of squares")
    out2, ssum2, ssq2 = m(x, return_gn_stats=True)
    assert torch.equal(out2, out) and torch.equal(ssum2, ssum) and torch.equal(ssq2, ssq), "not bit-reproducible"


@pytest.mark.parametrize("cin,cout,r,N", [(64, 64, 16, 2048), (32, 32, 8, 200), (192, 128, 8, 300)])
def test_dense_first_conv_on_sparse_grid(cin, cout, r, N):
    """N * 4 > r^3 keeps the dense first convolution, which skips the operand windows whose 64-row occupancy flags
    are all clear (the empty x-planes and corners of the scatter grid)"""
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.pvcnn2_ada import PVConv
    assert N * 4 > r ** 3
    mod = PVConv(cin, cout, 3, r, with_se=True, attention=False, cfg=default_prior_cfg())
    sd = synth_state_dict({k: list(v.shape) for k, v in mod.state_dict().items()}, 31)
    mod.load_state_dict(sd)
    mod = mod.cuda().eval()
    B = 2
    feats, coords, style = gen(74, B, cin, N), gen(75, B, 3, N, scale=0.4), gen(76, B, 128)
    out, *_ = mod((feats.cuda(), coords.cuda(), None, style.cuda()))
    blk = dict(kind="pvconv", cin=cin, cout=cout, r=r, attn=False)
    assert_close(out, ON.pvconv(sd, "", blk, feats, coords, style), 2e-3, "PVConv on a sparse grid")
    out2, *_ = mod((feats.cuda(), coords.cuda(), None, style.cuda()))
    assert torch.equal(out2, out), "PVConv is not bit-reproducible"
