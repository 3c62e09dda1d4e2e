"""3x3x3 weight slabs streamed in 3-tap parts (csrc/conv_tc.cu): every 3x3x3 shape class of the prior's step, ragged
grids and a sparse-input first convolution with occupancy skips compute bitwise the same outputs and GroupNorm sums
whether the slabs are streamed whole or in parts, and conv_tc_run takes the mode that test_conv_weight_parts_cpu.py
restates."""
import pytest
import torch

from lion_b200 import _lib as L
from tests.synth import synth_state_dict
from tests.test_conv_weight_parts_cpu import expected_taps
from tests.util import gen

pytestmark = pytest.mark.gpu


def _taps():
    return L.lib().lion_ctx_last_conv_stage_taps(L.ctx())


def _whole(on):
    L.check(L.lib().lion_ctx_set_conv_whole_slabs(L.ctx(), 1 if on else 0), "whole slabs")


@pytest.mark.parametrize("cin,cout,r,B", [
    (4, 32, 32, 32), (32, 32, 32, 32), (128, 64, 16, 32), (64, 64, 16, 32), (192, 128, 8, 32), (128, 128, 8, 32),
    (128, 128, 16, 32), (64, 64, 32, 32),
    (64, 64, 13, 3), (128, 128, 13, 3), (64, 128, 13, 32), (32, 32, 13, 3)])
def test_parts_equal_whole_slabs(cin, cout, r, B):
    from lion_b200.models.pvcnn2_ada import Conv3d
    m = Conv3d(cin, cout, 3, stride=1, padding=1)
    m.load_state_dict({"weight": gen(91, cout, cin, 3, 3, 3, scale=(27 * cin) ** -0.5), "bias": gen(92, cout, scale=0.1)})
    m = m.cuda().eval()
    x = gen(93, B, cin, r, r, r).cuda()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    try:
        _whole(True)
        ref = m(x, return_gn_stats=True)
        assert _taps() == 9
        _whole(False)
        got = m(x, return_gn_stats=True)
        assert _taps() == expected_taps(cin, cout, r, B, sms)
    finally:
        _whole(False)
    for a, b, name in zip(got, ref, ("out", "ssum", "ssq")):
        assert torch.equal(a, b), "%s differs between 3-tap parts and whole weight slabs" % name


@pytest.mark.parametrize("cin,cout,r,N", [(64, 64, 16, 2048), (192, 128, 8, 300)])
def test_sparse_first_conv_with_occupancy_skips_equal(cin, cout, r, N):
    """N * 4 > r^3 keeps the dense first convolution, which skips operand windows whose occupancy flags are clear (on
    128 channels with its weight slabs in 3-tap parts)"""
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.pvcnn2_ada import PVConv
    mod = PVConv(cin, cout, 3, r, with_se=True, attention=False, cfg=default_prior_cfg())
    sd = synth_state_dict({k: list(v.shape) for k, v in mod.state_dict().items()}, 41)
    mod.load_state_dict(sd)
    mod = mod.cuda().eval()
    B = 3
    feats, coords, style = gen(94, B, cin, N).cuda(), gen(95, B, 3, N, scale=0.4).cuda(), gen(96, B, 128).cuda()
    try:
        _whole(True)
        ref, *_ = mod((feats, coords, None, style))
        _whole(False)
        got, *_ = mod((feats, coords, None, style))
        # the block's last convolution, cout -> cout (the 128-channel grid streams its slabs in parts)
        assert _taps() == expected_taps(cout, cout, r, B, torch.cuda.get_device_properties(0).multi_processor_count)
    finally:
        _whole(False)
    assert torch.equal(got, ref), "PVConv output differs between 3-tap parts and whole weight slabs"
