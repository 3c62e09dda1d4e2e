"""4-block groups of the 128-channel 3x3x3 convolution (csrc/conv_tc.cu): a batch large enough to give every SM a
4-block group computes every shape bitwise like a single-shape call, which takes 2-block groups.  Each output's sum
order does not depend on the batch, so any reordering of the accumulation fails this test."""
import pytest
import torch

from lion_b200 import _lib as L
from tests.util import gen

pytestmark = pytest.mark.gpu


def _last_group():
    return L.lib().lion_ctx_last_conv_group(L.ctx())


@pytest.mark.parametrize("cin,cout,r", [(128, 128, 16), (64, 128, 13)])
def test_four_block_groups_equal_two_block_groups(cin, cout, r):
    from lion_b200.models.pvcnn2_ada import Conv3d
    m = Conv3d(cin, cout, 3, stride=1, padding=1)
    m.load_state_dict({"weight": gen(81, cout, cin, 3, 3, 3, scale=(27 * cin) ** -0.5), "bias": gen(82, cout, scale=0.1)})
    m = m.cuda().eval()
    B = 32
    x = gen(83, B, cin, r, r, r).cuda()
    out, _, _ = m(x, return_gn_stats=True)
    assert _last_group() == 4, "B = 32 should take 4-block groups"
    for b in range(B):
        one, _, _ = m(x[b:b + 1].contiguous(), return_gn_stats=True)
        assert _last_group() == 2, "B = 1 should take 2-block groups"
        assert torch.equal(one[0], out[b]), "shape %d differs between 4-block and 2-block groups" % b
