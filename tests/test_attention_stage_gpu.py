"""Stage-level float64 parity of the linear attention (k_attn_ctx / k_attn_apply and the two 1x1 convolutions around
them), which the module tests see only at N = 16, 100 and 1024 through a 2e-3 tolerance.  The softmax over the points is
split into 128-point chunks whose partial contexts k_attn_apply merges with an online maximum: the cases below put a
partial chunk after full ones (N = 129, 1000), hit the 32-chunk limit (N = 4096) and its refusal (N = 4097), and place
every channel's maximum of k in the last, partial chunk at |k| up to 50.  lion_attention_probe runs the product code and
returns qkv and the pre-projection output o; each reference is built from the probe's own previous stage.

Maximum errors measured on one H100 80GB HBM3 (SXM, 700 W power limit) are listed next to each tolerance below."""
import pytest
import torch

from lion_b200 import _lib as L
from tests import stage_ref as SR
from tests.test_stage_parity_gpu import _load
from tests.util import gen

pytestmark = pytest.mark.gpu

TOL_QKV = 2e-6         # qkv against trunc(x) @ rna(W), max-abs error / max-abs reference, per shape (measured 6.2e-7)
TOL_O = 1.5e-6         # o against float64 softmax / context / apply of the probe's qkv (4.9e-7)
TOL_OUT = 3.5e-6       # output against trunc(o) @ rna(W_out) + b (1.1e-6)


def _probe(m, x, heads):
    B, C, N = x.shape
    qkv = torch.empty(B, 3 * heads * 32, N, device="cuda")
    o = torch.empty(B, heads * 32, N, device="cuda")
    out = torch.empty(B, C, N, device="cuda")
    L.check(L.lib().lion_attention_probe(m.h, L.ptr(x), L.ptr(qkv), L.ptr(o), L.ptr(out), B, N, L.stream()), "attention_probe")
    torch.cuda.synchronize()
    return qkv, o, out


def _rel(got, ref):
    """max over shapes of max |got - ref| / max |ref| (float64)."""
    return ((got.double() - ref).abs().amax((1, 2)) / ref.abs().amax((1, 2)).clamp_min(1e-300)).max().item()


def _check(mod, sd, x, heads, label):
    m = L.model_for(mod, L.KIND_ATTN, [mod.dim, mod.heads], mod.lion_params())
    qkv, o, out = _probe(m, x, heads)
    e_qkv = _rel(qkv, SR.attn_qkv(x, sd["to_qkv.weight"]))
    e_o = _rel(o, SR.attn_core(qkv, heads))
    e_out = _rel(out, SR.attn_out(o, sd["to_out.weight"], sd["to_out.bias"]))
    print("attention %s: qkv %.2e, o %.2e, out %.2e" % (label, e_qkv, e_o, e_out))
    assert e_qkv <= TOL_QKV, "qkv: %.3e > %.1e" % (e_qkv, TOL_QKV)
    assert e_o <= TOL_O, "o: %.3e > %.1e" % (e_o, TOL_O)
    assert e_out <= TOL_OUT, "output: %.3e > %.1e" % (e_out, TOL_OUT)
    assert torch.equal(mod(x), out), "probe output differs from lion_linear_attention_fwd"
    return qkv


@pytest.mark.parametrize("B", [1, 3, 32])
@pytest.mark.parametrize("N", [16, 100, 127, 128, 129, 1000, 2048, 4096])
@pytest.mark.parametrize("C,heads", [(64, 4), (128, 8)])
def test_attention_stage(C, heads, N, B):
    from lion_b200.models.pvcnn2_ada import LinearAttention
    mod, sd = _load(LinearAttention(C, heads), 35)
    _check(mod, sd, gen(70 + N, B, C, N).cuda(), heads, (C, heads, N, B))


@pytest.mark.parametrize("C,heads", [(64, 4), (128, 8)])
def test_attention_maxima_in_the_last_partial_chunk(C, heads):
    """k spans about +-50 and every channel's maximum lies in the last chunk (points 896..999 of N = 1000): the partial
    contexts of the seven full chunks are rescaled by exp(max_c - max) of about e^-20 when they are merged."""
    from lion_b200.models.pvcnn2_ada import LinearAttention
    mod, sd = _load(LinearAttention(C, heads), 36)
    B, N, tail = 3, 1000, 896
    x = gen(71, B, C, N)
    x[:, :, tail:] *= 3.0                                 # the last chunk's points carry the extremes of every channel
    wk = sd["to_qkv.weight"].reshape(3, heads * 32, C)[1].cpu().double()
    k = torch.einsum("dc,bcn->bdn", wk, x.double())
    x = (x * (50.0 / k.abs().amax().item())).cuda()
    qkv = _check(mod, sd, x, heads, (C, heads, N, B, "k up to 50"))
    k = qkv.view(B, 3, heads * 32, N)[:, 1]
    assert (k.argmax(-1) >= tail).all(), "a channel's maximum of k is not in the last chunk"
    assert 45 < k.abs().max().item() < 55 and k.min().item() < -20


def test_attention_more_than_32_chunks_is_refused():
    from lion_b200.models.pvcnn2_ada import LinearAttention
    mod, _ = _load(LinearAttention(64, 4), 35)
    m = L.model_for(mod, L.KIND_ATTN, [mod.dim, mod.heads], mod.lion_params())
    B, N = 2, 4097
    x = gen(72, B, 64, N).cuda()
    qkv = torch.full((B, 3 * 128, N), 7.0, device="cuda")
    o = torch.full((B, 128, N), 7.0, device="cuda")
    out = torch.full((B, 64, N), 7.0, device="cuda")
    rc = L.lib().lion_attention_probe(m.h, L.ptr(x), L.ptr(qkv), L.ptr(o), L.ptr(out), B, N, L.stream())
    torch.cuda.synchronize()
    assert rc != 0 and b"too large" in L.lib().lion_last_error()
    assert (qkv == 7.0).all() and (o == 7.0).all() and (out == 7.0).all(), "a refused call wrote its outputs"
    with pytest.raises(L.LionError, match="too large"):
        mod(x)
