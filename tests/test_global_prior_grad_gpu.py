"""The differentiable global prior (Prior.forward's autograd route: lion_global_prior_forward_train and
lion_global_prior_backward) at network level.

  * Gradients of F.mse_loss(prior(x), noise) -- every parameter and x -- against float64 autograd of the same network
    on the same fp32 weights (tests/gp_grad_ref.py), as a relative Frobenius error per tensor, at full size (nf 2048,
    8 cells) for PriorSEDrop with dropout masks and PriorSEClip, scalar and per-shape t, embedding_scale 1 and 1000.
  * The reduced-width golden from the unmodified reference (tests/golden/global_prior_grad.npz).
  * Twenty Adam steps on a fixed batch follow the float64 trajectory.
  * Semantics: the route's output equals lion_global_prior_forward bit for bit without dropout; backward is
    deterministic; CUDA-graph replays equal eager; gradients accumulate; retain_graph; double backward raises.

Maximum errors measured on one H100 80GB HBM3 (SXM, 700 W power limit) are listed next to each tolerance."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lion_b200 import _lib as L
from tests import gp_grad_ref as GR
from tests import stage_ref as SR
from tests.synth import synth_state_dict
from tests.test_global_prior_grad_cpu import GOLDEN, SEEDS, small_net
from tests.test_global_prior_stage_gpu import gp_inputs, gp_net
from tests.util import gen

pytestmark = pytest.mark.gpu

# Network-level errors are dominated by ReLUs whose input lies within TF32 rounding of zero: there the library and float64
# take different branches, so whole gradient entries differ and a tensor's relative Frobenius error grows with the square
# root of the fraction of flipped units, not with the rounding error.  The stage tests bound the arithmetic itself.
TOL_NET = 0.15         # full size, any tensor, relative Frobenius error against float64 autograd          (6.9e-2)
TOL_GOLDEN = 0.02      # reduced width (nf 32), against the reference's float64 gradients                  (5.3e-3)
TOL_ADAM_LOSS = 5e-3   # relative loss difference along 20 Adam steps (loss 2.97 -> 0.72)                  (1.6e-3)
TOL_ADAM_PARAM = 5e-3  # final parameters, relative Frobenius error per tensor                             (1.3e-3)

DROP = (128, 2048, 128, 8, None, 1.0)
CLIP = (128, 2048, 128, 8, 512, 1.0)
DROP_1000 = (128, 2048, 128, 8, None, 1000.0)


def masks_for(net, B, seed, p=0.1):
    g = torch.Generator().manual_seed(seed)
    keep = (torch.rand(len(net.all_modules), B, net.nf, generator=g) >= p).float()
    return (keep / (1 - p)).cuda()


def rel_fro(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1).to(a.device)
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def grads_vs_f64(net, sd, x, t, clip, noise, masks, emb, scale):
    """Library gradients and float64 autograd's; returns {name: relative Frobenius error} (dx included)."""
    B = x.shape[0]
    net.zero_grad(set_to_none=True)
    xg = x.clone().requires_grad_(True)
    out = net(xg.view(B, -1, 1, 1), t, clip_feat=clip, _drop_mask=masks).view(B, -1)
    assert out.dtype == torch.float32
    F.mse_loss(out, noise).backward()
    tt = t.expand(B) if t.dim() == 0 or t.shape[0] == 1 else t
    pe = SR.gp_posemb(tt, emb, scale).cuda()
    _, dx, g64 = GR.mse_grads({k: v.cuda() for k, v in sd.items()}, x, pe, noise, clip, masks)
    e = {"dx": rel_fro(xg.grad, dx)}
    for k, p in net.named_parameters():
        e[k] = rel_fro(p.grad, g64[k])
    return e


NET_CASES = [(DROP, 32, "vector"), (DROP, 40, "scalar"), (CLIP, 32, "vector"), (CLIP, 5, "scalar"),
             (DROP_1000, 32, "vector"), (DROP_1000, 1, "vector")]


@pytest.mark.parametrize("spec,B,tkind", NET_CASES,
                         ids=["%s-B%d-%s-s%g" % ("clip" if s[4] else "drop", B, k, s[5]) for s, B, k in NET_CASES])
def test_gradients_against_float64(spec, B, tkind):
    net, sd = gp_net(*spec, seed=71)
    net = net.cuda().train()
    x, t, clip = gp_inputs(spec, B, 300 + B)
    x, t = x.cuda(), t.cuda()
    if tkind == "scalar":
        t = t[2].clone()           # 0-dim, 500: one embedding for all shapes
    clip = clip.cuda() if clip is not None else None
    noise = gen(400 + B, B, spec[0]).cuda()
    masks = masks_for(net, B, 500 + B) if spec[4] is None else None
    e = grads_vs_f64(net, sd, x, t, clip, noise, masks, spec[2], spec[5])
    worst = max(e, key=e.get)
    print("grad %s B=%d t=%s: worst %s %.2e, dx %.2e" % (spec, B, tkind, worst, e[worst], e["dx"]), flush=True)
    assert e[worst] <= TOL_NET, "%s: relative Frobenius error %.3e > %.1e" % (worst, e[worst], TOL_NET)


@pytest.mark.parametrize("tag", ["drop", "clip"])
def test_gradients_against_reference_golden(tag):
    z = np.load(GOLDEN)
    G = GR.golden(tag, z)
    net = small_net(tag == "clip")
    sd = synth_state_dict({k: list(v.shape) for k, v in net.state_dict().items()}, SEEDS[tag])
    net.load_state_dict(sd)
    net = net.cuda().train()
    B = G["x"].shape[0]
    x = G["x"].cuda().requires_grad_(True)
    clip = G["clip"].cuda() if G["clip"] is not None else None
    masks = G["mask"].float().cuda() if G["mask"] is not None else None
    out = net(x.view(B, -1, 1, 1), G["t"].cuda(), clip_feat=clip, _drop_mask=masks).view(B, -1)
    loss = F.mse_loss(out, G["noise"].cuda())
    loss.backward()
    e = {"loss": abs(loss.item() - G["loss"]) / abs(G["loss"]), "dx": rel_fro(x.grad, G["dx"])}
    for k, p in net.named_parameters():
        e[k] = rel_fro(p.grad, G["grads"][k])
    worst = max(e, key=e.get)
    print("golden %s: worst %s %.2e" % (tag, worst, e[worst]), flush=True)
    assert e[worst] <= TOL_GOLDEN, "%s: %.3e > %.1e" % (worst, e[worst], TOL_GOLDEN)


def test_adam_follows_float64_trajectory():
    spec = (128, 512, 128, 4, None, 1.0)
    net, sd = gp_net(*spec, seed=81)
    net = net.cuda().train()
    B = 32
    x, t, _ = gp_inputs(spec, B, 82)
    x, t = x.cuda(), t.cuda()
    noise = gen(83, B, spec[0]).cuda()
    masks = masks_for(net, B, 84)
    pe = SR.gp_posemb(t, spec[2], spec[5]).cuda()
    P64 = {k: v.detach().cuda().double().requires_grad_(True) for k, v in sd.items()}
    names = [k for k, _ in net.named_parameters()]
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    opt64 = torch.optim.Adam([P64[k] for k in names], lr=1e-4)
    l32, l64 = [], []
    for _ in range(20):
        opt.zero_grad()
        loss = F.mse_loss(net(x.view(B, -1, 1, 1), t, _drop_mask=masks).view(B, -1), noise)
        loss.backward()
        opt.step()
        opt64.zero_grad()
        loss64 = F.mse_loss(GR.prior_f64(P64, x.double(), pe, None, masks.double()), noise.double())
        loss64.backward()
        opt64.step()
        l32.append(loss.item())
        l64.append(loss64.item())
    dl = max(abs(a - b) / b for a, b in zip(l32, l64))
    dp = max(rel_fro(p, P64[k]) for k, p in net.named_parameters())
    print("adam: loss %.5f -> %.5f, max relative loss difference %.2e, parameters %.2e" % (l32[0], l32[-1], dl, dp))
    assert l32[-1] < l32[0] and l64[-1] < l64[0]
    assert dl <= TOL_ADAM_LOSS and dp <= TOL_ADAM_PARAM, (dl, dp)


# ---------------------------------------------------------------------------------------------------------------------
# semantics
# ---------------------------------------------------------------------------------------------------------------------
SEM = (36, 160, 40, 2, None, 1.0)


def _small(spec=SEM, train=True):
    net, _ = gp_net(*spec, seed=91)
    return net.cuda().train(train)


def _grads(net, x, t, masks, noise):
    net.zero_grad(set_to_none=True)
    xg = x.clone().requires_grad_(True)
    B = x.shape[0]
    F.mse_loss(net(xg.view(B, -1, 1, 1), t, _drop_mask=masks).view(B, -1), noise).backward()
    return [xg.grad.clone()] + [p.grad.clone() for p in net.parameters()]


@pytest.mark.parametrize("spec,B", [(SEM, 3), (DROP, 40), (CLIP, 32)])
def test_route_output_is_the_eval_forward(spec, B):
    """Without dropout (eval(), or PriorSEClip) the differentiable route gives lion_global_prior_forward's bits; so does
    a no-grad call in train() mode."""
    net, _ = gp_net(*spec, seed=92)
    net = net.cuda()
    x, t, clip = gp_inputs(spec, B, 93)
    x, t = x.cuda(), t.cuda()
    clip = clip.cuda() if clip is not None else None
    m = L.model_for(net, L.KIND_GLOBAL_PRIOR, net.lion_desc(), net.lion_params())
    ref = torch.empty_like(x)
    L.check(L.lib().lion_global_prior_forward(m.h, L.ptr(x), L.ptr(t), L.ptr(clip), L.ptr(ref), B, L.stream()), "fwd")
    xg = x.clone().requires_grad_(True)
    for mode in (False, True):
        net.train(mode)
        if mode and spec[4] is None:
            with torch.no_grad():
                out = net(x.view(B, -1, 1, 1), t, clip_feat=clip).view(B, -1)
        else:
            out = net(xg.view(B, -1, 1, 1), t, clip_feat=clip).view(B, -1)
            assert out.grad_fn is not None
        assert torch.equal(out, ref), "train=%s" % mode


def test_dropout_masks_drawn_in_train_mode():
    """train() with dropout p: each cell's conv1 output is kept with probability 1 - p and scaled by 1 / (1 - p)."""
    net = _small()
    B = 64
    drop = net._drop_masks(B, torch.device("cuda"))
    p = net.all_modules[0].dropout_ratio
    assert drop.shape == (len(net.all_modules), B, net.nf)
    vals = set(torch.unique(drop).tolist())
    assert vals <= {0.0, float(np.float32(1.0 / (1.0 - p)))}
    assert abs((drop == 0).float().mean().item() - p) < 0.02
    assert net.eval()._drop_masks(B, torch.device("cuda")) is None


def test_backward_deterministic_and_accumulates():
    net = _small()
    B = 33
    x, t, _ = gp_inputs(SEM, B, 94)
    x, t = x.cuda(), t.cuda()
    noise = gen(95, B, SEM[0]).cuda()
    masks = masks_for(net, B, 96)
    g1 = _grads(net, x, t, masks, noise)
    g2 = _grads(net, x, t, masks, noise)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2)), "two backward passes differ"
    # two backward() calls through one graph (retain_graph): .grad holds twice the gradient
    net.zero_grad(set_to_none=True)
    out = net(x.view(B, -1, 1, 1), t, _drop_mask=masks).view(B, -1)
    loss = F.mse_loss(out, noise)
    loss.backward(retain_graph=True)
    loss.backward()
    assert all(torch.equal(p.grad, 2 * g) for p, g in zip(net.parameters(), g1[1:]))


def test_eval_module_on_plain_input_returns_plain_tensor():
    """Sampling code calls an eval() module with grad mode on: parameters requiring grad do not make the output an
    autograd node unless x requires grad."""
    net = _small(train=False)
    x, t, _ = gp_inputs(SEM, 2, 101)
    out = net(x.cuda().view(2, -1, 1, 1), t.cuda())
    assert out.grad_fn is None and not out.requires_grad


def test_double_backward_raises():
    net = _small()
    x, t, _ = gp_inputs(SEM, 2, 97)
    x = x.cuda().requires_grad_(True)
    out = net(x.view(2, -1, 1, 1), t.cuda())
    with pytest.raises(L.LionError, match="double backward"):
        torch.autograd.grad(out.square().sum(), x, create_graph=True)


def test_graph_capture_replays_equal_eager():
    net = _small()
    B = 5
    x, t, _ = gp_inputs(SEM, B, 98)
    x, t = x.cuda(), t.cuda()
    noise = gen(99, B, SEM[0]).cuda()
    masks = masks_for(net, B, 100)
    params = list(net.parameters())

    def step():
        out = net(x.view(B, -1, 1, 1), t, _drop_mask=masks).view(B, -1)
        return torch.autograd.grad(F.mse_loss(out, noise), params)

    eager = step()          # also sizes the scratch arena outside the capture
    torch.cuda.synchronize()
    with L.capture_graph() as g:
        cap = step()
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(cap, eager)), "graph replay differs from eager"
