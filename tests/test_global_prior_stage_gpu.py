"""Stage-level parity of the global prior (csrc/global_prior.cu), which the network tests see only through whole-network
tolerances: the positional embedding (k_gp_posemb), every split-K Linear (k_gp_partial, TF32 mma.sync over K slices of
256, and k_gp_reduce with its fused bias / ReLU / sigmoid, SE gate and residual add).  lion_global_prior_probe runs
lion_global_prior_forward and copies out each Linear's output; each layer's float64 reference (tests/stage_ref.py) is
built from the probe's own recorded input, with the kernel's operand model: activations cvt.rna of fl32(x + add),
weights truncated (staged unrounded and read by the tensor core as fp32 bits).

The models reach the sampling shape (B = 32, one 32-shape chunk), chunks past the first, the CLIP cell's conv1 at
K = 4096 (16 K slices, the limit), partial output blocks and partial 64-column groups (O and K not multiples of 128 and
64), and an embedding wider than the 64 threads k_gp_posemb is launched with.

Maximum errors measured on one H100 80GB HBM3 (SXM, 700 W power limit) are listed next to each tolerance below.  A
Linear's error is |got - ref| / (|W~| |x~| + |b|) elementwise, W~ and x~ the modelled operands; the cell output's is
|got - ref| / (|gate bb| + |h|).  With the operand model swapped (weights rna, activations truncated) the same cases
measure at least 5.0e-5 on a Linear and 2.4e-4 on a cell output, so the tolerances tell the two models apart."""
import ctypes as C
import functools

import pytest
import torch

from lion_b200 import _lib as L
from tests import stage_ref as SR
from tests.synth import synth_state_dict
from tests.util import gen, rel_err

pytestmark = pytest.mark.gpu

TOL_EMB = 2.3e-7     # embedding, max-abs error (arguments up to 1e6 rad)                                 (7.8e-8)
TOL_LINEAR = 9.5e-7  # every Linear, error over |W~| |x~| + |b|                                              (3.2e-7)
TOL_CELL = 3.8e-6    # cell output sigmoid(fc2) bb + h, error over |gate bb| + |h|                          (1.3e-6)
# output against the float64 model run from x on its own activations, max-abs error / max-abs reference per shape: a
# wiring check.  The two chains' activations differ by fp32 rounding, and where that moves a value across a TF32
# rounding boundary the operands differ by a TF32 ulp, so this is far above the per-layer errors             (5.0e-4)
TOL_FREE = 1.5e-3
TIMES = [0.0, 1.0, 500.0, 999.0, 1000.0]

# (D, nf, emb, cells, clip_dim or None, embedding_scale)
DEFAULT = (128, 2048, 128, 8, None, 1.0)
CLIP = (128, 2048, 128, 8, 512, 1.0)
RAGGED = (36, 160, 40, 2, None, 1.0)         # O in {36, 160, 20}, K in {36, 40, 160, 20}: partial blocks and groups
RAGGED_CLIP = (36, 160, 40, 2, 36, 1.0)      # conv1 at K = 320: a second K slice of 64
WIDE = (128, 512, 256, 2, None, 1000.0)      # half = 128 frequencies; arguments up to 1e6 rad


def gp_net(D, nf, emb, cells, clip_dim=None, scale=1.0, seed=61):
    """PriorSEDrop / PriorSEClip built from default_prior_cfg() with the sde fields changed, synthetic weights of its own
    shapes.  Returns (module on the CPU, state dict)."""
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.score_sde.resnet import PriorSEClip, PriorSEDrop
    cfg = default_prior_cfg(clip=clip_dim is not None)
    cfg.sde.num_channels_dae, cfg.sde.embedding_dim, cfg.sde.num_cell_per_scale_dae = nf, emb, cells
    cfg.sde.embedding_scale = scale
    if clip_dim is not None:
        cfg.clipforge.feat_dim = clip_dim
    net = (PriorSEDrop if clip_dim is None else PriorSEClip)(cfg.sde, D, cfg)
    sd = synth_state_dict({k: list(v.shape) for k, v in net.state_dict().items()}, seed)
    net.load_state_dict(sd)
    return net.eval(), sd


@functools.lru_cache(maxsize=1)
def _net(spec):
    net, sd = gp_net(*spec)
    return net.cuda(), {k: v.cuda() for k, v in sd.items()}


def gp_inputs(spec, B, seed):
    """x [B, D], t (TIMES, then seeded integers in [1, 1000]), clip [B, clip_dim] or None, on the CPU."""
    D, clip_dim = spec[0], spec[4]
    g = torch.Generator().manual_seed(seed)
    t = torch.tensor(TIMES[:B] + torch.randint(1, 1001, (max(B - len(TIMES), 0),), generator=g).float().tolist())
    x = gen(seed + 1, B, D)
    clip = gen(seed + 2, B, clip_dim) if clip_dim is not None else None
    return x, t, clip


def _forward(net, x, t, clip):
    B = x.shape[0]
    return net(x.view(B, -1, 1, 1), t, clip_feat=clip).view(B, -1)


def _probe(net, x, t, clip):
    D, nf, emb, cells = net.lion_desc()[:4]
    B = x.shape[0]
    d = "cuda"
    P = {"pe": torch.empty(B, emb, device=d), "t0": torch.empty(B, 4 * emb, device=d), "temb": torch.empty(B, nf, device=d),
         "cmap": torch.empty(B, nf, device=d) if clip is not None else None, "h0": torch.empty(B, nf, device=d),
         "out": torch.empty(B, D, device=d)}
    taps = [P[k] for k in ("pe", "t0", "temb", "cmap", "h0")]
    for n, w in (("a", nf), ("bb", nf), ("s", nf // 8), ("h", nf)):
        P[n] = [torch.empty(B, w, device=d) for _ in range(cells)]
    for k in range(cells):
        taps += [P[n][k] for n in ("a", "bb", "s", "h")]
    arr = (C.c_void_p * len(taps))(*[None if p is None else p.data_ptr() for p in taps])
    m = L.model_for(net, L.KIND_GLOBAL_PRIOR, net.lion_desc(), net.lion_params())
    L.check(L.lib().lion_global_prior_probe(m.h, L.ptr(x), L.ptr(t), L.ptr(clip), L.ptr(P["out"]), arr, len(taps), B,
                                            L.stream()), "global_prior_probe")
    torch.cuda.synchronize()
    return P


def _lin_err(got, ref_bound):
    ref, bound = ref_bound
    return ((got.double() - ref) / bound.clamp_min(1e-30)).abs().max().item()


def layer_errors(P, sd, x, t, clip, emb, scale):
    """Per-layer errors of a probe record, each layer's reference from the probe's own input."""
    relu = lambda rb: (torch.relu(rb[0]), rb[1])
    e = {"emb": (P["pe"].double() - SR.gp_posemb(t, emb, scale).cuda()).abs().max().item()}
    e["t0"] = _lin_err(P["t0"], SR.gp_linear_f64(P["pe"], sd["temb_layer.0.weight"], sd["temb_layer.0.bias"]))
    e["temb"] = _lin_err(P["temb"], SR.gp_linear_f64(P["t0"], sd["temb_layer.1.weight"], sd["temb_layer.1.bias"]))
    if clip is not None:
        e["cmap"] = _lin_err(P["cmap"], SR.gp_linear_f64(clip, sd["clip_feat_mapping.weight"], sd["clip_feat_mapping.bias"]))
    e["h0"] = _lin_err(P["h0"], SR.gp_linear_f64(x, sd["input_layer.weight"], sd["input_layer.bias"]))
    for n in ("conv1", "conv2", "se0", "cell"):
        e[n] = 0.0
    h = P["h0"]
    for k in range(len(P["a"])):
        p = "all_modules.%d." % k
        a, bb, s = P["a"][k], P["bb"][k], P["s"][k]
        e["conv1"] = max(e["conv1"], _lin_err(a, relu(SR.gp_conv1_f64(h, P["temb"], P["cmap"], sd[p + "conv1.weight"],
                                                                      sd[p + "conv1.bias"]))))
        e["conv2"] = max(e["conv2"], _lin_err(bb, relu(SR.gp_linear_f64(a, sd[p + "conv2.weight"], sd[p + "conv2.bias"]))))
        e["se0"] = max(e["se0"], _lin_err(s, relu(SR.gp_linear_f64(bb, sd[p + "SE.fc.0.weight"], None))))
        e["cell"] = max(e["cell"], _lin_err(P["h"][k], SR.gp_cell_out(s, sd[p + "SE.fc.2.weight"], bb, h)))
        h = P["h"][k]
    e["out"] = _lin_err(P["out"], SR.gp_linear_f64(h, sd["output_layer.weight"], sd["output_layer.bias"]))
    return e


CASES = ([(DEFAULT, B) for B in (1, 5, 32, 33, 64)] + [(CLIP, B) for B in (3, 32, 40)] +
         [(RAGGED, B) for B in (1, 33)] + [(RAGGED_CLIP, B) for B in (1, 33)] + [(WIDE, B) for B in (2, 32)])


@pytest.mark.parametrize("spec,B", CASES, ids=["%s-B%d" % ("x".join(str(v) for v in s[:5]), B) for s, B in CASES])
def test_global_prior_stages(spec, B):
    net, sd = _net(spec)
    D, nf, emb, cells, clip_dim, scale = spec
    x, t, clip = gp_inputs(spec, B, 100 + B)
    x, t = x.cuda(), t.cuda()
    clip = clip.cuda() if clip is not None else None
    before = _forward(net, x, t, clip)
    P = _probe(net, x, t, clip)
    after = _forward(net, x, t, clip)

    # the probe computes what lion_global_prior_forward computes, and leaves it as it was; run to run, the same bits
    assert torch.equal(P["out"], before), "probe output differs from lion_global_prior_forward"
    assert torch.equal(after, before), "forward after the probe differs from the forward before it"
    again = _probe(net, x, t, clip)
    for k in ("pe", "t0", "temb", "h0", "out"):
        assert torch.equal(again[k], P[k]), "%s differs run to run" % k
    for n in ("a", "bb", "s", "h"):
        assert all(torch.equal(u, v) for u, v in zip(again[n], P[n])), "%s differs run to run" % n

    e = layer_errors(P, sd, x, t, clip, emb, scale)
    free = SR.gp_forward_f64(sd, x, t, clip, emb, scale)
    e["free"] = max(rel_err(P["out"][b], free["out"][b]) for b in range(B))
    print("global prior %s B=%d: %s" % (spec, B, ", ".join("%s %.2e" % kv for kv in e.items())), flush=True)
    assert e["emb"] <= TOL_EMB, "embedding: %.3e > %.1e" % (e["emb"], TOL_EMB)
    for n in ("t0", "temb", "cmap", "h0", "conv1", "conv2", "se0", "out"):
        if n in e:
            assert e[n] <= TOL_LINEAR, "%s: %.3e > %.1e" % (n, e[n], TOL_LINEAR)
    assert e["cell"] <= TOL_CELL, "cell output: %.3e > %.1e" % (e["cell"], TOL_CELL)
    assert e["free"] <= TOL_FREE, "output against the float64 model: %.3e > %.1e" % (e["free"], TOL_FREE)

    # every shape alone gives the bits of its row in the batch (rows past the first 32-shape chunk included)
    if B > 1:
        for b in range(B):
            one = _forward(net, x[b:b + 1], t[b:b + 1], None if clip is None else clip[b:b + 1])
            assert torch.equal(one, before[b:b + 1]), "row %d alone differs from its row in the batch of %d" % (b, B)


@pytest.mark.parametrize("spec,what", [((130, 160, 40, 1, None, 1.0), "K=130 must be a multiple of 4"),
                                       ((128, 2080, 128, 1, 512, 1.0), "K=4160 needs 17 K slices of 256, at most 16")])
def test_global_prior_refuses(spec, what):
    """A K that is not a multiple of 4 (D = 130), and a CLIP conv1 past 16 K slices (K = 2 nf = 4160), are refused with
    an error naming the limit, before anything is written to the output."""
    net, _ = _net(spec)
    x, t, clip = gp_inputs(spec, 2, 7)
    x, t = x.cuda(), t.cuda()
    clip = clip.cuda() if clip is not None else None
    out = torch.full((2, spec[0]), 1234.5, device="cuda")
    m = L.model_for(net, L.KIND_GLOBAL_PRIOR, net.lion_desc(), net.lion_params())
    with pytest.raises(L.LionError, match=what):
        L.check(L.lib().lion_global_prior_forward(m.h, L.ptr(x), L.ptr(t), L.ptr(clip), L.ptr(out), 2, L.stream()),
                "global_prior_forward")
    torch.cuda.synchronize()
    assert (out == 1234.5).all(), "a refused forward wrote to its output"
