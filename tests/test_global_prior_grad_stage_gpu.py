"""Stage-level parity of the global prior's backward (csrc/global_prior.cu): every Linear's dgrad (k_gpb_dgrad, TF32
mma.sync over slices of 256 outputs, and k_gpb_reduce with the elementwise backward in its epilogue) and wgrad
(k_gpb_wgrad, fp32 FFMA over the shapes).  lion_global_prior_forward_train records each Linear's input in the saved
buffer, lion_global_prior_backward_probe copies out the gradient between each pair of Linears; each stage's float64
reference is built from those recorded tensors, with the kernels' operand models:
  * dgrad: the gradient rounded with cvt.rna, the weights truncated (staged unrounded, read as fp32 bits);
  * wgrad: the gradient exact (fp32), the forward operand as the forward consumed it, cvt.rna of fl32(x + add).
A dgrad's error is |got - ref| / (|W~| |g~| + the magnitude of the elementwise terms), a wgrad's |got - ref| / (|g|^T |x~|),
elementwise.  The same comparison of every cell's conv2 with the dgrad operand model swapped (gradient truncated, weights rounded)
or with the wgrad operand unrounded is asserted to fail the tolerance, so the tolerances tell the models apart.

Cases: the sampling shape (B = 32), a second 32-shape chunk (B = 40), B = 1 and 5, the CLIP conv1 at K = 4096, and
ragged widths (O and K not multiples of the 256-row slices and 128-column tiles).
Maximum errors measured on one H100 80GB HBM3 (SXM, 700 W power limit) are listed next to each tolerance."""
import ctypes as C

import pytest
import torch

from lion_b200 import _lib as L
from tests import stage_ref as SR
from tests.test_global_prior_stage_gpu import gp_inputs, gp_net
from tests.util import gen

pytestmark = pytest.mark.gpu

TOL_DGRAD = 9.5e-7   # every dgrad and its epilogue, over the bound above    (5.0e-7; swapped model >= 7.9e-5)
TOL_WGRAD = 9.5e-7   # every weight and bias gradient, over |g|^T |x~|       (3.3e-7; unrounded x >= 4.5e-4)
TOL_ELEM = 6e-7      # d/d fc2 pre-sigmoid = gh * bb * gate * (1 - gate), relative                  (2.0e-7)

DEFAULT = (128, 2048, 128, 8, None, 1.0)
CLIP = (128, 2048, 128, 8, 512, 1.0)
RAGGED = (36, 160, 40, 2, None, 1.0)
RAGGED_CLIP = (36, 160, 40, 2, 36, 1.0)
CASES = [(DEFAULT, 32), (DEFAULT, 40), (DEFAULT, 1), (DEFAULT, 5), (CLIP, 32), (CLIP, 3), (RAGGED, 33),
         (RAGGED_CLIP, 5)]


def saved_views(saved, spec, B):
    D, nf, emb, cells, clip_dim = spec[:5]
    names = [("x", D), ("pe", emb), ("t0", 4 * emb), ("temb", nf)] + ([("cmap", nf)] if clip_dim else []) + [("h0", nf)]
    for k in range(cells):
        names += [("a.%d" % k, nf), ("bb.%d" % k, nf), ("s.%d" % k, nf // 8), ("gate.%d" % k, nf), ("h.%d" % k, nf)]
    S, off = {}, 0
    for n, w in names:
        S[n] = saved[off:off + B * w].view(B, w)
        off += B * w
    assert off == saved.numel()
    return S


def run(net, spec, B, seed):
    D, nf, emb, cells, clip_dim = spec[:5]
    x, t, clip = gp_inputs(spec, B, seed)
    x, t = x.cuda(), t.cuda()
    clip = clip.cuda() if clip is not None else None
    masks = None
    if clip_dim is None:
        g = torch.Generator().manual_seed(seed + 1)
        masks = ((torch.rand(cells, B, nf, generator=g) >= 0.2).float() / 0.8).cuda()
    m = L.model_for(net, L.KIND_GLOBAL_PRIOR, net.lion_desc(), net.lion_params())
    lib = L.lib()
    saved = torch.empty(lib.lion_global_prior_saved_floats(m.h, B), device="cuda")
    out = torch.empty(B, D, device="cuda")
    L.check(lib.lion_global_prior_forward_train(m.h, L.ptr(x), L.ptr(t), L.ptr(clip), L.ptr(masks), L.ptr(saved),
                                                L.ptr(out), B, L.stream()), "forward_train")
    gout = gen(seed + 2, B, D).cuda() / B
    gx = torch.empty(B, D, device="cuda")
    params = net.lion_params()
    gp = [torch.empty_like(p) for p in params]
    T = {"gtemb": torch.empty(B, nf, device="cuda"), "gt0": torch.empty(B, 4 * emb, device="cuda"),
         "gcmap": torch.empty(B, nf, device="cuda") if clip_dim else None, "gh0": torch.empty(B, nf, device="cuda")}
    taps = [T[k] for k in ("gtemb", "gt0", "gcmap", "gh0")]
    for k in range(cells):
        for n, w in (("gh", nf), ("gz", nf), ("gs", nf // 8), ("gbb", nf), ("gz1", nf)):
            T["%s.%d" % (n, k)] = torch.empty(B, w, device="cuda")
            taps.append(T["%s.%d" % (n, k)])
    arr = (C.c_void_p * len(gp))(*[p.data_ptr() for p in gp])
    tarr = (C.c_void_p * len(taps))(*[None if p is None else p.data_ptr() for p in taps])
    L.check(lib.lion_global_prior_backward_probe(m.h, L.ptr(saved), L.ptr(clip), L.ptr(masks), L.ptr(gout), L.ptr(gx),
                                                 arr, len(gp), tarr, len(taps), B, L.stream()), "backward_probe")
    # the probe's gradients are lion_global_prior_backward's, bit for bit
    gx2, gp2 = torch.empty_like(gx), [torch.empty_like(p) for p in params]
    arr2 = (C.c_void_p * len(gp2))(*[p.data_ptr() for p in gp2])
    L.check(lib.lion_global_prior_backward(m.h, L.ptr(saved), L.ptr(clip), L.ptr(masks), L.ptr(gout), L.ptr(gx2), arr2,
                                           len(gp2), B, L.stream()), "backward")
    torch.cuda.synchronize()
    assert torch.equal(gx, gx2) and all(torch.equal(a, b) for a, b in zip(gp, gp2))
    names = [k for k, _ in net.named_parameters()]
    order = {id(p): i for i, p in enumerate(params)}
    G = {n: gp[order[id(p)]] for n, p in net.named_parameters()}
    assert len(G) == len(names) == len(gp)
    return saved_views(saved, spec, B), T, G, gout, gx, clip, masks


def dgrad_ref(g, w, swap=False):
    """(g~ W~, |g~| |W~|) float64: g~ = rna(g), W~ = trunc(W); swapped: g~ = trunc(g), W~ = rna(W)."""
    gm, wm = (SR.tf32_trunc, SR.tf32_rna) if swap else (SR.tf32_rna, SR.tf32_trunc)
    gt = gm(g.float()).double()
    wt = wm(w.reshape(w.shape[0], -1).float().contiguous()).double()
    return gt @ wt, gt.abs() @ wt.abs()


def wgrad_ref(g, x, add=None, rounded=True):
    """(g^T x~, |g|^T |x~|) float64 with x~ = rna(fl32(x + add)) (unrounded: fl32(x + add))."""
    xs = x.float() if add is None else x.float() + add.float()
    xt = (SR.tf32_rna(xs) if rounded else xs).double()
    gd = g.double()
    return gd.T @ xt, gd.T.abs() @ xt.abs()


def err(got, ref, bound):
    return ((got.double().reshape(ref.shape) - ref) / bound.clamp_min(1e-30)).abs().max().item()


@pytest.mark.parametrize("spec,B", CASES, ids=["%s-B%d" % ("x".join(str(v) for v in s[:5]), B) for s, B in CASES])
def test_global_prior_backward_stages(spec, B):
    net, sd = gp_net(*spec, seed=111)
    net = net.cuda()
    D, nf, emb, cells, clip_dim = spec[:5]
    S, T, G, gout, gx, clip, masks = run(net, spec, B, 200 + B)
    sd = {k: v.cuda() for k, v in sd.items()}
    e = {"dgrad": 0.0, "wgrad": 0.0, "elem": 0.0, "swap_dgrad": float("inf"), "swap_wgrad": float("inf")}
    worst = {"dgrad": None, "wgrad": None}

    def dg(label, got, g, w, extra=None, post=None, swap_check=False):
        ref, bound = dgrad_ref(g, w)
        if extra is not None:
            ref, bound = ref + extra.double(), bound + extra.double().abs()
        if post is not None:
            ref, bound = ref * post, bound * post.abs()
        v = err(got, ref, bound)
        if v > e["dgrad"]:
            e["dgrad"], worst["dgrad"] = v, label
        if swap_check:
            r2, _ = dgrad_ref(g, w, swap=True)
            if extra is not None:
                r2 = r2 + extra.double()
            if post is not None:
                r2 = r2 * post
            e["swap_dgrad"] = min(e["swap_dgrad"], err(got, r2, bound))

    def wg(name, g, x, add=None, bias=True, swap_check=False):
        ref, bound = wgrad_ref(g, x, add)
        v = err(G[name + ".weight"], ref, bound)
        if v > e["wgrad"]:
            e["wgrad"], worst["wgrad"] = v, name
        if swap_check:
            r2, _ = wgrad_ref(g, x, add, rounded=False)
            e["swap_wgrad"] = min(e["swap_wgrad"], err(G[name + ".weight"], r2, bound))
        if bias:
            gd = g.double()
            e["wgrad"] = max(e["wgrad"], err(G[name + ".bias"], gd.sum(0), gd.abs().sum(0)))

    def se_gz(gh, k):
        bb, gate = S["bb.%d" % k].double(), S["gate.%d" % k].double()
        ref = gh.double() * bb * gate * (1 - gate)
        got = T["gz.%d" % k].double()
        e["elem"] = max(e["elem"], ((got - ref).abs() / ref.abs().clamp_min(1e-30)).max().item())

    last = cells - 1
    wg("output_layer", gout, S["h.%d" % last])
    dg("output_layer", T["gh.%d" % last], gout, sd["output_layer.weight"])
    gtemb_ref = gtemb_bound = 0
    gcmap_ref = gcmap_bound = 0
    for k in range(cells - 1, -1, -1):
        p = "all_modules.%d." % k
        gh = T["gh.%d" % k]
        se_gz(gh, k)
        gz, gs, gbb, gz1 = T["gz.%d" % k], T["gs.%d" % k], T["gbb.%d" % k], T["gz1.%d" % k]
        wg(p + "SE.fc.2", gz, S["s.%d" % k], bias=False)
        dg(p + "SE.fc.2", gs, gz, sd[p + "SE.fc.2.weight"], post=(S["s.%d" % k] > 0).double())
        wg(p + "SE.fc.0", gs, S["bb.%d" % k], bias=False)
        dg(p + "SE.fc.0", gbb, gs, sd[p + "SE.fc.0.weight"], extra=gh.double() * S["gate.%d" % k].double(),
           post=(S["bb.%d" % k] > 0).double())
        wg(p + "conv2", gbb, S["a.%d" % k], swap_check=True)
        post = (S["a.%d" % k] > 0).double() * (masks[k].double() if masks is not None else 1.0)
        dg(p + "conv2", gz1, gbb, sd[p + "conv2.weight"], post=post, swap_check=True)
        h_in = S["h.%d" % (k - 1)] if k else S["h0"]
        if clip_dim:
            wg(p + "conv1", gz1, torch.cat([h_in, S["cmap"]], 1), add=torch.cat([S["temb"], torch.zeros_like(S["cmap"])], 1))
        else:
            wg(p + "conv1", gz1, h_in, add=S["temb"])
        ref, bound = dgrad_ref(gz1, sd[p + "conv1.weight"])
        gtemb_ref, gtemb_bound = gtemb_ref + ref[:, :nf], gtemb_bound + bound[:, :nf]
        if clip_dim:
            gcmap_ref, gcmap_bound = gcmap_ref + ref[:, nf:], gcmap_bound + bound[:, nf:]
        nxt = T["gh.%d" % (k - 1)] if k else T["gh0"]
        dg(p + "conv1", nxt, gz1, sd[p + "conv1.weight"][:, :nf], extra=gh)
    for label, got, ref, bound in [("temb sum", T["gtemb"], gtemb_ref, gtemb_bound)] + (
            [("cmap sum", T["gcmap"], gcmap_ref, gcmap_bound)] if clip_dim else []):
        v = err(got, ref, bound)
        if v > e["dgrad"]:
            e["dgrad"], worst["dgrad"] = v, label
    if clip_dim:
        wg("clip_feat_mapping", T["gcmap"], clip)
    wg("input_layer", T["gh0"], S["x"])
    dg("input_layer", gx, T["gh0"], sd["input_layer.weight"])
    wg("temb_layer.1", T["gtemb"], S["t0"])
    dg("temb_layer.1", T["gt0"], T["gtemb"], sd["temb_layer.1.weight"])
    wg("temb_layer.0", T["gt0"], S["pe"])
    print("global prior backward %s B=%d: %s (worst at %s)" % (spec, B, ", ".join("%s %.2e" % kv for kv in e.items()),
                                                                worst), flush=True)
    assert e["dgrad"] <= TOL_DGRAD, "dgrad: %.3e > %.1e" % (e["dgrad"], TOL_DGRAD)
    assert e["wgrad"] <= TOL_WGRAD, "wgrad: %.3e > %.1e" % (e["wgrad"], TOL_WGRAD)
    assert e["elem"] <= TOL_ELEM, "SE gate backward: %.3e > %.1e" % (e["elem"], TOL_ELEM)
    assert e["swap_dgrad"] > TOL_DGRAD and e["swap_wgrad"] > TOL_WGRAD, "the tolerances do not tell the operand models apart"
