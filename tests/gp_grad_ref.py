"""Float64 restatement of the global prior's training forward (Prior.forward with SE cells and ResBlockSEDrop's dropout
as a multiplication by given scaled masks), for autograd: the gradients the library's backward is compared with.

Parameters are taken by state-dict name from a dict of float64 tensors; every Linear is W x + b on exact operands (no
TF32 model: the whole-network tests compare against this as the exact gradient)."""
import torch
import torch.nn.functional as F


def _lin(P, name, x, bias=True):
    w = P[name + ".weight"]
    y = x @ w.reshape(w.shape[0], -1).T
    return y + P[name + ".bias"] if bias else y


def prior_f64(P, x, pe, clip=None, masks=None):
    """x [B, D], pe [B, emb] (the positional embedding), clip [B, clip_dim] or None, masks [ncell, B, nf] or None,
    all float64 -> out [B, D]."""
    temb = _lin(P, "temb_layer.1", _lin(P, "temb_layer.0", pe))
    cm = _lin(P, "clip_feat_mapping", clip) if clip is not None else None
    h = _lin(P, "input_layer", x)
    k = 0
    while "all_modules.%d.conv1.weight" % k in P:
        p = "all_modules.%d." % k
        u = h + temb
        if cm is not None:
            u = torch.cat([u, cm], 1)
        a = torch.relu(_lin(P, p + "conv1", u))
        if masks is not None:
            a = a * masks[k]
        bb = torch.relu(_lin(P, p + "conv2", a))
        s = torch.relu(_lin(P, p + "SE.fc.0", bb, bias=False))
        h = h + bb * torch.sigmoid(_lin(P, p + "SE.fc.2", s, bias=False))
        k += 1
    return _lin(P, "output_layer", h)


def mse_grads(sd, x, pe, noise, clip=None, masks=None):
    """F.mse_loss(prior(x), noise) and its gradients in float64.  sd: {name: tensor}.  Returns (loss, dx, {name: grad})."""
    P = {k: v.detach().double().requires_grad_(True) for k, v in sd.items()}
    xd = x.detach().double().requires_grad_(True)
    out = prior_f64(P, xd, pe.double(), None if clip is None else clip.double(),
                    None if masks is None else masks.double())
    loss = F.mse_loss(out, noise.double())
    loss.backward()
    return loss.detach(), xd.grad, {k: v.grad for k, v in P.items()}


def golden(tag, z):
    """The inputs and results of one net of tests/golden/global_prior_grad.npz as tensors."""
    g = {k[len(tag) + 3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith(tag + "/g/")}
    get = lambda n: torch.from_numpy(z[tag + "/" + n]) if (tag + "/" + n) in z.files else None
    return {"x": get("x"), "t": get("t"), "pe": get("pe"), "noise": get("noise"), "clip": get("clip"),
            "mask": get("mask"), "loss": float(z[tag + "/loss"]), "dx": get("dx"), "grads": g}
