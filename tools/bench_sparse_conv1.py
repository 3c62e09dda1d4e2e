#!/usr/bin/env python
"""The sparse first convolution's output grid with and without the activity mask, at B = 32 (one GPU).

For every PVConv of a PVCNN2Prior forward whose first convolution runs sparse, the device time of the pair
k_sparse_conv_gather + the k_act_grid that reads its raw output, with the activity mask (default) and with the whole-grid
route (lion_ctx_set_sparse_conv1_dense), modes alternated.  Kernel times come from torch.profiler (CUPTI device
timestamps, one profiled forward per repetition); the whole forward is also timed with CUDA events in both modes.

Inputs: a Gaussian latent blob (the benchmark's x_T, N(0, 1) noise) and a surface-like cloud (points on a sphere with a
little radial noise).  Printed: the measured active fraction `a` of every sparse layer (r = 32: the latent points,
r = 16: their 1024 furthest-point centres), the bytes of raw1 each mode moves, the card name and power limit, and `a`
at the inputs of the steps t = 999, 500 and 0 of a real 1000-step sampling run of the same prior.

    python tools/bench_sparse_conv1.py [--reps 3] [--no-sampling]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from lion_b200 import _lib as L  # noqa: E402

B, NPTS = 32, 2048


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:          # (informational only)
        pl = "unknown (%s)" % e
    return name, pl


def prior():
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.latent_points_ada_localprior import PVCNN2Prior
    from tests.synth import synth_state_dict
    keys = json.load(open(os.path.join(ROOT, "tests", "golden", "keys.json")))
    cfg = default_prior_cfg()
    m = PVCNN2Prior(cfg.sde, 1, cfg)
    m.load_state_dict(synth_state_dict(keys["prior"], 11))
    return m.cuda().eval()


def inputs(kind):
    g = torch.Generator().manual_seed(5)
    if kind == "gauss":
        x = torch.randn(B, NPTS, 4, generator=g)
    else:
        d = torch.randn(B, NPTS, 3, generator=g)
        d = d / d.norm(dim=-1, keepdim=True) * (1 + 0.02 * torch.randn(B, NPTS, 1, generator=g))
        x = torch.cat([d, torch.randn(B, NPTS, 1, generator=g)], -1)
    return x.reshape(B, NPTS * 4, 1, 1).cuda()


_mask_models = {}


def active_fraction(xyz, r):
    """[B,3,n] points -> fraction of the r^3 voxels with an occupied neighbour, from the library's own mask"""
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.pvcnn2_ada import PVConv
    if r not in _mask_models:
        cin = 32 if r == 32 else 128
        _mask_models[r] = PVConv(cin, 64 if r == 16 else 32, 3, r, with_se=True, attention=False, cfg=default_prior_cfg()).cuda().eval()
    mod = _mask_models[r]
    m = L.model_for(mod, L.KIND_PVCONV, mod.lion_desc(), mod.lion_params())
    b, _, n = xyz.shape
    feats = torch.zeros(b, mod.lion_desc()[0], n, device="cuda")
    rp, W = r + 2, (r ** 3 + 31) // 32
    vg = torch.empty(b, rp, rp, rp, dtype=torch.int32, device="cuda")
    mask = torch.empty(b, W, dtype=torch.int32, device="cuda")
    L.check(L.lib().lion_pvconv_conv1_mask_probe(m.h, L.ptr(feats), L.ptr(xyz.contiguous()), L.ptr(vg), L.ptr(mask), b, n,
                                                 L.stream()), "conv1 mask probe")
    torch.cuda.synchronize()
    bits = sum(bin(w & 0xffffffff).count("1") for w in mask.flatten().tolist())
    return bits / float(b * r ** 3)


def level_fractions(x):
    from lion_b200.third_party.pvcnn.functional import furthest_point_sample_indices
    xyz = x.view(-1, NPTS, 4)[:, :, :3].transpose(1, 2).contiguous()
    idx = furthest_point_sample_indices(xyz, 1024).long()
    c1 = torch.gather(xyz, 2, idx[:, None, :].expand(-1, 3, -1)).contiguous()
    return {"r32": active_fraction(xyz, 32), "r16": active_fraction(c1, 16)}


def set_dense(on):
    L.check(L.lib().lion_ctx_set_sparse_conv1_dense(L.ctx(), 1 if on else 0), "sparse conv1 dense")


def profiled_pairs(m, x, style, t):
    """(C, r, gather us, k_act_grid us) of each sparse gather of one forward and the k_act_grid after it, in launch
    order; r from the gather's grid (cdiv(r^3, 128) blocks), read from the exported trace"""
    import tempfile
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m(x=x, t=t, condition_input=style)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        ev = json.load(open(path))["traceEvents"]
    ev = sorted([e for e in ev if e.get("cat") == "kernel"], key=lambda e: e["ts"])
    pairs = []
    for i, e in enumerate(ev):
        if "k_sparse_conv_gather" in e["name"]:
            c = 64 if "<64>" in e["name"] else 32
            r = {256: 32, 32: 16, 4: 8}[e["args"]["grid"][0]]
            act = next(f for f in ev[i + 1:] if "k_act_grid" in f["name"])
            pairs.append((c, r, e["dur"], act["dur"]))
    return pairs


def event_ms(m, x, style, t, n=20):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        m(x=x, t=t, condition_input=style)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-sampling", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    name, pl = card()
    m = prior()
    g = torch.Generator().manual_seed(7)
    style = torch.randn(B, 128, 1, 1, generator=g).cuda()
    t = torch.full((B,), 500.0).cuda()
    out = {"card": name, "power_limit": pl, "B": B, "inputs": {}}
    with torch.no_grad():
        for kind in ("gauss", "surface"):
            x = inputs(kind)
            for dense in (True, False):             # warm both modes (module load, arena sizing)
                set_dense(dense)
                m(x=x, t=t, condition_input=style)
            torch.cuda.synchronize()
            res = {"dense": [], "mask": []}
            fwd = {"dense": [], "mask": []}
            for _ in range(args.reps):
                for mode in ("dense", "mask"):
                    set_dense(mode == "dense")
                    res[mode].append(profiled_pairs(m, x, style, t))
                    fwd[mode].append(event_ms(m, x, style, t))
            set_dense(False)
            fr = level_fractions(x)
            layers = []
            for li, (c, r, _, _) in enumerate(res["mask"][0]):
                a = fr["r%d" % r]
                whole = 2 * B * r ** 3 * c * 4                        # raw1 stored by the gather and read by k_act_grid
                row = {"layer": li, "C": c, "r": r, "a": round(a, 4),
                       "raw1_bytes": {"dense": whole, "mask": int(round(whole * a))}}
                for mode in ("dense", "mask"):
                    row[mode + "_pair_us"] = [round(rep[li][2] + rep[li][3], 1) for rep in res[mode]]
                    row[mode + "_gather_us"] = round(min(rep[li][2] for rep in res[mode]), 1)
                    row[mode + "_act_us"] = round(min(rep[li][3] for rep in res[mode]), 1)
                layers.append(row)
            out["inputs"][kind] = {"active_fraction": fr, "layers": layers,
                                   "forward_ms": {k: [round(v, 3) for v in fwd[k]] for k in fwd}}
        if not args.no_sampling:
            from lion_b200.config import default_prior_cfg
            from lion_b200.utils.diffusion_pvd import DiffusionDiscretized
            cfg = default_prior_cfg(num_steps=1000)
            diff = DiffusionDiscretized(cfg.sde, None, cfg)
            torch.manual_seed(0)
            _, lst = diff.run_denoising_diffusion(m, B, [NPTS * 4, 1, 1], condition_input=style)
            hist = lst["pred_x"]              # hist[k]: the latent after the k-th step (t = 999 - k)
            xs = {"999": inputs("gauss"), "500": hist[498], "0": hist[998]}
            out["sampling_active_fraction"] = {tt: level_fractions(v) for tt, v in xs.items()}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
