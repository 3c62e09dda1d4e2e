#!/usr/bin/env python
"""The second 3x3x3 convolution of every PVConv whose first convolution runs sparse, with its class-valued 64-row blocks
skipped (default) and with every block computed (lion_ctx_set_conv2_class_mode(1)), at B = 32 (one GPU), modes alternated.

Kernel times come from torch.profiler (CUPTI device timestamps, one profiled PVCNN2Prior forward per repetition): per
layer the big k_conv_tc and, when skipping, the launches that prepare it (k_conv2_flags, the class grid's k_act_grid
and k_conv_tc).  The whole forward is also timed with CUDA events in both modes.

Flagged share: the class-valued blocks k_conv2_flags finds (lion_ctx_last_conv2_class_blocks) when a PVConv of that
resolution runs on the prior's points (r = 32: the latent points, r = 16: their 1024 furthest-point centres), for the
benchmark's Gaussian x_T, a surface-like cloud and the inputs of the steps t = 500 and t = 0 of a 1000-step sampling run.
Printed with the card name and power limit.

    python tools/bench_conv2_skip.py [--reps 3] [--no-sampling]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench_sparse_conv1 import B, NPTS, card, event_ms, inputs, prior  # noqa: E402
from lion_b200 import _lib as L  # noqa: E402


def set_mode(m):
    L.check(L.lib().lion_ctx_set_conv2_class_mode(L.ctx(), m), "conv2 class mode")


_models = {}


def flagged_share(xyz, r):
    """[B,3,n] points -> share of the row tiles' 64-row blocks that the second convolution of a PVConv at r skips"""
    from lion_b200.config import default_prior_cfg
    from lion_b200.models.pvcnn2_ada import PVConv
    if r not in _models:
        cin, cout = (32, 32) if r == 32 else (128, 64)
        _models[r] = PVConv(cin, cout, 3, r, with_se=True, attention=False, cfg=default_prior_cfg()).cuda().eval()
    mod = _models[r]
    b, _, n = xyz.shape
    feats = torch.zeros(b, mod.lion_desc()[0], n, device="cuda")
    style = torch.zeros(b, 128, device="cuda")
    mod((feats, xyz.contiguous(), None, style))
    f, t = C.c_longlong(0), C.c_longlong(0)
    L.check(L.lib().lion_ctx_last_conv2_class_blocks(L.ctx(), C.byref(f), C.byref(t)), "conv2 class blocks")
    return f.value / float(t.value)


def level_shares(x):
    from lion_b200.third_party.pvcnn.functional import furthest_point_sample_indices
    xyz = x.view(-1, NPTS, 4)[:, :, :3].transpose(1, 2).contiguous()
    idx = furthest_point_sample_indices(xyz, 1024).long()
    c1 = torch.gather(xyz, 2, idx[:, None, :].expand(-1, 3, -1)).contiguous()
    return {"r32": round(flagged_share(xyz, 32), 4), "r16": round(flagged_share(c1, 16), 4)}


def profiled_layers(m, x, style, t):
    """per sparse first convolution of one forward, in launch order: (C, r, conv2 us, preparation us), conv2 = the
    k_conv_tc right before the k_affine_prep that follows the layer's big k_act_grid"""
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
    main_stream = next(e for e in ev if "k_sparse_conv_gather" in e["name"])["args"].get("stream")
    ev = [e for e in ev if e["args"].get("stream") == main_stream]          # side-stream kernels interleave in time
    out = []
    for i, e in enumerate(ev):
        if "k_sparse_conv_gather" not in e["name"]:
            continue
        c = 64 if "<64>" in e["name"] else 32
        r = {256: 32, 32: 16, 4: 8}[e["args"]["grid"][0]]
        a = next(k for k in range(i + 1, len(ev)) if "k_act_grid" in ev[k]["name"])
        f = next(k for k in range(a + 1, len(ev)) if "k_affine_prep" in ev[k]["name"])
        assert "k_conv_tc" in ev[f - 1]["name"], ev[f - 1]["name"]
        prep = sum(ev[k]["dur"] for k in range(a + 1, f - 1))
        out.append((c, r, ev[f - 1]["dur"], prep))
    return out


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
    modes = {"computed": 1, "skipped": 0}
    with torch.no_grad():
        for kind in ("gauss", "surface"):
            x = inputs(kind)
            for mode in modes.values():             # warm both modes (module load, arena sizing)
                set_mode(mode)
                m(x=x, t=t, condition_input=style)
            torch.cuda.synchronize()
            res = {k: [] for k in modes}
            fwd = {k: [] for k in modes}
            for _ in range(args.reps):
                for k, mode in modes.items():
                    set_mode(mode)
                    res[k].append(profiled_layers(m, x, style, t))
                    fwd[k].append(event_ms(m, x, style, t))
            set_mode(0)
            layers = []
            for li, (c, r, _, _) in enumerate(res["skipped"][0]):
                row = {"layer": li, "C": c, "r": r}
                for k in modes:
                    row[k + "_conv2_us"] = [round(rep[li][2], 1) for rep in res[k]]
                row["skipped_prep_us"] = [round(rep[li][3], 1) for rep in res["skipped"]]
                layers.append(row)
            out["inputs"][kind] = {"flagged_share": level_shares(x), "layers": layers,
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
            out["sampling_flagged_share"] = {tt: level_shares(v) for tt, v in xs.items()}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
