"""One denoising step of both priors at the benchmarked batch, eager (no CUDA graph), bracketed by cudaProfilerStart/Stop
so that `ncu --profile-from-start off` sees exactly one step after a warm-up step:

    ncu --metrics <list> --clock-control none --profile-from-start off --csv --log-file step.csv python tools/profile_step.py

Where Nsight does not run, `python tools/profile_step.py --torch OUT.json` records the same step under torch.profiler
(CUDA activities) and prints -- and writes to OUT.json -- the GPU time per kernel name, largest first.

Weights: key-seeded synthetic (tests/synth.py), x / style: seeded noise -- the same shapes bench.py times."""
import json
import os
import sys
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lion_b200.config import default_prior_cfg
from lion_b200.models.latent_points_ada_localprior import PVCNN2Prior
from lion_b200.models.score_sde.resnet import PriorSEDrop
from tests.synth import synth_state_dict

B = int(os.environ.get("B", "32"))
cfg = default_prior_cfg()
shp = lambda m: {k: list(v.shape) for k, v in m.state_dict().items()}
gp = PriorSEDrop(cfg.sde, 128, cfg)
gp.load_state_dict(synth_state_dict(shp(gp), 14))
lp = PVCNN2Prior(cfg.sde, 1, cfg)
lp.load_state_dict(synth_state_dict(shp(lp), 11))
gp, lp = gp.cuda().eval(), lp.cuda().eval()
g = torch.Generator(device="cuda").manual_seed(0)
x = torch.randn(B, 8192, 1, 1, device="cuda", generator=g)
xg = torch.randn(B, 128, 1, 1, device="cuda", generator=g)
style = torch.randn(B, 128, 1, 1, device="cuda", generator=g)
t = torch.full((B,), 500.0, device="cuda")
for _ in range(2):                                  # warm-up: packs weights, sizes the arena, caches the style Linears
    gp(x=xg, t=t)
    lp(x=x, t=t, condition_input=style)
torch.cuda.synchronize()
if len(sys.argv) > 2 and sys.argv[1] == "--torch":
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gp(x=xg, t=t)
        lp(x=x, t=t, condition_input=style)
        torch.cuda.synchronize()
    per = defaultdict(lambda: [0.0, 0])            # kernel name -> [us, launches]
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            per[e.name][0] += e.time_range.elapsed_us()
            per[e.name][1] += 1
    total = sum(v[0] for v in per.values())
    rows = sorted(({"kernel": k, "us": round(v[0], 1), "launches": v[1], "share": round(v[0] / total, 4)}
                   for k, v in per.items()), key=lambda r: -r["us"])
    for r in rows[:25]:
        print("%9.1f us %5.1f %% %4d x  %s" % (r["us"], 100 * r["share"], r["launches"], r["kernel"][:110]))
    print("GPU time of one global-prior + one PVCNN2Prior forward at B=%d: %.3f ms" % (B, total / 1e3))
    with open(sys.argv[2], "w") as f:
        json.dump({"B": B, "device": torch.cuda.get_device_name(), "total_us": round(total, 1), "kernels": rows}, f, indent=1)
else:
    torch.cuda.profiler.start()
    gp(x=xg, t=t)
    lp(x=x, t=t, condition_input=style)
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
    print("profiled one global-prior + one PVCNN2Prior forward at B=%d" % B)
