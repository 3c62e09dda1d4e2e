"""TF32 against FP16 operands (torch.autocast("cuda", float16)) for the second 3x3x3 convolution of every PVConv.

    python tools/bench_autocast.py [--steps 1000] [--batch 32] [--out DIR] > autocast.jsonl

(a) Each second-convolution shape class at B = 32, both modes alternated in one call: the time of the convolution
    kernels alone (k_conv_tc, plus k_conv_stats on interior blocks) and the rate against the H100 SXM data-sheet peaks
    (dense TF32 495, FP16 989 TFLOP/s at 700 W).  The kernel time is taken from torch.profiler's CUDA activity over the
    stand-alone Conv3d rather than from CUDA events: events around the call would also time its layout conversions.
(s) One point-prior forward at B = 32 on the same finite input in both modes, CUDA events around `--iters` calls,
    modes alternated: the same work in both modes whatever the weights.  Profiler off.
(b) Shapes/s of full generate_samples_vada_2prior passes (global prior + point prior, `--steps` DDPM steps each, and the
    decoder) at B = 32, TF32 and FP16 alternated, the same seeds in both modes.  Profiler off.  With synthetic weights
    the trajectories leave the FP16 range; the first step whose point-prior state is non-finite is reported, and past
    it the data-dependent work (voxelisation, occupancy skips, FPS, ball query) is no longer that of the TF32 pass.
(c) The deviation of the FP16 pass's clouds from the TF32 pass's (report only: 1000 steps are chaotic).

The card's name and power limit are read in the same call and printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

CLASSES = [(32, 32, 32), (64, 64, 32), (64, 64, 16), (128, 128, 16), (128, 128, 8)]   # (cin, cout, r) of the second convolutions
PEAK = {"tf32": 495e12, "fp16": 989e12}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def conv_kernel_ms(m, x, fp16, iters):
    """mean GPU time per call of the convolution kernels of one Conv3d call (profiler, kernels named k_conv_*)."""
    from torch.profiler import ProfilerActivity, profile

    def call():
        with torch.autocast("cuda", dtype=torch.float16, enabled=fp16):
            m(x, return_gn_stats=True)

    for _ in range(3):
        call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            call()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "k_conv_tc" in e.key or "k_conv_stats" in e.key)
    return us / 1e3 / iters


def part_a(B, iters, rounds):
    from lion_b200.models.pvcnn2_ada import Conv3d
    out = []
    for cin, cout, r in CLASSES:
        m = Conv3d(cin, cout).cuda()
        g = torch.Generator(device="cuda").manual_seed(1)
        with torch.no_grad():
            m.weight.copy_(torch.randn(m.weight.shape, device="cuda", generator=g) * (27 * cin) ** -0.5)
        x = torch.randn(B, cin, r, r, r, device="cuda", generator=g)
        t = {"tf32": [], "fp16": []}
        for _ in range(rounds):                       # alternated: TF32, FP16, TF32, FP16, ...
            t["tf32"].append(conv_kernel_ms(m, x, False, iters))
            t["fp16"].append(conv_kernel_ms(m, x, True, iters))
        flops = 2.0 * B * r ** 3 * 27 * cin * cout
        row = {"part": "a", "cin": cin, "cout": cout, "r": r, "B": B}
        for k in ("tf32", "fp16"):
            ms = min(t[k])
            row[k + "_ms"] = round(ms, 4)
            row[k + "_ms_all"] = [round(v, 4) for v in t[k]]
            row[k + "_tflops"] = round(flops / ms / 1e9, 1)
            row[k + "_share_of_datasheet_peak"] = round(flops / ms / 1e-3 / PEAK[k], 3)
        row["fp16_speedup"] = round(min(t["tf32"]) / min(t["fp16"]), 3)
        print(json.dumps(row), flush=True)
        out.append(row)
        del m, x
        torch.cuda.empty_cache()
    return out


def part_step(B, iters, rounds):
    from bench import build_models
    from lion_b200.config import default_prior_cfg
    cfg = default_prior_cfg()
    lp = build_models(cfg, torch.device("cuda"))[0][1]
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(B, 8192, 1, 1, device="cuda", generator=g)
    style = torch.randn(B, 128, 1, 1, device="cuda", generator=g)
    t = torch.full((B,), 500.0, device="cuda")

    def timed(fp16, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.autocast("cuda", dtype=torch.float16, enabled=fp16):
            e0.record()
            for _ in range(n):
                y = lp(x=x, t=t, condition_input=style)
            e1.record()
        torch.cuda.synchronize()
        assert torch.isfinite(y).all()
        return e0.elapsed_time(e1) / n

    timed(False, 3)
    timed(True, 3)
    ms = {"tf32": [], "fp16": []}
    for _ in range(rounds):
        ms["tf32"].append(timed(False, iters))
        ms["fp16"].append(timed(True, iters))
    row = {"part": "s", "B": B, "what": "one point-prior forward, finite fixed input", "iters": iters}
    for k in ("tf32", "fp16"):
        row[k + "_ms"] = [round(v, 3) for v in ms[k]]
    row["fp16_speedup"] = round(min(ms["tf32"]) / min(ms["fp16"]), 3)
    print(json.dumps(row), flush=True)
    return row


def part_bc(B, steps, rounds, out_dir):
    from bench import build_models
    from lion_b200.config import default_prior_cfg
    from lion_b200.trainers.train_2prior import generate_samples_vada_2prior
    from lion_b200.utils.diffusion_pvd import DiffusionDiscretized
    cfg = default_prior_cfg(num_steps=steps)
    dae, vae = build_models(cfg, torch.device("cuda"))
    diff = DiffusionDiscretized(cfg.sde, None, cfg)
    shape = vae.latent_shape()

    first_bad = {}

    def one(fp16, seed):
        torch.manual_seed(seed)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = generate_samples_vada_2prior(shape, dae, diff, vae, B, fp16)
        torch.cuda.synchronize()
        secs = time.perf_counter() - t0
        # point-prior states after loop steps t = steps-1 .. 0: the first non-finite one
        bad = [k for k, h in enumerate(res[4]["eps_list"]["pred_x"]) if not bool(torch.isfinite(h).all())]
        first_bad["fp16" if fp16 else "tf32"] = steps - 1 - bad[0] if bad else None
        return secs, res[0]

    one(False, 0)                                     # warm-up: module packing, arena, both modes' first calls
    one(True, 0)
    secs = {"tf32": [], "fp16": []}
    imgs = {}
    for k in range(rounds):
        for mode, fp16 in (("tf32", False), ("fp16", True)):
            s, img = one(fp16, 100 + k)
            secs[mode].append(s)
            if k == 0:
                imgs[mode] = img.float().cpu()
    row = {"part": "b", "B": B, "ddpm_steps": steps, "passes_per_mode": rounds}
    for mode in ("tf32", "fp16"):
        row[mode + "_s_per_pass"] = [round(v, 3) for v in secs[mode]]
        row[mode + "_shapes_per_s"] = round(B / min(secs[mode]), 3)
    row["fp16_speedup"] = round(min(secs["tf32"]) / min(secs["fp16"]), 3)
    row["first_nonfinite_point_prior_step_t"] = first_bad       # None: finite throughout
    print(json.dumps(row), flush=True)
    a, b = imgs["fp16"].double(), imgs["tf32"].double()
    dev = {"part": "c", "max_abs_diff": (a - b).abs().max().item(), "max_abs_tf32": b.abs().max().item(),
           "rel_rms": ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item(),
           "finite_fp16": bool(torch.isfinite(a).all())}
    print(json.dumps(dev), flush=True)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        torch.save(imgs, os.path.join(out_dir, "autocast_clouds.pt"))
    return row, dev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--skip-a", action="store_true")
    ap.add_argument("--skip-b", action="store_true")
    ap.add_argument("--skip-s", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "tools/bench_autocast.py measures on the GPU; there is no CPU path"
    print(json.dumps({"card": card(), "torch": torch.__version__}), flush=True)
    if not args.skip_a:
        part_a(args.batch, args.iters, args.rounds)
    if not args.skip_s:
        part_step(args.batch, args.iters, args.rounds)
    if not args.skip_b:
        part_bc(args.batch, args.steps, args.rounds, args.out)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
