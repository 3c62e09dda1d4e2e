"""Forward + backward wall time of the style prior (PriorSEDrop, nf 2048, 8 cells, D 128) at B = 8, 32 and 64: the
library's differentiable route (lion_global_prior_forward_train + lion_global_prior_backward) against torch eager
autograd of the same float32 network (cuBLAS / cuDNN with TF32 allowed), both in train() mode with dropout.

One timed step = forward, F.mse_loss against fixed noise, backward into .grad (zeroed with set_to_none before each
step), CUDA events around ITERS steps after WARMUP steps; the two implementations alternate in REPEATS rounds and the
median is reported.  The weight and gradient traffic the backward cannot avoid is reading W once for the dgrads and
writing dW once (2 x 309 MB = 618 MB); the forward streams W once more (309 MB).  Reported: those 927 MB per step over
the step time (lion_gbs_3w), and the backward's 618 MB over the same time (lion_gbs_2w).  The card's name and power
limit are read in the same run.

    python tools/bench_global_prior_train.py            # ITERS=20 WARMUP=5 REPEATS=3
"""
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from lion_b200.config import default_prior_cfg  # noqa: E402
from lion_b200.models.score_sde.resnet import PriorSEDrop  # noqa: E402
from tests.synth import synth_state_dict  # noqa: E402


class TorchPrior(nn.Module):
    """The reference's PriorSEDrop forward (resnet.py:195-218 with ResBlockSEDrop and SE) in eager torch, same keys."""

    def __init__(self, lib_net):
        super().__init__()
        self.net = lib_net          # owns the parameters (state-dict keys of the reference)
        half = lib_net.embedding_dim // 2
        step = torch.log(torch.tensor(10000.0)) / (half - 1)
        self.register_buffer("freqs", torch.exp(torch.arange(half) * -step))

    def forward(self, x, t):
        n = self.net
        e = (t * n.embedding_scale)[:, None] * self.freqs[None, :]
        temb = n.temb_layer(torch.cat([torch.sin(e), torch.cos(e)], 1)[:, :, None, None])
        h = n.input_layer(x)
        for blk in n.all_modules:
            a = F.dropout(torch.relu(blk.conv1(h + temb)), blk.dropout_ratio, self.training)
            bb = torch.relu(blk.conv2(a))
            h = h + bb * blk.SE.fc(bb)
        return n.output_layer(h)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def main():
    assert torch.cuda.is_available(), "bench_global_prior_train.py measures on a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    iters, warmup, repeats = (int(os.environ.get(k, d)) for k, d in (("ITERS", 20), ("WARMUP", 5), ("REPEATS", 3)))
    cfg = default_prior_cfg()
    net = PriorSEDrop(cfg.sde, 128, cfg)
    net.load_state_dict(synth_state_dict({k: list(v.shape) for k, v in net.state_dict().items()}, 14))
    net = net.cuda().train()
    ref = TorchPrior(net).cuda().train()
    weight_bytes = sum(p.numel() for p in net.parameters()) * 4
    res = {"card": card(), "weights_mb": weight_bytes / 1e6, "iters": iters, "repeats": repeats, "rows": []}
    for B in (8, 32, 64):
        g = torch.Generator(device="cuda").manual_seed(B)
        x = torch.randn(B, 128, 1, 1, device="cuda", generator=g)
        t = torch.randint(1, 1001, (B,), device="cuda", generator=g).float()
        noise = torch.randn(B, 128, 1, 1, device="cuda", generator=g)

        def step_lib():
            net.zero_grad(set_to_none=True)
            F.mse_loss(net(x, t), noise).backward()

        def step_torch():
            net.zero_grad(set_to_none=True)
            F.mse_loss(ref(x, t), noise).backward()

        times = {"lion": [], "torch": []}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(repeats):
            for name, fn in (("lion", step_lib), ("torch", step_torch)):
                for _ in range(warmup):
                    fn()
                torch.cuda.synchronize()
                e0.record()
                for _ in range(iters):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / iters)
        lib_ms, torch_ms = statistics.median(times["lion"]), statistics.median(times["torch"])
        row = {"B": B, "lion_fwd_bwd_ms": lib_ms, "torch_eager_fwd_bwd_ms": torch_ms, "speedup": torch_ms / lib_ms,
               "lion_gbs_3w": 3 * weight_bytes / 1e6 / lib_ms, "lion_gbs_2w": 2 * weight_bytes / 1e6 / lib_ms,
               "spread_ms": {k: [min(v), max(v)] for k, v in times.items()}}
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
