import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from lion_b200.config import default_prior_cfg
from lion_b200.models.score_sde.resnet import PriorSEDrop
from tests.synth import synth_state_dict
cfg = default_prior_cfg()
m = PriorSEDrop(cfg.sde, 128, cfg)
m.load_state_dict(synth_state_dict({k: list(v.shape) for k, v in m.state_dict().items()}, 14))
m = m.cuda().eval()
B = int(os.environ.get("B", "32"))
x = torch.randn(B, 128, 1, 1, device="cuda"); t = torch.full((B,), 500.0, device="cuda")
for _ in range(3): m(x=x, t=t)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
n = int(os.environ.get("ITERS", "50"))
e0.record()
for _ in range(n): m(x=x, t=t)
e1.record(); torch.cuda.synchronize()
eager_us = e0.elapsed_time(e1) * 1000 / n
# the sampling loop replays the step from a CUDA graph: time that too (launch gaps are what the graph removes)
from lion_b200 import _lib as L
out = m(x=x, t=t)
with L.capture_graph() as g:
    out = m(x=x, t=t)
for _ in range(3): g.replay()
torch.cuda.synchronize()
e0.record()
for _ in range(n): g.replay()
e1.record(); torch.cuda.synchronize()
graph_us = e0.elapsed_time(e1) * 1000 / n
print(json.dumps({"global_prior_forward_us_eager": eager_us, "global_prior_forward_us_graph": graph_us, "B": B,
                  "launches_per_forward": L.last_launches(),
                  "weights_mb": sum(p.numel() for p in m.parameters()) * 4 / 1e6,
                  "hbm_gbs_graph": sum(p.numel() for p in m.parameters()) * 4 / 1e3 / graph_us}))
