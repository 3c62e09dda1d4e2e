import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tests.synth import synth_state_dict
from tests.util import gen, rel_err
from lion_b200.config import default_prior_cfg
from lion_b200.models.latent_points_ada_localprior import PVCNN2Prior
from lion_b200.models.pvcnn2_ada import PVConv
keys = json.load(open('tests/golden/keys.json'))
cfg = default_prior_cfg()
m = PVCNN2Prior(cfg.sde, 1, cfg); m.load_state_dict(synth_state_dict(keys['prior'], 11)); m = m.cuda().eval()
x, style = gen(31, 3, 8192, 1, 1).cuda(), gen(32, 3, 128, 1, 1).cuda()
t = torch.tensor([1000.0, 500.0, 1.0]).cuda()
a = m(x=x, t=t, condition_input=style); b = m(x=x, t=t, condition_input=style)
print("same-call repeat: bitwise", torch.equal(a, b), "rel", rel_err(a, b))
one = m(x=x[1:2], t=t[1:2], condition_input=style[1:2])
print("  B=3 vs B=1 rel", rel_err(one, a[1:2]))
for (cin, cout, r, N) in [(64, 64, 32, 2048), (128, 128, 8, 64), (4, 32, 32, 2048)]:
    pv = PVConv(cin, cout, 3, r, with_se=True, cfg=cfg)
    pv.load_state_dict(synth_state_dict({k: list(v.shape) for k, v in pv.state_dict().items()}, 23)); pv = pv.cuda().eval()
    f, c, s = gen(4, 3, cin, N).cuda(), gen(5, 3, 3, N, scale=0.4).cuda(), gen(6, 3, 128).cuda()
    o1 = pv((f, c, None, s))[0]; o2 = pv((f, c, None, s))[0]; o3 = pv((f[1:2], c[1:2], None, s[1:2]))[0]
    print("  pvconv", cin, cout, r, "repeat bitwise", torch.equal(o1, o2), "rel", rel_err(o1, o2), "B3 vs B1", rel_err(o3, o1[1:2]))
