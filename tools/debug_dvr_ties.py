"""Debug aid: tie-prone rays (tests/inputs.py::dvr_inputs_ties) three ways -- the reference's own CUDA
binary (oracle/_ref/ref_dvr.so), the C oracle, vidar_b200 -- and who disagrees with whom."""
import json, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import build_ref, dvr_ref
from tests.inputs import dvr_inputs_ties
from vidar_b200 import render
sigma, origin, points, tindex = dvr_inputs_ties(M=int(os.environ.get('TIES_M', '6000')))
dev = torch.device("cuda:0")
s, o, p, t = (torch.from_numpy(a).to(dev) for a in (sigma, origin, points, tindex))
grid = list(sigma.shape[1:])
ref = build_ref.load("ref_dvr")
out = {}
bad = lambda a, b: np.flatnonzero(np.abs(a - b) > 1e-5 * np.maximum(1.0, np.abs(b)))
for name, f_gpu, f_orc, f_ref in (
        ("fwd_test", lambda: render.dvr.render_forward(s, o, p, t, grid, "test")[0], lambda: dvr_ref.render_forward(sigma, origin, points, tindex, None, "test")[0],
         lambda: ref.render_forward(s, o, p, t, grid, "test")[0]),
        ("render_l1", lambda: render.dvr.render(s, o, p, t, "l1")[0], lambda: dvr_ref.render(sigma, origin, points, tindex, "l1")[0],
         lambda: ref.render(s, o, p, t, "l1")[0])):
    g, orc, r = f_gpu().cpu().numpy()[0], f_orc()[0], f_ref().cpu().numpy()[0]
    out[name] = {"gpu_vs_ref": bad(g, r).tolist()[:20], "oracle_vs_ref": bad(orc, r).tolist()[:20], "gpu_vs_oracle": bad(g, orc).tolist()[:20],
                 "frames_of_gpu_vs_ref": tindex[0, bad(g, r)].tolist()[:20],
                 "detail": [dict(i=int(i), point=points[0, i].tolist(), gpu=float(g[i]), oracle=float(orc[i]), ref=float(r[i])) for i in sorted(set(bad(g, orc).tolist() + bad(g, r).tolist()))[:12]]}
print(json.dumps(out))
