"""Per-kernel-family device time of a full-size step (development).
    python tools/gpu_families.py [pangu|sfno] [--steps N] [--members M]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from skyrim_b200.config import *
from skyrim_b200.engine import StepEngine
from skyrim_b200.weights import *
from skyrim_b200.verify import compare_fullsize, load_fixture, summarise

model = "sfno" if "sfno" in sys.argv else "pangu"
steps = int(sys.argv[sys.argv.index("--steps") + 1]) if "--steps" in sys.argv else 5
M = int(sys.argv[sys.argv.index("--members") + 1]) if "--members" in sys.argv else 1
if model == "pangu":
    cfg, ch = pangu_full(), PANGU_CHANNELS
    w = make_pangu_weights(cfg, 0)
else:
    cfg, ch = sfno_full(), FCNV2_CHANNELS
    w = dict(make_sfno_weights(cfg, 0)); w.update(sfno_tables(cfg))
eng = StepEngine(cfg, 0)
eng.load_weights(w); del w
x = torch.from_numpy(synthetic_state(ch, cfg.nlat, cfg.nlon, 0))[None].repeat(M, 1, 1, 1).cuda().contiguous()
y = torch.empty_like(x)
first = eng.step(x).clone()
s = summarise(compare_fullsize(first[0], load_fixture(model)))
for _ in range(2):
    eng.step(x, y)
torch.cuda.synchronize()
eng.profile_begin()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(steps):
    eng.step(x, y); x, y = y, x
e1.record(); torch.cuda.synchronize()
fam = eng.profile_end()
print(f"[{model} M={M}] {e0.elapsed_time(e1) / steps:.3f} ms/step (with profiling events); verify rel {s['rel']:.2e} block {s['block']:.2e}")
print("   " + "  ".join(f"{k} {v[0] / steps:.3f}" for k, v in sorted(fam.items(), key=lambda kv: -kv[1][0])))
