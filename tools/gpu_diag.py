"""Stage-by-stage parity of the CUDA Pangu step against the CPU oracle (run on the GPU box).
    python tools/gpu_diag.py [nlat nlon]
"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from skyrim_b200.config import pangu_small, PANGU_CHANNELS
from skyrim_b200.weights import make_pangu_weights, synthetic_state
from skyrim_b200.engine import StepEngine
from oracle.pangu_ref import PanguRef, rel_err_per_channel

nlat = int(sys.argv[1]) if len(sys.argv) > 1 else 41
nlon = int(sys.argv[2]) if len(sys.argv) > 2 else 96
cfg = pangu_small(nlat, nlon)
w = make_pangu_weights(cfg, 0)
x0 = synthetic_state(PANGU_CHANNELS, cfg.nlat, cfg.nlon, 0)
ref = PanguRef(cfg, w, torch.float32)
stages = ref.stages(x0)
names = ["embed", "layer0", "down", "layer1", "layer2", "up", "layer3"]
xin = torch.from_numpy(x0)[None].cuda()
eng = StepEngine(cfg, 0)
eng.load_weights(w)
print(f"== grid {nlat}x{nlon}", flush=True)
for i, nm in enumerate(names):
    eng.debug_set("stop_after", i)
    try:
        eng.step(xin)
        torch.cuda.synchronize()
    except Exception as e:
        print("  stage", nm, "FAILED:", e, flush=True)
        break
    r = stages[nm]
    which = "tokens2" if nm in ("down", "layer1", "layer2") else "tokens1"
    t = eng.debug_tensor(which, tuple(r.shape)).cpu()
    err = (t - r).norm() / r.norm()
    print(f"  {nm:7s} rel l2 err {err:.3e}  max abs {float((t - r).abs().max()):.3e}  nan={bool(torch.isnan(t).any())}", flush=True)
eng.debug_set("stop_after", 99)
try:
    y = eng.step(xin); torch.cuda.synchronize()
    e = rel_err_per_channel(y[0].cpu().numpy(), stages["out"].numpy())
    print(f"  OUTPUT per-channel rel err max {e.max():.3e} (ch {PANGU_CHANNELS[int(e.argmax())]}) median {np.median(e):.3e}", flush=True)
except Exception as e:
    print("  full step FAILED:", e, flush=True)
eng.close()
