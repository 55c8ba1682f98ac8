"""Pangu's 6-h chain against the hierarchical 6-h / 24-h schedule at 721x1440, in one process:

  * the card's name and power limit;
  * the device memory the 24-h handle adds (cudaMemGetInfo before and after building it, on the 6-h handle's workspace);
  * predict(lead_time=168) under both schedules: host clock around the call, which ends with the device->host copy of
    its two slices (a device synchronise), after two warm-up calls; forwards counted (28 against 10);
  * forecast(n_steps=28) under both schedules, which run the same number of forwards.

    python tools/time_pangu_schedule.py [--reps 3] [--out pangu_schedule.json]

Prints one JSON line.  The initial condition is built once and served from memory, so both schedules time the same
work apart from the forwards."""
import argparse
import datetime
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: these are GPU timings")
    from bench import gpu_identity
    from skyrim_b200 import Skyrim
    from skyrim_b200.config import PANGU_CHANNELS, pangu_full
    from skyrim_b200.core.models.base import SyntheticDataSource
    from skyrim_b200.engine import StepEngine
    from skyrim_b200.weights import make_pangu_weights

    cfg = pangu_full()
    w6, w24 = make_pangu_weights(cfg, 0), make_pangu_weights(cfg, 1)
    out = {"gpu": gpu_identity(0), "grid": [cfg.nlat, cfg.nlon]}

    # memory of the second handle: built after the first has stepped once (its workspace exists)
    x = torch.zeros((1, cfg.n_channels, cfg.nlat, cfg.nlon), dtype=torch.float32, device="cuda")
    y = torch.empty_like(x)
    e6 = StepEngine(cfg, 0)
    e6.load_weights(w6)
    e6.step(x, y)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    e24 = StepEngine(cfg, 0)
    e24.share_workspace(e6)
    e24.load_weights(w24)
    e24.step(x, y)
    torch.cuda.synchronize()
    out["second_handle_bytes"] = free0 - torch.cuda.mem_get_info()[0]
    e24.close()
    e6.close()
    del x, y

    t0 = datetime.datetime(2024, 5, 7)
    ic = {t0: SyntheticDataSource(PANGU_CHANNELS, cfg.nlat, cfg.nlon)[t0]}
    models = {"6h": Skyrim("pangu", ic_source=ic, cfg=cfg, weights=w6),
              "hierarchical": Skyrim("pangu", ic_source=ic, cfg=cfg, weights=w6, schedule="hierarchical",
                                     weights_24=w24)}
    calls = [0]
    step = StepEngine.step

    def counted(self, *a, **k):
        calls[0] += 1
        return step(self, *a, **k)
    StepEngine.step = counted

    def timed(fn):
        calls[0] = 0
        torch.cuda.synchronize()
        c = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - c, calls[0]

    work = {"predict_168h": lambda sk: sk.predict(date="20240507", time="0000", lead_time=168),
            "forecast_28": lambda sk: sk.forecast(t0, n_steps=28)}
    for name, fn in work.items():
        for sk in models.values():   # warm-up: eager first use of each buffer tuple, then graph capture
            fn(sk)
            fn(sk)
        res = {s: [] for s in models}
        for _ in range(args.reps):   # alternate the schedules
            for s, sk in models.items():
                res[s].append(timed(lambda: fn(sk)))
        out[name] = {s: {"seconds": [round(t, 4) for t, _ in r], "median_s": round(sorted(t for t, _ in r)[len(r) // 2], 4),
                         "forwards": r[0][1]} for s, r in res.items()}
    StepEngine.step = step
    for sk in models.values():
        sk.model.release_model()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
