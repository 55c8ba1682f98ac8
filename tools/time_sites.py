"""Timing of forecasts at sites on one GPU, in one process (DESIGN.md section 5, "Forecasts at sites"):

  1. sky_sample_sites at 721 x 1440 for 16 Pangu members x 69 channels at 1 000 and 10 000 random sites, both methods:
     ms (median of CUDA-event timings over repeated launches);
  2. the 16-member Pangu 6-h step with and without per-step site sampling plus its device->host copy
     (EnsembleRunner._walk against EnsembleRunner.iter_sites at 10 000 sites, all 69 channels): ms per step from a host
     clock around whole synchronised walks, alternated over three rounds, and the overhead in percent.

    python tools/time_sites.py [--steps 4] [--out time_sites.json]

Prints one JSON object with the card name, power limit and maximum SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [v.strip() for v in out.stdout.strip().splitlines()[0].split(",")])) if out.stdout else {}


def sites(n, seed=0):
    rng = np.random.default_rng(seed)
    return rng.uniform(-90, 90, n), rng.uniform(0, 360, n)


def time_sampling(x, reps=50):
    import torch
    from skyrim_b200.engine import SiteTable, sample_sites
    M, C, H, W = x.shape
    out = {}
    for n in (1000, 10000):
        for method in ("bilinear", "nearest"):
            t = SiteTable(*sites(n), H, W, method)
            v = sample_sites(x, t)
            torch.cuda.synchronize()
            times = []
            for _ in range(reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                sample_sites(x, t, out=v)
                b.record()
                b.synchronize()
                times.append(a.elapsed_time(b))
            out[f"{method}_{n}"] = float(np.median(times))
            t.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--members", type=int, default=16)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    from skyrim_b200.config import PANGU_CHANNELS, PanguConfig
    from skyrim_b200.engine import SiteTable, StepEngine
    from skyrim_b200.ensemble import EnsembleRunner
    from skyrim_b200.weights import channel_stats, make_pangu_weights, synthetic_state
    res = dict(gpu=gpu_info(), members=a.members, channels=len(PANGU_CHANNELS))
    cfg = PanguConfig()
    base = synthetic_state(PANGU_CHANNELS, cfg.nlat, cfg.nlon, 0)
    x = torch.from_numpy(base)[None].repeat(a.members, 1, 1, 1).cuda().contiguous()
    res["sample_ms"] = time_sampling(x)
    del x
    torch.cuda.empty_cache()
    eng = StepEngine(cfg, 0)
    eng.load_weights(make_pangu_weights(cfg, 0))
    run = EnsembleRunner(eng, base, channel_stats(PANGU_CHANNELS)[1], members_per_gpu=a.members, perturbation="gaussian")
    table = SiteTable(*sites(10000), cfg.nlat, cfg.nlon)

    def plain():
        for _ in run._walk(a.steps):
            pass

    def sampled():
        for _ in run.iter_sites(a.steps, table):
            pass

    for fn in (plain, sampled):   # warm-up: graph capture, pinned buffers
        fn()
    torch.cuda.synchronize()
    rounds = {"plain": [], "sampled": []}
    for _ in range(3):
        for name, fn in (("plain", plain), ("sampled", sampled)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            rounds[name].append((time.perf_counter() - t0) * 1e3 / a.steps)
    p, s = float(np.median(rounds["plain"])), float(np.median(rounds["sampled"]))
    res.update(step_ms=p, step_with_sites_ms=s, overhead_percent=100.0 * (s - p) / p, rounds_ms=rounds, sites=10000,
               steps=a.steps)
    table.close()
    eng.close()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
