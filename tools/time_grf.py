#!/usr/bin/env python
"""Time the spherical Gaussian random field perturbation and compare the Pangu ensemble spread it produces with K11's.

    python tools/time_grf.py [--iters 10] [--spread-steps 4] [--out result.json]

Prints one JSON object:
  grf_ms[L]       ms per ``engine.perturb_ic_grf`` call on 4 members x 69 channels at 721 x 1440, L in {90, 180, 360}
                  (CUDA events around --iters back-to-back calls after two warm-up calls; includes the workspace
                  allocation and spectrum upload the Python call makes, not the first call's Legendre table build)
  lon_tflops[L]   2 x fields x 721 x 1440 x 2 (L + 1) / time: the longitude synthesis' FLOPs over the whole call time
  kernel_ms[L]    device time per call of each kernel (torch.profiler, a run of its own)
  pangu_step_ms   one 4-member full-size Pangu step (synthetic weights), the same session
  spread          per perturbation ("gaussian" = K11, "spherical_grf"), at amp 0.05: the ensemble standard deviation over
                  the 4 members divided by amp sigma_c, averaged over the grid (cos-latitude weights), then the median
                  over the 69 channels, after 0, 1 and --spread-steps steps
  gpu             the card's name, power limit and maximum SM clock (the times depend on them)
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--spread-steps", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_grf.py measures on the GPU and found none")
    from bench import gpu_identity
    from skyrim_b200.config import PANGU_CHANNELS, pangu_full
    from skyrim_b200.engine import StepEngine, grf_legendre_table, perturb_ic_grf
    from skyrim_b200.ensemble import EnsembleRunner, mean_and_spread
    from skyrim_b200.weights import channel_stats, make_pangu_weights, synthetic_state

    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_identity(0), "grf_ms": {}, "lon_tflops": {}, "kernel_ms": {}}
    cfg = pangu_full()
    M, Cn, H, W = 4, len(PANGU_CHANNELS), cfg.nlat, cfg.nlon
    sig_np = channel_stats(PANGU_CHANNELS)[1]
    sigma = torch.from_numpy(sig_np).to(dev)
    x = torch.zeros((M, Cn, H, W), dtype=torch.float32, device=dev)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for L in (90, 180, 360):
        grf_legendre_table(H, L, dev)
        for _ in range(2):
            perturb_ic_grf(x, sigma, 0.05, seed=1, lmax=L)
        torch.cuda.synchronize()
        ev0.record()
        for i in range(args.iters):
            perturb_ic_grf(x, sigma, 0.05, seed=i, lmax=L)
        ev1.record()
        torch.cuda.synchronize()
        ms = ev0.elapsed_time(ev1) / args.iters
        res["grf_ms"][L] = round(ms, 3)
        res["lon_tflops"][L] = round(2.0 * M * Cn * H * W * 2 * (L + 1) / (ms * 1e-3) / 1e12, 2)
        # per-kernel device time of one call, from a profiled run of its own
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for i in range(3):
                perturb_ic_grf(x, sigma, 0.05, seed=i, lmax=L)
            torch.cuda.synchronize()
        per = {}
        for e in prof.events():
            if "grf" in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
                k = e.name.split("k_grf_")[1].split("(")[0] if "k_grf_" in e.name else e.name
                per[k] = per.get(k, 0.0) + e.device_time / 1e3 / 3
        res["kernel_ms"][L] = {k: round(v, 3) for k, v in per.items()}
    del x

    eng = StepEngine(cfg, 0)
    eng.load_weights(make_pangu_weights(cfg, 0))
    base = synthetic_state(PANGU_CHANNELS, H, W, 0)
    wlat = torch.cos(torch.linspace(np.pi / 2, -np.pi / 2, H, dtype=torch.float64, device=dev)).clamp_min(0)[:, None]
    wlat = wlat / (wlat.sum() * W)

    def spread_ratio(xm):
        _, sp = mean_and_spread(xm)
        r = (sp.double() * wlat).sum(dim=(1, 2)) / (0.05 * sigma.double())
        return float(r.median())

    res["spread"] = {}
    for name, kw in (("gaussian", {}), ("spherical_grf", dict(perturbation="spherical_grf"))):
        run = EnsembleRunner(eng, base, sig_np, members_per_gpu=M, rank=0, amp=0.05, seed=0, **kw)
        rec = {0: spread_ratio(run.x)}
        run.step(1)
        rec[1] = spread_ratio(run.x)
        if name == "gaussian":   # time the 4-member step on this runner's buffers (after the graph capture warm-up)
            run.step(3)
            torch.cuda.synchronize()
            ev0.record()
            run.step(args.iters)
            ev1.record()
            torch.cuda.synchronize()
            res["pangu_step_ms"] = round(ev0.elapsed_time(ev1) / args.iters, 3)
            run = EnsembleRunner(eng, base, sig_np, members_per_gpu=M, rank=0, amp=0.05, seed=0)
            run.step(1)
        run.step(args.spread_steps - 1)
        rec[args.spread_steps] = spread_ratio(run.x)
        res["spread"][name] = {k: round(v, 4) for k, v in rec.items()}
        del run
    eng.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
