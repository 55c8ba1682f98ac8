#!/usr/bin/env python
"""Time the forecast-score kernels and what scoring every lead adds to a full-size Pangu ensemble.

    python tools/time_scores.py [--iters 50] [--steps 8] [--out result.json]

Prints a table, then one JSON object:
  gpu      the card's name, power limit and maximum SM clock (the times depend on them)
  kernel   per (M, clim) at 721 x 1440, all 69 channels, one global region: ms per ``engine.forecast_scores`` call (both
           launches; CUDA events around --iters back-to-back calls after warm-up, median of three rounds), the bytes one
           call must read ((M + 1 + [clim]) x 69 planes of fp32), GB/s and the fraction of the H100 SXM data-sheet 3.35 TB/s
  pangu    4 full-size Pangu members, synthetic weights, three rounds alternating the three loops below; each loop is
           timed with a host clock (ending in a synchronise) over 2 and over 2 + --steps steps, and the per-step time is
           the slope between the two medians (the intercept, the loop's fixed cost of buffers and pinned memory, is
           reported as *_fixed_ms):
           bare     EnsembleRunner.step()
           stats    EnsembleRunner.iter_stats(): the step, mean and spread of all 69 channels, their device->host copy
                    under the next step
           scores   EnsembleRunner.iter_scores(): the step, the truth (one host fp32 (69, 721, 1440) array, 287 MB, per
                    lead) copied into pinned memory and uploaded on a copy stream, the scores of all 69 channels against it
                    and a climatology in two regions; the sums of every lead copied back at the end
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12    # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_scores.py measures on the GPU and found none")
    from bench import gpu_identity
    from skyrim_b200 import scores as S
    from skyrim_b200.config import PANGU_CHANNELS, pangu_full
    from skyrim_b200.core import Skyrim
    from skyrim_b200.engine import forecast_scores
    from skyrim_b200.ensemble import EnsembleRunner
    from skyrim_b200.timeloop import equiangular_grid
    from skyrim_b200.weights import channel_stats, synthetic_state

    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_identity(0), "kernel": [], "pangu": {}}
    print(f"{res['gpu']['name']}, power limit {res['gpu']['power_limit_w']} W, max SM clock {res['gpu']['sm_max_mhz']} MHz")
    cfg = pangu_full()
    names = PANGU_CHANNELS
    Cn, plane = len(names), cfg.nlat * cfg.nlon
    lat = equiangular_grid(cfg.nlat, cfg.nlon).lat
    rw = torch.from_numpy(S.region_weights(lat)[1]).to(dev)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g = torch.Generator(device=dev).manual_seed(0)
    truth = torch.randn((Cn, cfg.nlat, cfg.nlon), device=dev, generator=g)
    clim = torch.randn((Cn, cfg.nlat, cfg.nlon), device=dev, generator=g)
    print(f"{'M':>3} {'clim':>4} {'ms':>8} {'GB':>7} {'GB/s':>7} {'of 3.35 TB/s':>12}")
    for M in (1, 4, 8, 16, 64):
        x = torch.randn((M, Cn, cfg.nlat, cfg.nlon), device=dev, generator=g)
        for k in (None, clim):
            out = forecast_scores(x, truth, rw, None, k)
            for _ in range(5):
                forecast_scores(x, truth, rw, None, k, out=out)
            rounds = []
            for _ in range(3):
                torch.cuda.synchronize()
                ev0.record()
                for _ in range(args.iters):
                    forecast_scores(x, truth, rw, None, k, out=out)
                ev1.record()
                torch.cuda.synchronize()
                rounds.append(ev0.elapsed_time(ev1) / args.iters)
            ms = statistics.median(rounds)
            nbytes = 4 * plane * Cn * (M + 1 + (k is not None))
            row = dict(M=M, clim=k is not None, ms=round(ms, 4), bytes=nbytes, gb_s=round(nbytes / ms / 1e6, 1),
                       frac_hbm=round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3))
            res["kernel"].append(row)
            print(f"{M:>3} {int(k is not None):>4} {ms:>8.3f} {nbytes / 1e9:>7.3f} {row['gb_s']:>7.0f} {row['frac_hbm']:>12.3f}")
        del x
    del truth, clim
    torch.cuda.empty_cache()

    sk = Skyrim("pangu", cfg=cfg)
    eng = sk.model.model.engine
    base, sig = synthetic_state(names, cfg.nlat, cfg.nlon, 0), channel_stats(names)[1]
    run = EnsembleRunner(eng, base, sig, members_per_gpu=4, rank=0, amp=0.05, seed=0)
    run.step(3)   # graph capture of every (in, out) pair
    torch.cuda.synchronize()
    host_truth = base + np.float32(0.1) * sig[:, None, None]
    host_clim = np.broadcast_to(channel_stats(names)[0][:, None, None], base.shape).astype(np.float32)
    _, rw2 = S.region_weights(lat, {"global": (-90, 90), "tropics": (-20, 20)})
    run.iter_scores(2, lambda n: host_truth, host_clim, None, rw2)   # warm-up: pinned buffers, allocations
    short, long_ = 2, 2 + args.steps
    loops = {
        "bare": lambda n: run.step(n),
        "stats": lambda n: [None for _ in run.iter_stats(n)],
        "scores": lambda n: run.iter_scores(n, lambda k: host_truth, host_clim, None, rw2),
    }
    times = {k: {short: [], long_: []} for k in loops}
    for _ in range(3):
        for name, fn in loops.items():
            for n in (short, long_):
                torch.cuda.synchronize()
                c = time.perf_counter()
                fn(n)
                torch.cuda.synchronize()
                times[name][n].append((time.perf_counter() - c) * 1e3)
    p = res["pangu"]
    for name in loops:
        med = {n: statistics.median(v) for n, v in times[name].items()}
        slope = (med[long_] - med[short]) / args.steps
        p[f"{name}_step_ms"] = round(slope, 2)
        p[f"{name}_fixed_ms"] = round(med[short] - short * slope, 1)
    p["scores_over_stats"] = round(p["scores_step_ms"] / p["stats_step_ms"] - 1, 4)
    p["scores_over_bare"] = round(p["scores_step_ms"] / p["bare_step_ms"] - 1, 4)
    p["rounds"] = {name: {str(n): [round(v, 1) for v in t] for n, t in times[name].items()} for name in loops}
    print(f"Pangu 4 members, per step (slope between {short} and {long_} steps): bare {p['bare_step_ms']} ms, iter_stats "
          f"{p['stats_step_ms']} ms, iter_scores {p['scores_step_ms']} ms ({100 * p['scores_over_bare']:+.2f} % over bare, "
          f"{100 * p['scores_over_stats']:+.2f} % over iter_stats); fixed cost per call: bare {p['bare_fixed_ms']} ms, "
          f"iter_stats {p['stats_fixed_ms']} ms, iter_scores {p['scores_fixed_ms']} ms")
    sk.model.release_model()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
