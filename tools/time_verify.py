#!/usr/bin/env python
"""Time the rank-histogram and score-map kernels, and what a verification campaign adds to a full-size Pangu ensemble.

    python tools/time_verify.py [--iters 30] [--steps 8] [--out result.json]

Prints a table, then one JSON object:
  gpu      the card's name, power limit and maximum SM clock (the times depend on them)
  kernel   per M at 721 x 1440, all 69 channels, one global region: ms per call (CUDA events around --iters back-to-back
           calls after warm-up, median of three rounds) and the HBM bytes each call must move:
           hist   engine.forecast_rank_histogram, both launches: (M + 1) x 69 planes of fp32 read
           maps   engine.score_maps_accumulate: (M + 1) x 69 planes of fp32 read, 5 x 69 fp64 planes read and written
           with GB/s and the fraction of the H100 SXM data-sheet 3.35 TB/s
  pangu    4 full-size Pangu members, synthetic weights, three rounds alternating the two loops below, each timed with a
           host clock (ending in a synchronise) over 2 and over 2 + --steps steps; the per-lead time is the slope between
           the two medians:
           scores   EnsembleRunner.iter_scores() of all 69 channels against one truth array, as tools/time_scores.py
           campaign the same call with a rank histogram per lead and map accumulators of 4 channels at 2 map leads, on a
                    truth ring and device outputs allocated once, as GlobalModel.score_period runs each start date
           and the fixed cost per start date: the campaign's intercept, plus EnsembleRunner.restart (the next date's
           initial condition written into the members and perturbed), against the intercept of iter_scores alone, which
           allocates and pins its truth buffers on every call
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


def _events_ms(fn, iters):
    import torch
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(5):
        fn()
    rounds = []
    for _ in range(3):
        torch.cuda.synchronize()
        ev0.record()
        for _ in range(iters):
            fn()
        ev1.record()
        torch.cuda.synchronize()
        rounds.append(ev0.elapsed_time(ev1) / iters)
    return statistics.median(rounds)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_verify.py measures on the GPU and found none")
    from bench import gpu_identity
    from skyrim_b200 import scores as S
    from skyrim_b200.config import PANGU_CHANNELS, pangu_full
    from skyrim_b200.core import Skyrim
    from skyrim_b200.engine import MAP_TERMS, forecast_rank_histogram, score_maps_accumulate
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
    g = torch.Generator(device=dev).manual_seed(0)
    truth = torch.randn((Cn, cfg.nlat, cfg.nlon), device=dev, generator=g)
    maps = torch.zeros((Cn, MAP_TERMS, cfg.nlat, cfg.nlon), dtype=torch.float64, device=dev)
    print(f"{'M':>3} {'kernel':>6} {'ms':>8} {'GB':>7} {'GB/s':>7} {'of 3.35 TB/s':>12}")
    for M in (1, 4, 8, 16, 64):
        x = torch.randn((M, Cn, cfg.nlat, cfg.nlon), device=dev, generator=g)
        out = forecast_rank_histogram(x, truth, rw, 0, 0, 0)
        for kind, fn, nbytes in (
                ("hist", lambda: forecast_rank_histogram(x, truth, rw, 0, 0, 0, out=out), 4 * plane * Cn * (M + 1)),
                ("maps", lambda: score_maps_accumulate(x, truth, maps),
                 4 * plane * Cn * (M + 1) + 2 * 8 * MAP_TERMS * plane * Cn)):
            ms = _events_ms(fn, args.iters)
            row = dict(M=M, kernel=kind, ms=round(ms, 4), bytes=nbytes, gb_s=round(nbytes / ms / 1e6, 1),
                       frac_hbm=round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3))
            res["kernel"].append(row)
            print(f"{M:>3} {kind:>6} {ms:>8.3f} {nbytes / 1e9:>7.3f} {row['gb_s']:>7.0f} {row['frac_hbm']:>12.3f}")
        del x, out
    del truth, maps
    torch.cuda.empty_cache()

    sk = Skyrim("pangu", cfg=cfg)
    eng = sk.model.model.engine
    base, sig = synthetic_state(names, cfg.nlat, cfg.nlon, 0), channel_stats(names)[1]
    M = 4
    run = EnsembleRunner(eng, base, sig, members_per_gpu=M, rank=0, amp=0.05, seed=0)
    run.step(3)   # graph capture of every (in, out) pair
    torch.cuda.synchronize()
    host_truth = base + np.float32(0.1) * sig[:, None, None]
    _, rw1 = S.region_weights(lat)
    short, long_ = 2, 2 + args.steps
    mch = [names.index(c) for c in ("z500", "t850", "t2m", "msl")]
    ring = run.truth_ring(Cn)
    sums = torch.empty((long_ + 1, 1, Cn, 9), dtype=torch.float64, device=dev)
    hist = torch.empty((long_ + 1, 1, Cn, M + 1), dtype=torch.float64, device=dev)
    mp = torch.zeros((2, len(mch), MAP_TERMS, cfg.nlat, cfg.nlon), dtype=torch.float64, device=dev)

    def campaign(n):
        run.iter_scores(n, lambda k: host_truth, None, None, rw1, hist=hist[:n + 1], seed=0, date_index=0, maps=mp,
                        map_slot={1: 0, n: 1}, map_channels=mch, sums=sums[:n + 1], ring=ring)

    run.iter_scores(2, lambda n: host_truth, None, None, rw1)   # warm-up: pinned buffers, allocations
    campaign(2)
    loops = {"scores": lambda n: run.iter_scores(n, lambda k: host_truth, None, None, rw1), "campaign": campaign}
    times = {k: {short: [], long_: []} for k in loops}
    restart = []
    for _ in range(3):
        for name, fn in loops.items():
            for n in (short, long_):
                torch.cuda.synchronize()
                c = time.perf_counter()
                fn(n)
                torch.cuda.synchronize()
                times[name][n].append((time.perf_counter() - c) * 1e3)
        c = time.perf_counter()
        run.restart(base, 1)
        torch.cuda.synchronize()
        restart.append((time.perf_counter() - c) * 1e3)
    p = res["pangu"]
    for name in loops:
        med = {n: statistics.median(v) for n, v in times[name].items()}
        slope = (med[long_] - med[short]) / args.steps
        p[f"{name}_lead_ms"] = round(slope, 2)
        p[f"{name}_fixed_ms"] = round(med[short] - short * slope, 1)
    p["restart_ms"] = round(statistics.median(restart), 1)
    p["campaign_date_fixed_ms"] = round(p["campaign_fixed_ms"] + p["restart_ms"], 1)
    p["campaign_over_scores"] = round(p["campaign_lead_ms"] / p["scores_lead_ms"] - 1, 4)
    p["rounds"] = {name: {str(n): [round(v, 1) for v in t] for n, t in times[name].items()} for name in loops}
    print(f"Pangu {M} members, per lead (slope between {short} and {long_} steps): iter_scores {p['scores_lead_ms']} ms, "
          f"campaign (+ histogram, 4 map channels at 2 leads) {p['campaign_lead_ms']} ms "
          f"({100 * p['campaign_over_scores']:+.2f} %); fixed cost: iter_scores {p['scores_fixed_ms']} ms per call, "
          f"campaign {p['campaign_date_fixed_ms']} ms per date (restart {p['restart_ms']} ms)")
    sk.model.release_model()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
