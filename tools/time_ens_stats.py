#!/usr/bin/env python
"""Time the ensemble statistics kernel and what per-step statistics add to a full-size Pangu ensemble.

    python tools/time_ens_stats.py [--iters 50] [--steps 8] [--out result.json]

Prints a table, then one JSON object:
  gpu      the card's name, power limit and maximum SM clock (the times depend on them)
  kernel   per (M, n_q, n_events) at 721 x 1440, all 69 channels: ms per ``engine.ensemble_statistics`` call (CUDA events
           around --iters back-to-back calls after warm-up, median of three rounds), the bytes one call must move
           (M member planes read, 2 + n_q statistic planes per channel and n_events probability planes written), GB/s
           and the fraction of the H100 SXM data-sheet 3.35 TB/s
  pangu    4 full-size Pangu members, synthetic weights, --steps steps, three alternated rounds (medians):
           bare_step_ms        EnsembleRunner.step() per step (host clock, ends in a synchronise)
           stats_step_ms       EnsembleRunner.iter_stats() per step in steady state: step, reduction of all 69 channels with
                               3 quantiles and 4 events, device->host copy of the statistics under the next step
           fresh_step_ms       the slope of the wall time of a freshly built EnsembleRunner (spherical_grf) followed by n
                               bare steps, between n = 2 and n = 2 + --steps: what predict_ensemble runs minus the statistics
           predict_step_ms     the same slope for predict_ensemble(save=False): all 69 channels, 3 quantiles, 4 events
           predict_fixed_ms    its intercept (IC synthesis, perturbation, pinned host buffers, the returned arrays)
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12    # H100 SXM data sheet
Q3 = (0.1, 0.5, 0.9)
EVENTS = {"t2m": [273.15], "u10m": [15.0], "msl": [100000.0], "z500": [55000.0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import datetime

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_ens_stats.py measures on the GPU and found none")
    from bench import gpu_identity
    from skyrim_b200.config import PANGU_CHANNELS, pangu_full
    from skyrim_b200.core import Skyrim
    from skyrim_b200.engine import ensemble_statistics
    from skyrim_b200.ensemble import EnsembleRunner
    from skyrim_b200.weights import channel_stats, synthetic_state

    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_identity(0), "kernel": [], "pangu": {}}
    print(f"{res['gpu']['name']}, power limit {res['gpu']['power_limit_w']} W, max SM clock {res['gpu']['sm_max_mhz']} MHz")
    cfg = pangu_full()
    Cn, plane = len(PANGU_CHANNELS), cfg.nlat * cfg.nlon
    names = PANGU_CHANNELS
    ev_all = [(names.index(c), t) for c in names if c in EVENTS for t in EVENTS[c]]
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    g = torch.Generator(device=dev).manual_seed(0)
    print(f"{'M':>3} {'n_q':>3} {'n_ev':>4} {'ms':>8} {'GB':>7} {'GB/s':>7} {'of 3.35 TB/s':>12}")
    for M in (4, 8, 16):
        x = torch.randn((M, Cn, cfg.nlat, cfg.nlon), device=dev, generator=g)
        for q in ((), Q3):
            for ev in ((), ev_all):
                out = ensemble_statistics(x, None, q, ev)
                for _ in range(5):
                    ensemble_statistics(x, None, q, ev, out=out)
                rounds = []
                for _ in range(3):
                    torch.cuda.synchronize()
                    ev0.record()
                    for _ in range(args.iters):
                        ensemble_statistics(x, None, q, ev, out=out)
                    ev1.record()
                    torch.cuda.synchronize()
                    rounds.append(ev0.elapsed_time(ev1) / args.iters)
                ms = statistics.median(rounds)
                nbytes = 4 * plane * (M * Cn + (2 + len(q)) * Cn + len(ev))
                row = dict(M=M, n_q=len(q), n_events=len(ev), ms=round(ms, 4), bytes=nbytes,
                           gb_s=round(nbytes / ms / 1e6, 1), frac_hbm=round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3))
                res["kernel"].append(row)
                print(f"{M:>3} {len(q):>3} {len(ev):>4} {ms:>8.3f} {nbytes / 1e9:>7.3f} {row['gb_s']:>7.0f} {row['frac_hbm']:>12.3f}")
                del out
        del x
    torch.cuda.empty_cache()

    sk = Skyrim("pangu", cfg=cfg)
    eng = sk.model.model.engine
    base, sig = synthetic_state(names, cfg.nlat, cfg.nlon, 0), channel_stats(names)[1]
    run = EnsembleRunner(eng, base, sig, members_per_gpu=4, rank=0, amp=0.05, seed=0)
    run.step(3)   # graph capture of every (in, out) pair
    torch.cuda.synchronize()
    t0 = datetime.datetime(2024, 5, 7)
    kw = dict(members=4, quantiles=Q3, events=EVENTS, save=False)
    sk.model.predict_ensemble(t0, n_steps=2, **kw)   # warm-up: allocations, GRF tables
    bare, stats_steps, pred_short, pred_long, fresh_short, fresh_long = [], [], [], [], [], []

    def fresh(n):
        r = EnsembleRunner(eng, base, sig, members_per_gpu=4, rank=0, amp=0.05, seed=0, perturbation="spherical_grf")
        r.step(n)

    for _ in range(3):
        c = time.perf_counter()
        run.step(args.steps)
        torch.cuda.synchronize()
        bare.append((time.perf_counter() - c) * 1e3 / args.steps)
        it = run.iter_stats(args.steps, None, Q3, ev_all)
        next(it)
        c = time.perf_counter()
        for _ in it:
            pass
        stats_steps.append((time.perf_counter() - c) * 1e3 / args.steps)
        for n, acc, facc in ((2, pred_short, fresh_short), (2 + args.steps, pred_long, fresh_long)):
            for fn, a in ((lambda: fresh(n), facc), (lambda: sk.model.predict_ensemble(t0, n_steps=n, **kw), acc)):
                torch.cuda.synchronize()
                c = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                a.append((time.perf_counter() - c) * 1e3)
    p = res["pangu"]
    p["bare_step_ms"] = round(statistics.median(bare), 2)
    p["stats_step_ms"] = round(statistics.median(stats_steps), 2)
    slope = (statistics.median(pred_long) - statistics.median(pred_short)) / args.steps
    p["predict_step_ms"] = round(slope, 2)
    p["predict_fixed_ms"] = round(statistics.median(pred_short) - 2 * slope, 1)
    p["fresh_step_ms"] = round((statistics.median(fresh_long) - statistics.median(fresh_short)) / args.steps, 2)
    p["stats_overhead"] = round(p["stats_step_ms"] / p["bare_step_ms"] - 1, 4)
    p["predict_overhead"] = round(p["predict_step_ms"] / p["fresh_step_ms"] - 1, 4)
    p["rounds"] = dict(bare=[round(v, 2) for v in bare], stats=[round(v, 2) for v in stats_steps],
                       predict_short=[round(v, 1) for v in pred_short], predict_long=[round(v, 1) for v in pred_long],
                       fresh_short=[round(v, 1) for v in fresh_short], fresh_long=[round(v, 1) for v in fresh_long])
    print(f"Pangu 4 members: bare step {p['bare_step_ms']} ms, with statistics {p['stats_step_ms']} ms "
          f"({100 * p['stats_overhead']:+.2f} %); per step from a fresh runner {p['fresh_step_ms']} ms, predict_ensemble "
          f"{p['predict_step_ms']} ms ({100 * p['predict_overhead']:+.2f} %), fixed {p['predict_fixed_ms']} ms")
    sk.model.release_model()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
