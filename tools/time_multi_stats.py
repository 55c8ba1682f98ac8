#!/usr/bin/env python
"""Time the multi-source statistics kernel and a full-size Pangu + FourCastNet-v2 + GraphCast ensemble on one GPU.

    python tools/time_multi_stats.py [--iters 50] [--steps 3] [--out result.json]

Prints a table, then one JSON object:
  gpu      the card's name, power limit and maximum SM clock (the times depend on them)
  kernel   at 721 x 1440, 56 channels, 3 quantiles: ms per call (CUDA events around --iters back-to-back calls after
           warm-up, median of three rounds) of
             multi   engine.multi_model_statistics over 3 sources x 4 members (per-source means on)
             single  engine.ensemble_statistics over one 12-member tensor, the same channels
           with the bytes each must move (member planes read, statistic planes written), GB/s and the fraction of the
           H100 SXM data-sheet 3.35 TB/s
  trio     the three full-size engines (synthetic weights) on this GPU; for M = 1 and 4 members per model:
             step_ms        one step of all three engines plus the reduction, per step (host clock over --steps steps,
                            ends in a synchronise), and alone_ms each engine's own step over the same members
             used_gb        device memory in use (cudaMemGetInfo: free before building anything minus free after the run;
                            the allocator keeps what it reserved, so this is the peak of the run)
           A member count that does not fit is reported with the error instead of numbers.
"""
from __future__ import annotations

import argparse
import datetime
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12    # H100 SXM data sheet
Q3 = (0.1, 0.5, 0.9)
NAMES = ("pangu", "fourcastnet_v2", "graphcast")


def time_calls(fn, iters):
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
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_multi_stats.py measures on the GPU and found none")
    from bench import gpu_identity
    from skyrim_b200.config import FCNV2_CHANNELS, GRAPHCAST_CHANNELS, PANGU_CHANNELS
    from skyrim_b200.engine import ensemble_statistics, multi_model_statistics

    dev = torch.device("cuda", 0)
    res = {"gpu": gpu_identity(0), "kernel": {}, "trio": {}}
    print(f"{res['gpu']['name']}, power limit {res['gpu']['power_limit_w']} W, max SM clock {res['gpu']['sm_max_mhz']} MHz")
    free0 = torch.cuda.mem_get_info(dev)[0]

    nlat, nlon = 721, 1440
    plane = nlat * nlon
    shared = [c for c in PANGU_CHANNELS if c in FCNV2_CHANNELS and c in GRAPHCAST_CHANNELS]
    g = torch.Generator(device=dev).manual_seed(0)
    srcs = [torch.randn((4, len(n), nlat, nlon), device=dev, generator=g) for n in (PANGU_CHANNELS, FCNV2_CHANNELS)]
    gc = torch.randn((4, 2 * len(GRAPHCAST_CHANNELS), nlat, nlon), device=dev, generator=g)
    srcs.append(gc[:, len(GRAPHCAST_CHANNELS):])
    chans = [[n.index(c) for c in shared] for n in (PANGU_CHANNELS, FCNV2_CHANNELS, GRAPHCAST_CHANNELS)]
    one = torch.randn((12, len(PANGU_CHANNELS), nlat, nlon), device=dev, generator=g)
    out_m = multi_model_statistics(srcs, chans, Q3)
    out_s = ensemble_statistics(one, chans[0], Q3)
    nsel = len(shared)
    for name, fn, nbytes in (
            ("multi", lambda: multi_model_statistics(srcs, chans, Q3, out=out_m), 4 * plane * nsel * (12 + 2 + 3 + 3)),
            ("single", lambda: ensemble_statistics(one, chans[0], Q3, out=out_s), 4 * plane * nsel * (12 + 2 + 3))):
        ms = time_calls(fn, args.iters)
        row = dict(ms=round(ms, 4), bytes=nbytes, gb_s=round(nbytes / ms / 1e6, 1),
                   frac_hbm=round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3))
        res["kernel"][name] = row
        print(f"{name:>6}: {ms:.3f} ms, {nbytes / 1e9:.3f} GB, {row['gb_s']:.0f} GB/s, {row['frac_hbm']:.3f} of 3.35 TB/s")
    del srcs, gc, one, out_m, out_s
    torch.cuda.empty_cache()

    from skyrim_b200.core import Skyrim
    t0 = datetime.datetime(2024, 5, 7)
    sk = Skyrim(*NAMES)
    ens = sk.model
    res["trio"]["built_gb"] = round((free0 - torch.cuda.mem_get_info(dev)[0]) / 1e9, 2)
    sel = ens._shared_index(ens.shared_channels)
    for M in (1, 4):
        row = {}
        try:
            states = ens._initial_states(t0) if M == 1 else ens.ensemble_members(t0, M, "gaussian")
            q = () if M == 1 else Q3
            out = multi_model_statistics(ens._outputs(states), sel, q)

            def step():
                ens._step_all(states)
                multi_model_statistics(ens._outputs(states), sel, q, out=out)

            rounds = []
            for r in range(4):   # the first round warms up (graph capture of each (in, out) pair)
                torch.cuda.synchronize()
                c = time.perf_counter()
                for _ in range(args.steps):
                    step()
                torch.cuda.synchronize()
                if r:
                    rounds.append((time.perf_counter() - c) * 1e3 / args.steps)
            row["step_ms"] = round(statistics.median(rounds), 1)
            row["rounds"] = [round(v, 1) for v in rounds]
            alone = {}
            for k, (name, m) in enumerate(zip(NAMES, ens.models)):
                x = states[k]
                y = torch.empty_like(x)
                m.model.engine.step(x, y)
                torch.cuda.synchronize()
                c = time.perf_counter()
                for _ in range(args.steps):
                    m.model.engine.step(x, y)
                    x, y = y, x
                torch.cuda.synchronize()
                alone[name] = round((time.perf_counter() - c) * 1e3 / args.steps, 1)
            row["alone_ms"] = alone
            row["used_gb"] = round((free0 - torch.cuda.mem_get_info(dev)[0]) / 1e9, 2)
            del states, out
        except Exception as e:   # a member count that does not fit in memory
            row["error"] = f"{type(e).__name__}: {e}"[:300]
        torch.cuda.empty_cache()
        res["trio"][f"M{M}"] = row
        print(f"M = {M} per model: {row}")
    ens.release_model()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
