"""Timing of the model comparison on one GPU, in one process (DESIGN.md section 5, "Model comparison"):

  1. the three pooled verification entries (K = 3 sources x 4 members, 56 channels, 2 regions, with a climatology) against
     the single-source entries reading the same planes from one contiguous tensor: ms (median of CUDA-event timings) and
     the fraction of 3.35 TB/s for the member and truth bytes each reads;
  2. GlobalEnsemble.compare of the deterministic trio per lead, as the slope between 2 and 10 leads over three alternated
     rounds, against bare GlobalEnsemble._step_all;
  3. the device memory in use (cudaMemGetInfo) after a trio comparison at M = 1 and at the largest M per model that fits
     with one map channel.

    python tools/time_compare.py [--grid 721x1440] [--out time_compare.json]

Prints one JSON object with the card name, power limit and maximum SM clock read in the same run."""
import argparse
import datetime
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_BW = 3.35e12
NAMES = ("pangu", "fourcastnet_v2", "graphcast")
T0 = datetime.datetime(2024, 5, 7)


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [v.strip() for v in out.stdout.strip().splitlines()[0].split(",")])) if out.stdout else {}


def time_ms(fn, reps=20):
    import torch
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def kernels(H, W):
    import torch
    from skyrim_b200 import engine as E
    from skyrim_b200 import scores as S
    from skyrim_b200.timeloop import equiangular_grid
    g = torch.Generator(device="cuda").manual_seed(0)
    counts, M, n_sel = (69, 73, 83), 4, 56
    srcs = [torch.randn(M, c, H, W, device="cuda", generator=g) for c in counts[:2]]
    gc = torch.randn(M, 2 * counts[2], H, W, device="cuda", generator=g)
    srcs.append(gc[:, counts[2]:])
    rng = np.random.default_rng(0)
    chans = [sorted(int(c) for c in rng.permutation(c)[:n_sel]) for c in counts]
    pooled = torch.cat([x[:, ch] for x, ch in zip(srcs, chans)]).contiguous()   # (12, 56, H, W): source 0's order = 0..55
    truth = torch.randn(n_sel, H, W, device="cuda", generator=g)
    clim = torch.randn(n_sel, H, W, device="cuda", generator=g)
    _, w = S.region_weights(np.asarray(equiangular_grid(H, W).lat), {"global": (-90, 90), "tropics": (-20, 20)})
    rw = torch.as_tensor(w, device="cuda").contiguous()
    one = list(range(n_sel))
    maps = torch.zeros((n_sel, E.MAP_TERMS, H, W), dtype=torch.float64, device="cuda")
    plane = 4 * H * W
    runs = {
        "scores": (lambda: E.forecast_scores_multi(srcs, chans, truth, rw, clim),
                   lambda: E.forecast_scores(pooled, truth, rw, one, clim), (3 * M + 2) * n_sel * plane),
        "rank_histogram": (lambda: E.forecast_rank_histogram_multi(srcs, chans, truth, rw, 0, 0, 1),
                           lambda: E.forecast_rank_histogram(pooled, truth, rw, 0, 0, 1, one), (3 * M + 1) * n_sel * plane),
        "score_maps": (lambda: E.score_maps_accumulate_multi(srcs, chans, truth, maps),
                       lambda: E.score_maps_accumulate(pooled, truth, maps, one),
                       (3 * M + 1) * n_sel * plane + 2 * 8 * E.MAP_TERMS * n_sel * H * W),
    }
    out = {}
    for name, (multi, single, nbytes) in runs.items():
        tm, ts = time_ms(multi), time_ms(single)
        out[name] = dict(pooled_ms=tm, single_ms=ts, bytes=nbytes, pooled_frac_of_peak=nbytes / (tm * 1e-3) / PEAK_BW,
                         single_frac_of_peak=nbytes / (ts * 1e-3) / PEAK_BW, pooled_over_single=tm / ts)
    del srcs, gc, pooled, maps
    torch.cuda.empty_cache()
    return out


def trio_per_lead(sk):
    """the truth is a DataArray in host memory, so the per-lead host fetch is a slice, not a synthetic field drawn per call"""
    import torch
    from skyrim_b200 import xr_shim as xr
    ens = sk.model
    times = [T0 + n * ens.time_step for n in range(11)]
    first = ens.data_source[T0]
    truth = xr.DataArray(np.stack([np.asarray(ens.data_source[t].values, dtype=np.float32) for t in times]),
                         dims=["time", "channel", "lat", "lon"],
                         coords=dict(time=np.array([np.datetime64(t, "s") for t in times]),
                                     channel=np.asarray(first.coords["channel"]), lat=np.asarray(first.coords["lat"]),
                                     lon=np.asarray(first.coords["lon"])))

    def bare(n):
        states = ens._initial_states(T0)
        torch.cuda.synchronize()
        t = time.perf_counter()
        for i in range(n):
            ens._step_all(states, first=i == 0)
        torch.cuda.synchronize()
        return time.perf_counter() - t

    def comp(n):
        torch.cuda.synchronize()
        t = time.perf_counter()
        ens.compare([T0], n, truth=truth)
        torch.cuda.synchronize()
        return time.perf_counter() - t

    comp(1)                                        # warm-up: pinned buffers, graphs
    bare(2)
    rounds = []
    for _ in range(3):
        b = (bare(10) - bare(2)) / 8
        c = (comp(10) - comp(2)) / 8
        rounds.append(dict(bare_ms_per_lead=1e3 * b, compare_ms_per_lead=1e3 * c, overhead=c / b - 1))
    return rounds


def used_gb():
    import torch
    free, total = torch.cuda.mem_get_info()
    return (total - free) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", default="721x1440")
    ap.add_argument("--out", default="")
    ap.add_argument("--skip_trio", action="store_true")
    a = ap.parse_args()
    import torch
    from skyrim_b200.core.skyrim import Skyrim
    H, W = (int(v) for v in a.grid.split("x"))
    res = dict(gpu=gpu_info(), grid=[H, W], kernels=kernels(H, W))
    print(json.dumps(res["kernels"]), flush=True)
    if not a.skip_trio:
        sk = Skyrim(*NAMES)
        res["trio_per_lead"] = trio_per_lead(sk)
        print(json.dumps(res["trio_per_lead"]), flush=True)
        res["memory_gb"] = {"M=1": used_gb()}
        sk.model.compare([T0], 1)
        res["memory_gb"]["M=1"] = used_gb()
        for M in (4, 3, 2):
            try:
                sk.model.compare([T0], 1, members=M, map_leads=[6], map_channels=["z500"])
                torch.cuda.synchronize()
                res["memory_gb"][f"M={M} (largest that fits, one map channel)"] = used_gb()
                break
            except (RuntimeError, torch.cuda.OutOfMemoryError) as e:
                res["memory_gb"][f"M={M}"] = f"does not fit: {str(e)[:120]}"
                torch.cuda.empty_cache()
        sk.model.release_model()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
