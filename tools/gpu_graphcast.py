"""Full-size GraphCast step on the GPU: timing, per-family breakdown, comparison with the committed oracle fixture.

    python tools/gpu_graphcast.py [steps]      (run under gpurun; writes gpurun_out/graphcast_full.json)
"""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    from skyrim_b200 import icomesh, roofline as R
    from skyrim_b200.config import graphcast_full
    from skyrim_b200.engine import StepEngine, launch_count
    from skyrim_b200.timeloop import GraphcastTimeLoop
    from skyrim_b200.verify import compare_graphcast, load_fixture
    from skyrim_b200.weights import make_graphcast_weights, synthetic_graphcast_state
    cfg = graphcast_full()
    t0 = time.time()
    graph = icomesh.build_graph(cfg.nlat, cfg.nlon, cfg.mesh_levels, cfg.radius_frac)
    t_graph = time.time() - t0
    eng = StepEngine(cfg, 0, graph=graph)
    t0 = time.time()
    w = make_graphcast_weights(cfg, 0)
    eng.load_weights(w)
    torch.cuda.synchronize()
    t_load = time.time() - t0
    loop = GraphcastTimeLoop(eng)
    T0 = 1714521600.0
    x = torch.from_numpy(synthetic_graphcast_state(cfg, 0)).reshape(1, 2, cfg.n_state, cfg.nlat, cfg.nlon).cuda()
    loop.fill_forcing(x, T0)
    x = x.reshape(1, 2 * cfg.n_state, cfg.nlat, cfg.nlon).contiguous()
    y, z = torch.empty_like(x), torch.empty_like(x)
    print(f"graph {t_graph:.1f} s, weights + load {t_load:.1f} s, workspace {eng._L.sky_model_workspace_bytes(eng._h, 1) / 2**30:.1f} GiB, "
          f"allocated {torch.cuda.memory_allocated() / 2**30:.1f} GiB (torch) ", flush=True)
    eng.set_clock(T0)
    eng.step(x, z)
    torch.cuda.synchronize()
    cmp = compare_graphcast(z[0], x[0], w["norm.diff_std"], load_fixture("graphcast"), cfg)
    print("verify:", json.dumps(cmp), flush=True)
    # family breakdown
    eng.set_clock(T0)
    eng.profile_begin()
    eng.step(x, y)
    fam = eng.profile_end()
    fl, by = R.graphcast_flops(cfg, graph), R.graphcast_bytes(cfg, graph)
    rows = {}
    for k, (ms, n) in sorted(fam.items(), key=lambda kv: -kv[1][0]):
        rows[k] = dict(ms=round(ms, 3), launches=n, tflops=round(fl.get(k, 0) / ms / 1e9, 1), gbs=round(by.get(k, 0) / ms / 1e6, 1))
        print(f"{k:10s} {ms:8.3f} ms  {n:3d} launches  {rows[k]['tflops']:7.1f} TFLOP/s  {rows[k]['gbs']:7.1f} GB/s")
    # timed chain
    eng.set_clock(T0)
    for _ in range(3):
        eng.step(x, y); eng.step(y, z); eng.step(z, y)
    torch.cuda.synchronize()
    l0 = launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    src, dst = x, y
    for i in range(steps):
        eng.step(src, dst)
        src, dst = dst, (z if dst is y else y)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    rec = dict(ms_per_step=ms, steps=steps, launches_per_step=(launch_count() - l0) / steps, families=rows, verify=cmp,
               step_tflops=fl["total"] / ms / 1e9, flops=fl, bytes=by)
    print(f"GraphCast 721x1440: {ms:.2f} ms/step, {rec['step_tflops']:.0f} TFLOP/s algorithmic, finite {bool(torch.isfinite(src).all())}")
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(rec, open(os.path.join(ROOT, "gpurun_out", "graphcast_full.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
