"""The GraphCast engine unit by unit (debug_set "stop_launch" + raw debug_copy taps) against float64 references.

Graphs: six icosahedral ones — 41x96 / mesh 2 / 2 layers; 33x64 / mesh 1 / 3 layers; 49x120 / mesh 3 / 1 layer (one layer
that is first and last); 32x64 (n_grid a whole number of row tiles: no padding in the mesh2grid segments); 7x16 (112 grid
points: every grid-sized GEMM is one partial tile) and 8x16 (exactly one tile) — and a hand-built one
(oracle/graphcast_stages_ref.hand_graph) whose grid2mesh in-degrees are 0, 1, 3, 4, 5, 63, 64, 65, 127, 128, 129, 256, 257
and 4321 and whose mesh in-degrees are 0, 1, 64, 65 and 200.

- stage-local: every unit from the engine's own inputs to it, per element, zero outside, rows of a partial tile included;
- chained: every latent, update and aggregate against the fp64 oracle's taps, per row;
- a workspace full of NaN bytes, a previous step's leftovers and a NaN member change no valid bit;
- the feature-count limit, the range guard on partial tiles, the launch count of a step;
- the full 721 x 1440 grid with the refinement-6 multimesh and 16 layers: every unit on the rows of
  graphcast_stages_ref.full_size_rows (every mesh-node row, every mesh-edge row of the first and last two layers, the
  tiles around byte 2^31 of the mesh2grid images, every partial tile, every cut grid2mesh segment with all its edges),
  gathered on the device.
"""
import dataclasses
import functools
import resource
import time

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

T0 = 1714521600.0  # 2024-05-01T00:00:00Z
CASES = {"41x96-m2-L2": (41, 96, 2, 2, False), "33x64-m1-L3": (33, 64, 1, 3, False), "49x120-m3-L1": (49, 120, 3, 1, False),
         "32x64-m1-L1": (32, 64, 1, 1, False), "7x16-m1-L1": (7, 16, 1, 1, False), "8x16-m1-L1": (8, 16, 1, 1, False),
         "hand-41x96-m2-L1": (41, 96, 2, 1, True)}


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _inputs(case, seed=0, **cfg_kw):
    from oracle import graphcast_stages_ref as st
    from skyrim_b200 import icomesh
    from skyrim_b200.config import graphcast_small
    from skyrim_b200.weights import make_graphcast_weights
    nlat, nlon, levels, layers, hand = CASES[case]
    cfg = dataclasses.replace(graphcast_small(nlat, nlon, levels, 512, layers), **cfg_kw)
    graph = icomesh.build_graph(cfg.nlat, cfg.nlon, cfg.mesh_levels, cfg.radius_frac)
    if hand:
        graph = st.hand_graph(graph)
    return cfg, graph, make_graphcast_weights(cfg, 0), _state(cfg, seed)


def _state(cfg, seed):
    """the seeded state, its two toa forcing planes at T0 - 6 h and T0"""
    from oracle.graphcast_ref import toa_radiation
    from skyrim_b200.weights import synthetic_graphcast_state
    x = synthetic_graphcast_state(cfg, seed)
    lat = np.linspace(90.0, -90.0, cfg.nlat); lon = np.arange(cfg.nlon) * (360.0 / cfg.nlon)
    x[cfg.n_state - 1] = toa_radiation(T0 - 21600.0, lat, lon)
    x[2 * cfg.n_state - 1] = toa_radiation(T0, lat, lon)
    return x


def _engine(cfg, graph, w):
    from skyrim_b200.engine import StepEngine
    eng = StepEngine(cfg, 0, graph=graph)
    eng.load_weights(w)
    return eng


def _step(eng, x):
    eng.set_clock(T0)
    return eng.step(torch.from_numpy(np.ascontiguousarray(x)).reshape((-1,) + x.shape[-3:]).cuda()).cpu().numpy()


def _read_taps(eng, cfg, graph, x, fill=None):
    """{0: statics, n: taps of unit n}, decoded, valid rows only.  Every unit is read after a step of its own that stops
    right behind it (the workspace is reused); ``fill``: byte written over the whole workspace before each of those steps"""
    from oracle import graphcast_stages_ref as st
    sh = st.Shapes(cfg, graph)
    read = lambda name, rows, cols=None: sh.decode(name, eng.debug_tensor(name, (sh.tap_floats(name),)).cpu().numpy(), rows, cols)
    xs = torch.from_numpy(x)[None].cuda()
    ws = eng._workspace(1)
    rows0 = {"vm0": sh.Nm, "vm0_img": sh.Nm, "e_g2m_img": sh.Eg, "e_m2g_img": sh.m2g_rows, "e_mesh_img": sh.Em, "g2m_tr": sh.Nm}
    taps = {0: {k: read(k, r) for k, r in rows0.items()}}
    try:
        for n, (kind, name, outs) in enumerate(st.units(cfg, graph), 1):
            if fill is not None:
                ws.fill_(fill)
            eng.set_clock(T0)
            eng.debug_set("stop_launch", n)
            y = eng.step(xs)
            taps[n] = {tap: y[0].cpu().numpy() if tap == "x_out" else
                       read(tap, sh.Ng if tap == "feat" else sh.m2g_rows if kmajor else rows, cols)
                       for tap, (rows, kmajor, cols) in outs.items()}
    finally:
        eng.debug_set("stop_launch", -1)
    return taps


@functools.lru_cache(maxsize=None)
def _case(case):
    cfg, graph, w, x = _inputs(case)
    eng = _engine(cfg, graph, w)
    taps = _read_taps(eng, cfg, graph, x)
    y = _step(eng, x)[0]
    eng.close()
    return cfg, graph, w, x, taps, y


@pytest.mark.parametrize("case", list(CASES))
def test_units_against_stage_local_references(case):
    """every unit from the engine's own inputs: no element outside its bound, no NaN; one line per check.  Largest ratios
    to the bound per stage over the seven graphs: DESIGN.md, "GraphCast unit by unit"."""
    _need_gpu()
    from oracle import graphcast_stages_ref as st
    cfg, graph, w, x, taps, y = _case(case)
    res = st.check_step(cfg, graph, w, x, T0, taps)
    for n, kind, name, what, bad, wr in res:
        print(f"{case} unit {n:2d} {kind:8s} {name:20s} {what:24s} worst |D-R|/bound {wr:.3f}  outside {bad}")
    print(f"{case} per stage: " + ", ".join(f"{k} {v:.3f}" for k, v in st.by_stage(res).items()))
    assert not [r for r in res if r[4]], [r for r in res if r[4]]
    last = max(taps)
    assert np.array_equal(y, taps[last]["x_out"]), "a step stopped behind its last unit is the whole step"


@pytest.mark.parametrize("case", list(CASES))
def test_units_chained_against_the_oracle(case):
    """each tap against the fp64 oracle's, per ROW: relative L2 within 4x the largest row error of the oracle's own fp16
    emulation of that tap (at least 1e-3: two fp16 roundings of a row)"""
    _need_gpu()
    from oracle import graphcast_stages_ref as st
    cfg, graph, w, x, taps, y = _case(case)
    ref, tol = st.chain_bounds(cfg, graph, w, x, T0)
    bad = []
    for name, got in st.chain_pairs(cfg, graph, w, x, taps):
        e = st.row_rel(got, ref[name])
        print(f"{case} chained {name:14s} worst row rel L2 {e.max():.3e} (row {int(e.argmax())})  bound {tol[name]:.3e}")
        if not e.max() <= tol[name]:
            bad.append((name, float(e.max()), int(e.argmax()), tol[name]))
    assert not bad, bad


def _same_taps(a, b):
    return [(n, k) for n in a for k in a[n] if not np.array_equal(a[n][k], b[n][k], equal_nan=True)]


@pytest.mark.parametrize("case", ["hand-41x96-m2-L1", "7x16-m1-L1"])
def test_poisoned_workspace_reaches_no_valid_output(case):
    """workspace filled with 0xFF bytes (NaN in fp16 and in fp32) before every step: the new state and the valid rows of
    every tap equal, bit for bit, those of a zero-filled workspace — no padded row, stale buffer or row of a node without
    edges is read into a valid output"""
    _need_gpu()
    cfg, graph, w, x = _inputs(case)
    eng = _engine(cfg, graph, w)
    t0 = _read_taps(eng, cfg, graph, x, fill=0)
    t1 = _read_taps(eng, cfg, graph, x, fill=0xFF)
    eng._workspace(1).fill_(0xFF)
    y = _step(eng, x)[0]
    eng.close()
    assert np.isfinite(y).all()
    assert not _same_taps(t0, t1), _same_taps(t0, t1)
    assert np.array_equal(y, t0[max(t0)]["x_out"])


def test_a_previous_step_leaves_nothing_behind():
    """step(x_a) then step(x_b) on one engine = step(x_b) on a fresh one, bit for bit, on the graph with nodes without
    edges (their aggregate rows are rewritten with zeros every step)"""
    _need_gpu()
    cfg, graph, w, xa = _inputs("hand-41x96-m2-L1")
    xb = _inputs("hand-41x96-m2-L1", seed=7)[3]
    eng = _engine(cfg, graph, w)
    _step(eng, xa)
    y1 = _step(eng, xb)
    y1r = _step(eng, xb)           # and the captured / replayed launch sequence
    eng.close()
    eng = _engine(cfg, graph, w)
    y2 = _step(eng, xb)
    eng.close()
    assert np.isfinite(y2).all() and np.array_equal(y1, y2) and np.array_equal(y1r, y2)


def test_members_are_isolated_on_the_hand_built_graph():
    """B = 2: each member equals itself stepped alone; a NaN in member 1's input leaves member 0 bit-identical"""
    _need_gpu()
    cfg, graph, w, xa = _inputs("hand-41x96-m2-L1")
    xb = _inputs("hand-41x96-m2-L1", seed=5)[3]
    eng = _engine(cfg, graph, w)
    yb = _step(eng, np.stack([xa, xb]))
    for m, xm in enumerate((xa, xb)):
        assert np.array_equal(_step(eng, xm)[0], yb[m]), f"member {m} differs from itself stepped alone"
    xn = xb.copy(); xn[3, cfg.nlat - 1, cfg.nlon - 1] = np.nan
    yn = _step(eng, np.stack([xa, xn]))
    eng.close()
    assert not np.isfinite(yn[1]).all()
    assert np.array_equal(yn[0], yb[0])


def test_feature_count_is_bounded_by_the_feature_kernels_tile():
    """n_static = 5 (187 features) does not fit the 186 halves the feature kernel stages per grid point: load_weights
    refuses it before any launch.  n_static = 4 (186: the tile's full width) runs and passes the feature unit."""
    _need_gpu()
    from oracle import graphcast_stages_ref as st
    from skyrim_b200 import _ffi
    from skyrim_b200.engine import StepEngine, launch_count
    cfg, graph, w, x = _inputs("7x16-m1-L1", n_static=5)
    eng = StepEngine(cfg, 0, graph=graph)
    l0 = launch_count()
    with pytest.raises(_ffi.SkyError, match="features"):
        eng.load_weights(w)
    assert launch_count() == l0
    eng.close()
    cfg, graph, w, x = _inputs("7x16-m1-L1", n_static=4)
    assert cfg.n_features == 186
    eng = _engine(cfg, graph, w)
    taps = _read_taps(eng, cfg, graph, x)
    eng.close()
    res = st.check_step(cfg, graph, w, x, T0, taps)
    assert not [r for r in res if r[4]], [r for r in res if r[4]]


def test_range_guard_scans_the_rows_of_a_partial_tile():
    """41x96 / mesh 2: the largest hidden activation of the step (about 408: the mesh-node update after the grid2mesh
    aggregation, at the polar node 161) lies in the partial last row tile of the 162 mesh nodes.  The guarded step must
    report exactly that maximum; a guard that scans whole tiles only reports the runner-up."""
    _need_gpu()
    from oracle import graphcast_stages_ref as st
    cfg, graph, w, x = _inputs("41x96-m2-L2")
    eng = _engine(cfg, graph, w)
    sh = st.Shapes(cfg, graph)
    xs = torch.from_numpy(x)[None].cuda()
    best = (0.0, None, 0, 0)
    for n, (kind, name, outs) in enumerate(st.units(cfg, graph), 1):
        if kind != "hidden":
            continue
        (tap, (rows, kmajor, _)), = outs.items()
        eng.set_clock(T0); eng.debug_set("stop_launch", n)
        eng.step(xs)
        h = np.abs(sh.decode(tap, eng.debug_tensor(tap, (sh.tap_floats(tap),)).cpu().numpy(), sh.m2g_rows if kmajor else rows))
        if h.max() > best[0]:
            best = (float(h.max()), name, int(h.max(1).argmax()), rows)
    eng.debug_set("stop_launch", -1)
    eng.set_clock(T0)
    _, ranges = eng.step_guarded(xs)
    eng.close()
    print(f"largest hidden value {best[0]} in {best[1]} row {best[2]} of {best[3]}; guard saw {ranges['hidden_images']}")
    assert best[2] >= best[3] // 128 * 128, "the maximum is expected in a partial last tile on this graph"
    assert ranges["hidden_images"] == best[0], (ranges, best)


@pytest.mark.parametrize("case", ["41x96-m2-L2", "hand-41x96-m2-L1"])
def test_launches_per_step(case):
    """the clock kernel, then per member one launch per unit and a second aggregation kernel where a segment is cut"""
    _need_gpu()
    from oracle import graphcast_stages_ref as st
    from skyrim_b200.engine import launch_count
    cfg, graph, w, x = _inputs(case)
    split = lambda ptr: bool(st.chunk_plan(graph[ptr])[1])
    expect = len(st.units(cfg, graph)) + split("g2m.ptr") + cfg.layers * split("mesh.ptr")
    eng = _engine(cfg, graph, w)
    for B in (1, 2):
        counts = []
        for _ in range(3):            # eager, captured, replayed
            l0 = launch_count()
            _step(eng, np.stack([x] * B))
            counts.append(launch_count() - l0)
        print(f"{case} B = {B}: launches per step {counts}")
        assert counts == [1 + B * expect] * 3, (counts, expect)
    eng.close()


class _PlannedTaps:
    """``[n]``: a step that stops after unit n (n = 0: no step, the load-time taps), then the planned rows of each of its
    taps gathered on the device; a tap's raw device copy is freed before the next is read.  Units are read in order.
    ``host[n]``: the seconds the checker spent on unit n's references, from its read to the next one (``done`` closes
    the last)."""

    def __init__(self, eng, cfg, sh, p, xs):
        self.eng, self.cfg, self.sh, self.p, self.xs = eng, cfg, sh, p, xs
        self.y, self.seconds, self.bytes, self.host, self.t_read = None, 0.0, {}, {}, None

    def done(self):
        self.host[max(self.bytes)] = time.perf_counter() - self.t_read

    def __getitem__(self, n):
        from oracle import graphcast_stages_ref as st
        t0 = time.perf_counter()
        if n:
            self.host[n - 1] = t0 - self.t_read
        if n:
            self.eng.set_clock(T0)
            self.eng.debug_set("stop_launch", n)
            self.y = self.eng.step(self.xs)
        out = {}
        for tap, (rows, kmajor, cols) in self.p.reads[n].items():
            if tap == "x_out":
                idx = torch.from_numpy(rows).cuda()
                out[tap] = st.Rows(rows, self.y[0].reshape(2 * self.cfg.n_state, -1)[:, idx].T.cpu().numpy().astype(np.float64))
            else:
                raw = self.eng.debug_tensor(tap, (self.sh.tap_floats(tap),))
                out[tap] = self.sh.gather(tap, raw, rows, kmajor, cols)
                del raw
        self.bytes[n] = sum(len(r) * st.row_bytes(self.cfg, tap, cols) for tap, (r, _, cols) in self.p.reads[n].items())
        self.t_read = time.perf_counter()
        self.seconds += self.t_read - t0
        print(f"721x1440 stop {n:3d} read {self.bytes[n] / 2 ** 20:7.1f} MiB, {self.seconds:6.1f} s in stops and gathers", flush=True)
        return out


def test_full_size_units():
    """721 x 1440, refinement-6 multimesh, 16 layers, one member: each of the 115 units read after a step that stops
    behind it, on the rows of graphcast_stages_ref.full_size_rows, from the engine's own inputs to it.  No checked element
    outside its bound, no NaN; a step stopped behind its last unit is the whole step; a workspace of 0x00 and one of 0xFF
    bytes give the same state; launches per step.  Prints one line per unit, the wall time split into
    set-up, stops and gathers and host references per stage, and the memory used."""
    _need_gpu()
    from oracle import graphcast_stages_ref as st
    from skyrim_b200 import icomesh
    from skyrim_b200.config import graphcast_full
    from skyrim_b200.engine import StepEngine, launch_count
    from skyrim_b200.weights import make_graphcast_weights
    t_start = time.perf_counter()
    cfg = graphcast_full()
    t_graph = time.perf_counter()
    graph = icomesh.build_graph(cfg.nlat, cfg.nlon, cfg.mesh_levels, cfg.radius_frac)
    t_graph = time.perf_counter() - t_graph
    w = make_graphcast_weights(cfg, 0)
    x = _state(cfg, 0)
    sh = st.Shapes(cfg, graph)
    p = st.plan(cfg, graph, st.full_size_rows(cfg, graph))
    us = st.units(cfg, graph)
    assert len(us) == 115
    eng = StepEngine(cfg, 0, graph=graph)
    eng.load_weights(w)
    xs = torch.from_numpy(x)[None].cuda()
    taps = _PlannedTaps(eng, cfg, sh, p, xs)
    t_setup = time.perf_counter() - t_start
    try:
        res = st.check_step(cfg, graph, w, x, T0, taps, rows=p.checked)
        taps.done()
        stopped = taps.y.clone()
    finally:
        eng.debug_set("stop_launch", -1)
    for n in range(len(us) + 1):
        mine = [r for r in res if r[0] == n]
        kind, name = us[n - 1][:2] if n else ("static", "load-time")
        rows = sum(map(len, p.checked[0].values())) if n == 0 else len(p.checked[n])
        print(f"721x1440 unit {n:3d} {kind:8s} {name:20s} rows {rows:8d}  worst |D-R|/bound "
              f"{max(r[5] for r in mine):.3f}  outside {sum(r[4] for r in mine)}  host {taps.host[n]:5.1f} s")
    per_kind = {}
    for n, s in taps.host.items():
        k = us[n - 1][0] if n else "static"
        per_kind[k] = per_kind.get(k, 0.0) + s
    print(f"721x1440 set-up {t_setup:.1f} s (graph {t_graph:.1f} s); host references {sum(per_kind.values()):.1f} s: "
          + ", ".join(f"{k} {v:.1f}" for k, v in per_kind.items()) + f"; {st.WORKERS} threads")
    print("721x1440 per stage: " + ", ".join(f"{k} {v:.3f}" for k, v in st.by_stage(res).items()))
    m2g = sh.m2g_rows[p.reads[[n for n, u in enumerate(us, 1) if u[:2] == ("ln", "dec.m2g_edge")][0]]["yimg"][0]]
    print(f"721x1440 mesh2grid rows past byte 2^31 checked: {int((m2g >= 2 ** 31 // 1024).sum())}; most bytes read at one "
          f"stop {max(taps.bytes.values()) / 2 ** 20:.0f} MiB; stops and gathers {taps.seconds:.1f} s")
    ws = eng._workspace(1)
    whole = []
    for fill in (0x00, 0xFF):
        ws.fill_(fill)
        eng.set_clock(T0)
        whole.append(eng.step(xs))
    split = lambda ptr: bool(st.chunk_plan(graph[ptr])[1])
    expect = 1 + len(us) + split("g2m.ptr") + cfg.layers * split("mesh.ptr")
    counts = []
    for _ in range(3):            # eager, captured, replayed
        l0 = launch_count()
        eng.set_clock(T0)
        eng.step(xs)
        torch.cuda.synchronize()
        counts.append(launch_count() - l0)
    device_peak = torch.cuda.max_memory_allocated()
    eng.close()
    print(f"721x1440 launches per step {counts} (expected {expect}); wall time {time.perf_counter() - t_start:.0f} s, host "
          f"peak RSS {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20:.1f} GiB, device peak (torch) "
          f"{device_peak / 2 ** 30:.1f} GiB")
    assert not [r for r in res if r[4]], [r for r in res if r[4]]
    assert torch.equal(stopped, whole[0]), "a step stopped behind its last unit is the whole step"
    assert torch.isfinite(whole[0]).all() and torch.equal(whole[0], whole[1]), "0x00 and 0xFF workspaces"
    assert counts == [expect] * 3, (counts, expect)
