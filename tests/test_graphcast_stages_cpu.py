"""The GraphCast stage checker (oracle/graphcast_stages_ref.py) on its own, without a GPU.

A stand-in for the engine (graphcast_stages_ref.Emulator: the engine's formulation in numpy — fp16 where the engine
rounds, split first layers and per-node tables, chunked fp32 segment sums in the kernels' order) must pass every unit's
check on the icosahedral and the hand-built graphs and agree with the oracle's own fp16 emulation; each modelled engine
mistake planted into it must be named by the check of its own unit, and by none before it.
"""
import functools

import numpy as np
import pytest
import torch

from oracle import graphcast_stages_ref as st
from oracle.graphcast_ref import GraphCastRef, toa_radiation
from skyrim_b200 import icomesh
from skyrim_b200.config import graphcast_small
from skyrim_b200.weights import make_graphcast_weights, synthetic_graphcast_state

T0 = 1714521600.0
CASES = {"41x96-m2-L2": (41, 96, 2, 2, False), "33x64-m1-L3": (33, 64, 1, 3, False), "49x120-m3-L1": (49, 120, 3, 1, False),
         "32x64-m1-L1": (32, 64, 1, 1, False), "7x16-m1-L1": (7, 16, 1, 1, False), "8x16-m1-L1": (8, 16, 1, 1, False),
         "hand-41x96-m2-L1": (41, 96, 2, 1, True), "hand-33x64-m1-L2": (33, 64, 1, 2, True), "33x64-m1-L2": (33, 64, 1, 2, False)}


@functools.lru_cache(maxsize=None)
def _inputs(case):
    nlat, nlon, levels, layers, hand = CASES[case]
    cfg = graphcast_small(nlat, nlon, levels, 512, layers)
    graph = icomesh.build_graph(cfg.nlat, cfg.nlon, cfg.mesh_levels, cfg.radius_frac)
    if hand:
        graph = st.hand_graph(graph)
    w = make_graphcast_weights(cfg, 0)
    x = synthetic_graphcast_state(cfg, 0)
    lat = np.linspace(90.0, -90.0, cfg.nlat); lon = np.arange(cfg.nlon) * (360.0 / cfg.nlon)
    x[cfg.n_state - 1] = toa_radiation(T0 - 21600.0, lat, lon)
    x[2 * cfg.n_state - 1] = toa_radiation(T0, lat, lon)
    return cfg, graph, w, x


def test_chunk_plan_at_the_chunk_boundary():
    """exactly 64 edges are one chunk, 65 two, 4321 sixty-eight; a node without edges is one (empty) chunk that writes its
    row; the partial rows of the cut segments are numbered in node order"""
    deg = np.array([0, 64, 65, 4321, 1, 0])
    ptr = np.concatenate([[0], np.cumsum(deg)])
    chunks, multi = st.chunk_plan(ptr)
    per_node = [sum(1 for c in chunks if c[0] == n) for n in range(len(deg))]
    assert per_node == [1, 1, 2, 68, 1, 1]
    assert multi == [(2, 0, 2), (3, 2, 70)]
    assert [c for c in chunks if c[0] == 2] == [(2, 64, 128, 0), (2, 128, 129, 1)]
    assert chunks[0] == (0, 0, 0, -1) and chunks[-1] == (5, int(ptr[-1]), int(ptr[-1]), -1)
    assert all(e1 - e0 <= st.SEG_CHUNK for _, e0, e1, _ in chunks)
    assert sum(e1 - e0 for _, e0, e1, _ in chunks) == deg.sum()


def test_hand_built_graph_has_the_degrees_it_promises():
    cfg, graph, w, x = _inputs("hand-41x96-m2-L1")
    dg = np.diff(graph["g2m.ptr"]); dm = np.diff(graph["mesh.ptr"])
    assert set(st.G2M_DEGREES) <= set(dg.tolist()) and dg[0] == 0 and dg[-1] == 0
    assert set(st.MESH_DEGREES) <= set(dm.tolist()) and dm[0] == 0 and dm[-1] == 0
    assert {0, cfg.n_grid - 1} <= set(graph["g2m.senders"].tolist())
    for k in ("g2m", "mesh"):
        r = graph[k + ".receivers"]
        assert (np.diff(r) >= 0).all() and np.array_equal(np.repeat(np.arange(graph["n_mesh"]), np.diff(graph[k + ".ptr"])), r)
        assert len(graph[k + ".edge_feat"]) == len(r)
    s, r = graph["mesh.senders"], graph["mesh.receivers"]
    assert (s == r).any(), "a self-edge"
    assert len({(a, b) for a, b in zip(s.tolist(), r.tolist())}) < len(s), "a duplicated (sender, receiver) pair"
    assert st.chunk_plan(graph["mesh.ptr"])[1], "the mesh aggregation takes the partial-row route"


def test_tile_image_decoding_round_trips():
    cfg, graph, w, x = _inputs("7x16-m1-L1")
    sh = st.Shapes(cfg, graph)
    rng = np.random.default_rng(0)
    a = rng.standard_normal((sh.E3, st.L)).astype(np.float16)
    raw = np.zeros(sh.tap_floats("hid") * 4, np.uint8)
    img = st.gr.pack_tiles(a, 128, st.NKB)
    raw[:img.size] = img
    got = sh.decode("hid", raw.view(np.float32), sh.m2g_rows)
    want = a.astype(np.float64).reshape(3, sh.Ngp, st.L)[:, :sh.Ng].reshape(-1, st.L)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("case", [c for c in CASES if c != "33x64-m1-L2"])
def test_emulated_engine_passes_every_unit(case):
    cfg, graph, w, x = _inputs(case)
    e = st.emulate(cfg, graph, w, x, T0)
    assert len(e.taps) == len(st.units(cfg, graph)) + 1
    res = st.check_step(cfg, graph, w, x, T0, e.taps)
    assert not [r for r in res if r[4]], [r for r in res if r[4]]
    # the chain: the emulation's network output against the oracle's own fp16 emulation and against fp64
    t16 = GraphCastRef(cfg, w, graph, dtype=torch.float64, emulate="fp16s").tendency(x, T0).numpy()
    t64 = GraphCastRef(cfg, w, graph, dtype=torch.float64).tendency(x, T0).numpy()
    rel = lambda a, b: np.linalg.norm(a - b) / np.linalg.norm(b)
    print(f"{case}: emulation vs fp16s oracle {rel(e.tendency, t16):.2e}, vs fp64 {rel(e.tendency, t64):.2e}, fp16s vs fp64 {rel(t16, t64):.2e}")
    assert rel(e.tendency, t64) < 1.5 * rel(t16, t64) + 1e-4
    assert rel(e.tendency, t16) < 2.0 * rel(t16, t64) + 1e-4


# mutation -> (graph, the unit whose check must name it)
MUTATIONS = {
    "swap_tables": ("33x64-m1-L2", ("hidden", "proc0.edge")),           # sender table gathered with the receiver index
    "w1r_from_w1s": ("33x64-m1-L2", ("table", "proc0.edge")),           # W1r taken from the W1s columns
    "drop_last_chunk": ("33x64-m1-L2", ("agg", "g2m")),                 # the last chunk of the cut segments
    "skip_tail": ("33x64-m1-L2", ("agg", "g2m")),                       # the e % 4 tail of every chunk
    "swap_day_sincos": ("33x64-m1-L2", ("features", "features")),       # day sin / cos columns of t - 6h
    "no_residual_grid": ("33x64-m1-L2", ("ln", "enc.g2m_grid")),        # the grid stream's residual
    "stale_zero_degree": ("hand-33x64-m1-L2", ("agg", "g2m")),          # a node without edges keeps its previous row
    "shift_last_row": ("33x64-m1-L2", ("ln", "enc.grid_embed")),        # the last row of the partial tile holds its neighbour's
    "scale_last_row": ("33x64-m1-L2", ("ln", "enc.grid_embed")),        # the last row of the partial tile 10 % off
}
# the mutations that leave every latent tap of tests/test_graphcast_gpu.py::test_stage_taps_match_oracle (relative L2 over the
# whole tensor < 3e-3 against the oracle) inside its tolerance: measured by test_mutations_are_named_by_their_own_unit
MISSED_BY_WHOLE_TENSOR_NORM = {"scale_last_row"}


@functools.lru_cache(maxsize=None)
def _oracle_taps(case):
    cfg, graph, w, x = _inputs(case)
    ref = {}
    GraphCastRef(cfg, w, graph).tendency(x, T0, taps=ref)
    return {k: v.numpy() for k, v in ref.items()}


def _whole_tensor_errors(case, e):
    """the six latent taps of the existing whole-tensor check, emulated engine against the fp32 oracle"""
    cfg, graph, w, x = _inputs(case)
    ref = _oracle_taps(case)
    keys = ["grid_embed", "enc_mesh", "enc_grid", "dec_grid"] + [f"proc{i}_mesh" for i in range(cfg.layers)]
    got = dict(st.chain_pairs(cfg, graph, w, x, e.taps))
    return {k: float(np.linalg.norm(got[k] - ref[k]) / np.linalg.norm(ref[k])) for k in keys}


@pytest.mark.parametrize("mut", list(MUTATIONS))
def test_mutations_are_named_by_their_own_unit(mut):
    """each modelled mistake trips the check of the unit it belongs to and none before it.  Which of them a relative L2
    over whole tensors < 3e-3 lets through is recorded in MISSED_BY_WHOLE_TENSOR_NORM.  On this 2112-point grid the eight
    gross ones (swapped tables, W1r from the W1s columns, a dropped last chunk, a skipped e % 4 tail, swapped day sin / cos,
    a missing grid residual, a stale row of a node without edges, a row replaced by its neighbour) all move some latent by
    more than 3e-3 (the smallest: the skipped tail, 3.5e-3 on the decoder's grid latent, and the replaced row, 1.8e-2 —
    which shrinks with the square root of the grid size); what the norm misses is the last row of the partial tile being
    10 % off (2.2e-3).  The norm names no unit for any of them."""
    case, where = MUTATIONS[mut]
    cfg, graph, w, x = _inputs(case)
    e = st.emulate(cfg, graph, w, x, T0, mut=mut)
    res = st.check_step(cfg, graph, w, x, T0, e.taps)
    failing = [(n, kind, name, what, bad) for n, kind, name, what, bad, wr in res if bad]
    assert failing, f"{mut} passed every check"
    first = min(f[0] for f in failing)
    assert {(kind, name) for n, kind, name, what, bad in failing if n == first} == {where}, failing
    at = [n for n, (kind, name, _) in enumerate(st.units(cfg, graph), 1) if (kind, name) == where][0]
    assert first == at and all(f[0] >= at for f in failing), failing
    errs = _whole_tensor_errors(case, e)
    base = _whole_tensor_errors(case, st.emulate(cfg, graph, w, x, T0)) if mut == "swap_tables" else None
    missed = max(errs.values()) < 3e-3
    print(f"{mut}: first failing unit {first} {where}, {sum(f[4] for f in failing)} elements outside; whole-tensor errors "
          f"{ {k: round(v, 5) for k, v in errs.items()} } -> {'MISSED' if missed else 'caught'} by the 3e-3 norm"
          + (f"; clean emulation {max(base.values()):.2e}" if base else ""))
    assert missed == (mut in MISSED_BY_WHOLE_TENSOR_NORM), (mut, errs)


# ---------------------------------------------------------------------------------------------------------------------
# the sampled check: a read plan (Planner) and the Checker on chosen rows
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _emulated(case, mut=None):
    cfg, graph, w, x = _inputs(case)
    return st.emulate(cfg, graph, w, x, T0, mut=mut).taps


def _sampled(cfg, taps, p):
    """what a device gather of the plan would return: the planned rows of every tap, as Rows"""
    ns = cfg.n_state
    rows = lambda tap, v, r: np.asarray(v, np.float64).reshape(2 * ns, -1)[:, r].T if tap == "x_out" else np.asarray(v)[r]
    return {n: {tap: st.Rows(r, rows(tap, taps[n][tap], r)) for tap, (r, kmajor, cols) in p.reads[n].items()} for n in p.reads}


@pytest.mark.parametrize("case", [c for c in CASES if c != "33x64-m1-L2"])
def test_sampled_checker_on_every_row_is_check_step(case):
    """the every-row plan read as Rows gives check_step's counts and worst ratios exactly, and lists every valid row"""
    cfg, graph, w, x = _inputs(case)
    taps = _emulated(case)
    p = st.plan(cfg, graph)
    for n, (kind, name, outs) in enumerate(st.units(cfg, graph), 1):
        assert set(p.reads[n]) >= set(outs) and len(p.checked[n]) == (outs[next(iter(outs))][0] or cfg.n_grid)
    assert st.check_step(cfg, graph, w, x, T0, _sampled(cfg, taps, p), rows=p.checked) == st.check_step(cfg, graph, w, x, T0, taps)


SMALL = dict(n_grid=16, n_g2m_nodes=4, n_edges=16)       # the full-size rules with small seeded samples


@pytest.mark.parametrize("mut", list(MUTATIONS))
def test_full_size_rules_catch_every_mutation(mut):
    """the full-size sampling rules (first and partial last tile, first and last latitude row, cut and degree-0 nodes, a
    few seeded rows) applied to the small graphs name each modelled mistake in its own unit, as the every-row check does"""
    case, where = MUTATIONS[mut]
    cfg, graph, w, x = _inputs(case)
    p = st.plan(cfg, graph, st.full_size_rows(cfg, graph, **SMALL))
    assert any(len(r) < n for r, n in ((p.checked[1], cfg.n_grid), (p.checked[0]["e_g2m_img"], len(graph["g2m.senders"]))))
    res = st.check_step(cfg, graph, w, x, T0, _sampled(cfg, _emulated(case, mut), p), rows=p.checked)
    failing = [(n, kind, name, what, bad) for n, kind, name, what, bad, wr in res if bad]
    at = [n for n, (kind, name, _) in enumerate(st.units(cfg, graph), 1) if (kind, name) == where][0]
    assert failing and min(f[0] for f in failing) == at, (mut, failing)
    assert {(kind, name) for n, kind, name, what, bad in failing if n == at} == {where}, failing
    clean = st.check_step(cfg, graph, w, x, T0, _sampled(cfg, _emulated(case), p), rows=p.checked)
    assert not [r for r in clean if r[4]], [r for r in clean if r[4]]


def test_full_size_plan():
    """721 x 1440 / refinement-6 multimesh / 16 layers (the graph is built on the host): every mesh-node unit on every
    row; every mesh-edge row in layers 0, 1, 14 and 15; rows past byte 2^31 of the k-major mesh2grid images; every
    partial tile; all 3,234 nodes whose grid2mesh segment is cut, with all their edges in every grid2mesh unit.  Prints
    the most bytes a single stop reads."""
    from skyrim_b200.config import graphcast_full
    cfg = graphcast_full()
    graph = icomesh.build_graph(cfg.nlat, cfg.nlon, cfg.mesh_levels, cfg.radius_frac)
    sh = st.Shapes(cfg, graph)
    p = st.plan(cfg, graph, st.full_size_rows(cfg, graph))
    us = st.units(cfg, graph)
    assert len(us) == 115
    Ng, Nm, Em, Eg = cfg.n_grid, sh.Nm, sh.Em, sh.Eg
    last = lambda n: np.arange(n // 128 * 128, n)
    assert (Ng % 128, Nm % 128, Em % 128) == (32, 2, 108)
    for n, (kind, name, outs) in enumerate(us, 1):
        rows, kmajor, _ = next(iter(outs.values()))
        R = p.checked[n]
        if name == "g2m":
            continue
        if rows == Nm:
            assert len(R) == Nm, (n, name)
        elif kmajor:
            assert all(np.isin(k * Ng + last(Ng), R).all() for k in range(3)), (n, name)
        elif rows == Em:
            layer = int(name[4:name.index(".")])
            assert len(R) == Em if layer in (0, 1, 14, 15) else np.isin(last(Em), R).all() and R[0] == 0, (n, name)
        elif rows == Eg:
            assert np.isin(last(Eg), R).all() and R[0] == 0, (n, name)
        else:
            assert np.isin(last(Ng), R).all() and np.isin(np.arange(cfg.nlon), R).all(), (n, name)
    assert all(len(p.checked[0][k]) == Nm for k in ("vm0_img", "g2m_tr"))
    # the k-major mesh2grid images: tiles on either side of byte 2^31
    m2g = [n for n, (kind, name, outs) in enumerate(us, 1) if name == "dec.m2g_edge" and kind != "table"]
    for n in m2g:
        for tap, (rows, kmajor, _) in p.reads[n].items():
            byte = sh.m2g_rows[rows] // 128 * (st.NKB * st.TILE)
            assert kmajor and (byte >= 2 ** 31).sum() >= 128 and (byte == 2 ** 31 - st.NKB * st.TILE).any(), (n, tap)
    assert (sh.m2g_rows[p.checked[0]["e_m2g_img"]] >= 2 ** 31 // 1024).any()
    # every node whose grid2mesh segment is cut, with all its edges
    cut = np.array([node for node, p0, p1 in st.chunk_plan(graph["g2m.ptr"])[1]])
    agg = [n for n, (kind, name, _) in enumerate(us, 1) if name == "g2m"][0]
    assert len(cut) == 3234 and np.isin(cut, p.checked[agg]).all()
    cut_edges = st.seg_edges(graph["g2m.ptr"], cut)
    assert len(cut_edges) == 414552
    for n, (kind, name, _) in enumerate(us, 1):
        if name == "enc.g2m_edge" and kind != "table":
            assert np.isin(cut_edges, p.checked[n]).all()
    assert np.isin(cut_edges, p.checked[0]["e_g2m_img"]).all() and len(p.checked[0]["e_mesh_img"]) == Em
    per_stop = {n: sum(len(r) * st.row_bytes(cfg, tap, cols) for tap, (r, kmajor, cols) in taps.items())
                for n, taps in p.reads.items()}
    n = max(per_stop, key=per_stop.get)
    print(f"721x1440: most bytes read at one stop {per_stop[n] / 2 ** 20:.0f} MiB (stop {n}: {us[n - 1][:2] if n else 'load'}); "
          f"in all {sum(per_stop.values()) / 2 ** 30:.2f} GiB over {len(per_stop)} stops")


def test_device_gather_round_trips():
    """Shapes.gather on a host torch tensor: rows of a full tile, of the partial last tile and of the last tile of a
    k-major image, of a table and of an fp32 latent equal the whole decode"""
    cfg, graph, w, x = _inputs("7x16-m1-L1")
    sh = st.Shapes(cfg, graph)
    rng = np.random.default_rng(1)
    a = rng.standard_normal((sh.E3, st.L)).astype(np.float16)
    raw = np.zeros(sh.tap_floats("hid") * 4, np.uint8)
    img = st.gr.pack_tiles(a, 128, st.NKB)
    raw[:img.size] = img
    whole = sh.decode("hid", raw.view(np.float32), sh.m2g_rows)
    Ng = cfg.n_grid
    for rows in (np.arange(0, 128, 5), np.arange(Ng - 9, Ng), np.arange(2 * Ng, 3 * Ng)[[0, 7, -1]], np.array([Ng - 1, Ng, 2 * Ng + 3])):
        got = sh.gather("hid", torch.from_numpy(raw.view(np.float32)), rows, kmajor=True)
        assert np.array_equal(got.idx, rows) and np.array_equal(got.val, whole[rows]), rows
    plain = sh.gather("hid", torch.from_numpy(raw.view(np.float32)), np.array([0, 127, 128, sh.E3 - 1]))
    assert np.array_equal(plain.val, a[[0, 127, 128, sh.E3 - 1]].astype(np.float64))
    t = rng.standard_normal((sh.Nmp, 2 * st.L)).astype(np.float16)
    got = sh.gather("tm", torch.from_numpy(t.view(np.float32).reshape(-1)), [0, 5, sh.Nm - 1], cols=2 * st.L)
    assert np.array_equal(got.val, t[[0, 5, sh.Nm - 1]].astype(np.float64))
    v = rng.standard_normal((sh.Nm, st.L)).astype(np.float32)
    got = sh.gather("vm", torch.from_numpy(v.reshape(-1)), [1, sh.Nm - 1])
    assert np.array_equal(got.val, v[[1, sh.Nm - 1]].astype(np.float64))
    r = st.Rows(got.idx, got.val)
    assert np.array_equal(r[np.array([sh.Nm - 1])], got.val[1:]) and np.array_equal(r[1:sh.Nm].idx, [0, sh.Nm - 2])
    with pytest.raises(AssertionError, match="not read"):
        r[np.array([0])]
    with pytest.raises(AssertionError, match="not read"):
        r[np.array([sh.Nm])]
    empty = sh.gather("hid", torch.from_numpy(raw.view(np.float32)), np.zeros(0, np.int64), kmajor=True)
    assert empty.val.shape == (0, st.L) and empty[np.zeros(0, np.int64)].shape == (0, st.L)
    with pytest.raises(AssertionError, match="not read"):
        empty[np.array([0])]
