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
