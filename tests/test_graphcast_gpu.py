"""GraphCast step (SURVEY.md §8(a) A9 / §8(f) N1): CUDA engine through the C-ABI against the CPU oracle
(oracle/graphcast_ref.py) on the same seeded weights, graph tables and initial condition.

Tolerances: the north star's per-channel relative error <= 1e-3 on the stepped STATE, and — stricter in effect, because
the state is x + 0.1 sigma * tendency — a relative error <= 4e-3 per channel on the network's TENDENCY itself (fp16 tensor-core
operands through 2 + 2 x layers + 2 LayerNorm-ed MLPs: measured 1.2e-3 .. 1.4e-3, what the oracle's own fp16 emulation gives).
"""
import datetime

import numpy as np
import pytest
import torch

from oracle.graphcast_ref import GraphCastRef, rel_err_per_channel, toa_radiation
from skyrim_b200 import icomesh
from skyrim_b200.config import GRAPHCAST_CHANNELS, graphcast_small
from skyrim_b200.weights import make_graphcast_weights, synthetic_graphcast_state

pytestmark = pytest.mark.gpu

TOL = 1e-3        # per-channel relative error of the state (north star)
TOL_TEND = 4e-3   # per-channel relative error of the tendency (network output); measured 1.2e-3 .. 1.4e-3
T0 = 1714521600.0  # 2024-05-01T00:00:00Z


def _setup(nlat, nlon, levels, layers, seed=0):
    from skyrim_b200.engine import StepEngine
    cfg = graphcast_small(nlat, nlon, levels, 512, layers)
    graph = icomesh.build_graph(cfg.nlat, cfg.nlon, cfg.mesh_levels, cfg.radius_frac)
    w = make_graphcast_weights(cfg, seed)
    x = synthetic_graphcast_state(cfg, seed)
    lat = np.linspace(90.0, -90.0, cfg.nlat); lon = np.arange(cfg.nlon) * (360.0 / cfg.nlon)
    x[cfg.n_state - 1] = toa_radiation(T0 - 21600.0, lat, lon)
    x[2 * cfg.n_state - 1] = toa_radiation(T0, lat, lon)
    eng = StepEngine(cfg, 0, graph=graph)
    eng.load_weights(w)
    return cfg, graph, w, x, eng


def _tendency(cfg, y, x, w):
    ns, npg = cfg.n_state, cfg.n_prog
    return (y[ns:ns + npg] - x[ns:ns + npg]) / np.asarray(w["norm.diff_std"])[:npg, None, None]


def test_toa_radiation_matches_oracle():
    from skyrim_b200.engine import StepEngine
    cfg, graph, w, x, eng = _setup(41, 96, 2, 1)
    lat = np.linspace(90.0, -90.0, cfg.nlat); lon = np.arange(cfg.nlon) * (360.0 / cfg.nlon)
    for t in (T0, T0 + 3 * 3600.0, T0 + 200 * 86400.0 + 5000.0):
        got = eng.toa_radiation(t).cpu().numpy()
        ref = toa_radiation(t, lat, lon)
        assert np.abs(got - ref).max() <= 2e-5 * ref.max(), (t, np.abs(got - ref).max(), ref.max())
    eng.close()


@pytest.mark.parametrize("stage,tap,key", [(0, "vg", "grid_embed"), (1, "vm", "enc_mesh"), (1, "vg", "enc_grid"),
                                           (2, "vm", "proc0_mesh"), (3, "vm", "proc1_mesh"), (100, "vg", "dec_grid")])
def test_stage_taps_match_oracle(stage, tap, key):
    """latent taps after the grid embedding, the encoder, each processor layer and the decoder"""
    cfg, graph, w, x, eng = _setup(41, 96, 2, 2)
    taps = {}
    GraphCastRef(cfg, w, graph).tendency(x, T0, taps=taps)
    eng.set_clock(T0)
    eng.debug_set("stop_after", stage)
    eng.step(torch.from_numpy(x)[None].cuda())
    n = cfg.n_grid if tap == "vg" else graph["n_mesh"]
    got = eng.debug_tensor(tap, (n, cfg.latent)).cpu().numpy()
    ref = taps[key].numpy()
    err = np.linalg.norm(got - ref) / np.linalg.norm(ref)
    print(f"{key}: rel err {err:.3e}")
    assert err < 3e-3, (key, err)
    eng.close()


@pytest.mark.parametrize("shape", [(41, 96, 2, 2), (33, 64, 1, 3), (49, 120, 3, 1)])
def test_step_matches_oracle(shape):
    cfg, graph, w, x, eng = _setup(*shape)
    ref, tref = GraphCastRef(cfg, w, graph).step(x, T0, return_tendency=True)
    ref = ref.numpy()
    eng.set_clock(T0)
    y = eng.step(torch.from_numpy(x)[None].cuda())[0].cpu().numpy()
    assert np.isfinite(y).all()
    err = rel_err_per_channel(y, ref)
    terr = rel_err_per_channel(_tendency(cfg, y, x, w), _tendency(cfg, ref, x, w))
    print(f"GraphCast {shape}: state max per-channel rel err {err.max():.3e}, tendency {terr.max():.3e}")
    assert np.array_equal(y[:cfg.n_state], x[cfg.n_state:]), "slice 0 of the new state must be slice 1 of the old one"
    assert err.max() < TOL, err.max()
    assert terr.max() < TOL_TEND, terr.max()
    eng.close()


def test_mid_size_more_tiles_than_sms():
    """181 x 360 grid (509 row tiles of grid nodes, 1527 of mesh2grid edges), refinement-4 mesh, 3 layers: every
    persistent GEMM loop runs several tiles per CTA"""
    cfg, graph, w, x, eng = _setup(181, 360, 4, 3)
    ref = GraphCastRef(cfg, w, graph).step(x, T0).numpy()
    eng.set_clock(T0)
    y = eng.step(torch.from_numpy(x)[None].cuda())[0].cpu().numpy()
    err = rel_err_per_channel(y, ref)
    terr = rel_err_per_channel(_tendency(cfg, y, x, w), _tendency(cfg, ref, x, w))
    print(f"GraphCast 181x360 / mesh 4: state {err.max():.3e}, tendency {terr.max():.3e}")
    assert err.max() < TOL and terr.max() < TOL_TEND, (err.max(), terr.max())
    eng.close()


def test_two_chained_steps_advance_the_clock_and_are_reproducible():
    cfg, graph, w, x, eng = _setup(41, 96, 2, 2)
    oracle = GraphCastRef(cfg, w, graph)
    r1 = oracle.step(x, T0).numpy()
    r2 = oracle.step(r1, T0 + 21600.0).numpy()
    outs = []
    for _ in range(2):
        eng.set_clock(T0)
        a = eng.step(torch.from_numpy(x)[None].cuda())
        b = eng.step(a)
        outs.append(b[0].cpu().numpy())
    assert np.array_equal(outs[0], outs[1]), "the step must be run-to-run reproducible (no atomics in the aggregation)"
    err = rel_err_per_channel(outs[0], r2)
    print(f"two chained steps: max per-channel rel err {err.max():.3e}")
    assert err.max() < 2 * TOL
    # third call replays the captured CUDA graph: same clock handling
    eng.set_clock(T0)
    a = eng.step(torch.from_numpy(x)[None].cuda()); b = eng.step(a); c1 = eng.step(b)
    eng.set_clock(T0)
    a = eng.step(torch.from_numpy(x)[None].cuda()); b = eng.step(a); c2 = eng.step(b)
    assert torch.equal(c1, c2)
    eng.close()


def test_batched_members_match_single():
    cfg, graph, w, x, eng = _setup(41, 96, 2, 1)
    x2 = np.stack([x, x[::-1].copy() * 0 + synthetic_graphcast_state(cfg, 5)])
    eng.set_clock(T0)
    yb = eng.step(torch.from_numpy(x2).cuda()).cpu().numpy()
    for m in range(2):
        eng.set_clock(T0)
        ys = eng.step(torch.from_numpy(x2[m])[None].cuda())[0].cpu().numpy()
        assert np.array_equal(ys, yb[m])
    eng.close()


def test_skyrim_api_graphcast():
    """reference test shape (/root/reference/tests/core/test_graphcast.py:11-22): dims and the channel-name set"""
    from skyrim_b200.core import Skyrim
    cfg = graphcast_small(41, 96, 2, 512, 2)
    model = Skyrim("graphcast", ic_source="synthetic", cfg=cfg)
    pred, paths = model.predict("20240404", "0000", 12, save=False)
    assert set(pred.prediction.dims) == {"time", "channel", "lat", "lon"}
    assert pred.prediction.shape == (2, 83, 41, 96) and paths == []
    da = model.forecast(start_time=datetime.datetime(2024, 4, 4, 0, 0), n_steps=2)
    assert da.shape == (3, 83, 41, 96)
    assert set(model.model.out_channel_names) == set(GRAPHCAST_CHANNELS)
    # forecast step 2 == rollout's last slice (same chain)
    assert np.allclose(da.values[2], pred.prediction.values[1], rtol=0, atol=0)
    one = model.model.predict_one_step(datetime.datetime(2024, 4, 4, 0, 0))
    assert np.array_equal(one.values[1], da.values[1])


def test_rollout_saves_every_step_and_cli(tmp_path):
    """GraphcastModel.rollout(save=True) (graphcast.py:144-177): one file per step with two time slices, the forecast CLI
    drives the same path"""
    from skyrim_b200 import xr_shim as xr
    from skyrim_b200.core import Skyrim
    cfg = graphcast_small(41, 96, 2, 512, 2)
    model = Skyrim("graphcast", ic_source="synthetic", cfg=cfg)
    pred, paths = model.predict("20240404", "0600", 18, save=True, save_config=dict(output_dir=str(tmp_path), file_type="netcdf"))
    assert len(paths) == 3
    last = xr.open_dataarray(paths[-1])
    assert last.shape == (2, 83, 41, 96)
    assert np.array_equal(np.asarray(last.values, dtype=np.float32), pred.prediction.values.astype(np.float32))
    first = xr.open_dataarray(paths[0])
    second = xr.open_dataarray(paths[1])
    assert np.array_equal(first.values[1], second.values[0]), "successive files overlap by one time slice, as in the reference"
    from click.testing import CliRunner
    from skyrim_b200.forecast import main
    r = CliRunner().invoke(main, ["-m", "graphcast", "-d", "20240404", "-t", "0000", "-l", "12", "-o", str(tmp_path / "cli"),
                                  "--grid", "41x96"])
    assert r.exit_code == 0, r.output


def test_fp16_range_guard_graphcast():
    """guarded step: max |value| of the fp16 operand image classes stays far inside the fp16 range on synthetic weights; an
    inflated first-layer weight is refused"""
    from skyrim_b200 import _ffi
    cfg, graph, w, x, eng = _setup(41, 96, 2, 2)
    xs = torch.from_numpy(x)[None].cuda()
    eng.set_clock(T0)
    y_plain = eng.step(xs).clone()
    eng.set_clock(T0)
    y, ranges = eng.step_guarded(xs)
    assert torch.equal(y, y_plain)
    assert set(ranges) >= {"token_images", "hidden_images", "spectral_images"}, ranges
    assert all(0 < v < 2000 for v in ranges.values()), ranges
    eng.close()
    from skyrim_b200.engine import StepEngine
    w2 = dict(w); w2["proc0.edge.w1"] = w["proc0.edge.w1"] * 1.0e5
    eng2 = StepEngine(cfg, 0, graph=graph)
    eng2.load_weights(w2)
    eng2.set_clock(T0)
    with pytest.raises(_ffi.SkyError):
        eng2.step_guarded(xs)
    eng2.close()


def test_timeloop_generator_and_host_step_agree_with_the_stepper():
    """TimeLoop protocol (first yield = the initial condition's last slice), the stepper protocol of graphcast.py:110,118 and
    the host-in / host-out step of bench.py's e2e all run the same chain"""
    from skyrim_b200.timeloop import GraphcastTimeLoop
    cfg, graph, w, x, eng = _setup(41, 96, 2, 1)
    loop = GraphcastTimeLoop(eng)
    t0 = datetime.datetime(2024, 5, 1)
    x5 = torch.from_numpy(x).reshape(1, 2, cfg.n_state, cfg.nlat, cfg.nlon)
    gen = loop(t0, x5)
    t, first, _ = next(gen)
    assert t == t0 and torch.equal(first.cpu(), x5[:, 1])
    t1, y1, _ = next(gen)
    t2, y2, _ = next(gen)
    assert t2 == t0 + 2 * loop.time_step
    state = loop.stepper.initialize(x5, t0)
    state, o1 = loop.stepper.step(state)
    state, o2 = loop.stepper.step(state)
    assert torch.equal(o1, y1) and torch.equal(o2, y2) and state[0] == t2
    xh = x5.reshape(1, -1, cfg.nlat, cfg.nlon).contiguous().pin_memory()
    eng.set_clock(t0)
    h = loop.step_host(xh)
    h = loop.step_host(h)
    assert torch.equal(h[1], y2.cpu()) and torch.equal(h[0], y1.cpu())
    eng.close()
