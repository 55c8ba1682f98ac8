"""Pangu's hierarchical 6-h / 24-h schedule on the GPU: every entry point against the two handles stepped by hand, and
every forward against the oracle.  The Pangu step has no atomics and replays bit for bit, so "bitwise" is equality."""
import datetime

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

T0 = datetime.datetime(2024, 5, 7)


@pytest.fixture(scope="module")
def small():
    """one hierarchical and one 6-h Skyrim on pangu_small(41, 96): weight seeds 0 (6 h) and 1 (24 h)"""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from skyrim_b200 import Skyrim
    from skyrim_b200.config import pangu_small
    cfg = pangu_small(41, 96)
    hier = Skyrim("pangu", cfg=cfg, schedule="hierarchical")
    six = Skyrim("pangu", cfg=cfg)
    yield cfg, hier, six
    hier.model.release_model()
    six.model.release_model()


@pytest.fixture(scope="module")
def traj(small):
    """forecast(n_steps=12) under the hierarchical schedule"""
    _, hier, _ = small
    return hier.forecast(T0, n_steps=12).values


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a))[None].cuda()


def _host(t):
    return t[0].cpu().numpy()


def test_forecast_slices_are_the_hierarchy(small, traj):
    _, hier, _ = small
    loop = hier.model.model
    e6, e24 = loop.engine, loop.engine_24
    x0 = _dev(traj[0])
    assert np.array_equal(_host(e24.step(x0)), traj[4])
    assert np.array_equal(_host(e6.step(_dev(traj[4]))), traj[5])
    assert np.array_equal(_host(e6.step(e6.step(e6.step(x0)))), traj[3])
    assert np.array_equal(_host(e24.step(_dev(traj[4]))), traj[8])
    assert np.array_equal(traj[:10], hier.forecast(T0, n_steps=9).values)
    # predict_one_step is P6(x0)
    one = hier.model.predict_one_step(T0).values
    assert np.array_equal(one[1], traj[1])
    assert all(np.isfinite(s).all() for s in traj)


def test_every_forward_matches_the_oracle(small, traj):
    """each forward of the trajectory from the engine's own input for it, so errors do not compound.  The 24-h operator
    runs on weight seed 1, the suite's hardest weights (tests/test_pangu_gpu.py::test_step_parity_other_grids): with the
    default fp16 token stream the fp16 roundings alone cost about 1.1e-3 (from the initial condition) and 1.4e-3 (from
    slice 4) on H100 and in the oracle's emulation of that arithmetic alike, so the engine is held to 1.2 x that
    emulation and below 2e-3; with the fp32 token stream the 24-h forward of the initial condition must meet 1e-3."""
    from oracle.pangu_ref import PanguRef, rel_err_per_channel
    from skyrim_b200.engine import StepEngine
    from skyrim_b200.weights import make_pangu_weights
    cfg = small[0]
    w = {"6h": make_pangu_weights(cfg, 0), "24h": make_pangu_weights(cfg, 1)}
    ref = {op: PanguRef(cfg, w[op]) for op in w}
    for n in range(1, 10):
        d, k = divmod(n, 4)
        op, src = ("24h", 4 * (d - 1)) if k == 0 else ("6h", n - 1)
        want = ref[op].step(traj[src]).numpy()
        e = rel_err_per_channel(traj[n], want).max()
        if op == "6h":
            assert e < 1e-3, (n, op, e)
        else:
            em = rel_err_per_channel(PanguRef(cfg, w[op], emulate="fp16s").step(traj[src]).numpy(), want).max()
            assert e < 2e-3 and e < 1.2 * em, (n, op, e, em)
        print(f"\n[hierarchical 41x96] slice {n} ({op}): max per-channel rel err {e:.3e}")
    eng = StepEngine(cfg, 0)
    eng.load_weights(w["24h"])
    eng.debug_set("fp32_stream", 1)
    e = rel_err_per_channel(_host(eng.step(_dev(traj[0]))), ref["24h"].step(traj[0]).numpy()).max()
    eng.close()
    print(f"[hierarchical 41x96] 24-h forward of the IC, fp32 token stream: {e:.3e}")
    assert e < 1e-3, e


def test_6h_schedule_is_todays_chain(small):
    from skyrim_b200.timeloop import PanguHierarchicalTimeLoop, PanguTimeLoop
    _, _, six = small
    loop = six.model.model
    assert type(loop) is PanguTimeLoop and not isinstance(loop, PanguHierarchicalTimeLoop)
    da = six.forecast(T0, n_steps=5).values
    cur = _dev(da[0])
    for n in range(1, 6):
        cur = loop.engine.step(cur)
        assert np.array_equal(_host(cur), da[n])


@pytest.mark.parametrize("hours", [6, 18, 24, 30, 72])
def test_rollout_last_slices(small, traj, hours, monkeypatch):
    from skyrim_b200 import schedule
    from skyrim_b200.engine import StepEngine
    _, hier, _ = small
    n = hours // 6
    calls = []
    step = StepEngine.step
    monkeypatch.setattr(StepEngine, "step", lambda self, *a, **k: calls.append(self) or step(self, *a, **k))
    pred, paths = hier.model.rollout(T0, n_steps=n, save=False)
    assert paths == []
    assert np.array_equal(pred.values[0], traj[n - 1]) and np.array_equal(pred.values[1], traj[n])
    assert len(calls) == len(schedule.plan("hierarchical", n, every_slice=False).forwards)
    assert list(pred.coords["time"]) == [np.datetime64(T0 + (n - 1 + i) * datetime.timedelta(hours=6), "s")
                                         for i in range(2)]
    # predict goes the same way
    calls.clear()
    p = hier.predict(date="20240507", time="0000", lead_time=hours)[0]
    assert np.array_equal(p.prediction.values[1], traj[n]) and len(calls) == len(
        schedule.plan("hierarchical", n, every_slice=False).forwards)


def test_rollout_save_writes_every_slice(small, traj, tmp_path):
    from skyrim_b200 import xr_shim as xr
    _, hier, _ = small
    pred, paths = hier.model.rollout(T0, n_steps=9, save=True,
                                     save_config=dict(output_dir=str(tmp_path), file_type="netcdf"))
    assert len(paths) == 9
    for n, p in enumerate(paths, 1):
        v = xr.open_dataarray(p).values
        assert np.array_equal(v[0], traj[n - 1]) and np.array_equal(v[1], traj[n]), n
    assert np.array_equal(pred.values[1], traj[9])


def test_predict_ensemble_hierarchical(small, tmp_path):
    from skyrim_b200.engine import ensemble_statistics
    from skyrim_b200.ensemble import EnsembleRunner
    _, hier, _ = small
    m = hier.model
    loop = m.model
    n_steps, q = 6, (0.1, 0.9)
    got = {}
    for save in (False, True):
        res, paths = m.predict_ensemble(T0, n_steps=n_steps, members=3, quantiles=q, save=save,
                                        save_config=dict(output_dir=str(tmp_path / str(save))))
        assert len(paths) == (n_steps if save else 0)
        got[save] = res.stats.values
    assert np.array_equal(got[False], got[True])
    # the members by hand: the perturbed states predict_ensemble builds, then P6^k(P24^d(x))
    base, sigma, _ = m._ensemble_initial_state(T0)
    x = EnsembleRunner(loop.engine, base, sigma, members_per_gpu=3, amp=0.05, seed=0, perturbation="spherical_grf",
                       grf=dict(lmax=20)).x

    def at(n):
        d, k = divmod(n, 4)
        s = x
        for _ in range(d):
            s = loop.engine_24.step(s)
        for _ in range(k):
            s = loop.engine.step(s)
        return ensemble_statistics(s, quantiles=q)[0].cpu().numpy()
    assert np.array_equal(got[False][0], at(n_steps - 1)) and np.array_equal(got[False][1], at(n_steps))


def test_full_size_one_day():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from skyrim_b200 import Skyrim
    sk = Skyrim("pangu", schedule="hierarchical")
    try:
        loop = sk.model.model
        da = sk.forecast(T0, n_steps=4).values
        assert da.shape == (5, 69, 721, 1440) and np.isfinite(da).all()
        assert np.array_equal(_host(loop.engine_24.step(_dev(da[0]))), da[4])
    finally:
        sk.model.release_model()
