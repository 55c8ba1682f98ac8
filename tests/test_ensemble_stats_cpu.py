"""Ensemble statistics without a device: the C-ABI's argument refusals, the oracle, GlobalEnsemblePrediction, the
predict_ensemble host logic on a CPU fake of the member runner, its files and the forecast CLI options."""
import ctypes as C
import datetime
import os
import re

import numpy as np
import pytest
import torch

from oracle import ens_stats_ref
from skyrim_b200 import xr_shim as xr
from skyrim_b200.core.models.base import GlobalModel, GlobalPrediction
from skyrim_b200.core.models.ensemble import GlobalEnsemblePrediction, event_name, quantile_name
from skyrim_b200.timeloop import equiangular_grid

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CH = ["u10m", "v10m", "t2m", "msl"]
T0 = datetime.datetime(2024, 5, 7)


def test_export_present_and_declared():
    from skyrim_b200 import _ffi
    hdr = open(os.path.join(ROOT, "include", "skyrim_b200.h")).read()
    assert "sky_ensemble_stats" in set(re.findall(r"\b(sky_[a-z_0-9]+)\s*\(", hdr)) and "sky_ensemble_stats" in _ffi.EXPORTS
    assert hasattr(_ffi.lib(), "sky_ensemble_stats")


def _call(members=4, stride=None, plane=96, count=5, channels=(0, 4), quantiles=(0.5,), ev_sel=(0, 1), ev_thr=(1.0, 2.0),
          n_sel=None, n_q=None, n_events=None):
    from skyrim_b200 import _ffi
    L = _ffi.lib()
    bogus = C.c_void_p(0x1000)    # never inspected: every refusal below comes before the device-pointer check
    arr = lambda ct, v: (ct * max(len(v), 1))(*v)  # noqa: E731
    rc = L.sky_ensemble_stats(bogus, members, count * plane if stride is None else stride, plane, count,
                              arr(C.c_int32, channels), len(channels) if n_sel is None else n_sel,
                              arr(C.c_double, quantiles), len(quantiles) if n_q is None else n_q,
                              arr(C.c_int32, ev_sel), arr(C.c_float, ev_thr), len(ev_sel) if n_events is None else n_events,
                              bogus, bogus, None)
    return rc, L.sky_last_error().decode()


@pytest.mark.parametrize("kw, what", [
    (dict(members=0), "members"), (dict(members=65), "members"),
    (dict(channels=(0, 5)), "channel 5"), (dict(channels=(-1, 2)), "channel -1"),
    (dict(stride=5 * 96 - 1), "member_stride"), (dict(stride=-1), "member_stride"),
    (dict(quantiles=(1.5,)), "quantile"), (dict(quantiles=(-0.1,)), "quantile"), (dict(quantiles=(float("nan"),)), "quantile"),
    (dict(quantiles=(float("inf"),)), "quantile"),
    (dict(ev_sel=(0, 2)), "event_sel"), (dict(ev_sel=(1, 0)), "decreases"), (dict(ev_sel=(0, -1)), "event_sel"),
    (dict(ev_thr=(1.0, float("nan"))), "threshold"), (dict(ev_thr=(float("-inf"), 1.0)), "threshold"),
    (dict(channels=tuple(range(129)), count=200), "n_sel"), (dict(channels=()), "n_sel"),
    (dict(quantiles=(0.5,) * 9), "n_q"), (dict(ev_sel=(0,) * 65, ev_thr=(1.0,) * 65), "n_events"),
])
def test_library_refuses_bad_arguments_before_any_cuda_call(kw, what):
    rc, msg = _call(**kw)
    assert rc == -1 and what in msg, msg


def test_oracle_matches_numpy_definitions():
    rng = np.random.default_rng(0)
    x = rng.standard_normal((7, 3, 5, 6)).astype(np.float32) * 3 + 10
    s, p = ens_stats_ref.ensemble_stats(x, [2, 0], (0.0, 0.25, 1.0), [(0, 10.0), (1, 9.5)])
    v = x[:, [2, 0]].astype(np.float64)
    np.testing.assert_allclose(s[0], v.mean(0), rtol=1e-7)
    np.testing.assert_allclose(s[1], v.std(0), rtol=1e-6)
    np.testing.assert_array_equal(s[2], v.min(0).astype(np.float32))
    np.testing.assert_array_equal(s[4], v.max(0).astype(np.float32))
    np.testing.assert_array_equal(p[1], ((v[:, 1] > 9.5).sum(0) / 7).astype(np.float32))
    x[3, 0, 1, 2] = np.nan
    s, p = ens_stats_ref.ensemble_stats(x, [0], (0.5,), [(0, 0.0)])
    assert np.isnan(s[:, 0, 1, 2]).all() and np.isnan(p[0, 1, 2]) and np.isfinite(s[:, 0, 0]).all()
    y = np.zeros((3, 1, 1, 2), np.float32); y[:, 0, 0, 0] = [1.0, 2.0, 3.0]
    assert ens_stats_ref.ensemble_stats(y, [0], (), [(0, 2.0)])[1][0, 0, 0] == np.float32(1 / 3)   # strict: x == t not counted


def test_names():
    assert [quantile_name(q) for q in (0.1, 0.5, 0.9, 0.0, 1.0, 0.05)] == ["q0.1", "q0.5", "q0.9", "q0", "q1", "q0.05"]
    assert event_name("t2m", 273.15) == "t2m>273.15" and event_name("u10m", 15) == "u10m>15"


def _hand_made(n_ev=2):
    g = equiangular_grid(19, 36)
    stats = np.arange(2 * 4 * 3 * 19 * 36, dtype=np.float32).reshape(2, 4, 3, 19, 36)
    times = np.array(["2024-05-07T00", "2024-05-07T06"], dtype="datetime64[s]")
    sd = xr.DataArray(stats, dims=["time", "statistic", "channel", "lat", "lon"],
                      coords=dict(time=times, statistic=np.array(["mean", "spread", "q0.1", "q0.9"]),
                                  channel=np.array(["u10m", "v10m", "t2m"]), lat=np.array(g.lat), lon=np.array(g.lon)))
    prob = np.random.default_rng(1).random((2, n_ev, 19, 36)).astype(np.float32)
    pd = xr.DataArray(prob, dims=["time", "event", "lat", "lon"],
                      coords=dict(time=times, event=np.array(["t2m>273.15", "u10m>15"][:n_ev]), lat=np.array(g.lat),
                                  lon=np.array(g.lon)))
    return stats, prob, sd, pd


def test_prediction_accessors_on_hand_made_arrays():
    stats, prob, sd, pd = _hand_made()
    e = GlobalEnsemblePrediction(sd, pd, "pangu", 4)
    assert e.statistics == ["mean", "spread", "q0.1", "q0.9"] and e.channels == ["u10m", "v10m", "t2m"]
    assert e.events == ["t2m>273.15", "u10m>15"] and "members=4" in repr(e)
    for gp, k in ((e.mean, 0), (e.spread, 1), (e.quantile(0.1), 2), (e.quantile(0.9), 3)):
        assert isinstance(gp, GlobalPrediction)
        np.testing.assert_array_equal(gp.prediction.values, stats[:, k])
    # GlobalPrediction's accessors work unchanged: lon < 0 wraps, wind speed from u / v
    lon = float(np.asarray(sd.coords["lon"])[34])
    assert e.mean.point(lat=90.0, lon=lon - 360.0, channel="t2m") == stats[1, 0, 2, 0, 34]
    u, v = stats[1, 0, 0, 9, 1], stats[1, 0, 1, 9, 1]
    assert np.isclose(e.mean.wind_speed(0.0, 10.0, "10m"), (float(u) ** 2 + float(v) ** 2) ** 0.5)
    assert e.point(90.0, lon - 360.0, "t2m", statistic="q0.9", n_step=0) == stats[0, 3, 2, 0, 34]
    assert e.point(-90.0, 0.0, "u10m") == stats[1, 0, 0, 18, 0]
    np.testing.assert_array_equal(e.probability_of("u10m", 15.0), prob[1, 1])
    np.testing.assert_array_equal(e.probability_of("t2m", 273.15, n_step=0), prob[0, 0])
    with pytest.raises(KeyError):
        e.quantile(0.5)
    with pytest.raises(KeyError):
        e.probability_of("t2m", 280.0)
    with pytest.raises(KeyError):
        e.point(0.0, 0.0, "msl")


def test_netcdf_round_trip_of_both_arrays(tmp_path):
    from skyrim_b200.common import save_forecast
    stats, prob, sd, pd = _hand_made()
    t1 = T0 + datetime.timedelta(hours=6)
    cfg = dict(output_dir=str(tmp_path), forecast_id="f")
    ps = save_forecast(sd, "pangu-ens4", T0, t1, "synthetic", config=cfg)
    pp = save_forecast(pd, "pangu-ens4-prob", T0, t1, "synthetic", config=cfg)
    for path, da, vals in ((ps, sd, stats), (pp, pd, prob)):
        back = xr.open_dataarray(path)
        assert tuple(back.dims) == tuple(da.dims)
        np.testing.assert_array_equal(back.values, vals)
        for d in da.dims:
            np.testing.assert_array_equal(np.asarray(back.coords[d]), np.asarray(da.coords[d]))


# ---- predict_ensemble host logic on a CPU fake of EnsembleRunner ---------------------------------------------------------
class FakeLoop:
    n_history_levels = 1
    time_step = datetime.timedelta(hours=6)
    in_channel_names = out_channel_names = CH
    grid = equiangular_grid(19, 36)
    device = torch.device("cpu")
    engine = None

    def __call__(self, time, x):   # the single-forecast path (rollout): x -> x + 1 per step
        cur = x[:, -1].float()
        while True:
            yield time, cur.clone(), None
            cur, time = cur + 1.0, time + self.time_step


class FakeModel(GlobalModel):
    def __init__(self, ic_source="synthetic", **kw):
        super().__init__("pangu", ic_source=ic_source)

    def build_model(self):
        return FakeLoop()


class FakeRunner:
    """what EnsembleRunner.iter_stats yields, from CPU members that gain 1 per step, reduced by the oracle"""
    made = []

    def __init__(self, engine, base, sigma, members_per_gpu, rank=0, amp=0.05, seed=0, perturbation="gaussian", grf=None):
        rng = np.random.default_rng(seed)
        self.kw = dict(members=members_per_gpu, rank=rank, amp=amp, seed=seed, perturbation=perturbation, grf=grf)
        self.x = base[None] + amp * np.asarray(sigma)[:, None, None] * rng.standard_normal((members_per_gpu,) + base.shape)
        FakeRunner.made.append(self)

    def iter_stats(self, n_steps, channels=None, quantiles=(), events=(), channel_offset=0):
        self.reduced = []
        for n in range(n_steps + 1):
            self.reduced.append(self.x[:, channel_offset:])
            s, p = ens_stats_ref.ensemble_stats(self.x[:, channel_offset:], channels, quantiles, events)
            yield n, torch.from_numpy(s), torch.from_numpy(p)
            self.x = self.x + 1.0


@pytest.fixture
def fake_runner(monkeypatch):
    from skyrim_b200 import ensemble
    FakeRunner.made = []
    monkeypatch.setattr(ensemble, "EnsembleRunner", FakeRunner)
    return FakeRunner


def test_predict_ensemble_host_logic_and_files(tmp_path, fake_runner):
    gm = FakeModel()
    pred, paths = gm.predict_ensemble(T0, n_steps=3, members=5, quantiles=(0.1, 0.9), events={"t2m": [280.0, 300.0]},
                                      channels=["msl", "t2m"], seed=7, save=True,
                                      save_config=dict(output_dir=str(tmp_path), forecast_id="fid"))
    run = fake_runner.made[0]
    assert run.kw == dict(members=5, rank=0, amp=0.05, seed=7, perturbation="spherical_grf", grf=dict(lmax=9))
    assert pred.channels == ["t2m", "msl"] and pred.statistics == ["mean", "spread", "q0.1", "q0.9"]
    assert pred.events == ["t2m>280", "t2m>300"]
    assert len(run.reduced) == 4
    want = [ens_stats_ref.ensemble_stats(x, [2, 3], (0.1, 0.9), [(0, 280.0), (0, 300.0)]) for x in run.reduced[-2:]]
    np.testing.assert_array_equal(pred.stats.values, np.stack([w[0] for w in want]))
    np.testing.assert_array_equal(pred.probability.values, np.stack([w[1] for w in want]))
    assert list(np.asarray(pred.stats.coords["time"])) == [np.datetime64("2024-05-07T12:00:00"), np.datetime64("2024-05-07T18:00:00")]
    names = [os.path.basename(p) for p in paths]
    assert names == ["pangu-ens5__synthetic__20240507_00:00__20240507_06:00.nc",
                     "pangu-ens5-prob__synthetic__20240507_00:00__20240507_06:00.nc",
                     "pangu-ens5__file__20240507_06:00__20240507_12:00.nc",
                     "pangu-ens5-prob__file__20240507_06:00__20240507_12:00.nc",
                     "pangu-ens5__file__20240507_12:00__20240507_18:00.nc",
                     "pangu-ens5-prob__file__20240507_12:00__20240507_18:00.nc"]
    assert all(os.path.dirname(p) == str(tmp_path / "fid") for p in paths)
    last_s, last_p = xr.open_dataarray(paths[-2]), xr.open_dataarray(paths[-1])
    np.testing.assert_array_equal(last_s.values, pred.stats.values)
    np.testing.assert_array_equal(last_p.values, pred.probability.values)
    assert list(last_s.coords["statistic"]) == pred.statistics and list(last_p.coords["event"]) == pred.events


def test_predict_ensemble_filter_vars_select_on_the_device_and_no_events(tmp_path, fake_runner):
    gm = FakeModel()
    pred, paths = gm.predict_ensemble(T0, n_steps=1, members=2, perturbation="gaussian", save=True,
                                      save_config=dict(output_dir=str(tmp_path), filter_vars=["v10m"]))
    assert fake_runner.made[0].kw["grf"] is None
    assert pred.channels == ["v10m"] and pred.probability is None and len(paths) == 1
    assert pred.stats.shape == (2, 2, 1, 19, 36)
    pred, paths = gm.predict_ensemble(T0, n_steps=2, members=3, save=False)
    assert paths == [] and pred.channels == CH


@pytest.mark.parametrize("kw", [
    dict(events={"z500": 5000.0}), dict(channels=["nope"]), dict(save_config=dict(filter_vars=["nope"])),
    dict(quantiles=(1.5,)), dict(quantiles=(-0.01,)), dict(quantiles=(float("nan"),)), dict(quantiles=(0.5,) * 9),
    dict(members=0), dict(members=65), dict(n_steps=0), dict(events={"t2m": float("inf")}),
    dict(save=True, save_config=dict(file_type="zarr")),
])
def test_predict_ensemble_refuses_bad_arguments(kw, fake_runner):
    args = dict(start_time=T0, n_steps=1, members=4)
    args.update(kw)
    with pytest.raises(ValueError):
        FakeModel().predict_ensemble(**args)
    assert fake_runner.made == []       # refused before any member exists


def test_zarr_refusal_names_the_reason():
    with pytest.raises(ValueError, match="netCDF"):
        FakeModel().predict_ensemble(T0, 1, 4, save=True, save_config=dict(file_type="zarr"))


def test_forecast_cli_ensemble_options(tmp_path, monkeypatch, fake_runner):
    from click.testing import CliRunner
    from skyrim_b200 import forecast as F
    from skyrim_b200.core import models as M
    opts = {o.name: o for o in F.main.params}
    assert opts["members"].default == 1 and opts["perturbation"].default == "spherical_grf"
    assert opts["amp"].default == 0.05 and opts["seed"].default == 0
    monkeypatch.setitem(M.MODELS, "pangu", FakeModel)
    out = str(tmp_path)
    r = CliRunner().invoke(F.main, ["-m", "pangu", "-l", "12", "-o", out, "--members", "4", "--quantiles", "0.1,0.5,0.9",
                                    "--exceed", "t2m:273.15,u10m:15", "--seed", "3", "--amp", "0.1"])
    assert r.exit_code == 0, r.output
    paths = [ln for ln in r.output.splitlines() if ln.endswith(".nc")]
    assert len(paths) == 4 and sum("-ens4-prob__" in p for p in paths) == 2
    assert fake_runner.made[-1].kw == dict(members=4, rank=0, amp=0.1, seed=3, perturbation="spherical_grf", grf=dict(lmax=9))
    da = xr.open_dataarray(paths[0])
    assert list(da.coords["statistic"]) == ["mean", "spread", "q0.1", "q0.5", "q0.9"]
    assert list(xr.open_dataarray(paths[1]).coords["event"]) == ["u10m>15", "t2m>273.15"]
    # --members 1 keeps the single-forecast path: no runner, the rollout's file names
    n = len(fake_runner.made)
    r = CliRunner().invoke(F.main, ["-m", "pangu", "-l", "6", "-o", out, "-f", "t2m"])
    assert r.exit_code == 0, r.output
    assert len(fake_runner.made) == n
    paths = [ln for ln in r.output.splitlines() if ln.endswith(".nc")]
    assert len(paths) == 1 and os.path.basename(paths[0]).startswith("pangu__synthetic__")
    for bad in (["--members", "65"], ["--members", "0"], ["--quantiles", "0.5"], ["--members", "2", "--exceed", "t2m"],
                ["--members", "2", "--perturbation", "bred"]):
        assert CliRunner().invoke(F.main, ["-o", out] + bad).exit_code != 0, bad
    assert len(fake_runner.made) == n
