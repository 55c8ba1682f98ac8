"""Forecast scores without a device: the oracle's CRPS against its integral definition, the region weights, the metrics
from sums, the C-ABI's argument refusals, and GlobalModel.score's host logic on a CPU fake of the member runner (truth and
climatology adapters, the scorecard, its netCDF file and the forecast CLI options)."""
import ctypes as C
import datetime
import os
import re

import numpy as np
import pytest
import torch

from oracle import scores_ref
from skyrim_b200 import scores as S
from skyrim_b200 import xr_shim as xr
from skyrim_b200.core.models.base import GlobalModel
from skyrim_b200.timeloop import equiangular_grid

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CH = ["u10m", "v10m", "t2m", "msl"]
T0 = datetime.datetime(2024, 5, 7)
G = equiangular_grid(19, 36)


# ---- definitions ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1, 2, 3, 5, 8])
def test_oracle_crps_is_the_integral_of_the_squared_cdf_difference(M):
    rng = np.random.default_rng(M)
    for _ in range(3):
        xs, y = rng.standard_normal(M), float(rng.standard_normal())
        x = xs.reshape(M, 1, 1, 1)
        m = scores_ref.metrics(x, np.array([[[y]]]), np.ones((1, 1)), [0])[0, 0]
        assert np.isclose(m[5], scores_ref.crps_integral(xs, y), rtol=1e-12, atol=1e-15)
        pair = np.abs(xs[:, None] - xs[None, :]).sum()
        if M > 1:
            assert np.isclose(m[6], np.abs(xs - y).mean() - pair / (2 * M * (M - 1)), rtol=1e-13)
        else:
            assert np.isnan(m[6]) and np.isnan(m[3]) and np.isnan(m[4])
            assert m[5] == abs(xs[0] - y) and m[1] == abs(xs[0] - y) and m[0] == xs[0] - y
        assert np.isnan(m[2])   # no climatology


def test_region_weights():
    names, w = S.region_weights(G.lat, {"global": (-90, 90), "tropics": (-20, 20), "north": (20, 90)})
    assert names == ["global", "tropics", "north"] and w.shape == (3, 19) and w.dtype == np.float64
    assert (w[:, 0] == 0).all() and (w[:, -1] == 0).all()                       # poles exactly 0
    np.testing.assert_allclose(w.sum(1), 1.0, rtol=1e-15)
    lat = np.asarray(G.lat)
    assert w[1, np.isclose(lat, 20)] > 0 and w[1, np.isclose(lat, -20)] > 0 and w[2, np.isclose(lat, 20)] > 0  # ends in
    assert (w[1, np.abs(lat) > 20 + 1e-6] == 0).all()
    np.testing.assert_allclose(w[0] / w[0].max(), np.cos(np.deg2rad(lat)) / np.cos(np.deg2rad(lat)).max(), atol=1e-15)
    assert S.region_weights(G.lat)[0] == ["global"]
    for bad in ({"a": (10, -10)}, {"a": (-91, 0)}, {"pole": (90, 90)}, {f"r{i}": (-90, 90) for i in range(5)}, {}):
        with pytest.raises(ValueError):
            S.region_weights(G.lat, bad)


def test_metrics_from_sums_match_the_oracle():
    rng = np.random.default_rng(2)
    for M in (1, 2, 7):
        x = rng.standard_normal((M, 3, 19, 36)) * 2 + 1
        y, k = rng.standard_normal((2, 19, 36)), rng.standard_normal((2, 19, 36)) * 0.1
        names, w = S.region_weights(G.lat, {"g": (-90, 90), "s": (-90, -10)})
        sums, _ = scores_ref.score_sums(x, y, w, [2, 0], k)
        np.testing.assert_allclose(S.metrics_from_sums(sums, M), scores_ref.metrics(x, y, w, [2, 0], k), rtol=1e-10,
                                   equal_nan=True)
        x[M - 1, 0, 5, 5] = np.nan   # a weighted point of both regions? row 5 is at 40N: only "g"
        m = S.metrics_from_sums(scores_ref.score_sums(x, y, w, [2, 0], k)[0], M)
        assert np.isnan(m[0, 1]).all() and np.isfinite(m[1, 1, :3]).all() and np.isfinite(m[:, 0, :3]).all()


# ---- C-ABI refusals ---------------------------------------------------------------------------------------------------------
def test_export_present_and_declared():
    from skyrim_b200 import _ffi
    hdr = open(os.path.join(ROOT, "include", "skyrim_b200.h")).read()
    assert "sky_forecast_scores" in set(re.findall(r"\b(sky_[a-z_0-9]+)\s*\(", hdr)) and "sky_forecast_scores" in _ffi.EXPORTS
    assert hasattr(_ffi.lib(), "sky_forecast_scores")


def _call(members=4, stride=None, nlat=8, nlon=12, count=5, channels=(0, 4), n_sel=None, n_regions=1, pbytes=None,
          null_truth=False):
    from skyrim_b200 import _ffi
    L = _ffi.lib()
    bogus = C.c_void_p(0x1000)    # never inspected: every refusal below comes before the device-pointer check
    plane = nlat * nlon
    ns = len(channels) if n_sel is None else n_sel
    need = 8 * 128 * 9 * max(n_regions, 1) * max(ns, 1)
    rc = L.sky_forecast_scores(bogus, members, count * plane if stride is None else stride, nlat, nlon, count,
                               (C.c_int32 * max(len(channels), 1))(*channels), ns, None if null_truth else bogus, None,
                               bogus, n_regions, bogus, need if pbytes is None else pbytes, bogus, None)
    return rc, L.sky_last_error().decode()


@pytest.mark.parametrize("kw, what", [
    (dict(members=0), "members"), (dict(members=65), "members"),
    (dict(nlat=0), "nlat"), (dict(nlon=-1), "nlon"), (dict(nlat=65536, nlon=65536), "2^31"),
    (dict(count=0), "channel_count"),
    (dict(channels=(0, 5)), "channel 5"), (dict(channels=(-1, 2)), "channel -1"),
    (dict(stride=5 * 96 - 1), "member_stride"), (dict(stride=-1), "member_stride"),
    (dict(channels=tuple(range(129)), count=200), "n_sel"), (dict(channels=()), "n_sel"),
    (dict(n_regions=0), "n_regions"), (dict(n_regions=5), "n_regions"),
    (dict(pbytes=8 * 128 * 9 * 2 - 1), "partial_bytes"), (dict(null_truth=True), "null"),
])
def test_library_refuses_bad_arguments_before_any_cuda_call(kw, what):
    rc, msg = _call(**kw)
    assert rc == -1 and what in msg, msg


# ---- score() host logic on a CPU fake of EnsembleRunner ---------------------------------------------------------------------
class TimeSource:
    """seeded truth that changes with time: source[t] -> DataArray(channel, lat, lon)"""

    def __init__(self, channels=CH, grid=G, seed=0, missing=()):
        self.channels, self.grid, self.seed, self.missing = list(channels), grid, seed, set(missing)

    def __getitem__(self, t):
        if t in self.missing:
            raise KeyError(t)
        h = int((t - T0).total_seconds() // 3600)
        rng = np.random.default_rng(self.seed * 1000 + h + 7)
        v = (rng.standard_normal((len(self.channels), len(self.grid.lat), len(self.grid.lon))) + 0.1 * h).astype(np.float32)
        return xr.DataArray(v, dims=["channel", "lat", "lon"], coords=dict(channel=np.array(self.channels),
                            lat=np.array(self.grid.lat), lon=np.array(self.grid.lon)))


class FakeLoop:
    n_history_levels = 1
    time_step = datetime.timedelta(hours=6)
    in_channel_names = out_channel_names = CH
    grid = G
    device = torch.device("cpu")
    engine = None


class FakeModel(GlobalModel):
    def __init__(self, ic_source="synthetic", **kw):
        super().__init__("pangu", ic_source=ic_source)

    def build_model(self):
        return FakeLoop()


class FakeRunner:
    """what EnsembleRunner.iter_scores returns, from CPU members that gain 1 per step, scored by the oracle"""
    made = []

    def __init__(self, engine, base, sigma, members_per_gpu, rank=0, amp=0.05, seed=0, perturbation="gaussian", grf=None):
        rng = np.random.default_rng(seed)
        self.kw = dict(members=members_per_gpu, rank=rank, amp=amp, seed=seed, perturbation=perturbation, grf=grf)
        noise = 0.0 if perturbation == "none" else amp * np.asarray(sigma)[:, None, None] * rng.standard_normal(
            (members_per_gpu,) + base.shape)
        self.x = base[None] + noise
        FakeRunner.made.append(self)

    def iter_scores(self, n_steps, truth_at, clim=None, channels=None, row_weights=None, channel_offset=0):
        self.members, self.truths, out = [], [], []
        for n in range(n_steps + 1):
            y = truth_at(n)
            self.members.append(self.x[:, channel_offset:])
            self.truths.append(y)
            out.append(scores_ref.score_sums(self.x[:, channel_offset:], y, row_weights, channels, clim)[0])
            self.x = self.x + 1.0
        return list(range(n_steps + 1)), torch.from_numpy(np.stack(out))


@pytest.fixture
def fake_runner(monkeypatch):
    from skyrim_b200 import ensemble
    FakeRunner.made = []
    monkeypatch.setattr(ensemble, "EnsembleRunner", FakeRunner)
    return FakeRunner


def _clim(channels=CH):
    rng = np.random.default_rng(9)
    return xr.DataArray(rng.standard_normal((len(channels), 19, 36)).astype(np.float32) * 0.1, dims=["channel", "lat", "lon"],
                        coords=dict(channel=np.array(channels), lat=np.array(G.lat), lon=np.array(G.lon)))


def test_score_host_logic_scorecard_and_file(tmp_path, fake_runner):
    src = TimeSource()
    gm = FakeModel(ic_source=src)
    regions = {"global": (-90, 90), "tropics": (-20, 20)}
    card, paths = gm.score(T0, n_steps=3, climatology=_clim(), members=4, seed=3, channels=["msl", "t2m"], regions=regions,
                           save=True, save_config=dict(output_dir=str(tmp_path), forecast_id="fid"))
    run = fake_runner.made[0]
    assert run.kw == dict(members=4, rank=0, amp=0.05, seed=3, perturbation="spherical_grf", grf=dict(lmax=9))
    assert tuple(card.dims) == ("lead_time", "metric", "region", "channel") and card.values.dtype == np.float64
    assert list(card.coords["lead_time"]) == [0.0, 6.0, 12.0, 18.0] and list(card.coords["metric"]) == list(S.METRICS)
    assert list(card.coords["region"]) == ["global", "tropics"] and list(card.coords["channel"]) == ["t2m", "msl"]
    assert card.attrs == dict(model="pangu", members=4, start_time="2024-05-07T00:00:00")
    # the truth of lead n is source[T0 + 6n h], selected by name; the climatology too
    for n in range(4):
        want = src[T0 + n * datetime.timedelta(hours=6)].values[[2, 3]]
        np.testing.assert_array_equal(run.truths[n], want)
    _, w = S.region_weights(G.lat, regions)
    for n in range(4):
        ref = scores_ref.metrics(run.members[n], run.truths[n], w, [2, 3], _clim().values[[2, 3]])
        np.testing.assert_allclose(np.moveaxis(card.values[n], 0, -1), ref, rtol=1e-10, equal_nan=True)
    assert [os.path.basename(p) for p in paths] == ["pangu-score4__file__20240507_00:00__20240507_18:00.nc"]
    back = xr.open_dataarray(paths[0])
    assert tuple(back.dims) == tuple(card.dims) and back.attrs == card.attrs
    np.testing.assert_array_equal(back.values, card.values)
    for d in card.dims:
        np.testing.assert_array_equal(np.asarray(back.coords[d]), np.asarray(card.coords[d]))


def test_score_one_member_is_unperturbed_and_defaults(fake_runner):
    src = TimeSource()
    card, paths = FakeModel(ic_source=src).score(T0, n_steps=1)
    run = fake_runner.made[0]
    assert run.kw["perturbation"] == "none" and run.kw["members"] == 1 and paths == []
    assert list(card.coords["channel"]) == CH and list(card.coords["region"]) == ["global"]
    np.testing.assert_array_equal(run.members[0][0], src[T0].values)     # lead 0 is the truth itself
    m = card.values[0, :, 0]
    assert (m[[0, 1, 5]] == 0).all() and np.isnan(m[[2, 3, 4, 6]]).all()
    # truth as a DataArray with a time dimension gives the same card
    times = [T0, T0 + datetime.timedelta(hours=6)]
    da = xr.DataArray(np.stack([src[t].values for t in times]), dims=["time", "channel", "lat", "lon"],
                      coords=dict(time=np.array([np.datetime64(t, "s") for t in times]), channel=np.array(CH),
                                  lat=np.array(G.lat), lon=np.array(G.lon)))
    card2, _ = FakeModel(ic_source=src).score(T0, n_steps=1, truth=da)
    np.testing.assert_array_equal(card2.values, card.values)


@pytest.mark.parametrize("kw, what", [
    (dict(truth=TimeSource(grid=equiangular_grid(19, 37))), "lon"),
    (dict(truth=TimeSource(grid=equiangular_grid(21, 36))), "lat"),
    (dict(truth=TimeSource(channels=["u10m", "v10m", "t2m"])), "msl"),
    (dict(truth=TimeSource(missing={T0 + datetime.timedelta(hours=6)})), "2024-05-07T06:00:00"),
    (dict(climatology=_clim(["u10m", "t2m"])), "climatology lacks channel"),
    (dict(channels=["nope"]), "nope"), (dict(members=0), "members"), (dict(members=65), "members"),
    (dict(perturbation="bred"), "bred"), (dict(regions={"a": (30, 10)}), "band"),
    (dict(save=True, save_config=dict(file_type="zarr")), "netCDF"),
])
def test_score_refusals_name_the_problem(kw, what, fake_runner):
    args = dict(start_time=T0, n_steps=1)
    args.update(kw)
    with pytest.raises(ValueError, match=re.escape(what)):
        FakeModel(ic_source=TimeSource()).score(**args)


def test_truth_time_dimension_refusal():
    da = xr.DataArray(np.zeros((1, 4, 19, 36), np.float32), dims=["time", "channel", "lat", "lon"],
                      coords=dict(time=np.array([np.datetime64(T0, "s")]), channel=np.array(CH), lat=np.array(G.lat),
                                  lon=np.array(G.lon)))
    at = S.truth_fetcher(da, ["t2m"], G.lat, G.lon)
    assert at(T0).shape == (1, 19, 36)
    with pytest.raises(ValueError, match="no analysis"):
        at(T0 + datetime.timedelta(hours=6))


def test_graphcast_forcing_channel_is_not_scored():
    from skyrim_b200.core.models.graphcast import GraphcastModel
    assert GraphcastModel.forcing_channels == ("tp06",)


def test_multi_model_score_is_refused():
    from skyrim_b200.core.models.ensemble import GlobalEnsemble
    with pytest.raises(NotImplementedError, match="multi-model"):
        GlobalEnsemble.score(None, T0, 1)


def test_forecast_cli_score_options(tmp_path, monkeypatch, fake_runner):
    from click.testing import CliRunner
    from skyrim_b200 import forecast as F
    from skyrim_b200.core import models as M
    src = TimeSource()

    class SrcModel(FakeModel):
        def __init__(self, ic_source="synthetic", **kw):
            super().__init__(ic_source=src)
    monkeypatch.setitem(M.MODELS, "pangu", SrcModel)
    times = [T0 + datetime.timedelta(hours=6 * n) for n in range(3)]
    truth = xr.DataArray(np.stack([src[t].values for t in times]), dims=["time", "channel", "lat", "lon"],
                         coords=dict(time=np.array([np.datetime64(t, "s") for t in times]), channel=np.array(CH),
                                     lat=np.array(G.lat), lon=np.array(G.lon)))
    tp, cp = tmp_path / "truth.nc", tmp_path / "clim.nc"
    truth.to_netcdf(tp)
    _clim().to_netcdf(cp)
    out = str(tmp_path / "out")
    r = CliRunner().invoke(F.main, ["-m", "pangu", "-d", "20240507", "-l", "12", "-o", out, "--score", "--truth", str(tp),
                                    "--climatology", str(cp), "--members", "3", "--seed", "2"])
    assert r.exit_code == 0, r.output
    paths = [ln for ln in r.output.splitlines() if ln.endswith(".nc")]
    assert len(paths) == 1 and os.path.basename(paths[0]).startswith("pangu-score3__")
    assert fake_runner.made[-1].kw == dict(members=3, rank=0, amp=0.05, seed=2, perturbation="spherical_grf", grf=dict(lmax=9))
    card = xr.open_dataarray(paths[0])
    assert list(card.coords["lead_time"]) == [0.0, 6.0, 12.0] and np.isfinite(card.values[:, 2]).all()   # acc
    r = CliRunner().invoke(F.main, ["-m", "pangu", "-d", "20240507", "-l", "6", "-o", out, "--score"])
    assert r.exit_code == 0, r.output
    assert fake_runner.made[-1].kw["perturbation"] == "none"
    n = len(fake_runner.made)
    for bad in (["--truth", str(tp)], ["--climatology", str(cp)], ["--score", "--models", "pangu,graphcast"],
                ["--score", "--members", "2", "--quantiles", "0.5"]):
        assert CliRunner().invoke(F.main, ["-o", out] + bad).exit_code != 0, bad
    assert len(fake_runner.made) == n


def test_truth_array_missing_time_is_refused_before_any_member_exists(fake_runner):
    src = TimeSource()
    da = xr.DataArray(src[T0].values[None], dims=["time", "channel", "lat", "lon"],
                      coords=dict(time=np.array([np.datetime64(T0, "s")]), channel=np.array(CH), lat=np.array(G.lat),
                                  lon=np.array(G.lon)))
    with pytest.raises(ValueError, match="2024-05-07T06:00:00"):
        FakeModel(ic_source=src).score(T0, 1, truth=da)
    assert fake_runner.made == []
