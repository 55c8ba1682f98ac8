"""Forecasts at sites without a GPU: the site stencil of the fp64 reference (oracle/sites_ref.py), the refusals of the site
input, the observations and GlobalModel.predict_sites / score_sites before any engine call, the command line's usage
errors, the shim's site coordinates through netCDF, and SiteScores formed from hand-made sums."""
import datetime

import numpy as np
import pytest

from oracle import sites_ref as R
from skyrim_b200 import scores as S
from skyrim_b200 import sites as St
from skyrim_b200 import xr_shim as xr
from skyrim_b200.core.models.base import GlobalModel
from skyrim_b200.timeloop import equiangular_grid

T0 = datetime.datetime(2024, 5, 7)
STEP = datetime.timedelta(hours=6)
CH = ["t2m", "u10m", "v10m", "msl"]


# ---- the stencil -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nlat,nlon", [(41, 96), (721, 1440), (7, 5)])
def test_bilinear_weights_sum_to_one_and_stay_in_the_plane(nlat, nlon):
    rng = np.random.default_rng(nlat)
    lat, lon = rng.uniform(-90, 90, 500), rng.uniform(-720, 720, 500)
    idx, w = R.stencil(lat, lon, nlat, nlon)
    assert np.allclose(w.sum(1), 1.0, rtol=0, atol=1e-14) and (w >= 0).all()
    assert (idx >= 0).all() and (idx < nlat * nlon).all()
    idx, w = R.stencil(lat, lon, nlat, nlon, R.NEAREST)
    assert (w == np.array([1.0, 0, 0, 0])).all() and (idx >= 0).all() and (idx < nlat * nlon).all()


@pytest.mark.parametrize("method", [R.BILINEAR, R.NEAREST])
def test_grid_points_take_one_point_whole(method):
    g = equiangular_grid(41, 96)
    lat, lon = np.meshgrid(np.asarray(g.lat), np.asarray(g.lon), indexing="ij")
    idx, w = R.stencil(lat.ravel(), lon.ravel(), 41, 96, method)
    south = np.arange(41 * 96) >= 40 * 96
    assert (idx[~south, 0] == np.arange(40 * 96)).all()
    if method == R.NEAREST:
        assert (idx[south, 0] == np.arange(40 * 96, 41 * 96)).all()
    else:                      # the south pole row is reached as i0 = nlat - 2 with a = 1
        assert (w[~south] == np.array([1.0, 0, 0, 0])).all()
        assert (w[south] == np.array([0.0, 0, 1, 0])).all() and (idx[south, 2] == np.arange(40 * 96, 41 * 96)).all()


def test_poles_and_the_seam():
    nlat, nlon = 41, 96                                     # 4.5 x 3.75 degrees
    idx, w = R.stencil([90.0, -90.0], [17.0, 17.0], nlat, nlon)
    assert (idx[0, :2] // nlon == 0).all() and w[0, 2:].sum() == 0.0
    assert (idx[1, 2:] // nlon == nlat - 1).all() and w[1, :2].sum() == 0.0
    a, wa = R.stencil([10.0], [359.9], nlat, nlon)
    b, wb = R.stencil([10.0], [-0.1], nlat, nlon)
    assert (a == b).all() and (wa == wb).all()
    assert a[0, 0] % nlon == nlon - 1 and a[0, 1] % nlon == 0         # j1 wraps to column 0
    c, wc = R.stencil([10.0], [720.0], nlat, nlon)
    d, wd = R.stencil([10.0], [0.0], nlat, nlon)
    assert (c == d).all() and (wc == wd).all() and c[0, 0] % nlon == 0 and wc[0, 1] == 0.0
    n, _ = R.stencil([10.0, 10.0], [359.9, -0.1], nlat, nlon, R.NEAREST)
    assert (n[:, 0] % nlon == 0).all()                      # nearest measures longitude around the circle


def test_nearest_ties_go_south_and_east():
    nlat, nlon = 41, 96
    idx, _ = R.stencil([90.0 - 2.25, 0.0], [0.0, 3.75 / 2], nlat, nlon, R.NEAREST)
    assert idx[0, 0] == 1 * nlon                            # half a row below the pole: row 1
    assert idx[1, 0] == 20 * nlon + 1                       # half a column east of 0: column 1
    idx, _ = R.stencil([0.0], [360.0 - 3.75 / 2], nlat, nlon, R.NEAREST)
    assert idx[0, 0] == 20 * nlon                           # half a column west of 360: column 0


def test_sample_reference_skips_zero_weights():
    x = np.arange(2 * 3 * 5 * 8, dtype=np.float32).reshape(2, 3, 5, 8)
    x[:, :, 2, 3] = np.nan
    g = equiangular_grid(5, 8)
    idx, w = R.stencil([g.lat[2]], [g.lon[4]], 5, 8, R.NEAREST)
    v = R.sample(x, idx, w, [2, 0])
    assert v.shape == (2, 2, 1) and (v[:, :, 0] == x[:, [2, 0], 2, 4]).all()
    idx, w = R.stencil([g.lat[2]], [g.lon[3] + 1.0], 5, 8)
    assert np.isnan(R.sample(x, idx, w, [0])).all()


def test_site_terms_reference_missing_rule():
    rng = np.random.default_rng(1)
    v = rng.standard_normal((4, 2, 6)).astype(np.float32)
    y = rng.standard_normal((2, 6)).astype(np.float32)
    y[0, 1] = np.nan
    v[2, 1, 3] = np.nan
    t = R.site_terms(v, y)
    assert (t[0, 1] == 0).all() and t[1, 3, 0] == 1.0 and np.isnan(t[1, 3, 1:]).all()
    s, _ = R.site_sums(v, y)
    assert s[0, 0] == 5 and np.isnan(s[1, 1:]).all() and s[1, 0] == 6


# ---- site input and observations ------------------------------------------------------------------------------------------
def test_read_sites_forms_and_refusals(tmp_path):
    names, lat, lon = St.read_sites({"a": (1, 2), "b": (-3, 400)})
    assert names == ["a", "b"] and lat.tolist() == [1, -3] and lon.tolist() == [2, 400]
    p = tmp_path / "s.csv"
    p.write_text("name,lat,lon\nparis, 48.85, 2.35\n\noslo,59.9,10.7\n")
    assert St.read_sites(p)[0] == ["paris", "oslo"]
    assert St.read_sites((["x"], [0.5], [1.5]))[1].tolist() == [0.5]
    bad = [({"a": (91, 0)}, "lat must lie"), ({"a": (np.nan, 0)}, "must be finite"), ({"a": (0, np.inf)}, "finite"),
           ((["a", "a"], [0, 1], [0, 1]), "duplicate"), ((["a", "b"], [0], [0, 1]), "one of each"), ({}, "no sites"),
           ({"a": 3}, "maps each name")]
    for s, msg in bad:
        with pytest.raises(ValueError, match=msg):
            St.read_sites(s)
    p.write_text("a,1,2\nb,x,2\n")
    with pytest.raises(ValueError, match="line 2"):
        St.read_sites(p)
    p.write_text("a,1,2,3\n")
    with pytest.raises(ValueError, match="name,lat,lon"):
        St.read_sites(p)
    with pytest.raises(TypeError):
        St.read_sites(42)


def observations(times, names=("a", "b", "c"), channels=("t2m", "u10m"), seed=0):
    rng = np.random.default_rng(seed)
    v = rng.standard_normal((len(times), len(names), len(channels))).astype(np.float32)
    return xr.DataArray(v, dims=["time", "site", "channel"],
                        coords=dict(time=np.array([np.datetime64(t, "s") for t in times]), site=np.array(names),
                                    channel=np.array(channels), lat=("site", np.linspace(-60, 60, len(names))),
                                    lon=("site", np.linspace(0, 300, len(names)))))


def test_read_observations_refusals():
    obs = observations([T0, T0 + STEP])
    names, lat, lon, times, sel, vals = St.read_observations(obs, ["u10m"])
    assert names == ["a", "b", "c"] and sel == ["u10m"] and vals.shape == (2, 3, 1)
    assert (vals[..., 0] == obs.values[..., 1]).all()
    with pytest.raises(ValueError, match="lack channel"):
        St.read_observations(obs, ["msl"])
    with pytest.raises(ValueError, match="dims"):
        St.read_observations(xr.DataArray(obs.values[0], dims=["site", "channel"]))
    no_lat = xr.DataArray(obs.values, dims=obs.dims, coords={k: obs.coords[k] for k in ("time", "site", "channel")})
    with pytest.raises(ValueError, match="'lat'"):
        St.read_observations(no_lat)
    twice = observations([T0, T0])
    with pytest.raises(ValueError, match="twice"):
        St.read_observations(twice)


def test_check_equiangular():
    g = equiangular_grid(41, 96)
    St.check_equiangular(g.lat, g.lon)
    with pytest.raises(ValueError, match="not equiangular"):
        St.check_equiangular(np.linspace(89, -89, 41), g.lon)
    with pytest.raises(ValueError, match="not equiangular"):
        St.check_equiangular(g.lat, np.asarray(g.lon) + 0.5)


# ---- GlobalModel refusals, before any engine call -------------------------------------------------------------------------
class FakeLoop:
    n_history_levels = 1
    time_step = STEP
    in_channel_names = out_channel_names = CH
    grid = equiangular_grid(9, 16)
    engine = None


class FakeModel(GlobalModel):
    forcing_channels = ("msl",)

    def __init__(self, grid=None):
        self._grid = grid
        super().__init__("pangu", ic_source="synthetic")

    def build_model(self):
        loop = FakeLoop()
        if self._grid is not None:
            loop.grid = self._grid
        return loop

    def _score_runner(self, *a, **kw):
        raise AssertionError("the engine was reached")


def test_predict_sites_refusals():
    m = FakeModel()
    sites = {"a": (10, 20)}
    bad = [(dict(channels=["z999"]), "unknown channel"), (dict(members=0), "members"), (dict(members=65), "members"),
           (dict(method="cubic"), "unknown site method"), (dict(perturbation="big"), "unknown perturbation"),
           (dict(quantiles=[0.5]), "members > 1"), (dict(events={"t2m": 1.0}), "members > 1"),
           (dict(members=2, quantiles=[1.5]), "quantiles"), (dict(members=2, events={"t2m": np.nan}), "finite"),
           (dict(members=2, events={"q": 1.0}), "unknown channel"), (dict(sites={"a": (95, 0)}), "lat must lie"),
           (dict(n_steps=-1), "negative"), (dict(save=True, save_config={"file_type": "zarr"}), "netCDF")]
    for kw, msg in bad:
        args = dict(start_time=T0, n_steps=2, sites=sites)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            m.predict_sites(**args)
    big = (["s%d" % i for i in range(1 << 20)], np.zeros(1 << 20), np.zeros(1 << 20))
    with pytest.raises(ValueError, match="2\\^31"):
        m.predict_sites(T0, 40, big, members=4)
    crooked = type("G", (), dict(lat=np.linspace(88, -88, 9).tolist(), lon=FakeLoop.grid.lon))()
    with pytest.raises(ValueError, match="not equiangular"):
        FakeModel(crooked).predict_sites(T0, 2, sites)


def test_score_sites_refusals():
    m = FakeModel()
    obs = observations([T0, T0 + STEP], channels=("t2m", "msl"))
    bad = [(dict(channels=["msl"]), "forcings"), (dict(channels=["z999"]), "unknown channel"),
           (dict(start_times=[T0 + STEP, T0]), "sorted"), (dict(start_times=[]), "at least one"),
           (dict(seed=-1), "seed"), (dict(observations=observations([T0 + 100 * STEP])), "no value"),
           (dict(observations=observations([T0], channels=("q",))), "none of"), (dict(method="x"), "site method"),
           (dict(channels=["u10m"]), "lack channel")]
    for kw, msg in bad:
        args = dict(start_times=[T0], n_steps=1, observations=obs)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            m.score_sites(**args)
    empty = observations([T0])
    empty.values[:] = np.nan
    with pytest.raises(ValueError, match="no value"):
        m.score_sites([T0], 1, empty)


def test_multi_model_ensemble_refuses_sites():
    from skyrim_b200.core.models.ensemble import GlobalEnsemble
    for fn in (GlobalEnsemble.predict_sites, GlobalEnsemble.score_sites):
        with pytest.raises(NotImplementedError, match="Skyrim\\(name\\)"):
            fn(None)


# ---- the command line ---------------------------------------------------------------------------------------------------
def test_cli_usage_errors(tmp_path):
    from click.testing import CliRunner
    from skyrim_b200 import forecast as F
    out = str(tmp_path / "out")
    for bad in (["--site_method", "nearest"], ["--observations", "o.nc"],
                ["--sites", "s.csv", "--observations", "o.nc", "--truth", "t.nc"],
                ["--sites", "s.csv", "--observations", "o.nc", "--climatology", "c.nc"],
                ["--models", "pangu,graphcast", "--sites", "s.csv", "--observations", "o.nc", "--compare"],
                ["--sites", "s.csv", "--observations", "o.nc", "--map_channels", "t2m"],
                ["--sites", "s.csv", "--observations", "o.nc", "--map_leads", "6"],
                ["--sites", "s.csv", "--observations", "o.nc", "--members", "2", "--quantiles", "0.5"],
                ["--sites", "s.csv", "--models", "pangu,graphcast"], ["--sites", "s.csv", "--score"],
                ["--sites", "s.csv", "--until", "20240509"], ["--sites", "s.csv", "--truth", "t.nc"],
                ["--sites", "s.csv", "--quantiles", "0.5"]):
        r = CliRunner().invoke(F.main, ["-o", out, "-d", "20240507"] + bad)
        assert r.exit_code == 2 and "Usage" in r.output, (bad, r.output)


# ---- the shim ----------------------------------------------------------------------------------------------------------
def test_site_coordinates_survive_netcdf(tmp_path):
    obs = observations([T0, T0 + STEP])
    p = tmp_path / "o.nc"
    obs.to_netcdf(p)
    back = xr.open_dataarray(p)
    assert tuple(back.dims) == ("time", "site", "channel") and (back.values == obs.values).all()
    for c in ("lat", "lon"):
        assert np.asarray(back.coords[c]).dtype == np.float64
        assert (np.asarray(back.coords[c]) == np.asarray(obs.coords[c])).all()
    assert list(back.coords["site"]) == ["a", "b", "c"]
    sub = back.sel(site=["c", "a"])
    assert np.asarray(sub.coords["lat"]).tolist() == [60.0, -60.0]
    assert St.read_observations(sub)[0] == ["c", "a"]
    one = back.sel(site="b")
    assert tuple(one.dims) == ("time", "channel") and float(np.asarray(one.coords["lon"])) == 150.0


def test_files_without_site_coordinates_have_no_coordinates_attribute(tmp_path):
    da = xr.DataArray(np.ones((2, 3), np.float32), dims=["channel", "lat"],
                      coords=dict(channel=np.array(["a", "b"]), lat=np.array([1.0, 2.0, 3.0])))
    da.to_netcdf(tmp_path / "a.nc")
    assert b"coordinates" not in (tmp_path / "a.nc").read_bytes()


# ---- SiteScores -------------------------------------------------------------------------------------------------------------
def test_site_scores_from_hand_made_sums():
    M, D, L, Sn, n = 3, 2, 2, 1, 3
    sums = np.zeros((D, L, Sn, 6))
    sums[..., 0] = 4.0                                     # 4 observations per date and lead
    sums[..., 1] = 2.0                                     # e
    sums[..., 2] = 8.0                                     # e^2
    sums[..., 3] = 12.0                                    # var
    sums[..., 4] = 6.0                                     # mae
    sums[..., 5] = 3.0                                     # G
    acc = np.zeros((L, Sn, n, 6))
    acc[:, :, :2] = sums[0, :, :, None] * np.array([1.0, 1.0])[None, None, :, None]
    acc[:, :, 2] = 0.0                                     # site c: never observed
    res = St.SiteScores.build(sums, acc, M, [T0, T0 + 4 * STEP], [0.0, 6.0], ["a", "b", "c"], [1.0, 2.0, 3.0],
                              [4.0, 5.0, 6.0], ["t2m"], "pangu")
    card = res.card.values
    assert tuple(res.card.dims) == ("lead_time", "metric", "channel") and card.shape == (2, 6, 1)
    k = {m: i for i, m in enumerate(St.SITE_METRICS)}
    np.testing.assert_allclose(card[:, k["bias"]], 0.5)
    np.testing.assert_allclose(card[:, k["rmse"]], np.sqrt(2.0))
    np.testing.assert_allclose(card[:, k["spread"]], np.sqrt(12.0 / 2 / 4))
    np.testing.assert_allclose(card[:, k["ssr"]], np.sqrt(4 / 3) * np.sqrt(1.5) / np.sqrt(2.0))
    np.testing.assert_allclose(card[:, k["crps"]], (6.0 - 3.0 / 9) / 4)
    np.testing.assert_allclose(card[:, k["crps_fair"]], (6.0 - 3.0 / 6) / 4)
    assert res.cards.values.shape == (2, 2, 6, 1) and (res.cards.values[0] == card).all()
    assert tuple(res.sites.dims) == ("lead_time", "metric", "site", "channel") and res.sites.values.shape == (2, 6, 3, 1)
    np.testing.assert_allclose(res.sites.values[:, :, 0], card)
    assert np.isnan(res.sites.values[:, :, 2]).all()
    assert tuple(res.count.dims) == ("lead_time", "site", "channel")
    assert res.count.values[:, :, 0].tolist() == [[4, 4, 0], [4, 4, 0]]
    assert np.asarray(res.sites.coords["lat"]).tolist() == [1.0, 2.0, 3.0]
    want = S.metrics_from_sums(np.concatenate([sums.sum(0), np.full((L, Sn, 3), np.nan)], -1), M)
    np.testing.assert_array_equal(card, np.moveaxis(want[..., [S.METRICS.index(m) for m in St.SITE_METRICS]], -1, 1))
