"""sky_sample_sites and sky_site_scores on the device against the fp64 reference (oracle/sites_ref.py): bit for bit sampling
for both methods at 41 x 96 and 721 x 1440, site statistics, site scores with missing observations and NaN members, and
GlobalModel.predict_sites / score_sites end to end on the small grids."""
import datetime
import functools

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import ens_stats_ref  # noqa: E402
from oracle import sites_ref as R  # noqa: E402

T0 = datetime.datetime(2024, 5, 7)
STEP = datetime.timedelta(hours=6)


@pytest.fixture(autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def site_set(nlat, nlon, n=300, seed=0):
    """random sites, the poles, the 360-degree seam and grid points, in random order"""
    from skyrim_b200.timeloop import equiangular_grid
    g = equiangular_grid(nlat, nlon)
    rng = np.random.default_rng(seed)
    lat = list(rng.uniform(-90, 90, n)) + [90.0, -90.0, 90.0, -90.0, 12.3, -45.6, 0.0, 33.0]
    lon = list(rng.uniform(-400, 800, n)) + [0.0, 0.0, 359.99, 123.4, 359.9, -0.1, 360.0, 720.0]
    for i in rng.integers(0, nlat, 20):
        j = int(rng.integers(0, nlon))
        lat.append(g.lat[i])
        lon.append(g.lon[j])
    lat.append(g.lat[1])
    lon.append(360.0 - (360.0 / nlon) / 2)                   # a nearest tie on the seam
    order = rng.permutation(len(lat))
    return np.asarray(lat)[order], np.asarray(lon)[order]


def sample(x, lat, lon, method, channels, channel_offset=0):
    from skyrim_b200.engine import SiteTable, sample_sites
    H, W = x.shape[-2:]
    t = SiteTable(lat, lon, H, W, method)
    out = sample_sites(torch.as_tensor(x).cuda(), t, channels, channel_offset)
    torch.cuda.synchronize()
    t.close()
    return out[:, :, 0].cpu().numpy()


@pytest.mark.parametrize("grid", [(41, 96), (721, 1440)])
@pytest.mark.parametrize("M", [1, 3, 17, 64])
@pytest.mark.parametrize("method", ["bilinear", "nearest"])
def test_sampling_is_the_reference_bit_for_bit(grid, M, method):
    H, W = grid
    C = 4 if H < 100 else 2
    rng = np.random.default_rng(M)
    x = (rng.standard_normal((M, C, H, W)) * 40 + 250).astype(np.float32)
    lat, lon = site_set(H, W, seed=M)
    ch = [C - 1, 0]
    got = sample(x, lat, lon, method, ch)
    idx, w = R.stencil(lat, lon, H, W, method)
    want = R.sample(x, idx, w, ch)
    assert got.tobytes() == want.tobytes()
    whole = w[:, 0] == 1.0                                   # grid points (and every nearest site) take one value whole
    assert whole.sum() >= 20
    assert (got[:, :, whole] == x.reshape(M, C, -1)[:, ch][:, :, idx[whole, 0]]).all()


def test_graphcast_new_slice_through_the_channel_offset():
    M, C, off, H, W = 3, 10, 5, 41, 96
    x = np.random.default_rng(3).standard_normal((M, C, H, W)).astype(np.float32)
    lat, lon = site_set(H, W, 50, seed=3)
    got = sample(x, lat, lon, "bilinear", [0, 4], channel_offset=off)
    idx, w = R.stencil(lat, lon, H, W)
    assert got.tobytes() == R.sample(x[:, off:], idx, w, [0, 4]).tobytes()


def test_nan_beside_a_nearest_site_does_not_leak_in():
    from skyrim_b200.timeloop import equiangular_grid
    H, W = 41, 96
    g = equiangular_grid(H, W)
    x = np.ones((2, 1, H, W), np.float32)
    x[:, 0, 10, 21] = np.nan
    lat, lon = np.array([g.lat[10], g.lat[10] - 1.0]), np.array([g.lon[20] + 1.0, g.lon[21] + 0.5])
    near = sample(x, lat, lon, "nearest", [0])
    assert near[:, 0, 0].tolist() == [1.0, 1.0] and np.isnan(near[:, 0, 1]).all()
    bil = sample(x, lat, lon, "bilinear", [0])
    assert np.isnan(bil).all()


def test_site_statistics_are_ensemble_statistics_of_the_values():
    from skyrim_b200.engine import SiteTable, ensemble_statistics, sample_sites
    M, C, H, W = 9, 3, 41, 96
    x = (np.random.default_rng(5).standard_normal((M, C, H, W)) * 3 + 280).astype(np.float32)
    lat, lon = site_set(H, W, 100, seed=5)
    t = SiteTable(lat, lon, H, W)
    v = sample_sites(torch.as_tensor(x).cuda(), t, [2, 1])
    q, ev = [0.1, 0.5, 0.9], [(0, 280.0), (1, 281.5)]
    stats, prob = ensemble_statistics(v, None, q, ev)
    torch.cuda.synchronize()
    want_s, want_p = ens_stats_ref.ensemble_stats(v.cpu().numpy(), [0, 1], q, ev)
    assert stats.cpu().numpy().tobytes() == want_s.tobytes() and prob.cpu().numpy().tobytes() == want_p.tobytes()
    t.close()


def scores(values, obs, calls=1):
    from skyrim_b200.engine import site_scores
    v = torch.as_tensor(values).cuda()[:, :, None].contiguous()
    y = torch.as_tensor(obs).cuda()
    acc = torch.zeros(obs.shape + (6,), dtype=torch.float64, device="cuda")
    for _ in range(calls):
        s = site_scores(v, y, acc)
    torch.cuda.synchronize()
    return acc.cpu().numpy(), s.cpu().numpy()


@pytest.mark.parametrize("M", [1, 2, 5, 16, 33, 64])
def test_site_scores_match_the_reference(M):
    rng = np.random.default_rng(10 + M)
    S, n = 3, 1000
    v = (rng.standard_normal((M, S, n)) * 3 + 280).astype(np.float32)
    y = (rng.standard_normal((S, n)) * 3 + 280).astype(np.float32)
    y[rng.random((S, n)) < 0.2] = np.nan                   # missing observations
    acc, sums = scores(v, y, calls=2)
    t = R.site_terms(v, y)
    mag = np.abs(t) + 1e-300
    assert (np.abs(acc - 2 * t) <= 1e-12 * 2 * mag).all()
    want, wmag = R.site_sums(v, y)
    assert (np.abs(sums - want) <= 1e-12 * wmag + 1e-300).all()
    assert (sums[:, 0] == (~np.isnan(y)).sum(1)).all() and (acc[np.isnan(y)] == 0).all()


def test_nan_member_poisons_its_site_and_channel_only():
    rng = np.random.default_rng(2)
    v = rng.standard_normal((4, 3, 300)).astype(np.float32)
    y = rng.standard_normal((3, 300)).astype(np.float32)
    v[1, 1, 7] = np.nan
    v[2, 2, 9] = np.nan
    y[2, 9] = np.nan                                        # missing there: the NaN member is not read into anything
    acc, sums = scores(v, y)
    assert np.isnan(acc[1, 7, 1:]).all() and acc[1, 7, 0] == 1.0 and np.isnan(acc).sum() == 5
    assert np.isnan(sums[1, 1:]).all() and np.isfinite(sums[[0, 2]]).all() and sums[1, 0] == 300


def test_site_scores_are_reproducible_and_independent_of_the_channels():
    rng = np.random.default_rng(4)
    v = rng.standard_normal((8, 4, 700)).astype(np.float32)
    y = rng.standard_normal((4, 700)).astype(np.float32)
    y[:, ::5] = np.nan
    a1, s1 = scores(v, y, 3)
    a2, s2 = scores(v, y, 3)
    assert a1.tobytes() == a2.tobytes() and s1.tobytes() == s2.tobytes()
    a3, s3 = scores(v[:, 2:3].copy(), y[2:3].copy(), 3)
    assert a3[0].tobytes() == a1[2].tobytes() and s3[0].tobytes() == s1[2].tobytes()


def test_full_size_sampling_of_a_pangu_state():
    from skyrim_b200.config import PANGU_CHANNELS
    from skyrim_b200.weights import synthetic_state
    x = synthetic_state(PANGU_CHANNELS, 721, 1440, 0)[None].astype(np.float32)
    x = np.concatenate([x, x + 1.0])
    lat, lon = site_set(721, 1440, 5000, seed=9)
    for method in ("bilinear", "nearest"):
        ch = list(range(0, 69, 7))
        idx, w = R.stencil(lat, lon, 721, 1440, method)
        assert sample(x, lat, lon, method, ch).tobytes() == R.sample(x, idx, w, ch).tobytes()


# ---- end to end ------------------------------------------------------------------------------------------------------------
class TimeSource:
    """seeded analyses that change with time: source[t] = synthetic state + 0.05 sigma N(0, 1) drawn per hour"""

    def __init__(self, channels, nlat, nlon):
        from skyrim_b200.timeloop import equiangular_grid
        from skyrim_b200.weights import channel_stats, synthetic_state
        self.channels, self.grid = list(channels), equiangular_grid(nlat, nlon)
        self.base, self.sigma = synthetic_state(self.channels, nlat, nlon, 0), channel_stats(self.channels)[1]

    def __getitem__(self, t):
        from skyrim_b200 import xr_shim as xr
        h = int((t - datetime.datetime(2024, 1, 1)).total_seconds() // 3600)
        eps = np.random.default_rng(h).standard_normal(self.base.shape).astype(np.float32)
        v = (self.base + np.float32(0.05) * self.sigma[:, None, None] * eps).astype(np.float32)
        return xr.DataArray(v, dims=["channel", "lat", "lon"], coords=dict(channel=np.array(self.channels),
                            lat=np.array(self.grid.lat), lon=np.array(self.grid.lon)))


def _model(name, schedule=None):
    from skyrim_b200.config import (FCNV2_CHANNELS, GRAPHCAST_CHANNELS, PANGU_CHANNELS, graphcast_small, pangu_small,
                                    sfno_small)
    from skyrim_b200.core import Skyrim
    cfg, grid, ch = {"pangu": (pangu_small(41, 96), (41, 96), PANGU_CHANNELS),
                     "fourcastnet_v2": (sfno_small(49, 96), (49, 96), FCNV2_CHANNELS),
                     "graphcast": (graphcast_small(41, 96, 2, 512, 2), (41, 96), GRAPHCAST_CHANNELS)}[name]
    kw = dict(schedule=schedule) if schedule else {}
    return Skyrim(name, cfg=cfg, ic_source=TimeSource(ch, *grid), **kw)


def _runner_members(gm, t0, n_steps, M, seed):
    """the members an identically seeded runner holds at every lead (host (M, C, H, W) per lead)"""
    from skyrim_b200.ensemble import EnsembleRunner, HierarchicalEnsembleRunner
    base, sigma, off = gm._ensemble_initial_state(t0)
    make = EnsembleRunner
    if hasattr(gm.model, "engine_24"):
        make = functools.partial(HierarchicalEnsembleRunner, engine_24=gm.model.engine_24, every_slice=True)
    run = make(gm.model.engine, base, sigma, members_per_gpu=M, perturbation="spherical_grf" if M > 1 else "none",
               grf=dict(lmax=min(180, (len(gm.model.grid.lat) - 1) // 2)), seed=seed)
    return [m[:, off:].cpu().numpy() for _, m in run._walk(n_steps)]


CASES = [("pangu", None), ("pangu", "hierarchical"), ("fourcastnet_v2", None), ("graphcast", None)]


@pytest.mark.parametrize("name, schedule", CASES)
def test_predict_sites_end_to_end(name, schedule):
    gm = _model(name, schedule).model
    names = list(gm.out_channel_names)
    H, W = len(gm.model.grid.lat), len(gm.model.grid.lon)
    lat, lon = site_set(H, W, 40, seed=1)
    sites = ([f"s{i}" for i in range(lat.size)], lat, lon)
    n_steps = 2 if schedule is None else 5
    sel = [names[0], names[2], names[-2]]
    one, _ = gm.predict_sites(T0, n_steps, sites, channels=sel)
    fc = gm.forecast(T0, n_steps)
    fields = np.asarray(fc.values, dtype=np.float32)[-(n_steps + 1):]
    idx, w = R.stencil(lat, lon, H, W)
    cidx = [list(np.asarray(fc.coords["channel"])).index(c) for c in sel]
    for n in range(n_steps + 1):
        want = R.sample(fields[n][None], idx, w, cidx)                     # (1, S, n_sites)
        assert one.values.values[n].tobytes() == np.ascontiguousarray(want.transpose(0, 2, 1)).tobytes(), n
    assert one.stats is None and one.prob is None
    M, seed, thr = 4, 7, float(np.median(fields[0, cidx[0]]))
    ens, _ = gm.predict_sites(T0, n_steps, sites, members=M, seed=seed, method="nearest", channels=sel,
                              quantiles=[0.5], events={sel[0]: thr})
    idx, w = R.stencil(lat, lon, H, W, "nearest")
    for n, x in enumerate(_runner_members(gm, T0, n_steps, M, seed)):
        v = R.sample(x, idx, w, [names.index(c) for c in sel])              # (M, S, n_sites)
        assert ens.values.values[n].tobytes() == np.ascontiguousarray(v.transpose(0, 2, 1)).tobytes(), n
        s, p = ens_stats_ref.ensemble_stats(v[:, :, None], [0, 1, 2], [0.5], [(0, thr)])
        assert ens.stats.values[n].tobytes() == np.ascontiguousarray(s[:, :, 0].transpose(0, 2, 1)).tobytes()
        assert ens.prob.values[n].tobytes() == p[:, 0].tobytes()
    u = ens.point("s3", sel[1])
    assert u.values.shape == (n_steps + 1, M)
    gm.release_model()


@pytest.mark.parametrize("name, schedule", CASES)
def test_score_sites_end_to_end(name, schedule):
    from skyrim_b200 import sites as St
    from skyrim_b200 import xr_shim as xr
    gm = _model(name, schedule).model
    names = list(gm.out_channel_names)
    H, W = len(gm.model.grid.lat), len(gm.model.grid.lon)
    lat, lon = site_set(H, W, 60, seed=2)
    n_sites = lat.size
    sel = [c for c in names if c not in gm.forcing_channels][:3]
    n_steps, M, seed = (2 if schedule is None else 5), 3, 5
    starts = [T0, T0 + 2 * STEP]
    times = sorted({t + k * STEP for t in starts for k in range(n_steps + 1)})[:-1]     # the last valid time is absent
    idx, w = R.stencil(lat, lon, H, W)
    rng = np.random.default_rng(0)
    vals = np.stack([R.sample(gm.data_source[t].sel(channel=sel).values[None], idx, w, range(len(sel)))[0].T
                     for t in times])                                                # (time, site, channel)
    vals[rng.random(vals.shape) < 0.25] = np.nan                                     # holes
    obs = xr.DataArray(vals, dims=["time", "site", "channel"],
                       coords=dict(time=np.array([np.datetime64(t, "s") for t in times]),
                                   site=np.array([f"s{i}" for i in range(n_sites)]), channel=np.array(sel),
                                   lat=("site", lat), lon=("site", lon)))
    res, _ = gm.score_sites(starts, n_steps, obs, members=M, seed=seed)
    at = {np.datetime64(t, "s"): i for i, t in enumerate(times)}
    sums, acc, cidx = [], 0.0, [names.index(c) for c in sel]
    for d, t0 in enumerate(starts):
        per_lead, accs = [], []
        for k, x in enumerate(_runner_members(gm, t0, n_steps, M, seed + d)):
            v = R.sample(x, idx, w, cidx)
            i = at.get(np.datetime64(t0 + k * STEP, "s"))
            y = np.full((len(sel), n_sites), np.nan, np.float32) if i is None else vals[i].T
            per_lead.append(R.site_sums(v, y))
            accs.append(R.site_terms(v, y))
        sums.append(per_lead)
        acc = acc + np.stack(accs)
    want_sums = np.array([[s for s, _ in row] for row in sums])
    mag = np.array([[m for _, m in row] for row in sums]).sum(0)
    want_card = St.site_metrics(want_sums.sum(0), M)
    got_card = np.moveaxis(res.card.values, 1, -1)
    assert np.allclose(got_card, want_card, rtol=1e-10, atol=1e-10 * mag[..., :1].max(), equal_nan=True)
    want_sites = np.transpose(St.site_metrics(acc, M), (0, 3, 2, 1))
    assert np.allclose(res.sites.values, want_sites, rtol=1e-10, atol=1e-9, equal_nan=True)
    assert (res.count.values == np.swapaxes(acc[..., 0], 1, 2)).all()
    assert (res.count.values[-1].sum() < res.count.values[0].sum())                  # the absent time counts as missing
    gm.release_model()


def test_cli_writes_readable_site_files(tmp_path):
    from click.testing import CliRunner
    from skyrim_b200 import forecast as F
    from skyrim_b200 import xr_shim as xr
    csv = tmp_path / "sites.csv"
    csv.write_text("name,lat,lon\nparis,48.85,2.35\noslo,59.91,10.75\nquito,-0.18,-78.47\n")
    out = str(tmp_path / "out")
    r = CliRunner().invoke(F.main, ["-m", "pangu", "--grid", "41x96", "-d", "20240507", "-l", "12", "-o", out,
                                    "--sites", str(csv), "--members", "3", "--quantiles", "0.5", "--exceed", "t2m:280"])
    assert r.exit_code == 0, r.output
    paths = [ln for ln in r.output.splitlines() if ln.endswith(".nc")]
    assert len(paths) == 3
    v = xr.open_dataarray([p for p in paths if "-stats" not in p and "-prob" not in p][0])
    assert tuple(v.dims) == ("time", "member", "site", "channel") and v.values.shape[:3] == (3, 3, 3)
    assert np.asarray(v.coords["lat"]).tolist() == [48.85, 59.91, -0.18] and list(v.coords["site"])[2] == "quito"
    obs = xr.DataArray(np.full((3, 3, 1), 280.0, np.float32), dims=["time", "site", "channel"],
                       coords=dict(time=np.array(["2024-05-07T00", "2024-05-07T06", "2024-05-07T12"], dtype="datetime64[s]"),
                                   site=np.array(["paris", "oslo", "quito"]), channel=np.array(["t2m"]),
                                   lat=("site", np.array([48.85, 59.91, -0.18])), lon=("site", np.array([2.35, 10.75, -78.47]))))
    obs.to_netcdf(tmp_path / "obs.nc")
    r = CliRunner().invoke(F.main, ["-m", "pangu", "--grid", "41x96", "-d", "20240507", "-l", "12", "-o", out,
                                    "--sites", str(csv), "--observations", str(tmp_path / "obs.nc"), "--site_method",
                                    "nearest"])
    assert r.exit_code == 0, r.output
    paths = [ln for ln in r.output.splitlines() if ln.endswith(".nc")]
    assert len(paths) == 4
    card = xr.open_dataarray([p for p in paths if "-obs1__" in p][0])
    assert tuple(card.dims) == ("lead_time", "metric", "channel") and card.values.shape == (3, 6, 1)
    count = xr.open_dataarray([p for p in paths if "-count" in p][0])
    assert (count.values == 1).all()
