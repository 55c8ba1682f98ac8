"""sky_forecast_rank_histogram and sky_forecast_score_maps on the device against the fp64 reference (ranks, histograms,
forced ties, map accumulators), their properties (NaN rule, reproducibility, independence of the request, GraphCast's new
slice, a flat histogram for a reliable ensemble), one full-size call, and GlobalModel.score_period end to end."""
import datetime
import os
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import verify_period_ref as ref  # noqa: E402
from skyrim_b200 import scores as S  # noqa: E402

T0 = datetime.datetime(2024, 5, 7)
STEP = datetime.timedelta(hours=6)
REGIONS = {"global": (-90, 90), "tropics": (-20, 20), "north": (20, 90), "south": (-90, -24.75)}


@pytest.fixture(autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def dev(a):
    return a if torch.is_tensor(a) else torch.as_tensor(np.ascontiguousarray(a)).cuda()


def hist(x, truth, w, seed=0, date=0, lead=0, channels=None, channel_offset=0):
    from skyrim_b200.engine import forecast_rank_histogram
    out = forecast_rank_histogram(dev(x), dev(truth), dev(np.asarray(w, np.float64)), seed, date, lead, channels,
                                  channel_offset)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def maps_after(x, truth, calls=1, channels=None, channel_offset=0):
    from skyrim_b200.engine import score_maps_accumulate
    xd, yd = dev(x), dev(truth)
    H, W = yd.shape[-2:]
    m = torch.zeros((yd.shape[0], 5, H, W), dtype=torch.float64, device="cuda")
    for _ in range(calls):
        score_maps_accumulate(xd, yd, m, channels, channel_offset)
    torch.cuda.synchronize()
    return m.cpu().numpy()


def fields(M, C=5, H=41, W=96, seed=0, quantise=False):
    from skyrim_b200.timeloop import equiangular_grid
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((M, C, H, W)) * 3 + 280).astype(np.float32)
    y = (rng.standard_normal((3, H, W)) * 3 + 280).astype(np.float32)
    if quantise:
        x, y = np.round(x / 2) * 2, np.round(y / 2) * 2
    return x, y, np.asarray(equiangular_grid(H, W).lat)


@pytest.mark.parametrize("M", [1, 2, 3, 8, 17, 33, 64])
def test_kernels_match_the_reference(M):
    x, y, lat = fields(M, seed=M)
    x[M // 2, 1, :, ::3] = y[0, :, ::3]            # the truth equal to a member at every third point
    _, w = S.region_weights(lat, REGIONS)
    ch = [3, 1, 4]
    got = hist(x, y, w, 9, 2, 5, ch)
    want, wsum = ref.rank_histogram(x, y, w, ch, 9, 2, 5)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
    np.testing.assert_allclose(got.sum(-1), np.broadcast_to(wsum[:, None], got.shape[:2]), rtol=0, atol=1e-12)
    # the ranks themselves: each point alone in a one-point-wide "grid" row would cost a launch per point, so compare
    # the histogram of every single row instead (a row region holds one latitude)
    r = ref.ranks(x, y, ch, 9, 2, 5)
    for i in (3, 20, 37):
        wr = np.zeros((1, len(lat)))
        wr[0, i] = 1.0
        g = hist(x, y, wr, 9, 2, 5, ch)[0] * x.shape[-1]
        cnt = np.stack([(r[:, i] == k).sum(-1) for k in range(M + 1)], -1)
        np.testing.assert_array_equal(np.round(g).astype(int), cnt)
    t, mag = ref.map_terms(x, y, ch)
    m = maps_after(x, y, 3, ch)
    assert (np.abs(m - 3 * t) <= 1e-12 * 3 * mag + 1e-300).all()


def test_forced_ties_quantised_fields():
    for M in (1, 4, 16):
        x, y, lat = fields(M, seed=20 + M, quantise=True)
        _, w = S.region_weights(lat, REGIONS)
        got = hist(x, y, w, 1, 0, 0, [0, 2, 4])
        want, _ = ref.rank_histogram(x, y, w, [0, 2, 4], 1, 0, 0)
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)


def test_nan_rule():
    x, y, lat = fields(4, seed=3)
    _, w = S.region_weights(lat, REGIONS)
    x[2, 1, 5, 7] = np.nan                          # row 5 is at 67.5N: global and north only
    y[2, 30, 2] = np.nan                            # truth of selected channel 2, row 30 (-45): global and south
    h = hist(x, y, w, channels=[0, 1, 2])
    assert np.isnan(h[0, 1]).all() and np.isnan(h[2, 1]).all() and np.isfinite(h[1, 1]).all() and np.isfinite(h[3, 1]).all()
    assert np.isnan(h[0, 2]).all() and np.isnan(h[3, 2]).all() and np.isfinite(h[1:3, 2]).all()
    assert np.isfinite(h[:, 0]).all()
    m = maps_after(x, y, 1, [0, 1, 2])
    nan = np.isnan(m)
    assert nan[1, :, 5, 7].all() and nan[2, :, 30, 2].all() and nan.sum() == 10


def test_reproducible_and_independent_of_the_request():
    x, y, lat = fields(8, seed=4, quantise=True)
    _, w = S.region_weights(lat, REGIONS)
    a, b = hist(x, y, w, 3, 1, 2, [0, 1, 2]), hist(x, y, w, 3, 1, 2, [0, 1, 2])
    assert a.tobytes() == b.tobytes()
    sub = hist(x, y[1:2], w[[2, 0]], 3, 1, 2, [1])          # a channel subset and a region subset
    assert sub[0, 0].tobytes() == a[2, 1].tobytes() and sub[1, 0].tobytes() == a[0, 1].tobytes()
    m1, m2 = maps_after(x, y, 2, [0, 1, 2]), maps_after(x, y, 2, [0, 1, 2])
    assert m1.tobytes() == m2.tobytes()
    assert maps_after(x, y[2:], 2, [2])[0].tobytes() == m1[2].tobytes()


def test_channel_offset_reaches_a_graphcast_new_slice():
    M, Cn, off = 3, 10, 5
    x, y, lat = fields(M, C=Cn, seed=6, quantise=True)
    _, w = S.region_weights(lat, REGIONS)
    a = hist(x, y, w, 2, 0, 1, [0, 3, 4], channel_offset=off)
    want, _ = ref.rank_histogram(x[:, off:], y, w, [0, 3, 4], 2, 0, 1)    # channel words count from the offset
    np.testing.assert_allclose(a, want, rtol=0, atol=1e-12)
    m = maps_after(x, y, 1, [0, 3, 4], channel_offset=off)
    t, mag = ref.map_terms(x[:, off:], y, [0, 3, 4])
    assert (np.abs(m - t) <= 1e-12 * mag + 1e-300).all()


def test_reliable_ensemble_gives_a_flat_histogram():
    M, H, W = 9, 181, 360
    rng = np.random.default_rng(7)
    x = rng.standard_normal((M + 1, 1, H, W)).astype(np.float32)    # the truth is one more draw of the same law
    y = x[M:, 0]
    from skyrim_b200.timeloop import equiangular_grid
    _, w = S.region_weights(np.asarray(equiangular_grid(H, W).lat))
    h = hist(x[:M], y, w)[0, 0]
    n_eff = 1.0 / (np.sum(np.repeat(w[0] / W, W) ** 2))             # effective number of weighted points
    sd = np.sqrt((1 / (M + 1)) * (1 - 1 / (M + 1)) / n_eff)
    assert (np.abs(h - 1 / (M + 1)) < 5 * sd).all(), (h, sd)


def test_full_size():
    M, C, H, W = 4, 2, 721, 1440
    rng = np.random.default_rng(8)
    x = rng.standard_normal((M, C, H, W)).astype(np.float32)
    y = rng.standard_normal((C, H, W)).astype(np.float32)
    x[1, 0, ::7] = y[0, ::7]
    from skyrim_b200.timeloop import equiangular_grid
    _, w = S.region_weights(np.asarray(equiangular_grid(H, W).lat), REGIONS)
    got = hist(x, y, w, 5, 3, 2)
    want, _ = ref.rank_histogram(x, y, w, [0, 1], 5, 3, 2)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
    t, mag = ref.map_terms(x, y, [0, 1])
    assert (np.abs(maps_after(x, y, 1) - t) <= 1e-12 * mag + 1e-300).all()


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


def _runner_members(sk, t0, n_steps, M, seed, hierarchical=False):
    """the members an identically seeded runner holds at every lead (host (M, C, H, W) per lead), through the same
    schedule as the model"""
    import functools
    from skyrim_b200.ensemble import EnsembleRunner, HierarchicalEnsembleRunner
    gm = sk.model
    base, sigma, off = gm._ensemble_initial_state(t0)
    make = EnsembleRunner
    if hierarchical:
        make = functools.partial(HierarchicalEnsembleRunner, engine_24=gm.model.engine_24, every_slice=True)
    run = make(gm.model.engine, base, sigma, members_per_gpu=M, perturbation="spherical_grf" if M > 1 else "none",
               grf=dict(lmax=min(180, (len(gm.model.grid.lat) - 1) // 2)), seed=seed)
    return [m[:, off:].cpu().numpy() for _, m in run._walk(n_steps)], off


@pytest.mark.parametrize("name, schedule", [("pangu", None), ("pangu", "hierarchical"), ("fourcastnet_v2", None),
                                            ("graphcast", None)])
def test_score_period_end_to_end(name, schedule):
    sk = _model(name, schedule)
    gm = sk.model
    names = list(gm.out_channel_names)
    M, seed, n_steps = 4, 11, 2 if schedule is None else 5
    starts = [T0, T0 + 2 * STEP, T0 + 4 * STEP]
    mch = [names[0], names[3]]
    res, _ = gm.score_period(starts, n_steps, members=M, seed=seed, regions=REGIONS, map_leads=[6, 6 * n_steps],
                             map_channels=mch)
    sel = list(res.card.coords["channel"])
    idx = [names.index(c) for c in sel]
    midx = [names.index(c) for c in mch]
    _, w = S.region_weights(np.asarray(gm.model.grid.lat), REGIONS)
    H, W = len(gm.model.grid.lat), len(gm.model.grid.lon)
    acc = np.zeros((2, len(mch), 5, H, W))
    want_h, sums = 0.0, []
    for d, t0 in enumerate(starts):
        card, _ = gm.score(t0, n_steps, members=M, seed=seed + d, regions=REGIONS)
        assert res.cards.values[d].tobytes() == card.values.tobytes(), d       # bitwise the one-date card
        sums.append(_sums_of(gm, t0, n_steps, M, seed + d))
        members, _ = _runner_members(sk, t0, n_steps, M, seed + d, schedule == "hierarchical")
        hd = []
        for n, x in enumerate(members):
            src = gm.data_source[t0 + n * STEP]
            hd.append(ref.rank_histogram(x, src.sel(channel=sel).values, w, idx, seed, d, n)[0])
            if n in (1, n_steps):
                acc[int(n == n_steps)] += ref.map_terms(x, src.sel(channel=mch).values, midx)[0]
        want_h = want_h + np.stack(hd)
    np.testing.assert_allclose(res.rank_histogram.values, want_h / len(starts), rtol=0, atol=1e-12)
    np.testing.assert_array_equal(np.moveaxis(res.card.values, 1, -1), S.period_metrics(np.stack(sums), M))
    want_maps = np.swapaxes(S.map_metrics(acc, len(starts), M), 1, 2)
    scale = np.nanmax(np.abs(want_maps), axis=(-2, -1), keepdims=True)
    assert (np.abs(res.maps.values - want_maps) <= 1e-5 * scale).all()
    gm.release_model()


def _sums_of(gm, t0, n_steps, M, seed):
    names = list(gm.out_channel_names)
    times = [t0 + n * gm.time_step for n in range(n_steps + 1)]
    _, sel, _, rw, truth_at, clim = gm._score_setup(M, None, [], REGIONS, None, None, times, False, {})
    runner, off = gm._score_runner(t0, M, "spherical_grf", 0.05, seed, None)
    _, sums = runner.iter_scores(n_steps, lambda n: truth_at(times[n]), clim, [names.index(c) for c in sel], rw, off)
    return sums.numpy()


def test_one_member_at_lead_zero_against_its_own_initial_condition():
    sk = _model("pangu")
    gm = sk.model
    starts = [T0, T0 + STEP]
    res, _ = gm.score_period(starts, 0, members=1, seed=4, map_leads=[0], map_channels=["z500", "t2m"])
    for m in ("bias", "rmse", "crps"):
        assert (res.maps.sel(metric=m).values == 0).all(), m
    idx = list(range(len(res.card.coords["channel"])))
    _, w = S.region_weights(np.asarray(gm.model.grid.lat))
    want = 0.0
    for d, t0 in enumerate(starts):
        ic = gm.data_source[t0].values
        want = want + ref.rank_histogram(ic[None], ic, w, idx, 4, d, 0)[0]
    np.testing.assert_allclose(res.rank_histogram.values[0], want / 2, rtol=0, atol=1e-12)
    assert (res.rank_histogram.values[0] > 0.3).all()            # ties spread over both bins, not all in bin 0
    gm.release_model()


def test_cli_grid_score_period(tmp_path):
    from click.testing import CliRunner
    from skyrim_b200 import forecast as F
    from skyrim_b200 import xr_shim as xr
    r = CliRunner().invoke(F.main, ["-m", "pangu", "--grid", "41x96", "-d", "20240507", "-l", "12", "-o", str(tmp_path),
                                    "--score", "--until", "20240508", "--members", "2", "--map_channels", "z500,t850",
                                    "--map_leads", "12"])
    assert r.exit_code == 0, r.output
    paths = [ln for ln in r.output.splitlines() if ln.endswith(".nc")]
    assert len(paths) == 4
    maps = xr.open_dataarray([p for p in paths if "-maps" in p][0])
    assert maps.values.shape == (1, 4, 2, 41, 96) and np.isfinite(maps.values).all()
    cards = xr.open_dataarray([p for p in paths if "-cards" in p][0])
    assert cards.values.shape == (2, 3, 7, 1, 69)
