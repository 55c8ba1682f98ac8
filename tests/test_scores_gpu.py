"""sky_forecast_scores on the device: the sums against the fp64 oracle, reproducibility, independence of the request, the
NaN rule, GraphCast's new slice, the shared sort network, and GlobalModel.score end to end for the three models."""
import datetime

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import ens_stats_ref, scores_ref  # noqa: E402
from skyrim_b200 import scores as S  # noqa: E402

T0 = datetime.datetime(2024, 5, 7)
STEP = datetime.timedelta(hours=6)
REGIONS = {"global": (-90, 90), "tropics": (-20, 20), "north": (20, 90), "south": (-90, -24.75)}


@pytest.fixture(autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def sums(x, truth, w, channels=None, clim=None, channel_offset=0):
    from skyrim_b200.engine import forecast_scores
    dev = lambda a: None if a is None else torch.as_tensor(np.ascontiguousarray(a)).cuda()  # noqa: E731
    x = x if torch.is_tensor(x) else dev(x)
    out = forecast_scores(x, dev(truth), dev(np.asarray(w, np.float64)), channels, dev(clim), channel_offset)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def assert_sums(got, want, mag, rel=1e-12):
    """each sum within rel x the oracle's sum of w |term| (NaN where the oracle's is NaN)"""
    assert got.shape == want.shape
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    err = np.abs(got[ok] - want[ok])
    tol = rel * mag[ok]
    assert (err <= tol).all(), f"worst {np.max(err / np.maximum(tol, 1e-300)):.3g} of the bound"


def _fields(M, shape, kind, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        x = (rng.standard_normal((M,) + shape) * 10).astype(np.float32)
        y = (rng.standard_normal(shape) * 10).astype(np.float32)
    else:   # de-normalised geopotential-like fields: 5e4 +- 0.5
        x = (5e4 + rng.uniform(-0.5, 0.5, (M,) + shape)).astype(np.float32)
        y = (5e4 + rng.uniform(-0.5, 0.5, shape)).astype(np.float32)
    k = (y + rng.uniform(-0.3, 0.3, shape)).astype(np.float32)
    return x, y, k


@pytest.mark.parametrize("kind", ["random", "large_mean"])
@pytest.mark.parametrize("M", [1, 2, 3, 8, 17, 33, 64])
def test_kernel_matches_oracle(M, kind):
    from skyrim_b200.timeloop import equiangular_grid
    x, y, k = _fields(M, (6, 41, 96), kind, M)
    sel = [5, 0, 3]
    _, w = S.region_weights(equiangular_grid(41, 96).lat, REGIONS)
    for clim in (k[sel], None):
        got = sums(x, y[sel], w, sel, clim)
        want, mag = scores_ref.score_sums(x, y[sel], w, sel, clim)
        assert_sums(got, want, mag)
        if clim is None:
            assert np.isnan(got[..., 6:]).all() and np.isfinite(got[..., :6]).all()


def test_full_size_channel_subset():
    from skyrim_b200.timeloop import equiangular_grid
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn((4, 69, 721, 1440), device="cuda", generator=g) * 3 + 7
    sel = [68, 2]
    y = x[0, sel].cpu().numpy() + np.float32(0.5)
    k = np.full_like(y, 7.0)
    _, w = S.region_weights(equiangular_grid(721, 1440).lat, {"global": (-90, 90), "tropics": (-20, 20)})
    got = sums(x, y, w, sel, k)
    want, mag = scores_ref.score_sums(x[:, sel].cpu().numpy(), y, w, [0, 1], k)
    assert_sums(got, want, mag)
    assert got.shape == (2, 2, 9)
    np.testing.assert_allclose(got[:, :, 0], 1440.0, rtol=1e-13)   # the row weights sum to 1 per region


def test_reproducible_and_independent_of_the_request():
    from skyrim_b200.timeloop import equiangular_grid
    x, y, k = _fields(9, (7, 41, 96), "random", 3)
    names, w = S.region_weights(equiangular_grid(41, 96).lat, REGIONS)
    all_ = sums(x, y, w, None, k)
    np.testing.assert_array_equal(sums(x, y, w, None, k), all_)
    for c in (0, 4, 6):
        for r in range(len(names)):
            one = sums(x, y[[c]], w[[r]], [c], k[[c]])
            np.testing.assert_array_equal(one[0, 0], all_[r, c])


def test_nan_rule():
    from skyrim_b200.timeloop import equiangular_grid
    x, y, k = _fields(5, (4, 41, 96), "random", 4)
    names, w = S.region_weights(equiangular_grid(41, 96).lat, REGIONS)
    clean = sums(x, y, w, None, k)
    # NaN on a pole row (weight 0 in every region): nothing changes
    for arr, idx in ((x, (2, 1, 0, 7)), (y, (1, 40, 3)), (k, (3, 0, 50))):
        a = arr.copy()
        a[idx] = np.nan
        got = sums(a if arr is x else x, a if arr is y else y, w, None, a if arr is k else k)
        np.testing.assert_array_equal(got, clean)
    # NaN at a weighted point (row 10, 45 N: "global" and "north"): only that channel's scores in those regions
    for arr, idx, c in ((x, (4, 2, 10, 20), 2), (y, (1, 10, 5), 1), (k, (3, 10, 90), 3)):
        a = arr.copy()
        a[idx] = np.nan
        got = sums(a if arr is x else x, a if arr is y else y, w, None, a if arr is k else k)
        hit = [names.index("global"), names.index("north")]
        assert np.isnan(got[hit, c, 1:]).all() and (got[hit, c, 0] == clean[hit, c, 0]).all()
        got[hit, c] = clean[hit, c]
        np.testing.assert_array_equal(got, clean)
        m = S.metrics_from_sums(sums(a if arr is x else x, a if arr is y else y, w, None, a if arr is k else k), 5)
        assert np.isnan(m[hit, c]).all() and np.isfinite(m[:, [i for i in range(4) if i != c]]).all()


def test_channel_offset_reaches_a_graphcast_new_slice():
    from skyrim_b200.timeloop import equiangular_grid
    rng = np.random.default_rng(6)
    x = torch.from_numpy(rng.standard_normal((3, 166, 41, 96)).astype(np.float32)).cuda()
    sel = [0, 40, 81]
    y = rng.standard_normal((3, 41, 96)).astype(np.float32)
    _, w = S.region_weights(equiangular_grid(41, 96).lat)
    want = sums(x[:, 83:].contiguous(), y, w, sel)
    np.testing.assert_array_equal(sums(x, y, w, sel, channel_offset=83), want)
    np.testing.assert_array_equal(sums(x[:, 83:], y, w, sel), want)


@pytest.mark.parametrize("M", [2, 5, 8, 13, 16, 31, 32, 47, 64])
def test_shared_sort_network_keeps_ensemble_quantiles_exact(M):
    """a quantile at q = i / (M - 1) is the i-th sorted member bit for bit: the sort network is unchanged"""
    from skyrim_b200.engine import ensemble_statistics
    rng = np.random.default_rng(M)
    x = (rng.standard_normal((M, 3, 41, 96)) * 4).astype(np.float32)
    x[:, 1] = np.round(x[:, 1])          # ties
    qs = sorted({0, 1, M // 3, M // 2, M - 1})
    s, _ = ensemble_statistics(torch.from_numpy(x).cuda(), None, [i / (M - 1) for i in qs])
    s = s.cpu().numpy()
    srt = np.sort(x, axis=0)
    for j, i in enumerate(qs):
        np.testing.assert_array_equal(s[2 + j], srt[i])
    ws, _ = ens_stats_ref.ensemble_stats(x, range(3), [i / (M - 1) for i in qs])
    np.testing.assert_array_equal(s[2:], ws[2:])


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


def climatology(channels, nlat, nlon):
    from skyrim_b200 import xr_shim as xr
    from skyrim_b200.timeloop import equiangular_grid
    from skyrim_b200.weights import channel_stats
    g = equiangular_grid(nlat, nlon)
    mu = channel_stats(channels)[0]
    return xr.DataArray(np.broadcast_to(mu[:, None, None], (len(channels), nlat, nlon)).astype(np.float32),
                        dims=["channel", "lat", "lon"], coords=dict(channel=np.array(channels), lat=np.array(g.lat),
                                                                    lon=np.array(g.lon)))


def assert_card(card, members_per_lead, truths, clim, regions, sel_idx, lat):
    """the scorecard against the oracle's metrics of the given members (per lead) and truths"""
    _, w = S.region_weights(lat, regions)
    for n, (x, y) in enumerate(zip(members_per_lead, truths)):
        want = scores_ref.metrics(x, y, w, sel_idx, clim)                    # (region, channel, metric)
        got = np.moveaxis(card.values[n], 0, -1)
        np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
        ok = ~np.isnan(want)
        scale = (np.abs(want) + want[..., 1:2])[ok]                         # + rmse: bias and crps may be near 0
        assert (np.abs(got[ok] - want[ok]) <= 1e-9 * scale).all(), n


@pytest.mark.parametrize("model", ["pangu", "fourcastnet_v2", "graphcast"])
def test_one_member_scores_the_forecast(model, tmp_path):
    from skyrim_b200 import xr_shim as xr
    from skyrim_b200.config import graphcast_small, pangu_small, sfno_small
    from skyrim_b200.core import Skyrim
    cfg, (nlat, nlon) = {"pangu": (pangu_small(41, 96), (41, 96)), "fourcastnet_v2": (sfno_small(49, 96), (49, 96)),
                         "graphcast": (graphcast_small(41, 96, 2, 512, 2), (41, 96))}[model]
    sk = Skyrim(model, cfg=cfg, ic_source=TimeSource(_channels(model), nlat, nlon))
    names = list(sk.model.out_channel_names)
    sel = [c for c in names if c != "tp06"]
    clim = climatology(sel, nlat, nlon)
    regions = {"global": (-90, 90), "tropics": (-20, 20)}
    card, paths = sk.score("20240507", "0000", lead_time=12, climatology=clim, regions=regions, save=True,
                           save_config=dict(output_dir=str(tmp_path)))
    assert tuple(card.dims) == ("lead_time", "metric", "region", "channel") and list(card.coords["channel"]) == sel
    assert list(card.coords["lead_time"]) == [0.0, 6.0, 12.0] and card.attrs["members"] == 1
    lead0 = card.values[0]
    for m in ("rmse", "bias", "crps"):
        assert (lead0[list(S.METRICS).index(m)] == 0).all(), m
    assert (lead0[list(S.METRICS).index("acc")] == 1).all()
    fc = sk.forecast(T0, n_steps=2, channels=sel).values                      # (3, S, H, W) host output
    src = sk.model.data_source
    truths = [src[T0 + n * STEP].sel(channel=sel).values for n in range(3)]
    assert_card(card, [fc[n][None] for n in range(3)], truths, clim.values, regions, range(len(sel)),
                sk.model.model.grid.lat)
    back = xr.open_dataarray(paths[0])
    np.testing.assert_array_equal(back.values, card.values)
    assert back.attrs["model"] == model
    sk.model.release_model()


def _channels(model):
    from skyrim_b200.config import FCNV2_CHANNELS, GRAPHCAST_CHANNELS, PANGU_CHANNELS
    return {"pangu": PANGU_CHANNELS, "fourcastnet_v2": FCNV2_CHANNELS, "graphcast": GRAPHCAST_CHANNELS}[model]


def test_ensemble_scores_the_runner_members():
    from skyrim_b200.config import PANGU_CHANNELS, pangu_small
    from skyrim_b200.core import Skyrim
    from skyrim_b200.ensemble import EnsembleRunner
    from skyrim_b200.weights import channel_stats
    src = TimeSource(PANGU_CHANNELS, 41, 96)
    sk = Skyrim("pangu", cfg=pangu_small(41, 96), ic_source=src)
    sel = ["z500", "t850", "t2m", "msl"]
    clim = climatology(sel, 41, 96)
    card, _ = sk.score("20240507", "0000", lead_time=12, members=4, climatology=clim, channels=sel, regions=REGIONS)
    run = EnsembleRunner(sk.model.model.engine, src[T0].values, channel_stats(PANGU_CHANNELS)[1], members_per_gpu=4,
                         perturbation="spherical_grf", grf=dict(lmax=20))
    members = [run.x.cpu().numpy()] + [run.step().cpu().numpy() for _ in range(2)]
    assert list(card.coords["channel"]) == ["z500", "t850", "msl", "t2m"]   # the model's channel order
    idx = [PANGU_CHANNELS.index(c) for c in card.coords["channel"]]
    truths = [src[T0 + n * STEP].values[idx] for n in range(3)]
    assert_card(card, members, truths, clim.sel(channel=list(card.coords["channel"])).values, REGIONS, idx,
                sk.model.model.grid.lat)
    m = card.sel(metric="spread").values
    assert np.isfinite(m).all() and (m[1:] > 0).all() and np.isfinite(card.sel(metric="ssr").values).all()
    sk.model.release_model()


def test_pangu_hierarchical_scores_its_slices():
    from skyrim_b200.config import PANGU_CHANNELS, pangu_small
    from skyrim_b200.core import Skyrim
    src = TimeSource(PANGU_CHANNELS, 41, 96)
    sk = Skyrim("pangu", cfg=pangu_small(41, 96), schedule="hierarchical", ic_source=src)
    card, _ = sk.score("20240507", "0000", lead_time=36)                      # 6 slices: the 24-h operator at slice 4
    fc = sk.forecast(T0, n_steps=6).values
    truths = [src[T0 + n * STEP].values for n in range(7)]
    assert_card(card, [fc[n][None] for n in range(7)], truths, None, S.DEFAULT_REGIONS, range(69), sk.model.model.grid.lat)
    sk.model.release_model()


def test_cli_grid_score(tmp_path):
    from click.testing import CliRunner
    from skyrim_b200 import forecast as F
    from skyrim_b200 import xr_shim as xr
    r = CliRunner().invoke(F.main, ["-m", "pangu", "--grid", "41x96", "-d", "20240507", "-l", "12", "-o", str(tmp_path),
                                    "--score", "--members", "2"])
    assert r.exit_code == 0, r.output
    paths = [ln for ln in r.output.splitlines() if ln.endswith(".nc")]
    card = xr.open_dataarray(paths[0])
    assert card.values.shape == (3, 7, 1, 69) and card.attrs["members"] == 2
