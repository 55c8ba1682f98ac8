"""Verification over many start dates without a device: the rank-histogram and score-map reference, the period metrics,
the C-ABI's new exports and refusals, and GlobalModel.score_period's host logic on a CPU fake of the member runner (the
date range, the seeds, the refusals, the files and the forecast CLI options)."""
import ctypes as C
import datetime
import os
import re
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import verify_period_ref as ref  # noqa: E402
from oracle import scores_ref  # noqa: E402
from skyrim_b200 import scores as S  # noqa: E402
from skyrim_b200 import xr_shim as xr  # noqa: E402
from skyrim_b200.core.models.base import GlobalModel  # noqa: E402
from skyrim_b200.timeloop import equiangular_grid  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CH = ["u10m", "v10m", "t2m", "msl"]
T0 = datetime.datetime(2024, 5, 7)
STEP = datetime.timedelta(hours=6)
G = equiangular_grid(19, 36)


# ---- the reference ----------------------------------------------------------------------------------------------------------
def test_rank_histogram_without_ties_is_weighted_searchsorted_counts():
    rng = np.random.default_rng(0)
    M = 5
    x, y = rng.standard_normal((M, 3, 19, 36)), rng.standard_normal((2, 19, 36))
    _, w = S.region_weights(G.lat, {"g": (-90, 90), "t": (-20, 20)})
    h, wsum = ref.rank_histogram(x, y, w, [2, 0], 7, 1, 3)
    for r in range(2):
        for s, c in enumerate([2, 0]):
            xs = np.sort(x[:, c].astype(np.float32), axis=0)
            rk = np.array([[np.searchsorted(xs[:, i, j], np.float32(y[s, i, j])) for j in range(36)] for i in range(19)])
            want = [(w[r][:, None] * (rk == k)).sum() / 36 for k in range(M + 1)]
            np.testing.assert_allclose(h[r, s], want, rtol=1e-13, atol=1e-16)
    np.testing.assert_allclose(h.sum(-1), np.broadcast_to(wsum[:, None], h.shape[:2]), rtol=1e-13)
    np.testing.assert_allclose(wsum, 1.0, rtol=1e-13)


def test_all_members_tied_to_the_truth_give_the_philox_ranks():
    M, y = 3, np.full((1, 19, 36), 2.5)
    x = np.full((M, 2, 19, 36), 2.5)
    r = ref.ranks(x, y, [1], 11, 2, 4)
    u = ref.tie_words(11, 2, 4, [1], 19, 36)
    np.testing.assert_array_equal(r, (u * 4) >> 32)
    assert set(np.unique(r)) == {0, 1, 2, 3}               # all four bins are reached
    assert not np.array_equal(r, ref.ranks(x, y, [1], 11, 3, 4))   # the date index changes the draws
    # one member with the truth below / above it
    assert (ref.ranks(x[:1] + 1, y, [1], 0, 0, 0) == 0).all() and (ref.ranks(x[:1] - 1, y, [1], 0, 0, 0) == 1).all()


def test_every_histogram_sums_to_one():
    rng = np.random.default_rng(1)
    for M in (1, 2, 8):
        x = np.round(rng.standard_normal((M, 2, 19, 36)))        # quantised: many ties
        y = np.round(rng.standard_normal((2, 19, 36)))
        _, w = S.region_weights(G.lat, {"g": (-90, 90), "n": (20, 90), "s": (-90, -30)})
        h, _ = ref.rank_histogram(x, y, w, [0, 1], 3, 0, 1)
        np.testing.assert_allclose(h.sum(-1), 1.0, rtol=1e-13)


def test_map_terms_sum_to_the_score_sums():
    rng = np.random.default_rng(2)
    x, y = rng.standard_normal((4, 3, 19, 36)), rng.standard_normal((2, 19, 36))
    t, _ = ref.map_terms(x, y, [2, 1])
    _, w = S.region_weights(G.lat)
    sums, _ = scores_ref.score_sums(x, y, w, [2, 1])
    np.testing.assert_allclose((t * w[0][None, None, :, None]).sum((2, 3)), sums[0][:, 1:6], rtol=1e-12)


# ---- period metrics ---------------------------------------------------------------------------------------------------------
def _sums(rng, D, M):
    out = []
    for d in range(D):
        x = rng.standard_normal((M, 3, 19, 36)) * (1 + d) + d
        y, k = rng.standard_normal((3, 19, 36)), rng.standard_normal((3, 19, 36)) * 0.1
        out.append(scores_ref.score_sums(x, y, S.region_weights(G.lat, {"g": (-90, 90), "t": (-20, 20)})[1], [0, 1, 2], k)[0])
    return np.stack(out)


def test_one_date_gives_metrics_from_sums_bitwise():
    s = _sums(np.random.default_rng(3), 1, 4)
    np.testing.assert_array_equal(S.period_metrics(s, 4), S.metrics_from_sums(s[0], 4))


@pytest.mark.parametrize("M", [1, 5])
def test_period_metrics_over_several_dates(M):
    s = _sums(np.random.default_rng(4), 3, M)
    got = S.period_metrics(s, M)
    per = S.metrics_from_sums(s, M)
    w, e, e2, var, mae, g = (s[..., i] for i in range(6))
    ix = list(S.METRICS).index
    np.testing.assert_allclose(got[..., ix("acc")], per[..., ix("acc")].mean(0), rtol=1e-14)
    np.testing.assert_allclose(got[..., ix("bias")], (e / w).mean(0), rtol=1e-12)
    np.testing.assert_allclose(got[..., ix("rmse")], np.sqrt((e2 / w).mean(0)), rtol=1e-12)
    np.testing.assert_allclose(got[..., ix("crps")], ((mae - g / M ** 2) / w).mean(0), rtol=1e-12)
    if M > 1:
        spread = np.sqrt((var / (M - 1) / w).mean(0))
        np.testing.assert_allclose(got[..., ix("spread")], spread, rtol=1e-12)
        np.testing.assert_allclose(got[..., ix("ssr")], np.sqrt((M + 1) / M) * spread / np.sqrt((e2 / w).mean(0)),
                                   rtol=1e-12)
    with pytest.raises(ValueError):
        S.period_metrics(s[:0], M)


def test_map_metrics_form_the_maps_as_the_scalars():
    rng = np.random.default_rng(5)
    acc = np.abs(rng.standard_normal((2, 1, 5, 3, 4)))
    got = S.map_metrics(acc, 3, 4)
    e, e2, var, mae, g = (acc[:, :, i] for i in range(5))
    np.testing.assert_allclose(got[:, :, 0], e / 3, rtol=1e-6)
    np.testing.assert_allclose(got[:, :, 1], np.sqrt(e2 / 3), rtol=1e-6)
    np.testing.assert_allclose(got[:, :, 2], np.sqrt(var / 3 / 3), rtol=1e-6)
    np.testing.assert_allclose(got[:, :, 3], (mae - g / 16) / 3, rtol=1e-6)
    assert got.dtype == np.float32


# ---- C-ABI ------------------------------------------------------------------------------------------------------------------
NEW = ("sky_forecast_rank_histogram", "sky_forecast_score_maps")


def test_exports_present_and_declared():
    from skyrim_b200 import _ffi
    hdr = open(os.path.join(ROOT, "include", "skyrim_b200.h")).read()
    declared = set(re.findall(r"\b(sky_[a-z_0-9]+)\s*\(", hdr))
    for name in NEW:
        assert name in declared and name in _ffi.EXPORTS and hasattr(_ffi.lib(), name)


def _hist(members=4, stride=None, nlat=8, nlon=12, count=5, channels=(0, 4), n_sel=None, n_regions=1, seed=0, date=0,
          lead=0, cbytes=None, null_truth=False):
    from skyrim_b200 import _ffi
    L = _ffi.lib()
    bogus = C.c_void_p(0x1000)    # never inspected: every refusal below comes before the device-pointer check
    plane = nlat * nlon
    ns = len(channels) if n_sel is None else n_sel
    need = 4 * max(ns, 1) * nlat * (members + 2)
    rc = L.sky_forecast_rank_histogram(bogus, members, count * plane if stride is None else stride, nlat, nlon, count,
                                       (C.c_int32 * max(len(channels), 1))(*channels), ns, None if null_truth else bogus,
                                       bogus, n_regions, seed, date, lead, bogus, need if cbytes is None else cbytes,
                                       bogus, None)
    return rc, L.sky_last_error().decode()


def _maps(members=4, stride=None, nlat=8, nlon=12, count=5, channels=(0, 4), n_sel=None, null_maps=False):
    from skyrim_b200 import _ffi
    L = _ffi.lib()
    bogus = C.c_void_p(0x1000)
    plane = nlat * nlon
    ns = len(channels) if n_sel is None else n_sel
    rc = L.sky_forecast_score_maps(bogus, members, count * plane if stride is None else stride, nlat, nlon, count,
                                   (C.c_int32 * max(len(channels), 1))(*channels), ns, bogus,
                                   None if null_maps else bogus, None)
    return rc, L.sky_last_error().decode()


COMMON = [
    (dict(members=0), "members"), (dict(members=65), "members"),
    (dict(nlat=0), "nlat"), (dict(nlon=-1), "nlon"), (dict(nlat=65536, nlon=65536), "2^31"),
    (dict(count=0), "channel_count"),
    (dict(channels=(0, 5)), "channel 5"), (dict(channels=(-1, 2)), "channel -1"),
    (dict(stride=5 * 96 - 1), "member_stride"), (dict(stride=-1), "member_stride"),
    (dict(channels=tuple(range(129)), count=200), "n_sel"), (dict(channels=()), "n_sel"),
]


@pytest.mark.parametrize("kw, what", COMMON + [
    (dict(n_regions=0), "n_regions"), (dict(n_regions=5), "n_regions"), (dict(seed=2 ** 32), "seed"),
    (dict(date=-1), "date_index"), (dict(lead=-2), "lead_index"),
    (dict(cbytes=4 * 2 * 8 * 6 - 1), "counts_bytes"), (dict(null_truth=True), "null"),
])
def test_rank_histogram_refuses_bad_arguments_before_any_cuda_call(kw, what):
    rc, msg = _hist(**kw)
    assert rc == -1 and what in msg, msg


@pytest.mark.parametrize("kw, what", COMMON + [(dict(null_maps=True), "null")])
def test_score_maps_refuse_bad_arguments_before_any_cuda_call(kw, what):
    rc, msg = _maps(**kw)
    assert rc == -1 and what in msg, msg


# Every statistics and verification entry reads one field of members: here 5 channels of 8 x 12 points per member, with
# every other argument valid and bogus pointers that are never inspected.
def _field_entry(name, members=4, stride=5 * 96, channels=(0, 4)):
    from skyrim_b200 import _ffi
    L = _ffi.lib()
    bogus, plane, big = C.c_void_p(0x1000), 96, 1 << 40
    sel, n_sel = (C.c_int32 * max(len(channels), 1))(*channels), len(channels)
    if name == "sky_ensemble_stats":
        rc = L.sky_ensemble_stats(bogus, members, stride, plane, 5, sel, n_sel, None, 0, None, None, 0, bogus, None, None)
    elif name == "sky_ensemble_stats_multi":
        one = lambda ct, v: (ct * 1)(v)  # noqa: E731
        rc = L.sky_ensemble_stats_multi(1, one(C.c_void_p, 0x1000), one(C.c_int32, members), one(C.c_int64, stride),
                                        one(C.c_int32, 5), sel, n_sel, plane, None, 0, None, None, 0, bogus, None, None, None)
    elif name == "sky_forecast_scores":
        rc = L.sky_forecast_scores(bogus, members, stride, 8, 12, 5, sel, n_sel, bogus, None, bogus, 1, bogus, big, bogus,
                                   None)
    elif name == "sky_forecast_rank_histogram":
        rc = L.sky_forecast_rank_histogram(bogus, members, stride, 8, 12, 5, sel, n_sel, bogus, bogus, 1, 0, 0, 0, bogus, big,
                                           bogus, None)
    else:
        rc = L.sky_forecast_score_maps(bogus, members, stride, 8, 12, 5, sel, n_sel, bogus, bogus, None)
    return rc, L.sky_last_error().decode()


@pytest.mark.parametrize("entry", ["sky_ensemble_stats", "sky_ensemble_stats_multi", "sky_forecast_scores",
                                   "sky_forecast_rank_histogram", "sky_forecast_score_maps"])
@pytest.mark.parametrize("kw, what", [
    (dict(members=0), "members"), (dict(members=65), "members"), (dict(stride=5 * 96 - 1), "member_stride"),
    (dict(channels=(0, 5)), "channel 5"), (dict(channels=()), "n_sel"), (dict(channels=(0,) * 129), "n_sel"),
])
def test_every_entry_refuses_a_bad_member_field_before_any_cuda_call(entry, kw, what):
    rc, msg = _field_entry(entry, **kw)
    assert rc == -1 and what in msg, msg


# ---- score_period() host logic on a CPU fake of EnsembleRunner --------------------------------------------------------------
class TimeSource:
    """seeded truth that changes with time: source[t] -> DataArray(channel, lat, lon)"""

    def __init__(self, channels=CH, grid=G, seed=0):
        self.channels, self.grid, self.seed = list(channels), grid, seed

    def __getitem__(self, t):
        h = int((t - T0).total_seconds() // 3600)
        rng = np.random.default_rng(self.seed * 1000 + h + 7)
        v = (rng.standard_normal((len(self.channels), len(self.grid.lat), len(self.grid.lon))) + 0.1 * h).astype(np.float32)
        return xr.DataArray(v, dims=["channel", "lat", "lon"], coords=dict(channel=np.array(self.channels),
                            lat=np.array(self.grid.lat), lon=np.array(self.grid.lon)))


class FakeLoop:
    n_history_levels = 1
    time_step = STEP
    in_channel_names = out_channel_names = CH
    grid = G
    device = torch.device("cpu")
    engine = None


class FakeModel(GlobalModel):
    forcing_channels = ("msl",)

    def __init__(self, ic_source="synthetic", **kw):
        super().__init__("pangu", ic_source=ic_source)

    def build_model(self):
        return FakeLoop()


class FakeRunner:
    """EnsembleRunner's campaign interface on CPU members that gain 1 per step, scored by the references"""
    made = []

    def __init__(self, engine, base, sigma, members_per_gpu, rank=0, amp=0.05, seed=0, perturbation="gaussian", grf=None):
        self.M, self.amp, self.sigma, self.perturbation = members_per_gpu, amp, np.asarray(sigma), perturbation
        self.kw = dict(members=members_per_gpu, rank=rank, amp=amp, seed=seed, perturbation=perturbation, grf=grf)
        self.seeds, self.rings, self.calls = [], 0, []
        self.restart(base, seed)
        FakeRunner.made.append(self)

    def restart(self, base, seed):
        rng = np.random.default_rng(seed)
        noise = 0.0 if self.perturbation == "none" else self.amp * self.sigma[:, None, None] * rng.standard_normal(
            (self.M,) + base.shape)
        self.x0 = base[None] + noise
        self.x = torch.from_numpy(self.x0)
        self.seeds.append(seed)

    def truth_ring(self, n_sel):
        self.rings += 1
        return object()

    def iter_scores(self, n_steps, truth_at, clim=None, channels=None, row_weights=None, channel_offset=0, hist=None,
                    seed=0, date_index=0, maps=None, map_slot=None, map_channels=(), sums=None, ring=None):
        self.calls.append(dict(seed=seed, date_index=date_index, ring=ring, truths=[]))
        x, map_slot = self.x0, map_slot or {}
        if sums is None:                   # score(): a host tensor of sums and nothing else
            sums = torch.empty((n_steps + 1, len(row_weights), len(channels), 9), dtype=torch.float64)
        for n in range(n_steps + 1):
            y = truth_at(n)
            self.calls[-1]["truths"].append(y)
            sums[n] = torch.from_numpy(scores_ref.score_sums(x, y, row_weights, channels, clim)[0])
            if hist is not None:
                hist[n] = torch.from_numpy(ref.rank_histogram(x, y, row_weights, channels, seed, date_index, n)[0])
            if n in map_slot:
                t, _ = ref.map_terms(x, y[list(map_channels)], [channels[k] for k in map_channels])
                maps[map_slot[n]] += torch.from_numpy(t)
            x = x + 1.0
        return list(range(n_steps + 1)), sums


@pytest.fixture
def fake_runner(monkeypatch):
    from skyrim_b200 import ensemble
    FakeRunner.made = []
    monkeypatch.setattr(ensemble, "EnsembleRunner", FakeRunner)
    return FakeRunner


def _truth_array(src, starts, n_steps, drop=None):
    times = sorted({t + n * STEP for t in starts for n in range(n_steps + 1)} - {drop})
    return xr.DataArray(np.stack([src[t].values for t in times]), dims=["time", "channel", "lat", "lon"],
                        coords=dict(time=np.array([np.datetime64(t, "s") for t in times]), channel=np.array(CH),
                                    lat=np.array(G.lat), lon=np.array(G.lon)))


def test_period_start_times():
    from skyrim_b200.core.skyrim import period_start_times
    assert period_start_times("20240507", "20240509", "1200", 24) == [datetime.datetime(2024, 5, d, 12) for d in (7, 8, 9)]
    got = period_start_times("20240507", "20240508", "0600", 12)
    assert got == [datetime.datetime(2024, 5, 7, 6), datetime.datetime(2024, 5, 7, 18), datetime.datetime(2024, 5, 8, 6),
                   datetime.datetime(2024, 5, 8, 18)]
    assert period_start_times("20240507", "20240507") == [T0]
    for bad in (dict(every=5), dict(every=0), dict(end="20240506")):
        args = dict(start="20240507", end="20240509", time="0000", every=24)
        args.update(bad)
        with pytest.raises(ValueError):
            period_start_times(**args)


def test_score_period_host_logic_and_files(tmp_path, fake_runner):
    src = TimeSource()
    gm = FakeModel(ic_source=src)
    starts = [T0, T0 + 2 * STEP, T0 + 4 * STEP]
    regions = {"global": (-90, 90), "tropics": (-20, 20)}
    res, paths = gm.score_period(starts, 2, members=3, seed=5, channels=["t2m", "u10m"], regions=regions,
                                 map_leads=(12, 0), map_channels=["t2m"], save=True,
                                 save_config=dict(output_dir=str(tmp_path), forecast_id="fid"))
    assert len(fake_runner.made) == 1
    run = fake_runner.made[0]
    assert run.seeds == [5, 6, 7] and run.kw["seed"] == 5 and run.rings == 1
    assert [c["date_index"] for c in run.calls] == [0, 1, 2] and all(c["seed"] == 5 for c in run.calls)
    assert len({id(c["ring"]) for c in run.calls}) == 1
    for d, t0 in enumerate(starts):        # date d's truth at lead n is source[t0 + 6n h]
        for n in range(3):
            np.testing.assert_array_equal(run.calls[d]["truths"][n], src[t0 + n * STEP].values[[0, 2]])
    sel = ["u10m", "t2m"]
    assert tuple(res.cards.dims) == ("start_time", "lead_time", "metric", "region", "channel")
    assert list(res.cards.coords["start_time"]) == [str(np.datetime64(t, "s")) for t in starts]
    assert list(res.card.coords["channel"]) == sel and list(res.card.coords["lead_time"]) == [0.0, 6.0, 12.0]
    # each date's card is what score() computes for that date with seed + d
    for d, t0 in enumerate(starts):
        card, _ = gm.score(t0, 2, members=3, seed=5 + d, channels=["t2m", "u10m"], regions=regions)
        np.testing.assert_array_equal(res.cards.values[d], card.values)
    _, w = S.region_weights(G.lat, regions)
    sums = np.stack([np.stack([scores_ref.score_sums(FakeRunner(None, src[t0].values, run.sigma, 3, seed=5 + d).x0 + n,
                                                     src[t0 + n * STEP].values[[0, 2]], w, [0, 2])[0]
                               for n in range(3)]) for d, t0 in enumerate(starts)])
    np.testing.assert_allclose(np.moveaxis(res.card.values, 1, -1), S.period_metrics(sums, 3), rtol=1e-12, atol=1e-15)
    assert tuple(res.rank_histogram.dims) == ("lead_time", "region", "channel", "rank")
    np.testing.assert_allclose(res.rank_histogram.values.sum(-1), 1.0, rtol=1e-12)
    assert tuple(res.maps.dims) == ("lead_time", "metric", "channel", "lat", "lon") and res.maps.values.dtype == np.float32
    assert list(res.maps.coords["lead_time"]) == [0.0, 12.0] and list(res.maps.coords["metric"]) == list(S.MAP_METRICS)
    # lead 0 of the map: the members are the perturbed truth of each date
    acc = sum(ref.map_terms(FakeRunner(None, src[t0].values, run.sigma, 3, seed=5 + d).x0, src[t0].values[[2]], [2])[0]
              for d, t0 in enumerate(starts))
    np.testing.assert_allclose(res.maps.values[0, :, 0], S.map_metrics(acc, 3, 3)[0], rtol=1e-6)
    names = sorted(os.path.basename(p).split("__")[0] for p in paths)
    assert names == ["pangu-period3", "pangu-period3-cards", "pangu-period3-maps", "pangu-period3-rank"]
    for p in paths:
        back = xr.open_dataarray(p)
        da = {"": res.card, "-cards": res.cards, "-maps": res.maps,
              "-rank": res.rank_histogram}[os.path.basename(p).split("__")[0][len("pangu-period3"):]]
        assert tuple(back.dims) == tuple(da.dims) and back.attrs == da.attrs
        assert back.values.dtype.newbyteorder("=") == da.values.dtype
        np.testing.assert_array_equal(back.values, da.values)
        for d in da.dims:
            np.testing.assert_array_equal(np.asarray(back.coords[d]), np.asarray(da.coords[d]))


def test_score_period_without_maps(fake_runner):
    res, paths = FakeModel(ic_source=TimeSource()).score_period([T0], 1)
    assert res.maps is None and paths == [] and fake_runner.made[0].kw["perturbation"] == "none"
    assert list(res.card.coords["channel"]) == ["u10m", "v10m", "t2m"]          # the forcing is not scored
    assert res.rank_histogram.values.shape == (2, 1, 3, 2)


@pytest.mark.parametrize("kw, what", [
    (dict(map_leads=[6], map_channels=["nope"]), "nope"),
    (dict(map_leads=[6], map_channels=["msl"]), "forcings"),
    (dict(map_leads=[6], map_channels=["t2m"], channels=["u10m"]), "not among the scored"),
    (dict(map_leads=[3], map_channels=["t2m"]), "map lead"),
    (dict(map_leads=[18], map_channels=["t2m"]), "map lead"),
    (dict(map_leads=[-6], map_channels=["t2m"]), "map lead"),
    (dict(map_leads=[6]), "go together"),
    (dict(start_times=[T0 + STEP, T0]), "sorted"), (dict(start_times=[T0, T0]), "distinct"),
    (dict(start_times=[]), "at least one"),
    (dict(seed=2 ** 32), "seed"), (dict(members=65), "members"),
    (dict(truth="drop"), "2024-05-07T18:00:00"),
])
def test_score_period_refusals_name_the_problem_before_any_member_exists(kw, what, fake_runner):
    src = TimeSource()
    args = dict(start_times=[T0, T0 + STEP], n_steps=2)
    args.update(kw)
    if args.get("truth") == "drop":       # the second date's last valid time is missing
        args["truth"] = _truth_array(src, [T0, T0 + STEP], 2, drop=T0 + 3 * STEP)
    with pytest.raises(ValueError, match=re.escape(what)):
        FakeModel(ic_source=src).score_period(**args)
    assert fake_runner.made == []


def test_multi_model_score_period_is_refused():
    from skyrim_b200.core.models.ensemble import GlobalEnsemble
    with pytest.raises(NotImplementedError, match="multi-model"):
        GlobalEnsemble.score_period(None, [T0], 1)


def test_forecast_cli_period_options(tmp_path, monkeypatch, fake_runner):
    from click.testing import CliRunner
    from skyrim_b200 import forecast as F
    from skyrim_b200.core import models as M
    src = TimeSource()

    class SrcModel(FakeModel):
        def __init__(self, ic_source="synthetic", **kw):
            super().__init__(ic_source=src)
    monkeypatch.setitem(M.MODELS, "pangu", SrcModel)
    out = str(tmp_path / "out")
    r = CliRunner().invoke(F.main, ["-m", "pangu", "-d", "20240507", "-l", "12", "-o", out, "--score", "--until", "20240508",
                                    "--every", "12", "--members", "2", "--seed", "3", "--map_channels", "t2m",
                                    "--map_leads", "6,12"])
    assert r.exit_code == 0, r.output
    paths = [ln for ln in r.output.splitlines() if ln.endswith(".nc")]
    assert sorted(os.path.basename(p).split("__")[0] for p in paths) == [
        "pangu-period2", "pangu-period2-cards", "pangu-period2-maps", "pangu-period2-rank"]
    run = fake_runner.made[-1]
    assert run.seeds == [3, 4, 5, 6] and run.kw["perturbation"] == "spherical_grf"
    cards = xr.open_dataarray([p for p in paths if "-cards" in p][0])
    assert list(cards.coords["start_time"]) == ["2024-05-07T00:00:00", "2024-05-07T12:00:00", "2024-05-08T00:00:00",
                                                "2024-05-08T12:00:00"]
    maps = xr.open_dataarray([p for p in paths if "-maps" in p][0])
    assert list(maps.coords["lead_time"]) == [6.0, 12.0] and list(maps.coords["channel"]) == ["t2m"]
    n = len(fake_runner.made)
    for bad in (["--until", "20240508"], ["--every", "12"], ["--map_channels", "t2m"], ["--map_leads", "6"],
                ["--score", "--until", "20240508", "--map_leads", "six"], ["--score", "--until", "20240508", "--every", "5"]):
        assert CliRunner().invoke(F.main, ["-o", out, "-d", "20240507"] + bad).exit_code != 0, bad
    assert len(fake_runner.made) == n
