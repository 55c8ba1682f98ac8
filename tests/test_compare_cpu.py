"""Model comparison without a device: the paired differences against the plain-loop oracle, the *_multi exports and their
refusals before any CUDA call, and GlobalEnsemble.compare's host logic on CPU fakes of the models and the scoring entries
(the refusals, the initial states, the entries, the files) and the forecast CLI's --compare."""
import ctypes as C
import datetime
import os
import re
import sys

import numpy as np
import pytest
import torch
from scipy import stats as st

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import verify_period_ref as ref  # noqa: E402
from oracle import compare_ref, scores_ref  # noqa: E402
from skyrim_b200 import scores as S  # noqa: E402
from skyrim_b200 import xr_shim as xr  # noqa: E402
from skyrim_b200.core.models.base import GlobalModel  # noqa: E402
from skyrim_b200.timeloop import equiangular_grid  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T0 = datetime.datetime(2024, 5, 7)
STEP = datetime.timedelta(hours=6)
G = equiangular_grid(19, 36)


# ---- paired differences ------------------------------------------------------------------------------------------------------
def _check(d):
    got = S.paired_difference_stats(np.asarray(d, dtype=np.float64)[:, None])[0]
    want = np.array(compare_ref.paired_stats(d))
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-15, equal_nan=True)
    return got


def test_ar1_series_with_known_lag1_autocorrelation():
    rng = np.random.default_rng(0)
    d = np.empty(4000)
    d[0] = rng.standard_normal()
    for t in range(1, d.size):
        d[t] = 0.6 * d[t - 1] + rng.standard_normal()
    got = _check(d + 0.1)
    r1 = got[4] and (d.size - got[4]) / (d.size + got[4])      # n_eff = D (1 - r1) / (1 + r1)
    assert abs(r1 - 0.6) < 0.05
    assert got[4] < d.size / 3                                    # inflated variance: far fewer effective dates


def test_negative_autocorrelation_is_the_t_test():
    d = np.array([0.3, -0.1, 0.5, -0.2, 0.6, 0.0, 0.4, -0.3, 0.7, 0.1])
    got = _check(d)
    assert got[4] == d.size
    t = st.ttest_1samp(d, 0.0)
    ci = t.confidence_interval(0.95)
    np.testing.assert_allclose(got[3], t.pvalue, rtol=1e-10)
    np.testing.assert_allclose(got[1:3], [ci.low, ci.high], rtol=1e-10)


def test_zero_variance_nan_and_two_dates():
    got = _check([0.25, 0.25, 0.25, 0.25])
    assert list(got[:4]) == [0.25, 0.25, 0.25, 0.0]
    got = _check([0.0, 0.0, 0.0])
    assert list(got[:4]) == [0.0, 0.0, 0.0, 1.0]
    assert np.isnan(_check([1.0, np.nan, 2.0, 3.0])).all()
    got = _check([1.0, 2.0])
    assert got[0] == 1.5 and np.isnan(got[1:]).all()


def test_paired_differences_layout_and_sign():
    rng = np.random.default_rng(1)
    a = rng.random((5, 2, len(S.METRICS), 1, 3))
    b = a.copy()
    b[:, :, S.METRICS.index("rmse")] += 1.0 + 0.1 * rng.random((5, 2, 1, 3))
    d = S.paired_differences(a, b)
    assert d.shape == (3, 5, 2, 1, 3)
    assert (d[0, 0] < -0.9).all() and (d[0, 3] < 1e-3).all()     # a better in rmse, significantly
    np.testing.assert_array_equal(d[1], S.paired_difference_stats(np.zeros((5, 2, 1, 3)))[..., :].transpose(3, 0, 1, 2))


# ---- the C-ABI ------------------------------------------------------------------------------------------------------------------
MULTI = ("sky_forecast_scores_multi", "sky_forecast_rank_histogram_multi", "sky_forecast_score_maps_multi")


def test_exports_present_and_declared():
    from skyrim_b200 import _ffi
    hdr = open(os.path.join(ROOT, "include", "skyrim_b200.h")).read()
    declared = set(re.findall(r"\b(sky_[a-z_0-9]+)\s*\(", hdr))
    for name in MULTI:
        assert name in declared and name in _ffi.EXPORTS and hasattr(_ffi.lib(), name)
    assert _ffi.lib().sky_abi_version() == 1


def _multi(entry, n_sources=2, members=(3, 2), strides=None, counts=(5, 4), channels=((0, 4), (3, 1)), nlat=4, nlon=24,
           n_regions=1, ws_bytes=None, seed=0, date=0, lead=0, null=None, n_sel=None):
    from skyrim_b200 import _ffi
    L = _ffi.lib()
    bogus = C.c_void_p(0x1000)    # never inspected: every refusal below comes before the device-pointer check
    arr = lambda ct, v: (ct * max(len(v), 1))(*v)  # noqa: E731
    plane = nlat * nlon
    strides = [c * plane for c in counts] if strides is None else strides
    xs = [0 if null == "x" else 0x1000] * len(members)
    ptr = lambda name: None if null == name else bogus  # noqa: E731
    n_sel = len(channels[0]) if n_sel is None else n_sel
    head = (n_sources, arr(C.c_void_p, xs), arr(C.c_int32, members), arr(C.c_int64, strides), arr(C.c_int32, counts),
            arr(C.c_int32, [c for ch in channels for c in ch]), n_sel, nlat, nlon)
    total = sum(members)
    if entry == "scores":
        need = n_regions * n_sel * 9 * 128 * 8 if ws_bytes is None else ws_bytes
        rc = L.sky_forecast_scores_multi(*head, ptr("truth"), None, ptr("rw"), n_regions, ptr("ws"), need, ptr("out"), None)
    elif entry == "hist":
        need = n_sel * nlat * (total + 2) * 4 if ws_bytes is None else ws_bytes
        rc = L.sky_forecast_rank_histogram_multi(*head, ptr("truth"), ptr("rw"), n_regions, seed, date, lead, ptr("ws"),
                                                 need, ptr("out"), None)
    else:
        rc = L.sky_forecast_score_maps_multi(*head, ptr("truth"), ptr("out"), None)
    return rc, L.sky_last_error().decode()


SOURCE_BAD = [
    (dict(n_sources=0), "n_sources"), (dict(n_sources=5, members=(1,) * 5, counts=(5,) * 5, channels=((0,),) * 5), "n_sources"),
    (dict(members=(0, 2)), "members[0]"), (dict(members=(3, 65)), "members[1]"), (dict(members=(40, 25)), "total members"),
    (dict(counts=(5, 0)), "channel_count[1]"), (dict(strides=(5 * 96, 4 * 96 - 1)), "member_stride[1]"),
    (dict(channels=((0, 5), (3, 1))), "channel 5 of source 0"), (dict(channels=((0, 4), (4, 1))), "channel 4 of source 1"),
    (dict(channels=((0, 4), (-1, 1))), "channel -1"), (dict(n_sel=0), "n_sel"),
    (dict(channels=(tuple(range(129)), tuple(range(129))), counts=(200, 200)), "n_sel"),
    (dict(nlat=0), "nlat"), (dict(null="x"), "x[0]"), (dict(null="truth"), "must not be null"),
    (dict(null="out"), "must not be null"),
]


@pytest.mark.parametrize("entry", ["scores", "hist", "maps"])
@pytest.mark.parametrize("kw, what", SOURCE_BAD)
def test_multi_entries_refuse_bad_sources_before_any_cuda_call(entry, kw, what):
    rc, msg = _multi(entry, **kw)
    assert rc == -1 and what in msg, msg


@pytest.mark.parametrize("entry, kw, what", [
    ("scores", dict(n_regions=0), "n_regions"), ("scores", dict(n_regions=5), "n_regions"),
    ("scores", dict(ws_bytes=8), "partial_bytes"), ("scores", dict(null="rw"), "must not be null"),
    ("scores", dict(null="ws"), "must not be null"),
    ("hist", dict(n_regions=0), "n_regions"), ("hist", dict(seed=2 ** 32), "seed"), ("hist", dict(date=-1), "date_index"),
    ("hist", dict(lead=-1), "lead_index"), ("hist", dict(ws_bytes=4), "counts_bytes"), ("hist", dict(null="rw"), "must not"),
])
def test_multi_entries_refuse_their_own_arguments_before_any_cuda_call(entry, kw, what):
    rc, msg = _multi(entry, **kw)
    assert rc == -1 and what in msg, msg


# ---- compare() on CPU fakes -------------------------------------------------------------------------------------------------
class TimeSource:
    def __init__(self, channels, grid=G):
        self.channels, self.grid = list(channels), grid

    def __getitem__(self, t):
        h = int((t - T0).total_seconds() // 3600)
        rng = np.random.default_rng(h + 1000)
        v = (rng.standard_normal((len(self.channels), len(self.grid.lat), len(self.grid.lon))) + 0.1 * h).astype(np.float32)
        return xr.DataArray(v, dims=["channel", "lat", "lon"], coords=dict(channel=np.array(self.channels),
                            lat=np.array(self.grid.lat), lon=np.array(self.grid.lon)))


def _fake_model(name, channels, forcing=()):
    class Loop:
        n_history_levels = 1
        time_step = STEP
        in_channel_names = out_channel_names = list(channels)
        grid = G
        device = torch.device("cpu")
        engine = None
        guard_first_step = False

    class Fake(GlobalModel):
        forcing_channels = tuple(forcing)

        def __init__(self, ic_source="synthetic", **kw):
            super().__init__(name, ic_source=ic_source)

        def build_model(self):
            return Loop()

        def release_model(self):
            pass
    return Fake


CH_A, CH_B = ["u10m", "v10m", "t2m", "msl", "z500"], ["z500", "t2m", "tp06", "u10m"]


@pytest.fixture
def fakes(monkeypatch):
    """two fake models on the CPU whose engine adds 1 per step, scored by the references"""
    from skyrim_b200 import engine as E
    from skyrim_b200 import ensemble as ens_mod
    from skyrim_b200.core import models as Mo
    from skyrim_b200.core.models.ensemble import GlobalEnsemble
    monkeypatch.setitem(Mo.MODELS, "pangu", _fake_model("pangu", CH_A, ("msl",)))
    monkeypatch.setitem(Mo.MODELS, "graphcast", _fake_model("graphcast", CH_B, ("tp06",)))
    calls = dict(engine=0, lead0=[], lead=None)

    def step_all(self, states, first=False):
        calls["engine"] += 1
        for k in range(len(states)):
            states[k] = states[k] + 1.0

    class Ev:
        def record(self, *a):
            pass
    monkeypatch.setattr(GlobalEnsemble, "_step_all", step_all)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: None)
    monkeypatch.setattr(ens_mod, "truth_ring", lambda *a: dict(scored=[Ev(), Ev()]))

    def upload(ring, i, y, main):
        calls["lead"] = i
        return torch.from_numpy(np.array(y))
    monkeypatch.setattr(ens_mod, "upload_truth", upload)

    def pooled(srcs, chans):
        C0 = srcs[0].shape[1]
        out = np.zeros((sum(x.shape[0] for x in srcs), C0) + tuple(srcs[0].shape[-2:]))
        r = 0
        for x, ch in zip(srcs, chans):
            out[r:r + x.shape[0], chans[0]] = x.numpy()[:, ch]
            r += x.shape[0]
        return out

    def fs(x, truth, rw, channels, clim=None, channel_offset=0, out=None):
        if calls["lead"] == 0:             # per date: each model's members, then the pooled members
            calls["lead0"].append(x.numpy().copy())
        out[...] = torch.from_numpy(scores_ref.score_sums(x.numpy()[:, channel_offset:], truth.numpy(), rw.numpy(), channels,
                                                          None if clim is None else clim.numpy())[0])
        return out

    def rh(x, truth, rw, seed, d, n, channels, channel_offset=0, out=None):
        out[...] = torch.from_numpy(ref.rank_histogram(x.numpy()[:, channel_offset:], truth.numpy(), rw.numpy(), channels,
                                                       seed, d, n)[0])
        return out

    def sm(x, truth, maps, channels, channel_offset=0):
        maps += torch.from_numpy(ref.map_terms(x.numpy()[:, channel_offset:], truth.numpy(), channels)[0])
        return maps
    monkeypatch.setattr(E, "forecast_scores", fs)
    monkeypatch.setattr(E, "forecast_rank_histogram", rh)
    monkeypatch.setattr(E, "score_maps_accumulate", sm)
    monkeypatch.setattr(E, "forecast_scores_multi", lambda s, c, t, rw, clim=None, out=None: fs(
        torch.from_numpy(pooled(s, c)), t, rw, c[0], clim, 0, out))
    monkeypatch.setattr(E, "forecast_rank_histogram_multi", lambda s, c, t, rw, seed, d, n, out=None: rh(
        torch.from_numpy(pooled(s, c)), t, rw, seed, d, n, c[0], 0, out))
    monkeypatch.setattr(E, "score_maps_accumulate_multi", lambda s, c, t, maps: sm(torch.from_numpy(pooled(s, c)), t, maps,
                                                                                   c[0]))
    return calls


def _ensemble():
    from skyrim_b200.core.models.ensemble import GlobalEnsemble
    return GlobalEnsemble(["pangu", "graphcast"], ic_source=TimeSource(["u10m", "v10m", "t2m", "msl", "z500", "tp06"]))


@pytest.mark.parametrize("kw, what", [
    (dict(start_times=[T0, T0 + STEP, T0 + 3 * STEP]), "equally spaced"),
    (dict(start_times=[T0 + STEP, T0]), "sorted"), (dict(start_times=[]), "at least one"),
    (dict(members=33), "64"), (dict(members=0), "members"), (dict(seed=2 ** 32), "seed"), (dict(n_steps=-1), "n_steps"),
    (dict(channels=["msl"]), "not shared"), (dict(channels=["v10m"]), "not shared"),
    (dict(map_leads=[6], map_channels=["nope"]), "not shared"), (dict(map_leads=[3], map_channels=["t2m"]), "map lead"),
    (dict(map_leads=[6]), "go together"), (dict(perturbation="bogus"), "perturbation"),
    (dict(save=True, save_config=dict(file_type="zarr")), "netCDF"), (dict(regions={"x": (10, 5)}), "band"),
    (dict(truth="drop"), "2024-05-07T18:00:00"),
])
def test_compare_refusals_name_the_problem_before_any_engine_call(kw, what, fakes):
    ge = _ensemble()
    args = dict(start_times=[T0, T0 + STEP], n_steps=2)
    args.update(kw)
    if args.get("truth") == "drop":
        src = ge.data_source
        times = [t for t in sorted({T0 + n * STEP for n in range(4)}) if t != T0 + 3 * STEP]
        args["truth"] = xr.DataArray(np.stack([src[t].values for t in times]), dims=["time", "channel", "lat", "lon"],
                                     coords=dict(time=np.array([np.datetime64(t, "s") for t in times]),
                                                 channel=np.asarray(src[T0].coords["channel"]), lat=np.array(G.lat),
                                                 lon=np.array(G.lon)))
    with pytest.raises(ValueError, match=re.escape(what)):
        ge.compare(**args)
    assert fakes["engine"] == 0


def test_compare_host_logic_and_files(tmp_path, fakes):
    ge = _ensemble()
    assert ge.shared_channels == ["u10m", "t2m", "z500"]
    starts = [T0, T0 + 2 * STEP, T0 + 4 * STEP]
    res, paths = ge.compare(starts, 2, regions={"global": (-90, 90), "tropics": (-20, 20)}, map_leads=[12],
                            map_channels=["t2m"], seed=4, save=True,
                            save_config=dict(output_dir=str(tmp_path), forecast_id="fid"))
    assert res.entries == ["pangu", "graphcast", "pooled"] and res.pairs == ["pangu-graphcast", "pangu-pooled",
                                                                              "graphcast-pooled"]
    assert list(res.card.coords["channel"]) == ["u10m", "t2m", "z500"]
    assert res.scores["pooled"].rank_histogram.values.shape == (3, 2, 3, 3)
    assert res.card.values.shape == (3, 3, len(S.METRICS), 2, 3)
    np.testing.assert_array_equal(res.differences.values[1], S.paired_differences(res.scores["pangu"].cards.values,
                                                                                  res.scores["pooled"].cards.values))
    label = "graphcast_pangu-compare1"
    want = {"": res.card, "-cards": None, "-maps": None, "-diff": res.differences,
            "-rank-pangu": res.scores["pangu"].rank_histogram, "-rank-graphcast": res.scores["graphcast"].rank_histogram,
            "-rank-pooled": res.scores["pooled"].rank_histogram}
    names = sorted(os.path.basename(p).split("__")[0] for p in paths)
    assert names == sorted(label + k for k in want)
    dims = {"-cards": ("model", "start_time", "lead_time", "metric", "region", "channel"),
            "-maps": ("model", "lead_time", "metric", "channel", "lat", "lon")}
    for p in paths:
        suffix = os.path.basename(p).split("__")[0][len(label):]
        back = xr.open_dataarray(p)
        if want[suffix] is None:
            assert tuple(back.dims) == dims[suffix]
            field = suffix[1:]
            np.testing.assert_array_equal(back.values, np.stack([getattr(res.scores[e], field).values for e in res.entries]))
        else:
            da = want[suffix]
            assert tuple(back.dims) == tuple(da.dims)
            np.testing.assert_array_equal(back.values, da.values)
            for d in da.dims:
                np.testing.assert_array_equal(np.asarray(back.coords[d]), np.asarray(da.coords[d]))


def test_first_model_members_are_its_own_score_period_members(fakes, monkeypatch):
    from skyrim_b200 import ensemble as ens_mod
    ge = _ensemble()
    starts = [T0, T0 + STEP]
    ge.compare(starts, 0)
    held = []

    class Runner:
        def __init__(self, engine, base, sigma, members_per_gpu, **kw):
            self.x = torch.from_numpy(np.repeat(np.asarray(base)[None], members_per_gpu, 0))
            held.append(self.x.numpy().copy())

        def truth_ring(self, n):
            return None

        def restart(self, base, seed):
            self.x = torch.from_numpy(np.asarray(base)[None].copy())
            held.append(self.x.numpy().copy())

        def iter_scores(self, n_steps, truth_at, clim, channels, rw, offset, hist=None, sums=None, maps=None, **kw):
            return [0], sums
    monkeypatch.setattr(ens_mod, "EnsembleRunner", Runner)
    ge.models[0].score_period(starts, 0)
    assert len(held) == 2 and len(fakes["lead0"]) == 6
    for d in range(2):
        assert fakes["lead0"][3 * d].tobytes() == held[d].astype(np.float32).tobytes()


def test_forecast_cli_compare(tmp_path, fakes):
    from click.testing import CliRunner
    from skyrim_b200 import forecast as F
    out = str(tmp_path / "out")
    r = CliRunner().invoke(F.main, ["--models", "pangu,graphcast", "--compare", "-d", "20240507", "--until", "20240508",
                                    "--every", "12", "-l", "12", "-o", out, "--map_channels", "t2m", "--map_leads", "6"])
    assert r.exit_code == 0, r.output
    paths = [ln for ln in r.output.splitlines() if ln.endswith(".nc")]
    label = "graphcast_pangu-compare1"
    assert sorted(os.path.basename(p).split("__")[0] for p in paths) == sorted(
        label + s for s in ("", "-cards", "-maps", "-diff", "-rank-pangu", "-rank-graphcast", "-rank-pooled"))
    cards = xr.open_dataarray([p for p in paths if "-cards" in p][0])
    assert cards.values.shape[:3] == (3, 4, 3) and list(cards.coords["model"]) == ["pangu", "graphcast", "pooled"]
    diff = xr.open_dataarray([p for p in paths if "-diff" in p][0])
    assert tuple(diff.dims) == ("pair", "metric", "stat", "lead_time", "region", "channel") and diff.values.shape[:3] == (3, 3, 5)
    r = CliRunner().invoke(F.main, ["--models", "pangu,graphcast", "--compare", "-d", "20240507", "-l", "6", "-o", out])
    assert r.exit_code == 0, r.output
    for bad in (["--compare"], ["-m", "pangu", "--compare"], ["--models", "pangu,graphcast", "--compare", "--score"],
                ["--models", "pangu,graphcast", "--compare", "--members", "2", "--quantiles", "0.5"],
                ["--models", "pangu,graphcast", "--compare", "--members", "2", "--exceed", "t2m:1"],
                ["--models", "pangu,graphcast", "--until", "20240508"], ["--models", "pangu,graphcast", "--truth", "a.nc"]):
        assert CliRunner().invoke(F.main, ["-o", out, "-d", "20240507"] + bad).exit_code != 0, bad
