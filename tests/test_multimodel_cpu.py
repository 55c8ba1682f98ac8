"""Multi-model ensembles without a device: the shared and union channels, the channel view, keyword routing, every
refusal of GlobalEnsemble, the file labels, the sky_ensemble_stats_multi export and its argument refusals, and the
oracle against a hand computation."""
import ctypes as C
import datetime
import os
import re

import numpy as np
import pytest

from oracle import multi_stats_ref
from skyrim_b200.config import FCNV2_CHANNELS, GRAPHCAST_CHANNELS, PANGU_CHANNELS
from skyrim_b200.core.models.base import GlobalModel, SyntheticDataSource
from skyrim_b200.core.models.ensemble import GlobalEnsemble, SourceView
from skyrim_b200.timeloop import equiangular_grid
from skyrim_b200.weights import synthetic_state

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T0 = datetime.datetime(2024, 5, 7)


class FakeLoop:
    time_step = datetime.timedelta(hours=6)

    def __init__(self, names, nlat, nlon):
        self.in_channel_names = self.out_channel_names = list(names)
        self.grid = equiangular_grid(nlat, nlon)


def fake(name, names):
    class Fake(GlobalModel):
        made = []

        def __init__(self, ic_source="synthetic", nlat=19, nlon=36, channels=None, **kw):
            self.kw, self.shape, self.names = kw, (nlat, nlon), list(channels or names)
            Fake.made.append(self)
            super().__init__(name, ic_source=ic_source)

        def build_model(self):
            return FakeLoop(self.names, *self.shape)

        def release_model(self):
            self.released = True
    return Fake


@pytest.fixture
def fakes(monkeypatch):
    from skyrim_b200.core import models as M
    out = {"pangu": fake("pangu", PANGU_CHANNELS), "fourcastnet_v2": fake("fourcastnet_v2", FCNV2_CHANNELS),
           "graphcast": fake("graphcast", GRAPHCAST_CHANNELS)}
    for k, v in out.items():
        monkeypatch.setitem(M.MODELS, k, v)
    return out


def test_shared_channels_are_the_intersection_in_the_first_models_order(fakes):
    ens = GlobalEnsemble(["pangu", "fourcastnet_v2", "graphcast"])
    want = [f"{v}{p}" for v in "ztuv" for p in (50, 100, 150, 200, 250, 300, 400, 500, 600, 700, 850, 925, 1000)]
    assert ens.shared_channels == [c for c in PANGU_CHANNELS if c in want + ["msl", "u10m", "v10m", "t2m"]]
    assert len(ens.shared_channels) == 56 and ens.out_channel_names == ens.shared_channels
    assert GlobalEnsemble(["pangu", "graphcast"]).shared_channels == PANGU_CHANNELS                  # all 69
    assert GlobalEnsemble(["fourcastnet_v2", "pangu"]).shared_channels[:3] == ["u10m", "v10m", "t2m"]  # SFNO's order


def test_union_source_and_views_reproduce_each_models_channels(fakes):
    ens = GlobalEnsemble(["pangu", "fourcastnet_v2", "graphcast"])
    union = ens.channel_names
    assert union[:69] == PANGU_CHANNELS and len(union) == len(set(union))
    assert union[69:] == [c for c in FCNV2_CHANNELS if c not in PANGU_CHANNELS] + \
        [c for c in GRAPHCAST_CHANNELS if c not in PANGU_CHANNELS + FCNV2_CHANNELS]
    assert isinstance(ens.data_source, SyntheticDataSource) and ens.data_source.channel_names == union
    full = ens.data_source[T0].values
    # synthetic_state draws channel by channel: the first model's view is its own synthetic state, bit for bit
    np.testing.assert_array_equal(SourceView(ens.data_source, PANGU_CHANNELS)[T0].values, synthetic_state(PANGU_CHANNELS, 19, 36))
    for m in ens.models:
        v = m.data_source[T0]
        assert isinstance(m.data_source, SourceView) and list(v.coords["channel"]) == m.in_channel_names
        np.testing.assert_array_equal(v.values, full[[union.index(c) for c in m.in_channel_names]])
    # a user-supplied source is used as it is
    src = SyntheticDataSource(union, 19, 36, seed=3)
    assert GlobalEnsemble(["pangu", "graphcast"], ic_source=src).data_source is src


def test_keywords_named_after_a_model_go_to_that_model_only(fakes):
    GlobalEnsemble(["pangu", "graphcast"], pangu=dict(weight_seed=4), graphcast=dict(weight_seed=5, device=1), device=0)
    assert fakes["pangu"].made[-1].kw == dict(weight_seed=4, device=0)
    assert fakes["graphcast"].made[-1].kw == dict(weight_seed=5, device=1)


def test_refusals_at_construction(fakes):
    with pytest.raises(ValueError, match="duplicate"):
        GlobalEnsemble(["pangu", "pangu"])
    assert fakes["pangu"].made == []                         # refused before any model is built
    with pytest.raises(ValueError, match="grid"):
        GlobalEnsemble(["pangu", "graphcast"], graphcast=dict(nlat=21))
    assert fakes["pangu"].made[-1].released                  # what was built is released
    with pytest.raises(ValueError, match="grid"):
        GlobalEnsemble(["pangu", "graphcast"], graphcast=dict(nlon=40))
    with pytest.raises(ValueError, match="share no"):
        GlobalEnsemble(["pangu", "fourcastnet_v2"], fourcastnet_v2=dict(channels=["sp", "tcwv"]))
    with pytest.raises(ValueError):
        GlobalEnsemble(["pangu", "nope"])


@pytest.mark.parametrize("kw", [
    dict(members=22), dict(members=0), dict(channels=["sp"]), dict(channels=["nope"]), dict(events={"tcwv": 30.0}),
    dict(events={"w500": 0.1}), dict(save_config=dict(filter_vars=["q500"])), dict(quantiles=(1.5,)), dict(n_steps=0),
    dict(events={"t2m": float("nan")}), dict(save=True, save_config=dict(file_type="zarr")), dict(perturbation="bred"),
    dict(perturbation="gaussian", grf=dict(lmax=4)),
])
def test_predict_ensemble_refusals(fakes, kw, monkeypatch):
    ens = GlobalEnsemble(["pangu", "fourcastnet_v2", "graphcast"])
    monkeypatch.setattr(GlobalEnsemble, "ensemble_members", lambda *a, **k: pytest.fail("members were built"))
    args = dict(start_time=T0, n_steps=1, members=3)
    args.update(kw)
    with pytest.raises(ValueError):
        ens.predict_ensemble(**args)


def test_sixty_four_members_in_all_is_the_limit(fakes, monkeypatch):
    ens = GlobalEnsemble(["pangu", "fourcastnet_v2", "graphcast"])
    monkeypatch.setattr(GlobalEnsemble, "ensemble_members", lambda *a, **k: (_ for _ in ()).throw(RuntimeError("built")))
    with pytest.raises(RuntimeError, match="built"):         # 3 x 21 = 63 passes validation
        ens.predict_ensemble(T0, 1, 21)
    with pytest.raises(ValueError, match="64"):
        ens.predict_ensemble(T0, 1, 22)


def test_forecast_refuses_unshared_channels_and_labels(fakes):
    ens = GlobalEnsemble(["pangu", "fourcastnet_v2", "graphcast"])
    with pytest.raises(ValueError, match="shared"):
        ens.forecast(T0, 1, channels=["q500"])
    assert ens.label == "fourcastnet_v2_graphcast_pangu"
    with pytest.raises(NotImplementedError):
        ens.predict_one_step(T0)


def test_facade_builds_an_ensemble_for_several_names(fakes):
    from skyrim_b200.core.skyrim import Skyrim
    sk = Skyrim("graphcast", "pangu", pangu=dict(weight_seed=2))
    assert isinstance(sk.model, GlobalEnsemble) and sk.model.model_names == ["graphcast", "pangu"]
    assert fakes["pangu"].made[-1].kw == dict(weight_seed=2)
    assert sk.model.shared_channels[0] == GRAPHCAST_CHANNELS[0] and sk.model.time_steps(24) == 4
    assert isinstance(Skyrim("pangu").model, fakes["pangu"])
    with pytest.raises(ValueError):
        Skyrim("pangu", "pangu")


def test_cli_models_option(fakes):
    from click.testing import CliRunner
    from skyrim_b200 import forecast as F
    assert {o.name: o for o in F.main.params}["models"].default == ""
    for bad in (["--models", "pangu,nope"], ["--models", "pangu,pangu"], ["--models", "pangu"],
                ["--models", "pangu,graphcast,fourcastnet_v2", "--members", "22"]):
        assert CliRunner().invoke(F.main, bad).exit_code != 0, bad
    assert fakes["pangu"].made == []


def test_export_present_and_declared():
    from skyrim_b200 import _ffi
    hdr = open(os.path.join(ROOT, "include", "skyrim_b200.h")).read()
    assert "sky_ensemble_stats_multi" in set(re.findall(r"\b(sky_[a-z_0-9]+)\s*\(", hdr))
    assert "sky_ensemble_stats_multi" in _ffi.EXPORTS and hasattr(_ffi.lib(), "sky_ensemble_stats_multi")


def _call(n_sources=2, members=(3, 2), strides=None, counts=(5, 4), channels=((0, 4), (3, 1)), plane=96, quantiles=(0.5,),
          ev_sel=(0, 1), ev_thr=(1.0, 2.0), n_sel=None, n_q=None, n_events=None):
    from skyrim_b200 import _ffi
    L = _ffi.lib()
    bogus = 0x1000    # never inspected: every refusal below comes before the device-pointer check
    arr = lambda ct, v: (ct * max(len(v), 1))(*v)  # noqa: E731
    strides = [c * plane for c in counts] if strides is None else strides
    flat = [c for ch in channels for c in ch]
    rc = L.sky_ensemble_stats_multi(n_sources, arr(C.c_void_p, [bogus] * len(members)), arr(C.c_int32, members),
                                    arr(C.c_int64, strides), arr(C.c_int32, counts), arr(C.c_int32, flat),
                                    len(channels[0]) if n_sel is None else n_sel, plane, arr(C.c_double, quantiles),
                                    len(quantiles) if n_q is None else n_q, arr(C.c_int32, ev_sel), arr(C.c_float, ev_thr),
                                    len(ev_sel) if n_events is None else n_events, C.c_void_p(bogus), C.c_void_p(bogus),
                                    C.c_void_p(bogus), None)
    return rc, L.sky_last_error().decode()


@pytest.mark.parametrize("kw, what", [
    (dict(n_sources=0), "n_sources"), (dict(n_sources=5, members=(1,) * 5, counts=(5,) * 5, channels=((0,),) * 5), "n_sources"),
    (dict(members=(0, 2)), "members[0]"), (dict(members=(3, 65)), "members[1]"),
    (dict(members=(40, 25)), "total members"), (dict(plane=0), "plane"),
    (dict(counts=(5, 0)), "channel_count[1]"), (dict(strides=(5 * 96, 4 * 96 - 1)), "member_stride[1]"),
    (dict(channels=((0, 5), (3, 1))), "channel 5 of source 0"), (dict(channels=((0, 4), (4, 1))), "channel 4 of source 1"),
    (dict(channels=((0, 4), (-1, 1))), "channel -1"),
    (dict(quantiles=(1.5,)), "quantile"), (dict(quantiles=(float("nan"),)), "quantile"),
    (dict(ev_sel=(0, 2)), "event_sel"), (dict(ev_sel=(1, 0)), "decreases"),
    (dict(ev_thr=(1.0, float("inf"))), "threshold"), (dict(ev_thr=(float("nan"), 1.0)), "threshold"),
    (dict(channels=(tuple(range(129)), tuple(range(129))), counts=(200, 200)), "n_sel"), (dict(n_sel=0), "n_sel"),
    (dict(quantiles=(0.5,) * 9), "n_q"), (dict(ev_sel=(0,) * 65, ev_thr=(1.0,) * 65), "n_events"),
])
def test_library_refuses_bad_arguments_before_any_cuda_call(kw, what):
    rc, msg = _call(**kw)
    assert rc == -1 and what in msg, msg


def test_oracle_against_a_hand_computation():
    a = np.zeros((2, 3, 1, 2), np.float32)            # source 0: 2 members, 3 channels
    b = np.zeros((3, 2, 1, 2), np.float32)            # source 1: 3 members, 2 channels
    a[:, 2, 0, 0], a[:, 0, 0, 0] = [1.0, 2.0], [7.0, 7.0]
    b[:, 1, 0, 0], b[:, 0, 0, 0] = [3.0, 4.0, 10.0], [5.0, 5.0, 5.0]
    # selected channel 0 is a[2] / b[1], channel 1 is a[0] / b[0]
    s, p, m = multi_stats_ref.multi_source_stats([a, b], [[2, 0], [1, 0]], (0.0, 0.5, 1.0), [(0, 3.0), (1, 6.0)])
    v = np.array([1.0, 2.0, 3.0, 4.0, 10.0])
    assert s[0, 0, 0, 0] == np.float32(4.0) and np.isclose(s[1, 0, 0, 0], np.sqrt(((v - 4.0) ** 2).mean()))
    assert (s[2, 0, 0, 0], s[3, 0, 0, 0], s[4, 0, 0, 0]) == (1.0, 3.0, 10.0)
    assert s[0, 1, 0, 0] == np.float32(29.0 / 5) and p[0, 0, 0] == np.float32(0.4) and p[1, 0, 0] == np.float32(0.4)
    assert (m[0, 0, 0, 0], m[1, 0, 0, 0], m[0, 1, 0, 0], m[1, 1, 0, 0]) == (1.5, np.float32(17 / 3), 7.0, 5.0)
    assert s.shape == (5, 2, 1, 2) and m.shape == (2, 2, 1, 2) and (s[:, :, 0, 1] == 0).all()
    b[1, 1, 0, 1] = np.nan
    s, p, m = multi_stats_ref.multi_source_stats([a, b], [[2, 0], [1, 0]], (0.5,), [(0, 0.0)])
    assert np.isnan(s[:, 0, 0, 1]).all() and np.isnan(p[0, 0, 1]) and np.isnan(m[1, 0, 0, 1]) and m[0, 0, 0, 1] == 0.0
