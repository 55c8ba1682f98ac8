"""Multi-model ensembles on the GPU: sky_ensemble_stats_multi against the fp64 oracle and against sky_ensemble_stats, and
Pangu + FourCastNet-v2 + GraphCast side by side on one 49x96 grid (predict, predict_ensemble, forecast) against the
single-model paths."""
import datetime

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from oracle import multi_stats_ref  # noqa: E402
from skyrim_b200 import xr_shim as xr  # noqa: E402
from skyrim_b200._ffi import SkyError  # noqa: E402
from skyrim_b200.config import graphcast_small, pangu_small, sfno_small  # noqa: E402
from skyrim_b200.engine import ensemble_statistics, multi_model_statistics  # noqa: E402

T0 = datetime.datetime(2024, 5, 7)
H, W = 49, 96


def within_ulp(got, want, n=1):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    same_nan = np.isnan(got) == np.isnan(want)
    tol = n * np.spacing(np.maximum(np.abs(got), np.abs(want)))
    ok = np.isnan(got) | (np.abs(got.astype(np.float64) - want.astype(np.float64)) <= tol)
    return bool(same_nan.all() and ok.all())


def make_sources(Ms, counts, pad=0, gc_slice=None, seed=0):
    """device sources (M_k, C_k, H, W); ``pad`` extra planes per member (a free member stride); source ``gc_slice`` is
    the second half of a (M, 2, C, H, W) two-slice state, as a GraphCast state is reduced"""
    g = torch.Generator().manual_seed(seed)
    out = []
    for k, (M, Cn) in enumerate(zip(Ms, counts)):
        if k == gc_slice:
            full = (torch.randn(M, 2 * Cn, H, W, generator=g) * 3 + 10 * k).cuda()
            out.append(full[:, Cn:])
        else:
            full = (torch.randn(M, Cn + pad, H, W, generator=g) * 3 + 10 * k).cuda()
            out.append(full[:, :Cn])
    return out


@pytest.mark.parametrize("Ms, counts, pad, gc", [
    ((5,), (7,), 0, None), ((3, 4), (7, 9), 2, None), ((4, 4, 4), (69, 73, 83), 0, 2), ((1, 1, 1), (7, 8, 9), 0, 2),
    ((16, 16, 16, 16), (6, 7, 8, 9), 1, 1), ((20, 30), (6, 9), 0, 0), ((1, 63), (5, 6), 3, None),
])
def test_kernel_against_oracle(Ms, counts, pad, gc):
    srcs = make_sources(Ms, counts, pad, gc)
    rng = np.random.default_rng(len(Ms))
    chans = [list(rng.permutation(c)[:5]) for c in counts]
    q, ev = (0.0, 0.1, 0.5, 0.9, 1.0), [(0, 1.0), (2, 11.0), (2, 12.0), (4, 25.0)]
    s, p, m = multi_model_statistics(srcs, chans, q, ev)
    ws, wp, wm = multi_stats_ref.multi_source_stats([x.cpu().numpy() for x in srcs], chans, q, ev)
    torch.cuda.synchronize()
    assert within_ulp(s.cpu().numpy(), ws) and within_ulp(m.cpu().numpy(), wm)
    np.testing.assert_array_equal(p.cpu().numpy(), wp)


@pytest.mark.parametrize("M, q", [(1, ()), (7, (0.25, 0.75)), (16, (0.5,)), (33, (0.1, 0.9)), (64, ())])
def test_one_source_is_bitwise_sky_ensemble_stats(M, q):
    (x,) = make_sources((M,), (9,), pad=2, seed=M)
    chans, ev = [8, 0, 3], [(0, 2.0), (1, 1.0)]
    s, p, m = multi_model_statistics([x], [chans], q, ev)
    s1, p1 = ensemble_statistics(x, chans, q, ev)
    assert torch.equal(s, s1) and torch.equal(p, p1) and torch.equal(m[0], s1[0])


def test_source_means_are_bitwise_the_single_source_means_and_selection_does_not_matter():
    srcs = make_sources((3, 5, 2), (7, 8, 9), 0, 2, seed=5)
    chans = [[0, 1, 2, 3], [4, 5, 6, 7], [8, 7, 6, 5]]
    s, p, m = multi_model_statistics(srcs, chans, (0.3,), [(1, 12.0)])
    for k, x in enumerate(srcs):
        assert torch.equal(m[k], ensemble_statistics(x, chans[k])[0][0])
    sub = [[c[1], c[3]] for c in chans]
    s2, p2, m2 = multi_model_statistics(srcs, sub, (0.3,), [(0, 12.0)])
    assert torch.equal(s2, s[:, [1, 3]]) and torch.equal(m2, m[:, [1, 3]]) and torch.equal(p2, p)
    s3, p3, m3 = multi_model_statistics(srcs, chans, (0.3,), [(1, 12.0)], source_means=False)
    assert m3 is None and torch.equal(s3, s) and torch.equal(p3, p)


def test_nan_in_a_member():
    srcs = make_sources((3, 4), (5, 6), seed=9)
    srcs[1][2, 4, 10, 20] = float("nan")
    s, p, m = multi_model_statistics(srcs, [[0, 1], [3, 4]], (0.5,), [(1, 0.0)])
    s, p, m = s.cpu().numpy(), p.cpu().numpy(), m.cpu().numpy()
    assert np.isnan(s[:, 1, 10, 20]).all() and np.isnan(p[0, 10, 20]) and np.isnan(m[1, 1, 10, 20])
    assert np.isfinite(m[0, 1, 10, 20]) and np.isfinite(s[:, 0]).all() and np.isfinite(s[:, 1, 10, 21]).all()


def test_refusals_on_the_device():
    import ctypes as C
    from skyrim_b200 import _ffi
    srcs = make_sources((2, 2), (5, 5))
    host = srcs[1].cpu().pin_memory()
    out = torch.empty(2, 1, H, W, device="cuda")
    arr = lambda ct, v: (ct * len(v))(*v)  # noqa: E731
    L = _ffi.lib()
    for xs, stats in (([srcs[0].data_ptr(), host.data_ptr()], out.data_ptr()), ([srcs[0].data_ptr()] * 2, host.data_ptr())):
        rc = L.sky_ensemble_stats_multi(2, arr(C.c_void_p, xs), arr(C.c_int32, [2, 2]), arr(C.c_int64, [5 * H * W] * 2),
                                        arr(C.c_int32, [5, 5]), arr(C.c_int32, [0, 0]), 1, H * W, None, 0, None, None, 0,
                                        stats, None, None, None)
        assert rc == -1 and "device memory" in L.sky_last_error().decode()
    with pytest.raises(ValueError):
        multi_model_statistics([srcs[0], host], [[0], [0]])
    with pytest.raises(SkyError, match="total members"):
        multi_model_statistics(make_sources((40, 25), (2, 2)), [[0], [0]])
    with pytest.raises(ValueError):
        multi_model_statistics(srcs, [[0], [0, 1]])
    with pytest.raises(ValueError):
        multi_model_statistics(srcs * 3, [[0]] * 6)


# ---- three models side by side ---------------------------------------------------------------------------------------
CFG = dict(pangu=dict(cfg=pangu_small(H, W)), fourcastnet_v2=dict(cfg=sfno_small(H, W, 64, 3)),
           graphcast=dict(cfg=graphcast_small(H, W, 2, 512, 2)))
NAMES = ("pangu", "fourcastnet_v2", "graphcast")


@pytest.fixture(scope="module")
def trio():
    from skyrim_b200.core.skyrim import Skyrim
    sk = Skyrim(*NAMES, **CFG)
    yield sk
    sk.model.release_model()


def test_predict_matches_each_model_alone_and_the_oracle_mean(trio, tmp_path):
    from skyrim_b200.core.models.ensemble import SourceView
    from skyrim_b200.core.skyrim import Skyrim
    ens = trio.model
    pred, paths = trio.predict("20240507", "0000", lead_time=12, save=True, save_config=dict(output_dir=str(tmp_path)))
    states = []
    for name in NAMES:
        single = Skyrim(name, ic_source=SourceView(ens.data_source, ens.models[NAMES.index(name)].in_channel_names),
                        **CFG[name])
        want, _ = single.model.rollout(T0, 2, save=True, save_config=dict(output_dir=str(tmp_path / "alone")))
        single.model.release_model()
        got = ens.model_predictions[name]
        np.testing.assert_array_equal(got.values, want.values)
        assert list(got.coords["channel"]) == list(want.coords["channel"])
        states.append(want.values)
    chans = ens._shared_index(ens.shared_channels)
    for t in range(2):
        ref = multi_stats_ref.multi_source_stats([s[t][None] for s in states], chans)[0][0]
        assert within_ulp(pred.prediction.values[t], ref)
    assert list(pred.prediction.coords["channel"]) == ens.shared_channels and len(ens.shared_channels) == 56
    assert len(paths) == 2 and all("fourcastnet_v2_graphcast_pangu__" in p for p in paths)
    np.testing.assert_array_equal(xr.open_dataarray(paths[-1]).values, pred.prediction.values)
    for name in NAMES:
        assert len(ens.model_paths[name]) == 2 and f"/{name}__" in ens.model_paths[name][0]
        np.testing.assert_array_equal(xr.open_dataarray(ens.model_paths[name][-1]).values, ens.model_predictions[name].values)


def test_predict_ensemble_against_members_stepped_by_hand(trio, tmp_path):
    from skyrim_b200.ensemble import EnsembleRunner
    ens, M, q, seed = trio.model, 3, (0.1, 0.5, 0.9), 11
    ev = {"t2m": [280.0, 290.0], "z500": 55000.0}
    pred, paths = trio.predict_ensemble("20240507", "0000", lead_time=12, members=M, quantiles=q, events=ev, seed=seed,
                                        save=True, save_config=dict(output_dir=str(tmp_path)))
    grf = dict(lmax=(H - 1) // 2)
    states = ens.ensemble_members(T0, M, "spherical_grf", 0.05, seed, grf)
    # the first model's members are those of its own predict_ensemble
    pangu = ens.models[0]
    base, sigma, _ = pangu._ensemble_initial_state(T0)
    run = EnsembleRunner(pangu.model.engine, base, sigma, members_per_gpu=M, amp=0.05, seed=seed,
                         perturbation="spherical_grf", grf=grf)
    assert torch.equal(run.x, states[0])
    for _ in range(2):
        for k, m in enumerate(ens.models):
            states[k] = m.model.engine.step(states[k])
    outs = [x.cpu().numpy() for x in ens._outputs(states)]
    sel = pred.channels
    ev_list = [(sel.index("z500"), 55000.0)] + [(sel.index("t2m"), t) for t in ev["t2m"]]
    ev_list.sort(key=lambda e: e[0])
    ws, wp, wm = multi_stats_ref.multi_source_stats(outs, ens._shared_index(sel), q, ev_list)
    got = pred.stats.values[1]
    assert pred.statistics == ["mean", "spread", "q0.1", "q0.5", "q0.9"] + [f"mean:{n}" for n in NAMES]
    assert within_ulp(got[:5], ws) and within_ulp(got[5:], wm)
    np.testing.assert_array_equal(pred.probability.values[1], wp)
    for k, n in enumerate(NAMES):
        np.testing.assert_array_equal(pred.model_mean(n).prediction.values[1], got[5 + k])
    assert len(paths) == 4 and "fourcastnet_v2_graphcast_pangu-ens3-prob__" in paths[1]
    np.testing.assert_array_equal(xr.open_dataarray(paths[-2]).values, pred.stats.values)


def test_forecast_starts_from_the_mean_of_the_initial_conditions(trio):
    ens = trio.model
    da = trio.forecast(T0, n_steps=2, channels=["t2m", "z500"])
    assert da.shape == (3, 2, H, W)
    ics = [np.asarray(m.data_source[T0].values) for m in ens.models]
    want = multi_stats_ref.multi_source_stats([x[None] for x in ics], ens._shared_index(["t2m", "z500"]))[0][0]
    assert within_ulp(da.values[0], want)
    pred, _ = ens.rollout(T0, 2, save=False)
    np.testing.assert_array_equal(da.values[1:], pred.sel(channel=["t2m", "z500"]).values)
