"""sky_ensemble_stats on the device: against the fp64 oracle, edge cases, invariances, bounds, refusals, and
predict_ensemble end to end for the three models."""
import ctypes as C
import datetime

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from oracle import ens_stats_ref  # noqa: E402

Q = (0.0, 0.1, 0.5, 0.9, 1.0)


@pytest.fixture(autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def stats(x, channels=None, quantiles=(), events=(), channel_offset=0, out=None):
    from skyrim_b200.engine import ensemble_statistics
    s, p = ensemble_statistics(x, channels, quantiles, events, channel_offset, out)
    torch.cuda.synchronize()
    return s.cpu().numpy(), p.cpu().numpy()


def assert_ulp(got, want, n=1):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    g, w = got[ok], want[ok]
    tol = n * np.spacing(np.maximum(np.abs(g), np.abs(w))).astype(np.float64)
    d = np.abs(g.astype(np.float64) - w)
    assert (d <= tol).all(), f"max {np.max(d / np.maximum(tol, 1e-300)):.2f} ulp"


def _events(x):
    """nondecreasing channel indices; thresholds that include member values (equality must not count)"""
    return [(0, 0.0), (0, float(x[0, 0, 5, 5])), (3, float(x[1 % x.shape[0], 3, 7, 8])), (3, 1.0), (68, -1.0),
            (68, float(np.median(x[:, 68])))]


@pytest.mark.parametrize("kind", ["random", "large_mean"])
@pytest.mark.parametrize("M", [1, 2, 3, 5, 8, 17, 33, 64])
def test_kernel_matches_oracle(M, kind):
    rng = np.random.default_rng(M)
    shape = (M, 69, 41, 96)
    if kind == "random":
        x = (rng.standard_normal(shape) * 10).astype(np.float32)
    else:   # de-normalised geopotential-like field: 5e4 +- 0.5
        x = (5e4 + rng.uniform(-0.5, 0.5, shape)).astype(np.float32)
    ev = _events(x)
    s, p = stats(torch.from_numpy(x).cuda(), None, Q, ev)
    ws, wp = ens_stats_ref.ensemble_stats(x, range(69), Q, ev)
    assert_ulp(s, ws)
    np.testing.assert_array_equal(p, wp)


def test_full_size_subset():
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn((4, 69, 721, 1440), device="cuda", generator=g) * 3 + 7
    sel, q = [68, 2, 30, 5], (0.1, 0.5, 0.9)
    ev = [(0, 7.0), (1, 6.0), (1, 9.5), (3, 0.0)]
    s, p = stats(x, sel, q, ev)
    assert s.shape == (5, 4, 721, 1440) and p.shape == (4, 721, 1440)
    ws, wp = ens_stats_ref.ensemble_stats(x[:, sel].cpu().numpy(), range(4), q, ev)
    assert_ulp(s, ws)
    np.testing.assert_array_equal(p, wp)


def test_edge_cases():
    rng = np.random.default_rng(0)
    one = rng.standard_normal((1, 3, 41, 96)).astype(np.float32)
    s, p = stats(torch.from_numpy(one).cuda(), None, Q, [(1, 0.0)])
    assert (s[1] == 0).all()
    for k in [0] + list(range(2, 2 + len(Q))):
        np.testing.assert_array_equal(s[k], one[0])
    for M in (5, 17, 33):
        same = np.repeat(one, M, axis=0)
        s, _ = stats(torch.from_numpy(same).cuda(), None, (0.3,))
        assert (s[1] == 0).all()
        np.testing.assert_array_equal(s[0], one[0])
        np.testing.assert_array_equal(s[2], one[0])
    # a threshold equal to a member value is not counted
    x = np.zeros((3, 1, 2, 64), np.float32)
    x[:, 0] = np.array([1.0, 2.0, 3.0], np.float32)[:, None, None]
    _, p = stats(torch.from_numpy(x).cuda(), None, (), [(0, 2.0), (0, 3.0), (0, 0.5)])
    assert (p[0] == np.float32(1 / 3)).all() and (p[1] == 0).all() and (p[2] == 1).all()
    # NaN at one (member, channel, point): every output there is NaN, nothing else changes
    x = rng.standard_normal((6, 4, 41, 96)).astype(np.float32)
    ev = [(0, 0.0), (2, 0.0), (2, 1.0)]
    clean_s, clean_p = stats(torch.from_numpy(x).cuda(), None, (0.5, 0.9), ev)
    x[4, 2, 10, 20] = np.nan
    s, p = stats(torch.from_numpy(x).cuda(), None, (0.5, 0.9), ev)
    assert np.isnan(s[:, 2, 10, 20]).all() and np.isnan(p[1:, 10, 20]).all()
    s[:, 2, 10, 20] = clean_s[:, 2, 10, 20]
    p[1:, 10, 20] = clean_p[1:, 10, 20]
    np.testing.assert_array_equal(s, clean_s)
    np.testing.assert_array_equal(p, clean_p)


def test_channel_alone_and_member_permutation():
    rng = np.random.default_rng(3)
    x = torch.from_numpy((rng.standard_normal((9, 69, 41, 96)) * 5 + 2).astype(np.float32)).cuda()
    ev = [(0, 2.0), (7, 0.0), (68, 3.0)]
    s_all, p_all = stats(x, None, Q, ev)
    for c, e in ((0, 0), (7, 1), (68, 2)):
        s, p = stats(x, [c], Q, [(0, ev[e][1])])
        np.testing.assert_array_equal(s[:, 0], s_all[:, c])
        np.testing.assert_array_equal(p[0], p_all[e])
    perm = torch.from_numpy(rng.permutation(9)).cuda()
    s, p = stats(x[perm].contiguous(), None, Q, ev)
    np.testing.assert_array_equal(s[2:], s_all[2:])
    np.testing.assert_array_equal(p, p_all)
    assert_ulp(s[:2], s_all[:2])


def test_strided_graphcast_slice_equals_contiguous_copy():
    rng = np.random.default_rng(4)
    x = torch.from_numpy(rng.standard_normal((5, 166, 41, 96)).astype(np.float32)).cuda()
    sel, ev = [0, 40, 82], [(1, 0.5), (2, -0.5)]
    want = stats(x[:, 83:].contiguous(), sel, (0.25, 0.75), ev)
    for got in (stats(x, sel, (0.25, 0.75), ev, channel_offset=83), stats(x[:, 83:], sel, (0.25, 0.75), ev)):
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[1], want[1])


def test_no_writes_out_of_bounds():
    rng = np.random.default_rng(5)
    x = torch.from_numpy(rng.standard_normal((7, 5, 41, 96)).astype(np.float32)).cuda()
    pad, plane = 4096, 41 * 96
    shapes = ((2 + 3, 2, 41, 96), (3, 41, 96))
    bufs = [torch.full((int(np.prod(s)) + 2 * pad,), float("nan"), device="cuda") for s in shapes]
    out = tuple(b[pad:-pad].view(s) for b, s in zip(bufs, shapes))
    s, p = stats(x, [4, 1], (0.1, 0.5, 0.9), [(0, 0.0), (1, 0.0), (1, 1.0)], out=out)
    assert np.isfinite(s).all() and np.isfinite(p).all() and plane % 128 != 0
    for b in bufs:
        h = b.cpu().numpy()
        assert np.isnan(h[:pad]).all() and np.isnan(h[-pad:]).all()


def test_refusals_launch_nothing():
    from skyrim_b200 import _ffi
    from skyrim_b200.engine import ensemble_statistics, launch_count
    L = _ffi.lib()
    x = torch.zeros((4, 3, 41, 96), device="cuda")
    st, pr = torch.empty((3, 3, 41, 96), device="cuda"), torch.empty((1, 41, 96), device="cuda")
    hx, hs, hp = np.zeros(x.numel(), np.float32), np.zeros(st.numel(), np.float32), np.zeros(pr.numel(), np.float32)
    plane = 41 * 96

    def call(xp=x.data_ptr(), sp=st.data_ptr(), pp=pr.data_ptr(), members=4, stride=3 * plane, chans=(0, 1, 2), q=(0.5,),
             ev=(1,), thr=(0.0,)):
        return L.sky_ensemble_stats(xp, members, stride, plane, 3, (C.c_int32 * 3)(*chans), len(chans),
                                    (C.c_double * 1)(*q), len(q), (C.c_int32 * 1)(*ev), (C.c_float * 1)(*thr), len(ev), sp,
                                    pp, torch.cuda.current_stream().cuda_stream)
    n0 = launch_count()
    assert call() == 0
    torch.cuda.synchronize()
    assert launch_count() == n0 + 1
    n0 = launch_count()
    for kw in (dict(xp=hx.ctypes.data), dict(sp=hs.ctypes.data), dict(pp=hp.ctypes.data), dict(members=65),
               dict(stride=3 * plane - 1), dict(chans=(0, 1, 3)), dict(q=(1.01,)), dict(ev=(3,)), dict(thr=(float("nan"),))):
        assert call(**kw) == -1, kw
    for bad in (dict(quantiles=(2.0,)), dict(channels=[7]), dict(events=[(1, 0.0), (0, 0.0)])):
        with pytest.raises(_ffi.SkyError):
            ensemble_statistics(x, **bad)
    with pytest.raises(ValueError):
        ensemble_statistics(x.cpu())
    with pytest.raises(ValueError):
        ensemble_statistics(x.transpose(2, 3))
    assert launch_count() == n0


def test_host_pointer_refusal_message():
    from skyrim_b200 import _ffi
    L = _ffi.lib()
    x = torch.zeros((2, 1, 4, 32), device="cuda")
    h = np.zeros(2 * 128, np.float32)
    one = (C.c_int32 * 1)(0)
    rc = L.sky_ensemble_stats(x.data_ptr(), 2, 128, 128, 1, one, 1, None, 0, None, None, 0, h.ctypes.data, None, None)
    assert rc == -1 and "stats must be device memory" in L.sky_last_error().decode()


# ---- end to end ------------------------------------------------------------------------------------------------------------
def _expected_events(names, events):
    return [(i, t) for i, c in enumerate(names) for t in np.atleast_1d(events.get(c, ()))]


def test_pangu_predict_ensemble_end_to_end(tmp_path):
    from skyrim_b200 import xr_shim as xr
    from skyrim_b200.config import PANGU_CHANNELS, pangu_small
    from skyrim_b200.core import Skyrim
    from skyrim_b200.engine import ensemble_statistics
    from skyrim_b200.ensemble import EnsembleRunner
    from skyrim_b200.weights import channel_stats, synthetic_state
    q, events = (0.1, 0.5, 0.9), {"t2m": [280.0, 290.0], "u10m": [2.0]}
    sk = Skyrim("pangu", cfg=pangu_small(41, 96))
    pred, paths = sk.predict_ensemble("20240507", "0000", lead_time=18, members=4, quantiles=q, events=events, save=True,
                                      save_config=dict(output_dir=str(tmp_path)))
    assert len(paths) == 6 and pred.channels == PANGU_CHANNELS and pred.statistics == ["mean", "spread", "q0.1", "q0.5", "q0.9"]
    assert list(np.asarray(pred.stats.coords["time"])) == [np.datetime64("2024-05-07T12:00:00"), np.datetime64("2024-05-07T18:00:00")]
    ev = _expected_events(PANGU_CHANNELS, events)
    eng = sk.model.model.engine
    base, sig = synthetic_state(PANGU_CHANNELS, 41, 96, 0), channel_stats(PANGU_CHANNELS)[1]

    def runner():
        return EnsembleRunner(eng, base, sig, members_per_gpu=4, rank=0, amp=0.05, seed=0, perturbation="spherical_grf",
                              grf=dict(lmax=20))
    plain, run = [], runner()
    for n in range(4):
        if n:
            run.step()
        s, p = ensemble_statistics(run.x, None, q, ev)
        plain.append((s.cpu().numpy(), p.cpu().numpy()))
        if n == 3:
            members = run.x.cpu().numpy()
    for k, n in enumerate((2, 3)):
        np.testing.assert_array_equal(pred.stats.values[k], plain[n][0])
        np.testing.assert_array_equal(pred.probability.values[k], plain[n][1])
    ws, wp = ens_stats_ref.ensemble_stats(members, range(69), q, ev)
    assert_ulp(pred.stats.values[1], ws)
    np.testing.assert_array_equal(pred.probability.values[1], wp)
    over = [(n, s.numpy().copy(), p.numpy().copy()) for n, s, p in runner().iter_stats(3, None, q, ev)]
    assert [o[0] for o in over] == [0, 1, 2, 3]
    for (_, s, p), (ps, pp) in zip(over, plain):
        np.testing.assert_array_equal(s, ps)
        np.testing.assert_array_equal(p, pp)
    back_s, back_p = xr.open_dataarray(paths[-2]), xr.open_dataarray(paths[-1])
    np.testing.assert_array_equal(back_s.values, pred.stats.values)
    np.testing.assert_array_equal(back_p.values, pred.probability.values)
    assert list(back_p.coords["event"]) == pred.events
    assert pred.probability_of("t2m", 280.0).shape == (41, 96)
    sk.model.release_model()


def test_sfno_predict_ensemble_matches_hand_driven_runner():
    from skyrim_b200.config import FCNV2_CHANNELS, sfno_small
    from skyrim_b200.core import Skyrim
    from skyrim_b200.engine import ensemble_statistics
    from skyrim_b200.ensemble import EnsembleRunner
    from skyrim_b200.weights import channel_stats, synthetic_state
    sk = Skyrim("fourcastnet_v2", cfg=sfno_small(49, 96, embed=64, layers=3))
    pred, _ = sk.predict_ensemble("20240507", "0600", lead_time=6, members=3, quantiles=(0.5,), events={"t2m": 280.0},
                                  channels=["t2m", "z500"])
    assert pred.channels == [c for c in FCNV2_CHANNELS if c in ("t2m", "z500")]
    sel = [FCNV2_CHANNELS.index(c) for c in pred.channels]
    run = EnsembleRunner(sk.model.model.engine, synthetic_state(FCNV2_CHANNELS, 49, 96, 0), channel_stats(FCNV2_CHANNELS)[1],
                         members_per_gpu=3, perturbation="spherical_grf", grf=dict(lmax=24))
    run.step()
    s, p = ensemble_statistics(run.x, sel, (0.5,), [(pred.channels.index("t2m"), 280.0)])
    np.testing.assert_array_equal(pred.stats.values[1], s.cpu().numpy())
    np.testing.assert_array_equal(pred.probability.values[1], p.cpu().numpy())
    assert float(pred.stats.values[1, 1].mean()) > 0
    sk.model.release_model()


def test_graphcast_predict_ensemble_reduces_the_new_slice():
    from skyrim_b200.config import GRAPHCAST_CHANNELS, graphcast_small
    from skyrim_b200.core import Skyrim
    from skyrim_b200.ensemble import EnsembleRunner
    sk = Skyrim("graphcast", cfg=graphcast_small(41, 96, 2, 512, 2))
    pred, _ = sk.predict_ensemble("20240507", "0000", lead_time=12, members=3, quantiles=(0.1, 0.9), events={"t2m": 280.0})
    assert pred.channels == GRAPHCAST_CHANNELS
    gm = sk.model
    base, sigma, offset = gm._ensemble_initial_state(datetime.datetime(2024, 5, 7))   # sets the engine's clock
    assert offset == 83 and tuple(base.shape) == (166, 41, 96) and sigma[82] == 0 and sigma[165] == 0
    run = EnsembleRunner(gm.model.engine, base, sigma, members_per_gpu=3, perturbation="spherical_grf", grf=dict(lmax=20))
    run.step(2)
    members = run.x[:, 83:].cpu().numpy()
    ev = _expected_events(GRAPHCAST_CHANNELS, {"t2m": 280.0})
    ws, wp = ens_stats_ref.ensemble_stats(members, range(83), (0.1, 0.9), ev)
    assert_ulp(pred.stats.values[1], ws)
    np.testing.assert_array_equal(pred.probability.values[1], wp)
    # the forcing channel is not perturbed and is recomputed per step: identical in every member
    assert (pred.stats.values[1, 1, GRAPHCAST_CHANNELS.index("tp06")] == 0).all()
    assert float(pred.stats.values[1, 1, GRAPHCAST_CHANNELS.index("t2m")].mean()) > 0
    gm.release_model()
