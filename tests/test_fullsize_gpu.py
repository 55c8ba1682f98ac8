"""Full-size (BASELINE.json shape, 721x1440) GPU tests.

Oracle parity at full size: the CUDA step against the committed sampled fixture of ONE real oracle step
(tests/golden/{pangu,sfno,graphcast}_721x1440_seed0.npz, tools/make_golden_full.py: point sample, 48x48 block means
over every pixel, last latitude row, per-channel norms).  Tolerance is the north star's: per-channel relative
L2 error <= 1e-3; the block means / normalised errors are bounded in units of the channel's standard deviation.
Mid-size grids with more tiles than SMs are compared with the oracle evaluated in the test (persistent-loop
coverage: ring phase wrap, accumulator staging over the ring, several tiles per CTA).  Then size-independent properties."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pangu_full_engine():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from skyrim_b200.config import PANGU_CHANNELS, pangu_full
    from skyrim_b200.engine import StepEngine
    from skyrim_b200.weights import make_pangu_weights, synthetic_state
    cfg = pangu_full()
    w = make_pangu_weights(cfg, 0)
    w["const.masks"] = np.zeros_like(w["const.masks"])   # constant fields would break the longitude symmetry
    eng = StepEngine(cfg, 0)
    eng.load_weights(w)
    x0 = torch.from_numpy(synthetic_state(PANGU_CHANNELS, cfg.nlat, cfg.nlon, 0))[None].cuda()
    yield cfg, w, eng, x0
    eng.close()


TOL = 1e-3          # per-channel relative L2 (north star)
TOL_SIGMA = 5e-3    # point-sample RMS error and 48x48 block-mean error, in channel standard deviations


def _report(tag, c):
    from skyrim_b200.verify import summarise
    s = summarise(c)
    print(f"\n[{tag} 721x1440 vs oracle fixture] max per-channel: rel {s['rel']:.3e}  nrm {s['nrm']:.3e}  "
          f"block {s['block']:.3e}  last-row {s['last']:.3e}  norm {s['norm']:.3e}")
    return s


def test_pangu_full_size_oracle_parity():
    """One CUDA step at the BASELINE shape against the oracle's step on the same seeded weights and IC."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from skyrim_b200.config import PANGU_CHANNELS, pangu_full
    from skyrim_b200.engine import StepEngine
    from skyrim_b200.verify import compare_fullsize, load_fixture
    from skyrim_b200.weights import make_pangu_weights, synthetic_state
    fx = load_fixture("pangu")
    cfg = pangu_full()
    x0 = synthetic_state(PANGU_CHANNELS, cfg.nlat, cfg.nlon, 0)
    np.testing.assert_array_equal(x0[:, ::64, ::64], fx["x0_sample"])     # same IC as the oracle run
    eng = StepEngine(cfg, 0)
    eng.load_weights(make_pangu_weights(cfg, 0))
    y = eng.step(torch.from_numpy(x0)[None].cuda())[0]
    s = _report("pangu", compare_fullsize(y, fx))
    eng.close()
    assert s["finite"] and s["rel"] < TOL and s["norm"] < TOL, s
    assert s["nrm"] < TOL_SIGMA and s["block"] < TOL_SIGMA and s["last"] < 4 * TOL_SIGMA, s


def test_sfno_full_size_oracle_parity():
    """FourCastNet-v2 SFNO (E=384, L=8) at 721x1440 against the oracle fixture."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from skyrim_b200.config import FCNV2_CHANNELS, sfno_full
    from skyrim_b200.engine import StepEngine
    from skyrim_b200.verify import compare_fullsize, load_fixture
    from skyrim_b200.weights import make_sfno_weights, sfno_tables, synthetic_state
    fx = load_fixture("sfno")
    cfg = sfno_full()
    x0 = synthetic_state(FCNV2_CHANNELS, cfg.nlat, cfg.nlon, 0)
    np.testing.assert_array_equal(x0[:, ::64, ::64], fx["x0_sample"])
    w = dict(make_sfno_weights(cfg, 0)); w.update(sfno_tables(cfg))
    eng = StepEngine(cfg, 0)
    eng.load_weights(w)
    del w
    y = eng.step(torch.from_numpy(x0)[None].cuda())[0]
    s = _report("sfno", compare_fullsize(y, fx))
    eng.close()
    assert s["finite"] and s["rel"] < TOL and s["norm"] < TOL, s
    assert s["nrm"] < TOL_SIGMA and s["block"] < TOL_SIGMA and s["last"] < 4 * TOL_SIGMA, s


def test_graphcast_full_size_oracle_parity():
    """BASELINE config 4's step: GraphCast on the 0.25 deg grid with the refinement-6 multimesh (40,962 nodes, 327,660 mesh
    edges, 1.63 M grid2mesh and 3.11 M mesh2grid edges, 16 layers) against ONE real oracle step (135 s on 8 host threads),
    for the stepped state (north-star tolerance) and for the network's tendency itself."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from skyrim_b200.config import graphcast_full
    from skyrim_b200.engine import StepEngine
    from skyrim_b200.timeloop import GraphcastTimeLoop
    from skyrim_b200.verify import compare_graphcast, load_fixture
    from skyrim_b200.weights import make_graphcast_weights, synthetic_graphcast_state
    cfg = graphcast_full()
    w = make_graphcast_weights(cfg, 0)
    eng = StepEngine(cfg, 0)
    eng.load_weights(w)
    fx = load_fixture("graphcast")
    t0 = float(fx["t0"])
    x = torch.from_numpy(synthetic_graphcast_state(cfg, 0)).reshape(1, 2, cfg.n_state, cfg.nlat, cfg.nlon).cuda()
    GraphcastTimeLoop(eng).fill_forcing(x, t0)
    x = x.reshape(1, 2 * cfg.n_state, cfg.nlat, cfg.nlon).contiguous()
    xs, ref = x[0, :, ::64, ::64].cpu().numpy(), fx["x0_sample"]
    forcing = [cfg.n_state - 1, 2 * cfg.n_state - 1]        # toa radiation: fp32 CUDA formula here, fp64 numpy in the fixture
    prog = [c for c in range(2 * cfg.n_state) if c not in forcing]
    assert np.array_equal(xs[prog], ref[prog]), "seeded IC differs from the fixture's"
    assert np.abs(xs[forcing] - ref[forcing]).max() <= 2e-5 * ref[forcing].max(), "toa forcing differs from the fixture's"
    eng.set_clock(t0)
    y = eng.step(x)
    s = compare_graphcast(y[0], x[0], w["norm.diff_std"], fx, cfg)
    print(f"\n[graphcast 721x1440 vs oracle fixture] state: rel {s['rel']:.3e} nrm {s['nrm']:.3e} block {s['block']:.3e} last {s['last']:.3e} "
          f"norm {s['norm']:.3e}; tendency: rel {s['t_rel']:.3e} block {s['t_block']:.3e} norm {s['t_norm']:.3e}")
    assert s["finite"] and s["slice0_is_old_slice1"]
    assert s["rel"] < TOL and s["norm"] < TOL and s["nrm"] < TOL_SIGMA and s["block"] < TOL_SIGMA and s["last"] < TOL_SIGMA
    assert s["t_rel"] < 4e-3 and s["t_norm"] < 2e-3, "tendency (network output) error (measured 1.4e-3 / 5.1e-4)"
    eng.close()


@pytest.mark.parametrize("nlat,nlon", [(181, 480), (121, 384)])
def test_pangu_mid_size_parity_more_tiles_than_sms(nlat, nlon):
    """181x480: 43,200 / 10,800 tokens = 338 / 85 row tiles, 1,014 QKV tiles on 132 SMs
    -> every persistent loop runs several tiles per CTA; compared with the oracle evaluated here."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle.pangu_ref import PanguRef, rel_err_per_channel
    from skyrim_b200.config import PANGU_CHANNELS, pangu_small
    from skyrim_b200.engine import StepEngine
    from skyrim_b200.weights import make_pangu_weights, synthetic_state
    cfg = pangu_small(nlat, nlon)
    w = make_pangu_weights(cfg, 2)
    x0 = synthetic_state(PANGU_CHANNELS, nlat, nlon, 4)
    eng = StepEngine(cfg, 0)
    eng.load_weights(w)
    y = eng.step(torch.from_numpy(x0)[None].cuda())[0].cpu().numpy()
    y2 = eng.step(torch.from_numpy(np.stack([x0, x0[:, ::-1].copy()])).cuda())[0].cpu().numpy()   # 2 stacked members
    eng.close()
    ref = PanguRef(cfg, w).step(x0).numpy()
    e = rel_err_per_channel(y, ref)
    print(f"\n[pangu {nlat}x{nlon}] max per-channel rel err {e.max():.3e}")
    assert np.isfinite(y).all() and e.max() < TOL, e.max()
    assert np.array_equal(y, y2)


def test_sfno_mid_size_parity_more_tiles_than_sms():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle.pangu_ref import rel_err_per_channel
    from oracle.sfno_ref import SFNORef
    from skyrim_b200.config import FCNV2_CHANNELS, sfno_small
    from skyrim_b200.engine import StepEngine
    from skyrim_b200.weights import make_sfno_weights, sfno_tables, synthetic_state
    cfg = sfno_small(241, 480, embed=128, layers=2)     # 115,680 pixels = 904 row tiles
    w = make_sfno_weights(cfg, 3)
    x0 = synthetic_state(FCNV2_CHANNELS, cfg.nlat, cfg.nlon, 1)
    allw = dict(w); allw.update(sfno_tables(cfg))
    eng = StepEngine(cfg, 0)
    eng.load_weights(allw)
    y = eng.step(torch.from_numpy(x0)[None].cuda())[0].cpu().numpy()
    eng.close()
    e = rel_err_per_channel(y, SFNORef(cfg, w).step(x0).numpy())
    print(f"\n[sfno 241x480 E128 L2] max per-channel rel err {e.max():.3e}")
    assert np.isfinite(y).all() and e.max() < TOL, e.max()


def test_pangu_full_size_finite_and_in_climatological_range(pangu_full_engine):
    cfg, w, eng, x0 = pangu_full_engine
    y = eng.step(x0)
    assert bool(torch.isfinite(y).all())
    z = (y[0] - torch.from_numpy(w["norm.mean"]).cuda()[:, None, None]) / torch.from_numpy(w["norm.std"]).cuda()[:, None, None]
    assert 0.2 < float(z.std()) < 5.0 and float(z.abs().max()) < 50.0


def test_pangu_full_size_longitude_periodicity(pangu_full_engine):
    """No mask along W (longitude is periodic): rolling the input by one coarse-window span
    (12 tokens x 2 (merge) x 4 (patch) = 96 grid columns) rolls the output by the same amount."""
    cfg, w, eng, x0 = pangu_full_engine
    y0 = eng.step(x0).clone()
    y1 = eng.step(torch.roll(x0, 96, dims=-1).contiguous())
    d = (torch.roll(y0, 96, dims=-1) - y1).abs().amax(dim=(0, 2, 3)) / torch.from_numpy(w["norm.std"]).cuda()
    assert float(d.max()) < 1e-4, float(d.max())
    y2 = eng.step(torch.roll(x0, 40, dims=-1).contiguous())   # not a window multiple: must differ
    d2 = (torch.roll(y0, 40, dims=-1) - y2).abs().amax(dim=(0, 2, 3)) / torch.from_numpy(w["norm.std"]).cuda()
    assert float(d2.max()) > 1e-3


def test_pangu_full_size_members_are_independent(pangu_full_engine):
    cfg, w, eng, x0 = pangu_full_engine
    xb = torch.cat([x0, torch.roll(x0, 7, dims=-2)]).contiguous()
    yb = eng.step(xb).clone()
    for m in range(2):
        ys = eng.step(xb[m:m + 1].contiguous())
        assert torch.equal(ys[0], yb[m]), m


def test_pangu_full_size_rollout_stays_bounded(pangu_full_engine):
    cfg, w, eng, x0 = pangu_full_engine
    x = x0
    sd = torch.from_numpy(w["norm.std"]).cuda()[:, None, None]
    mu = torch.from_numpy(w["norm.mean"]).cuda()[:, None, None]
    for _ in range(8):
        x = eng.step(x)
    z = (x[0] - mu) / sd
    assert bool(torch.isfinite(x).all()) and 0.2 < float(z.std()) < 5.0
