"""Spherical Gaussian random field perturbation on the GPU against the fp64 oracle (oracle/grf_ref.py)."""
import numpy as np
import pytest

from oracle import grf_ref

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

FIELD_TOL = 1e-5      # max |device - fp64 oracle| of a unit-variance field (amp = sigma = 1)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _tri_index(lmax):
    """(l, m) of every entry of the m-major (m, l) triangle the library writes"""
    ls, ms = [], []
    for m in range(lmax + 1):
        ls += list(range(m, lmax + 1))
        ms += [m] * (lmax + 1 - m)
    return np.array(ls), np.array(ms)


def _device_draw(spec, seed, member0, members, channels, dev):
    """sky_grf_draw -> complex64 [members, channels, triangle] (numpy)"""
    from skyrim_b200 import _ffi
    lmax = len(spec) - 1
    T = (lmax + 1) * (lmax + 2) // 2
    s = torch.as_tensor(np.asarray(spec, np.float32), device=dev)
    out = torch.empty((members, channels, T, 2), dtype=torch.float32, device=dev)
    L = _ffi.lib()
    _ffi.check(L.sky_grf_draw(out.data_ptr(), s.data_ptr(), seed, member0, members, channels, lmax,
                              torch.cuda.current_stream(dev).cuda_stream), "sky_grf_draw", L)
    o = out.cpu().numpy()
    return o[..., 0] + 1j * o[..., 1]


def _field(nlat, nlon, lmax, seed, member0, members, channels, dev, sigma=None, amp=1.0, x=None):
    from skyrim_b200.engine import perturb_ic_grf
    if x is None:
        x = torch.zeros((members, channels, nlat, nlon), dtype=torch.float32, device=dev)
    sig = torch.ones(channels, dtype=torch.float32, device=dev) if sigma is None else sigma
    perturb_ic_grf(x, sig, amp, seed, member0=member0, lmax=lmax)
    torch.cuda.synchronize()
    return x


def test_device_coefficients_match_oracle_to_one_ulp(dev):
    from skyrim_b200.engine import grf_spectrum
    lmax = 90
    spec32 = grf_spectrum(2.0, 3.0, lmax)[0].astype(np.float32)
    got = _device_draw(spec32, 0x1234_5678_9ABC, 5, 3, 4, dev)
    ls, ms = _tri_index(lmax)
    want = grf_ref.coefficients(spec32.astype(np.float64), 0x1234_5678_9ABC, [5, 6, 7], 4)[..., ls, ms]
    for part in (np.real, np.imag):
        g, w = part(got).astype(np.float32), part(want).astype(np.float32)
        ulp = np.spacing(np.abs(w)).astype(np.float64)
        d = np.abs(g.astype(np.float64) - w.astype(np.float64))
        assert (d <= ulp).all(), d.max()
    assert (np.imag(got)[..., ms == 0] == 0).all()


@pytest.mark.parametrize("nlat, nlon, lmax, members, channels", [
    (41, 96, 20, 2, 3), (181, 360, 90, 2, 3), (721, 1440, 180, 2, 3),
])
def test_field_matches_fp64_oracle(dev, nlat, nlon, lmax, members, channels):
    seed, member0 = 77, 1
    f = _field(nlat, nlon, lmax, seed, member0, members, channels, dev).cpu().numpy().astype(np.float64)
    from skyrim_b200.engine import grf_spectrum
    spec32 = grf_spectrum(2.0, 3.0, lmax)[0].astype(np.float32).astype(np.float64)
    a = grf_ref.coefficients(spec32, seed, list(range(member0, member0 + members)), channels)
    ref = grf_ref.synthesize(a, nlat, nlon)
    err = np.abs(f - ref).max()
    print(f"GRF {nlat}x{nlon} lmax {lmax}: max |device - fp64 oracle| = {err:.3e}, field rms {np.sqrt((ref ** 2).mean()):.3f}")
    assert err <= FIELD_TOL, err
    # pole rows are bitwise constant along longitude
    for k in (0, nlat - 1):
        row = f[..., k, :]
        assert (row == row[..., :1]).all()


def test_zero_sigma_channels_and_other_members_untouched(dev):
    nlat, nlon, lmax = 41, 96, 20
    g = torch.Generator(device="cpu").manual_seed(0)
    base = torch.randn((3, 4, nlat, nlon), generator=g).to(dev)
    sig = torch.tensor([1.0, 0.0, 2.0, 0.0], device=dev)
    x = base.clone()
    # only members 1..2 are perturbed (a view of a contiguous tail is itself contiguous)
    _field(nlat, nlon, lmax, 5, 1, 2, 4, dev, sigma=sig, amp=0.5, x=x[1:])
    assert torch.equal(x[0], base[0])
    assert torch.equal(x[1:, 1], base[1:, 1]) and torch.equal(x[1:, 3], base[1:, 3])
    assert not torch.equal(x[1:, 0], base[1:, 0]) and not torch.equal(x[1:, 2], base[1:, 2])
    # channel 2 got twice channel 0's amplitude of its own field: compare with a lone sigma = 1 run of the same member
    one = _field(nlat, nlon, lmax, 5, 1, 2, 4, dev)
    d = (x[1:] - base[1:]).cpu().numpy()
    ref = one.cpu().numpy()
    np.testing.assert_allclose(d[:, 0], 0.5 * ref[:, 0], atol=2e-6)
    np.testing.assert_allclose(d[:, 2], 1.0 * ref[:, 2], atol=4e-6)


def test_member_alone_equals_member_in_batch(dev):
    nlat, nlon, lmax, C_ = 181, 360, 90, 5
    batch = _field(nlat, nlon, lmax, 3, 0, 4, C_, dev)
    solo = _field(nlat, nlon, lmax, 3, 2, 1, C_, dev)
    assert torch.equal(solo[0], batch[2])


def test_raw_draws_do_not_depend_on_lmax(dev):
    a90 = _device_draw(np.ones(91, np.float32), 42, 3, 2, 3, dev)
    a180 = _device_draw(np.ones(181, np.float32), 42, 3, 2, 3, dev)
    l90, m90 = _tri_index(90)
    l180, m180 = _tri_index(180)
    pos180 = {(l, m): i for i, (l, m) in enumerate(zip(l180, m180))}
    idx = np.array([pos180[(l, m)] for l, m in zip(l90, m90)])
    assert np.array_equal(a90, a180[..., idx])


def test_forward_sht_of_device_field_recovers_draws(dev):
    nlat, nlon, lmax = 181, 360, 90
    from skyrim_b200.engine import grf_spectrum
    spec32 = grf_spectrum(2.0, 3.0, lmax)[0].astype(np.float32)
    f = _field(nlat, nlon, lmax, 8, 0, 2, 2, dev).cpu().numpy().astype(np.float64)
    a = _device_draw(spec32, 8, 0, 2, 2, dev).astype(np.complex128)
    ls, ms = _tri_index(lmax)
    back = grf_ref.analyze(f, lmax)[..., ls, ms]
    rel = np.abs(back - a).max() / np.abs(a).max()
    print(f"forward SHT of the device field vs drawn a_lm: max rel err {rel:.3e}")
    assert rel <= 1e-5, rel


def test_per_degree_power_follows_chi_square(dev):
    """Q_l = sum over fields of |a_l0|^2 / s_l^2 + 2 sum_{m>0} |a_lm|^2 / s_l^2 = sum of F (2l + 1) squared N(0, 1):
    Q_l ~ chi^2 with F (2l + 1) degrees of freedom, exactly.  Q_l / (F (2l + 1)) is the mean of |a_lm|^2 / s_l^2 per
    degree over its 2l + 1 real degrees of freedom; it must lie within the two-sided chi^2 quantiles at a family-wise
    false-alarm probability of 1e-6 over all degrees (Bonferroni)."""
    from scipy.stats import chi2
    from skyrim_b200.engine import grf_spectrum
    lmax, members, channels = 180, 4, 69
    spec32 = grf_spectrum(2.0, 3.0, lmax)[0].astype(np.float32)
    a = _device_draw(spec32, 2024, 0, members, channels, dev).astype(np.complex128).reshape(members * channels, -1)
    ls, ms = _tri_index(lmax)
    keep = ls >= 1                                                  # s_0 = 0: the field has zero mean
    a, ls, ms = a[:, keep], ls[keep], ms[keep]
    w = np.where(ms == 0, 1.0, 2.0)
    p = np.abs(a) ** 2 * w / spec32.astype(np.float64)[ls] ** 2
    Fn = a.shape[0]
    q = np.bincount(ls, weights=p.sum(0), minlength=lmax + 1)[1:]
    dof = Fn * (2 * np.arange(1, lmax + 1) + 1)
    pfa = 1e-6 / (2 * lmax)
    lo, hi = chi2.ppf(pfa, dof), chi2.isf(pfa, dof)
    assert ((q >= lo) & (q <= hi)).all(), np.nonzero((q < lo) | (q > hi))
    assert abs(q.sum() / dof.sum() - 1.0) < 5 * np.sqrt(2.0 / dof.sum())


def test_library_refuses_host_pointers_and_short_workspace(dev):
    from skyrim_b200 import _ffi
    from skyrim_b200.engine import grf_legendre_table, grf_spectrum
    L = _ffi.lib()
    nlat, nlon, lmax = 41, 96, 20
    x = torch.zeros((1, 2, nlat, nlon), device=dev)
    sig = torch.ones(2, device=dev)
    s = torch.as_tensor(grf_spectrum(2.0, 3.0, lmax)[0].astype(np.float32), device=dev)
    leg = grf_legendre_table(nlat, lmax, dev)
    need = L.sky_grf_workspace_bytes(1, 2, nlat, nlon, lmax)
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    host = np.zeros(nlat * nlon * 2, np.float32)
    args = [x.data_ptr(), sig.data_ptr(), 1.0, 0, 0, 1, 2, nlat, nlon, lmax, s.data_ptr(), leg.data_ptr(), ws.data_ptr(), need,
            None]
    for i in (0, 1, 10, 11, 12):
        bad = list(args)
        bad[i] = host.ctypes.data
        assert L.sky_perturb_ic_grf(*bad) == -1, i
        assert b"device memory" in L.sky_last_error()
    bad = list(args)
    bad[13] = need - 1
    assert L.sky_perturb_ic_grf(*bad) == -1 and b"workspace" in L.sky_last_error()
    torch.cuda.synchronize()
    assert torch.count_nonzero(x) == 0
    assert L.sky_perturb_ic_grf(*args) == 0
    torch.cuda.synchronize()
    assert torch.count_nonzero(x) > 0


def test_ensemble_runner_spherical_grf_members_stay_solo_equal(dev):
    from skyrim_b200.config import PANGU_CHANNELS, pangu_small
    from skyrim_b200.engine import StepEngine
    from skyrim_b200.ensemble import EnsembleRunner
    from skyrim_b200.weights import channel_stats, make_pangu_weights, synthetic_state
    cfg = pangu_small(41, 96)
    eng = StepEngine(cfg, 0)
    eng.load_weights(make_pangu_weights(cfg, 0))
    base = synthetic_state(PANGU_CHANNELS, cfg.nlat, cfg.nlon, 0)
    sig = channel_stats(PANGU_CHANNELS)[1]
    kw = dict(amp=0.05, seed=3, perturbation="spherical_grf", grf=dict(lmax=20))
    run = EnsembleRunner(eng, base, sig, members_per_gpu=4, rank=0, **kw)
    solo = EnsembleRunner(eng, base, sig, members_per_gpu=1, rank=2, **kw)
    gauss = EnsembleRunner(eng, base, sig, members_per_gpu=1, rank=2, amp=0.05, seed=3)
    assert torch.equal(solo.x[0], run.x[2])
    assert not torch.equal(solo.x[0], gauss.x[0])
    # the perturbation is amp sigma_c times a unit-variance field
    d = (run.x[:, :, 1:-1] - torch.as_tensor(base, device=dev)[None, :, 1:-1]).double()
    ratio = (d.pow(2).mean(dim=(0, 2, 3)).sqrt() / (0.05 * torch.as_tensor(sig, device=dev).double())).cpu().numpy()
    assert 0.3 < np.median(ratio) < 3.0, ratio
    run.step(2)
    solo.step(2)
    assert torch.equal(solo.x[0], run.x[2])
    mean, spread = run.mean_and_spread(world=1)
    assert bool(torch.isfinite(spread).all()) and float(spread.mean()) > 0
    eng.close()
