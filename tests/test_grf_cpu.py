"""Spherical Gaussian random field perturbation: oracle, spectrum and C-ABI checks that need no GPU."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import scipy.special as sp

from oracle import grf_ref, sht_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("ctr, key, want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_oracle_philox_known_answers(ctr, key, want):
    """Random123's Philox4x32-10 known-answer vectors"""
    got = grf_ref.philox4x32_10(np.array(ctr, dtype=np.uint32), key)
    assert tuple(int(v) for v in got) == want


@pytest.mark.parametrize("alpha, tau, lmax", [(2.0, 3.0, 180), (2.0, 3.0, 20), (3.0, 1.0, 90), (1.5, 10.0, 360)])
def test_spectrum_is_normalised(alpha, tau, lmax):
    from skyrim_b200.engine import grf_spectrum
    s, kept = grf_spectrum(alpha, tau, lmax)
    l = np.arange(lmax + 1)
    assert s.shape == (lmax + 1,) and s[0] == 0.0 and (s[1:] > 0).all()
    assert abs(np.sum(s ** 2 * (2 * l + 1)) / (4 * np.pi) - 1.0) < 1e-13
    np.testing.assert_allclose(s, grf_ref.spectrum(alpha, tau, lmax), rtol=1e-13)
    # truncation keeps a fraction that grows with lmax towards 1; for alpha = 2 the tail is ~ 1 / (lmax^2 (...))
    assert 0.0 < kept < 1.0
    assert grf_spectrum(alpha, tau, 2 * lmax)[1] > kept


def test_spectrum_retained_fraction_against_direct_sum():
    from skyrim_b200.engine import grf_spectrum
    l = np.arange(1, 4_000_001, dtype=np.float64)
    g = (2 * l + 1) * (l * (l + 1) + 9.0) ** -2.0
    want = g[:180].sum() / (g.sum() + 1.0 / (4e6 * 4e6))     # tail beyond 4e6 ~ 1 / l^2
    assert abs(grf_spectrum(2.0, 3.0, 180)[1] - want) < 1e-9
    with pytest.raises(ValueError):
        grf_spectrum(1.0, 3.0, 180)


def test_oracle_synthesis_matches_scipy_spherical_harmonics():
    nlat, nlon, lmax = 13, 24, 5
    a = grf_ref.coefficients(grf_ref.spectrum(2.0, 3.0, lmax), 11, [3], 2)
    f = grf_ref.synthesize(a, nlat, nlon)
    theta = np.pi * np.arange(nlat) / (nlat - 1)
    phi = 2 * np.pi * np.arange(nlon) / nlon
    T, P = np.meshgrid(theta, phi, indexing="ij")
    ref = np.zeros((1, 2, nlat, nlon))
    for l in range(lmax + 1):
        for m in range(l + 1):
            y = sp.sph_harm_y(l, m, T, P)
            term = a[..., l, m, None, None] * y[None, None]
            ref += term.real if m == 0 else 2.0 * term.real
    np.testing.assert_allclose(f, ref, atol=1e-12, rtol=0)


@pytest.mark.parametrize("nlat, nlon, lmax", [(41, 96, 20), (21, 41, 10), (181, 360, 90)])
def test_oracle_forward_sht_recovers_coefficients(nlat, nlon, lmax):
    a = grf_ref.coefficients(grf_ref.spectrum(2.0, 3.0, lmax), 5, [0, 7], 3)
    p, w = grf_ref.legendre(nlat, lmax)
    back = grf_ref.analyze(grf_ref.synthesize(a, nlat, nlon, p), lmax, p, w)
    assert np.abs(back - a).max() < 1e-12 * np.abs(a).max()


def test_oracle_pole_rows_are_constant():
    a = grf_ref.coefficients(grf_ref.spectrum(2.0, 3.0, 20), 1, [0, 1], 2)
    f = grf_ref.synthesize(a, 41, 96)
    for k in (0, -1):
        assert np.ptp(f[..., k, :], axis=-1).max() < 1e-14


def test_oracle_draws_do_not_depend_on_lmax():
    z_small = grf_ref.normal_draws(9, [4], 3, 10)
    z_big = grf_ref.normal_draws(9, [4], 3, 30)
    for s, b in zip(z_small, z_big):
        np.testing.assert_array_equal(s, b[..., :11, :11])


def test_oracle_variance_is_one_by_addition_theorem():
    """E f^2 = sum_l s_l^2 sum_m |Pbar_l^m|^2 (m > 0 twice) = sum_l s_l^2 (2l + 1) / 4 pi = 1 at every latitude"""
    lmax, nlat = 60, 121
    s = grf_ref.spectrum(2.0, 3.0, lmax)
    p, _ = grf_ref.legendre(nlat, lmax)
    c = np.where(np.arange(lmax + 1) == 0, 1.0, 2.0)
    var = np.einsum("l,m,mlk->k", s ** 2, c, p ** 2)    # E|a_lm|^2 = s_l^2 (m = 0), s_l^2 / 2 (m > 0), times 2^2 / 2
    np.testing.assert_allclose(var, 1.0, atol=1e-12)


def test_grf_symbols_exported_and_declared():
    from skyrim_b200 import _ffi
    hdr = open(os.path.join(ROOT, "include", "skyrim_b200.h")).read()
    declared = set(re.findall(r"\b(sky_[a-z_0-9]+)\s*\(", hdr))
    new = {"sky_grf_workspace_bytes", "sky_grf_draw", "sky_perturb_ic_grf"}
    assert new <= declared and new <= set(_ffi.EXPORTS)
    L = _ffi.lib()
    for name in new:
        assert hasattr(L, name), name


@pytest.mark.parametrize("nlat, nlon, lmax, what", [
    (41, 96, 41, "nlat"), (41, 96, 60, "nlat"), (41, 40, 20, "nlon"), (721, 1440, 720, "nlon"), (41, 96, 0, "lmax"),
])
def test_library_refuses_shape_errors_before_any_cuda_call(nlat, nlon, lmax, what):
    """the shape checks run first: the pointers (bogus here) are never inspected, so this needs no device"""
    from skyrim_b200 import _ffi
    L = _ffi.lib()
    bogus = C.c_void_p(0x1000)
    assert L.sky_grf_workspace_bytes(4, 69, nlat, nlon, lmax) == 0
    rc = L.sky_perturb_ic_grf(bogus, bogus, 1.0, 0, 0, 4, 69, nlat, nlon, lmax, bogus, bogus, bogus, 1 << 30, None)
    assert rc == -1
    assert what in L.sky_last_error().decode()


def test_workspace_stays_under_512_mb():
    from skyrim_b200 import _ffi
    L = _ffi.lib()
    sizes = {lmax: L.sky_grf_workspace_bytes(4, 69, 721, 1440, lmax) for lmax in (1, 90, 180, 360)}
    assert all(0 < b <= 512 << 20 for b in sizes.values()), sizes
    assert L.sky_grf_workspace_bytes(32, 69, 721, 1440, 360) <= 512 << 20
    # one field's coefficients + Legendre stage at lmax 180: 16471 complex64 + 2 x 181 x 721 fp32
    one = L.sky_grf_workspace_bytes(1, 1, 721, 1440, 180)
    assert one >= 16471 * 8 + 2 * 181 * 721 * 4 + 1440 * 8


def test_ensemble_runner_rejects_unknown_perturbation():
    from skyrim_b200.ensemble import EnsembleRunner
    with pytest.raises(ValueError):
        EnsembleRunner(None, np.zeros((1, 2, 2), np.float32), np.ones(1), 1, perturbation="bred")
    with pytest.raises(ValueError):
        EnsembleRunner(None, np.zeros((1, 2, 2), np.float32), np.ones(1), 1, grf=dict(lmax=4))
