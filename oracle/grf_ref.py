"""ORACLE — test infrastructure, not product code.

The spherical Gaussian random field perturbation (include/skyrim_b200.h sky_perturb_ic_grf) restated in numpy, fp64,
without any code from ``skyrim_b200``:

  * Philox4x32-10 (Salmon et al., SC'11) and the Box-Muller transform, restated here;
  * the spectrum s_l = k (l (l + 1) + tau^2)^(-alpha / 2), s_0 = 0, sum_l s_l^2 (2l + 1) / 4 pi = 1, restated here;
  * Pbar_l^m on the equiangular grid from ``oracle/sht_ref.py`` (scipy, Waldvogel nodes), not ``sht.legpoly``;
  * the longitude sum by ``numpy.fft.irfft`` (norm="forward"), not a cos / sin table.
"""
from __future__ import annotations

import numpy as np

from . import sht_ref

GRF_TAG = 0x47524631          # "GRF1": second counter word
_M0, _M1 = 0xD2511F53, 0xCD9E8D57
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """ctr: uint32 array (..., 4); key: (k0, k1) ints or uint32 arrays broadcastable to ctr[..., 0].  -> uint32 (..., 4)"""
    c = [np.asarray(ctr, dtype=np.uint64)[..., i].copy() for i in range(4)]
    k0 = np.asarray(key[0], dtype=np.uint64) & _MASK
    k1 = np.asarray(key[1], dtype=np.uint64) & _MASK
    for _ in range(10):
        p0 = np.uint64(_M0) * c[0]
        p1 = np.uint64(_M1) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(_MASK)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(_MASK)
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0 = (k0 + np.uint64(_W0)) & np.uint64(_MASK)
        k1 = (k1 + np.uint64(_W1)) & np.uint64(_MASK)
    return np.stack(c, axis=-1).astype(np.uint32)


def spectrum(alpha: float, tau: float, lmax: int) -> np.ndarray:
    l = np.arange(lmax + 1, dtype=np.float64)
    s = np.where(l > 0, (l * (l + 1) + tau ** 2) ** (-alpha / 2), 0.0)
    return s / np.sqrt(np.sum(s ** 2 * (2 * l + 1)) / (4 * np.pi))


def normal_draws(seed: int, members, channels: int, lmax: int):
    """z0, z1 float64 [len(members), channels, lmax + 1 (l), lmax + 1 (m)] for the global member ids ``members``
    (entries with m > l are unused)."""
    g = np.asarray(members, dtype=np.uint64)[:, None, None, None]
    c = np.arange(channels, dtype=np.uint64)[None, :, None, None]
    l = np.arange(lmax + 1, dtype=np.uint64)[None, None, :, None]
    m = np.arange(lmax + 1, dtype=np.uint64)[None, None, None, :]
    shape = np.broadcast_shapes(g.shape, c.shape, l.shape, m.shape)
    ctr = np.stack([np.broadcast_to(l | (m << np.uint64(16)), shape), np.full(shape, GRF_TAG, np.uint64),
                    np.broadcast_to(c, shape), np.broadcast_to(g, shape)], axis=-1)
    w = philox4x32_10(ctr, (seed & _MASK, seed >> 32)).astype(np.float64)
    u0, u1 = (w[..., 0] + 0.5) * 2.0 ** -32, (w[..., 1] + 0.5) * 2.0 ** -32
    r = np.sqrt(-2.0 * np.log(u0))
    return r * np.cos(2.0 * np.pi * u1), r * np.sin(2.0 * np.pi * u1)


def coefficients(spec, seed: int, members, channels: int) -> np.ndarray:
    """a_lm complex128 [members, channels, lmax + 1 (l), lmax + 1 (m)], zero for m > l.  ``spec``: s_l [lmax + 1]."""
    spec = np.asarray(spec, dtype=np.float64)
    lmax = spec.size - 1
    z0, z1 = normal_draws(seed, members, channels, lmax)
    s = spec[:, None]
    a = np.where(np.arange(lmax + 1)[None, :] == 0, s * z0 + 0j, s * (z0 + 1j * z1) / np.sqrt(2.0))
    return np.where(np.arange(lmax + 1)[None, :] <= np.arange(lmax + 1)[:, None], a, 0.0)


def legendre(nlat: int, lmax: int):
    """Pbar[m, l, k] on the equiangular grid (sht_ref: scipy) and the Clenshaw-Curtis weights"""
    cost, w = sht_ref.cc_nodes_weights(nlat)
    return sht_ref.pbar(lmax + 1, lmax + 1, cost), w


def synthesize(a: np.ndarray, nlat: int, nlon: int, pbar=None) -> np.ndarray:
    """f float64 [..., nlat, nlon] from a_lm [..., l, m]: F_m(theta_k) = sum_l Pbar a_lm, then irfft over longitude"""
    lmax = a.shape[-1] - 1
    p = legendre(nlat, lmax)[0] if pbar is None else pbar
    F = np.einsum("mlk,...lm->...km", p, a)
    F = F.copy()
    F[..., 0] = F[..., 0].real                     # irfft ignores Im of the m = 0 mode (it is 0 here anyway)
    return np.fft.irfft(F, n=nlon, axis=-1, norm="forward")


def analyze(f: np.ndarray, lmax: int, pbar=None, weights=None) -> np.ndarray:
    """forward real SHT (torch-harmonics conventions): a_lm complex128 [..., l, m] of f [..., nlat, nlon].  Exact for
    band-limited fields with lmax <= (nlat - 1) / 2 and 2 lmax < nlon."""
    nlat, nlon = f.shape[-2:]
    if pbar is None:
        pbar, weights = legendre(nlat, lmax)
    F = 2.0 * np.pi * np.fft.rfft(f, axis=-1, norm="forward")[..., : lmax + 1]
    return np.einsum("mlk,k,...km->...lm", pbar, weights, F)
