"""fp64 numpy restatement of the site entries (include/skyrim_b200.h sky_sites_create, sky_sample_sites,
sky_site_scores): the stencil with the same operations in the same order, sampling with the same summation order, and the
six site terms with the missing-observation rule, taken from the scores oracle's per-point terms."""
import numpy as np

from oracle.scores_ref import point_terms

BILINEAR, NEAREST = "bilinear", "nearest"


def stencil(lat, lon, nlat: int, nlon: int, method: str = BILINEAR):
    """(idx int64 (n, 4) flat plane indices, w fp64 (n, 4) weights) of the sites at (lat, lon) degrees"""
    lat = np.asarray(lat, dtype=np.float64).reshape(-1)
    lon = np.asarray(lon, dtype=np.float64).reshape(-1)
    dphi, dlam = 180.0 / (nlat - 1), 360.0 / nlon
    lp = np.fmod(lon, 360.0)
    lp = np.where(lp < 0.0, lp + 360.0, lp)
    u = lp / dlam
    t = (90.0 - lat) / dphi
    n = lat.size
    idx, w = np.zeros((n, 4), np.int64), np.zeros((n, 4), np.float64)
    if method == NEAREST:
        i0 = np.floor(t + 0.5).astype(np.int64)
        j0 = np.floor(u + 0.5).astype(np.int64) % nlon
        idx[:] = (i0 * nlon + j0)[:, None]
        w[:, 0] = 1.0
        return idx, w
    if method != BILINEAR:
        raise ValueError(method)
    jf = np.floor(u)
    b = u - jf
    j0 = jf.astype(np.int64) % nlon
    j1 = (j0 + 1) % nlon
    i0 = np.minimum(np.floor(t).astype(np.int64), nlat - 2)
    a = t - i0
    idx[:, 0], idx[:, 1] = i0 * nlon + j0, i0 * nlon + j1
    idx[:, 2], idx[:, 3] = (i0 + 1) * nlon + j0, (i0 + 1) * nlon + j1
    w[:, 0], w[:, 1], w[:, 2], w[:, 3] = (1.0 - a) * (1.0 - b), (1.0 - a) * b, a * (1.0 - b), a * b
    return idx, w


def sample(x, idx, w, channels):
    """fp32 (M, n_sel, n_sites) of the members x (M, C, H, W) at the sites of the stencil (idx, w): per member, channel and
    site, 0 + w_0 x_0 + w_1 x_1 + ... in stencil order in fp64, entries of weight 0 skipped, rounded once to fp32"""
    x = np.asarray(x, dtype=np.float32)
    M = x.shape[0]
    flat = x.reshape(M, x.shape[1], -1)[:, list(channels)].astype(np.float64)    # (M, S, plane)
    acc = np.zeros(flat.shape[:2] + (idx.shape[0],))
    for k in range(idx.shape[1]):
        keep = w[:, k] != 0.0
        term = w[:, k] * flat[:, :, idx[:, k]]
        acc = np.where(keep, acc + np.where(keep, term, 0.0), acc)
    return acc.astype(np.float32)


def site_terms(values, obs):
    """fp64 (n_sel, n_sites, 6) terms 1, e, e^2, var, mae / M, G of ``values`` fp32 (M, n_sel, n_sites) against ``obs``
    fp32 (n_sel, n_sites): 0 where the observation is NaN (missing); terms 1..5 NaN where a member is NaN and the
    observation is not"""
    v = np.asarray(values, dtype=np.float32)
    y = np.asarray(obs, dtype=np.float32)
    missing = np.isnan(y)
    t = point_terms(v[:, :, None, :], np.where(missing, 0.0, y)[:, None, :], None, range(v.shape[1]))[:6, :, 0]
    t = np.moveaxis(t, 0, -1)                                              # (S, n, 6)
    t[missing] = 0.0
    return t


def site_sums(values, obs):
    """fp64 (n_sel, 6) sums over the sites with an observation, and the sums of |term| (the scale of their rounding)"""
    t = site_terms(values, obs)
    return t.sum(axis=1), np.abs(t).sum(axis=1)
