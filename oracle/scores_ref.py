"""fp64 numpy restatement of the forecast verification scores (skyrim_b200/scores.py, include/skyrim_b200.h
sky_forecast_scores), straight from the fields: the nine weighted sums per (region, channel), with the CRPS spread term G
summed pairwise in O(M^2) rather than from sorted values, and the metrics formed from the fields without the sums."""
import numpy as np


def _fields(x, truth, clim, channels):
    v = np.asarray(x, dtype=np.float64)[:, list(channels)]               # (M, S, H, W)
    y = np.asarray(truth, dtype=np.float64)                              # (S, H, W)
    k = None if clim is None else np.asarray(clim, dtype=np.float64)
    M = v.shape[0]
    s = np.zeros(v.shape[1:])
    for m in range(M):                                                   # member order, as the kernel sums
        s = s + v[m]
    return v, y, k, s / M


def point_terms(x, truth, clim, channels):
    """(9, S, H, W) unweighted per-point terms (SUMS order), NaN where a member, the truth or the climatology is NaN"""
    v, y, k, xb = _fields(x, truth, clim, channels)
    M = v.shape[0]
    e = xb - y
    g = np.zeros(xb.shape)
    for m in range(M):
        for j in range(m + 1, M):
            g = g + np.abs(v[m] - v[j])
    t = [np.ones(xb.shape), e, e * e, ((v - xb) ** 2).sum(0), np.abs(v - y).sum(0) / M, g]
    if k is None:
        t += [np.full(xb.shape, np.nan)] * 3
    else:
        f, o = xb - k, y - k
        t += [f * o, f * f, o * o]
    t = np.stack(t)
    nan = np.isnan(v).any(0) | np.isnan(y) | (np.zeros(y.shape, bool) if k is None else np.isnan(k))
    t[1:, nan] = np.nan
    return t


def score_sums(x, truth, row_weights, channels, clim=None):
    """fp64 (n_regions, n_sel, 9) sums and (n_regions, n_sel, 9) sums of w |term| (the scale of each sum's rounding).
    x (M, C, H, W); truth, clim (n_sel, H, W); row_weights (n_regions, H).  Rows of weight 0 in a region are left out."""
    t = point_terms(x, truth, clim, channels)                            # (9, S, H, W)
    out, mag = [], []
    for w in np.asarray(row_weights, dtype=np.float64):
        rows = w > 0
        tw = t[:, :, rows] * w[rows][None, None, :, None]
        out.append(tw.sum(axis=(2, 3)).T)
        mag.append(np.abs(tw).sum(axis=(2, 3)).T)
    return np.stack(out), np.stack(mag)


def metrics(x, truth, row_weights, channels, clim=None):
    """fp64 (n_regions, n_sel, 7) metrics (bias, rmse, acc, spread, ssr, crps, crps_fair) formed from the fields with
    normalised weights, independently of skyrim_b200.scores.metrics_from_sums"""
    v, y, k, xb = _fields(x, truth, clim, channels)
    M = v.shape[0]
    res = []
    for w in np.asarray(row_weights, dtype=np.float64):
        W = np.broadcast_to(w[:, None], xb.shape[1:]) / (w.sum() * xb.shape[-1])
        keep = W > 0
        avg = lambda a: np.where(keep, a * W, 0.0).sum(axis=(-2, -1))    # noqa: E731
        nan = np.where(keep, np.isnan(v).any(0) | np.isnan(y) | (False if k is None else np.isnan(k)), False).any((-2, -1))
        e = xb - y
        bias, rmse = avg(e), np.sqrt(avg(e * e))
        if k is None:
            acc = np.full(bias.shape, np.nan)
        else:
            f, o = xb - k, y - k
            acc = avg(f * o) / np.sqrt(avg(f * f) * avg(o * o))
        pair = np.zeros(xb.shape)
        for m in range(M):
            for j in range(M):
                pair = pair + np.abs(v[m] - v[j])
        mae = np.abs(v - y).mean(0)
        crps = avg(mae - pair / (2 * M * M))
        if M > 1:
            spread = np.sqrt(avg(((v - xb) ** 2).sum(0) / (M - 1)))
            ssr = np.sqrt((M + 1) / M) * spread / rmse
            crps_fair = avg(mae - pair / (2 * M * (M - 1)))
        else:
            spread = ssr = crps_fair = np.full(bias.shape, np.nan)
        m_ = np.stack([bias, rmse, acc, spread, ssr, crps, crps_fair], axis=-1)
        m_[nan] = np.nan
        res.append(m_)
    return np.stack(res)


def crps_integral(members, y):
    """CRPS of one scalar forecast by its definition: the integral of (F_M(z) - 1{z >= y})^2 dz, F_M the empirical CDF.
    The integrand is constant between consecutive members and y, so the midpoint rule on those intervals is exact."""
    xs = np.asarray(members, dtype=np.float64)
    z = np.unique(np.append(xs, y))
    mid = 0.5 * (z[1:] + z[:-1])
    F = (xs[None, :] <= mid[:, None]).mean(1)
    d = (F - (mid >= y)) ** 2
    return float(np.sum(d * np.diff(z)))
