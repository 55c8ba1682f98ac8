"""fp64 numpy restatement of the per-point verification (include/skyrim_b200.h sky_forecast_rank_histogram and
sky_forecast_score_maps), straight from the fields and without code from ``skyrim_b200``: ranks by counting, ties broken
with the oracle's own Philox (``oracle/grf_ref.py``), and the map terms with G summed pairwise in O(M^2)."""
import numpy as np

from oracle.grf_ref import philox4x32_10

RANK_TAG = 0x524E4B31          # "RNK1": second counter word of the tie-breaking draws


def tie_words(seed, date_index, lead_index, channels, nlat, nlon):
    """uint64 (n_sel, H, W): the first Philox output word at key (seed, date), counter (point, "RNK1", channel, lead)"""
    S, P = len(channels), nlat * nlon
    ctr = np.zeros((S, P, 4), np.uint64)
    ctr[..., 0] = np.arange(P, dtype=np.uint64)[None]
    ctr[..., 1] = RANK_TAG
    ctr[..., 2] = np.asarray(channels, np.uint64)[:, None]
    ctr[..., 3] = lead_index
    return philox4x32_10(ctr, (seed, date_index))[..., 0].astype(np.uint64).reshape(S, nlat, nlon)


def ranks(x, truth, channels, seed, date_index, lead_index):
    """int64 (n_sel, H, W) rank of the truth among the members, -1 where a member or the truth is NaN.
    x (M, C, H, W); truth (n_sel, H, W)"""
    v = np.asarray(x, dtype=np.float32)[:, list(channels)]
    y = np.asarray(truth, dtype=np.float32)
    lt, eq = (v < y).sum(0), (v == y).sum(0)
    u = tie_words(seed, date_index, lead_index, channels, *y.shape[-2:])
    r = lt + ((u * (eq + 1).astype(np.uint64)) >> np.uint64(32)).astype(np.int64)
    nan = np.isnan(v).any(0) | np.isnan(y)
    return np.where(nan, -1, r)


def rank_histogram(x, truth, row_weights, channels, seed, date_index, lead_index):
    """fp64 (n_regions, n_sel, M + 1): sum over the points with w > 0 of (w / nlon) 1{rank = k}, NaN for a region and
    channel with a NaN point of positive weight; and fp64 (n_regions,) sum of the point weights"""
    M = np.asarray(x).shape[0]
    r = ranks(x, truth, channels, seed, date_index, lead_index)
    nlon = r.shape[-1]
    out, wsum = [], []
    for w in np.asarray(row_weights, dtype=np.float64):
        rows = w > 0
        rr = r[:, rows]                                                   # (S, rows, W)
        h = np.stack([((rr == k) * (w[rows] / nlon)[None, :, None]).sum((1, 2)) for k in range(M + 1)], -1)
        h[(rr < 0).any((1, 2))] = np.nan
        out.append(h)
        wsum.append(w[rows].sum())
    return np.stack(out), np.array(wsum)


def map_terms(x, truth, channels):
    """fp64 (n_sel, 5, H, W): e = x_bar - y, e^2, sum_m (x_m - x_bar)^2, (1/M) sum_m |x_m - y|, G = sum_{m<k} |x_m - x_k|,
    NaN where a member or the truth is NaN; and the per-term magnitudes for a rounding bound"""
    v = np.asarray(x, dtype=np.float64)[:, list(channels)]
    y = np.asarray(truth, dtype=np.float64)
    M = v.shape[0]
    xb = np.zeros(y.shape)
    for m in range(M):                                                    # member order, as the kernel sums
        xb = xb + v[m]
    xb = xb / M
    g = np.zeros(y.shape)
    for m in range(M):
        for k in range(m + 1, M):
            g = g + np.abs(v[m] - v[k])
    e = xb - y
    t = np.stack([e, e * e, ((v - xb) ** 2).sum(0), np.abs(v - y).sum(0) / M, g], axis=1)
    nan = np.isnan(v).any(0) | np.isnan(y)
    t[np.broadcast_to(nan[:, None], t.shape)] = np.nan
    a = np.abs(xb) + np.abs(y)
    mag = np.stack([a, a * a, ((np.abs(v) + np.abs(xb)) ** 2).sum(0), (np.abs(v) + np.abs(y)).mean(0),
                    (M - 1) * np.abs(v).sum(0)], axis=1)
    return t, mag
