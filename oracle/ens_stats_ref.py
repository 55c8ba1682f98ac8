"""fp64 numpy restatement of sky_ensemble_stats (include/skyrim_b200.h): per-point ensemble mean, population spread,
numpy-"linear" quantiles and strict exceedance probabilities, with NaN propagation, each rounded once to fp32."""
import numpy as np


def ensemble_stats(x, channels, quantiles=(), events=()):
    """x: (M, C, H, W) array; channels: indices into C; events: (i, threshold) with i an index into ``channels``.
    Returns (stats fp32 (2 + n_q, n_sel, H, W), prob fp32 (n_events, H, W))."""
    v = np.asarray(x, dtype=np.float64)[:, list(channels)]
    M = v.shape[0]
    s = np.zeros(v.shape[1:])
    for m in range(M):              # member order, as the kernel sums
        s = s + v[m]
    mu = s / M
    ss = np.zeros(v.shape[1:])
    for m in range(M):
        d = v[m] - mu
        ss = ss + d * d
    out = [mu, np.sqrt(ss / M)]
    nan = np.isnan(v).any(axis=0)
    for q in quantiles:
        r = np.quantile(v, q, axis=0, method="linear")
        out.append(np.where(nan, np.nan, r))
    prob = []
    for i, t in events:
        p = (v[:, i] > np.float64(np.float32(t))).sum(axis=0) / M     # the kernel compares against the fp32 threshold
        prob.append(np.where(nan[i], np.nan, p))
    shape = v.shape[2:]
    return (np.stack(out).astype(np.float32),
            np.stack(prob).astype(np.float32) if prob else np.zeros((0,) + shape, np.float32))
