"""fp64 numpy restatement of sky_ensemble_stats_multi (include/skyrim_b200.h): the statistics of ens_stats_ref over members
pooled from several sources in source-then-member order, plus each source's own mean."""
import numpy as np

from .ens_stats_ref import ensemble_stats


def multi_source_stats(sources, channels_per_source, quantiles=(), events=()):
    """sources: (M_k, C_k, H, W) arrays; channels_per_source[k]: for every selected channel, its index in source k;
    events: (i, threshold) with i an index into the selection.  Returns (stats fp32 (2 + n_q, n_sel, H, W),
    prob fp32 (n_events, H, W), means fp32 (K, n_sel, H, W))."""
    picked = [np.asarray(x, dtype=np.float64)[:, list(c)] for x, c in zip(sources, channels_per_source)]
    pool = np.concatenate(picked, axis=0)
    stats, prob = ensemble_stats(pool, range(pool.shape[1]), quantiles, events)
    means = []
    for v in picked:
        s = np.zeros(v.shape[1:])
        for m in range(v.shape[0]):      # member order, as the kernel sums
            s = s + v[m]
        means.append(s / v.shape[0])
    return stats, prob, np.stack(means).astype(np.float32)
