"""Forecast verification: latitude-weighted scores per channel, region and lead time against supplied analyses, as
earth2mip's ``score_deterministic`` / ``score_ensemble`` report them.  The device writes weighted fp64 sums
(``engine.forecast_scores``, include/skyrim_b200.h sky_forecast_scores); this module holds the definitions, forms the
metrics from the sums, and adapts truth and climatology sources to the model's grid and channels.

Notation: channel c, region r, lead n; members x_1..x_M; ensemble mean x_bar, summed in member order in fp64 (the
unrounded mean of ``k_ens_stats``); truth y; optional climatology k.  A region is a latitude band [lat_min, lat_max], both
ends included (at most 4; default ``{"global": (-90, 90)}``).  The weight of point p in region r is
w_p = cos(phi_p) / sum_{q in r} cos(phi_q), phi the latitude, with the pole rows weighted exactly 0 (earth2mip's cos-latitude
convention; cell-area weights are not offered).  With all sums over the points of the region:

    bias       sum w (x_bar - y)                                             M = 1: the forecast bias
    rmse       sqrt(sum w (x_bar - y)^2)                                     M = 1: the deterministic RMSE
    acc        sum w f'o' / sqrt(sum w f'^2 sum w o'^2), f' = x_bar - k, o' = y - k (uncentred, earth2mip's
               ``weighted_acc``)                                              NaN without a climatology
    spread     sqrt(sum w s^2), s^2 = sum_m (x_m - x_bar)^2 / (M - 1)          M = 1: NaN
    ssr        sqrt((M + 1) / M) spread / rmse (Fortin et al. 2014)           M = 1: NaN
    crps       sum w [(1/M) sum_m |x_m - y| - 1/(2 M^2) sum_{m,k} |x_m - x_k|] (the empirical-CDF CRPS, as properscoring
               computes it)                                                   M = 1: the MAE
    crps_fair  the same with 1/(2 M (M - 1)) in the second term              M = 1: NaN

A NaN member, truth or climatology value at a point with w > 0 in a region makes that channel's scores for that region NaN;
points with w = 0 are not read into that region's sums; scores never depend on which other channels or regions were
requested.
"""
from __future__ import annotations

import datetime

import numpy as np

METRICS = ("bias", "rmse", "acc", "spread", "ssr", "crps", "crps_fair")
# the nine sums the device writes per (region, channel), in order (G = sum_{m<k} |x_m - x_k|)
SUMS = ("w", "w_e", "w_e2", "w_var", "w_mae", "w_g", "w_fo", "w_ff", "w_oo")
MAX_REGIONS = 4
DEFAULT_REGIONS = {"global": (-90.0, 90.0)}
_LAT_EPS = 1e-9   # degrees: a band end equal to a grid latitude up to rounding includes that row


def region_weights(lat, regions=None):
    """(names, fp64 (n_regions, nlat) row weights): for region r, row i gets cos(lat_i) if lat_i lies in the band (both
    ends included), else 0; the pole rows get exactly 0; each region's row weights sum to 1 (the weight of a point is its
    row's weight over nlon)."""
    regions = dict(DEFAULT_REGIONS if regions is None else regions)
    if not 1 <= len(regions) <= MAX_REGIONS:
        raise ValueError(f"{len(regions)} regions: 1 to {MAX_REGIONS} latitude bands")
    lat = np.asarray(lat, dtype=np.float64)
    cos = np.cos(np.deg2rad(lat))
    cos[np.abs(np.abs(lat) - 90.0) <= _LAT_EPS] = 0.0
    cos = np.maximum(cos, 0.0)
    names, rows = [], []
    for name, band in regions.items():
        lo, hi = (float(v) for v in band)
        if not -90.0 <= lo <= hi <= 90.0:
            raise ValueError(f"region {name!r}: band ({lo}, {hi}) must satisfy -90 <= lat_min <= lat_max <= 90")
        w = np.where((lat >= lo - _LAT_EPS) & (lat <= hi + _LAT_EPS), cos, 0.0)
        if not w.sum() > 0.0:
            raise ValueError(f"region {name!r}: band ({lo}, {hi}) holds no grid row of positive weight")
        names.append(str(name))
        rows.append(w / w.sum())
    return names, np.stack(rows)


def metrics_from_sums(sums, members: int):
    """fp64 (..., 7) metrics (``METRICS`` order) from fp64 (..., 9) sums of ``members`` members (``SUMS`` order)."""
    s = np.asarray(sums, dtype=np.float64)
    M = int(members)
    if M < 1:
        raise ValueError(f"members = {M} must be at least 1")
    w, e, e2, var, mae, g, fo, ff, oo = (s[..., i] for i in range(9))
    nan = np.full(w.shape, np.nan)
    with np.errstate(divide="ignore", invalid="ignore"):
        bias = e / w
        rmse = np.sqrt(e2 / w)
        acc = fo / np.sqrt(ff * oo)
        if M > 1:
            spread = np.sqrt(var / (M - 1) / w)
            ssr = np.sqrt((M + 1) / M) * spread / rmse
            crps_fair = (mae - g / (M * (M - 1))) / w
        else:
            spread = ssr = crps_fair = nan
        crps = (mae - g / (M * M)) / w
    return np.stack([bias, rmse, acc, spread, ssr, crps, crps_fair], axis=-1)


def period_metrics(sums_per_date, members: int):
    """fp64 (..., 7) metrics of a verification period from fp64 (n_dates, ..., 9) per-date sums.  acc is the mean over the
    dates of each date's acc (WeatherBench2 averages ACC per initial time); every other metric is formed from the sums
    added over the dates: rmse = sqrt(mean MSE), bias = mean bias, spread = sqrt(mean variance), crps = mean crps, and
    ssr from the period's spread and rmse.  One date gives ``metrics_from_sums`` of its sums exactly."""
    s = np.asarray(sums_per_date, dtype=np.float64)
    if s.ndim < 2 or s.shape[0] < 1 or s.shape[-1] != len(SUMS):
        raise ValueError(f"sums of shape {s.shape}: (n_dates >= 1, ..., {len(SUMS)}) needed")
    m = metrics_from_sums(s.sum(axis=0), members)
    m[..., METRICS.index("acc")] = metrics_from_sums(s, members)[..., METRICS.index("acc")].mean(axis=0)
    return m


MAP_METRICS = ("bias", "rmse", "spread", "crps")
MAP_TERMS = ("e", "e2", "var", "mae", "g")    # the five per-point accumulators of sky_forecast_score_maps, in order


def map_metrics(acc, n_dates: int, members: int):
    """fp32 (..., 4, H, W) maps (``MAP_METRICS`` order) from fp64 (..., 5, H, W) per-point accumulators summed over
    ``n_dates`` start dates, formed point by point as ``metrics_from_sums`` forms the scalars (each point with weight 1
    per date)."""
    a = np.asarray(acc, dtype=np.float64)
    lead = a.shape[:-3]
    out = np.empty(lead + (len(MAP_METRICS),) + a.shape[-2:], dtype=np.float32)
    pick = [METRICS.index(k) for k in MAP_METRICS]
    for idx in np.ndindex(*lead):            # one (5, H, W) block at a time: the (H, W, 9) sums stay small
        t = np.moveaxis(a[idx], 0, -1)
        s9 = np.concatenate([np.full(t.shape[:-1] + (1,), float(n_dates)), t, np.full(t.shape[:-1] + (3,), np.nan)], -1)
        out[idx] = np.moveaxis(metrics_from_sums(s9, members)[..., pick], -1, 0)
    return out


# ---- truth and climatology ------------------------------------------------------------------------------------------------
def _check_grid(da, lat, lon, what):
    for name, want in (("lat", lat), ("lon", lon)):
        have = np.asarray(da.coords[name], dtype=np.float64) if name in da.coords else None
        if have is None or have.shape != np.shape(want) or not np.allclose(have, want, rtol=0.0, atol=1e-6):
            n = "none" if have is None else len(have)
            raise ValueError(f"{what}'s {name} ({n} values) differs from the model's grid ({len(want)} values); "
                             "regrid it onto the model grid first")


def _select(da, channels, what):
    have = [str(c) for c in np.asarray(da.coords["channel"])] if "channel" in da.coords else []
    missing = [c for c in channels if c not in have]
    if missing:
        raise ValueError(f"{what} lacks channel(s) {missing}")
    vals = np.asarray(da.values, dtype=np.float32)
    ax = list(da.dims).index("channel")
    return np.ascontiguousarray(np.take(vals, [have.index(c) for c in channels], axis=ax))


def truth_fetcher(truth, channels, lat, lon, times=()):
    """``time -> fp32 (n_sel, nlat, nlon)`` from ``truth``: a data source (``source[time] -> DataArray(channel, lat,
    lon)``, the ``ic_source`` protocol) or a DataArray with dims (time, channel, lat, lon).  Refuses a grid that differs
    from the model's, a missing channel and a missing time, each by name; a DataArray is checked for every one of
    ``times`` at once, a data source when each time is fetched."""
    if hasattr(truth, "dims") and "time" in tuple(truth.dims):
        if tuple(truth.dims) != ("time", "channel", "lat", "lon"):
            raise ValueError(f"truth dims {tuple(truth.dims)}: (time, channel, lat, lon) needed")
        _check_grid(truth, lat, lon, "truth")
        have = np.asarray(truth.coords["time"]).astype("datetime64[s]")
        vals = _select(truth, channels, "truth")

        def at(t):
            hit = np.nonzero(have == np.datetime64(t, "s"))[0]
            if hit.size == 0:
                raise ValueError(f"truth has no analysis at {np.datetime64(t, 's')}")
            return vals[hit[0]]
        for t in times:
            at(t)
        return at
    if not hasattr(truth, "__getitem__") or isinstance(truth, str):
        raise TypeError("truth must be a data source (source[time] -> DataArray) or a DataArray with a time dimension")

    def at(t):
        try:
            da = truth[t]
        except KeyError as e:
            raise ValueError(f"truth has no analysis at {np.datetime64(t, 's')}") from e
        if tuple(da.dims)[-2:] != ("lat", "lon") or "channel" not in da.dims:
            raise ValueError(f"truth[{t}] has dims {tuple(da.dims)}: (channel, lat, lon) needed")
        _check_grid(da, lat, lon, "truth")
        v = _select(da, channels, "truth")
        return v[-1] if v.ndim == 4 else v
    return at


def climatology_fields(clim, channels, lat, lon):
    """fp32 (n_sel, nlat, nlon) of a static climatology DataArray (channel, lat, lon), or None"""
    if clim is None:
        return None
    if tuple(clim.dims) != ("channel", "lat", "lon"):
        raise ValueError(f"climatology dims {tuple(clim.dims)}: (channel, lat, lon) needed")
    _check_grid(clim, lat, lon, "climatology")
    return _select(clim, channels, "climatology")


def scorecard(sums, members: int, leads_hours, regions, channels, model: str, start_time: datetime.datetime):
    """DataArray (lead_time, metric, region, channel) of fp64 metrics from fp64 sums (lead, region, channel, 9); lead_time in
    hours (0: the initial condition); the model, members and start time in attrs."""
    from . import xr_shim as xr
    m = metrics_from_sums(sums, members)                     # (lead, region, channel, metric)
    return xr.DataArray(np.ascontiguousarray(np.moveaxis(m, -1, 1)), dims=["lead_time", "metric", "region", "channel"],
                        coords=dict(lead_time=np.asarray(leads_hours, dtype=np.float64), metric=np.array(METRICS),
                                    region=np.array(list(regions)), channel=np.array(list(channels))),
                        attrs=dict(model=str(model), members=int(members),
                                   start_time=str(np.datetime64(start_time, "s"))))


class PeriodScores:
    """What ``GlobalModel.score_period`` returns: DataArrays of a verification period over several start dates.
        card            fp64 (lead_time, metric, region, channel): the period's metrics (``period_metrics``)
        cards           fp64 (start_time, lead_time, metric, region, channel): each date's scorecard
        rank_histogram  fp64 (lead_time, region, channel, rank): the rank histograms averaged over the dates
        maps            fp32 (lead_time, metric, channel, lat, lon) of ``MAP_METRICS`` over the period, or None"""

    def __init__(self, card, cards, rank_histogram, maps=None):
        self.card, self.cards, self.rank_histogram, self.maps = card, cards, rank_histogram, maps

    @classmethod
    def build(cls, sums, hist, maps, members: int, start_times, leads_hours, map_leads, step_hours: float, regions,
              channels, map_channels, model: str, lat, lon):
        """from host fp64 sums (date, lead, region, channel, 9), histograms (date, lead, region, channel, M + 1) and map
        accumulators (map lead, map channel, 5, lat, lon) summed over the dates, or None; ``map_leads`` lists the steps of
        the map slots in slot order"""
        from . import xr_shim as xr
        starts = np.array([str(np.datetime64(t, "s")) for t in start_times])
        attrs = dict(model=str(model), members=int(members), first_start=str(starts[0]), last_start=str(starts[-1]),
                     n_dates=len(starts))
        common = dict(lead_time=np.asarray(leads_hours, dtype=np.float64), region=np.array(list(regions)),
                      channel=np.array(list(channels)))
        card = xr.DataArray(np.ascontiguousarray(np.moveaxis(period_metrics(sums, members), -1, 1)),
                            dims=["lead_time", "metric", "region", "channel"],
                            coords=dict(common, metric=np.array(METRICS)), attrs=dict(attrs))
        cards = xr.DataArray(np.ascontiguousarray(np.moveaxis(metrics_from_sums(sums, members), -1, 2)),
                             dims=["start_time", "lead_time", "metric", "region", "channel"],
                             coords=dict(common, start_time=starts, metric=np.array(METRICS)), attrs=dict(attrs))
        rank = xr.DataArray(np.ascontiguousarray(np.asarray(hist, dtype=np.float64).mean(axis=0)),
                            dims=["lead_time", "region", "channel", "rank"],
                            coords=dict(common, rank=np.arange(members + 1, dtype=np.float64)), attrs=dict(attrs))
        mp = None
        if maps is not None:
            mp = xr.DataArray(np.ascontiguousarray(np.swapaxes(map_metrics(maps, len(starts), members), 1, 2)),
                              dims=["lead_time", "metric", "channel", "lat", "lon"],
                              coords=dict(lead_time=np.array([n * step_hours for n in map_leads], dtype=np.float64),
                                          metric=np.array(MAP_METRICS), channel=np.array(list(map_channels)),
                                          lat=np.asarray(lat, dtype=np.float64), lon=np.asarray(lon, dtype=np.float64)),
                              attrs=dict(attrs))
        return cls(card, cards, rank, mp)


# ---- model comparison -------------------------------------------------------------------------------------------------------
DIFF_METRICS = ("rmse", "crps", "acc")
DIFF_STATS = ("mean", "ci_low", "ci_high", "p_value", "n_eff")


def paired_difference_stats(d):
    """fp64 (..., 5) statistics (``DIFF_STATS`` order) of per-date score differences d, fp64 (D, ...) along the first
    axis, with dates equally spaced.  d̄ the mean, s the sample standard deviation (ddof 1), r1 = sum_{t<D-1} (d_t - d̄)
    (d_{t+1} - d̄) / sum_t (d_t - d̄)^2 the lag-1 autocorrelation (0 when the denominator is 0), n_eff = D (1 - r1) /
    (1 + r1) clipped to [2, D] (AR(1) variance inflation, Geer 2016), se = s / sqrt(n_eff); then p = 2 stdtr(n_eff - 1,
    -|d̄ / se|) and the 95 % interval d̄ -/+ stdtrit(n_eff - 1, 0.975) se.  s = 0 gives the interval [d̄, d̄] with p = 1
    when d̄ = 0 and 0 otherwise.  With D < 3 every statistic but the mean is NaN; a NaN d_t makes every statistic NaN."""
    from scipy.special import stdtr, stdtrit
    d = np.asarray(d, dtype=np.float64)
    D = d.shape[0]
    out = np.full(d.shape[1:] + (len(DIFF_STATS),), np.nan)
    mean = d.sum(axis=0) / D
    out[..., 0] = mean
    if D < 3:
        return out
    dev = d - mean
    den = (dev * dev).sum(axis=0)
    num = (dev[:-1] * dev[1:]).sum(axis=0)
    s = np.sqrt(den / (D - 1))
    with np.errstate(divide="ignore", invalid="ignore"):
        r1 = np.where(den > 0.0, num / den, 0.0)
        n_eff = np.clip(D * (1.0 - r1) / (1.0 + r1), 2.0, float(D))
        se = s / np.sqrt(n_eff)
        q = stdtrit(n_eff - 1.0, 0.975)
        p = 2.0 * stdtr(n_eff - 1.0, -np.abs(mean / se))
    flat = s == 0.0
    out[..., 1] = np.where(flat, mean, mean - q * se)
    out[..., 2] = np.where(flat, mean, mean + q * se)
    out[..., 3] = np.where(flat, np.where(mean == 0.0, 1.0, 0.0), p)
    out[..., 4] = n_eff
    out[np.isnan(d).any(axis=0)] = np.nan
    return out


def paired_differences(cards_a, cards_b):
    """fp64 (metric, stat, lead_time, region, channel) statistics (``DIFF_METRICS`` x ``DIFF_STATS``) of the per-date
    differences a - b of two entries' per-date cards, fp64 (start_time, lead_time, metric, region, channel) in ``METRICS``
    order: negative means a is better for rmse and crps, positive for acc."""
    a, b = np.asarray(cards_a, dtype=np.float64), np.asarray(cards_b, dtype=np.float64)
    pick = [METRICS.index(m) for m in DIFF_METRICS]
    st = paired_difference_stats(a[:, :, pick] - b[:, :, pick])      # (lead, metric, region, channel, stat)
    return np.ascontiguousarray(np.moveaxis(np.moveaxis(st, -1, 0), 2, 0))


class ModelComparison:
    """What ``GlobalEnsemble.compare`` returns: several models and their pooled ensemble verified over the same start
    dates against one truth.
        entries      the model names, then "pooled"
        scores       {entry: PeriodScores} (members: M per model, K M for the pooled entry)
        card         fp64 (model, lead_time, metric, region, channel): the entries' period cards stacked
        differences  fp64 (pair, metric, stat, lead_time, region, channel): ``paired_differences`` of the per-date cards
                     of every pair "a-b" with a before b in ``entries``, over ``DIFF_METRICS`` and ``DIFF_STATS``"""

    def __init__(self, entries, scores, card, differences):
        self.entries, self.scores, self.card, self.differences = list(entries), dict(scores), card, differences

    def __repr__(self) -> str:
        return f"ModelComparison(entries={self.entries},dates={self.card.attrs.get('n_dates')})"

    @property
    def pairs(self):
        return [str(p) for p in np.asarray(self.differences.coords["pair"])]

    @classmethod
    def build(cls, scores: dict):
        """from {entry: PeriodScores} in entry order, all over the same dates, leads, regions and channels"""
        from . import xr_shim as xr
        entries = list(scores)
        first = scores[entries[0]].card
        attrs = {k: v for k, v in first.attrs.items() if k not in ("model", "members")}
        attrs["members"] = [int(scores[e].card.attrs["members"]) for e in entries]
        coords = {d: np.asarray(first.coords[d]) for d in first.dims}
        card = xr.DataArray(np.stack([scores[e].card.values for e in entries]),
                            dims=["model"] + list(first.dims), coords=dict(coords, model=np.array(entries)),
                            attrs=dict(attrs))
        pairs = [(a, b) for i, a in enumerate(entries) for b in entries[i + 1:]]
        diff = np.stack([paired_differences(scores[a].cards.values, scores[b].cards.values) for a, b in pairs])
        differences = xr.DataArray(diff, dims=["pair", "metric", "stat", "lead_time", "region", "channel"],
                                   coords=dict(pair=np.array([f"{a}-{b}" for a, b in pairs]),
                                               metric=np.array(DIFF_METRICS), stat=np.array(DIFF_STATS),
                                               lead_time=coords["lead_time"], region=coords["region"],
                                               channel=coords["channel"]), attrs=dict(attrs))
        return cls(entries, scores, card, differences)
