"""Forecasts at sites and their verification against station observations.  The device samples every member at the sites
(``engine.sample_sites``, include/skyrim_b200.h sky_sample_sites) and accumulates the site scores
(``engine.site_scores``); this module reads the sites and the observations, and shapes the results.

Sites are a dict ``{name: (lat, lon)}``, a tuple ``(names, lats, lons)`` of arrays, or a CSV file of ``name,lat,lon``
rows (a header row is skipped), in degrees north and east.  Observations are a DataArray (time, site, channel) in the
model's units (K, Pa, m s^-1), NaN where missing, with ``lat`` / ``lon`` coordinates along ``site``.

Site scores are formed per (lead, site, channel) from the observations used there (``count``), as
``scores.metrics_from_sums`` forms the scalars with w = count (each observation of weight 1); there is no acc at sites:

    bias       mean e, e = x_bar - y             rmse       sqrt(mean e^2)
    spread     sqrt(mean sum_m (x_m - x_bar)^2 / (M - 1))       ssr  sqrt((M + 1) / M) spread / rmse
    crps       mean [(1/M) sum_m |x_m - y| - G / M^2]           crps_fair  the same with G / (M (M - 1))

A site and lead without observations has count 0 and NaN metrics.
"""
from __future__ import annotations

import csv
from collections import Counter
from pathlib import Path

import numpy as np

from . import scores as S

SITE_METRICS = ("bias", "rmse", "spread", "ssr", "crps", "crps_fair")
SITE_TERMS = ("n", "e", "e2", "var", "mae", "g")   # the six accumulators of sky_site_scores, in order
RETURN_LIMIT = 2 ** 31                            # bytes of arrays predict_sites returns


def read_sites(sites):
    """(names, lat fp64, lon fp64) of ``sites`` (module docstring), refusing duplicate names, a lat outside [-90, 90] and
    non-finite coordinates"""
    if isinstance(sites, (str, Path)):
        rows = []
        with open(sites, newline="") as f:
            for i, row in enumerate(csv.reader(f)):
                row = [c.strip() for c in row]
                if not row or not any(row):
                    continue
                if len(row) != 3:
                    raise ValueError(f"{sites} line {i + 1}: {len(row)} fields, name,lat,lon needed")
                try:
                    rows.append((row[0], float(row[1]), float(row[2])))
                except ValueError:
                    if i == 0 and not rows:   # a header
                        continue
                    raise ValueError(f"{sites} line {i + 1}: lat and lon must be numbers ({row[1]!r}, {row[2]!r})")
        names, lat, lon = [r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows]
    elif isinstance(sites, dict):
        names = [str(k) for k in sites]
        try:
            lat, lon = [float(v[0]) for v in sites.values()], [float(v[1]) for v in sites.values()]
        except (TypeError, IndexError):
            raise ValueError("a site dict maps each name to (lat, lon)")
    elif isinstance(sites, (tuple, list)) and len(sites) == 3:
        names, lat, lon = ([str(n) for n in sites[0]], np.asarray(sites[1], dtype=np.float64).reshape(-1),
                           np.asarray(sites[2], dtype=np.float64).reshape(-1))
    else:
        raise TypeError("sites must be a dict {name: (lat, lon)}, a tuple (names, lats, lons) or a CSV file name,lat,lon")
    lat, lon = np.asarray(lat, dtype=np.float64), np.asarray(lon, dtype=np.float64)
    if not len(names):
        raise ValueError("no sites given")
    if not len(names) == lat.size == lon.size:
        raise ValueError(f"{len(names)} names, {lat.size} latitudes and {lon.size} longitudes: one of each per site")
    dup = sorted(n for n, k in Counter(names).items() if k > 1)
    if dup:
        raise ValueError(f"duplicate site name(s) {dup}")
    bad = [n for n, a, b in zip(names, lat, lon) if not (np.isfinite(a) and np.isfinite(b) and -90.0 <= a <= 90.0)]
    if bad:
        raise ValueError(f"site(s) {bad}: lat must lie in [-90, 90] and lat, lon must be finite")
    return names, lat, lon


def check_equiangular(lat, lon):
    """refuses a grid that is not the equiangular one of ``timeloop.equiangular_grid`` (the site stencil assumes it)"""
    lat, lon = np.asarray(lat, dtype=np.float64), np.asarray(lon, dtype=np.float64)
    want_lat, want_lon = np.linspace(90.0, -90.0, lat.size), np.arange(lon.size) * (360.0 / max(lon.size, 1))
    if lat.size < 2 or not (np.allclose(lat, want_lat, rtol=0, atol=1e-9) and np.allclose(lon, want_lon, rtol=0, atol=1e-9)):
        raise ValueError(f"the model grid ({lat.size} x {lon.size}) is not equiangular (lat 90 .. -90, lon from 0): sites "
                         "are sampled on that grid only")


def read_observations(obs, channels=None):
    """(names, lat, lon, times datetime64[s], channel names, values fp32 (time, site, channel)) of an observation
    DataArray (module docstring), with ``channels`` selected (default: all of them)"""
    if not (hasattr(obs, "dims") and tuple(obs.dims) == ("time", "site", "channel")):
        raise ValueError(f"observations dims {tuple(getattr(obs, 'dims', ()))}: (time, site, channel) needed")
    for c in ("time", "site", "channel", "lat", "lon"):
        if c not in obs.coords:
            raise ValueError(f"observations lack the {c!r} coordinate (lat / lon lie along site)")
    names = [str(n) for n in np.asarray(obs.coords["site"])]
    lat = np.asarray(obs.coords["lat"], dtype=np.float64).reshape(-1)
    lon = np.asarray(obs.coords["lon"], dtype=np.float64).reshape(-1)
    names, lat, lon = read_sites((names, lat, lon))
    times = np.asarray(obs.coords["time"]).astype("datetime64[s]")
    if len(set(times.tolist())) != times.size:
        raise ValueError("observations hold a valid time twice")
    have = [str(c) for c in np.asarray(obs.coords["channel"])]
    sel = list(have) if channels is None else list(channels)
    missing = [c for c in sel if c not in have]
    if missing:
        raise ValueError(f"observations lack channel(s) {missing}")
    vals = np.asarray(obs.values, dtype=np.float32)[:, :, [have.index(c) for c in sel]]
    return names, lat, lon, times, sel, np.ascontiguousarray(vals)


def _sums9(terms):
    """fp64 (..., 9) sums of ``scores.SUMS`` from fp64 (..., 6) site terms (the climatology sums NaN)"""
    t = np.asarray(terms, dtype=np.float64)
    return np.concatenate([t, np.full(t.shape[:-1] + (3,), np.nan)], axis=-1)


def site_metrics(terms, members: int):
    """fp64 (..., 6) ``SITE_METRICS`` from fp64 (..., 6) terms summed over observations (w = the count)"""
    pick = [S.METRICS.index(k) for k in SITE_METRICS]
    return S.metrics_from_sums(_sums9(terms), members)[..., pick]


class SiteForecast:
    """What ``GlobalModel.predict_sites`` returns.
        values  fp32 (time, member, site, channel): every member at every site, time from lead 0
        stats   fp32 (time, statistic, site, channel): mean, spread and quantiles, or None with one member
        prob    fp32 (time, event, site): exceedance probabilities, or None without events
    Each has the site's ``lat`` / ``lon`` along ``site``."""

    def __init__(self, values, stats=None, prob=None, model: str = "", members: int = 1):
        self.values, self.stats, self.prob, self.model, self.members = values, stats, prob, model, members

    def __repr__(self) -> str:
        return f"SiteForecast(model={self.model},members={self.members},shape={tuple(self.values.shape)})"

    @property
    def sites(self):
        return [str(n) for n in np.asarray(self.values.coords["site"])]

    def point(self, site: str, channel: str):
        """(time, member) series of ``channel`` at ``site``"""
        return self.values.sel(site=site, channel=channel)

    def wind_speed(self, site: str, pressure_level=10):
        """(time, member) wind speed sqrt(u^2 + v^2) at ``site`` from each member's interpolated u and v: channels
        u<level> / v<level> (``pressure_level`` 1000 for u1000, "10m" or 10 for u10m)"""
        level = "10m" if str(pressure_level) in ("10", "10m") else str(pressure_level)
        u, v = self.point(site, f"u{level}"), self.point(site, f"v{level}")
        uv = np.asarray(u.values, dtype=np.float64), np.asarray(v.values, dtype=np.float64)
        from . import xr_shim as xr
        return xr.DataArray(np.sqrt(uv[0] ** 2 + uv[1] ** 2).astype(np.float32), dims=list(u.dims),
                            coords={d: np.asarray(u.coords[d]) for d in u.dims})


class SiteScores:
    """What ``GlobalModel.score_sites`` returns: site scores over one or more start dates.
        card   fp64 (lead_time, metric, channel): over all sites and dates
        cards  fp64 (start_time, lead_time, metric, channel): per start date
        sites  fp64 (lead_time, metric, site, channel): per site over the dates
        count  (lead_time, site, channel): the number of observations used
    metrics ``SITE_METRICS``; ``sites`` and ``count`` have the site's ``lat`` / ``lon`` along ``site``."""

    def __init__(self, card, cards, sites, count):
        self.card, self.cards, self.sites, self.count = card, cards, sites, count

    @classmethod
    def build(cls, sums, acc, members: int, start_times, leads_hours, names, lat, lon, channels, model: str):
        """from host fp64 sums (date, lead, channel, 6) and per-site accumulators (lead, channel, site, 6) summed over the
        dates"""
        from . import xr_shim as xr
        sums, acc = np.asarray(sums, dtype=np.float64), np.asarray(acc, dtype=np.float64)
        starts = np.array([str(np.datetime64(t, "s")) for t in start_times])
        attrs = dict(model=str(model), members=int(members), first_start=str(starts[0]), last_start=str(starts[-1]),
                     n_dates=len(starts))
        lead = np.asarray(leads_hours, dtype=np.float64)
        ch, met = np.array(list(channels)), np.array(SITE_METRICS)
        where = dict(site=np.array(list(names)), lat=("site", np.asarray(lat, np.float64)),
                     lon=("site", np.asarray(lon, np.float64)))
        card = xr.DataArray(np.ascontiguousarray(np.moveaxis(site_metrics(sums.sum(axis=0), members), -1, 1)),
                            dims=["lead_time", "metric", "channel"], coords=dict(lead_time=lead, metric=met, channel=ch),
                            attrs=dict(attrs))
        cards = xr.DataArray(np.ascontiguousarray(np.moveaxis(site_metrics(sums, members), -1, 2)),
                             dims=["start_time", "lead_time", "metric", "channel"],
                             coords=dict(start_time=starts, lead_time=lead, metric=met, channel=ch), attrs=dict(attrs))
        m = site_metrics(acc, members)                                       # (lead, channel, site, metric)
        per_site = xr.DataArray(np.ascontiguousarray(np.transpose(m, (0, 3, 2, 1))),
                                dims=["lead_time", "metric", "site", "channel"],
                                coords=dict(where, lead_time=lead, metric=met, channel=ch), attrs=dict(attrs))
        count = xr.DataArray(np.ascontiguousarray(np.swapaxes(acc[..., 0], 1, 2)), dims=["lead_time", "site", "channel"],
                             coords=dict(where, lead_time=lead, channel=ch), attrs=dict(attrs))
        return cls(card, cards, per_site, count)
