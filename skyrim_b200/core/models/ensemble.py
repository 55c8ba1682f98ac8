"""GlobalEnsemblePrediction — the class /root/reference/skyrim/core/models/ensemble.py:131-133 names and leaves empty: the
per-step statistics of a perturbed-initial-condition ensemble (``GlobalModel.predict_ensemble``), reduced on the GPU."""
from __future__ import annotations

import numpy as np

from .base import GlobalPrediction


def quantile_name(q: float) -> str:
    """"q0.1" for q = 0.1: the shortest decimal that reads back as the fp64 quantile"""
    return "q" + np.format_float_positional(float(q), trim="-")


def event_name(channel: str, threshold: float) -> str:
    """"t2m>273.15": the shortest decimal of the fp32 threshold the kernel compares against"""
    return f"{channel}>" + np.format_float_positional(np.float32(threshold), trim="-")


class GlobalEnsemblePrediction:
    """``stats``: DataArray (time, statistic, channel, lat, lon) with statistic = ["mean", "spread", "q0.1", ...];
    ``probability``: DataArray (time, event, lat, lon) with event = ["t2m>273.15", ...], or None without events.  ``time``
    holds the previous and the last step, as a rollout's prediction does."""

    def __init__(self, stats, probability=None, model_name: str = "", members: int = 0):
        self.stats, self.probability, self.model, self.members = stats, probability, model_name, members

    def __repr__(self) -> str:
        ev = 0 if self.probability is None else len(self.events)
        return (f"GlobalEnsemblePrediction(model={self.model},members={self.members},statistics={self.statistics},"
                f"channels={len(self.channels)},events={ev})")

    @property
    def statistics(self):
        return [str(s) for s in np.asarray(self.stats.coords["statistic"])]

    @property
    def channels(self):
        return [str(c) for c in np.asarray(self.stats.coords["channel"])]

    @property
    def events(self):
        return [] if self.probability is None else [str(e) for e in np.asarray(self.probability.coords["event"])]

    def _statistic(self, name: str) -> GlobalPrediction:
        if name not in self.statistics:
            raise KeyError(f"statistic {name!r} was not computed (have {self.statistics})")
        return GlobalPrediction(self.stats.sel(statistic=name), model_name=self.model)

    @property
    def mean(self) -> GlobalPrediction:
        return self._statistic("mean")

    @property
    def spread(self) -> GlobalPrediction:
        return self._statistic("spread")

    def quantile(self, q: float) -> GlobalPrediction:
        return self._statistic(quantile_name(q))

    def probability_of(self, channel: str, threshold: float, n_step: int = 1) -> np.ndarray:
        """(lat, lon) fp32 P(channel > threshold) at time slice ``n_step`` (1: the last step)"""
        name = event_name(channel, threshold)
        if name not in self.events:
            raise KeyError(f"event {name!r} was not computed (have {self.events})")
        return np.asarray(self.probability.sel(event=name).isel(time=n_step).values)

    def point(self, lat: float, lon: float, channel: str, statistic: str = "mean", n_step: int = 1) -> float:
        """one statistic at the grid point nearest (lat, lon); lon < 0 wraps as in GlobalPrediction.point"""
        if lon < 0:
            lon = 360 + lon
        if statistic not in self.statistics or channel not in self.channels:
            raise KeyError(f"({statistic!r}, {channel!r}) not in {self.statistics} x {self.channels}")
        lats, lons = np.asarray(self.stats.coords["lat"]), np.asarray(self.stats.coords["lon"])
        i, j = int(np.abs(lats - lat).argmin()), int(np.abs(lons - lon).argmin())
        v = np.asarray(self.stats.values)[n_step, self.statistics.index(statistic), self.channels.index(channel), i, j]
        return float(v)
