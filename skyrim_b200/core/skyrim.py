"""Facade — mirrors /root/reference/skyrim/core/skyrim.py:12-95 (same constructor, ``predict``,
``forecast``, ``list_available_models``)."""
from __future__ import annotations

import datetime

from loguru import logger

from .models import MODELS
from .models.base import GlobalModel, GlobalPrediction, adjust_lead_time
from .models.ensemble import GlobalEnsemble


class Skyrim:
    def __init__(self, *model_names: str, ic_source="synthetic", **model_kw):
        missing_names = [name for name in model_names if name not in MODELS]
        if missing_names:
            raise ValueError(f"Invalid model name(s): {missing_names}")
        if not model_names:
            raise NotImplementedError("give at least one model name")
        self.model_names = model_names
        self.ic_source = ic_source
        if len(model_names) > 1:
            # the reference's GlobalEnsemble (ensemble.py:10-128): every model on this GPU, reduced on the device
            self.model: GlobalModel | GlobalEnsemble = GlobalEnsemble(model_names, ic_source=ic_source, **model_kw)
        else:
            self.model = MODELS[model_names[0]](ic_source=ic_source, **model_kw)
        logger.debug(f"Initialized {self.model} model with initial conditions from {ic_source}")

    def __repr__(self) -> str:
        return f"Skyrim(models={self.model_names},ic={self.ic_source})"

    @staticmethod
    def list_available_models():
        return list(MODELS.keys())

    def forecast(self, start_time: datetime.datetime, n_steps: int = 4, channels: list = []):
        start_time = start_time.replace(second=0, microsecond=0)
        return self.model.forecast(start_time=start_time, n_steps=n_steps, channels=channels)

    def predict(self, date: str, time: str, lead_time: int = 6, save: bool = False, save_config: dict = {}):
        """Predict a single lead-time snapshot, optionally saving every intermediate step
        (skyrim.py:60-95: YYYYMMDD / HHMM parsing, lead time floored to a multiple of 6 h)."""
        start_time = datetime.datetime(int(date[:4]), int(date[4:6]), int(date[6:8]), int(time[:2]), int(time[2:4]))
        lead_time = adjust_lead_time(lead_time, step_size=6)
        logger.debug(f"Lead time adjusted to nearest multiple of 6: {lead_time} hours")
        n_steps = int(lead_time // (self.model.time_step.total_seconds() / 3600))
        logger.debug(f"Number of prediction steps: {n_steps}")
        pred, output_paths = self.model.rollout(start_time=start_time, n_steps=n_steps, save=save,
                                                save_config=save_config)
        logger.debug("Prediction completed successfully")
        return GlobalPrediction(pred, model_name=self.model_names), output_paths

    def predict_ensemble(self, date: str, time: str, lead_time: int = 6, members: int = 4, **kw):
        """Perturbed-initial-condition ensemble forecast reduced to per-step statistics on the GPU: the date, time and lead
        time are read as ``predict`` reads them, ``kw`` goes to ``GlobalModel.predict_ensemble`` (perturbation, amp, seed,
        quantiles, events, channels, save, save_config, grf); with several models, to ``GlobalEnsemble.predict_ensemble``
        (``members`` per model).  Returns (GlobalEnsemblePrediction, paths)."""
        start_time = datetime.datetime(int(date[:4]), int(date[4:6]), int(date[6:8]), int(time[:2]), int(time[2:4]))
        n_steps = self.model.time_steps(lead_time)
        logger.debug(f"Ensemble of {members} members, {n_steps} steps")
        return self.model.predict_ensemble(start_time=start_time, n_steps=n_steps, members=members, **kw)

    def score(self, date: str, time: str, lead_time: int = 6, **kw):
        """Forecast verification (``GlobalModel.score``): the date, time and lead time are read as ``predict`` reads them,
        ``kw`` goes to ``GlobalModel.score`` (truth, climatology, members, perturbation, amp, seed, grf, channels, regions,
        save, save_config).  Returns (scorecard DataArray (lead_time, metric, region, channel), paths)."""
        start_time = datetime.datetime(int(date[:4]), int(date[4:6]), int(date[6:8]), int(time[:2]), int(time[2:4]))
        n_steps = self.model.time_steps(lead_time)
        logger.debug(f"Scoring {n_steps} steps")
        return self.model.score(start_time=start_time, n_steps=n_steps, **kw)

    def score_period(self, start: str, end: str, time: str = "0000", every: int = 24, lead_time: int = 6, **kw):
        """Verification over a period (``GlobalModel.score_period``): start dates from ``start`` (YYYYMMDD) at ``time``
        (HHMM) every ``every`` hours (a multiple of 6) through the date ``end``, inclusive; the lead time is read as
        ``predict`` reads it; ``kw`` goes to ``GlobalModel.score_period`` (truth, climatology, members, perturbation, amp,
        seed, grf, channels, regions, map_leads, map_channels, save, save_config).  Returns (PeriodScores, paths)."""
        return self.model.score_period(start_times=period_start_times(start, end, time, every),
                                       n_steps=self.model.time_steps(lead_time), **kw)

    def compare(self, start: str, end: str | None = None, time: str = "0000", every: int = 24, lead_time: int = 6, **kw):
        """Head-to-head verification of several models and their pooled ensemble (``GlobalEnsemble.compare``): start
        dates as ``score_period`` reads them, ``end = None`` meaning the single date ``start``; ``kw`` goes to
        ``GlobalEnsemble.compare`` (truth, climatology, members, perturbation, amp, seed, grf, channels, regions,
        map_leads, map_channels, save, save_config).  Returns (ModelComparison, paths)."""
        if not isinstance(self.model, GlobalEnsemble):
            raise ValueError(f"compare needs two to four models, e.g. Skyrim('pangu', 'graphcast'); this Skyrim runs "
                             f"{self.model_names[0]} alone")
        return self.model.compare(start_times=period_start_times(start, start if end is None else end, time, every),
                                  n_steps=self.model.time_steps(lead_time), **kw)


    def predict_sites(self, date: str, time: str, lead_time: int = 6, sites=None, **kw):
        """Forecast at sites (``GlobalModel.predict_sites``): the date, time and lead time are read as ``predict`` reads
        them, ``kw`` goes to ``GlobalModel.predict_sites`` (members, method, channels, quantiles, events, perturbation,
        amp, seed, grf, save, save_config).  Returns (SiteForecast, paths)."""
        start_time = datetime.datetime(int(date[:4]), int(date[4:6]), int(date[6:8]), int(time[:2]), int(time[2:4]))
        return self.model.predict_sites(start_time=start_time, n_steps=self.model.time_steps(lead_time), sites=sites, **kw)

    def score_sites(self, date: str, time: str, lead_time: int = 6, observations=None, until: str | None = None,
                    every: int = 24, **kw):
        """Verification against station observations (``GlobalModel.score_sites``) over the start dates from ``date`` at
        ``time`` every ``every`` hours through ``until`` (default: ``date`` alone), as ``score_period`` reads them; ``kw``
        goes to ``GlobalModel.score_sites`` (members, method, channels, perturbation, amp, seed, grf, save,
        save_config).  Returns (SiteScores, paths)."""
        return self.model.score_sites(start_times=period_start_times(date, until or date, time, every),
                                      n_steps=self.model.time_steps(lead_time), observations=observations, **kw)


def period_start_times(start: str, end: str, time: str = "0000", every: int = 24):
    """start times from ``start`` + ``time`` every ``every`` hours (a positive multiple of 6) while their date is at most
    ``end``"""
    if every <= 0 or every % 6:
        raise ValueError(f"every = {every} h: a positive multiple of 6 h needed")
    t = datetime.datetime(int(start[:4]), int(start[4:6]), int(start[6:8]), int(time[:2]), int(time[2:4]))
    stop = datetime.datetime(int(end[:4]), int(end[4:6]), int(end[6:8])) + datetime.timedelta(days=1)
    if t >= stop:
        raise ValueError(f"end date {end} lies before the first start time {t}")
    out = []
    while t < stop:
        out.append(t)
        t += datetime.timedelta(hours=every)
    return out
