"""GlobalModel / GlobalPrediction — mirrors /root/reference/skyrim/core/models/base.py
(adjust_lead_time :13-15, GlobalModel :18-146, GlobalPrediction :149-274,
GlobalPredictionRollout :277-303), with the back-end replaced by the CUDA step engine."""
from __future__ import annotations

import datetime
import functools
import time
from pathlib import Path
from typing import List

import numpy as np
from loguru import logger

from ... import xr_shim as xr
from ...common import generate_forecast_id, save_forecast
from .utils import run_basic_inference


def adjust_lead_time(lead_time: int, step_size: int = 6):
    """Adjust lead time to the nearest multiple of step_size (base.py:13-15)."""
    return max(step_size, (lead_time // step_size) * step_size)


class SyntheticDataSource:
    """Seeded synthetic initial conditions (SURVEY.md §8(d)).  The reference's sources
    (cds / gfs / ifs, libs/ic/__init__.py:25-34) download GRIB over the network and stay with
    the reference package; any object with ``source[time] -> DataArray(channel, lat, lon)`` works."""

    def __init__(self, channel_names, nlat=721, nlon=1440, seed=0):
        self.channel_names, self.nlat, self.nlon, self.seed = list(channel_names), nlat, nlon, seed

    def __getitem__(self, t):
        from ...weights import synthetic_state
        from ...timeloop import equiangular_grid
        g = equiangular_grid(self.nlat, self.nlon)
        x = synthetic_state(self.channel_names, self.nlat, self.nlon, self.seed)
        return xr.DataArray(x, dims=["channel", "lat", "lon"],
                            coords=dict(channel=np.array(self.channel_names), lat=np.array(g.lat), lon=np.array(g.lon)))


class GlobalModel:
    # channels that are forcings rather than forecasts (GraphCast's toa radiation): never scored
    forcing_channels: tuple = ()

    def __init__(self, model_name: str, ic_source: str = "synthetic", **engine_kw):
        clock = time.time()
        self.model_name = model_name
        self.ic_source = ic_source
        self.engine_kw = engine_kw
        logger.debug(f"Building {model_name} model...")
        self.model = self.build_model()
        logger.debug(f"Building {self.ic_source} data source...")
        self.data_source = self.build_datasource()
        logger.success(f"Initialized {model_name} in {time.time() - clock:.1f} seconds")

    def build_model(self):
        raise NotImplementedError

    def build_datasource(self):
        if self.ic_source == "synthetic":
            return SyntheticDataSource(self.model.in_channel_names, len(self.model.grid.lat), len(self.model.grid.lon))
        if hasattr(self.ic_source, "__getitem__") and not isinstance(self.ic_source, str):
            return self.ic_source  # a user-supplied data source object
        raise NotImplementedError(
            f"ic_source='{self.ic_source}' downloads initial conditions over the network (reference "
            "libs/ic/__init__.py:25-34); pass ic_source='synthetic' or a data-source object")

    def release_model(self):
        self.model.engine.close()

    @property
    def time_step(self):
        return self.model.time_step

    def time_steps(self, lead_time: int):
        lead_time = adjust_lead_time(lead_time, step_size=6)
        return int(lead_time // (self.time_step.total_seconds() / 3600))

    @property
    def in_channel_names(self):
        return self.model.in_channel_names

    @property
    def out_channel_names(self):
        return self.model.out_channel_names

    def __repr__(self) -> str:
        return f"{self.__class__.__name__}(model_name={self.model_name})"

    def predict_one_step(self, start_time: datetime.datetime, initial_condition=None):
        return run_basic_inference(model=self.model, n=1, data_source=self.data_source, time=start_time,
                                   x=initial_condition)

    def forecast(self, start_time: datetime.datetime, n_steps: int = 3, channels: List[str] = []):
        """All steps from the IC in one device-resident generator (base.py:94-117)."""
        da = run_basic_inference(model=self.model, n=n_steps, data_source=self.data_source, time=start_time, x=None)
        return da.sel(channel=list(channels)) if channels else da

    def rollout(self, start_time: datetime.datetime, n_steps: int = 3, save: bool = True, save_config: dict = {},
                initial_condition=None):
        """Chained 6-h steps; returns (last prediction with 2 time slices, paths) like base.py:119-146.
        Unlike the reference (which round-trips the state through the host and re-uploads it every
        step, utils.py:24-31), the state stays resident in HBM; only what is saved / returned is
        copied back.  ``initial_condition`` (DataArray / path) resumes a rollout (TODO at base.py:127)."""
        import torch
        pred, output_paths, source = None, [], self.ic_source if isinstance(self.ic_source, str) else "file"
        save_config = dict(save_config)
        save_config.setdefault("forecast_id", generate_forecast_id())
        if initial_condition is None:
            ic = self.data_source[start_time]
        else:
            ic = xr.open_dataarray(initial_condition) if isinstance(initial_condition, str) else initial_condition
            source = "file"
        vals = np.asarray(ic.values, dtype=np.float32)
        vals = vals[-1] if vals.ndim == 4 else vals
        x = torch.from_numpy(np.ascontiguousarray(vals))[None, None]

        def pair(t0, a0, t1, a1):
            return xr.DataArray(np.stack([a0, a1]), dims=["time", "channel", "lat", "lon"],
                                coords=dict(time=np.array([np.datetime64(t0, "s"), np.datetime64(t1, "s")]),
                                            channel=np.array(self.out_channel_names),
                                            lat=np.array(self.model.grid.lat), lon=np.array(self.model.grid.lon)))

        if not save and n_steps > 0 and hasattr(self.model, "last_slices"):
            # a schedule that can skip slices (Pangu's hierarchical one) computes only the two returned ones
            (t_prev, prev), (t_cur, cur) = self.model.last_slices(start_time, x, n_steps)
            logger.success(f"Rollout to step {n_steps} completed")
            return pair(t_prev, prev.cpu().numpy()[0], t_cur, cur.cpu().numpy()[0]), output_paths
        if save and hasattr(self.model, "iter_host"):
            # every state is needed on the host: device->host copy of step n overlaps step n+1 (timeloop.iter_host)
            gen = ((t, h[0].numpy(), None) for t, h in self.model.iter_host(start_time, x, n_steps))
            to_host = lambda a: a
        else:
            gen = self.model(start_time, x)
            to_host = lambda a: a.cpu().numpy()[0]
        t_prev, prev, _ = next(gen)
        prev_host = np.array(to_host(prev))   # own copy: the iterator's host buffers are a ring of two
        for n in range(n_steps):
            t_cur, cur, _ = next(gen)
            need_host = save or n == n_steps - 1
            if need_host:
                pred = pair(t_prev, prev_host, t_cur, to_host(cur))
                if save:
                    output_paths.append(save_forecast(pred, self.model_name, t_prev, t_cur, source, config=save_config))
                prev_host = pred.values[1]
            t_prev, source = t_cur, "file"
            logger.success(f"Rollout step {n+1}/{n_steps} completed")
        return pred, output_paths

    def _ensemble_initial_state(self, start_time: datetime.datetime):
        """(unperturbed state (C, H, W), per-channel perturbation sigma (C,), offset of the reduced channels in the state)"""
        from ...weights import channel_stats
        vals = np.asarray(self.data_source[start_time].values, dtype=np.float32)
        return np.ascontiguousarray(vals[-1] if vals.ndim == 4 else vals), channel_stats(self.in_channel_names)[1], 0

    def predict_ensemble(self, start_time: datetime.datetime, n_steps: int, members: int, perturbation: str = "spherical_grf",
                         amp: float = 0.05, seed: int = 0, quantiles=(), events: dict = {}, channels: List[str] = [],
                         save: bool = False, save_config: dict = {}, grf: dict | None = None):
        """Perturbed-initial-condition ensemble of ``members`` (1..64) on this model's GPU, reduced on the device to
        per-step statistics: mean, spread and ``quantiles`` of ``channels`` (default: save_config's filter_vars, else all),
        and P(x > t) for ``events`` = {channel: threshold or [thresholds]} (their channels are reduced too).  Member m is
        the state ``EnsembleRunner(members_per_gpu=members, rank=0, amp=amp, seed=seed, perturbation=...)`` produces;
        "spherical_grf" defaults to the degree limit min(180, (nlat - 1) // 2) unless ``grf`` says otherwise.  Only the
        statistics are copied to the host, each step's copy under the next step.  ``save`` writes one netCDF file of
        statistics per step (model "<model>-ens<M>") and, with events, one of probabilities ("<model>-ens<M>-prob").
        Returns (GlobalEnsemblePrediction of the last step with 2 time slices, paths)."""
        from ... import engine as E
        from .ensemble import GlobalEnsemblePrediction, event_name, quantile_name
        names = list(self.out_channel_names)
        if not 1 <= members <= E.ENS_MAX_MEMBERS:
            raise ValueError(f"members = {members} must lie in [1, {E.ENS_MAX_MEMBERS}]")
        if n_steps < 1:
            raise ValueError(f"n_steps = {n_steps} must be at least 1")
        q = [float(v) for v in quantiles]
        if len(q) > E.ENS_MAX_QUANTILES or not all(0.0 <= v <= 1.0 for v in q):
            raise ValueError(f"quantiles {q}: at most {E.ENS_MAX_QUANTILES}, each in [0, 1]")
        ev = {c: [float(t) for t in np.atleast_1d(thr)] for c, thr in dict(events).items()}
        filt = list(save_config.get("filter_vars", ()))
        unknown = [c for c in list(channels) + filt + list(ev) if c not in names]
        if unknown:
            raise ValueError(f"unknown channel(s) {unknown} for {self.model_name}")
        if not all(np.isfinite(t) for ts in ev.values() for t in ts):
            raise ValueError(f"event thresholds must be finite: {ev}")
        if save and save_config.get("file_type", "netcdf") == "zarr":
            raise ValueError("ensemble statistics are written as netCDF only: the zarr writer holds one variable per "
                             "forecast id")
        wanted = set(channels or filt or names) | set(ev)
        sel = [c for c in names if c in wanted]
        ev_list = [(i, t) for i, c in enumerate(sel) for t in ev.get(c, ())]
        if len(sel) > E.ENS_MAX_CHANNELS or len(ev_list) > E.ENS_MAX_EVENTS:
            raise ValueError(f"{len(sel)} channels and {len(ev_list)} events: at most {E.ENS_MAX_CHANNELS} and "
                             f"{E.ENS_MAX_EVENTS}")
        from ...ensemble import EnsembleRunner, HierarchicalEnsembleRunner
        if perturbation == "spherical_grf" and grf is None:
            grf = dict(lmax=min(180, (len(self.model.grid.lat) - 1) // 2))
        base, sigma, offset = self._ensemble_initial_state(start_time)
        make = EnsembleRunner
        if hasattr(self.model, "engine_24"):   # Pangu's hierarchical schedule: without save, the last two steps only
            make = functools.partial(HierarchicalEnsembleRunner, engine_24=self.model.engine_24, every_slice=save)
        runner = make(self.model.engine, base, sigma, members_per_gpu=members, rank=0, amp=amp, seed=seed,
                      perturbation=perturbation, grf=grf)
        save_config = {k: v for k, v in save_config.items() if k != "filter_vars"}   # selected on the device already
        save_config.setdefault("forecast_id", generate_forecast_id())
        label, source = f"{self.model_name}-ens{members}", self.ic_source if isinstance(self.ic_source, str) else "file"
        lat, lon = np.array(self.model.grid.lat), np.array(self.model.grid.lon)
        stat_names = np.array(["mean", "spread"] + [quantile_name(v) for v in q])
        ev_names = np.array([event_name(sel[i], t) for i, t in ev_list])
        result, paths, prev, t_prev = None, [], None, start_time
        # the host buffers of step n - 1 stay valid while step n is handled (iter_stats: rings of two)
        for n, s, p in runner.iter_stats(n_steps, [names.index(c) for c in sel], q, ev_list, offset):
            t_cur = start_time + n * self.time_step
            if n > 0 and (save or n == n_steps):
                times = np.array([np.datetime64(t_prev, "s"), np.datetime64(t_cur, "s")])
                stats = xr.DataArray(np.stack([prev[0].numpy(), s.numpy()]), dims=["time", "statistic", "channel", "lat", "lon"],
                                     coords=dict(time=times, statistic=stat_names, channel=np.array(sel), lat=lat, lon=lon))
                prob = None
                if ev_list:
                    prob = xr.DataArray(np.stack([prev[1].numpy(), p.numpy()]), dims=["time", "event", "lat", "lon"],
                                        coords=dict(time=times, event=ev_names, lat=lat, lon=lon))
                if save:
                    paths.append(save_forecast(stats, label, t_prev, t_cur, source, config=save_config))
                    if prob is not None:
                        paths.append(save_forecast(prob, f"{label}-prob", t_prev, t_cur, source, config=save_config))
                result = GlobalEnsemblePrediction(stats, prob, self.model_name, members)
            if n > 0:
                source = "file"
                logger.success(f"Ensemble step {n}/{n_steps} completed")
            prev, t_prev = (s, p), t_cur
        return result, paths

    def score(self, start_time: datetime.datetime, n_steps: int, truth=None, climatology=None, members: int = 1,
              perturbation: str | None = None, amp: float = 0.05, seed: int = 0, grf: dict | None = None,
              channels: List[str] = [], regions: dict | None = None, save: bool = False, save_config: dict = {}):
        """Verifies the forecast from ``start_time`` at every lead 0, 6, .., 6 ``n_steps`` h against ``truth`` and returns
        (scorecard, paths): a DataArray (lead_time, metric, region, channel) of the latitude-weighted scores of
        ``skyrim_b200/scores.py`` (bias, rmse, acc, spread, ssr, crps, crps_fair) in fp64, lead_time in hours (0: the
        initial condition), attrs model / members / start_time.  ``truth`` is a data source (``source[time] ->
        DataArray(channel, lat, lon)``) or a DataArray (time, channel, lat, lon) on the model's grid; it defaults to the
        model's own data source, as earth2mip verifies against its IC source.  ``climatology``: DataArray (channel, lat,
        lon), needed for acc.  ``members = 1`` scores the model's own unperturbed trajectory; above 1, ``perturbation``
        defaults to "spherical_grf" (as ``predict_ensemble``, with the same ``amp``, ``seed`` and ``grf``).  ``channels``
        default to the forecast channels (forcings excluded), ``regions`` to ``{"global": (-90, 90)}`` (at most 4 latitude
        bands).  The scores are formed on the device and the sums of all leads cross to the host once.  ``save`` writes
        the scorecard as one netCDF file, model "<model>-score<M>", under the forecast id."""
        from ... import scores as S
        if n_steps < 0:
            raise ValueError(f"n_steps = {n_steps} must not be negative")
        times = [start_time + n * self.time_step for n in range(n_steps + 1)]
        perturbation, sel, region_names, row_weights, truth_at, clim = self._score_setup(
            members, perturbation, channels, regions, truth, climatology, times, save, save_config)
        names = list(self.out_channel_names)
        runner, offset = self._score_runner(start_time, members, perturbation, amp, seed, grf)
        leads, sums = runner.iter_scores(n_steps, lambda n: truth_at(times[n]), clim,
                                         [names.index(c) for c in sel], row_weights, offset)
        hours = [n * self.time_step.total_seconds() / 3600 for n in leads]
        card = S.scorecard(np.asarray(sums), members, hours, region_names, sel, self.model_name, start_time)
        logger.success(f"Scored {len(leads)} leads of {members} member(s) on {len(sel)} channels")
        paths = []
        if save:
            save_config = {k: v for k, v in save_config.items() if k != "filter_vars"}   # selected on the device already
            save_config.setdefault("forecast_id", generate_forecast_id())
            source = self.ic_source if isinstance(self.ic_source, str) else "file"
            paths.append(save_forecast(card, f"{self.model_name}-score{members}", start_time,
                                       start_time + n_steps * self.time_step, source, config=save_config))
        return card, paths

    def _score_setup(self, members, perturbation, channels, regions, truth, climatology, times, save, save_config):
        """the checks and host inputs shared by ``score`` and ``score_period``, before any engine call: (perturbation,
        scored channel names, region names, row weights, truth fetcher, climatology fields)"""
        from ... import engine as E
        from ... import scores as S
        names = list(self.out_channel_names)
        if not 1 <= members <= E.ENS_MAX_MEMBERS:
            raise ValueError(f"members = {members} must lie in [1, {E.ENS_MAX_MEMBERS}]")
        if perturbation is None:
            perturbation = "none" if members == 1 else "spherical_grf"
        if perturbation not in ("none", "gaussian", "spherical_grf"):
            raise ValueError(f"unknown perturbation {perturbation!r} (none, gaussian, spherical_grf)")
        if save and save_config.get("file_type", "netcdf") == "zarr":
            raise ValueError("a scorecard is written as netCDF only: the zarr writer appends along time")
        filt = list(save_config.get("filter_vars", ()))
        wanted = list(channels) or filt
        unknown = [c for c in wanted if c not in names]
        if unknown:
            raise ValueError(f"unknown channel(s) {unknown} for {self.model_name}")
        forcing = [c for c in wanted if c in self.forcing_channels]
        if forcing:
            raise ValueError(f"{forcing} are forcings, not forecasts, and are not scored")
        sel = [c for c in names if (c in wanted if wanted else c not in self.forcing_channels)]
        if len(sel) > E.ENS_MAX_CHANNELS:
            raise ValueError(f"{len(sel)} channels: at most {E.ENS_MAX_CHANNELS}")
        lat, lon = np.array(self.model.grid.lat), np.array(self.model.grid.lon)
        region_names, row_weights = S.region_weights(lat, regions)
        if truth is None:
            truth = self.data_source
            if truth is None:
                raise ValueError(f"{self.model_name} has no data source to verify against (synthetic initial conditions): "
                                 "pass truth=")
        truth_at = S.truth_fetcher(truth, sel, lat, lon, times)
        clim = S.climatology_fields(climatology, sel, lat, lon)
        return perturbation, sel, region_names, row_weights, truth_at, clim

    def _score_runner(self, start_time, members, perturbation, amp, seed, grf):
        """(member runner of the forecast from ``start_time``, offset of the scored channels in its state)"""
        from ...ensemble import EnsembleRunner, HierarchicalEnsembleRunner
        if perturbation == "spherical_grf" and grf is None:
            grf = dict(lmax=min(180, (len(self.model.grid.lat) - 1) // 2))
        base, sigma, offset = self._ensemble_initial_state(start_time)
        make = EnsembleRunner
        if hasattr(self.model, "engine_24"):   # Pangu's hierarchical schedule: every slice is scored
            make = functools.partial(HierarchicalEnsembleRunner, engine_24=self.model.engine_24, every_slice=True)
        runner = make(self.model.engine, base, sigma, members_per_gpu=members, rank=0, amp=amp, seed=seed,
                      perturbation=perturbation, grf=grf)
        return runner, offset

    def score_period(self, start_times, n_steps: int, truth=None, climatology=None, members: int = 1,
                     perturbation: str | None = None, amp: float = 0.05, seed: int = 0, grf: dict | None = None,
                     channels: List[str] = [], regions: dict | None = None, map_leads=(), map_channels=(),
                     save: bool = False, save_config: dict = {}):
        """Verifies the forecasts from every one of ``start_times`` (distinct, increasing) at leads 0, 6, .., 6 ``n_steps`` h
        and returns (``scores.PeriodScores``, paths).  Date d is the forecast ``score(start_times[d], seed=seed + d)``
        verifies, with the same arguments; its scorecard is ``.cards[d]`` bit for bit.  ``.card`` holds the period's
        metrics (``scores.period_metrics``), ``.rank_histogram`` the rank histogram (lead_time, region, channel, rank)
        averaged over the dates, with ties broken by Philox draws keyed by (``seed``, d).  With ``map_leads`` (hours,
        multiples of the time step in [0, lead]) and ``map_channels`` (scored forecast channels), ``.maps`` holds per-point
        bias, rmse, spread and crps over the period, fp32 (lead_time, metric, channel, lat, lon).  Everything is checked
        before the first engine call, a truth DataArray for every valid time of every date.  One member runner serves all
        dates, restarted in place, and the truth buffers, the sums, histograms and map accumulators are allocated once;
        only the results cross to the host, at the end.  ``save`` writes the period card, the per-date cards, the rank
        histogram and the maps as netCDF files, models "<model>-period<M>[-cards|-rank|-maps]", under one forecast id."""
        import torch
        from ... import engine as E
        from ... import scores as S
        names = list(self.out_channel_names)
        starts = list(start_times)
        if not starts:
            raise ValueError("score_period needs at least one start time")
        if any(b <= a for a, b in zip(starts, starts[1:])):
            raise ValueError(f"start times must be distinct and sorted: {[str(np.datetime64(t, 's')) for t in starts]}")
        if n_steps < 0:
            raise ValueError(f"n_steps = {n_steps} must not be negative")
        if not 0 <= seed < 2 ** 32:
            raise ValueError(f"seed = {seed} must lie in [0, 2^32)")
        step_h = self.time_step.total_seconds() / 3600
        check_map_leads(map_leads, map_channels, n_steps, step_h)
        times = sorted({t + n * self.time_step for t in starts for n in range(n_steps + 1)})
        perturbation, sel, region_names, row_weights, truth_at, clim = self._score_setup(
            members, perturbation, channels, regions, truth, climatology, times, save, save_config)
        mch, slots = map_plan(map_leads, map_channels, sel, names, self.forcing_channels, step_h,
                              f"unknown map channel(s) {{}} for {self.model_name}")
        D, L, R, Sn, M = len(starts), n_steps + 1, len(region_names), len(sel), members
        runner = None
        for d, t0 in enumerate(starts):
            if runner is None:
                runner, offset = self._score_runner(t0, members, perturbation, amp, seed, grf)
                dev = runner.x.device
                H, W = runner.x.shape[-2:]
                sums = torch.empty((D, L, R, Sn, len(S.SUMS)), dtype=torch.float64, device=dev)
                hist = torch.empty((D, L, R, Sn, M + 1), dtype=torch.float64, device=dev)
                maps = torch.zeros((len(slots), len(mch), E.MAP_TERMS, H, W), dtype=torch.float64, device=dev)
                ring = runner.truth_ring(Sn)
            else:
                runner.restart(self._ensemble_initial_state(t0)[0], seed + d)
            valid = [t0 + n * self.time_step for n in range(L)]
            runner.iter_scores(n_steps, lambda n: truth_at(valid[n]), clim, [names.index(c) for c in sel], row_weights,
                               offset, hist=hist[d], seed=seed, date_index=d, maps=maps, map_slot=slots,
                               map_channels=[sel.index(c) for c in mch], sums=sums[d], ring=ring)
            logger.success(f"Scored start date {d + 1}/{D}: {np.datetime64(t0, 's')}")
        sums, hist = sums.cpu().numpy(), hist.cpu().numpy()
        hours = [n * step_h for n in range(L)]
        res = S.PeriodScores.build(sums, hist, maps.cpu().numpy() if mch else None, members, starts, hours,
                                   sorted(slots, key=slots.get), step_h, region_names, sel, mch, self.model_name,
                                   np.array(self.model.grid.lat), np.array(self.model.grid.lon))
        paths = []
        if save:
            save_config = {k: v for k, v in save_config.items() if k != "filter_vars"}   # selected on the device already
            save_config.setdefault("forecast_id", generate_forecast_id())
            source = self.ic_source if isinstance(self.ic_source, str) else "file"
            label, t_end = f"{self.model_name}-period{members}", starts[-1] + n_steps * self.time_step
            for suffix, da in (("", res.card), ("-cards", res.cards), ("-rank", res.rank_histogram), ("-maps", res.maps)):
                if da is not None:
                    paths.append(save_forecast(da, label + suffix, starts[0], t_end, source, config=save_config))
        return res, paths

    def _site_channels(self, channels, save_config, default):
        """the checked channel names of a site request, in model order: ``channels``, else save_config's filter_vars,
        else ``default``"""
        from ... import engine as E
        names = list(self.out_channel_names)
        wanted = list(channels) or list(save_config.get("filter_vars", ())) or list(default)
        unknown = [c for c in wanted if c not in names]
        if unknown:
            raise ValueError(f"unknown channel(s) {unknown} for {self.model_name}")
        sel = [c for c in names if c in wanted]
        if len(sel) > E.ENS_MAX_CHANNELS:
            raise ValueError(f"{len(sel)} channels: at most {E.ENS_MAX_CHANNELS}")
        return sel

    def _site_checks(self, members, perturbation, method):
        """the checks shared by ``predict_sites`` and ``score_sites``, before any engine call: the perturbation ("none"
        for one member, else "spherical_grf", unless given)"""
        from ... import engine as E
        from ... import sites as St
        if not 1 <= members <= E.ENS_MAX_MEMBERS:
            raise ValueError(f"members = {members} must lie in [1, {E.ENS_MAX_MEMBERS}]")
        if perturbation is None:
            perturbation = "none" if members == 1 else "spherical_grf"
        if perturbation not in ("none", "gaussian", "spherical_grf"):
            raise ValueError(f"unknown perturbation {perturbation!r} (none, gaussian, spherical_grf)")
        if method not in E.SITES_METHODS:
            raise ValueError(f"unknown site method {method!r} ({', '.join(E.SITES_METHODS)})")
        St.check_equiangular(self.model.grid.lat, self.model.grid.lon)
        return perturbation

    def predict_sites(self, start_time: datetime.datetime, n_steps: int, sites, members: int = 1,
                      method: str = "bilinear", channels: List[str] = [], quantiles=(), events: dict = {},
                      perturbation: str | None = None, amp: float = 0.05, seed: int = 0, grf: dict | None = None,
                      save: bool = False, save_config: dict = {}):
        """Forecast at ``sites`` (``sites.read_sites``: {name: (lat, lon)}, (names, lats, lons) or a CSV file) for leads 0,
        6, .., 6 ``n_steps`` h: every member sampled on the device with the site stencil ``method`` ("bilinear" or
        "nearest", include/skyrim_b200.h sky_sites_create).  ``members = 1`` (perturbation "none") samples the model's own
        trajectory; above 1 the members are ``predict_ensemble``'s (perturbation, amp, seed, grf), and the site
        statistics (mean, spread, ``quantiles``) and P(x > t) for ``events`` = {channel: threshold(s)} are reduced on the
        device too.  Only the site arrays cross to the host, each step's copy under the next step's forwards.  Refused
        before any engine call: unknown channels, a grid that is not equiangular, and returned arrays above 2^31 bytes.
        ``save`` writes the values, statistics and probabilities as netCDF files, models "<model>-sites<M>[-stats|-prob]".
        Returns (``sites.SiteForecast``, paths)."""
        from ... import engine as E
        from ... import sites as St
        from .ensemble import event_name, quantile_name
        perturbation = self._site_checks(members, perturbation, method)
        if n_steps < 0:
            raise ValueError(f"n_steps = {n_steps} must not be negative")
        names, lat, lon = St.read_sites(sites)
        ev = {c: [float(t) for t in np.atleast_1d(thr)] for c, thr in dict(events).items()}
        q = [float(v) for v in quantiles]
        if members == 1 and (q or ev):
            raise ValueError("quantiles and events describe an ensemble: give members > 1")
        if len(q) > E.ENS_MAX_QUANTILES or not all(0.0 <= v <= 1.0 for v in q):
            raise ValueError(f"quantiles {q}: at most {E.ENS_MAX_QUANTILES}, each in [0, 1]")
        if not all(np.isfinite(t) for ts in ev.values() for t in ts):
            raise ValueError(f"event thresholds must be finite: {ev}")
        if save and save_config.get("file_type", "netcdf") == "zarr":
            raise ValueError("site forecasts are written as netCDF only: the zarr writer holds one variable per forecast id")
        unknown = [c for c in ev if c not in self.out_channel_names]
        if unknown:
            raise ValueError(f"unknown channel(s) {unknown} for {self.model_name}")
        wanted = set(self._site_channels(channels, save_config, self.out_channel_names)) | set(ev)
        sel = [c for c in self.out_channel_names if c in wanted]
        ev_list = [(i, t) for i, c in enumerate(sel) for t in ev.get(c, ())]
        if len(sel) > E.ENS_MAX_CHANNELS or len(ev_list) > E.ENS_MAX_EVENTS:
            raise ValueError(f"{len(sel)} channels and {len(ev_list)} events: at most {E.ENS_MAX_CHANNELS} and "
                             f"{E.ENS_MAX_EVENTS}")
        T, n, Sn = n_steps + 1, len(names), len(sel)
        nbytes = 4 * T * n * (members * Sn + ((2 + len(q)) * Sn + len(ev_list) if members > 1 else 0))
        if nbytes > St.RETURN_LIMIT:
            raise ValueError(f"the site arrays of this request take {nbytes} bytes, above the 2^31 returned at most: "
                             "ask for fewer steps, members, channels or sites")
        runner, offset = self._score_runner(start_time, members, perturbation, amp, seed, grf)
        table = E.SiteTable(lat, lon, len(self.model.grid.lat), len(self.model.grid.lon), method, runner.x.device.index)
        values = np.empty((T, members, n, Sn), np.float32)
        stats = np.empty((T, 2 + len(q), n, Sn), np.float32) if members > 1 else None
        prob = np.empty((T, len(ev_list), n), np.float32) if ev_list else None
        idx = [list(self.out_channel_names).index(c) for c in sel]
        try:
            for n_, v, *rest in runner.iter_sites(n_steps, table, idx, q, ev_list, offset):
                values[n_] = v.numpy()[:, :, 0].transpose(0, 2, 1)
                if stats is not None:
                    stats[n_] = rest[0].numpy()[:, :, 0].transpose(0, 2, 1)
                if prob is not None:
                    prob[n_] = rest[1].numpy()[:, 0]
        finally:
            table.close()
        times = np.array([np.datetime64(start_time + k * self.time_step, "s") for k in range(T)])
        where = dict(site=np.array(names), lat=("site", lat), lon=("site", lon))
        attrs = dict(model=self.model_name, members=int(members), method=method)
        res = St.SiteForecast(
            xr.DataArray(values, dims=["time", "member", "site", "channel"],
                         coords=dict(where, time=times, member=np.arange(members, dtype=np.float64), channel=np.array(sel)),
                         attrs=dict(attrs)),
            None if stats is None else xr.DataArray(
                stats, dims=["time", "statistic", "site", "channel"],
                coords=dict(where, time=times, statistic=np.array(["mean", "spread"] + [quantile_name(v) for v in q]),
                            channel=np.array(sel)), attrs=dict(attrs)),
            None if prob is None else xr.DataArray(
                prob, dims=["time", "event", "site"],
                coords=dict(where, time=times, event=np.array([event_name(sel[i], t) for i, t in ev_list])),
                attrs=dict(attrs)),
            self.model_name, members)
        logger.success(f"Sampled {members} member(s) at {n} site(s) for {T} leads")
        paths = []
        if save:
            save_config = {k: v for k, v in save_config.items() if k != "filter_vars"}   # selected on the device already
            save_config.setdefault("forecast_id", generate_forecast_id())
            source = self.ic_source if isinstance(self.ic_source, str) else "file"
            label, t_end = f"{self.model_name}-sites{members}", start_time + n_steps * self.time_step
            for suffix, da in (("", res.values), ("-stats", res.stats), ("-prob", res.prob)):
                if da is not None:
                    paths.append(save_forecast(da, label + suffix, start_time, t_end, source, config=save_config))
        return res, paths

    def score_sites(self, start_times, n_steps: int, observations, members: int = 1, method: str = "bilinear",
                    channels: List[str] = [], perturbation: str | None = None, amp: float = 0.05, seed: int = 0,
                    grf: dict | None = None, save: bool = False, save_config: dict = {}):
        """Verifies the forecasts from every one of ``start_times`` (distinct, increasing) at leads 0, 6, .., 6 ``n_steps``
        h against station ``observations`` (``sites.read_observations``: a DataArray (time, site, channel) with lat / lon
        along site, NaN where missing), sampling the members at the observation sites with ``method``.  Date d is the
        forecast ``predict_sites`` makes with ``seed + d`` (one runner restarted per date); ``channels`` default to the
        observations' channels.  A valid time absent from the observations counts as missing everywhere; the call is
        refused, before any engine call, if no observation is usable at all, and for forcing channels.  The site terms
        are accumulated on the device and cross to the host once, at the end.  ``save`` writes the card, the per-date
        cards, the per-site scores and the counts as netCDF files, models "<model>-obs<M>[-cards|-sites|-count]".
        Returns (``sites.SiteScores``, paths)."""
        import torch
        from ... import engine as E
        from ... import sites as St
        from ...ensemble import upload_truth, truth_ring
        perturbation = self._site_checks(members, perturbation, method)
        starts = list(start_times)
        if not starts:
            raise ValueError("score_sites needs at least one start time")
        if any(b <= a for a, b in zip(starts, starts[1:])):
            raise ValueError(f"start times must be distinct and sorted: {[str(np.datetime64(t, 's')) for t in starts]}")
        if n_steps < 0:
            raise ValueError(f"n_steps = {n_steps} must not be negative")
        if not 0 <= seed < 2 ** 32:
            raise ValueError(f"seed = {seed} must lie in [0, 2^32)")
        if save and save_config.get("file_type", "netcdf") == "zarr":
            raise ValueError("site scores are written as netCDF only: the zarr writer appends along time")
        have = St.read_observations(observations)[4]
        wanted = list(channels) or list(save_config.get("filter_vars", ()))
        forcing = [c for c in wanted if c in self.forcing_channels]
        if forcing:
            raise ValueError(f"{forcing} are forcings, not forecasts, and are not scored")
        sel = self._site_channels(channels, save_config, [c for c in have if c in self.out_channel_names
                                                          and c not in self.forcing_channels])
        if not sel:
            raise ValueError(f"the observations hold none of {self.model_name}'s forecast channels ({have})")
        names, lat, lon, times, sel, obs = St.read_observations(observations, sel)
        D, L, Sn, n = len(starts), n_steps + 1, len(sel), len(names)
        at = {t: i for i, t in enumerate(times.tolist())}
        slot = [[at.get(np.datetime64(t0 + k * self.time_step, "s").tolist()) for k in range(L)] for t0 in starts]
        if not any(i is not None and np.isfinite(obs[i]).any() for row in slot for i in row):
            raise ValueError("the observations hold no value at any valid time of these forecasts: nothing to verify")
        missing = np.full((Sn, n), np.nan, np.float32)
        runner = None
        for d, t0 in enumerate(starts):
            if runner is None:
                runner, offset = self._score_runner(t0, members, perturbation, amp, seed, grf)
                dev = runner.x.device
                table = E.SiteTable(lat, lon, len(self.model.grid.lat), len(self.model.grid.lon), method, dev.index)
                sums = torch.empty((D, L, Sn, E.SITE_TERMS), dtype=torch.float64, device=dev)
                acc = torch.zeros((L, Sn, n, E.SITE_TERMS), dtype=torch.float64, device=dev)
                values = torch.empty((members, Sn, 1, n), dtype=torch.float32, device=dev)
                ring = truth_ring(dev, Sn, 1, n)
                main = torch.cuda.current_stream(dev)
                idx = [list(self.out_channel_names).index(c) for c in sel]
            else:
                runner.restart(self._ensemble_initial_state(t0)[0], seed + d)
            for i, (k, members_x) in enumerate(runner._walk(n_steps, every_slice=True)):
                j = slot[d][k]
                y = upload_truth(ring, i, (missing if j is None else obs[j].T)[:, None, :], main)
                E.sample_sites(members_x, table, idx, offset, out=values)
                E.site_scores(values, y.view(Sn, n), acc[k], out=sums[d, k])
                ring["scored"][i % 2].record(main)
            logger.success(f"Scored start date {d + 1}/{D} at {n} site(s): {np.datetime64(t0, 's')}")
        table.close()
        step_h = self.time_step.total_seconds() / 3600
        res = St.SiteScores.build(sums.cpu().numpy(), acc.cpu().numpy(), members, starts, [k * step_h for k in range(L)],
                                  names, lat, lon, sel, self.model_name)
        paths = []
        if save:
            save_config = {k: v for k, v in save_config.items() if k != "filter_vars"}   # selected on the device already
            save_config.setdefault("forecast_id", generate_forecast_id())
            source = self.ic_source if isinstance(self.ic_source, str) else "file"
            label, t_end = f"{self.model_name}-obs{members}", starts[-1] + n_steps * self.time_step
            for suffix, da in (("", res.card), ("-cards", res.cards), ("-sites", res.sites), ("-count", res.count)):
                paths.append(save_forecast(da, label + suffix, starts[0], t_end, source, config=save_config))
        return res, paths


def check_map_leads(map_leads, map_channels, n_steps: int, step_h: float):
    """refuses map leads (hours) that are not multiples of the time step in [0, n_steps steps], and map leads without map
    channels or the reverse"""
    bad = [h for h in map_leads if not (0 <= h <= n_steps * step_h and float(h) / step_h == int(float(h) / step_h))]
    if bad:
        raise ValueError(f"map lead(s) {list(bad)} h: multiples of the {step_h:g}-h time step in [0, {n_steps * step_h:g}] "
                         "needed")
    if bool(len(map_leads)) != bool(len(map_channels)):
        raise ValueError("map_leads and map_channels go together: give both or neither")


def map_plan(map_leads, map_channels, sel, names, forcing_channels, step_h: float, unknown_msg: str):
    """(map channels in the order of the scored channels ``sel``, {step: slot} of the map leads in increasing order),
    refusing a map channel not in ``names`` (``unknown_msg`` formatted with the list), a forcing or one not scored"""
    mch = list(dict.fromkeys(map_channels))
    unknown = [c for c in mch if c not in names]
    if unknown:
        raise ValueError(unknown_msg.format(unknown))
    forcing = [c for c in mch if c in forcing_channels]
    if forcing:
        raise ValueError(f"map channel(s) {forcing} are forcings, not forecasts, and are not scored")
    unscored = [c for c in mch if c not in sel]
    if unscored:
        raise ValueError(f"map channel(s) {unscored} are not among the scored channels {sel}")
    mch = [c for c in sel if c in mch]
    return mch, {int(round(h / step_h)): i for i, h in enumerate(sorted({float(h) for h in map_leads}))}


class GlobalPrediction:
    filepath: Path | None = None
    prediction = None

    def __init__(self, source, model_name: str = ""):
        self.model = model_name
        if isinstance(source, (str, Path)):
            self.filepath = Path(source)
            self.prediction = xr.open_dataarray(source).squeeze()
        elif hasattr(source, "dims") and hasattr(source, "values"):
            self.filepath = None
            self.prediction = source.squeeze()
        else:
            raise ValueError("Invalid source type.")

    @property
    def coords(self):
        return self.prediction.coords

    @property
    def size(self):
        return self.prediction.size

    @property
    def channels(self):
        return self.prediction.channel

    def __repr__(self) -> str:
        info = self.filepath if self.filepath else f"{type(self.prediction).__name__} with shape {self.prediction.shape}"
        return f"GlobalPrediction(model={self.model},source={info})"

    def slice(self, lat: slice | None = None, lon: slice | None = None, channel: str | None = None,
              n_step: slice | None = None):
        if channel is None:
            data = self.prediction
        else:
            assert channel in self.channels, f"Variable {channel} not found in dataset."
            data = self.prediction.sel(channel=channel)
        if lat:
            data = data.sel(lat=lat)
        if lon:
            data = data.sel(lon=lon)
        if n_step and "time" in data.dims:
            data = data.isel(time=n_step)
        return data

    def point(self, lat: float, lon: float, channel: str, n_step: int | None = 1):
        """The value of the grid point nearest to (lat, lon), as the reference reads it: longitudes are compared on
        [0, 360) without wrapping, so near 360 degrees this can pick a different point than ``predict_sites(...,
        method="nearest")``, which measures longitude distance around the circle, and it does not interpolate."""
        if lon < 0:
            lon = 360 + lon
        assert channel in self.channels, f"Variable {channel} not found in dataset."
        lats, lons = np.asarray(self.prediction.coords["lat"]), np.asarray(self.prediction.coords["lon"])
        if lat not in lats or lon not in lons:
            lat = float(lats[np.abs(lats - lat).argmin()])
            lon = float(lons[np.abs(lons - lon).argmin()])
            logger.warning(f"Exact coordinates not found. Using nearest values: Lat {lat}, Lon {lon}")
        data = self.prediction.sel(lat=lat, lon=lon, channel=channel)
        if "time" in data.dims:
            data = data.isel(time=n_step)
        return data.item()

    def point_wind_uv(self, lat: float, lon: float, pressure_level: int = 1000, n_step: int | None = 1):
        u = self.point(lat=lat, lon=lon, channel=f"u{pressure_level}", n_step=n_step)
        v = self.point(lat=lat, lon=lon, channel=f"v{pressure_level}", n_step=n_step)
        return u, v

    def wind_speed(self, lat: float, lon: float, pressure_level: int, n_step: int | None = 1):
        u, v = self.point_wind_uv(lat, lon, pressure_level, n_step)
        return (u ** 2 + v ** 2) ** 0.5

    def surface_wind_speed(self, lat: float, lon: float, n_step: int | None = 1):
        return self.wind_speed(lat, lon, pressure_level=1000, n_step=n_step)


class GlobalPredictionRollout:
    def __init__(self, rollout: list):
        self.rollout = [GlobalPrediction(source) for source in rollout]
        self.time_steps = [np.asarray(r.prediction.coords["time"])[-1] for r in self.rollout]

    def __repr__(self):
        return f"<GlobalPredictionRollout with {len(self.rollout)} predictions, last times: {self.time_steps}>"

    def wind_speed(self, lat: float, lon: float, pressure_level: int, n_step: int | None = 1):
        return [pred.wind_speed(lat, lon, pressure_level, n_step) for pred in self.rollout]

    def surface_wind_speed(self, lat: float, lon: float, n_step: int | None = 1):
        return self.wind_speed(lat, lon, pressure_level=1000, n_step=n_step)
