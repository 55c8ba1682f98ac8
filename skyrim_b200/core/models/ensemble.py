"""GlobalEnsemblePrediction — the class /root/reference/skyrim/core/models/ensemble.py:131-133 names and leaves empty: the
per-step statistics of a perturbed-initial-condition ensemble (``GlobalModel.predict_ensemble``), reduced on the GPU; and
GlobalEnsemble (ensemble.py:10-128 there): several models side by side on one GPU, reduced on the device every step."""
from __future__ import annotations

import datetime
from typing import List

import numpy as np
from loguru import logger

from ... import xr_shim as xr
from ...common import generate_forecast_id, save_forecast
from ...engine import ENS_MAX_MEMBERS, ENS_MAX_SOURCES
from .base import GlobalPrediction, SyntheticDataSource, check_map_leads, map_plan
from .graphcast import GraphcastModel


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

    def model_mean(self, name: str) -> GlobalPrediction:
        """the mean of one model's own members (statistic "mean:<name>" of a multi-model ensemble)"""
        return self._statistic(f"mean:{name}")


class SourceView:
    """Channel-selecting view of a data source: ``view[t]`` is ``source[t]`` restricted to ``channel_names``, in that order.
    ``Skyrim(name, ic_source=SourceView(ensemble.data_source, names))`` starts one model from exactly the initial condition
    it gets inside a ``GlobalEnsemble``."""

    def __init__(self, source, channel_names):
        self.source, self.channel_names = source, list(channel_names)

    def __getitem__(self, t):
        return self.source[t].sel(channel=self.channel_names)


class GlobalEnsemble:
    """Several models side by side on one GPU, reduced on the device every step (the reference's multi-model mean,
    ensemble.py:10-128, which runs the models one after the other and averages the last step on the host).

    ``Skyrim("pangu", "graphcast", pangu=dict(cfg=...), device=0)``: a keyword named after a model goes to that model only,
    every other keyword to all of them.  The models must share one grid.  They start from one atmosphere: a data source
    over the union of their channels (the first model's channels in its order, then each later model's new ones), which
    every model reads by name through a ``SourceView``.  The shared channels, the ones every model forecasts, are kept in
    the first model's order; the mean and the statistics are taken over them."""

    def __init__(self, model_names, ic_source="synthetic", **model_kw):
        from . import MODELS
        names = list(model_names)
        if len(set(names)) != len(names):
            raise ValueError(f"duplicate model names in {names}")
        missing = [n for n in names if n not in MODELS]
        if missing:
            raise ValueError(f"Invalid model name(s): {missing}")
        if not 1 <= len(names) <= ENS_MAX_SOURCES:
            raise ValueError(f"{len(names)} models: a multi-model ensemble holds 1 to {ENS_MAX_SOURCES}")
        common = {k: v for k, v in model_kw.items() if k not in names}
        if "pangu" in names and {**common, **dict(model_kw.get("pangu", {}))}.get("schedule", "6h") != "6h":
            # the models step in lockstep (_step_all): a schedule that skips or re-anchors steps is not built here
            raise ValueError("a multi-model run steps Pangu on its 6-h schedule only; the hierarchical schedule runs "
                             "with Pangu alone")
        self.model_names, self.ic_source = names, ic_source
        self.models = []
        try:
            for n in names:
                self.models.append(MODELS[n](ic_source=ic_source, **{**common, **dict(model_kw.get(n, {}))}))
            first = self.models[0].model.grid
            for n, m in zip(names[1:], self.models[1:]):
                g = m.model.grid
                if not (np.array_equal(g.lat, first.lat) and np.array_equal(g.lon, first.lon)):
                    raise ValueError(f"{n}'s grid ({len(g.lat)}x{len(g.lon)}) differs from {names[0]}'s "
                                     f"({len(first.lat)}x{len(first.lon)}): the models must share one grid")
            self.shared_channels = [c for c in self.models[0].out_channel_names
                                    if all(c in m.out_channel_names for m in self.models[1:])]
            if not self.shared_channels:
                raise ValueError(f"{names} share no output channel")
        except Exception:
            self.release_model()
            raise
        union = list(self.models[0].in_channel_names)
        for m in self.models[1:]:
            union += [c for c in m.in_channel_names if c not in union]
        self.channel_names = union
        nlat, nlon = len(first.lat), len(first.lon)
        if ic_source == "synthetic":
            self.data_source = SyntheticDataSource(union, nlat, nlon)
        elif hasattr(ic_source, "__getitem__") and not isinstance(ic_source, str):
            self.data_source = ic_source
        else:
            raise NotImplementedError(f"ic_source='{ic_source}': pass 'synthetic' or a data-source object")
        for m in self.models:
            m.data_source = SourceView(self.data_source, m.in_channel_names)
        self.model_predictions, self.model_paths = {}, {}

    def release_model(self):
        for m in self.models:
            m.release_model()

    def __repr__(self) -> str:
        return f"GlobalEnsemble({self.model_names})"

    @property
    def time_step(self):
        return self.models[0].time_step

    def time_steps(self, lead_time: int):
        return self.models[0].time_steps(lead_time)

    @property
    def in_channel_names(self):
        return self.channel_names

    @property
    def out_channel_names(self):
        return self.shared_channels

    @property
    def label(self) -> str:
        """the model name of the files: the reference's "_".join(sorted(names))"""
        return "_".join(sorted(self.model_names))

    def predict_one_step(self, start_time: datetime.datetime, initial_condition=None):
        raise NotImplementedError("a multi-model ensemble steps through rollout / forecast (as the reference's)")

    def score(self, *args, **kw):
        raise NotImplementedError("forecast scores are computed per model: score each model with Skyrim(name).score, or "
                                  "compare the models with compare(); multi-model scoring through score is not built")

    def score_period(self, *args, **kw):
        raise NotImplementedError("forecast scores are computed per model: verify a period for each model with "
                                  "Skyrim(name).score_period, or compare the models with compare(); multi-model scoring "
                                  "through score_period is not built")

    def predict_sites(self, *args, **kw):
        raise NotImplementedError("site forecasts are made per model: sample each model with Skyrim(name).predict_sites; "
                                  "multi-model site forecasts are not built")

    def score_sites(self, *args, **kw):
        raise NotImplementedError("site scores are computed per model: verify each model with Skyrim(name).score_sites; "
                                  "multi-model site verification is not built")

    # -- device states ---------------------------------------------------------------------------------------------------
    def _layout(self, m):
        """(state channels, offset of the output slice in the state): a GraphCast state holds two time slices"""
        if isinstance(m, GraphcastModel):
            ns = m._cfg.n_state
            return 2 * ns, ns
        return len(m.in_channel_names), 0

    def _initial_states(self, start_time):
        """one (1, C_state, H, W) device state per model, assembled as that model's own rollout assembles it"""
        import torch
        states = []
        for m in self.models:
            if isinstance(m, GraphcastModel):
                x = m._initial_fields(start_time)
                m.model.engine.set_clock(start_time)
            else:
                vals = np.asarray(m.data_source[start_time].values, dtype=np.float32)
                x = torch.from_numpy(np.ascontiguousarray(vals[-1] if vals.ndim == 4 else vals))[None].to(m.model.device)
            states.append(x.reshape(x.shape[0], -1, *x.shape[-2:]).contiguous())
        return states

    def _step_all(self, states, first: bool = False):
        """one step of every model, in turn on the current stream (each engine's persistent kernels fill the GPU)"""
        import torch
        for k, m in enumerate(self.models):
            nxt = torch.empty_like(states[k])
            if first and m.model.guard_first_step:
                _, m.model.last_ranges = m.model.engine.step_guarded(states[k], nxt)
            else:
                m.model.engine.step(states[k], nxt)
            states[k] = nxt

    def _outputs(self, states):
        """each model's newest slice, (B, C_out, H, W) views of the states"""
        return [x[:, self._layout(m)[1]:] for m, x in zip(self.models, states)]

    def _shared_index(self, channels):
        return [[m.out_channel_names.index(c) for c in channels] for m in self.models]

    def _model_da(self, k, state, prev, times):
        """model k's (2, C, H, W) DataArray of the step ending at times[1], as its own rollout returns it"""
        m, (cs, off) = self.models[k], self._layout(self.models[k])
        if off:
            vals = state[0].cpu().numpy().reshape(2, off, *state.shape[-2:])
        else:
            vals = np.stack([prev, state[0].cpu().numpy()])
        return xr.DataArray(vals, dims=["time", "channel", "lat", "lon"],
                            coords=dict(time=np.array([np.datetime64(t, "s") for t in times]),
                                        channel=np.array(m.out_channel_names), lat=np.array(m.model.grid.lat),
                                        lon=np.array(m.model.grid.lon)))

    def _mean_da(self, mean_prev, mean_cur, times, channels):
        g = self.models[0].model.grid
        return xr.DataArray(np.stack([mean_prev, mean_cur]), dims=["time", "channel", "lat", "lon"],
                            coords=dict(time=np.array([np.datetime64(t, "s") for t in times]), channel=np.array(channels),
                                        lat=np.array(g.lat), lon=np.array(g.lon)))

    # -- deterministic: one member per model ------------------------------------------------------------------------------
    def rollout(self, start_time: datetime.datetime, n_steps: int = 3, save: bool = True, save_config: dict = {}):
        """Steps every model from the shared initial condition and reduces the K states after each step with one kernel.
        Returns (DataArray of the model mean over the shared channels with 2 time slices, paths of the per-step mean files,
        model "<sorted names joined by _>").  With ``save``, every model also writes its own step files as its rollout
        would; they are in ``model_paths[name]``.  ``model_predictions[name]`` holds each model's last step."""
        import torch
        from ... import engine as E
        if n_steps < 1:
            raise ValueError(f"n_steps = {n_steps} must be at least 1")
        save_config = dict(save_config)
        save_config.setdefault("forecast_id", generate_forecast_id())
        filt = list(save_config.get("filter_vars", ()))
        mean_config = dict(save_config, filter_vars=[c for c in filt if c in self.shared_channels])
        model_config = {n: dict(save_config, filter_vars=[c for c in filt if c in m.out_channel_names])
                        for n, m in zip(self.model_names, self.models)}
        source = self.ic_source if isinstance(self.ic_source, str) else "file"
        chans = self._shared_index(self.shared_channels)
        states = self._initial_states(start_time)
        ring = [E.multi_model_statistics(self._outputs(states), chans, source_means=False)]
        ring.append(tuple(None if t is None else torch.empty_like(t) for t in ring[0]))
        prev = [o[0].cpu().numpy() for o in self._outputs(states)]
        paths, model_paths, mean = [], {n: [] for n in self.model_names}, None
        t_prev = start_time
        for n in range(1, n_steps + 1):
            t_cur = t_prev + self.time_step
            self._step_all(states, first=n == 1)
            E.multi_model_statistics(self._outputs(states), chans, source_means=False, out=ring[n % 2])
            if save or n == n_steps:
                for k, name in enumerate(self.model_names):
                    da = self._model_da(k, states[k], prev[k], (t_prev, t_cur))
                    prev[k] = da.values[1]
                    self.model_predictions[name] = da
                    if save:
                        model_paths[name].append(save_forecast(da, name, t_prev, t_cur, source,
                                                               config=model_config[name]))
                mean = self._mean_da(ring[(n - 1) % 2][0][0].cpu().numpy(), ring[n % 2][0][0].cpu().numpy(),
                                     (t_prev, t_cur), self.shared_channels)
                if save:
                    paths.append(save_forecast(mean, self.label, t_prev, t_cur, source, config=mean_config))
            t_prev, source = t_cur, "file"
            logger.success(f"Multi-model rollout step {n}/{n_steps} completed")
        self.model_paths = model_paths
        return mean, paths

    def forecast(self, start_time: datetime.datetime, n_steps: int = 3, channels: List[str] = []):
        """(n_steps + 1, channel, lat, lon) model mean over the shared channels (or ``channels``, which must be shared),
        the first slice being the mean of the initial conditions"""
        from ... import engine as E
        sel = list(channels) or self.shared_channels
        unknown = [c for c in sel if c not in self.shared_channels]
        if unknown:
            raise ValueError(f"channel(s) {unknown} are not shared by {self.model_names}")
        chans = self._shared_index(sel)
        states = self._initial_states(start_time)
        means = [E.multi_model_statistics(self._outputs(states), chans, source_means=False)[0][0].cpu().numpy()]
        for n in range(n_steps):
            self._step_all(states, first=n == 0)
            means.append(E.multi_model_statistics(self._outputs(states), chans, source_means=False)[0][0].cpu().numpy())
            logger.success(f"Multi-model forecast step {n + 1}/{n_steps} completed")
        g = self.models[0].model.grid
        times = [start_time + i * self.time_step for i in range(n_steps + 1)]
        return xr.DataArray(np.stack(means), dims=["time", "channel", "lat", "lon"],
                            coords=dict(time=np.array([np.datetime64(t, "s") for t in times]), channel=np.array(sel),
                                        lat=np.array(g.lat), lon=np.array(g.lon)))

    # -- verification: the models head to head ------------------------------------------------------------------------
    def compare(self, start_times, n_steps: int, truth=None, climatology=None, members: int = 1,
                perturbation: str | None = None, amp: float = 0.05, seed: int = 0, grf: dict | None = None,
                channels: List[str] = [], regions: dict | None = None, map_leads=(), map_channels=(), save: bool = False,
                save_config: dict = {}):
        """Verifies every model and their pooled ensemble over the same start dates against one truth, and returns
        (``scores.ModelComparison``, paths).

        The models (2 to 4, K x ``members`` at most 64) step in lockstep from each of ``start_times`` (distinct,
        increasing and equally spaced: the paired significance assumes it) through leads 0 .. ``n_steps``.  ``members = 1``
        starts each model from exactly the state its own ``score_period`` starts from (perturbation "none"); above 1,
        ``perturbation`` defaults to "spherical_grf" and date d's members are ``ensemble_members(t, members, ..., seed +
        d)``, the same perturbation of the same variable for every model.  The scored channels are the shared channels
        that are no model's forcing (``channels`` must name shared channels); ``truth`` defaults to the ensemble's data
        source.  Per lead every model's forwards are launched, the truth is fetched on the host under them and uploaded
        once (``ensemble.upload_truth``); each model is scored with the single-source entries (its own channel indices and
        state slice, so its per-date cards, rank histograms and maps are bitwise its own ``score_period``'s), and the K x
        ``members`` pooled members with the ``*_multi`` entries, off the same buffer.  Only the sums, histograms and maps
        reach the host, at the end.  Everything ``score_period`` checks is checked before the first engine call.

        ``.scores[entry]`` is that entry's ``PeriodScores``, ``.card`` the period cards stacked (model, lead_time, metric,
        region, channel), ``.differences`` the paired differences of every pair (``scores.paired_differences``).  ``save``
        writes netCDF files under one forecast id, label "<sorted names joined by _>-compare<M>": "" the card, "-cards",
        "-rank-<entry>", "-maps" (with map leads) and "-diff"."""
        import torch
        from ... import engine as E
        from ... import scores as S
        from ...ensemble import truth_ring, upload_truth
        K, names = len(self.models), self.shared_channels
        if not 2 <= K <= ENS_MAX_SOURCES:
            raise ValueError(f"{K} model(s): a comparison holds 2 to {ENS_MAX_SOURCES} models")
        if not 1 <= members or K * members > ENS_MAX_MEMBERS:
            raise ValueError(f"members = {members} per model: {K} models x members must lie in [1, {ENS_MAX_MEMBERS}]")
        starts = list(start_times)
        if not starts:
            raise ValueError("compare needs at least one start time")
        if any(b <= a for a, b in zip(starts, starts[1:])):
            raise ValueError(f"start times must be distinct and sorted: {[str(np.datetime64(t, 's')) for t in starts]}")
        gaps = [b - a for a, b in zip(starts, starts[1:])]
        uneven = [(a, b) for a, b, g in zip(starts, starts[1:], gaps) if g != gaps[0]]
        if uneven:
            a, b = uneven[0]
            raise ValueError(f"start times must be equally spaced (the paired significance assumes it): the gap "
                             f"{np.datetime64(a, 's')} -> {np.datetime64(b, 's')} is {b - a}, not {gaps[0]}")
        if n_steps < 0:
            raise ValueError(f"n_steps = {n_steps} must not be negative")
        if not 0 <= seed < 2 ** 32:
            raise ValueError(f"seed = {seed} must lie in [0, 2^32)")
        if perturbation is None:
            perturbation = "none" if members == 1 else "spherical_grf"
        if perturbation not in ("none", "gaussian", "spherical_grf"):
            raise ValueError(f"unknown perturbation {perturbation!r} (none, gaussian, spherical_grf)")
        if grf and perturbation != "spherical_grf":
            raise ValueError("grf options need perturbation='spherical_grf'")
        if save and save_config.get("file_type", "netcdf") == "zarr":
            raise ValueError("a comparison is written as netCDF only: the zarr writer appends along time")
        step_h = self.time_step.total_seconds() / 3600
        check_map_leads(map_leads, map_channels, n_steps, step_h)
        forcings = {c for m in self.models for c in m.forcing_channels}
        wanted = list(channels) or list(save_config.get("filter_vars", ()))
        unknown = [c for c in wanted if c not in names]
        if unknown:
            raise ValueError(f"channel(s) {unknown} are not shared by {self.model_names}")
        forcing = [c for c in wanted if c in forcings]
        if forcing:
            raise ValueError(f"{forcing} are forcings, not forecasts, and are not scored")
        sel = [c for c in names if (c in wanted if wanted else c not in forcings)]
        if len(sel) > E.ENS_MAX_CHANNELS:
            raise ValueError(f"{len(sel)} channels: at most {E.ENS_MAX_CHANNELS}")
        mch, slots = map_plan(map_leads, map_channels, sel, names, forcings, step_h,
                              f"map channel(s) {{}} are not shared by {self.model_names}")
        g = self.models[0].model.grid
        lat, lon = np.array(g.lat), np.array(g.lon)
        region_names, row_weights = S.region_weights(lat, regions)
        times = sorted({t + n * self.time_step for t in starts for n in range(n_steps + 1)})
        truth_at = S.truth_fetcher(self.data_source if truth is None else truth, sel, lat, lon, times)
        clim = S.climatology_fields(climatology, sel, lat, lon)
        if perturbation == "spherical_grf" and grf is None:
            grf = dict(lmax=min(180, (len(g.lat) - 1) // 2))

        entries = list(self.model_names) + ["pooled"]
        chans = [[m.out_channel_names.index(c) for c in sel] for m in self.models]
        offsets = [self._layout(m)[1] for m in self.models]
        mpos = [sel.index(c) for c in mch]
        D, L, R, Sn = len(starts), n_steps + 1, len(region_names), len(sel)
        init, states = None, None
        for d, t0 in enumerate(starts):
            if perturbation == "none":
                fresh = [torch.as_tensor(m._ensemble_initial_state(t0)[0], dtype=torch.float32, device=m.model.device)
                         [None].expand(members, -1, -1, -1) for m in self.models]
            else:
                fresh = self.ensemble_members(t0, members, perturbation, amp, seed + d, grf)
            if init is None:   # the member states, the results and the truth ring: allocated once for the campaign
                init = [f.contiguous() for f in fresh]
                dev = init[0].device
                H, W = init[0].shape[-2:]
                main = torch.cuda.current_stream(dev)
                sums = torch.empty((K + 1, D, L, R, Sn, len(S.SUMS)), dtype=torch.float64, device=dev)
                hist = [torch.empty((D, L, R, Sn, (K if e == K else 1) * members + 1), dtype=torch.float64, device=dev)
                        for e in range(K + 1)]
                maps = torch.zeros((K + 1, len(slots), len(mch), E.MAP_TERMS, H, W), dtype=torch.float64, device=dev)
                rw = torch.as_tensor(row_weights, dtype=torch.float64, device=dev).contiguous()
                kd = None if clim is None else torch.from_numpy(np.ascontiguousarray(clim, dtype=np.float32)).to(dev)
                ring = truth_ring(dev, Sn, H, W)
            else:
                for x, f in zip(init, fresh):
                    x.copy_(f)
            states = list(init)
            valid = [t0 + n * self.time_step for n in range(L)]
            for n in range(L):
                if n > 0:
                    self._step_all(states, first=n == 1)
                y = upload_truth(ring, n, truth_at(valid[n]), main)   # the host fetch runs under the forwards
                for k in range(K):
                    E.forecast_scores(states[k], y, rw, chans[k], kd, offsets[k], out=sums[k, d, n])
                    E.forecast_rank_histogram(states[k], y, rw, seed, d, n, chans[k], offsets[k], out=hist[k][d, n])
                    if n in slots:
                        for j, c in enumerate(mpos):
                            E.score_maps_accumulate(states[k], y[c:c + 1], maps[k, slots[n], j:j + 1], [chans[k][c]],
                                                    offsets[k])
                outs = self._outputs(states)
                E.forecast_scores_multi(outs, chans, y, rw, kd, out=sums[K, d, n])
                E.forecast_rank_histogram_multi(outs, chans, y, rw, seed, d, n, out=hist[K][d, n])
                if n in slots:
                    for j, c in enumerate(mpos):
                        E.score_maps_accumulate_multi(outs, [[ch[c]] for ch in chans], y[c:c + 1], maps[K, slots[n], j:j + 1])
                ring["scored"][n % 2].record(main)
            logger.success(f"Compared start date {d + 1}/{D}: {np.datetime64(t0, 's')}")
        sums, maps = sums.cpu().numpy(), maps.cpu().numpy()
        hours = [n * step_h for n in range(L)]
        scores = {e: S.PeriodScores.build(sums[i], hist[i].cpu().numpy(), maps[i] if mch else None,
                                          members * (K if i == K else 1), starts, hours, sorted(slots, key=slots.get),
                                          step_h, region_names, sel, mch, e, lat, lon)
                  for i, e in enumerate(entries)}
        res = S.ModelComparison.build(scores)
        paths = []
        if save:
            save_config = {k: v for k, v in save_config.items() if k != "filter_vars"}   # selected on the device already
            save_config.setdefault("forecast_id", generate_forecast_id())
            source = self.ic_source if isinstance(self.ic_source, str) else "file"
            label, t_end = f"{self.label}-compare{members}", starts[-1] + n_steps * self.time_step
            files = [("", res.card), ("-cards", _stack(res, "cards", "model"))]
            files += [(f"-rank-{e}", res.scores[e].rank_histogram) for e in entries]
            if mch:
                files.append(("-maps", _stack(res, "maps", "model")))
            files.append(("-diff", res.differences))
            for suffix, da in files:
                paths.append(save_forecast(da, label + suffix, starts[0], t_end, source, config=save_config))
        return res, paths

    # -- perturbed members ------------------------------------------------------------------------------------------------
    def predict_ensemble(self, start_time: datetime.datetime, n_steps: int, members: int, perturbation: str = "spherical_grf",
                         amp: float = 0.05, seed: int = 0, quantiles=(), events: dict = {}, channels: List[str] = [],
                         save: bool = False, save_config: dict = {}, grf: dict | None = None):
        """``GlobalModel.predict_ensemble`` over K models with ``members`` members each (K members at most 64 in all).

        The perturbation is drawn once, on the (members, union channels, H, W) initial condition, by ``perturb_ic`` /
        ``perturb_ic_grf`` (channel ids are union indices; GraphCast's forcing channel has sigma 0).  Member m of every
        model is gathered from member m of that tensor by channel name, so every model sees the same perturbation of the
        same variable; GraphCast adds it to both history slices and refills the forcing.  The union starts with the first
        model's channels in its order, so when the first model is Pangu or FourCastNet-v2 its members are bitwise those of
        its own ``predict_ensemble`` with the same seed, amplitude and perturbation.  Each step the K engines step in turn
        and one kernel reduces all K x members; only the statistics are copied to the host, each step's copy under the next
        step.  ``statistic`` is "mean", "spread", the quantiles, then "mean:<model>" for each model
        (``GlobalEnsemblePrediction.model_mean``).  ``channels`` and ``events`` must be shared channels.  Files are named
        "<sorted names joined by _>-ens<M>" and "...-prob"."""
        import torch
        from ... import engine as E
        K, names = len(self.models), self.shared_channels
        if not 1 <= members or K * members > ENS_MAX_MEMBERS:
            raise ValueError(f"members = {members} per model: {K} models x members must lie in [1, {ENS_MAX_MEMBERS}]")
        if n_steps < 1:
            raise ValueError(f"n_steps = {n_steps} must be at least 1")
        q = [float(v) for v in quantiles]
        if len(q) > E.ENS_MAX_QUANTILES or not all(0.0 <= v <= 1.0 for v in q):
            raise ValueError(f"quantiles {q}: at most {E.ENS_MAX_QUANTILES}, each in [0, 1]")
        ev = {c: [float(t) for t in np.atleast_1d(thr)] for c, thr in dict(events).items()}
        filt = list(save_config.get("filter_vars", ()))
        unknown = [c for c in list(channels) + filt + list(ev) if c not in names]
        if unknown:
            raise ValueError(f"channel(s) {unknown} are not shared by {self.model_names}")
        if not all(np.isfinite(t) for ts in ev.values() for t in ts):
            raise ValueError(f"event thresholds must be finite: {ev}")
        if save and save_config.get("file_type", "netcdf") == "zarr":
            raise ValueError("ensemble statistics are written as netCDF only: the zarr writer holds one variable per "
                             "forecast id")
        if perturbation not in ("gaussian", "spherical_grf"):
            raise ValueError(f"unknown perturbation {perturbation!r} (gaussian, spherical_grf)")
        if grf and perturbation != "spherical_grf":
            raise ValueError("grf options need perturbation='spherical_grf'")
        wanted = set(channels or filt or names) | set(ev)
        sel = [c for c in names if c in wanted]
        ev_list = [(i, t) for i, c in enumerate(sel) for t in ev.get(c, ())]
        if len(sel) > E.ENS_MAX_CHANNELS or len(ev_list) > E.ENS_MAX_EVENTS:
            raise ValueError(f"{len(sel)} channels and {len(ev_list)} events: at most {E.ENS_MAX_CHANNELS} and "
                             f"{E.ENS_MAX_EVENTS}")
        g = self.models[0].model.grid
        if perturbation == "spherical_grf" and grf is None:
            grf = dict(lmax=min(180, (len(g.lat) - 1) // 2))
        states = self.ensemble_members(start_time, members, perturbation, amp, seed, grf)
        chans = self._shared_index(sel)
        shapes = ((2 + len(q) + K, len(sel)) + tuple(states[0].shape[-2:]), (len(ev_list),) + tuple(states[0].shape[-2:]))

        def reduce(out):
            stats, prob = out
            E.multi_model_statistics(self._outputs(states), chans, q, ev_list,
                                     out=(stats[:2 + len(q)], prob, stats[2 + len(q):]))

        save_config = {k: v for k, v in save_config.items() if k != "filter_vars"}   # selected on the device already
        save_config.setdefault("forecast_id", generate_forecast_id())
        label, source = f"{self.label}-ens{members}", self.ic_source if isinstance(self.ic_source, str) else "file"
        lat, lon = np.array(g.lat), np.array(g.lon)
        stat_names = np.array(["mean", "spread"] + [quantile_name(v) for v in q] + [f"mean:{n}" for n in self.model_names])
        ev_names = np.array([event_name(sel[i], t) for i, t in ev_list])
        result, paths, prev, t_prev = None, [], None, start_time
        dev = states[0].device
        main, copy = torch.cuda.current_stream(dev), torch.cuda.Stream(dev)
        # EnsembleRunner.iter_stats' pattern over K engines: rings of two device and two pinned host buffers
        ring = [tuple(torch.empty(s, dtype=torch.float32, device=dev) for s in shapes) for _ in range(2)]
        host = [tuple(torch.empty(s, dtype=torch.float32).pin_memory() for s in shapes) for _ in range(2)]
        done = [torch.cuda.Event() for _ in range(2)]
        copied = torch.cuda.Event()
        reduce(ring[0])
        done[0].record(main)
        for n in range(n_steps + 1):
            if n < n_steps:   # launch step n + 1 and its reduction before waiting for the copy of step n
                self._step_all(states, first=n == 0)
                reduce(ring[(n + 1) % 2])
                done[(n + 1) % 2].record(main)
            copy.wait_event(done[n % 2])
            with torch.cuda.stream(copy):
                for h, d in zip(host[n % 2], ring[n % 2]):
                    h.copy_(d, non_blocking=True)
                copied.record(copy)
            copied.synchronize()   # also orders the next reduction into ring[n % 2] (launched at n + 1) after this copy
            s, p = host[n % 2]
            t_cur = start_time + n * self.time_step
            if n > 0 and (save or n == n_steps):
                times = np.array([np.datetime64(t_prev, "s"), np.datetime64(t_cur, "s")])
                stats = xr.DataArray(np.stack([prev[0], s.numpy()]), dims=["time", "statistic", "channel", "lat", "lon"],
                                     coords=dict(time=times, statistic=stat_names, channel=np.array(sel), lat=lat, lon=lon))
                prob = None
                if ev_list:
                    prob = xr.DataArray(np.stack([prev[1], p.numpy()]), dims=["time", "event", "lat", "lon"],
                                        coords=dict(time=times, event=ev_names, lat=lat, lon=lon))
                if save:
                    paths.append(save_forecast(stats, label, t_prev, t_cur, source, config=save_config))
                    if prob is not None:
                        paths.append(save_forecast(prob, f"{label}-prob", t_prev, t_cur, source, config=save_config))
                result = GlobalEnsemblePrediction(stats, prob, self.label, K * members)
            if n > 0:
                source = "file"
                logger.success(f"Multi-model ensemble step {n}/{n_steps} completed")
            prev, t_prev = (s.numpy().copy(), p.numpy().copy()), t_cur
        return result, paths

    def ensemble_members(self, start_time: datetime.datetime, members: int, perturbation: str = "spherical_grf",
                         amp: float = 0.05, seed: int = 0, grf: dict | None = None):
        """The perturbed initial states ``predict_ensemble`` steps: one (members, C_state, H, W) device tensor per model
        (a GraphCast state holds both slices)."""
        import torch
        from ...engine import perturb_ic, perturb_ic_grf
        from ...weights import channel_stats
        dev = self.models[0].model.device
        base = torch.from_numpy(np.ascontiguousarray(np.asarray(self.data_source[start_time].values, dtype=np.float32)))
        base = base.to(dev)
        sigma = channel_stats(self.channel_names)[1].copy()
        for m in self.models:
            if isinstance(m, GraphcastModel):
                sigma[self.channel_names.index(m.out_channel_names[m._cfg.n_state - 1])] = 0.0   # the toa forcing
        sigma = torch.as_tensor(sigma, device=dev)
        x = base[None].repeat(members, 1, 1, 1).contiguous()
        if perturbation == "gaussian":
            perturb_ic(x, sigma, amp, seed=seed)
        else:
            perturb_ic_grf(x, sigma, amp, seed=seed, **(grf or {}))
        states = []
        for m in self.models:
            idx = torch.tensor([self.channel_names.index(c) for c in m.in_channel_names], device=dev)
            xm = x.index_select(1, idx)
            if isinstance(m, GraphcastModel):
                # the same perturbation on both history slices: slice 0 = source[t - 6 h] + (member - source[t])
                prev = torch.from_numpy(np.asarray(m.data_source[start_time - m.time_step].values, dtype=np.float32))
                s0 = prev.to(dev)[None] + (xm - base.index_select(0, idx)[None])
                xm = m.model.fill_forcing(torch.stack([s0, xm], 1), start_time)
                m.model.engine.set_clock(start_time)
            states.append(xm.reshape(members, -1, *xm.shape[-2:]).contiguous())
        return states


def _stack(res, field: str, dim: str):
    """the entries' ``field`` DataArrays of a ModelComparison stacked along a new first dimension ``dim``"""
    das = [getattr(res.scores[e], field) for e in res.entries]
    first = das[0]
    return xr.DataArray(np.stack([da.values for da in das]), dims=[dim] + list(first.dims),
                        coords=dict({d: np.asarray(first.coords[d]) for d in first.dims}, **{dim: np.array(res.entries)}),
                        attrs=dict(res.card.attrs))
