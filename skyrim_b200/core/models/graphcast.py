"""GraphcastModel — mirrors /root/reference/skyrim/core/models/graphcast.py:44-177: ``build_model`` returns the CUDA
TimeLoop instead of ``graphcast.load_time_loop_operational(registry.get_model("e2mip://graphcast"))`` (:51-54); the
stepper protocol (``stepper.initialize`` / ``stepper.step``, :102-118), ``forecast`` (:122-142) and ``rollout`` (:144-177)
keep their signatures.  The state lives in HBM as a (B, 2, 83, nlat, nlon) tensor instead of an xarray Dataset."""
from __future__ import annotations

import datetime
from typing import List

import numpy as np
from loguru import logger

from ... import xr_shim as xr
from ...common import generate_forecast_id, save_forecast
from ...config import GRAPHCAST_CHANNELS, GraphCastConfig, graphcast_full
from .base import GlobalModel

# the reference's CHANNELS (:17-26) lists the same 83 names with z first; _to_global_da (:68-91) emits this order
CHANNELS = GRAPHCAST_CHANNELS


class GraphcastModel(GlobalModel):
    model_name = "graphcast"
    forcing_channels = (CHANNELS[-1],)   # "tp06", the toa radiation the engine recomputes every step

    def __init__(self, *args, cfg: GraphCastConfig | None = None, weights=None, weight_seed: int = 0, device: int = 0,
                 graph=None, **kwargs):
        self._cfg, self._weights, self._seed, self._device, self._graph = cfg or graphcast_full(), weights, weight_seed, device, graph
        super().__init__(self.model_name, *args, **kwargs)

    def build_model(self):
        from ...engine import StepEngine
        from ...timeloop import GraphcastTimeLoop
        from ...weights import make_graphcast_weights
        eng = StepEngine(self._cfg, self._device, graph=self._graph)
        # no network here: the JAX checkpoint the reference downloads is replaced by seeded synthetic parameters
        eng.load_weights(self._weights if self._weights is not None else make_graphcast_weights(self._cfg, self._seed))
        return GraphcastTimeLoop(eng)

    def build_datasource(self):
        if self.ic_source == "synthetic":
            return None   # _initial_state synthesises both history slices
        return super().build_datasource()

    @property
    def device(self):
        return self.model.device

    # -- state <-> DataArray ---------------------------------------------------------------------------------------
    def _to_global_da(self, fields, times) -> "xr.DataArray":
        """state tensor (1, T, 83, lat, lon) or array (T, 83, lat, lon) -> DataArray(time, channel, lat, lon) with the
        given valid times (graphcast.py:68-91 followed by the assign_coords of :139-142 / :163,177)"""
        vals = fields[0].cpu().numpy() if hasattr(fields, "cpu") else np.asarray(fields)
        g = self.model.grid
        return xr.DataArray(vals, dims=["time", "channel", "lat", "lon"],
                            coords=dict(time=np.array([np.datetime64(t, "s") for t in times]),
                                        channel=np.array(self.out_channel_names), lat=np.array(g.lat), lon=np.array(g.lon)))

    def _initial_state(self, start_time: datetime.datetime):
        """what get_initial_condition_for_model + stepper.initialize do upstream (graphcast.py:104-110)"""
        return self.model.stepper.initialize(self._initial_fields(start_time), start_time)

    def _ensemble_initial_state(self, start_time: datetime.datetime):
        """both slices, forcing filled, as one (2 * 83, H, W) state; the toa channels are not perturbed (sigma 0), the
        engine's clock is set, and the statistics are taken over slice 1 (the newest)"""
        from ...weights import channel_stats
        ns = self._cfg.n_state
        x = self._initial_fields(start_time)
        self.model.engine.set_clock(start_time)
        sigma = np.tile(channel_stats(self.out_channel_names)[1], 2)
        sigma[ns - 1] = sigma[2 * ns - 1] = 0.0
        return x.reshape(2 * ns, self._cfg.nlat, self._cfg.nlon), sigma, ns

    def _initial_fields(self, start_time: datetime.datetime):
        """(1, 2, 83, H, W) device tensor of the slices at start_time - 6 h and start_time, toa forcing filled"""
        import torch
        cfg = self._cfg
        if self.data_source is None:
            from ...weights import synthetic_graphcast_state
            x = torch.from_numpy(synthetic_graphcast_state(cfg, 0)).reshape(1, 2, cfg.n_state, cfg.nlat, cfg.nlon)
        else:
            step = self.time_step
            x = torch.from_numpy(np.stack([np.asarray(self.data_source[start_time - step].values, dtype=np.float32),
                                           np.asarray(self.data_source[start_time].values, dtype=np.float32)]))[None]
        x = x.to(self.model.device)
        return self.model.fill_forcing(x, start_time)

    def _predict_one_step(self, start_time: datetime.datetime, initial_condition: tuple | None = None):
        self.stepper = self.model.stepper
        state = self._initial_state(start_time) if initial_condition is None else initial_condition
        state, _ = self.stepper.step(state)
        logger.debug(f"state[0]: {state[0]}")
        return state

    def predict_one_step(self, start_time: datetime.datetime, initial_condition=None):
        state = self._predict_one_step(start_time, initial_condition)
        return self._to_global_da(state[1], [start_time, start_time + self.time_step])

    def forecast(self, start_time: datetime.datetime, n_steps: int = 4, channels: List[str] = []) -> "xr.DataArray":
        """(n_steps + 1, channel, lat, lon) from one device-resident chain (graphcast.py:122-142).  The reference flips
        the latitude axis here and not in rollout (:138 vs :164-166, SURVEY.md §3.4); the engine's grid is already the
        north-to-south order of the other models, so no flip is needed and both methods agree."""
        times = [start_time + i * self.time_step for i in range(n_steps + 1)]
        state, slices = None, []
        for n in range(n_steps):
            state = self._predict_one_step(start_time, initial_condition=state)
            logger.success(f"Forecast step {n + 1}/{n_steps} completed")
            slices.append((state[1][0] if n == 0 else state[1][0, -1:]).cpu().numpy())
        da = self._to_global_da(np.concatenate(slices, axis=0), times)
        return da.sel(channel=list(channels)) if channels else da

    def rollout(self, start_time: datetime.datetime, n_steps: int = 3, save: bool = True, save_config: dict = {},
                initial_condition=None):
        """(last prediction with 2 time slices, paths) like graphcast.py:144-177; ``initial_condition`` = a stepper state."""
        times = [start_time + i * self.time_step for i in range(n_steps + 1)]
        pred, output_paths, source = initial_condition, [], self.ic_source if isinstance(self.ic_source, str) else "file"
        save_config = dict(save_config)
        save_config.setdefault("forecast_id", generate_forecast_id())
        t = start_time
        for n in range(n_steps):
            pred = self._predict_one_step(t, initial_condition=pred)
            pred_time = t + self.time_step
            if save:
                output_paths.append(save_forecast(self._to_global_da(pred[1], [t, pred_time]), self.model_name, t, pred_time, source,
                                                  config=save_config))
            t, source = pred_time, "file"
            logger.success(f"Rollout step {n + 1}/{n_steps} completed")
        return self._to_global_da(pred[1], times[-2:]), output_paths
