"""`forecast` command line — mirrors /root/reference/skyrim/forecast.py:19-151 (same option names, short flags and
defaults; same `run_forecast` signature and return value) on top of the H100 engine:

    python -m skyrim_b200.forecast -m pangu -d 20240507 -t 0000 -l 24 -o outputs
    python -m skyrim_b200.forecast -m pangu -l 24 --members 8 --quantiles 0.1,0.5,0.9 --exceed t2m:273.15 -o outputs
    python -m skyrim_b200.forecast --models pangu,fourcastnet_v2,graphcast -l 24 --members 4 -o outputs
    python -m skyrim_b200.forecast -m pangu -l 168 --pangu_schedule hierarchical -o outputs
    python -m skyrim_b200.forecast -m pangu -l 72 --score --truth era5.nc --climatology clim.nc -o outputs
    python -m skyrim_b200.forecast -m pangu -d 20240501 -l 72 --score --until 20240531 --map_channels z500,t850 \
        --map_leads 24,72 --truth era5.nc -o outputs
    python -m skyrim_b200.forecast --models pangu,fourcastnet_v2,graphcast --compare -d 20240501 --until 20240531 -l 72 \
        --truth era5.nc --climatology clim.nc --map_channels z500 --map_leads 24,72 -o outputs
    python -m skyrim_b200.forecast -m pangu -l 72 --members 16 --sites cities.csv --quantiles 0.1,0.9 -o outputs
    python -m skyrim_b200.forecast -m pangu -d 20240501 --until 20240531 -l 72 --sites stations.csv \
        --observations synop.nc -o outputs

The second form runs a perturbed-initial-condition ensemble and saves its per-step statistics (mean, spread, quantiles)
and exceedance probabilities instead of the members.  The third runs several models side by side on one GPU
(``GlobalEnsemble``): with ``--members 1`` it saves every model's steps and their mean, above 1 the pooled statistics.
The fifth verifies the forecast (``--members`` members) against analyses and saves one scorecard of latitude-weighted
scores per lead time (``GlobalModel.score``).  With ``--until`` (or ``--every`` / ``--map_channels`` / ``--map_leads``) it
verifies every start date through the last one (``GlobalModel.score_period``) and saves the period's scorecard, the
per-date scorecards, the rank histogram and, for ``--map_channels`` at ``--map_leads``, per-point score maps.  The last
compares the ``--models`` head to head (``GlobalEnsemble.compare``) over the start dates ``--date`` .. ``--until`` (one
date without ``--until``): every model and their pooled ensemble are scored off one upload of each analysis, and the
stacked period card, the per-date cards, each entry's rank histogram, the maps and the paired score differences of
every pair of entries (mean, 95 % interval, p-value) are saved.  ``--sites`` saves the forecast of every member at the
sites of a CSV file (``GlobalModel.predict_sites``, bilinear or ``--site_method nearest``), with the site statistics above
one member; with ``--observations`` it verifies the forecast against station observations at those sites
(``GlobalModel.score_sites``) over the start dates ``--date`` .. ``--until``.

Differences, all forced by the scope of this build (SURVEY.md section 2): `--initial_conditions` accepts `synthetic`
(the default here: the network IC providers cds / ifs / gfs are the reference's `libs/ic`, out of scope, and raise a clear
error) or a path to a netCDF / .npy state; `--modal` (remote execution through Modal) is not available and says so;
`--weight_seed`, `--device` and `--grid` select the synthetic weight seed, the GPU and a coarse test grid."""
from __future__ import annotations

from datetime import datetime, timedelta
from pathlib import Path

import click
import numpy as np
from loguru import logger

from .common import AVAILABLE_MODELS
from .schedule import SCHEDULES

yesterday = (datetime.now() - timedelta(days=1)).date().isoformat().replace("-", "")


def run_forecast(model_name: str, date: str, time: str, lead_time: int, list_models: bool, initial_conditions: str,
                 output_dir: str, filter_vars: str, **model_kw):
    from .core import Skyrim
    if list_models:
        print("Available models:", Skyrim.list_available_models())
        return []
    logger.debug(f"Starting forecast run with model_name={model_name}, date={date}, time={time}, lead_time={lead_time}, "
                 f"initial_conditions={initial_conditions}, output_dir={output_dir}, filter_vars={filter_vars}")
    names = [model_name] if isinstance(model_name, str) else list(model_name)
    model = Skyrim(*names, ic_source=initial_conditions, **model_kw)
    pred, output_paths = model.predict(
        date=date, time=time, lead_time=lead_time, save=True,
        save_config={"output_dir": output_dir or str(Path.cwd() / "outputs"),
                     "filter_vars": [v.strip() for v in filter_vars.split(",") if v.strip()]})
    return output_paths


def run_ensemble_forecast(model_name: str, date: str, time: str, lead_time: int, initial_conditions: str, output_dir: str,
                          filter_vars: str, members: int, perturbation: str, amp: float, seed: int, quantiles=(),
                          events: dict = {}, **model_kw):
    """``--members`` > 1: ``Skyrim.predict_ensemble(save=True)``; returns the statistics and probability file paths"""
    from .core import Skyrim
    names = [model_name] if isinstance(model_name, str) else list(model_name)
    model = Skyrim(*names, ic_source=initial_conditions, **model_kw)
    _, paths = model.predict_ensemble(
        date=date, time=time, lead_time=lead_time, members=members, perturbation=perturbation, amp=amp, seed=seed,
        quantiles=quantiles, events=events, save=True,
        save_config={"output_dir": output_dir or str(Path.cwd() / "outputs"),
                     "filter_vars": [v.strip() for v in filter_vars.split(",") if v.strip()]})
    return paths


def run_score(model_name: str, date: str, time: str, lead_time: int, initial_conditions: str, output_dir: str,
              filter_vars: str, members: int, perturbation: str, amp: float, seed: int, truth: str = "",
              climatology: str = "", **model_kw):
    """``--score``: ``Skyrim.score(save=True)`` against the netCDF analyses ``truth`` (time, channel, lat, lon; default: the
    initial-condition source) and climatology (channel, lat, lon); returns the scorecard's path"""
    from . import xr_shim as xr
    from .core import Skyrim
    model = Skyrim(model_name, ic_source=initial_conditions, **model_kw)
    _, paths = model.score(
        date=date, time=time, lead_time=lead_time, members=members, perturbation=perturbation if members > 1 else None,
        amp=amp, seed=seed, truth=xr.open_dataarray(truth) if truth else None,
        climatology=xr.open_dataarray(climatology) if climatology else None, save=True,
        save_config={"output_dir": output_dir or str(Path.cwd() / "outputs"),
                     "filter_vars": [v.strip() for v in filter_vars.split(",") if v.strip()]})
    return paths


def run_score_period(model_name: str, date: str, time: str, lead_time: int, until: str, every: int, map_channels,
                     map_leads, initial_conditions: str, output_dir: str, filter_vars: str, members: int,
                     perturbation: str, amp: float, seed: int, truth: str = "", climatology: str = "", **model_kw):
    """``--score --until``: ``Skyrim.score_period(save=True)`` over the start dates ``date`` .. ``until``; returns the
    paths of the period card, the per-date cards, the rank histogram and the maps"""
    from . import xr_shim as xr
    from .core import Skyrim
    model = Skyrim(model_name, ic_source=initial_conditions, **model_kw)
    _, paths = model.score_period(
        start=date, end=until, time=time, every=every, lead_time=lead_time, members=members,
        perturbation=perturbation if members > 1 else None, amp=amp, seed=seed,
        truth=xr.open_dataarray(truth) if truth else None,
        climatology=xr.open_dataarray(climatology) if climatology else None, map_leads=map_leads,
        map_channels=map_channels, save=True,
        save_config={"output_dir": output_dir or str(Path.cwd() / "outputs"),
                     "filter_vars": [v.strip() for v in filter_vars.split(",") if v.strip()]})
    return paths


def run_compare(model_names, date: str, time: str, lead_time: int, until: str, every: int, map_channels, map_leads,
                initial_conditions: str, output_dir: str, filter_vars: str, members: int, perturbation: str, amp: float,
                seed: int, truth: str = "", climatology: str = "", **model_kw):
    """``--compare``: ``Skyrim(*model_names).compare(save=True)`` over the start dates ``date`` .. ``until``; returns the
    paths of the stacked card, the per-date cards, the rank histograms, the maps and the differences"""
    from . import xr_shim as xr
    from .core import Skyrim
    model = Skyrim(*model_names, ic_source=initial_conditions, **model_kw)
    _, paths = model.compare(
        start=date, end=until, time=time, every=every, lead_time=lead_time, members=members,
        perturbation=perturbation if members > 1 else None, amp=amp, seed=seed,
        truth=xr.open_dataarray(truth) if truth else None,
        climatology=xr.open_dataarray(climatology) if climatology else None, map_leads=map_leads,
        map_channels=map_channels, save=True,
        save_config={"output_dir": output_dir or str(Path.cwd() / "outputs"),
                     "filter_vars": [v.strip() for v in filter_vars.split(",") if v.strip()]})
    return paths


def run_sites(model_name: str, date: str, time: str, lead_time: int, sites: str, method: str, initial_conditions: str,
              output_dir: str, filter_vars: str, members: int, perturbation: str, amp: float, seed: int, quantiles=(),
              events: dict = {}, **model_kw):
    """``--sites``: ``Skyrim.predict_sites(save=True)`` at the sites of the CSV file ``sites`` (name,lat,lon); returns the
    paths of the site values, statistics and probabilities"""
    from .core import Skyrim
    model = Skyrim(model_name, ic_source=initial_conditions, **model_kw)
    _, paths = model.predict_sites(
        date=date, time=time, lead_time=lead_time, sites=sites, members=members, method=method,
        perturbation=perturbation if members > 1 else None, amp=amp, seed=seed, quantiles=quantiles, events=events,
        save=True, save_config={"output_dir": output_dir or str(Path.cwd() / "outputs"),
                                "filter_vars": [v.strip() for v in filter_vars.split(",") if v.strip()]})
    return paths


def run_score_sites(model_name: str, date: str, time: str, lead_time: int, until: str, every: int, sites: str, method: str,
                    observations: str, initial_conditions: str, output_dir: str, filter_vars: str, members: int,
                    perturbation: str, amp: float, seed: int, **model_kw):
    """``--sites --observations``: ``Skyrim.score_sites(save=True)`` against the netCDF observations (time, site, channel)
    at the sites of the CSV file ``sites``, chosen by name; returns the paths of the card, the per-date cards, the
    per-site scores and the counts"""
    from . import sites as St
    from . import xr_shim as xr
    from .core import Skyrim
    names = St.read_sites(sites)[0]
    obs = xr.open_dataarray(observations)
    have = [str(n) for n in np.asarray(obs.coords["site"])] if "site" in obs.coords else []
    unknown = [n for n in names if n not in have]
    if unknown:
        raise click.UsageError(f"--observations {observations} holds no site named {unknown}")
    model = Skyrim(model_name, ic_source=initial_conditions, **model_kw)
    _, paths = model.score_sites(
        date=date, time=time, lead_time=lead_time, observations=obs.sel(site=names), until=until, every=every,
        members=members, method=method, perturbation=perturbation if members > 1 else None, amp=amp, seed=seed,
        save=True, save_config={"output_dir": output_dir or str(Path.cwd() / "outputs"),
                                "filter_vars": [v.strip() for v in filter_vars.split(",") if v.strip()]})
    return paths


def parse_quantiles(text: str):
    """"0.1,0.5,0.9" -> [0.1, 0.5, 0.9]"""
    return [float(v) for v in text.split(",") if v.strip()]


def parse_exceed(text: str):
    """"t2m:273.15,u10m:15" -> {"t2m": [273.15], "u10m": [15.0]} (a channel may appear more than once)"""
    events = {}
    for item in (v.strip() for v in text.split(",")):
        if item:
            name, sep, thr = item.partition(":")
            if not sep:
                raise ValueError(f"--exceed item {item!r} is not channel:threshold")
            events.setdefault(name.strip(), []).append(float(thr))
    return events


@click.command()
@click.option("--model_name", "-m", type=click.Choice(AVAILABLE_MODELS, case_sensitive=False), default="pangu", help="Select model")
@click.option("--date", "-d", type=str, default=yesterday, help="YYYYMMDD")
@click.option("--time", "-t", type=str, default="0000", help="HHMM")
@click.option("--lead_time", "-l", type=int, default=6, help="Lead time in hours (floored to a multiple of 6)")
@click.option("--list_models", "-lm", is_flag=True, help="List all available models and exit")
@click.option("--initial_conditions", "-ic", type=str, default="synthetic",
              help="Initial conditions: 'synthetic' (seeded state) or a path to a netCDF / .npy state; cds / ifs / gfs need the "
                   "reference's network data sources")
@click.option("--output_dir", "-o", type=str, default="", help="Output directory (local)")
@click.option("--filter_vars", "-f", type=str, default="", help="Filter variables such as t2m (temperature) before saving forecasts.")
@click.option("--modal", "-mo", is_flag=True, help="(reference option) run on Modal — not available in this build")
@click.option("--weight_seed", type=int, default=0, help="seed of the synthetic weights (no checkpoint download here)")
@click.option("--device", type=int, default=0, help="CUDA device ordinal")
@click.option("--grid", type=str, default="", help="NLATxNLON coarse test grid (default: the model's 721x1440)")
@click.option("--members", type=int, default=1, help="Ensemble members (1..64); above 1, per-step ensemble statistics are saved")
@click.option("--perturbation", type=click.Choice(["spherical_grf", "gaussian"]), default="spherical_grf",
              help="Initial-condition perturbation of the ensemble members")
@click.option("--amp", type=float, default=0.05, help="Perturbation amplitude in units of each channel's standard deviation")
@click.option("--seed", type=int, default=0, help="Perturbation seed")
@click.option("--quantiles", type=str, default="", help="Ensemble quantiles such as 0.1,0.5,0.9")
@click.option("--exceed", type=str, default="", help="Exceedance events channel:threshold such as t2m:273.15,u10m:15")
@click.option("--models", type=str, default="",
              help="Several models side by side on one GPU, such as pangu,graphcast (replaces -m); --members counts per model")
@click.option("--pangu_schedule", type=click.Choice(SCHEDULES), default=None,
              help="Pangu alone: '6h' (default) chains the 6-h model; 'hierarchical' interleaves the 6-h and 24-h models "
                   "as earth2mip's PanguInference does")
@click.option("--score", is_flag=True, help="Verify the forecast (--members members) against analyses and save a scorecard")
@click.option("--compare", is_flag=True, help="Verify the --models and their pooled ensemble head to head over the start "
              "dates --date .. --until and save scores and paired differences")
@click.option("--truth", type=str, default="", help="--score / --compare: netCDF analyses (time, channel, lat, lon) on the model grid "
              "(default: the initial-condition source)")
@click.option("--climatology", type=str, default="", help="--score / --compare: netCDF climatology (channel, lat, lon) for "
              "the ACC")
@click.option("--until", type=str, default="", help="--score / --compare: the last start date YYYYMMDD; verifies every start "
              "date from --date through it and saves period scores and a rank histogram")
@click.option("--every", type=int, default=None, help="--score --until / --compare: hours between start dates (a multiple "
              "of 6; default 24)")
@click.option("--map_channels", type=str, default="", help="--score --until / --compare: channels of per-point score maps "
              "such as z500,t850")
@click.option("--map_leads", type=str, default="", help="--score --until / --compare: lead times in hours of the maps such "
              "as 24,72")
@click.option("--sites", type=str, default="", help="CSV file of sites name,lat,lon: save every member (and with --members > 1 "
              "the statistics) at those sites instead of the grid")
@click.option("--site_method", type=click.Choice(["bilinear", "nearest"]), default=None,
              help="--sites: interpolation to the sites (default bilinear)")
@click.option("--observations", type=str, default="", help="--sites: netCDF station observations (time, site, channel) with "
              "lat / lon along site; verifies the forecast at the --sites named there, from --date through --until")
def main(model_name, date, time, lead_time, list_models, initial_conditions, output_dir, filter_vars, modal, weight_seed, device, grid,
         members, perturbation, amp, seed, quantiles, exceed, models, pangu_schedule, score, compare, truth, climatology, until,
         every, map_channels, map_leads, sites="", site_method=None, observations=""):
    if modal:
        raise click.UsageError("--modal: remote execution through Modal is outside this build (SURVEY.md section 2); run locally")
    if not 1 <= members <= 64:
        raise click.UsageError(f"--members {members}: an ensemble holds 1 to 64 members on one GPU")
    try:
        q, events = parse_quantiles(quantiles), parse_exceed(exceed)
    except ValueError as e:
        raise click.UsageError(str(e))
    if compare and (not models.strip() or score or q or events or list_models):
        raise click.UsageError("--compare verifies several models (--models), without -m alone, --score, --quantiles, "
                               "--exceed or --list_models")
    if members == 1 and (q or events):
        raise click.UsageError("--quantiles and --exceed describe an ensemble: give --members > 1")
    kw = {"weight_seed": weight_seed, "device": device}
    names = [v.strip() for v in models.split(",") if v.strip()]
    unknown = [n for n in names if n not in AVAILABLE_MODELS]
    if unknown or len(set(names)) != len(names) or len(names) == 1 or len(names) * members > 64:
        raise click.UsageError(f"--models {models}: two to four distinct models of {AVAILABLE_MODELS}, at most 64 members "
                               "in all")
    if pangu_schedule is not None:
        if names or model_name != "pangu":
            raise click.UsageError("--pangu_schedule applies to -m pangu alone, not to --models or another model")
        kw["schedule"] = pangu_schedule
    if grid:
        from .config import graphcast_small, pangu_small, sfno_small
        nlat, nlon = (int(v) for v in grid.lower().split("x"))
        small = lambda n: (pangu_small(nlat, nlon) if n == "pangu" else graphcast_small(nlat, nlon) if n == "graphcast"  # noqa: E731
                           else sfno_small(nlat, nlon))
        if names:
            kw.update({n: dict(cfg=small(n)) for n in names})
        else:
            kw["cfg"] = small(model_name)
    if names:
        model_name = names
    if site_method is not None and not sites:
        raise click.UsageError("--site_method belongs to --sites")
    if observations and not sites:
        raise click.UsageError("--observations verifies at sites: give --sites too")
    if observations and (truth or climatology or compare or map_channels or map_leads):
        raise click.UsageError("--observations verifies against station observations, without --truth, --climatology, "
                               "--compare, --map_channels or --map_leads")
    if sites and (names or score or compare or list_models):
        raise click.UsageError("--sites forecasts one model (-m) at sites, without --models, --score, --compare or "
                               "--list_models")
    if observations and (q or events):
        raise click.UsageError("--observations verifies the forecast: --quantiles and --exceed belong to --sites alone")
    if sites and not observations and (until or every is not None or truth or climatology or map_channels or map_leads):
        raise click.UsageError("--sites alone forecasts: --until and --every need --observations, and --truth, "
                               "--climatology, --map_channels and --map_leads belong to --score or --compare")
    if observations:
        paths = run_score_sites(model_name, date, time, lead_time, until or date, 24 if every is None else every, sites,
                                site_method or "bilinear", observations, initial_conditions, output_dir, filter_vars,
                                members, perturbation, amp, seed, **kw)
        for p in paths:
            print(p)
        return paths
    if sites:
        paths = run_sites(model_name, date, time, lead_time, sites, site_method or "bilinear", initial_conditions,
                          output_dir, filter_vars, members, perturbation, amp, seed, q, events, **kw)
        for p in paths:
            print(p)
        return paths
    if (truth or climatology) and not (score or compare):
        raise click.UsageError("--truth and --climatology belong to --score or --compare")
    if score and (names or q or events or list_models):
        raise click.UsageError("--score verifies one model (-m), without --models, --quantiles, --exceed or --list_models")
    period = bool(until or every is not None or map_channels or map_leads)
    if period and not (score or compare):
        raise click.UsageError("--until, --every, --map_channels and --map_leads belong to --score or --compare")
    if period or compare:
        try:
            m_leads = [float(v) for v in map_leads.split(",") if v.strip()]
        except ValueError:
            raise click.UsageError(f"--map_leads {map_leads}: lead times in hours such as 24,72")
        m_chans = [v.strip() for v in map_channels.split(",") if v.strip()]
    if compare:
        paths = run_compare(model_name, date, time, lead_time, until or date, 24 if every is None else every, m_chans, m_leads,
                            initial_conditions, output_dir, filter_vars, members, perturbation, amp, seed, truth,
                            climatology, **kw)
    elif period:
        paths = run_score_period(model_name, date, time, lead_time, until or date, 24 if every is None else every, m_chans,
                                 m_leads, initial_conditions, output_dir, filter_vars, members, perturbation, amp, seed,
                                 truth, climatology, **kw)
    elif score:
        paths = run_score(model_name, date, time, lead_time, initial_conditions, output_dir, filter_vars, members,
                          perturbation, amp, seed, truth, climatology, **kw)
    elif members > 1 and not list_models:
        paths = run_ensemble_forecast(model_name, date, time, lead_time, initial_conditions, output_dir, filter_vars, members,
                                      perturbation, amp, seed, q, events, **kw)
    else:
        paths = run_forecast(model_name, date, time, lead_time, list_models, initial_conditions, output_dir, filter_vars, **kw)
    for p in paths:
        print(p)
    return paths


if __name__ == "__main__":
    main()
