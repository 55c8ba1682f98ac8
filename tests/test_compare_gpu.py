"""Model comparison on the GPU: the three *_multi verification entries bitwise against their single-source entries on the
pooled members, one case against the fp64 oracle, and GlobalEnsemble.compare on the Pangu + FourCastNet-v2 + GraphCast trio
against each model's own score_period / score."""
import datetime

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from oracle import scores_ref  # noqa: E402
from skyrim_b200 import engine as E  # noqa: E402
from skyrim_b200 import scores as S  # noqa: E402
from skyrim_b200 import xr_shim as xr  # noqa: E402
from skyrim_b200.config import graphcast_small, pangu_small, sfno_small  # noqa: E402
from skyrim_b200.timeloop import equiangular_grid  # noqa: E402

T0 = datetime.datetime(2024, 5, 7)
STEP = datetime.timedelta(hours=6)
H, W = 49, 96
REGIONS = {"global": (-90, 90), "tropics": (-20, 20)}


def make_sources(Ms, counts, pad=0, gc_slice=None, seed=0, quantise=False):
    """device sources (M_k, C_k, H, W): ``pad`` extra planes per member, source ``gc_slice`` the second half of a two-slice
    state (a GraphCast state's new slice); ``quantise`` rounds to integers, so members and truth tie often"""
    g = torch.Generator().manual_seed(seed)
    out = []
    for k, (M, Cn) in enumerate(zip(Ms, counts)):
        if k == gc_slice:
            full = torch.randn(M, 2 * Cn, H, W, generator=g) * 3 + 10
            full = (full.round() if quantise else full).cuda()
            out.append(full[:, Cn:])
        else:
            full = torch.randn(M, Cn + pad, H, W, generator=g) * 3 + 10
            full = (full.round() if quantise else full).cuda()
            out.append(full[:, :Cn])
    return out


def pooled_tensor(srcs, chans):
    """one contiguous tensor of the pooled members in source-then-member order, in source 0's channel layout"""
    C0 = srcs[0].shape[1]
    rows = []
    for x, ch in zip(srcs, chans):
        y = torch.zeros((x.shape[0], C0, H, W), device="cuda")
        y[:, chans[0]] = x[:, ch]
        rows.append(y)
    return torch.cat(rows).contiguous()


CASES = [((5,), (7,), 0, None), ((3, 4), (7, 9), 2, None), ((4, 4, 4), (69, 73, 83), 0, 2), ((1, 1, 1), (7, 8, 9), 0, 2),
         ((16, 16, 16, 16), (6, 7, 8, 9), 1, 1), ((1, 63), (5, 6), 3, None), ((1,), (4,), 0, None), ((2, 7), (5, 6), 0, 0)]


@pytest.mark.parametrize("quantise", [False, True])
@pytest.mark.parametrize("Ms, counts, pad, gc", CASES)
def test_multi_entries_are_bitwise_the_single_source_entries_on_the_pooled_members(Ms, counts, pad, gc, quantise):
    srcs = make_sources(Ms, counts, pad, gc, seed=sum(Ms), quantise=quantise)
    rng = np.random.default_rng(len(Ms) + sum(counts))
    chans = [[int(c) for c in rng.permutation(c)[:4]] for c in counts]
    pooled = pooled_tensor(srcs, chans)
    g = torch.Generator().manual_seed(7)
    truth = torch.randn(4, H, W, generator=g) * 3 + 10
    truth = (truth.round() if quantise else truth).cuda().contiguous()
    clim = (torch.randn(4, H, W, generator=g) + 10).cuda().contiguous()
    _, w = S.region_weights(np.asarray(equiangular_grid(H, W).lat), REGIONS)
    rw = torch.as_tensor(w, device="cuda").contiguous()
    got = E.forecast_scores_multi(srcs, chans, truth, rw, clim)
    want = E.forecast_scores(pooled, truth, rw, chans[0], clim)
    assert torch.equal(got, want)
    got = E.forecast_rank_histogram_multi(srcs, chans, truth, rw, 5, 3, 2)
    want = E.forecast_rank_histogram(pooled, truth, rw, 5, 3, 2, chans[0])
    assert torch.equal(got, want) and got.shape[-1] == sum(Ms) + 1
    maps = torch.zeros((4, E.MAP_TERMS, H, W), dtype=torch.float64, device="cuda")
    want_maps = torch.zeros_like(maps)
    for _ in range(2):
        E.score_maps_accumulate_multi(srcs, chans, truth, maps)
        E.score_maps_accumulate(pooled, truth, want_maps, chans[0])
    torch.cuda.synchronize()
    assert torch.equal(maps, want_maps)


def test_sixty_four_members_in_all_and_the_oracle():
    srcs = make_sources((20, 20, 24), (6, 7, 8), 1, 2, seed=3)
    chans = [[0, 5, 2], [6, 1, 3], [7, 0, 4]]
    pooled = pooled_tensor(srcs, chans)
    truth = (torch.randn(3, H, W) * 3 + 10).cuda().contiguous()
    clim = (torch.randn(3, H, W) + 10).cuda().contiguous()
    _, w = S.region_weights(np.asarray(equiangular_grid(H, W).lat), REGIONS)
    rw = torch.as_tensor(w, device="cuda").contiguous()
    got = E.forecast_scores_multi(srcs, chans, truth, rw, clim)
    assert torch.equal(got, E.forecast_scores(pooled, truth, rw, chans[0], clim))
    want, _ = scores_ref.score_sums(pooled.cpu().numpy(), truth.cpu().numpy(), w, chans[0], clim.cpu().numpy())
    np.testing.assert_allclose(got.cpu().numpy(), want, rtol=1e-9, atol=1e-9)


def test_refusals_on_the_device():
    srcs = make_sources((2, 2), (5, 5))
    host = srcs[1].cpu().pin_memory()
    truth = torch.zeros(1, H, W, device="cuda")
    rw = torch.ones(1, H, dtype=torch.float64, device="cuda") / H
    with pytest.raises(ValueError, match="CUDA"):
        E.forecast_scores_multi([srcs[0], host], [[0], [0]], truth, rw)
    with pytest.raises(E._ffi.SkyError, match="total members"):
        E.forecast_scores_multi(make_sources((40, 25), (2, 2)), [[0], [0]], truth, rw)


# ---- the trio head to head -------------------------------------------------------------------------------------------------
CFG = dict(pangu=dict(cfg=pangu_small(H, W)), fourcastnet_v2=dict(cfg=sfno_small(H, W, 64, 3)),
           graphcast=dict(cfg=graphcast_small(H, W, 2, 512, 2)))
NAMES = ("pangu", "fourcastnet_v2", "graphcast")


class TimeSource:
    """seeded analyses that change with time over the union channels"""

    def __init__(self, channels, nlat, nlon):
        from skyrim_b200.weights import channel_stats, synthetic_state
        self.channels, self.grid = list(channels), equiangular_grid(nlat, nlon)
        self.base, self.sigma = synthetic_state(self.channels, nlat, nlon, 0), channel_stats(self.channels)[1]

    def __getitem__(self, t):
        h = int((t - datetime.datetime(2024, 1, 1)).total_seconds() // 3600)
        eps = np.random.default_rng(h).standard_normal(self.base.shape).astype(np.float32)
        v = (self.base + np.float32(0.05) * self.sigma[:, None, None] * eps).astype(np.float32)
        return xr.DataArray(v, dims=["channel", "lat", "lon"], coords=dict(channel=np.array(self.channels),
                            lat=np.array(self.grid.lat), lon=np.array(self.grid.lon)))


def _union():
    from skyrim_b200.config import FCNV2_CHANNELS, GRAPHCAST_CHANNELS, PANGU_CHANNELS
    u = list(PANGU_CHANNELS)
    for ch in (FCNV2_CHANNELS, GRAPHCAST_CHANNELS):
        u += [c for c in ch if c not in u]
    return u


@pytest.fixture(scope="module")
def trio():
    from skyrim_b200.core.skyrim import Skyrim
    sk = Skyrim(*NAMES, ic_source=TimeSource(_union(), H, W), **CFG)
    yield sk
    sk.model.release_model()


def _own(ens, name):
    """the ensemble's own handle of a model: a GlobalModel reading the shared source through a SourceView, as
    Skyrim(name, ic_source=SourceView(ens.data_source, its channels)) does, on the same engine"""
    return ens.models[ens.model_names.index(name)]


def _clim(trio):
    da = trio.model.data_source[T0 - 30 * STEP]
    return xr.DataArray(da.values * np.float32(0.999), dims=["channel", "lat", "lon"], coords=dict(
        channel=np.asarray(da.coords["channel"]), lat=np.asarray(da.coords["lat"]), lon=np.asarray(da.coords["lon"])))


def test_trio_members_1_against_each_model_alone(trio):
    ens = trio.model
    starts, n_steps, seed = [T0, T0 + 2 * STEP, T0 + 4 * STEP], 2, 9
    clim = _clim(trio)
    mch = ["z500", "t850"]
    res, _ = ens.compare(starts, n_steps, climatology=clim, regions=REGIONS, map_leads=[6, 12], map_channels=mch, seed=seed)
    sel = list(res.card.coords["channel"])
    assert res.entries == list(NAMES) + ["pooled"] and tuple(res.card.dims) == ("model", "lead_time", "metric", "region",
                                                                                "channel")
    assert res.differences.values.shape == (6, 3, 5, n_steps + 1, 2, len(sel))
    for name in NAMES:
        own, _ = _own(ens, name).score_period(starts, n_steps, climatology=clim, channels=sel, regions=REGIONS,
                                              map_leads=[6, 12], map_channels=mch, seed=seed)
        got = res.scores[name]      # the comparison keeps the shared channels in the first model's order: select by name
        assert got.cards.values.tobytes() == own.cards.sel(channel=sel).values.tobytes(), name
        assert got.rank_histogram.values.tobytes() == own.rank_histogram.sel(channel=sel).values.tobytes(), name
        assert got.maps.values.tobytes() == own.maps.sel(channel=mch).values.tobytes(), name
    # the pooled entry: the single-source entries on the concatenated states, stepped by hand
    _, w = S.region_weights(np.asarray(ens.models[0].model.grid.lat), REGIONS)
    rw = torch.as_tensor(w, device="cuda").contiguous()
    chans = ens._shared_index(sel)
    kd = torch.from_numpy(S.climatology_fields(clim, sel, ens.models[0].model.grid.lat, ens.models[0].model.grid.lon)).cuda()
    for d, t0 in enumerate(starts):
        states = [torch.as_tensor(m._ensemble_initial_state(t0)[0], device="cuda")[None].contiguous() for m in ens.models]
        for n in range(n_steps + 1):
            if n:
                ens._step_all(states, first=n == 1)
            y = torch.from_numpy(np.ascontiguousarray(ens.data_source[t0 + n * STEP].sel(channel=sel).values)).cuda()
            pooled = pooled_tensor(ens._outputs(states), chans)
            sums = E.forecast_scores(pooled, y, rw, chans[0], kd).cpu().numpy()
            want = np.moveaxis(S.metrics_from_sums(sums, 3), -1, 0)
            assert res.scores["pooled"].cards.values[d, n].tobytes() == want.tobytes(), (d, n)
    np.testing.assert_array_equal(res.differences.values[0], S.paired_differences(res.scores["pangu"].cards.values,
                                                                                  res.scores["fourcastnet_v2"].cards.values))


def test_trio_members_2(trio):
    ens = trio.model
    starts, seed = [T0, T0 + 4 * STEP], 3
    res, _ = ens.compare(starts, 1, members=2, regions=REGIONS, seed=seed)
    sel = list(res.card.coords["channel"])
    own, _ = _own(ens, "pangu").score_period(starts, 1, members=2, channels=sel, regions=REGIONS, seed=seed)
    assert res.scores["pangu"].cards.values.tobytes() == own.cards.values.tobytes()
    h = res.scores["pooled"].rank_histogram.values
    assert h.shape[-1] == 2 * 3 + 1
    np.testing.assert_allclose(h.sum(-1), 1.0, rtol=1e-12)


def test_cli_compare_until(tmp_path):
    from click.testing import CliRunner
    from skyrim_b200 import forecast as F
    r = CliRunner().invoke(F.main, ["--models", "pangu,fourcastnet_v2,graphcast", "--grid", "49x96", "--compare", "-d",
                                    "20240507", "--until", "20240508", "-l", "6", "-o", str(tmp_path),
                                    "--map_channels", "z500", "--map_leads", "6"])
    assert r.exit_code == 0, r.output
    paths = [ln for ln in r.output.splitlines() if ln.endswith(".nc")]
    label = "fourcastnet_v2_graphcast_pangu-compare1"
    assert sorted(p.split("/")[-1].split("__")[0] for p in paths) == sorted(
        [label, label + "-cards", label + "-maps", label + "-diff"] + [f"{label}-rank-{e}" for e in NAMES + ("pooled",)])
    for p in paths:
        assert np.isfinite(np.asarray(xr.open_dataarray(p).values, dtype=np.float64)).any()


def test_full_size_deterministic_trio():
    from skyrim_b200.core.skyrim import Skyrim
    sk = Skyrim(*NAMES)
    ens = sk.model
    starts = [T0, T0 + 4 * STEP]
    res, _ = ens.compare(starts, 1)
    sel = list(res.card.coords["channel"])
    for name in NAMES:
        for d, t0 in enumerate(starts):
            card, _ = _own(ens, name).score(t0, 1, channels=sel)
            assert res.scores[name].cards.values[d].tobytes() == card.sel(channel=sel).values.tobytes(), (name, d)
    ens.release_model()
