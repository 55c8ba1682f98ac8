"""CPU tests: the oracle against the committed golden fixtures, structural properties of the
restated architecture, the fp16-operand error budget, and the host-side plumbing."""
import os
import re

import numpy as np
import pytest
import torch

from oracle.pangu_ref import PanguRef, position_index, rel_err_per_channel, shift_mask
from skyrim_b200.config import PANGU_CHANNELS, FCNV2_CHANNELS, pangu_full, pangu_small
from skyrim_b200.weights import (channel_stats, make_pangu_weights, n_params, pangu_param_shapes,
                                 synthetic_state)

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def small():
    cfg = pangu_small(41, 96)
    w = make_pangu_weights(cfg, 0)
    x0 = synthetic_state(PANGU_CHANNELS, cfg.nlat, cfg.nlon, 0)
    return cfg, w, x0


def test_channel_orders_match_reference():
    # /root/reference/skyrim/core/models/pangu.py:6-13, fourcastnet_v2.py:12-20
    assert len(PANGU_CHANNELS) == 69 and PANGU_CHANNELS[0] == "z1000" and PANGU_CHANNELS[13] == "q1000"
    assert PANGU_CHANNELS[64] == "v50" and PANGU_CHANNELS[65:] == ["msl", "u10m", "v10m", "t2m"]
    assert len(FCNV2_CHANNELS) == 73 and FCNV2_CHANNELS[:8] == ["u10m", "v10m", "u100m", "v100m", "t2m", "sp", "msl", "tcwv"]
    assert FCNV2_CHANNELS[8] == "u50" and FCNV2_CHANNELS[-1] == "r1000"


def test_full_config_geometry():
    c = pangu_full()
    assert (c.Z, c.H, c.W, c.H2, c.W2) == (8, 181, 360, 91, 180)
    assert c.padded_h(c.H) == 186 and c.padded_h(c.H2) == 96
    assert c.n_window_types(c.H) == 124 and c.n_window_types(c.H2) == 64 and c.bias_table_len == 3312
    shapes = pangu_param_shapes(c)
    total = sum(int(np.prod(s)) for k, s in shapes.items() if k != "const.masks")
    assert 60e6 < total < 70e6  # ~64 M parameters (SURVEY.md §8(d))


def test_oracle_matches_golden(small):
    cfg, w, x0 = small
    g = np.load(os.path.join(GOLD, "pangu_41x96_seed0.npz"))
    np.testing.assert_array_equal(x0[:, ::8, ::16], g["x0_sample"])
    y = PanguRef(cfg, w, torch.float32).step(x0).numpy()
    ys = y[:, ::5, ::12]
    scale = np.abs(g["y_sample"]).max(axis=(1, 2), keepdims=True)
    assert np.abs(ys - g["y_sample"]).max() / scale.max() < 1e-4
    assert np.max(np.abs(ys - g["y_sample"]) / scale) < 1e-4
    np.testing.assert_allclose(np.sqrt((y.astype(np.float64) ** 2).sum(axis=(1, 2))), g["y_norm"], rtol=1e-5)


def test_position_index_properties():
    idx = position_index((2, 6, 12))
    assert idx.shape == (144, 144) and int(idx.min()) == 0 and int(idx.max()) == 3311
    assert len(torch.unique(idx)) == 3312  # every table entry is addressed
    # relative in longitude: shifting both tokens along w by one keeps the index
    i = torch.arange(144).reshape(2, 6, 12)
    a, b = i[:, :, :-1].reshape(-1), i[:, :, 1:].reshape(-1)
    assert torch.equal(idx[a][:, a], idx[b][:, b])


def test_shift_mask_structure():
    cfg = pangu_full()
    m = shift_mask(cfg, 8, 186, 360, torch.float32)
    assert m.shape == (4 * 31, 144, 144)
    m = m.reshape(4, 31, 144, 144)
    assert float(m[:3, :30].abs().max()) == 0.0          # interior windows are unmasked
    assert float(m[3, 0].min()) == cfg.mask_value           # last z-window mixes both ends of Z
    assert torch.equal(m[3, 5], m[3, 5].transpose(0, 1))   # symmetric


def test_operator_is_periodic_in_longitude():
    """No mask along W: shifting the input by one coarse-window span of longitude (96 grid
    columns = 12 coarse tokens x 2 x 4) shifts the output by the same amount."""
    cfg = pangu_small(25, 192)
    w = make_pangu_weights(cfg, 2)
    w["const.masks"] = np.zeros_like(w["const.masks"])  # constant fields would break the symmetry
    x0 = synthetic_state(PANGU_CHANNELS, cfg.nlat, cfg.nlon, 1)
    ref = PanguRef(cfg, w)
    y0 = ref.step(x0)
    y1 = ref.step(np.roll(x0, 96, axis=-1))
    e = rel_err_per_channel(torch.roll(y0, 96, -1).numpy(), y1.numpy())
    assert e.max() < 1e-5, e.max()
    y2 = ref.step(np.roll(x0, 40, axis=-1))  # not a window multiple: no equivariance expected
    assert rel_err_per_channel(torch.roll(y0, 40, -1).numpy(), y2.numpy()).max() > 1e-4


def test_fp16_operand_error_budget(small):
    """What the tensor-core GEMMs do (fp16 operands, fp32 accumulate) stays inside the 1e-3 budget;
    bf16 operands would not — the reason the engine computes in fp16."""
    cfg, w, x0 = small
    y64 = PanguRef(cfg, w, torch.float64).step(x0).numpy()
    e16 = rel_err_per_channel(PanguRef(cfg, w, emulate="fp16").step(x0).numpy(), y64)
    eb16 = rel_err_per_channel(PanguRef(cfg, w, emulate="bf16").step(x0).numpy(), y64)
    assert e16.max() < 1e-3 and eb16.max() > 1e-3, (e16.max(), eb16.max())
    # the engine keeps the token stream only as its fp16 operand image (one extra rounding per residual add): still inside
    e16s = rel_err_per_channel(PanguRef(cfg, w, emulate="fp16s").step(x0).numpy(), y64)
    assert e16s.max() < 7.5e-4 and e16s.max() < 1.25 * e16.max(), (e16.max(), e16s.max())


def test_weights_are_deterministic_and_order_free(small):
    cfg, w, _ = small
    w2 = make_pangu_weights(cfg, 0)
    assert all(np.array_equal(w[k], w2[k]) for k in w)
    w3 = make_pangu_weights(cfg, 1)
    assert not np.array_equal(w["layer0.block0.qkv.w"], w3["layer0.block0.qkv.w"])
    assert n_params(w) == sum(int(np.prod(s)) for s in pangu_param_shapes(cfg).values())


def test_synthetic_state_statistics():
    x = synthetic_state(PANGU_CHANNELS, 61, 96, 0)
    mu, sd = channel_stats(PANGU_CHANNELS)
    z = (x - mu[:, None, None]) / sd[:, None, None]
    assert x.dtype == np.float32 and np.isfinite(x).all()
    assert np.abs(z.mean(axis=(1, 2))).max() < 0.6 and 0.3 < z.std() < 1.2


# ---- host plumbing / C-ABI ---------------------------------------------------------------
def test_pack_arena_roundtrip(small):
    from skyrim_b200.engine import pack_arena
    cfg, w, _ = small
    arena, man = pack_arena(w)
    assert arena.dtype == np.float32 and len(man) == len(w)
    for d, (k, a) in zip(man, w.items()):
        assert d.name.decode() == k and d.offset % 4 == 0
        np.testing.assert_array_equal(arena[d.offset:d.offset + d.count], a.reshape(-1))


def test_library_exports_every_declared_symbol():
    from skyrim_b200 import _ffi
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(__file__)), "include", "skyrim_b200.h")).read()
    declared = set(re.findall(r"\b(sky_[a-z_0-9]+)\s*\(", hdr))
    assert declared >= {"sky_model_create", "sky_model_step", "sky_model_load_weights", "sky_perturb_ic"}
    L = _ffi.lib()
    for name in declared:
        assert hasattr(L, name), name
    assert declared == set(_ffi.EXPORTS), declared ^ set(_ffi.EXPORTS)
    assert L.sky_abi_version() == 1


def test_no_cpu_fallback():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from skyrim_b200 import _ffi
    from skyrim_b200.engine import StepEngine
    with pytest.raises(_ffi.SkyError):
        StepEngine(pangu_small(41, 96), 0)
