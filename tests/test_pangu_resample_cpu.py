"""CPU checks of the float64 references of Pangu's down-sample, up-sample and patch recovery (oracle/pangu_resample_ref.py)
that tests/test_pangu_resample_gpu.py compares the engine against: with unrounded inputs they are the model
(PanguRef), a float32 / fp16 emulation of each kernel's arithmetic stays within their bounds, and each modelled kernel
mistake leaves the bounds at some element on inputs of the GPU cases' shapes and scale."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle import gemm_ref as gr
from oracle import pangu_resample_ref as pr
from oracle.pangu_ref import PanguRef
from skyrim_b200.config import pangu_small
from skyrim_b200.weights import make_pangu_weights

GRIDS = [(41, 96), (33, 96), (45, 192), (24, 96)]      # those of the GPU cases: H 11, 9 (odd), 12, 6 (even)
# token scales of the engine's streams at these grids (PanguRef stages, weights seed 1, state seed 3): skip and x1 std
# about 2, the level-2 stream after layer 2 std about 5
SKIP_STD, X1_STD, X2_STD = 2.0, 2.0, 5.0
F32 = np.float32


def _tokens(rng, rows, cols, std, round16=True):
    x = rng.standard_normal((rows, cols)) * std
    return x.astype(np.float16).astype(np.float64) if round16 else x


def _inputs(cfg, B, seed, round16=True):
    """level-1 tokens (the down-sample's input), level-2 tokens (the up-sample's), and the skip and x1 tokens of the
    recovery, at the scale of the engine's streams"""
    rng = np.random.default_rng(seed)
    T1, T2, C = cfg.Z * cfg.H * cfg.W, cfg.Z * cfg.H2 * cfg.W2, cfg.dim
    return (_tokens(rng, B * T1, C, SKIP_STD, round16), _tokens(rng, B * T2, 2 * C, X2_STD, round16),
            _tokens(rng, B * T1, C, SKIP_STD, round16), _tokens(rng, B * T1, C, X1_STD, round16))


# ---------------------------------------------------------------------------------------------------------------------
# workspace layout and index maps
# ---------------------------------------------------------------------------------------------------------------------
def test_workspace_layout_by_hand():
    """41 x 96, B = 1: T1 = 8 * 11 * 24 = 2112 (17 row tiles), T2 = 8 * 6 * 12 = 576 (5 tiles); window tiles: g1 4 * 2 * 2
    = 16 windows x 3 head pairs = 48, g2 4 * 1 * 1 windows x 6 pairs = 24"""
    lay = pr.workspace_layout(pangu_small(41, 96), 1)
    x1, x2 = 2112 * 192 * 4, 576 * 384 * 4
    img1 = 17 * 3 * 16384
    assert lay["x1"] == 0 and lay["x2"] == x1 and lay["x1h"] == x1 + x2
    assert lay["skiph"] == lay["x1h"] + img1 and lay["x2h"] == lay["skiph"] + img1
    assert lay["qkv"] == lay["x2h"] + 5 * 6 * 16384
    assert lay["atth"] == lay["qkv"] + 3 * 48 * 18432
    assert lay["hidh"] == lay["atth"] + max(17 * 3, 5 * 6) * 16384
    assert lay["total"] == lay["hidh"] + max(17 * 12, 5 * 24) * 16384
    assert all(v % 1024 == 0 for v in lay.values())


@pytest.mark.parametrize("nlat,nlon", GRIDS)
def test_index_maps_cover_each_element_once(nlat, nlon):
    cfg, B = pangu_small(nlat, nlon), 3
    T1 = cfg.Z * cfg.H * cfg.W
    src = pr.merge_sources(cfg, B)
    s = np.sort(src[src >= 0])
    assert np.array_equal(s, np.arange(B * T1)), "every level-1 token in exactly one merge slot"
    assert (src < 0).sum() == (cfg.H % 2) * B * cfg.Z * cfg.W2 * 2
    coarse, sub = pr.shuffle_sources(cfg, B)
    assert (coarse >= 0).all()
    assert np.unique(coarse * 4 + sub).size == B * T1
    flat, _, _ = pr.recover_targets(cfg, B)
    f = np.sort(flat[flat >= 0])
    assert np.array_equal(f, np.arange(B * cfg.n_channels * nlat * nlon)), "every output element written exactly once"


# ---------------------------------------------------------------------------------------------------------------------
# same model: unrounded inputs and weights give PanguRef's downsample, upsample and patch_recover
# ---------------------------------------------------------------------------------------------------------------------
def _model_cases():
    return [((nlat, nlon), 2) for nlat, nlon in GRIDS] + [((721, 1440), 1)]


@pytest.mark.parametrize("grid,B", _model_cases(), ids=lambda v: f"{v[0]}x{v[1]}" if isinstance(v, tuple) else f"B{v}")
def test_references_equal_the_model(grid, B):
    cfg = pangu_small(*grid)
    w = make_pangu_weights(cfg, 1)
    gw = pr.gemm_weights(cfg, w, round16=False)
    model = PanguRef(cfg, w, dtype=torch.float64)
    C, Z, H, W, H2, W2 = cfg.dim, cfg.Z, cfg.H, cfg.W, cfg.H2, cfg.W2
    T1 = Z * H * W
    x1, x2, skip, xu = _inputs(cfg, B, 5, round16=False)
    chunk = 1 << 16

    def close(got, want):
        scale = np.abs(want).max()
        assert np.abs(got - want).max() <= 1e-12 * scale, float(np.abs(got - want).max() / scale)

    # down-sample: merge + LayerNorm, then the down GEMM
    R2 = B * Z * H2 * W2
    down = np.concatenate([pr.linear_plain(pr.down_merge_ln(cfg, w, x1, B, np.arange(s, min(s + chunk, R2)))[0], gw["down"])[0]
                           for s in range(0, R2, chunk)])
    for m in range(B):
        want = model.downsample(torch.from_numpy(x1[m * T1:(m + 1) * T1].reshape(Z, H, W, C))).numpy()
        close(down.reshape(B, Z, H2, W2, 2 * C)[m], want)
    del down
    # up-sample: linear1 + shuffle + crop + LayerNorm, then linear2
    R1 = B * T1
    up = np.concatenate([pr.linear_plain(pr.up_shuffle(cfg, w, x2, gw["up1"], B, np.arange(s, min(s + chunk, R1)))[0], gw["up2"])[0]
                         for s in range(0, R1, chunk)])
    T2 = Z * H2 * W2
    for m in range(B):
        want = model.upsample(torch.from_numpy(x2[m * T2:(m + 1) * T2].reshape(Z, H2, W2, 2 * C))).numpy()
        close(up.reshape(B, Z, H, W, C)[m], want)
    del up
    # recovery: [skip | x1] -> de-normalised state
    a = np.concatenate([skip, xu], 1)
    out = np.full(B * cfg.n_channels * cfg.nlat * cfg.nlon, np.nan)
    for s in range(0, R1, chunk):
        r = np.arange(s, min(s + chunk, R1))
        flat, ref, _ = pr.recover(cfg, w, a[r], gw["rec"], B, r)
        out[flat] = ref
    out = out.reshape(B, cfg.n_channels, cfg.nlat, cfg.nlon)
    assert not np.isnan(out).any()
    for m in range(B):
        xm = torch.from_numpy(a[m * T1:(m + 1) * T1].reshape(Z, H, W, 2 * C))
        close(out[m], model.patch_recover(xm).numpy())


# ---------------------------------------------------------------------------------------------------------------------
# the bounds hold: float32 / fp16 emulations of the kernels' arithmetic
# ---------------------------------------------------------------------------------------------------------------------
def _warp_sum(v):
    """warp_sum over the lane axis (last): xor butterfly 16, 8, 4, 2, 1 in fp32"""
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., lanes ^ o]).astype(F32)
    return v


def _emulate_merge_ln(cfg, w, x, B):
    """k_down_merge_ln in fp32: lane l holds features 4 l + 128 i + j, per-lane sums in the kernel's order"""
    src = pr.merge_sources(cfg, B)
    v = np.where((src >= 0)[:, :, None], x[np.maximum(src, 0)], 0.0).astype(F32).reshape(-1, 6, 32, 4)   # [row, i, lane, j]
    s = np.zeros((v.shape[0], 32), F32)
    for i in range(6):
        s = (s + ((v[:, i, :, 0] + v[:, i, :, 1]) + (v[:, i, :, 2] + v[:, i, :, 3]))).astype(F32)
    mean = (_warp_sum(s)[:, :1] / F32(768)).astype(F32)                   # [row, 1]
    ss = np.zeros_like(s)
    for i in range(6):
        for j in range(4):
            d = (v[:, i, :, j] - mean).astype(F32)
            ss = (ss.astype(np.float64) + d.astype(np.float64) * d).astype(F32)   # fma
    var = (_warp_sum(ss)[:, :1] / F32(768)).astype(F32)
    rstd = (1.0 / np.sqrt((var + F32(cfg.ln_eps)).astype(np.float64))).astype(F32)
    g = np.asarray(w["down.ln.g"], F32).reshape(1, 6, 32, 4)
    b = np.asarray(w["down.ln.b"], F32).reshape(1, 6, 32, 4)
    yn = ((v - mean[:, :, None, None]).astype(F32) * rstd[:, :, None, None]).astype(F32)
    return ((yn * g).astype(F32) + b).astype(F32).reshape(-1, 768).astype(np.float16)


def _emulate_gemm(a, wt):
    return np.asarray(a, F32) @ np.asarray(wt, F32).T


def _emulate_shuffle(cfg, w, x2, wu1, B):
    C = cfg.dim
    coarse, sub = pr.shuffle_sources(cfg, B)
    acc = _emulate_gemm(x2, wu1).reshape(-1, 4, C)[coarse, sub]            # [R1, C] fp32
    s = np.cumsum(acc, 1, dtype=F32)[:, -1:]                              # sequential fp32 sums, as one thread adds them
    mean = (s / F32(C)).astype(F32)
    d = (acc - mean).astype(F32)                                           # second pass, about the mean
    var = (np.cumsum((d * d).astype(F32), 1, dtype=F32)[:, -1:] / F32(C)).astype(F32)
    rstd = (1.0 / np.sqrt((var + F32(cfg.ln_eps)).astype(np.float64))).astype(F32)
    yn = ((acc - mean).astype(F32) * rstd).astype(F32)
    return ((yn * np.asarray(w["up.ln.g"], F32)).astype(F32) + np.asarray(w["up.ln.b"], F32)).astype(np.float16)


def _emulate_recover(cfg, w, a, wrec, B):
    flat, bidx, sch = pr.recover_targets(cfg, B)
    acc = _emulate_gemm(a, wrec)
    bias = np.concatenate([w["recover.upper.b"], w["recover.surf.b"]]).astype(F32)
    y = (((acc + bias[bidx]).astype(F32) * np.asarray(w["norm.std"], F32)[sch]).astype(F32)
         + np.asarray(w["norm.mean"], F32)[sch]).astype(F32)
    return flat[flat >= 0], y[flat >= 0]


@pytest.mark.parametrize("nlat,nlon", [(41, 96), (24, 96)])
def test_bounds_hold_for_emulated_kernels(nlat, nlon):
    cfg, B = pangu_small(nlat, nlon), 3
    w = make_pangu_weights(cfg, 1)
    gw = pr.gemm_weights(cfg, w)
    x1, x2, skip, xu = _inputs(cfg, B, 6)
    checks = []
    ref, bnd = pr.down_merge_ln(cfg, w, x1, B)
    hid = _emulate_merge_ln(cfg, w, x1, B)
    checks.append(("merge + LayerNorm", hid, ref, bnd))
    ref, bnd = pr.linear_plain(hid, gw["down"])
    acc = _emulate_gemm(hid, gw["down"])
    checks += [("down GEMM fp32", acc, ref, bnd), ("down GEMM fp16", acc.astype(np.float16), ref, gr.f16_bound(ref, bnd))]
    ref, bnd = pr.up_shuffle(cfg, w, x2, gw["up1"], B)
    hid = _emulate_shuffle(cfg, w, x2, gw["up1"], B)
    checks.append(("up-sample linear1 + shuffle", hid, ref, bnd))
    ref, bnd = pr.linear_plain(hid, gw["up2"])
    acc = _emulate_gemm(hid, gw["up2"])
    checks += [("up-sample linear2 fp32", acc, ref, bnd), ("up-sample linear2 fp16", acc.astype(np.float16), ref, gr.f16_bound(ref, bnd))]
    a = np.concatenate([skip, xu], 1)
    flat, ref, bnd = pr.recover(cfg, w, a, gw["rec"], B)
    eflat, got = _emulate_recover(cfg, w, a, gw["rec"], B)
    assert np.array_equal(flat, eflat)
    checks.append(("recovery", got, ref, bnd))
    for name, got, ref, bnd in checks:
        assert np.isfinite(ref).all() and (bnd > 0).all(), name
        r = gr.worst(got, ref, bnd)
        print(f"[pangu resample emulation] {nlat}x{nlon} {name}: largest |error| / bound {r:.3f}")
        assert r <= 1, (name, r)
        # the bound is tight enough to notice a few ulps: 4 fp16 ulps off at one element leave it
        if got.dtype == np.float16:
            bad = got.astype(np.float64)
            i = np.unravel_index(np.argmax(np.abs(ref)), ref.shape)
            bad[i] += 4 * gr.ulp16(ref[i])
            assert gr.exceed(bad, ref, bnd)[i], name


# ---------------------------------------------------------------------------------------------------------------------
# the bounds catch mistakes: each modelled kernel mistake leaves the bound at some element
# ---------------------------------------------------------------------------------------------------------------------
def _ratio(got, ref, bnd):
    """largest |got - ref| / bound; an element one of them leaves unwritten (NaN) counts as infinitely far"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    d = np.abs(got - ref) / bnd
    return float(np.where(np.isnan(d), np.inf, d).max())


@pytest.mark.parametrize("nlat,nlon", GRIDS)
def test_bounds_flag_every_mutation(nlat, nlon):
    """at every grid of the GPU cases with B = 3: a kernel making one of these mistakes lands within its own bound
    (about the same) of the mutated reference, so the mutated reference must be > 3 bounds from the correct one"""
    cfg, B = pangu_small(nlat, nlon), 3
    w = make_pangu_weights(cfg, 1)
    gw = pr.gemm_weights(cfg, w)
    x1, x2, skip, xu = _inputs(cfg, B, 7)
    T1, T2 = cfg.Z * cfg.H * cfg.W, cfg.Z * cfg.H2 * cfg.W2
    odd = cfg.H % 2 == 1
    res = {}

    ref, bnd = pr.down_merge_ln(cfg, w, x1, B)
    for name, kw in [("merge: (hs, ws) swapped", dict(swap=True))] + [("merge: padding zeros left out of the statistics",
                                                                       dict(pad_stats=False))] * odd:
        res[name] = _ratio(pr.down_merge_ln(cfg, w, x1, B, **kw)[0], ref, bnd)
    res["merge: member stride (Z - 1) H W"] = _ratio(
        pr.down_merge_ln(cfg, w, pr.restride(x1, B, T1, T1 - cfg.H * cfg.W), B)[0], ref, bnd)
    # the down GEMM and linear2 are plain products over whole rows: their only index is the member's, on the A rows
    hid = ref.astype(np.float16)
    ref, bnd = pr.linear_plain(hid, gw["down"])
    res["down GEMM: member stride"] = _ratio(pr.linear_plain(pr.restride(hid, B, T2, T2 - cfg.H2 * cfg.W2), gw["down"])[0],
                                             ref, bnd)

    ref, bnd = pr.up_shuffle(cfg, w, x2, gw["up1"], B)
    muts = {"shuffle: (hs, ws) swapped": dict(swap=True), "shuffle: crop at H - 1": dict(h_lim=cfg.H - 1),
            "shuffle: LayerNorm over 4C": dict(ln_cols=4 * cfg.dim)}
    if odd:
        muts["shuffle: crop at H + 1"] = dict(h_lim=cfg.H + 1)
    for name, kw in muts.items():
        res[name] = _ratio(pr.up_shuffle(cfg, w, x2, gw["up1"], B, **kw)[0], ref, bnd)
    res["shuffle: member stride"] = _ratio(
        pr.up_shuffle(cfg, w, pr.restride(x2, B, T2, T2 - cfg.H2 * cfg.W2), gw["up1"], B)[0], ref, bnd)
    hid = ref.astype(np.float16)
    ref, bnd = pr.linear_plain(hid, gw["up2"])
    res["up linear2: member stride"] = _ratio(
        pr.linear_plain(pr.restride(hid, B, T1, T1 - cfg.H * cfg.W), gw["up2"])[0], ref, bnd)

    shape = (B, cfg.n_channels, nlat, nlon)
    a = np.concatenate([skip, xu], 1)
    flat, ref, bnd = pr.recover(cfg, w, a, gw["rec"], B)
    ref, bnd = pr.scatter(flat, ref, shape), pr.scatter(flat, bnd, shape)
    for name, kw in [("recovery: dz swapped", dict(dz_swap=True)), ("recovery: level pair from z", dict(level_from_z=True)),
                     ("recovery: surface bias of the next variable", dict(surf_nb_bias=True)),
                     ("recovery: surface statistics of the next variable", dict(surf_nb_stats=True))]:
        f, r, _ = pr.recover(cfg, w, a, gw["rec"], B, **kw)
        res[name] = _ratio(pr.scatter(f, r, shape), ref, bnd)
    f, r, _ = pr.recover(cfg, w, pr.restride(a, B, T1, T1 - cfg.H * cfg.W), gw["rec"], B)
    res["recovery: member stride"] = _ratio(pr.scatter(f, r, shape), ref, bnd)

    assert len(res) == 13 + 2 * odd
    for name, r in res.items():
        print(f"[pangu resample discrimination] {nlat}x{nlon} B {B} {name}: max |mutated - ref| / bound = {r:.1f}")
    low = {k: r for k, r in res.items() if not r > 3}
    assert not low, low
