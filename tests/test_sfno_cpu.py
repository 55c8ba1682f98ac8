"""CPU tests of the SFNO restatement: SHT tables, truncated-DFT matrices, oracle precision."""
import numpy as np
import pytest
import torch

from oracle.pangu_ref import rel_err_per_channel
from oracle.sfno_ref import SFNORef
from skyrim_b200.config import FCNV2_CHANNELS, sfno_full, sfno_small
from skyrim_b200.sht import RealSHT, clenshaw_curtis, dft_matrices, legendre_gauss, legpoly
from skyrim_b200.weights import make_sfno_weights, sfno_param_shapes, sfno_tables, synthetic_state


def test_quadrature_rules():
    for n in (13, 32):
        x, w = clenshaw_curtis(n)
        assert abs(w.sum() - 2.0) < 1e-13 and abs((w * x ** 2).sum() - 2.0 / 3.0) < 1e-12
        x, w = legendre_gauss(n)
        assert abs(w.sum() - 2.0) < 1e-13 and abs((w * x ** 4).sum() - 2.0 / 5.0) < 1e-12


def test_legendre_orthonormality():
    x, w = legendre_gauss(40)
    p = legpoly(17, 16, x)
    for m in (0, 3, 9):
        g = 2 * np.pi * np.einsum("lk,jk,k->lj", p[m], p[m], w)
        ll = np.arange(16)
        mask = (ll[:, None] >= m) & (ll[None, :] >= m)
        assert np.abs(g - np.eye(16))[mask].max() < 1e-12


@pytest.mark.parametrize("nlat,nlon,grid", [(49, 96, "equiangular"), (16, 32, "legendre-gauss")])
def test_sht_roundtrip_and_dft_matrices(nlat, nlon, grid):
    lmax, mmax = 16, 17
    s = RealSHT(nlat, nlon, lmax, mmax, grid)
    rng = np.random.default_rng(0)
    X = rng.standard_normal((lmax, mmax)) + 1j * rng.standard_normal((lmax, mmax))
    X[:, 0] = X[:, 0].real
    for m in range(mmax):
        X[:m, m] = 0
    if mmax - 1 == nlon // 2:
        X[:, -1] = 0
    x = s.inverse(X)
    assert np.abs(s.forward(x) - X).max() < 1e-12
    f, i = dft_matrices(nlon, mmax)
    F = x @ f.T
    ref = 2 * np.pi * np.fft.rfft(x, axis=-1, norm="forward")[:, :mmax]
    assert np.abs((F[:, 0::2] + 1j * F[:, 1::2]) - ref).max() < 1e-12
    assert np.abs(F @ i.T - np.fft.irfft(ref, n=nlon, axis=-1, norm="forward")).max() < 1e-11


def test_full_config_shapes():
    c = sfno_full()
    assert (c.h, c.w, c.lmax, c.mmax) == (240, 480, 240, 241)
    sh = sfno_param_shapes(c)
    assert sh["blk0.spec.w"] == (240, 384, 384, 2) and sh["dec.fc1.w"] == (384, 457)
    assert len(FCNV2_CHANNELS) == 73


def test_oracle_precision_and_stability():
    cfg = sfno_small(49, 96, embed=64, layers=3)
    w = make_sfno_weights(cfg, 0)
    x0 = synthetic_state(FCNV2_CHANNELS, cfg.nlat, cfg.nlon, 0)
    y64 = SFNORef(cfg, w, torch.float64).step(x0).numpy()
    y32 = SFNORef(cfg, w, torch.float32).step(x0).numpy()
    assert rel_err_per_channel(y32, y64).max() < 1e-5
    t = sfno_tables(cfg)
    assert t["sht.fwd_big"].shape == (cfg.mmax, cfg.lmax, cfg.nlat) and t["dft.inv_int"].shape == (cfg.w, 2 * cfg.mmax)
    # autoregressive use neither explodes nor collapses
    r = SFNORef(cfg, w)
    x = torch.from_numpy(x0)
    mu, sd = r.w["norm.mean"][:, None, None], r.w["norm.std"][:, None, None]
    for _ in range(4):
        x = r.step(x)
    s = float(((x - mu) / sd).std())
    assert 0.1 < s < 3.0, s


def test_three_term_fp16_split_is_fp32_grade():
    """hi + lo fp16 split used for the SFNO GEMM operands: a*b ~= ah*bh + al*bh + ah*bl."""
    rng = np.random.default_rng(1)
    a = rng.standard_normal((64, 256)).astype(np.float32)
    b = (rng.standard_normal((256, 48)) * 0.05).astype(np.float32)
    ah, bh = a.astype(np.float16), b.astype(np.float16)
    al = (a - ah.astype(np.float32)).astype(np.float16)
    bl = (b - bh.astype(np.float32)).astype(np.float16)
    f = lambda u, v: u.astype(np.float32) @ v.astype(np.float32)
    exact = a.astype(np.float64) @ b.astype(np.float64)
    one = np.abs(f(ah, bh) - exact).max() / np.abs(exact).max()
    three = np.abs(f(ah, bh) + f(al, bh) + f(ah, bl) - exact).max() / np.abs(exact).max()
    assert one > 1e-4 and three < 3e-6, (one, three)


def test_oracle_matches_golden():
    """The fp32 oracle against the committed fp64 fixture (tools/make_golden.py): pins the restatement across
    refactors; the reference itself ships no golden vector for this path (DESIGN.md section 2)."""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "sfno_49x96_seed0.npz"))
    cfg = sfno_small(49, 96, embed=64, layers=3)
    w = make_sfno_weights(cfg, 0)
    x0 = synthetic_state(FCNV2_CHANNELS, cfg.nlat, cfg.nlon, 0)
    np.testing.assert_array_equal(x0[:, ::8, ::16], g["x0_sample"])
    y = SFNORef(cfg, w, torch.float32).step(x0).numpy()
    scale = np.abs(g["y_sample"]).max(axis=(1, 2), keepdims=True)
    assert np.max(np.abs(y[:, ::6, ::12] - g["y_sample"]) / scale) < 1e-4
    np.testing.assert_allclose(np.sqrt((y.astype(np.float64) ** 2).sum(axis=(1, 2))), g["y_norm"], rtol=1e-5)


@pytest.mark.parametrize("nlat,grid", [(49, "equiangular"), (97, "equiangular"), (32, "legendre-gauss"), (80, "legendre-gauss")])
def test_product_tables_agree_with_independent_oracle_tables(nlat, grid):
    """skyrim_b200/sht.py (recurrence + cosine-sum Clenshaw-Curtis / numpy leggauss: what the engine's weight arena
    carries) against oracle/sht_ref.py (scipy.special.sph_legendre_p, Waldvogel FFT weights, roots_legendre):
    two algorithms, one convention — orthonormal Pbar with Condon-Shortley phase, north pole first."""
    from oracle import sht_ref
    from skyrim_b200.sht import sht_tables, grid_nodes
    lmax, mmax = 33, 34
    f1, i1, cost1, w1 = sht_ref.tables(nlat, lmax, mmax, grid)
    f2, i2 = sht_tables(nlat, lmax, mmax, grid)
    cost2, w2 = grid_nodes(nlat, grid)
    assert np.abs(cost1 - cost2).max() < 1e-14 and np.abs(w1 - w2).max() < 1e-14
    assert np.abs(f1 - f2).max() < 1e-12 and np.abs(i1 - i2).max() < 1e-12
    # Condon-Shortley: Pbar_1^1(cos theta) = -sqrt(3/(8 pi)) sin(theta)
    th = np.arccos(cost1)
    assert np.abs(i1[1, :, 1] + np.sqrt(3.0 / (8.0 * np.pi)) * np.sin(th)).max() < 1e-14


def test_full_size_fixtures_match_the_seeded_inputs():
    """tests/golden/*_721x1440_seed0.npz (one real oracle step each, tools/make_golden_full.py): the committed IC
    sample must equal what skyrim_b200.weights regenerates, or the GPU-side comparison would be meaningless."""
    from skyrim_b200.config import PANGU_CHANNELS
    from skyrim_b200.verify import BLOCK_PX, SAMPLE_STEP, load_fixture
    for model, names in (("pangu", PANGU_CHANNELS), ("sfno", FCNV2_CHANNELS)):
        fx = load_fixture(model)
        x0 = synthetic_state(names, 721, 1440, 0)
        np.testing.assert_array_equal(x0[:, ::64, ::64], fx["x0_sample"])
        assert fx["y_sample"].shape == (len(names), -(-721 // SAMPLE_STEP[0]), -(-1440 // SAMPLE_STEP[1]))
        assert fx["y_block"].shape == (len(names), 720 // BLOCK_PX, 1440 // BLOCK_PX) and np.isfinite(fx["y_block"]).all()
        assert (fx["y_std"] > 0).all() and float(fx["oracle_seconds"]) > 1.0


def test_engine_rewrites_are_identities_of_the_oracle():
    """The CUDA engine restructures the block algebraically (skyrim_b200/csrc/sfno_engine.cu); each rewrite is checked here
    on the fp64 oracle, so that the GPU parity tests measure rounding only:
      1. grid-changing blocks: iSHT(W_l X) + V iSHT(X) + b = iSHT((W_l + V) X) + b  (inner skip folded into the mixing);
      2. an instance norm in front of a 1x1 convolution folds into its weights:  W (sc*g + sh) + b = (W diag(sc)) g + (W sh + b);
      3. the norm's affine commutes with the (linear, per-channel) forward transform:  SHT(sc*x + sh) = sc*SHT(x) + sh*SHT(1)."""
    cfg = sfno_small(49, 96, embed=16, layers=3)
    w = make_sfno_weights(cfg, 5)
    x0 = synthetic_state(FCNV2_CHANNELS, cfg.nlat, cfg.nlon, 5)
    ref = SFNORef(cfg, w, dtype=torch.float64)
    y = ref.step(x0).numpy()
    # 1. fold the inner skip of the first and last block into their mixing matrices, zero the pixel-space weights
    wf = {k: np.array(v, dtype=np.float64) for k, v in w.items()}
    for i in (0, cfg.layers - 1):
        wf[f"blk{i}.spec.w"][..., 0] += wf[f"blk{i}.inner.w"][None]
        wf[f"blk{i}.inner.w"][:] = 0.0
    yf = SFNORef(cfg, wf, dtype=torch.float64).step(x0).numpy()
    assert rel_err_per_channel(yf, y).max() < 1e-10
    # 2. / 3. on one block's tensors
    g = torch.randn(cfg.embed, cfg.h, cfg.w, dtype=torch.float64)
    sc, sh = torch.rand(cfg.embed, dtype=torch.float64) + 0.5, torch.randn(cfg.embed, dtype=torch.float64)
    W1, b1 = ref.w["blk1.fc1.w"], ref.w["blk1.fc1.b"]
    lhs = ref._conv1x1(g * sc[:, None, None] + sh[:, None, None], W1, b1)
    rhs = ref._conv1x1(g, W1 * sc[None, :], W1 @ sh + b1)
    assert torch.allclose(lhs, rhs, rtol=1e-12, atol=1e-12)
    X1 = ref.sht(torch.ones(1, cfg.h, cfg.w, dtype=torch.float64), "int")[0]
    lhs = ref.sht(g * sc[:, None, None] + sh[:, None, None], "int")
    rhs = ref.sht(g, "int") * sc[:, None, None] + sh[:, None, None] * X1[None]
    assert torch.allclose(lhs, rhs, rtol=1e-11, atol=1e-11)
    # ... and SHT(1) lives in the (l = 0, m = 0) coefficient alone: the engine adds sh * (row sum of the DFT table) to the
    # m = 0 real row before the Legendre transform
    mask = torch.ones_like(X1.real, dtype=torch.bool); mask[0, 0] = False
    assert X1[mask].abs().max() < 1e-12 * X1[0, 0].abs()
