"""The SFNO engine stage by stage (debug_set "stop_after" + debug_copy taps) against float64 references.

Shapes: the 49x96 baseline (E 64, L 3); the single-block path (E 192, L 1: one block that is first and last, BLOCK_N 192);
the full-size BLOCK_N dispatch and 384 statistics channels (E 384, L 2); 385x768 (lmax 128 = one tile, mmax 129 = one row
past it: the first shape where the mixing's triangular schedule skips tiles and the forward DFT has three row tiles) and
433x864 (lmax 144, mmax 145).

- stage-local: every stage from the engine's own input to it (oracle/sfno_stages_ref.py), per element, zero outside;
- chained: every tap against the fp64 oracle's (SFNORef.step(taps=...)), per-channel relative L2;
- end to end at 2e-4 per channel;
- members, run-to-run, eager / graph replay and NaN isolation, bit for bit;
- channels with |mean| / std of 10, 100 and 1000 at the block input (an offset in the encoder's fc2 bias).
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

SHAPES = [(49, 96, 64, 3), (49, 96, 192, 1), (49, 96, 384, 2), (385, 768, 64, 3), (433, 864, 64, 2)]
IDS = ["49x96-E64-L3", "49x96-E192-L1", "49x96-E384-L2", "385x768-E64-L3", "433x864-E64-L2"]
E2E_TOL = 2e-4


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _setup(shape, w=None, seed=0):
    from skyrim_b200.config import FCNV2_CHANNELS, sfno_small
    from skyrim_b200.engine import StepEngine
    from skyrim_b200.weights import make_sfno_weights, sfno_tables, synthetic_state
    nlat, nlon, E, L = shape
    cfg = sfno_small(nlat, nlon, embed=E, layers=L)
    w = make_sfno_weights(cfg, 0) if w is None else w
    tabs = sfno_tables(cfg)
    eng = StepEngine(cfg, 0)
    allw = dict(w); allw.update(tabs)
    eng.load_weights(allw)
    x0 = synthetic_state(FCNV2_CHANNELS, cfg.nlat, cfg.nlon, seed)
    return cfg, w, tabs, x0, eng


def _stage_names(sh, stage):
    """the taps live after stop_after = stage (0: encoder, 1 + i: block i, 99: the whole step)"""
    if stage == 0:
        return ["in_img", "hidden_img", "x_img", "sums0"] + (["x"] if sh.L == 1 else [])
    if stage == 99:
        return ["in_img", "x_img", "g_img"]
    i = stage - 1
    Hi, _, Ho, _ = sh.grids(i)
    names = ["norm0", "li", "si", "mi", "di", "g_img", "sums", "norm1", "fc1_bias", "hidden_img", "x_img"]
    names += ["f1", "inner_bias"] if Hi == Ho else ["mi2", "rpm"]
    names += ["x", "sums0"] if i + 1 < sh.L else []
    return names


def _read_taps(eng, sh, x, stage):
    eng.debug_set("stop_after", stage)
    try:
        y = eng.step(x)
        torch.cuda.synchronize()
        t = {n: eng.debug_tensor(n, (sh.tap_floats(n),)).cpu().numpy() for n in _stage_names(sh, stage)}
    finally:
        eng.debug_set("stop_after", 99)
    if stage == 99:
        t["state"] = y[0].cpu().numpy()
    return t


def _all_taps(eng, sh, x0):
    x = torch.from_numpy(x0)[None].cuda()
    return [_read_taps(eng, sh, x, s) for s in range(sh.L + 1)] + [_read_taps(eng, sh, x, 99)]


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_stages_against_stage_local_references(shape):
    """every stage from the engine's own input to it: zero elements outside the per-element bound, no NaN.  Largest
    ratios to the bound measured on an H100 80GB HBM3 at 700 W over the five shapes (hi + lo): inverse Legendre 1.00 (an
    element whose lo lands on an fp16 subnormal step), forward DFT 0.99, forward Legendre 0.69, inverse DFT + skip + GELU
    0.48, mixing 0.47, the pointwise GEMMs 0.21-0.36, statistics and norm affines below 0.05"""
    _need_gpu()
    from oracle import sfno_stages_ref as st
    cfg, w, tabs, x0, eng = _setup(shape)
    sh = st.Shapes(cfg)
    taps = _all_taps(eng, sh, x0)
    eng.close()
    checks, bad = st.stage_input(sh, x0, w, taps[0]["in_img"])
    assert bad == 0, f"{bad} input elements differ from the split of the fused fp32 normalisation"
    checks += st.stage_encoder(sh, w, taps[0]["in_img"], taps[0]["hidden_img"], taps[0]["x_img"], taps[0]["sums0"],
                               taps[0].get("x"))
    for i in range(sh.L):
        t = dict(taps[1 + i]); t["_tables"] = tabs
        checks += [(f"b{i} {n}", *rest) for n, *rest in st.stage_block_spectral(sh, w, i, t, taps[i])]
        checks += [(f"b{i} {n}", *rest) for n, *rest in st.stage_block_tail(sh, w, i, t, taps[i])]
    checks += st.stage_decoder(sh, w, taps[-1]["x_img"], taps[-1]["in_img"], taps[-1]["g_img"], taps[-1]["state"])
    res = st.evaluate(checks)
    for name, n, wr in res:
        print(f"{shape} {name:44s} worst |D-R|/bound {wr:.3f}  outside {n}")
    bad = [(name, n, wr) for name, n, wr in res if n]
    assert not bad, bad


def _chain_pairs(sh, taps, ref):
    """(name, engine [rows, channels], oracle [rows, channels]) of every tap; the per-channel vectors (norm affine, folded
    biases) as one column: their entries near zero have no relative error of their own"""
    from oracle import sfno_stages_ref as st
    E, Hd, P1 = sh.E, sh.Hd, sh.P1
    img = lambda raw, rows, cols: (lambda h, l: h + l)(*st.decode(raw, rows, cols, -(-cols // 64)))
    out = [("input", img(taps[0]["in_img"], P1, 128)[:, :sh.Cin], ref["in"]),
           ("enc hidden", img(taps[0]["hidden_img"], P1, E), ref["enc.hidden"]),
           ("enc x", img(taps[0]["x_img"], P1, E), ref["enc.x"])]
    for i in range(sh.L):
        t, k = taps[1 + i], f"b{i}."
        Hi, Wi, Ho, Wo = sh.grids(i)
        n2, mm, lm = 2 * E, sh.mmax, sh.lmax
        bat = lambda raw, nb, rows, cols: (lambda h, l: h + l)(*st.decode(raw, rows, cols, cols // 64, nb, st.img_bytes(rows, cols)))
        out += [(k + "norm0 scale", t["norm0"][:E, None], ref[k + "norm0"][:E, None]),
                (k + "norm0 shift", t["norm0"][E:, None], ref[k + "norm0"][E:, None]),
                (k + "li", bat(t["li"], mm, Hi, n2).reshape(-1, n2), ref[k + "li"].reshape(-1, n2)),
                (k + "si", bat(t["si"], lm, mm, n2).reshape(-1, n2), ref[k + "si"].reshape(-1, n2)),
                (k + "mi", bat(t["mi"], mm, lm, n2).reshape(-1, n2), ref[k + "mi"].reshape(-1, n2)),
                (k + "di", bat(t["di"], Ho, 2 * mm, E).reshape(-1, E), ref[k + "di"].reshape(-1, E)),
                (k + "g", img(t["g_img"], Ho * Wo, E), ref[k + "g"]),
                (k + "norm1 scale", t["norm1"][:E, None], ref[k + "norm1"][:E, None]),
                (k + "norm1 shift", t["norm1"][E:, None], ref[k + "norm1"][E:, None]),
                (k + "fc1 bias", t["fc1_bias"][:, None], ref[k + "fc1_bias"][:, None]),
                (k + "hidden", img(t["hidden_img"], Ho * Wo, Hd), ref[k + "hidden"]),
                (k + "x", img(t["x_img"], Ho * Wo, E), ref[k + "x"])]
        if Hi == Ho:
            out += [(k + "f1", t["f1"].reshape(-1, E)[:Ho * Wo], ref[k + "f1"]),
                    (k + "inner bias", t["inner_bias"][:, None], ref[k + "inner_bias"][:, None])]
        else:
            out += [(k + "mi2", bat(t["mi2"], mm, lm, n2).reshape(-1, n2), ref[k + "mi2"].reshape(-1, n2)),
                    (k + "rpm", t["rpm"].reshape(-1, E)[:Ho * Wo], ref[k + "rpm"])]
    out.append(("dec hidden", img(taps[-1]["g_img"], P1, E), ref["dec.hidden"]))
    return out


def _rel_per_channel(got, ref):
    got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
    num = np.sqrt(((got - ref) ** 2).sum(0)); den = np.sqrt((ref ** 2).sum(0))
    keep = den > 1e-6 * den.max()      # channels the stage leaves (numerically) empty: the m = mmax - 1 imaginary rows
    return float(np.max(num[keep] / den[keep])) if np.isfinite(num).all() else float("inf")


# Largest per-channel relative L2 error of any field tap against the fp64 oracle, measured on an H100 80GB HBM3 at 700 W:
# 49x96/E64/L3 1.0e-5 (block hidden), E192/L1 9.6e-6 (decoder hidden), E384/L2 1.3e-5 (decoder hidden), 385x768/E64/L3
# 2.1e-5 (decoder hidden), 433x864/E64/L2 2.3e-5 (decoder hidden); the end-to-end state 7.8e-6, 8.6e-6, 1.2e-5, 2.0e-5 and
# 2.0e-5.  One bound for every tap and shape, 3x or more above each of them.
CHAIN_TOL = 1e-4


@pytest.mark.parametrize("shape", SHAPES, ids=IDS)
def test_stages_chained_against_the_oracle(shape):
    """each tap against the fp64 oracle's, per channel; then the final state end to end (2e-4)"""
    _need_gpu()
    from oracle.pangu_ref import rel_err_per_channel
    from oracle.sfno_ref import SFNORef
    from oracle import sfno_stages_ref as st
    cfg, w, tabs, x0, eng = _setup(shape)
    sh = st.Shapes(cfg)
    taps = _all_taps(eng, sh, x0)
    y = eng.step(torch.from_numpy(x0)[None].cuda())[0].cpu().numpy()
    eng.close()
    ref = {}
    yref = SFNORef(cfg, w, torch.float64).step(x0, taps=ref).numpy()
    ref = {k: v.numpy() for k, v in ref.items()}
    tol = CHAIN_TOL
    worst = []
    for name, got, r in _chain_pairs(sh, taps, ref):
        e = _rel_per_channel(got, r)
        print(f"{shape} chained {name:16s} max per-channel rel L2 {e:.3e}")
        worst.append((e, name))
    e2e = rel_err_per_channel(y, yref)
    print(f"{shape} end to end: max per-channel rel err {e2e.max():.3e}")
    assert max(worst)[0] <= tol, max(worst)
    assert np.isfinite(y).all() and e2e.max() <= E2E_TOL, e2e.max()
    assert np.array_equal(y, taps[-1]["state"]), "reading taps changed what the next step computes"


def test_members_runs_graph_replay_and_nan_isolation():
    """B = 3 different ICs: each member bitwise equal to that member stepped alone; two runs bitwise equal; the eager
    first call and the graph replay bitwise equal; a NaN IC in the middle member leaves the other two bitwise unchanged"""
    _need_gpu()
    from skyrim_b200.config import FCNV2_CHANNELS
    from skyrim_b200.weights import synthetic_state
    cfg, w, tabs, x0, eng = _setup((49, 96, 64, 3))
    xs = np.stack([synthetic_state(FCNV2_CHANNELS, cfg.nlat, cfg.nlon, s) for s in (1, 2, 3)])
    xb = torch.from_numpy(xs).cuda()
    yb = [eng.step(xb).cpu().numpy() for _ in range(3)]            # eager, captured, replayed
    assert np.array_equal(yb[0], yb[1]) and np.array_equal(yb[0], yb[2])
    for m in range(3):
        ya = eng.step(xb[m:m + 1].contiguous()).cpu().numpy()[0]
        assert np.array_equal(ya, yb[0][m]), f"member {m} differs from itself stepped alone"
    xn = xs.copy(); xn[1, 5, 10, 20] = np.nan
    yn = eng.step(torch.from_numpy(xn).cuda()).cpu().numpy()
    assert not np.isfinite(yn[1]).all()
    assert np.array_equal(yn[0], yb[0][0]) and np.array_equal(yn[2], yb[0][2])
    eng.close()


@pytest.mark.parametrize("ratio,e2e_tol", [(10, E2E_TOL), (100, E2E_TOL), (1000, 5e-4)])
def test_norm_statistics_under_large_channel_offsets(ratio, e2e_tol):
    """k * sigma_c added to enc.fc2.b for four channels (|mean| / std about `ratio` at the first block's input): norm0's
    scale and shift within the stage bound of the two-pass fp64 norm, and the step within the end-to-end budget.

    Measured on an H100 80GB HBM3 at 700 W, end to end: 8.0e-6, 2.2e-5 and 2.0e-4 at ratios 10, 100 and 1000 (7.9e-6,
    1.9e-5 and 9.9e-4 when the statistics were unshifted sums of x and x^2); worst norm0 ratio to the bound 0.043.  At
    ratio 1000 what remains is the storage of the block input itself: fp32 x carries 2^-24 |x| ~ 6e-5 std and its hi / lo
    split 2^-22 |x| ~ 2.4e-4 std per element before any normalisation, which the fp64 oracle does not have; hence 5e-4
    there, which the unshifted statistics miss."""
    _need_gpu()
    import torch.nn.functional as F
    from oracle.pangu_ref import rel_err_per_channel
    from oracle.sfno_ref import SFNORef
    from oracle import sfno_stages_ref as st
    from skyrim_b200.config import FCNV2_CHANNELS, sfno_small
    from skyrim_b200.weights import make_sfno_weights, synthetic_state
    cfg = sfno_small(49, 96, embed=64, layers=3)
    w = make_sfno_weights(cfg, 0)
    r = SFNORef(cfg, w, torch.float64)
    enc = {}
    r.step(synthetic_state(FCNV2_CHANNELS, cfg.nlat, cfg.nlon, 0), taps=enc)
    sd = enc["enc.x"].numpy().std(0)
    w["enc.fc2.b"] = w["enc.fc2.b"].copy()
    chans = [3, 17, 40, 63]
    for j, c in enumerate(chans):
        w["enc.fc2.b"][c] += np.float32((-1) ** j * ratio * sd[c])
    cfg, w, tabs, x0, eng = _setup((49, 96, 64, 3), w=w)
    sh = st.Shapes(cfg)
    x = torch.from_numpy(x0)[None].cuda()
    t0, t1 = _read_taps(eng, sh, x, 0), _read_taps(eng, sh, x, 1)
    y = eng.step(x)[0].cpu().numpy()
    eng.close()
    x_hi, x_lo = st.decode(t0["x_img"], sh.P1, sh.E, sh.E // 64)
    xm = x_hi + x_lo
    print(f"ratio {ratio}: |mean|/std at the block input {np.abs(xm.mean(0) / xm.std(0))[chans]}")
    res = st.evaluate(st.stage_norm("norm0", sh, x_hi, x_lo, w["blk0.norm0.g"], w["blk0.norm0.b"], t1["norm0"]))
    for name, n, wr in res:
        print(f"ratio {ratio}: {name} worst |D-R|/bound {wr:.3f} outside {n}")
    assert not [x for x in res if x[1]], res
    e = rel_err_per_channel(y, SFNORef(cfg, w, torch.float64).step(x0).numpy())
    print(f"ratio {ratio}: end to end max per-channel rel err {e.max():.3e}")
    assert e.max() <= e2e_tol, e.max()
