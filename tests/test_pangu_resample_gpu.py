"""Pangu's down-sample, up-sample and patch recovery element by element against float64 (oracle/pangu_resample_ref.py).

Each case runs the engine's own step to a tap (debug_set("stop_after", n)) and reads the workspace regions the units
read and write (their offsets: pr.workspace_layout, the mirror of PanguEngine::carve).  Every reference starts from the
exact bytes the kernel read in that run and the fp16 packed weights, so each unit is checked on its own:
  stop_after 2   k_down_merge_ln's image (hidh) from the skip image (fp16 stream) or the fp32 rows x1 (fp32 stream);
                 the down GEMM's x2h (and x2 with the fp32 stream) from those hidh bytes
  stop_after 5   Epi2UpShuffle's image (hidh) from x2h; linear2's x1h (and x1) from those hidh bytes
  whole step     Epi2Recover at BLOCK_N 224 from skiph and x1h: every element of the output, filled with NaN before
Grids 41 x 96, 33 x 96 (odd H: the merge's zero padding row and the up-sample's crop row), 45 x 192, 24 x 96 (even H),
with one and three members and both token streams: the last row tile is partial at both grid levels at 41 x 96 and
33 x 96, at level 2 only at 24 x 96, and whole at 45 x 192.  And the full 721 x 1440 grid with one member (partial
tiles), there on every token of the first and last latitude row of each level and a seeded random sample (every output
element of the recovery is still checked for being written).  The workspace starts as 0xFF bytes (an fp16 NaN): image rows past the last token keep them, and so does
the fp32 level-2 stream with the fp16 token stream.  Under -s each case prints its largest |error| / bound per unit."""
import numpy as np
import pytest

from oracle import gemm_ref as gr
from oracle import pangu_resample_ref as pr

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

GRIDS = [(41, 96), (33, 96), (45, 192), (24, 96)]
FULL = (721, 1440)
CASES = [(g, B) for g in GRIDS for B in (1, 3)] + [(FULL, 1)]
SAMPLE_SEED, SAMPLE_ROWS = 11, 4096


@pytest.fixture(scope="module")
def engines():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from skyrim_b200.config import pangu_small
    from skyrim_b200.engine import StepEngine
    from skyrim_b200.weights import make_pangu_weights
    made = {}

    def get(grid):
        if grid not in made:
            cfg = pangu_small(*grid)
            w = make_pangu_weights(cfg, 1)
            eng = StepEngine(cfg, 0)
            eng.load_weights(w)
            made[grid] = (cfg, w, pr.gemm_weights(cfg, w), eng)
        return made[grid]
    yield get
    for *_, eng in made.values():
        eng.close()


def _case_id(v):
    return f"{v[0]}x{v[1]}" if isinstance(v, tuple) else f"B{v}"


def _step(cfg, eng, B, stream, stop, x_out=None):
    """one step to tap `stop` from states of seeds 3 + m on a 0xFF workspace; returns the workspace and its layout"""
    from skyrim_b200.config import PANGU_CHANNELS
    from skyrim_b200.weights import synthetic_state
    x = np.stack([synthetic_state(PANGU_CHANNELS, cfg.nlat, cfg.nlon, 3 + m) for m in range(B)])
    eng.debug_set("fp32_stream", int(stream == "fp32"))
    eng.debug_set("stop_after", stop)
    try:
        ws = eng._workspace(B)
        ws.fill_(0xFF)
        eng.step(torch.from_numpy(x).cuda(), x_out)
        torch.cuda.synchronize()
    finally:
        eng.debug_set("stop_after", 99)
    lay = pr.workspace_layout(cfg, B)
    assert eng._L.sky_model_workspace_bytes(eng._h, B) == lay["total"]
    return ws, lay


def _image(ws, lay, name, rows, cols):
    """fp16 tile image at region `name` -> (float64 [rows, cols], the raw bytes [tiles, cols / 64, 128, 128])"""
    tiles, nkb = -(-rows // 128), cols // 64
    raw = ws[lay[name]: lay[name] + tiles * nkb * pr.G2_A_BYTES].cpu().numpy()
    return gr.unpack_tiles(raw, 128, nkb, rows, cols).astype(np.float64), raw.reshape(tiles, nkb, 128, 128)


def _f32_rows(ws, lay, name, rows, cols):
    return ws[lay[name]: lay[name] + rows * cols * 4].cpu().numpy().view(np.float32).reshape(rows, cols)


def _sample(B, Z, H, W):
    """every token of the first and last latitude row of each (member, level) slab, and a seeded random sample"""
    q = np.arange(B * Z)[:, None, None]
    edge = ((q * H + np.array([0, H - 1])[None, :, None]) * W + np.arange(W)[None, None, :]).reshape(-1)
    rnd = np.random.default_rng(SAMPLE_SEED).choice(B * Z * H * W, SAMPLE_ROWS, replace=False)
    return np.unique(np.concatenate([edge, rnd]))


def _rows(cfg, B, level):
    Z, H, W = (cfg.Z, cfg.H, cfg.W) if level == 1 else (cfg.Z, cfg.H2, cfg.W2)
    return _sample(B, Z, H, W) if (cfg.nlat, cfg.nlon) == FULL else np.arange(B * Z * H * W)


def _check(tag, name, got, ref, bound, rows, dims, worst):
    """every element within its bound; on failure the first offending (member, z, h, w, feature)"""
    r = gr.worst(got, ref, bound)
    worst[name] = max(worst.get(name, 0.0), r)
    print(f"{tag} {name}: largest |error| / bound {r:.3f}")
    bad = gr.exceed(got, ref, bound)
    if bad.any():
        i, f = np.argwhere(bad)[0]
        Z, H, W = dims
        t = int(rows[i])
        m, z, h, w = t // (Z * H * W), t // (H * W) % Z, t // W % H, t % W
        pytest.fail(f"{tag} {name}: {int(bad.sum())} elements out of bound, first at member {m}, z {z}, h {h}, w {w}, "
                    f"feature {f}: got {got[i, f]!r}, reference {ref[i, f]!r}, bound {bound[i, f]:.3g}")


WORST = {}


@pytest.mark.parametrize("stream", ["fp16", "fp32"])
@pytest.mark.parametrize("grid,B", CASES, ids=_case_id)
def test_down_sample(engines, grid, B, stream):
    cfg, w, gw, eng = engines(grid)
    C = cfg.dim
    R1, R2 = B * cfg.Z * cfg.H * cfg.W, B * cfg.Z * cfg.H2 * cfg.W2
    ws, lay = _step(cfg, eng, B, stream, 2)
    if stream == "fp16":
        xin, _ = _image(ws, lay, "skiph", R1, C)
    else:
        xin = _f32_rows(ws, lay, "x1", R1, C).astype(np.float64)
    hid, _ = _image(ws, lay, "hidh", R2, 4 * C)
    x2h, x2h_raw = _image(ws, lay, "x2h", R2, 2 * C)
    x2 = _f32_rows(ws, lay, "x2", R2, 2 * C)
    tag, dims = f"{cfg.nlat}x{cfg.nlon} B={B} {stream} stream, down-sample", (cfg.Z, cfg.H2, cfg.W2)
    rows = _rows(cfg, B, 2)
    ref, bnd = pr.down_merge_ln(cfg, w, xin, B, rows)
    _check(tag, "merge + LayerNorm (hidh)", hid[rows], ref, bnd, rows, dims, WORST)
    ref, bnd = pr.linear_plain(hid[rows], gw["down"])
    _check(tag, "down GEMM (x2h)", x2h[rows], ref, gr.f16_bound(ref, bnd), rows, dims, WORST)
    if stream == "fp32":
        _check(tag, "down GEMM (x2 rows)", x2[rows], ref, bnd, rows, dims, WORST)
    else:
        assert (x2.view(np.uint8) == 0xFF).all(), "fp32 level-2 rows written in the image-only stream mode"
    assert (x2h_raw[-1, :, R2 - (x2h_raw.shape[0] - 1) * 128:] == 0xFF).all(), "x2h rows past the last token written"


@pytest.mark.parametrize("stream", ["fp16", "fp32"])
@pytest.mark.parametrize("grid,B", CASES, ids=_case_id)
def test_up_sample(engines, grid, B, stream):
    cfg, w, gw, eng = engines(grid)
    C = cfg.dim
    R1, R2 = B * cfg.Z * cfg.H * cfg.W, B * cfg.Z * cfg.H2 * cfg.W2
    ws, lay = _step(cfg, eng, B, stream, 5)
    x2h, _ = _image(ws, lay, "x2h", R2, 2 * C)
    hid, _ = _image(ws, lay, "hidh", R1, C)
    x1h, x1h_raw = _image(ws, lay, "x1h", R1, C)
    tag, dims = f"{cfg.nlat}x{cfg.nlon} B={B} {stream} stream, up-sample", (cfg.Z, cfg.H, cfg.W)
    rows = _rows(cfg, B, 1)
    ref, bnd = pr.up_shuffle(cfg, w, x2h, gw["up1"], B, rows)
    _check(tag, "linear1 + shuffle + LayerNorm (hidh)", hid[rows], ref, bnd, rows, dims, WORST)
    ref, bnd = pr.linear_plain(hid[rows], gw["up2"])
    _check(tag, "linear2 (x1h)", x1h[rows], ref, gr.f16_bound(ref, bnd), rows, dims, WORST)
    if stream == "fp32":
        x1 = _f32_rows(ws, lay, "x1", R1, C)
        _check(tag, "linear2 (x1 rows)", x1[rows], ref, bnd, rows, dims, WORST)
    assert (x1h_raw[-1, :, R1 - (x1h_raw.shape[0] - 1) * 128:] == 0xFF).all(), "x1h rows past the last token written"


def _token_of(cfg, flat):
    """output element (member, channel, lat, lon) -> the token (member, z, h, w) that writes it and its weight column"""
    nl, nup = cfg.n_levels, cfg.n_upper_vars * cfg.n_levels
    m, rest = divmod(int(flat), cfg.n_channels * cfg.nlat * cfg.nlon)
    ch, rest = divmod(rest, cfg.nlat * cfg.nlon)
    lat, lon = divmod(rest, cfg.nlon)
    dh, dw = lat % 4, lon % 4
    if ch < nup:
        v, lev = divmod(ch, nl)
        z, col = 1 + lev // 2, ((v * 2 + lev % 2) * 4 + dh) * 4 + dw
    else:
        z, col = 0, pr.REC_UPPER + ((ch - nup) * 4 + dh) * 4 + dw
    return m, z, lat // 4, lon // 4, col, (m, ch, lat, lon)


@pytest.mark.parametrize("stream", ["fp16", "fp32"])
@pytest.mark.parametrize("grid,B", CASES, ids=_case_id)
def test_patch_recovery(engines, grid, B, stream):
    cfg, w, gw, eng = engines(grid)
    C = cfg.dim
    R1 = B * cfg.Z * cfg.H * cfg.W
    x_out = torch.full((B, cfg.n_channels, cfg.nlat, cfg.nlon), float("nan"), device="cuda")
    ws, lay = _step(cfg, eng, B, stream, 99, x_out)
    skip, _ = _image(ws, lay, "skiph", R1, C)
    x1h, _ = _image(ws, lay, "x1h", R1, C)
    out = x_out.cpu().numpy().reshape(-1)
    tag = f"{cfg.nlat}x{cfg.nlon} B={B} {stream} stream, patch recovery"
    nan = np.flatnonzero(np.isnan(out))
    assert nan.size == 0, f"{tag}: {nan.size} output elements not written, first {_token_of(cfg, nan[0])}"
    rows = _rows(cfg, B, 1)
    flat, ref, bnd = pr.recover(cfg, w, np.concatenate([skip[rows], x1h[rows]], 1), gw["rec"], B, rows)
    if (cfg.nlat, cfg.nlon) != FULL:
        assert flat.size == out.size
    got = out[flat]
    r = gr.worst(got, ref, bnd)
    WORST["recovery (x_out)"] = max(WORST.get("recovery (x_out)", 0.0), r)
    print(f"{tag} (BLOCK_N 224): largest |error| / bound {r:.3f}")
    bad = gr.exceed(got, ref, bnd)
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        m, z, h, w_, col, el = _token_of(cfg, flat[i])
        pytest.fail(f"{tag}: {int(bad.sum())} elements out of bound, first at member {m}, z {z}, h {h}, w {w_}, feature {col} "
                    f"(output {el}): got {got[i]!r}, reference {ref[i]!r}, bound {bnd[i]:.3g}")


def test_summary():
    """the largest |error| / bound per unit over the cases that ran in this session (print only)"""
    for name, r in sorted(WORST.items()):
        print(f"[pangu resample] worst {name}: {r:.3f}")
