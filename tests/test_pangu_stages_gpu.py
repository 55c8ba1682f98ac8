"""Pangu's transformer blocks unit by unit inside the engine (debug_set "stop_launch" + raw debug_copy taps) against the
float64 references of oracle/pangu_stages_ref.py.

Grids pangu_small(41, 96) (latitude padding 1 at level 1; a single window row at level 2), (33, 96) (padding 3 and 1)
and (45, 192) (no padding), with one and three members (partial last 128-row tiles) and both token streams: the image-only
fp16 stream (fused MLP at C = 192) and the fp32 rows beside it (debug_set "fp32_stream" 1: fc1 + fc2 at C = 192).

- stage-local: every unit of every block from the engine's own inputs to it (QKV: the stream image; attention: the window
  image; projection and fc2: the attention output or hidden image and the residual of the stream mode; fc1 and the fused
  MLP: the stream image), per element, no NaN; the workspace starts as the fp16 sentinel 0x7D5A before every stopped step,
  and the rows past B T of every stream image, and in layer 0 of the attention and hidden images and the window image
  region past its three parts, still hold it.  The fused MLP leaves the hidden image untouched;
- chained: the stream after every block against PanguRef in float64, per row, within graphcast_stages_ref's rule on the
  oracle's own fp16 emulation of that block;
- a workspace of 0x00 bytes and one of 0xFF bytes give the same bits in every tap's valid region and the same state;
- a step stopped after its last unit is the whole step; eager and graph-replayed steps agree; launches per step;
- the full 721 x 1440 grid, one member, fp16 stream: the first two blocks of layers 0 and 1 on every window of the first
  and last window rows and a seeded sample of windows.
pytest -s prints the largest err / bound of every check; test_summary the largest per unit kind (DESIGN.md)."""
import numpy as np
import pytest

from oracle import gemm_ref as gr
from oracle import pangu_kernels_ref as pk
from oracle import pangu_resample_ref as pr
from oracle import pangu_stages_ref as ps

torch = pytest.importorskip("torch")

from test_pangu_kernels_gpu import SENT, image_rows, sample_windows  # noqa: E402

pytestmark = pytest.mark.gpu

GRIDS = [(41, 96), (33, 96), (45, 192)]
FULL = (721, 1440)
CASES = [(g, B, s) for g in GRIDS for B in (1, 3) for s in ("fp16", "fp32")]
WORST = {}


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
            made[grid] = (cfg, w, eng)
        return made[grid]
    yield get
    for *_, eng in made.values():
        eng.close()


def _case_id(v):
    return f"{v[0]}x{v[1]}" if isinstance(v, tuple) else f"B{v}" if isinstance(v, int) else v


def _states(cfg, B):
    from skyrim_b200.config import PANGU_CHANNELS
    from skyrim_b200.weights import synthetic_state
    return np.stack([synthetic_state(PANGU_CHANNELS, cfg.nlat, cfg.nlon, 3 + m) for m in range(B)])


def _fill(ws, fill):
    if fill == "sentinel":
        ws.view(torch.int16).fill_(SENT)
    else:
        ws.fill_(fill)


def _img_bytes(g, B, nkb):
    return -(-B * g.T // 128) * nkb * pr.G2_A_BYTES


def _tap(eng, name, B, nbytes):
    """raw tap, int16 on the device"""
    return eng.debug_tensor(name, (nbytes // 4,), B).view(torch.int16)


def block_taps(eng, cfg, B, stream, li, bi, xs, fill="sentinel", sentinels=None):
    """{unit kind: {tap: device tensor}} of block (li, bi), each unit read after a step of its own that stops right behind
    it on a workspace filled with `fill`.  sentinels: list collecting (what, ok) of the regions that must keep the
    sentinel"""
    g = ps.level(cfg, li)
    nkb, R = g.C // 64, B * g.T
    at = ps.unit_index(cfg, stream)
    ws = eng._workspace(B)
    lay = pr.workspace_layout(cfg, B)
    img = _img_bytes(g, B, nkb)
    taps = {}
    for kind in ("qkv", "attn", "proj") + ps.mlp_kinds(g.C, stream):
        _fill(ws, fill)
        eng.debug_set("stop_launch", at[(kind, li, bi)])
        eng.step(xs)
        t = {}
        if kind == "qkv":
            t["qkv"] = _tap(eng, "qkv", B, 3 * B * g.nWin * g.pairs * pk.TILE_B)
        if kind == "attn":
            t["att_h"] = _tap(eng, "att_h", B, img)
        if kind == "fc1":
            t["hid_h"] = _tap(eng, "hid_h", B, 4 * img)
        if kind in ("qkv", "proj", "fc2", "mlp"):
            t["stream_h"] = _tap(eng, "stream_h", B, img)
            if stream == "fp32":
                t["rows"] = eng.debug_tensor("tokens1" if g.C == cfg.dim else "tokens2", (R, g.C), B)
            elif sentinels is not None and R <= 1 << 16 and kind != "qkv":
                # the expanded stream tap follows the stream: the skip image in layer 0, x1h in layer 3
                exp = eng.debug_tensor("tokens1" if g.C == cfg.dim else "tokens2", (R, g.C), B).cpu().numpy()
                sentinels.append((f"debug_copy tokens after {kind} = the stream image",
                                  np.array_equal(exp, image_rows(t["stream_h"], np.arange(R), nkb).astype(np.float32))))
        if sentinels is not None and fill == "sentinel":
            for name, v in t.items():
                if name == "rows" or R % 128 == 0 or name == "qkv":
                    continue
                n = v.numel() // (-(-R // 128) * 128 * 64)          # k-blocks of the image
                tail = v.view(-1, n, 128, 64)[-1, :, R % 128:]
                if name == "stream_h" or li == 0:
                    sentinels.append((f"{name} rows past B T after {kind}", bool((tail == SENT).all())))
            if li == 0 and kind == "qkv":
                gap = ws[lay["qkv"] + 3 * B * g.nWin * g.pairs * pk.TILE_B: lay["atth"]].view(torch.int16)
                sentinels.append(("window image past its three parts", bool((gap == SENT).all())))
            if li == 0 and kind == "mlp":
                hid = ws[lay["hidh"]: lay["total"]].view(torch.int16)
                sentinels.append(("hidden image untouched by the fused MLP", bool((hid == SENT).all())))
        taps[kind] = t
    return taps


def _check(tag, name, got, ref, bound, worst_key):
    r = gr.worst(got, ref, bound)
    WORST[worst_key] = max(WORST.get(worst_key, 0.0), r)
    print(f"{tag} {name}: largest |error| / bound {r:.3f}")
    bad = gr.exceed(got, ref, bound)
    return [] if not bad.any() else [f"{tag} {name}: {int(bad.sum())} elements out of bound (worst ratio {r:.3g})"]


def check_block(cfg, w, B, stream, li, bi, taps, wins, tag):
    """stage-local checks of block (li, bi) on windows wins (member * nWin + window) and the tokens they hold; returns the
    failures"""
    g = ps.level(cfg, li)
    nkb, R, roll = g.C // 64, B * g.T, bi & 1
    bw = ps.block_weights(w, li, bi)
    eps = cfg.ln_eps
    tag = f"{tag} layer {li} block {bi}"
    fails = []
    # QKV from the stream image it read
    idx = ps.window_rows(g, B, roll, wins)
    toks = np.unique(idx[idx >= 0])
    x = np.zeros((R, g.C), np.float16)
    x[toks] = image_rows(taps["qkv"]["stream_h"], toks, nkb)
    ref, bnd = ps.qkv_unit(g, B, roll, wins, x, bw)
    tiles = torch.from_numpy(np.array([wi * g.pairs + p for wi in wins for p in range(g.pairs)])).cuda()
    sel = taps["qkv"]["qkv"].view(3, -1, pk.NTOK * 64)[:, tiles].cpu().numpy()
    qkv = pk.unpack_tiles(sel.reshape(3, len(wins), g.pairs, pk.NTOK * 64)).reshape(3, len(wins), g.heads, pk.NTOK, 32)
    fails += _check(tag, "QKV window image", qkv, ref, bnd, "QKV (window image)")
    # attention from the window image as the kernel read it
    tok, ref, bnd = ps.attention_unit(g, B, roll, wins, qkv, bw, cfg.mask_value)
    order = np.argsort(tok)
    tok, ref, bnd = tok[order], ref[order], bnd[order]
    att = image_rows(taps["attn"]["att_h"], tok, nkb).astype(np.float64)
    fails += _check(tag, "attention output image", att, ref, bnd, "attention (output image)")
    # projection + ln1 + residual
    rows32 = (lambda k: taps[k]["rows"][torch.from_numpy(tok).cuda()].double().cpu().numpy()) if stream == "fp32" else None
    res = rows32("qkv") if stream == "fp32" else x[tok].astype(np.float64)
    y, yb = ps.proj_unit(att, bw, res, eps, stream)
    x1 = image_rows(taps["proj"]["stream_h"], tok, nkb).astype(np.float64)
    fails += _check(tag, "projection + LayerNorm (image)", x1, y, gr.f16_bound(y, yb), "projection + LayerNorm")
    if stream == "fp32":
        fails += _check(tag, "projection + LayerNorm (fp32 rows)", rows32("proj"), y, yb, "projection + LayerNorm")
    res = rows32("proj") if stream == "fp32" else x1
    # MLP
    if "mlp" in taps:
        y, yb = ps.mlp_unit(x1, bw, res, eps, stream)
        out = image_rows(taps["mlp"]["stream_h"], tok, nkb).astype(np.float64)
        fails += _check(tag, "fused MLP + LayerNorm (image)", out, y, gr.f16_bound(y, yb), "fused MLP + LayerNorm")
    else:
        h, hb = ps.fc1_unit(x1, bw)
        hid = image_rows(taps["fc1"]["hid_h"], tok, 4 * nkb).astype(np.float64)
        fails += _check(tag, "fc1 + GELU (hidden image)", hid, h, hb, "fc1 + GELU")
        y, yb = ps.fc2_unit(hid, bw, res, eps, stream)
        out = image_rows(taps["fc2"]["stream_h"], tok, nkb).astype(np.float64)
        fails += _check(tag, "fc2 + LayerNorm (image)", out, y, gr.f16_bound(y, yb), "fc2 + LayerNorm")
        if stream == "fp32":
            fails += _check(tag, "fc2 + LayerNorm (fp32 rows)", rows32("fc2"), y, yb, "fc2 + LayerNorm")
    return fails


def _stream_rows(taps, stream, g, B):
    last = taps["mlp" if "mlp" in taps else "fc2"]
    if stream == "fp32":
        return last["rows"].double().cpu().numpy()
    return image_rows(last["stream_h"], np.arange(B * g.T), g.C // 64).astype(np.float64)


@pytest.mark.parametrize("grid,B,stream", CASES, ids=_case_id)
def test_blocks_unit_by_unit(engines, grid, B, stream):
    """stage-local: every unit of all 16 blocks within its bound, sentinels intact; chained: the stream after every
    block within the row bound of the oracle's fp16 emulation"""
    cfg, w, eng = engines(grid)
    eng.debug_set("fp32_stream", int(stream == "fp32"))
    xs = torch.from_numpy(_states(cfg, B)).cuda()
    ref, tol = ps.chain_bounds(cfg, w, list(_states(cfg, B)))
    tag = f"{cfg.nlat}x{cfg.nlon} B={B} {stream} stream"
    fails, sent, chained = [], [], []
    try:
        for li in range(4):
            for bi in range(cfg.depths[li]):
                g = ps.level(cfg, li)
                taps = block_taps(eng, cfg, B, stream, li, bi, xs, sentinels=sent)
                fails += check_block(cfg, w, B, stream, li, bi, taps, np.arange(B * g.nWin), tag)
                e = ps.row_rel(_stream_rows(taps, stream, g, B), ref[(li, bi)])
                print(f"{tag} chained layer {li} block {bi}: worst row rel L2 {e.max():.3e} (row {int(e.argmax())}), "
                      f"bound {tol[(li, bi)]:.3e}")
                if not e.max() <= tol[(li, bi)]:
                    chained.append((li, bi, float(e.max()), tol[(li, bi)]))
                del taps
    finally:
        eng.debug_set("stop_launch", -1)
        eng.debug_set("fp32_stream", 0)
    assert not fails, fails
    assert all(ok for _, ok in sent), [s for s, ok in sent if not ok]
    assert not chained, chained


def _read_all(eng, cfg, B, stream, xs, fill):
    """every block's taps, valid regions only, on the host"""
    out = {}
    for li in range(4):
        g = ps.level(cfg, li)
        nkb, R = g.C // 64, B * g.T
        for bi in range(cfg.depths[li]):
            for kind, t in block_taps(eng, cfg, B, stream, li, bi, xs, fill).items():
                for name, v in t.items():
                    if name in ("stream_h", "att_h", "hid_h"):
                        v = image_rows(v, np.arange(R), nkb * (4 if name == "hid_h" else 1)).view(np.int16)
                    else:
                        v = v.cpu().numpy()
                    out[(li, bi, kind, name)] = v
    return out


@pytest.mark.parametrize("stream", ["fp16", "fp32"])
@pytest.mark.parametrize("grid", GRIDS, ids=_case_id)
def test_poisoned_workspace_reaches_no_valid_output(engines, grid, stream):
    """workspace of 0x00 bytes, then of 0xFF bytes (NaN in fp16 and fp32), before every stopped step, B = 3: every tap's
    valid region and the new state are equal bit for bit"""
    cfg, w, eng = engines(grid)
    B = 3
    eng.debug_set("fp32_stream", int(stream == "fp32"))
    xs = torch.from_numpy(_states(cfg, B)).cuda()
    try:
        t0 = _read_all(eng, cfg, B, stream, xs, 0)
        t1 = _read_all(eng, cfg, B, stream, xs, 0xFF)
        eng.debug_set("stop_launch", -1)
        ys = []
        for fill in (0, 0xFF):
            eng._workspace(B).fill_(fill)
            ys.append(eng.step(xs).cpu().numpy())
    finally:
        eng.debug_set("stop_launch", -1)
        eng.debug_set("fp32_stream", 0)
    diff = [k for k in t0 if not np.array_equal(t0[k], t1[k])]
    assert not diff, diff
    assert np.isfinite(ys[0]).all() and np.array_equal(ys[0], ys[1])


@pytest.mark.parametrize("stream", ["fp16", "fp32"])
@pytest.mark.parametrize("grid", GRIDS, ids=_case_id)
def test_stops_graphs_and_launches(engines, grid, stream):
    """a step stopped after its last unit is the whole step, bit for bit; with stop_launch back at -1 the eager, captured
    and replayed steps agree bit for bit; launches per step = the unit list's, for B = 1 and 3"""
    from skyrim_b200.engine import launch_count
    cfg, w, eng = engines(grid)
    eng.debug_set("fp32_stream", int(stream == "fp32"))
    u = ps.units(cfg, stream)
    try:
        for B in (1, 3):
            xs = torch.from_numpy(_states(cfg, B)).cuda()
            y = torch.empty_like(xs)
            eng.debug_set("stop_launch", len(u))
            l0 = launch_count()
            stopped = eng.step(xs).cpu().numpy()
            counts = [launch_count() - l0]
            eng.debug_set("stop_launch", -1)
            outs = []
            for _ in range(3):           # eager, captured, replayed
                l0 = launch_count()
                eng.step(xs, y)
                torch.cuda.synchronize()
                counts.append(launch_count() - l0)
                outs.append(y.cpu().numpy())
            print(f"{cfg.nlat}x{cfg.nlon} {stream} stream B = {B}: launches per step {counts}, unit list "
                  f"{sum(n for *_, n in u)}")
            assert counts == [sum(n for *_, n in u)] * 4
            assert np.isfinite(outs[0]).all()
            assert all(np.array_equal(o, outs[0]) for o in outs) and np.array_equal(stopped, outs[0])
    finally:
        eng.debug_set("stop_launch", -1)
        eng.debug_set("fp32_stream", 0)


def test_full_size_first_blocks():
    """721 x 1440, one member, fp16 stream: the first two blocks of layers 0 and 1, every window of the first and last
    window rows and a seeded sample"""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from skyrim_b200.config import pangu_full
    from skyrim_b200.engine import StepEngine
    from skyrim_b200.weights import make_pangu_weights
    cfg = pangu_full()
    w = make_pangu_weights(cfg, 1)
    eng = StepEngine(cfg, 0)
    eng.load_weights(w)
    B, fails, sent = 1, [], []
    xs = torch.from_numpy(_states(cfg, B)).cuda()
    try:
        for li, bi in [(0, 0), (0, 1), (1, 0), (1, 1)]:
            g = ps.level(cfg, li)
            wins = np.array([b * g.nWin + wi for b, wi in sample_windows(g, B, True, seed=11 + li)])
            taps = block_taps(eng, cfg, B, "fp16", li, bi, xs, sentinels=sent)
            fails += check_block(cfg, w, B, "fp16", li, bi, taps, wins, f"721x1440 B=1 fp16 stream ({len(wins)} windows)")
            del taps
    finally:
        eng.debug_set("stop_launch", -1)
        eng.close()
    assert not fails, fails
    assert all(ok for _, ok in sent), [s for s, ok in sent if not ok]


def test_summary():
    """the largest |error| / bound per unit kind over the cases that ran in this session (print only)"""
    for name, r in sorted(WORST.items()):
        print(f"[pangu stages] worst {name}: {r:.3f}")
