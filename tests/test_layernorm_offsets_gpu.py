"""The LayerNorm GEMM epilogues on rows whose |mean| is up to 3000 times their standard deviation, element by element
against the fp64 bound of oracle/gemm_ref.py.

LayerNorm does not change when a constant is added to every element of a row, but a variance taken in one pass as
ss / n - mean^2 in fp32 loses it to cancellation once |mean| / std reaches ~100.  The epilogues take their statistics
about the mean (gemm2.cuh LnStat); gemm_ref.layer_norm's bound is linear in |mean| / std (tests/test_layernorm_offsets_cpu.py
checks it against fp32 emulations of every path), so these cases fail for one-pass statistics from a ratio of 100 on.

Kernel level, through libskyrim_b200_probe.so: one A column holds a per-row fp16 value a_r and the matching W column is 1,
so every output of row r is shifted by a_r, with a_r / std cycling over 0, 10, 100, 1000 and 3000:
  * single CTAs at BLOCK_N 192: Epi2F32Img<true, 1> (fp32 rows and their image), <true, 2> (the fp16 image in place) and
    its fragment path FragEpi<Epi2F32Img<true, 2>>;
  * CTA pairs at 2 x 192 with the same three, and GraphCast's Epi2F32Img<true, 0 / 1 / 2> at 2 x 256;
  * the fused MLP (mlp_fused.cuh) at C = 192 and 384, with a constant offset of 10, 100 and 1000 row deviations on b2,
    which must also stay bit for bit what fc1 + fc2 write.
Each runs at M = 300 and at Pangu's full token count (a sampled set of rows), on all SMs and on one CTA (pair).  As in
tests/test_gemm_fragment_epilogue_gpu.py the stream image sits between guard bands of an fp16 NaN sentinel, the A rows past
M and the image rows past M hold it too, and pytest -s prints the worst err / bound of every ratio.

Model level, with shifts that LayerNorm removes: Pangu steps with the projection and fc2 biases of one block per layer
shifted by 10, 100 and 1000 row deviations (both stream modes, against the oracle), GraphCast's units with every MLP's b2
shifted (each against its fp64 bound from the engine's own inputs), and Pangu's up-sample with the up.w1 rows of one
sub-position shifted by a common vector.
"""
from __future__ import annotations

import numpy as np
import pytest

from oracle import gemm_probe as gp
from oracle import gemm_ref as gr

torch = pytest.importorskip("torch")

from test_gemm_fragment_epilogue_gpu import T, Guarded, image, image_rows, run, sample_rows  # noqa: E402
from test_pangu_mlp_fused_gpu import EPS, Mlp  # noqa: E402

pytestmark = pytest.mark.gpu

EPI_LN_IMG_FRAG = 19
RATIOS = [0, 10, 100, 1000, 3000]
K = 192
SD = 1.0 / 3.0   # std of a row of A W^T + bias with A ~ U[-1, 1), W ~ U[-1, 1) / sqrt(K), bias ~ U[-0.1, 0.1]

# name: (kernel, epilogue, BLOCK_N, residual source: "rows" fp32 rows in place, "img" the image in place, None)
EPIS = {
    "W/LN": (gp.W, gp.EPI_LN, 192, "rows"),
    "W/LN_IMG": (gp.W, gp.EPI_LN_IMG, 192, "img"),
    "W/LN_IMG_FRAG": (gp.W, EPI_LN_IMG_FRAG, 192, "img"),
    "PAIR/LN": (gp.PAIR, gp.EPI_LN, 192, "rows"),
    "PAIR/LN_IMG": (gp.PAIR, gp.EPI_LN_IMG, 192, "img"),
    "PAIR/LN_IMG_FRAG": (gp.PAIR, EPI_LN_IMG_FRAG, 192, "img"),
    "PAIR/GC_LN0": (gp.PAIR, gp.EPI_GC_LN0, 256, None),
    "PAIR/GC_LN1": (gp.PAIR, gp.EPI_GC_LN1, 256, "rows"),
    "PAIR/GC_LN2": (gp.PAIR, gp.EPI_GC_LN2, 256, "img"),
}


def model(epi: int, bn: int, pair: bool) -> dict:
    """gemm_ref.layer_norm's depth and shift of the epilogue's statistics"""
    if epi == EPI_LN_IMG_FRAG:
        return dict(depth=gr.ln_depth(bn // 16 + 2, 2 + pair))
    return dict(depth=gr.ln_depth(bn // 8 + 2, 1 + pair), shift=gr.ln_shift(bn))


def offset_operands(M: int, N: int, seed: int):
    """A image (int16, device) with column 0 = a_r, and W [N, K] fp16 with column 0 = 1; the target ratio of every row"""
    nkb = K // 64
    a = image(M, nkb, seed)
    rng = np.random.default_rng(seed)
    target = np.asarray(RATIOS, np.float64)[np.arange(M) % len(RATIOS)]
    ar = (target * SD * rng.choice([-1.0, 1.0], M)).astype(np.float16)
    r = torch.arange(M, device="cuda")
    v = a.view(-1, nkb, 128, 8, 8)
    v[r // 128, 0, r % 128, (r % 128) & 7, 0] = torch.from_numpy(ar.view(np.int16)).cuda()
    w = (rng.uniform(-1.0, 1.0, (N, K)) / np.sqrt(K)).astype(np.float16)
    w[:, 0] = 1.0
    return a, w, target


def report(name: str, got, ref, bound, target, rows) -> float:
    """worst err / bound per target ratio (printed); the overall worst"""
    parts, worst = [], 0.0
    for t in RATIOS:
        m = target[rows] == t
        if m.any():
            r = gr.worst(got[m], ref[m], bound[m])
            worst = max(worst, r)
            parts.append(f"{t}: {r:.3f}")
    print(f"[ln offsets] {name}: max err/bound by |mean|/std " + ", ".join(parts))
    return worst


CASES = [(name, M, grid) for name in EPIS for M in ("300", "full") for grid in ("all", "one")]


@pytest.mark.parametrize("name,M,grid", CASES)
def test_layer_norm_row_offsets(name, M, grid):
    kernel, epi, bn, res = EPIS[name]
    pair = kernel == gp.PAIR
    N = 2 * bn if pair else bn
    M = 300 if M == "300" else T[192 if N == 192 else 384]
    grid = 0 if grid == "all" else (2 if pair else 1)
    nkb, onkb = K // 64, N // 64
    a, w, target = offset_operands(M, N, N + M + grid)
    dw = torch.from_numpy(gr.pack_w(w, bn, nkb).copy()).cuda()
    rng = np.random.default_rng(M + bn)
    bias, gamma, beta = (rng.uniform(-0.1, 0.1, N).astype(np.float32), (rng.uniform(-1.0, 1.0, N) + 1.0).astype(np.float32),
                         rng.uniform(-0.1, 0.1, N).astype(np.float32))
    dv = [torch.from_numpy(v).cuda() for v in (bias, gamma, beta)]
    x0 = image(M, onkb, M + 1)
    nbytes = x0.numel() * 2
    img = Guarded(nbytes, x0 if res == "img" else None)
    kw = dict(hi=img.ptr, img_bytes=nbytes, img_nkb=onkb)
    xr = yimg = None
    if epi in (gp.EPI_LN, gp.EPI_GC_LN0, gp.EPI_GC_LN1):   # fp32 rows: the residual (read and rewritten) or the output
        gen = torch.Generator(device="cuda").manual_seed(M)
        xr = (torch.rand(M, N, generator=gen, device="cuda") * 2 - 1).half().float() if res else torch.zeros(M, N, device="cuda")
        kw.update(out=xr.data_ptr(), out_bytes=xr.numel() * 4, ldo=N)
        if epi == gp.EPI_GC_LN1:
            kw.update(xin=xr.data_ptr(), xin_bytes=xr.numel() * 4)
    if epi in (gp.EPI_GC_LN0, gp.EPI_GC_LN1, gp.EPI_GC_LN2):
        yimg = Guarded(nbytes)
        kw.update(yimg=yimg.ptr)
        if epi == gp.EPI_GC_LN2:
            kw.update(xin_img=img.ptr, xin_bytes=nbytes)
    rows = sample_rows(M, N + M)
    resid = (image_rows(x0, rows, onkb).astype(np.float64) if res == "img" else
             xr[torch.from_numpy(rows).cuda()].double().cpu().numpy() if res == "rows" else np.zeros((len(rows), N)))
    run(gp.make_case(kernel=kernel, epi=epi, block_n=bn, n=N, n_valid=N, batches=1, grid_sms=grid, nseg=1, m=M, a=[a.data_ptr()],
                     a_bytes=[a.numel() * 2], a_batch_stride=[0], a_nkb=[nkb], w=dw.data_ptr(), w_bytes=dw.numel(), num_kb=nkb,
                     bias=dv[0].data_ptr(), gamma=dv[1].data_ptr(), beta=dv[2].data_ptr(), vec_floats=N, eps=1e-5, **kw))
    img.check(M, onkb, "stream image")
    R, S = gr.linear([(image_rows(a, rows, nkb), w)])
    d = model(epi, bn, pair)
    ref, bound = gr.layer_norm(R, S, bias[None, :], gamma[None, :], beta[None, :], resid, 1e-5, **d)
    y = R + bias[None, :]
    ratio = np.abs(y.mean(1)) / y.std(1)
    assert ratio[target[rows] == 3000].min() > 2000 and ratio[target[rows] == 0].max() < 1.0
    tag = f"{name} M={M} grid={grid}"
    worst = report(tag + " fp16 image", image_rows(img.inner(), rows, onkb).astype(np.float64), ref, gr.f16_bound(ref, bound),
                   target, rows)
    if xr is not None:
        got = xr[torch.from_numpy(rows).cuda()].double().cpu().numpy()
        worst = max(worst, report(tag + " fp32 rows", got, ref, bound, target, rows))
    if yimg is not None:
        yimg.check(M, onkb, "update image")
        yr, yb = gr.layer_norm(R, S, bias[None, :], gamma[None, :], beta[None, :], 0.0, 1e-5, **d)
        worst = max(worst, report(tag + " y image", image_rows(yimg.inner(), rows, onkb).astype(np.float64), yr,
                                  gr.f16_bound(yr, yb), target, rows))
    assert worst <= 1.0, f"{tag}: LayerNorm error exceeds its bound by {worst:.3f}x"


@pytest.mark.parametrize("grid", [0, 1])
@pytest.mark.parametrize("M", ["300", "full"])
@pytest.mark.parametrize("C", [192, 384])
def test_fused_mlp_b2_offset(C, M, grid):
    """fc2's bias shifted by k row deviations, k = 10, 100, 1000: the fused MLP within the fp64 bound built from the hidden
    image of fc1 + fc2, and bit for bit what fc1 + fc2 write"""
    if M == "full" and grid:
        pytest.skip("the full token count runs on all SMs only, as in tests/test_pangu_mlp_fused_gpu.py")
    NKB = C // 64
    M = 300 if M == "300" else T[C]
    grid = grid if C == 192 else 2 * grid
    mlp = Mlp(C + M + grid, C)
    x0 = image(M, NKB, M + 3)
    rows = sample_rows(M, C + M)
    x = image_rows(x0, rows, NKB).astype(np.float64)
    b2 = mlp.b2.copy()
    sd = None
    for k in (0, 10, 100, 1000):
        mlp.b2 = (b2 + np.float32(k * sd if k else 0.0)).astype(np.float32)
        mlp.db2 = torch.from_numpy(mlp.b2).cuda()
        two, hid = mlp.two_gemm(x0, M, grid)
        got = mlp.fused(x0, M, grid)
        got.check(M, NKB, "stream image")
        assert torch.equal(got.t, two.t), f"k={k}: the fused MLP differs from fc1 + fc2"
        R2, S2 = gr.linear([(image_rows(hid.inner(), rows, 4 * NKB), mlp.w2)])
        if sd is None:
            sd = float(np.median((R2 + b2[None, :]).std(1)))
        y, yb = gr.layer_norm(R2, S2, mlp.b2[None, :], mlp.gamma[None, :], mlp.beta[None, :], x, EPS,
                              depth=gr.ln_depth(192 // 16 + 2, 2 + (C == 384)))
        r = gr.worst(image_rows(got.inner(), rows, NKB).astype(np.float64), y, gr.f16_bound(y, yb))
        print(f"[ln offsets] fused MLP C={C} M={M} grid={grid} b2 + {k} sd: max err/bound {r:.3f}")
        assert r <= 1.0, f"fused MLP, b2 + {k} sd: error exceeds its bound by {r:.3f}x"


# ---------------------------------------------------------------------------------------------------------------------
# model level: Pangu with the projection and fc2 biases of one block per layer shifted by k row deviations
# ---------------------------------------------------------------------------------------------------------------------
def _ln_input_sd(ref, x0):
    """median row deviation of every LayerNorm input of one oracle step, by the name of its gamma; the step"""
    import torch.nn.functional as F
    names = {id(t): k[: -len(".g")] for k, t in ref.w.items() if k.endswith(".g")}
    sd, layer_norm = {}, F.layer_norm

    def capture(y, shape, weight=None, bias=None, eps=1e-5):
        sd.setdefault(names[id(weight)], float(y.reshape(-1, shape[-1]).std(-1).median()))
        return layer_norm(y, shape, weight, bias, eps)

    F.layer_norm = capture
    try:
        out = ref.step(x0).numpy()
    finally:
        F.layer_norm = layer_norm
    return sd, out


@pytest.fixture(scope="module")
def pangu_small_case():
    from oracle.pangu_ref import PanguRef
    from skyrim_b200.config import PANGU_CHANNELS, pangu_small
    from skyrim_b200.weights import make_pangu_weights, synthetic_state
    cfg = pangu_small(41, 96)
    w = make_pangu_weights(cfg, 0)
    x0 = synthetic_state(PANGU_CHANNELS, cfg.nlat, cfg.nlon, 0)
    sd, _ = _ln_input_sd(PanguRef(cfg, w, dtype=torch.float64), x0)
    return cfg, w, x0, PanguRef(cfg, w).step(x0).numpy(), sd


@pytest.mark.parametrize("stream", ["fp32", "fp16"])
def test_pangu_step_with_shifted_biases(pangu_small_case, stream):
    """Block 0 of every layer gets proj.b + k sd(ln1 input) and fc2.b + k sd(ln2 input), k = 10, 100, 1000: LayerNorm
    removes the shift, so the step must stay within the north star's 1e-3 of the unshifted oracle and within 1.5 x of the
    unshifted engine step's error (fp32_stream runs the staged epilogues, the fp16 stream the fragment path and the fused
    MLP).  With one-pass statistics a shift of 100 already costs the LayerNorm outputs ~6e-3."""
    from oracle.pangu_ref import rel_err_per_channel
    from skyrim_b200.engine import StepEngine
    cfg, w, x0, ref, sd = pangu_small_case
    errs = {}
    for k in (0, 10, 100, 1000):
        ws = dict(w)
        for li in range(len(cfg.depths)):
            p = f"layer{li}.block0."
            ws[p + "proj.b"] = (np.asarray(w[p + "proj.b"], np.float64) + k * sd[p + "ln1"]).astype(np.float32)
            ws[p + "fc2.b"] = (np.asarray(w[p + "fc2.b"], np.float64) + k * sd[p + "ln2"]).astype(np.float32)
        eng = StepEngine(cfg, 0)
        eng.load_weights(ws)
        if stream == "fp32":
            eng.debug_set("fp32_stream", 1)
        y = eng.step(torch.from_numpy(x0)[None].cuda())[0].cpu().numpy()
        eng.close()
        errs[k] = float(rel_err_per_channel(y, ref).max())
    print(f"[ln offsets] Pangu 41x96 {stream} stream: max per-channel rel err by bias shift (row deviations) "
          + ", ".join(f"{k}: {e:.3e}" for k, e in errs.items()))
    for k in (10, 100, 1000):
        assert errs[k] < 1e-3 and errs[k] <= 1.5 * errs[0], f"{stream} stream, shift {k} sd: rel err {errs[k]:.3e} ({errs[0]:.3e} unshifted)"


# ---------------------------------------------------------------------------------------------------------------------
# model level: GraphCast with every LayerNorm MLP's b2 shifted by k row deviations
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [10, 100, 1000])
def test_graphcast_units_with_shifted_b2(k):
    """41 x 96 grid, refinement-2 mesh, 2 processor layers: b2 of every MLP that ends in a LayerNorm + k sd of that
    LayerNorm's input rows (from an oracle step); every unit of the step within its fp64 bound from the engine's own inputs
    (graphcast_stages_ref.check_step), as tests/test_graphcast_stages_gpu.py checks the unshifted step"""
    import torch.nn.functional as F
    from oracle import graphcast_stages_ref as st
    from oracle.graphcast_ref import GraphCastRef
    from test_graphcast_stages_gpu import T0, _engine, _inputs, _read_taps
    cfg, graph, w, x = _inputs("41x96-m2-L2")
    ref = GraphCastRef(cfg, w, graph)
    names = {id(t): n[: -len(".ln.g")] for n, t in ref.w.items() if n.endswith(".ln.g")}
    sd, layer_norm = {}, F.layer_norm

    def capture(y, shape, weight=None, bias=None, eps=1e-5):
        sd.setdefault(names[id(weight)], float(y.reshape(-1, shape[-1]).std(-1).median()))
        return layer_norm(y, shape, weight, bias, eps)

    F.layer_norm = capture
    try:
        ref.step(x, T0)
    finally:
        F.layer_norm = layer_norm
    assert sd, "no LayerNorm seen in the oracle step"
    ws = dict(w)
    for name, s in sd.items():
        ws[name + ".b2"] = (np.asarray(w[name + ".b2"], np.float64) + k * s).astype(np.float32)
    eng = _engine(cfg, graph, ws)
    taps = _read_taps(eng, cfg, graph, x)
    eng.close()
    res = st.check_step(cfg, graph, ws, x, T0, taps)
    worst = st.by_stage(res)
    print(f"[ln offsets] GraphCast 41x96-m2-L2, {len(sd)} MLPs with b2 + {k} sd: worst err/bound per stage "
          + ", ".join(f"{n} {v:.3f}" for n, v in worst.items()))
    assert not [r for r in res if r[4]], [r for r in res if r[4]]


# ---------------------------------------------------------------------------------------------------------------------
# model level: Pangu's up-sample (Epi2UpShuffle) with the up.w1 rows of one sub-position shifted by a common vector
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stream", ["fp16", "fp32"])
@pytest.mark.parametrize("k", [10, 100, 1000])
def test_up_sample_with_shifted_sub_position(k, stream):
    """41 x 96 grid, weights of seed 1: all C rows of up.w1 that feed sub-position (1, 0) get the same vector v added, so
    every fine token from that sub-position gets the offset x2h_r . v; v is scaled so that the median |offset| / row sd
    is k.  The LayerNorm image (hidh) is read at the up-sample's tap and held to the bound of the fp16 operands the
    engine packs (oracle/pangu_resample_ref.up_shuffle), as tests/test_pangu_resample_gpu.py checks it unshifted"""
    from oracle import pangu_resample_ref as pr
    from skyrim_b200.config import pangu_small
    from skyrim_b200.engine import StepEngine
    from skyrim_b200.weights import make_pangu_weights
    from test_pangu_resample_gpu import _image, _step
    cfg, B, sub = pangu_small(41, 96), 1, 2
    C = cfg.dim
    R1, R2 = B * cfg.Z * cfg.H * cfg.W, B * cfg.Z * cfg.H2 * cfg.W2
    w = make_pangu_weights(cfg, 1)
    x2h = None
    v = np.random.default_rng(k).choice([-1.0, 1.0], 2 * C) / np.sqrt(2 * C)
    scale = None
    for shift in (False, True):
        ws = dict(w)
        if shift:
            w1 = np.asarray(w["up.w1"], np.float64).copy()
            w1[sub * C:(sub + 1) * C] += scale * v[None, :]
            ws["up.w1"] = w1.astype(np.float32)
        eng = StepEngine(cfg, 0)
        eng.load_weights(ws)
        try:
            wsp, lay = _step(cfg, eng, B, stream, 5)
            x2h, _ = _image(wsp, lay, "x2h", R2, 2 * C)
            hid, _ = _image(wsp, lay, "hidh", R1, C)
        finally:
            eng.close()
        gw = pr.gemm_weights(cfg, ws)
        coarse, subs = pr.shuffle_sources(cfg, B)
        rows = np.flatnonzero((subs == sub) & (coarse >= 0))
        if not shift:   # |offset| / sd of the unshifted rows -> the scale of v
            y = x2h[coarse[rows]] @ np.asarray(gw["up1"], np.float64)[sub * C:(sub + 1) * C].T
            scale = k * float(np.median(y.std(1) / np.abs(x2h[coarse[rows]] @ v)))
            continue
        ref, bnd = pr.up_shuffle(cfg, ws, x2h, gw["up1"], B, rows)
        y = x2h[coarse[rows]] @ np.asarray(gw["up1"], np.float64)[sub * C:(sub + 1) * C].T
        ratio = np.abs(y.mean(1)) / y.std(1)
        r = gr.worst(hid[rows], ref, bnd)
        print(f"[ln offsets] up-sample 41x96 {stream} stream, sub-position {sub} + v: median |mean|/sd {np.median(ratio):.0f} "
              f"(max {ratio.max():.0f}), max err/bound {r:.3f} over {len(rows)} tokens")
        assert np.median(ratio) > 0.3 * k
        assert r <= 1.0, f"up-sample, median ratio {np.median(ratio):.0f}: error exceeds its bound by {r:.3f}x"
