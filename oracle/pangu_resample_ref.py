"""ORACLE — test infrastructure, not product code.

Float64 references of the Pangu step's units between the transformer layers as the engine computes them
(skyrim_b200/csrc/pangu_engine.cu, gemm2.cuh), for tests/test_pangu_resample_gpu.py, and the mirror of the engine's
workspace layout (PanguEngine::carve) that the engine-level tests read raw regions through:

  down-sample   k_down_merge_ln<24>: 2x2 (lat, lon) merge of the level-1 tokens into rows of 4C = (hs, ws, c) features,
                zero rows where 2 h2 + hs >= H, two-pass fp32 LayerNorm over all 4C (the zeros included), fp16 image;
                then the down GEMM (Epi2F32Img<false, 0>: the plain product, fp16 image and, with the fp32 token stream,
                fp32 rows)
  up-sample     linear1 on Epi2UpShuffle: n-tile `sub` = (hs, ws) of the 4C outputs, two-pass LayerNorm over its C
                columns, stored at the fine token (z, 2 h2 + hs, 2 w2 + ws) when 2 h2 + hs < H; then linear2
                (Epi2F32Img<false, 0>)
  recovery      Epi2Recover on k_gemm2 at BLOCK_N 224: A = [skip | x1] along K, weight columns ((v 2 + dz) 4 + dh) 4 + dw
                (upper air, slab z >= 1, level 2 (z - 1) + dz, level 13 dropped) and 160 + (v 4 + dh) 4 + dw (surface,
                slab 0), latitude 4 h + dh cropped at nlat, + bias of the variable, * std + mean of the channel

Inputs are the exact operands the kernels read (fp16 images, or fp32 rows with the fp32 token stream) and the fp16
packed weights (gemm_weights); with float64 inputs and unrounded weights the same functions are the model
(oracle/pangu_ref.py), which tests/test_pangu_resample_cpu.py checks.  Tokens are rows (member, z, h, w) of the grid
level's natural order.  Every function returns (reference, per-element bound); the bounds of fp16 stores include the
store's half ulp.  `rows` restricts a reference to some output rows (the full-size case checks a sample).

Bound of k_down_merge_ln (two-pass statistics; u = 2^-24, n = 4C = 768, 24 values per lane, first order in u):
  mean   each lane adds its 24 values as 6 sums ((a + b) + (c + d)) onto its running sum, the warp adds the 32 lane sums
         in 5 butterfly steps: no value passes more than 2 + 1 + 5 + 5 = 13 fp32 additions, and s / n is one correctly
         rounded division: |mu' - mu| <= 13 u sum|v| / n + u |mu| <= dmu = 16 u mean|v| (margin for the second order);
  var    d_i = fl(v_i - mu') = (v_i - mu')(1 + e), squared (2u), multiplied (u), 24 sequential additions per lane and 5
         warp steps (29u), divided by n (u): V' = (V + (mu - mu')^2)(1 + 33u), because sum (v_i - mu')^2 = n V + n
         (mu - mu')^2 exactly; + eps adds u (V + eps);
  rstd   rsqrtf is within 2 ulp (CUDA C Programming Guide, Mathematical Functions): 2^-22 relative, so
         |r' - r| / r <= rho = rel / 2 + 2^-22 with rel = (dmu^2 + 35u (V + eps + dmu^2)) / (V + eps);
  out    fl(fl(fl(d_i r') g) + b) = g r (v_i - mu) + g r (mu - mu') + g r (v_i - mu') theta + rounding of the sum, with
         |theta| <= rho + 3u: |out' - out| <= |g| r dmu + |g yn| (rho + 4u) + u |b| (yn = (v_i - mu) r), then the fp16
         store (half an fp16 ulp).
The LayerNorm of Epi2UpShuffle is gemm_ref.layer_norm's model with bias 0 and residual 0: one lane adds its row's C
values in sequence (the mean, ln_depth(C, 0) roundings), then their squared deviations from that mean; the variance is
taken about the mean, so the bound stays linear in |mean| / std, as for k_down_merge_ln.
"""
from __future__ import annotations

import numpy as np

from oracle import gemm_ref as gr
from oracle import pangu_kernels_ref as pk

U = gr.U32
G2_A_BYTES = 128 * 128          # one 128-row x 128-byte tile of an operand image
REC_UPPER = 160                 # upper-air columns of the recovery weight (5 variables x 2 levels x 4 x 4)
REC_N = 224                     # + 64 surface columns (4 variables x 4 x 4): the GEMM's N and BLOCK_N


# ---------------------------------------------------------------------------------------------------------------------
# workspace layout
# ---------------------------------------------------------------------------------------------------------------------
def workspace_layout(cfg, B: int) -> dict:
    """byte offset of every region of the engine's workspace for B members, and "total" (PanguEngine::carve): each
    region starts on a 1 KiB boundary"""
    g1, g2 = pk.grids(cfg)
    C = cfg.dim
    R1, R2 = B * g1.T, B * g2.T
    t1, t2 = -(-R1 // 128), -(-R2 // 128)
    x1h = t1 * (C // 64) * G2_A_BYTES
    wt = max(B * g1.nWin * g1.pairs, B * g2.nWin * g2.pairs)
    sizes = [("x1", R1 * C * 4), ("x2", R2 * 2 * C * 4), ("x1h", x1h), ("skiph", x1h), ("x2h", t2 * (2 * C // 64) * G2_A_BYTES),
             ("qkv", 3 * wt * pk.TILE_B), ("atth", max(t1 * (C // 64), t2 * (2 * C // 64)) * G2_A_BYTES),
             ("hidh", max(t1 * (4 * C // 64), t2 * (8 * C // 64)) * G2_A_BYTES)]
    out, off = {}, 0
    for name, n in sizes:
        out[name] = off
        off += -(-n // 1024) * 1024
    out["total"] = off
    return out


# ---------------------------------------------------------------------------------------------------------------------
# weights and index maps
# ---------------------------------------------------------------------------------------------------------------------
def packed(a, round16: bool = True) -> np.ndarray:
    """a weight as k_pack_weight packs it (fp16 of the fp32 value), as float64; round16=False: the weight itself"""
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float64) if round16 else np.asarray(a, np.float64)


def gemm_weights(cfg, w, round16: bool = True) -> dict:
    """the [N, K] weights of the down, up1, up2 and recovery GEMMs as the engine packs them (k_pack_weight: fp16 of the
    fp32 value; recovery: upper-air | surface columns of the transposed weights), as float64"""
    C = cfg.dim
    f = lambda a: packed(a, round16)   # noqa: E731
    rec = np.concatenate([np.asarray(w["recover.upper.w"]).reshape(2 * C, -1).T, np.asarray(w["recover.surf.w"]).reshape(2 * C, -1).T])
    assert rec.shape == (REC_N, 2 * C)
    return {"down": f(w["down.w"]), "up1": f(w["up.w1"]), "up2": f(w["up.w2"]), "rec": f(rec)}


def restride(x: np.ndarray, B: int, T: int, stride: int) -> np.ndarray:
    """the rows a kernel reads for members 0..B-1 when it steps `stride` rows per member instead of T (a modelled
    mistake: stride = (Z - 1) H W, the upper-air embedding's member stride)"""
    idx = (np.arange(B)[:, None] * stride + np.arange(T)[None, :]).reshape(-1)
    return np.asarray(x)[idx]


def _rows(rows, n):
    return np.arange(n) if rows is None else np.asarray(rows, np.int64)


def merge_sources(cfg, B: int, rows=None, swap: bool = False) -> np.ndarray:
    """[rows, 4] level-1 token of each (hs, ws) sub-position of down-sample rows (member, z, h2, w2), -1 for the zero
    padding row at odd H.  swap models a kernel that takes hs from the low bit of the sub-position"""
    H, W, H2, W2 = cfg.H, cfg.W, cfg.H2, cfg.W2
    r = _rows(rows, B * cfg.Z * H2 * W2)
    q, h2, w2 = r // (H2 * W2), (r // W2) % H2, r % W2
    sub = np.arange(4)
    hs, ws = (sub & 1, sub >> 1) if swap else (sub >> 1, sub & 1)
    h = 2 * h2[:, None] + hs[None]
    w_ = 2 * w2[:, None] + ws[None]
    return np.where(h < H, (q[:, None] * H + h) * W + w_, -1)


def shuffle_sources(cfg, B: int, rows=None, swap: bool = False, h_lim: int | None = None) -> tuple[np.ndarray, np.ndarray]:
    """(coarse row, sub-position) of Epi2UpShuffle's output at fine tokens `rows` (-1: no store reaches the row).
    h_lim models a crop at h < h_lim instead of h < H: at H - 1 the last row is never written; at H + 1 (odd H) the
    merge's padding row lands on the next slab's first row."""
    H, W, H2, W2 = cfg.H, cfg.W, cfg.H2, cfg.W2
    r = _rows(rows, B * cfg.Z * H * W)
    q, h, w_ = r // (H * W), (r // W) % H, r % W
    lim = H if h_lim is None else h_lim
    if lim > H and H % 2:              # the store of the padding row h = H of slab q - 1 overwrites row (q, 0)
        spill = (h == 0) & (q > 0)
        q = np.where(spill, q - 1, q)
        h = np.where(spill, H, h)
    hs, ws = h % 2, w_ % 2
    sub = ws * 2 + hs if swap else hs * 2 + ws
    coarse = (q * H2 + h // 2) * W2 + w_ // 2
    return np.where(h < lim, coarse, -1), sub


def recover_targets(cfg, B: int, rows=None, *, dz_swap: bool = False, level_from_z: bool = False,
                    surf_nb_bias: bool = False, surf_nb_stats: bool = False):
    """Epi2Recover's scatter: for token rows (member, z, h, w) and the 224 weight columns, the flat index into the
    (B, 69, nlat, nlon) output (-1: dropped), the bias entry and the channel of the de-normalisation statistics.  The
    knobs model mistakes: dz read the other way round, the level pair taken from z instead of z - 1, the surface bias or
    statistics of the neighbouring variable."""
    H, W, T = cfg.H, cfg.W, cfg.Z * cfg.H * cfg.W
    nu, nl, ns = cfg.n_upper_vars, cfg.n_levels, cfg.n_surface_vars
    nup, nch, nlat, nlon = nu * nl, cfg.n_channels, cfg.nlat, cfg.nlon
    r = _rows(rows, B * T)[:, None]
    b, t = r // T, r % T
    z, h, w_ = t // (H * W), (t // W) % H, t % W
    col = np.arange(REC_N)[None, :]
    upper = col < REC_UPPER
    cs = col - REC_UPPER
    dz = (col >> 4) & 1
    if dz_swap:
        dz = 1 - dz
    lev = 2 * (z if level_from_z else z - 1) + dz
    v_s = (cs >> 4) % ns
    ch = np.where(upper, (col >> 5) * nl + lev, nup + v_s)
    bidx = np.where(upper, col >> 5, nu + (v_s + surf_nb_bias) % ns)
    sch = np.where(upper, ch, nup + (v_s + surf_nb_stats) % ns)
    dh = np.where(upper, col >> 2, cs >> 2) & 3
    lat, lon = 4 * h + dh, 4 * w_ + (col & 3)
    keep = np.where(upper, (z > 0) & (lev >= 0) & (lev < nl), z == 0) & (lat < nlat)
    flat = ((b * nch + ch) * nlat + np.minimum(lat, nlat - 1)) * nlon + lon
    return np.where(keep, flat, -1), np.broadcast_to(bidx, flat.shape), np.where(keep, sch, 0)


# ---------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------
def down_merge_ln(cfg, w, x: np.ndarray, B: int, rows=None, *, swap: bool = False, pad_stats: bool = True):
    """k_down_merge_ln: tokens x [B T1, C] -> the fp16 image rows [rows, 4C] (reference, bound; module docstring).
    pad_stats=False models a kernel that leaves the padding zeros out of the statistics."""
    C, n = cfg.dim, 4 * cfg.dim
    src = merge_sources(cfg, B, rows, swap)
    x = np.asarray(x, np.float64)
    v = np.where((src >= 0)[:, :, None], x[np.maximum(src, 0)], 0.0).reshape(-1, n)
    g = np.asarray(w["down.ln.g"], np.float64)[None]
    bt = np.asarray(w["down.ln.b"], np.float64)[None]
    if pad_stats:
        mu = v.mean(1, keepdims=True)
        var = ((v - mu) ** 2).mean(1, keepdims=True)
    else:
        m = np.repeat(src >= 0, C, axis=1)
        cnt = m.sum(1, keepdims=True)
        mu = (v * m).sum(1, keepdims=True) / cnt
        var = (((v - mu) * m) ** 2).sum(1, keepdims=True) / cnt
    eps = cfg.ln_eps
    r = 1.0 / np.sqrt(var + eps)
    yn = (v - mu) * r
    out = yn * g + bt
    dmu = 16 * U * np.abs(v).mean(1, keepdims=True)
    rel = (dmu * dmu + 35 * U * (var + eps + dmu * dmu)) / (var + eps)
    rho = 0.5 * rel * (1 + rel) + 2.0 ** -22
    bound = np.abs(g) * r * dmu * (1 + 2.0 ** -20) + np.abs(g * yn) * (rho + 4 * U) + U * np.abs(bt)
    return out, gr.f16_bound(out, bound)


def linear_plain(a: np.ndarray, wt: np.ndarray):
    """Epi2F32Img<false, 0> without bias (down GEMM, up-sample linear2): the fp32 rows' (reference, bound); the fp16
    image's bound is gr.f16_bound of them"""
    R, S = gr.linear([(a, wt)])
    return gr.epi_affine(R, S)


def up_shuffle(cfg, w, x2: np.ndarray, wu1: np.ndarray, B: int, rows=None, *, swap: bool = False,
               h_lim: int | None = None, ln_cols: int | None = None):
    """Epi2UpShuffle: level-2 tokens x2 [B T2, 2C] (the fp16 image) and the up1 weight [4C, 2C] -> the fp16 image rows
    of fine tokens `rows` [rows, C] (reference, bound); NaN where no store reaches a row.  ln_cols = 4C models
    statistics over the whole 4C row instead of the sub-position's C columns."""
    C = cfg.dim
    coarse, sub = shuffle_sources(cfg, B, rows, swap, h_lim)
    x2 = np.asarray(x2, np.float64)
    g = np.asarray(w["up.ln.g"], np.float64)[None]
    bt = np.asarray(w["up.ln.b"], np.float64)[None]
    out = np.full((len(sub), C), np.nan)
    bnd = np.full((len(sub), C), np.nan)
    for s in range(4):
        sel = np.flatnonzero((sub == s) & (coarse >= 0))
        if ln_cols == 4 * C:           # every sub-position's columns, then keep sub-position s
            R, S = gr.linear([(x2[coarse[sel]], wu1)])
            o, b = gr.layer_norm(R, S, 0.0, np.tile(g, 4), np.tile(bt, 4), 0.0, cfg.ln_eps)
            o, b = o[:, s * C:(s + 1) * C], b[:, s * C:(s + 1) * C]
        else:
            R, S = gr.linear([(x2[coarse[sel]], wu1[s * C:(s + 1) * C])])
            o, b = gr.layer_norm(R, S, 0.0, g, bt, 0.0, cfg.ln_eps)
        out[sel], bnd[sel] = o, b
    return out, gr.f16_bound(out, bnd)


def recover(cfg, w, a: np.ndarray, wrec: np.ndarray, B: int, rows=None, **knobs):
    """Epi2Recover: A rows [skip | x1] [rows, 2C] of tokens `rows` and the [224, 2C] weight -> (flat index into the
    (B, 69, nlat, nlon) output, reference, bound) of every element those tokens write.  knobs: recover_targets'."""
    flat, bidx, sch = recover_targets(cfg, B, rows, **knobs)
    R, S = gr.linear([(a, wrec)])
    bias = np.concatenate([np.asarray(w["recover.upper.b"], np.float32), np.asarray(w["recover.surf.b"], np.float32)])
    y, by = gr.epi_affine(R, S, bias.astype(np.float64)[bidx])
    keep = flat >= 0
    sd = np.asarray(w["norm.std"], np.float64)[sch]
    mu = np.asarray(w["norm.mean"], np.float64)[sch]
    ref = y * sd + mu
    bound = sd * by + 4 * U * (np.abs(sd * y) + np.abs(mu))
    return flat[keep], ref[keep], bound[keep]


def scatter(flat: np.ndarray, vals: np.ndarray, shape) -> np.ndarray:
    """dense array of `shape` holding vals at flat indices, NaN elsewhere (the later of two writes wins)"""
    out = np.full(int(np.prod(shape)), np.nan)
    out[flat] = vals
    return out.reshape(shape)
