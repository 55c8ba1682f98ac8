"""ORACLE — test infrastructure, not product code.

Stage-local float64 references of the SFNO engine (skyrim_b200/csrc/sfno_engine.cu), for tests/test_sfno_stages_gpu.py
(engine taps read with debug_copy after ``debug_set("stop_after", n)``) and tests/test_sfno_stages_cpu.py (this module on
its own).  Each stage starts from the ENGINE's own input to that stage (the decoded previous tap), so errors do not
accumulate and every stage gets a per-element bound of the form

    |D - R| <= TAU * k_scale(K) * sum |a| |w|  +  epilogue rounding (gemm_ref.epi_affine / epi_gelu / split_bound / col_stats)

where R is formed in float64 from the exact fp16 hi / lo operands the engine reads (the 3-term product
hi*hi + lo*hi + hi*lo) and the same fp32 tables and folded weights it packs.

Layouts (the header comment of sfno_engine.cu): pixel images [(lat, lon)][c]; DFT rows LI [m][lat][(ri, c)]; spectra
SI [l][m][(ri, c)]; mixing output MI / Legendre copy MI2 [m][l][(ro, o)]; inverse-Legendre output DI [lat][(m, ro)][o];
fp32 fields pixel-major [(lat, lon)][c].  Every image is a stack of 128-row x 64-column SWIZZLE_128B tiles
(gemm_ref.unpack_tiles); a tap of an image is its hi bytes followed by its lo bytes.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import gemm_ref as gr

TILE = 16384      # bytes of one 128-row x 64-column fp16 tile


def cdiv(a, b):
    return -(-a // b)


def img_bytes(rows, K, batches=1):
    return batches * cdiv(rows, 128) * cdiv(K, 64) * TILE


class Shapes:
    """the engine's buffer geometry for one config"""

    def __init__(self, cfg):
        self.cfg = cfg
        self.E, self.Cin, self.L = cfg.embed, cfg.n_channels, cfg.layers
        self.Hd = cfg.mlp_ratio * cfg.embed
        self.H1, self.W1, self.H2, self.W2 = cfg.nlat, cfg.nlon, cfg.h, cfg.w
        self.lmax, self.mmax = cfg.lmax, cfg.mmax
        self.P1 = self.H1 * self.W1

    def grids(self, i):
        """(Hi, Wi, Ho, Wo) of block i"""
        big_in, big_out = i == 0, i == self.L - 1
        return ((self.H1, self.W1) if big_in else (self.H2, self.W2)) + ((self.H1, self.W1) if big_out else (self.H2, self.W2))

    def tap_floats(self, name):
        E, n2, Hd, P1 = self.E, 2 * self.E, self.Hd, self.P1
        b = {"in_img": img_bytes(P1, self.Cin), "x_img": img_bytes(P1 + 128, E), "g_img": img_bytes(P1 + 128, Hd),
             "hidden_img": img_bytes(P1 + 128, Hd), "li": img_bytes(self.H1, n2, self.mmax),
             "si": img_bytes(self.mmax, n2, self.lmax), "mi": img_bytes(self.lmax, n2, self.mmax),
             "mi2": img_bytes(self.lmax, n2, self.mmax), "di": img_bytes(2 * self.mmax, E, self.H1)}
        if name in b:
            return 2 * b[name] // 4
        return {"x": P1 * E, "rpm": P1 * E, "f1": P1 * E, "norm0": 2 * E, "norm1": 2 * E, "fc1_bias": Hd, "inner_bias": E,
                "sums0": 4 * E, "sums": 4 * E}[name]


# ---------------------------------------------------------------------------------------------------------------------
# decoding taps
# ---------------------------------------------------------------------------------------------------------------------
def halves(raw):
    """raw tap (any dtype) -> (hi bytes, lo bytes)"""
    u = np.ascontiguousarray(raw).reshape(-1).view(np.uint8)
    n = u.size // 2
    return u[:n], u[n:]


def decode(raw, rows, cols, nkb, batches=1, batch_bytes=0):
    """image tap -> (hi, lo) float64 arrays [batches, rows, cols] (or [rows, cols] when batches == 1 and batch_bytes == 0)"""
    out = []
    for part in halves(raw):
        if batch_bytes:
            x = np.stack([gr.unpack_tiles(part[b * batch_bytes:(b + 1) * batch_bytes], 128, nkb, rows, cols) for b in range(batches)])
        else:
            x = gr.unpack_tiles(part, 128, nkb, rows, cols)
        out.append(x.astype(np.float64))
    return out[0], out[1]


def f64(raw):
    return np.ascontiguousarray(raw).reshape(-1).view(np.float64)


# ---------------------------------------------------------------------------------------------------------------------
# building blocks
# ---------------------------------------------------------------------------------------------------------------------
def wsplit(w32):
    """fp32 weights / table -> float64 (hi, lo) as the packer writes them (k_pack_w3: hi = rn(w), lo = rn(w - hi))"""
    h, l = gr.split16(np.asarray(w32, np.float32))
    return h.astype(np.float64), l.astype(np.float64)


def k_scale(K):
    """factor on S = sum |a w| that makes gemm_ref's TAU * S the accumulation bound of a 3-term product over K: the
    tensor cores round the fp32 accumulator once per 16-wide k-step, by at most 2^-23 of the running sum, so a long
    contraction whose terms share a sign (the DFT's m = 0 row of a channel with a mean) can reach (3 K / 16) 2^-23 of
    sum |a w|; TAU (32 x 2^-23, gemm_ref) is the floor measured at short K"""
    return max(1.0, 3 * cdiv(K, 64) * 4 * 2.0 ** -23 / gr.TAU)


def data_gemm(a_hi, a_lo, w32):
    """pointwise GEMM: activations [M, K] (hi, lo) x fp32 weights [N, K] -> (R, S) [M, N], S scaled by k_scale(K)"""
    w_hi, w_lo = wsplit(w32)
    R, S = gr.linear(gr.split_pairs(a_hi, a_lo, w_hi, w_lo))
    return R, S * k_scale(a_hi.shape[-1])


def table_gemm(t32, x_hi, x_lo):
    """table x data: fp32 table(s) [(B,) M, K] x data [(B,) K, N] (hi, lo) -> (R, S) [(B,) M, N]; the 3-term product with
    the table on the A side (t_hi x_hi + t_hi x_lo + t_lo x_hi); S scaled by k_scale(K)"""
    t_hi, t_lo = wsplit(t32)
    R = t_hi @ x_hi + t_hi @ x_lo + t_lo @ x_hi
    at_hi, at_lo, ax_hi, ax_lo = np.abs(t_hi), np.abs(t_lo), np.abs(x_hi), np.abs(x_lo)
    S = at_hi @ ax_hi + at_hi @ ax_lo + at_lo @ ax_hi
    return R, S * k_scale(t_hi.shape[-1])


def fold_bias(W32, shift32, bias32):
    """k_fold_bias: bias + W @ shift in fp32 (one warp per output: 32 lanes of fmaf, then a shuffle tree)"""
    W = np.asarray(W32, np.float64); sh = np.asarray(shift32, np.float64)
    ref = np.asarray(bias32, np.float64) + W @ sh
    K = W.shape[1]
    return ref, (cdiv(K, 32) + 6) * gr.U32 * (np.abs(W) @ np.abs(sh) + np.abs(bias32))


def norm_affine(x, g, b, eps, dec_err):
    """(scale, shift) of an instance norm (k_finalize_norm) against a two-pass fp64 instance norm of the decoded image x
    [P, E], with its bound.  The engine's statistics are fp32 sums of 32 rows, combined in fp64; the bound is that of such
    sums of the DEVIATIONS x - mean (plus the decoding error of the image against the fp32 values the sums saw), i.e. what
    a computation that does not depend on the channel's offset delivers; a variance formed as E[x^2] - mean^2 from
    unshifted sums leaves it once |mean| >> std."""
    P = x.shape[0]
    mean = x.mean(0)
    dev = x - mean
    var = (dev * dev).mean(0)
    g = np.asarray(g, np.float64); b = np.asarray(b, np.float64)
    rstd = 1.0 / np.sqrt(var + eps)
    sc = g * rstd
    sh = b - mean * sc
    d_mean = (dec_err.sum(0) + 64 * gr.U32 * np.abs(dev).sum(0)) / P
    d_var = (2 * (np.abs(dev) * dec_err).sum(0) + 64 * gr.U32 * (dev * dev).sum(0)) / P + d_mean ** 2
    b_sc = np.abs(sc) * (0.5 * d_var / (var + eps) + 3 * gr.U32)
    b_sh = np.abs(sc) * d_mean + np.abs(mean) * b_sc + 3 * gr.U32 * np.abs(mean * sc) + 2 * gr.U32 * np.abs(sh)
    return sc, sh, b_sc, b_sh


def dec_err(hi, lo):
    """distance of a decoded hi + lo value from the fp32 value it was split from (gemm_ref.split_bound)"""
    return 2.0 ** -22 * np.abs(hi + lo) + gr.SUB16


def mixing_matrix(spec32_l, inner32=None):
    """k_pack_w3 mode 1: the real [(ro, o)][(ri, i)] matrix of degree l; inner: the folded inner skip (fp32 add at load)"""
    wr = np.asarray(spec32_l[..., 0], np.float32)
    if inner32 is not None:
        wr = (wr + np.asarray(inner32, np.float32)).astype(np.float32)
    wi = np.asarray(spec32_l[..., 1], np.float32)
    return np.block([[wr, -wi], [wi, wr]])


# ---------------------------------------------------------------------------------------------------------------------
# stages: each returns a list of checks (name, got, ref, bound); `zero` checks carry bound 0
# ---------------------------------------------------------------------------------------------------------------------
def stage_input(sh: Shapes, x_in, w, in_img):
    """k_pack_tile: v = fma(x, 1/sigma, -mu/sigma) in fp32, then hi = rn(v), lo = rn(v - hi); columns Cin..127 zero.
    Returns (checks, mismatches of the bit-exact split)."""
    std = np.asarray(w["norm.std"], np.float32); mu = np.asarray(w["norm.mean"], np.float32)
    sc = (np.float32(1.0) / std).astype(np.float32)
    shf = (-mu / std).astype(np.float32)
    x = np.asarray(x_in, np.float32).reshape(sh.Cin, -1).T                      # [P1, Cin]
    v64 = x.astype(np.float64) * sc.astype(np.float64) + shf.astype(np.float64)
    hi, lo = decode(in_img, sh.P1, 128, 2)
    # the split of some fp32 v within one ulp of the fused result
    v32 = v64.astype(np.float32)
    ok = np.zeros(v32.shape, bool)
    for cand in (v32, np.nextafter(v32, np.float32(np.inf)), np.nextafter(v32, np.float32(-np.inf))):
        ch, cl = gr.split16(cand)
        ok |= (ch.astype(np.float64) == hi[:, :sh.Cin]) & (cl.astype(np.float64) == lo[:, :sh.Cin])
    bad = int((~ok).sum())
    checks = [("input pack hi+lo", hi[:, :sh.Cin] + lo[:, :sh.Cin], v64, 2.0 ** -22 * np.abs(v64) + 2 * gr.U32 * np.abs(v64) + gr.SUB16),
              ("input pack padding", np.concatenate([hi[:, sh.Cin:], lo[:, sh.Cin:]], 1), 0.0, 0.0)]
    return checks, bad


def _split_checks(name, hi, lo, f, fb):
    b_hi, b_sum = gr.split_bound(f, fb)
    return [(name + " hi", hi, f, b_hi), (name + " hi+lo", hi + lo, f, b_sum)]


def stage_encoder(sh: Shapes, w, in_img, hidden_img, x_img, sums0, x32=None):
    """encoder fc1 + GELU (hidden image), fc2 + positional embedding (x image, fp32 x when L == 1, norm0 statistics)"""
    E, P = sh.E, sh.P1
    a_hi, a_lo = decode(in_img, P, 128, 2)
    w1 = np.zeros((E, 128), np.float32); w1[:, :sh.Cin] = w["enc.fc1.w"]
    R, S = data_gemm(a_hi, a_lo, w1)
    f, fb = gr.epi_gelu(*gr.epi_affine(R, S, np.asarray(w["enc.fc1.b"], np.float64)[None]))
    h_hi, h_lo = decode(hidden_img, P, E, E // 64)
    checks = _split_checks("enc fc1+gelu", h_hi, h_lo, f, fb)
    R, S = data_gemm(h_hi, h_lo, w["enc.fc2.w"])
    pos = np.asarray(w["pos_embed"], np.float64).reshape(E, -1).T
    bias = np.asarray(w["enc.fc2.b"], np.float64)
    f, fb = gr.epi_affine(R, S, bias[None], pos)
    x_hi, x_lo = decode(x_img, P, E, E // 64)
    checks += _split_checks("enc fc2+pos", x_hi, x_lo, f, fb)
    if x32 is not None:
        checks.append(("enc fc2+pos fp32", x32.reshape(-1, E)[:P], f, fb))
    checks += _stats_checks("enc sums0", f64(sums0), f - bias[None], fb)
    return checks


def _stats_checks(name, got, f, fb):
    n = f.shape[1]
    s, q, bs, bq = gr.col_stats(f, fb)
    return [(name + " sum", got[:n], s, bs), (name + " sumsq", got[n:2 * n], q, bq)]


def stage_norm(name, sh: Shapes, x_hi, x_lo, g, b, got):
    """norm affine (scale | shift) against the two-pass fp64 norm of the decoded image"""
    sc, shf, b_sc, b_sh = norm_affine(x_hi + x_lo, g, b, sh.cfg.eps, dec_err(x_hi, x_lo))
    got = np.asarray(got, np.float64).reshape(-1)
    return [(name + " scale", got[:sh.E], sc, b_sc), (name + " shift", got[sh.E:2 * sh.E], shf, b_sh)]


def stage_dft(sh: Shapes, tab, x_img, Hi, Wi, norm0, li):
    """forward DFT per latitude of the raw block input, the norm affine folded behind it:
    LI = fma(T x, sc, sh * t1), t1 = row sums of the fp32 table (k_row_sums)"""
    E, mm = sh.E, sh.mmax
    T = np.asarray(tab, np.float32)                                          # [(m, ri), lon]
    x_hi, x_lo = decode(x_img, Hi * Wi, E, E // 64)
    R, S = table_gemm(T, x_hi.reshape(Hi, Wi, E), x_lo.reshape(Hi, Wi, E))    # [lat, (m, ri), c]
    n0 = np.asarray(norm0, np.float64).reshape(-1)
    sc, shf = n0[:E], n0[E:2 * E]
    t1 = T.astype(np.float64).sum(1)
    t1_err = (cdiv(Wi, 32) + 6) * gr.U32 * np.abs(T.astype(np.float64)).sum(1)
    f = R * sc + (shf[None, :] * t1[:, None])[None]
    fb = gr.TAU * S * np.abs(sc) + (np.abs(shf)[None, :] * (t1_err + gr.U32 * np.abs(t1))[:, None])[None] + 2 * gr.U32 * np.abs(f)
    # -> [m][lat][(ri, c)]
    f = f.reshape(Hi, mm, 2, E).transpose(1, 0, 2, 3).reshape(mm, Hi, 2 * E)
    fb = fb.reshape(Hi, mm, 2, E).transpose(1, 0, 2, 3).reshape(mm, Hi, 2 * E)
    g_hi, g_lo = decode(li, Hi, 2 * E, 2 * E // 64, mm, img_bytes(Hi, 2 * E))
    return _split_checks("forward DFT", g_hi, g_lo, f, fb)


def stage_legendre(sh: Shapes, tab, li, Hi, si, mi2=None):
    """forward Legendre per m: S_m = P_m LI_m -> SI [l][m][(ri, c)] (and MI2 [m][l][(ri, c)]); m > l exactly zero"""
    E, mm, lm = sh.E, sh.mmax, sh.lmax
    d_hi, d_lo = decode(li, Hi, 2 * E, 2 * E // 64, mm, img_bytes(Hi, 2 * E))
    R, S = table_gemm(np.asarray(tab, np.float32), d_hi, d_lo)              # [m, l, (ri, c)]
    f, fb = gr.epi_affine(R, S)
    tri = np.arange(mm)[:, None] <= np.arange(lm)[None, :]                  # [m, l]: m <= l
    g_hi, g_lo = decode(si, mm, 2 * E, 2 * E // 64, lm, img_bytes(mm, 2 * E))
    g_hi, g_lo = g_hi.transpose(1, 0, 2), g_lo.transpose(1, 0, 2)           # -> [m, l, (ri, c)]
    checks = _split_checks("forward Legendre", g_hi[tri], g_lo[tri], f[tri], fb[tri])
    checks.append(("forward Legendre m > l", np.concatenate([g_hi[~tri], g_lo[~tri]]), 0.0, 0.0))
    if mi2 is not None:
        m_hi, m_lo = decode(mi2, lm, 2 * E, 2 * E // 64, mm, img_bytes(lm, 2 * E))
        checks += _split_checks("forward Legendre (inverse layout)", m_hi[tri], m_lo[tri], f[tri], fb[tri])
    return checks


def stage_mixing(sh: Shapes, spec32, inner32, si, mi):
    """per-degree complex mixing MI[m][l] = SI[l][m] W_l^T on the rows m <= l (the rows the triangular schedule computes)"""
    E, mm, lm = sh.E, sh.mmax, sh.lmax
    a_hi, a_lo = decode(si, mm, 2 * E, 2 * E // 64, lm, img_bytes(mm, 2 * E))   # [l, m, (ri, i)]
    g_hi, g_lo = decode(mi, lm, 2 * E, 2 * E // 64, mm, img_bytes(lm, 2 * E))   # [m, l, (ro, o)]
    f = np.zeros((lm, mm, 2 * E)); fb = np.zeros_like(f)
    for l in range(lm):
        R, S = data_gemm(a_hi[l], a_lo[l], mixing_matrix(spec32[l], inner32))
        f[l], fb[l] = gr.epi_affine(R, S)
    f, fb = f.transpose(1, 0, 2), fb.transpose(1, 0, 2)
    tri = np.arange(mm)[:, None] <= np.arange(lm)[None, :]
    return _split_checks("mixing", g_hi[tri], g_lo[tri], f[tri], fb[tri])


def inverse_legendre(sh: Shapes, tab, mi, Ho):
    """inverse Legendre per m of the decoded MI (every row, whatever the skipped tiles hold) -> [lat][(m, ro)][o]"""
    E, mm, lm = sh.E, sh.mmax, sh.lmax
    d_hi, d_lo = decode(mi, lm, 2 * E, 2 * E // 64, mm, img_bytes(lm, 2 * E))
    R, S = table_gemm(np.asarray(tab, np.float32), d_hi, d_lo)              # [m, lat, (ro, o)]
    f, fb = gr.epi_affine(R, S)
    perm = lambda a: a.reshape(mm, Ho, 2, E).transpose(1, 0, 2, 3).reshape(Ho, 2 * mm, E)
    return perm(f), perm(fb)


def stage_inverse_legendre(sh: Shapes, tab, mi, Ho, di):
    f, fb = inverse_legendre(sh, tab, mi, Ho)
    g_hi, g_lo = decode(di, 2 * sh.mmax, sh.E, sh.E // 64, Ho, img_bytes(2 * sh.mmax, sh.E))
    return _split_checks("inverse Legendre", g_hi, g_lo, f, fb)


def inverse_dft(sh: Shapes, tab, di, Ho, Wo):
    """inverse DFT per latitude of the decoded DI: (R, S) [(lat, lon), o]"""
    E = sh.E
    d_hi, d_lo = decode(di, 2 * sh.mmax, E, E // 64, Ho, img_bytes(2 * sh.mmax, E))
    R, S = table_gemm(np.asarray(tab, np.float32), d_hi, d_lo)              # [lat, lon, o]
    return R.reshape(Ho * Wo, E), S.reshape(Ho * Wo, E)


def stage_block_tail(sh: Shapes, w, i, taps, prev):
    """the block from the inverse DFT on: inverse DFT (+ inner skip) + GELU -> g image and norm1 statistics; norm1,
    fc1 bias, fc1 + GELU -> hidden image; fc2 + outer skip -> x (image, fp32, next norm0 statistics).
    taps: this block's engine taps; prev: the taps of the stage before (block input x / x_img)."""
    E, Hd = sh.E, sh.Hd
    Hi, Wi, Ho, Wo = sh.grids(i)
    Po, Pi = Ho * Wo, Hi * Wi
    p = f"blk{i}."
    big = Ho == sh.H1
    tabs = taps["_tables"]
    R, S = inverse_dft(sh, tabs["dft.inv_big" if big else "dft.inv_int"], taps["di"], Ho, Wo)
    n0 = np.asarray(taps["norm0"], np.float64)
    checks = []
    if Hi == Ho:
        f1 = taps["f1"].reshape(-1, E)[:Po].astype(np.float64)
        checks.append(("inverse DFT (f1)", f1, R, gr.TAU * S + 2 * gr.U32 * np.abs(R)))
        ib_ref, ib_b = fold_bias(w[p + "inner.w"], taps["norm0"][E:], w[p + "inner.b"])
        checks.append(("inner bias", taps["inner_bias"], ib_ref, ib_b))
        x_hi, x_lo = decode(prev["x_img"], Pi, E, E // 64)
        Wf = (np.asarray(w[p + "inner.w"], np.float32) * np.asarray(taps["norm0"][:E], np.float32)[None]).astype(np.float32)
        R2, S2 = data_gemm(x_hi, x_lo, Wf)
        g, gb = gr.epi_gelu(*gr.epi_affine(R2, S2, np.asarray(taps["inner_bias"], np.float64)[None], f1))
    else:
        g, gb = gr.epi_gelu(*gr.epi_affine(R, S, np.asarray(w[p + "inner.b"], np.float64)[None]))
    g_hi, g_lo = decode(taps["g_img"], Po, E, E // 64)
    checks += _split_checks("inverse DFT + skip + GELU (g)", g_hi, g_lo, g, gb)
    checks += _stats_checks("norm1 statistics", f64(taps["sums"]), g, gb)
    checks += stage_norm("norm1", sh, g_hi, g_lo, w[p + "norm1.g"], w[p + "norm1.b"], taps["norm1"])
    fb_ref, fb_b = fold_bias(w[p + "fc1.w"], taps["norm1"][E:], w[p + "fc1.b"])
    checks.append(("fc1 bias", taps["fc1_bias"], fb_ref, fb_b))
    W1 = (np.asarray(w[p + "fc1.w"], np.float32) * np.asarray(taps["norm1"][:E], np.float32)[None]).astype(np.float32)
    R, S = data_gemm(g_hi, g_lo, W1)
    h, hb = gr.epi_gelu(*gr.epi_affine(R, S, np.asarray(taps["fc1_bias"], np.float64)[None]))
    a_hi, a_lo = decode(taps["hidden_img"], Po, Hd, Hd // 64)
    checks += _split_checks("fc1 + GELU (hidden)", a_hi, a_lo, h, hb)
    R, S = data_gemm(a_hi, a_lo, w[p + "fc2.w"])
    bias = np.asarray(w[p + "fc2.b"], np.float64)
    if Hi == Ho:
        xin = prev["x"].reshape(-1, E)[:Pi].astype(np.float64)
        f, fb = gr.epi_affine(R, S, bias[None], n0[E:2 * E][None], xin * n0[:E][None])
    else:
        f, fb = gr.epi_affine(R, S, bias[None], taps["rpm"].reshape(-1, E)[:Po].astype(np.float64))
    x_hi, x_lo = decode(taps["x_img"], Po, E, E // 64)
    checks += _split_checks("fc2 + outer skip (x)", x_hi, x_lo, f, fb)
    if i + 1 < sh.L:
        checks.append(("fc2 + outer skip (x fp32)", taps["x"].reshape(-1, E)[:Po], f, fb))
        checks += _stats_checks("norm0 statistics", f64(taps["sums0"]), f - bias[None], fb)
    return checks


def stage_rpm(sh: Shapes, i, taps):
    """grid-changing block: the resampled residual iSHT(MI2) (inverse Legendre into DI', split, inverse DFT) -> fp32 Rpm;
    the bound carries DI''s rounding through the second GEMM"""
    E = sh.E
    Hi, Wi, Ho, Wo = sh.grids(i)
    big = Ho == sh.H1
    tabs = taps["_tables"]
    d, db = inverse_legendre(sh, tabs["sht.inv_big" if big else "sht.inv_int"], taps["mi2"], Ho)   # [lat, (m, ro), o]
    _, b_sum = gr.split_bound(d, db)
    T = np.asarray(tabs["dft.inv_big" if big else "dft.inv_int"], np.float64)                      # [lon, (m, ri)]
    R = T @ d
    bound = (2 * gr.TAU * k_scale(T.shape[1]) * (np.abs(T) @ (np.abs(d) + b_sum)) + np.abs(T) @ b_sum
             + 2.0 ** -21 * (np.abs(T) @ np.abs(d)) + 2 * gr.U32 * np.abs(R))
    got = taps["rpm"].reshape(-1, E)[:Ho * Wo]
    return [("resampled residual (rpm)", got, R.reshape(Ho * Wo, E), bound.reshape(Ho * Wo, E))]


def stage_block_spectral(sh: Shapes, w, i, taps, prev):
    """norm0, forward DFT, forward Legendre (and its inverse-layout copy), mixing, inverse Legendre of block i"""
    E = sh.E
    Hi, Wi, Ho, Wo = sh.grids(i)
    p = f"blk{i}."
    tabs = taps["_tables"]
    bi, bo = ("big" if Hi == sh.H1 else "int"), ("big" if Ho == sh.H1 else "int")
    x_hi, x_lo = decode(prev["x_img"], Hi * Wi, E, E // 64)
    checks = stage_norm("norm0", sh, x_hi, x_lo, w[p + "norm0.g"], w[p + "norm0.b"], taps["norm0"])
    checks += stage_dft(sh, tabs[f"dft.fwd_{bi}"], prev["x_img"], Hi, Wi, taps["norm0"], taps["li"])
    checks += stage_legendre(sh, tabs[f"sht.fwd_{bi}"], taps["li"], Hi, taps["si"], taps.get("mi2") if Hi != Ho else None)
    checks += stage_mixing(sh, w[p + "spec.w"], w[p + "inner.w"] if Hi != Ho else None, taps["si"], taps["mi"])
    checks += stage_inverse_legendre(sh, tabs[f"sht.inv_{bo}"], taps["mi"], Ho, taps["di"])
    if Hi != Ho:
        checks += stage_rpm(sh, i, taps)
    return checks


def stage_decoder(sh: Shapes, w, x_img, in_img, g_img, state):
    """decoder fc1 + GELU on [x | normalised input] (K-concatenated images), fc2 -> de-normalised state"""
    E, P, Cin = sh.E, sh.P1, sh.Cin
    x_hi, x_lo = decode(x_img, P, E, E // 64)
    i_hi, i_lo = decode(in_img, P, 128, 2)
    a_hi, a_lo = np.concatenate([x_hi, i_hi], 1), np.concatenate([x_lo, i_lo], 1)
    w1 = np.zeros((E, E + 128), np.float32); w1[:, :E + Cin] = w["dec.fc1.w"]
    R, S = data_gemm(a_hi, a_lo, w1)
    f, fb = gr.epi_gelu(*gr.epi_affine(R, S, np.asarray(w["dec.fc1.b"], np.float64)[None]))
    g_hi, g_lo = decode(g_img, P, E, E // 64)
    checks = _split_checks("decoder fc1 + GELU", g_hi, g_lo, f, fb)
    R, S = data_gemm(g_hi, g_lo, w["dec.fc2.w"])
    std = np.asarray(w["norm.std"], np.float64); mu = np.asarray(w["norm.mean"], np.float64)
    y = R + np.asarray(w["dec.fc2.b"], np.float64)[None]
    ref = y * std[None] + mu[None]
    bound = std[None] * (gr.TAU * S + 2 * gr.U32 * np.abs(y)) + 2 * gr.U32 * np.abs(ref)
    checks.append(("decoder fc2 (state)", np.asarray(state, np.float64).reshape(Cin, -1).T, ref, bound))
    return checks


# ---------------------------------------------------------------------------------------------------------------------
# report
# ---------------------------------------------------------------------------------------------------------------------
def evaluate(checks):
    """[(name, n_outside, worst ratio)] of a list of checks; NaN counts as outside"""
    out = []
    for name, got, ref, bound in checks:
        got = np.asarray(got, np.float64)
        ref = np.broadcast_to(np.asarray(ref, np.float64), got.shape)
        bound = np.broadcast_to(np.asarray(bound, np.float64), got.shape)
        n = int(gr.exceed(got, ref, bound).sum())
        if np.all(bound == 0):
            wr = 0.0 if n == 0 else math.inf
        else:
            wr = gr.worst(got, ref, bound)
        out.append((name, n, wr))
    return out
