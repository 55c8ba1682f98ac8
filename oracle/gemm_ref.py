"""ORACLE — test infrastructure, not product code.

Layouts and float64 references of the wgmma GEMM (skyrim_b200/csrc/gemm2.cuh, gemm_tb.cuh) at kernel level, for
tests/test_gemm_kernels_gpu.py (which launches the kernel through libskyrim_b200_probe.so) and
tests/test_gemm_probe_cpu.py (which checks this module on its own).

Layouts.  Every operand the kernel reads is a SWIZZLE_128B fp16 tile image: tiles of T rows x 64 halves (128 bytes per
row), the 16-byte chunk k of row r stored at position k ^ (r & 7).  Packing here is written from that one sentence,
independently of the CUDA packers (k_pack_img, k_pack_w3), so a layout error on either side shows as a mismatch:
  A image     [ceil(M/128)][nkb][128 rows x 128 B]             pack_tiles(a, 128, nkb)
  W image     [N/BN][nkb][BN rows x 128 B], per batch           pack_tiles(w, BN, nkb); with w_rep: [hi | lo] along K
  TB table    [M/128][hi | lo][128 rows x 128 B]                a W image with BN = 128
  TB data     rows = contraction index, 64 channels per chunk row: an A image of X[k, n]

References are float64 and start from the exact fp16 values the kernel reads.  Bounds are per element, never norms:
the linear part |D - R| <= tau * sum_k |a_k w_k|; a nonlinear epilogue adds its Lipschitz factor and, for every fp16
output, half an fp16 ulp of the reference.
"""
from __future__ import annotations

import numpy as np
import scipy.special as sp

# fp32-accumulation bound of the tensor-core GEMM relative to sum_k |a_k w_k|: 32 x 2^-23.  Largest measured ratio
# |D - R| / (2^-23 sum_k |a_k w_k|) on an H100 80GB HBM3 at 700 W: 7.0 (3-term split), 3.1 (single fp16 products); the
# per-case figures are in tests/test_gemm_kernels_gpu.py
TAU = 2.0 ** -18
U32 = 2.0 ** -24          # fp32 unit roundoff
GELU_LIP = 1.13           # max |gelu'(x)| = 1.1289
GELU_ABS = 1.0e-5         # the kernel's polynomial erf-GELU: max abs error 0.61 * 1.2e-5 (sky_common.cuh)
SUB16 = 2.0 ** -25        # half the smallest fp16 subnormal


# ---------------------------------------------------------------------------------------------------------------------
# layouts
# ---------------------------------------------------------------------------------------------------------------------
def _swz_index(rows) -> np.ndarray:
    """[R, 8] for the row numbers ``rows`` (an int T: rows 0 .. T - 1): stored chunk p of row r holds logical chunk
    p ^ (r & 7) (and vice versa: XOR is an involution)."""
    r = np.arange(rows) if np.isscalar(rows) else np.asarray(rows)
    return np.arange(8)[None, :] ^ (r[:, None] & 7)


def pack_tiles(x: np.ndarray, tile_rows: int, nkb: int, row_fill=0.0, col_fill=0.0, rows_pad: int | None = None) -> np.ndarray:
    """fp16 matrix [R, K] -> image bytes [ceil(R/T)][nkb][T rows x 128 B].  Rows >= R are `row_fill`, columns >= K of
    the valid rows `col_fill` (NaN rows of an A image show any leak; the K padding must stay finite, it meets zeros)."""
    x = np.asarray(x, dtype=np.float16)
    R, K = x.shape
    assert K <= nkb * 64 and tile_rows % 8 == 0
    nt = -(-max(R, rows_pad or 0) // tile_rows)
    buf = np.full((nt * tile_rows, nkb * 64), col_fill, dtype=np.float16)
    buf[R:] = row_fill
    buf[:R, :K] = x
    v = buf.reshape(nt, tile_rows, nkb, 8, 8).transpose(0, 2, 1, 3, 4)      # [tile][kb][row][chunk][8]
    idx = np.broadcast_to(_swz_index(tile_rows)[None, None, :, :, None], v.shape)
    return np.ascontiguousarray(np.take_along_axis(v, idx, axis=3)).reshape(-1).view(np.uint8)


def unpack_tiles(img: np.ndarray, tile_rows: int, nkb: int, rows: int, cols: int | None = None) -> np.ndarray:
    """inverse of pack_tiles: image bytes -> fp16 [rows, cols]"""
    h = np.asarray(img).reshape(-1).view(np.float16)
    nt = h.size // (tile_rows * nkb * 64)
    v = h[: nt * tile_rows * nkb * 64].reshape(nt, nkb, tile_rows, 8, 8)
    idx = np.broadcast_to(_swz_index(tile_rows)[None, None, :, :, None], v.shape)
    x = np.take_along_axis(v, idx, axis=3).transpose(0, 2, 1, 3, 4).reshape(nt * tile_rows, nkb * 64)
    return x[:rows, : (cols if cols is not None else nkb * 64)]


def unpack_rows(pieces: np.ndarray, rows) -> np.ndarray:
    """gathered rows of a tile image -> fp16 [n, nkb * 64].  pieces: [n, nkb, 128 B], piece kb of row r taken from byte
    img_offset(r, 64 kb, nkb); the rows' own numbers undo the swizzle"""
    pieces = np.ascontiguousarray(pieces)
    if len(rows) == 0:
        return np.zeros((0, pieces.shape[1] * 64), np.float16)
    h = pieces.view(np.float16).reshape(len(rows), -1, 8, 8)
    idx = np.broadcast_to(_swz_index(rows)[:, None, :, None], h.shape)
    return np.take_along_axis(h, idx, axis=2).reshape(len(rows), -1)


def img_offset(row: int, col: int, nkb: int, tile_rows: int = 128) -> int:
    """byte offset of element (row, col) in a tile image (gemm2.cuh img_offset, for T = 128)"""
    t, r = divmod(row, tile_rows)
    return (t * nkb + col // 64) * tile_rows * 128 + r * 128 + ((((col % 64) // 8) ^ (r & 7)) << 4) + (col % 8) * 2


def pack_w(w: np.ndarray, bn: int, nkb: int) -> np.ndarray:
    """weights [N, K] fp16 -> [N/BN][nkb][BN x 128 B]"""
    assert w.shape[0] % bn == 0
    return pack_tiles(w, bn, nkb)


def pack_w_split(w_hi: np.ndarray, w_lo: np.ndarray, bn: int, nkb: int) -> np.ndarray:
    """3-term weights: [N/BN][hi: nkb | lo: nkb][BN x 128 B] (read hi, hi, lo against A = [hi | lo | hi])"""
    K = w_hi.shape[1]
    pad = np.zeros((w_hi.shape[0], nkb * 64 - K), np.float16)
    return pack_w(np.concatenate([w_hi, pad, w_lo, pad], axis=1), bn, 2 * nkb)


def split16(x: np.ndarray):
    """fp32/fp64 -> (hi, lo) fp16 with hi = rn(x), lo = rn(x - hi) (computed in fp32, as the kernels do)"""
    x = np.asarray(x, np.float32)
    hi = x.astype(np.float16)
    lo = (x - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def ulp16(x: np.ndarray) -> np.ndarray:
    """one fp16 ulp at |x| (subnormal spacing below 2^-14)"""
    a = np.maximum(np.abs(np.asarray(x, np.float64)), 2.0 ** -14)
    return 2.0 ** (np.floor(np.log2(a)) - 10)


# ---------------------------------------------------------------------------------------------------------------------
# linear part
# ---------------------------------------------------------------------------------------------------------------------
def linear(pairs) -> tuple[np.ndarray, np.ndarray]:
    """sum over (A_s [M, K_s], W_s [N, K_s]) of A_s W_s^T in float64, and sum_k |a_k w_k| (the scale of the bound)"""
    R = S = 0.0
    for a, w in pairs:
        a = np.asarray(a, np.float64)
        w = np.asarray(w, np.float64)
        R = R + a @ w.T
        S = S + np.abs(a) @ np.abs(w).T
    return R, S


def linear_naive(pairs) -> tuple[np.ndarray, np.ndarray]:
    """the same by explicit loops (tests of the vectorised version only)"""
    a0, w0 = pairs[0]
    M, N = a0.shape[0], w0.shape[0]
    R = np.zeros((M, N)); S = np.zeros((M, N))
    for a, w in pairs:
        for i in range(M):
            for j in range(N):
                for k in range(a.shape[1]):
                    p = float(a[i, k]) * float(w[j, k])
                    R[i, j] += p; S[i, j] += abs(p)
    return R, S


def split_pairs(a_hi, a_lo, w_hi, w_lo):
    """the 3-term product the kernel forms: hi*hi + lo*hi + hi*lo"""
    return [(a_hi, w_hi), (a_lo, w_hi), (a_hi, w_lo)]


# ---------------------------------------------------------------------------------------------------------------------
# epilogues: each returns (reference, bound) per element
# ---------------------------------------------------------------------------------------------------------------------
def gelu(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, np.float64)
    return 0.5 * x * (1.0 + sp.erf(x / np.sqrt(2.0)))


def epi_affine(R, S, *terms, tau=TAU):
    """acc + sum(terms) in fp32 (bias, addend, previous value): tau * S plus a few fp32 roundings of the magnitudes"""
    ref = R + sum(np.asarray(t, np.float64) for t in terms)
    mag = np.abs(R) + sum(np.abs(np.asarray(t, np.float64)) for t in terms)
    return ref, tau * S + 4 * U32 * mag


def epi_gelu(x_ref, x_bound):
    g = gelu(x_ref)
    return g, GELU_LIP * x_bound + GELU_ABS + 4 * U32 * np.abs(g)


SILU_LIP = 1.1                       # max |silu'(x)| = 1.0998
SILU_REL = 2.0 ** -20                # the kernel's silu: ex2.approx and rcp.approx


def silu(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, np.float64)
    return x * sp.expit(x)


def epi_silu(x_ref, x_bound):
    s = silu(x_ref)
    return s, SILU_LIP * x_bound + SILU_REL * (np.abs(s) + np.abs(x_ref)) + 1e-30


def f16_bound(ref, bound):
    """bound of an fp16 store of a value within `bound` of `ref`: half an fp16 ulp on top"""
    return bound + 0.5 * ulp16(np.abs(ref) + bound)


def split_bound(ref, bound):
    """bounds of the hi / lo pair written for a value within `bound` of `ref`: hi alone (half an fp16 ulp) and hi + lo
    (22 bits: lo's own rounding is at most 2^-12 of |x - hi| <= 2^-23 |x|, plus subnormal underflow)"""
    b_hi = bound + 0.5 * ulp16(np.abs(ref) + bound)
    b_sum = bound + 2.0 ** -22 * np.abs(ref) + SUB16
    return b_hi, b_sum


def col_stats(f_ref, f_bound, rows_per_sum: int = 32):
    """per-column sum and sum of squares of f (rows x cols) with bounds: the element bounds add up, plus the kernel's fp32
    partial sums (32 rows per fp32 sum before the fp64 accumulation)"""
    f = np.asarray(f_ref, np.float64); b = np.asarray(f_bound, np.float64)
    s = f.sum(0); q = (f * f).sum(0)
    bs = b.sum(0) + rows_per_sum * 2 * U32 * np.abs(f).sum(0)
    bq = (2 * np.abs(f) * b + b * b).sum(0) + rows_per_sum * 2 * U32 * (f * f).sum(0)
    return s, q, bs, bq


def ln_depth(chain: int, merges: int) -> int:
    """fp32 roundings a LayerNorm row mean passes through in a kernel (first order, a value's error is u |value| per
    addition its partial sum passes through): `chain`, the most additions any one value meets in a thread's sum, two per
    merge of partial statistics (ln_merge: weighted means and their sum), one for the division and one for the product
    mean * rstd that the normalisation adds.  The paths of gemm2.cuh, BN columns per CTA:
      FragEpi<Epi2F32Img>   chain BN / 16 + 2 (pairs of columns onto two running sums), merges 2 (lane quad) + 1 in a pair
      Epi2F32Img::run       chain BN / 8 + 2 (four-column trees onto a running sum, every other 32-column group),
                            merges 1 (the two warps of a lane quarter) + 1 in a pair
      Epi2UpShuffle         chain BN (one lane adds its row in sequence), no merge"""
    return chain + 2 * merges + 2


def ln_shift(bn: int) -> tuple[int, int]:
    """Epi2F32Img::run's one pass (the `shift` of layer_norm): each lane sums its BN / 2 columns about the mean of its
    first 32"""
    return 32, bn // 2


def layer_norm(R, S, bias, gamma, beta, res, eps, tau=TAU, depth=None, shift=None):
    """Epi2F32Img<true, kRes> (Pangu's and GraphCast's LayerNorm epilogue) and Epi2UpShuffle: out = LN(acc + bias) * gamma
    + beta + res over whole rows, with its bound; res = 0 for kRes 0.

    The kernels take the statistics of a thread's m columns about their mean, as (mean, m2 = sum of squared deviations),
    and merge partials of disjoint columns with Chan's formula (gemm2.cuh ln_merge).  A thread either makes two passes
    (shift None: the mean, then the squared deviations from it) or one pass about k, the mean of its first q columns
    (shift = (q, m), ln_shift: mean = k + s / m, m2 = ss - s^2 / m with s, ss the sums of y - k and its square).
    First order in u = 2^-24, with e the error of each y = acc + bias (tau S and its fp32 roundings), n the row width,
    sd its standard deviation, and `depth` the roundings of a thread's sum (ln_depth; default n + 2, more than any path):
      mean  the propagated e.mean() and the summation error dsum.  Two passes: depth u mean|y|, linear in the row's
            |mean|.  One pass: (k - mean_t)^2 <= m2_t / q for the thread's columns (their first q deviate by k - mean_t
            on average) and m2_t <= m2, so mean|y - k| <= (1 + sqrt(m / q)) sqrt(n / m) sd, and dsum = depth u (1 +
            sqrt(m / q)) sqrt(n / m) sd + 10 u |mean| (k + s / m, two per merge, the product mean * rstd);
      var   sum (y_i - mu')^2 = n var + n (mu - mu')^2 exactly, so the mean's error enters a thread's m2 only to second
            order (dsum^2); a merge's d^2 na nb / n term carries the local means' summation error to first order, at
            most 2 sqrt(m2 n / 4) dsum <= n sd dsum per level of the merge tree, 4 levels at most (quad, lane quarter,
            pair); the propagated 2 |y - mu| e; the roundings of the positive sum of squares and its division, depth + 4
            of them (two passes), or 3 depth + 3 of the sum about k, which is at most 1 + m / q times m2 (one pass);
      rstd  rsqrtf within 2 ulp: 2^-21 on top of half the variance's relative error.
    """
    y = R + bias
    e = tau * S + 2 * U32 * np.abs(y)
    n = y.shape[1]
    depth = n + 2 if depth is None else depth
    mu = y.mean(1, keepdims=True)
    var = y.var(1, keepdims=True)
    sd = np.sqrt(var)
    rstd = 1.0 / np.sqrt(var + eps)
    yn = (y - mu) * rstd
    out = yn * gamma + beta + res
    if shift is None:
        dsum = depth * U32 * np.abs(y).mean(1, keepdims=True)
        rounding = depth + 4
    else:
        q, m = shift
        dsum = U32 * (10 * np.abs(mu) + depth * (1 + np.sqrt(m / q)) * np.sqrt(n / m) * sd)
        rounding = (3 * depth + 3) * (1 + m / q)
    e_mu = e.mean(1, keepdims=True) + dsum
    rel_var = (2 * (np.abs(y - mu) * e).mean(1, keepdims=True) + 4 * dsum * sd + dsum * dsum + rounding * U32 * var) / (var + eps)
    bound = (np.abs(gamma) * rstd * (e + e_mu) + np.abs(gamma * yn) * (0.5 * rel_var + 2.0 ** -21)
             + 4 * U32 * (np.abs(gamma * yn) + np.abs(beta) + np.abs(res)))
    return out, bound


def remap_dest(b, r, c, *, bdiv, kmul, kdiv, rb, same):
    """EpiSplitRemap: source (batch b, row r, column c) -> destination (batch', row', k')"""
    if same:
        return b, r, c
    return r // bdiv, b * rb + c // kdiv, (r % bdiv) * kmul + c % kdiv


# ---------------------------------------------------------------------------------------------------------------------
# comparison
# ---------------------------------------------------------------------------------------------------------------------
def exceed(got, ref, bound) -> np.ndarray:
    """mask of elements outside their bound (NaN counts as outside)"""
    got = np.asarray(got, np.float64)
    return ~(np.abs(got - ref) <= bound)


def worst(got, ref, bound) -> float:
    """largest |got - ref| / bound (inf when a NaN is present)"""
    got = np.asarray(got, np.float64)
    d = np.abs(got - ref)
    if not np.all(np.isfinite(d)):
        return float("inf")
    return float((d / np.maximum(bound, 1e-300)).max()) if d.size else 0.0
