"""The LayerNorm bound of oracle/gemm_ref.py against fp32 emulations of the GEMM epilogues' statistics, on rows whose
|mean| is up to 3000 times their standard deviation.

Every LayerNorm epilogue of the wgmma GEMM (gemm2.cuh) takes its row statistics in fp32 from values spread over threads:
  frag     FragEpi<Epi2F32Img<true, 2>> (Pangu's projection and fc2, and the fused MLP): a thread holds BN / 4 columns of
           a row (8 i + 2 (l & 3) + {0, 1}) and adds even and odd i in two chains, the lane quad merges by two xor
           shuffles, a CTA pair merges the two halves;
  staged   Epi2F32Img<true, kRes>::run (Pangu's fp32 stream, GraphCast's MLPs): the row's owner lane in each of the two
           warps of a lane quarter adds every other 32-column group, four columns at a time, in one pass about the mean
           of its first 32 columns; the warps merge through their patches, a CTA pair merges the two halves;
  shuffle  Epi2UpShuffle (Pangu's up-sample): one lane adds its whole row in sequence.
Each is emulated here value by value in numpy fp32 in the kernel's order, both as the epilogues compute now (each
thread's mean and sum of squared deviations from it; partials merged with Chan's formula) and as they computed before
(one pass over the sum and the sum of squares, var = ss / n - mean^2).  The bound must accept the first at every ratio of
|mean| / std from 0 to 3000, for gamma and beta drawn as the GPU tests draw them, and must reject the second from a ratio
of 100 on, where the one-pass variance has cancelled.  So the bound is checked without a GPU, before the GPU tests rely
on it.  pytest -s prints the worst err / bound of every path and ratio.
"""
from __future__ import annotations

import numpy as np
import pytest

from oracle import gemm_ref as gr

F32 = np.float32
EPS = 1e-5
RATIOS = [0, 1, 10, 30, 100, 300, 1000, 3000]
ROWS = 500   # per ratio


def fma(a, b, c):
    """fp32 fused multiply-add: the product is exact in fp64, one rounding to fp32 (double rounding aside)"""
    return (np.asarray(a, np.float64) * b + c).astype(F32)


def rsqrt(x):
    return (1.0 / np.sqrt(np.asarray(x, np.float64))).astype(F32)


def merge(a, na, b, nb):
    """gemm2.cuh ln_merge in fp32: (mean, m2) of na and nb columns"""
    n = F32(na + nb)
    d = b[0] - a[0]
    wa, wb, wab = F32(na) / n, F32(nb) / n, F32(na) * F32(nb) / n
    return (wa * a[0] + wb * b[0]).astype(F32), ((a[1] + b[1]) + (d * d) * wab).astype(F32)


def finish(y, stat, width, old, gamma, beta):
    """(sum, sum of squares) or (mean, m2) of the whole row -> fma(fma(y, rstd, -mean rstd), gamma, beta)"""
    if old:
        mean = (stat[0] / F32(width)).astype(F32)
        var = np.maximum((stat[1] / F32(width) - mean * mean).astype(F32), F32(0))
    else:
        mean, var = stat[0], (stat[1] / F32(width)).astype(F32)
    rs = rsqrt((var + F32(EPS)).astype(F32))
    ns = (-mean * rs).astype(F32)
    return fma(fma(y, rs[:, None], ns[:, None]), gamma, beta)


def frag_half(y, old):
    """statistics of one CTA's BN columns, merged over the lane quad (the same in all four lanes)"""
    bn = y.shape[1]
    lanes = []
    for l in range(4):
        v = y.reshape(-1, bn // 8, 8)[:, :, 2 * l: 2 * l + 2]
        s = np.zeros(len(y), F32); q = np.zeros(len(y), F32)
        if old:
            for i in range(bn // 8):
                s = (s + (v[:, i, 0] + v[:, i, 1])).astype(F32)
                q = (q + fma(v[:, i, 1], v[:, i, 1], v[:, i, 0] * v[:, i, 0])).astype(F32)
        else:   # two chains (even and odd 8-column groups) per pass
            a = [np.zeros(len(y), F32), np.zeros(len(y), F32)]
            for i in range(bn // 8):
                a[i & 1] = (a[i & 1] + (v[:, i, 0] + v[:, i, 1])).astype(F32)
            s = ((a[0] + a[1]).astype(F32) * F32(1 / (bn // 4))).astype(F32)
            a = [np.zeros(len(y), F32), np.zeros(len(y), F32)]
            for i in range(bn // 8):
                a0, a1 = (v[:, i, 0] - s).astype(F32), (v[:, i, 1] - s).astype(F32)
                a[i & 1] = (a[i & 1] + fma(a1, a1, a0 * a0)).astype(F32)
            q = (a[0] + a[1]).astype(F32)
        lanes.append((s, q))
    n = bn // 4
    for o in (1, 2):
        lanes = [(lanes[l][0] + lanes[l ^ o][0], lanes[l][1] + lanes[l ^ o][1]) if old else merge(lanes[l], n, lanes[l ^ o], n)
                 for l in range(4)]
        n *= 2
    return lanes[0]


def staged_half(y, old):
    """statistics of one CTA's BN columns: two warps of a lane quarter, every other 32-column group each"""
    bn = y.shape[1]
    ng = bn // 32
    parts = []
    for p in range(2):
        s = np.zeros(len(y), F32); q = np.zeros(len(y), F32)
        groups = range(p, ng, 2)
        for g in groups if old else ():
            v = y[:, 32 * g: 32 * g + 32]
            for j in range(0, 32, 4):
                s = (s + ((v[:, j] + v[:, j + 1]) + (v[:, j + 2] + v[:, j + 3]))).astype(F32)
                q = (q + (fma(v[:, j + 1], v[:, j + 1], v[:, j] * v[:, j]) + fma(v[:, j + 3], v[:, j + 3], v[:, j + 2] * v[:, j + 2]))).astype(F32)
        if not old:   # one pass about k, the mean of the lane's first 32 columns
            v = y[:, 32 * p: 32 * p + 32]
            k = np.zeros(len(y), F32)
            for j in range(0, 32, 4):
                k = (k + ((v[:, j] + v[:, j + 1]) + (v[:, j + 2] + v[:, j + 3]))).astype(F32)
            k = (k * F32(1 / 32)).astype(F32)
            for g in groups:
                d = (y[:, 32 * g: 32 * g + 32] - k[:, None]).astype(F32)
                for j in range(0, 32, 4):
                    s = (s + ((d[:, j] + d[:, j + 1]) + (d[:, j + 2] + d[:, j + 3]))).astype(F32)
                    q = (q + (fma(d[:, j + 1], d[:, j + 1], d[:, j] * d[:, j]) + fma(d[:, j + 3], d[:, j + 3], d[:, j + 2] * d[:, j + 2]))).astype(F32)
            dm = (s / F32(32 * len(groups))).astype(F32)
            s, q = (k + dm).astype(F32), np.maximum((q - s * dm).astype(F32), F32(0))
        parts.append(((s, q), 32 * len(groups)))
    if old:
        return parts[0][0][0] + parts[1][0][0], parts[0][0][1] + parts[1][0][1]
    return merge(parts[0][0], parts[0][1], parts[1][0], parts[1][1])


def emulate(path, y, bn, pair, old, gamma, beta):
    """the epilogue's fp32 output LN(y) * gamma + beta for rows y [R, width]"""
    if path == "shuffle":
        s = np.zeros(len(y), F32); q = np.zeros(len(y), F32)
        for j in range(y.shape[1]):
            s = (s + y[:, j]).astype(F32)
            if old:
                q = fma(y[:, j], y[:, j], q)
        if not old:
            s = (s / F32(y.shape[1])).astype(F32)
            for j in range(y.shape[1]):
                d = (y[:, j] - s).astype(F32)
                q = fma(d, d, q)
        return finish(y, (s, q), y.shape[1], old, gamma, beta)
    half = frag_half if path == "frag" else staged_half
    st = half(y[:, :bn], old)
    if pair:
        pst = half(y[:, bn:], old)
        st = (st[0] + pst[0], st[1] + pst[1]) if old else merge(st, bn, pst, bn)
    return finish(y, st, y.shape[1], old, gamma, beta)


def depth(path, bn, pair):
    """gemm_ref.ln_depth of each path"""
    if path == "frag":
        return gr.ln_depth(bn // 16 + 2, 2 + pair)
    if path == "staged":
        return gr.ln_depth(bn // 8 + 2, 1 + pair)
    return gr.ln_depth(bn, 0)


def rows(width: int, seed: int):
    """ROWS rows per ratio: mean = ratio * sd (either sign), sd log-uniform in [0.1, 10], N(0, 1) shape; fp32"""
    rng = np.random.default_rng(seed)
    ratio = np.repeat(np.asarray(RATIOS, np.float64), ROWS)
    sd = np.exp(rng.uniform(np.log(0.1), np.log(10.0), len(ratio)))
    sign = rng.choice([-1.0, 1.0], len(ratio))
    y = (sign * ratio * sd)[:, None] + sd[:, None] * rng.standard_normal((len(ratio), width))
    return y.astype(F32), ratio


PATHS = [("frag", 192, False), ("frag", 192, True), ("staged", 192, False), ("staged", 192, True), ("staged", 256, True),
         ("shuffle", 192, False)]


@pytest.mark.parametrize("path,bn,pair", PATHS)
def test_bound_accepts_statistics_about_the_mean_and_rejects_one_pass(path, bn, pair):
    width = bn * (2 if pair else 1)
    y, ratio = rows(width, bn + 7 * pair + len(path))
    rng = np.random.default_rng(width)
    gamma = (rng.uniform(-1.0, 1.0, width) + 1.0).astype(F32)
    beta = rng.uniform(-0.1, 0.1, width).astype(F32)
    ref, bound = gr.layer_norm(y.astype(np.float64), 0.0, 0.0, gamma[None, :].astype(np.float64), beta[None, :].astype(np.float64),
                               0.0, EPS, depth=depth(path, bn, pair), shift=gr.ln_shift(bn) if path == "staged" else None)
    line = []
    for old in (False, True):
        out = emulate(path, y, bn, pair, old, gamma[None, :], beta[None, :])
        for r in RATIOS:
            m = ratio == r
            w = gr.worst(out[m], ref[m], bound[m])
            line.append(f"{'one-pass' if old else 'about the mean'}@{r}: {w:.3g}")
            if not old:
                assert w <= 1.0, f"{path} bn={bn} pair={pair}: statistics about the mean exceed the bound by {w:.3g}x at ratio {r}"
            elif r >= 100:
                assert w > 1.0, f"{path} bn={bn} pair={pair}: the bound accepts one-pass statistics at ratio {r} ({w:.3g})"
    print(f"[ln offsets] {path} bn={bn} pair={pair} depth={depth(path, bn, pair)}: " + ", ".join(line))


def test_merge_is_symmetric_and_exact_in_fp64():
    """Chan's merge: the same bits in either order (both CTAs of a pair, all lanes of a quad agree), and in fp64 the
    statistics of the whole row"""
    rng = np.random.default_rng(3)
    a, b = rng.standard_normal((64, 48)) + 1000.0, rng.standard_normal((64, 144)) + 1000.0
    sa = (a.mean(1).astype(F32), (a.var(1) * 48).astype(F32))
    sb = (b.mean(1).astype(F32), (b.var(1) * 144).astype(F32))
    ab, ba = merge(sa, 48, sb, 144), merge(sb, 144, sa, 48)
    assert np.array_equal(ab[0], ba[0]) and np.array_equal(ab[1], ba[1])
    n = 192.0
    d = b.mean(1) - a.mean(1)
    m2 = a.var(1) * 48 + b.var(1) * 144 + d * d * 48 * 144 / n
    whole = np.concatenate([a, b], 1)
    np.testing.assert_allclose(m2, whole.var(1) * n, rtol=1e-12)
    np.testing.assert_allclose((48 * a.mean(1) + 144 * b.mean(1)) / n, whole.mean(1), rtol=1e-15)
