"""CPU checks of the kernel-level GEMM test machinery (oracle/gemm_ref.py, oracle/gemm_probe.py): the layouts, the
float64 references, that the comparator at the chosen TAU catches the errors a tiled kernel makes, and that the probe
refuses inconsistent cases on the host (without touching a device)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from oracle import gemm_probe as gp
from oracle import gemm_ref as gr


@pytest.mark.parametrize("tile_rows,nkb,R,K", [(128, 1, 1, 5), (128, 3, 129, 150), (16, 2, 48, 128), (80, 2, 160, 100),
                                               (240, 1, 240, 64), (384, 2, 384, 128)])
def test_pack_unpack_identity(tile_rows, nkb, R, K):
    rng = np.random.default_rng(R + K)
    x = rng.standard_normal((R, K)).astype(np.float16)
    img = gr.pack_tiles(x, tile_rows, nkb)
    assert img.size == -(-R // tile_rows) * tile_rows * nkb * 128
    back = gr.unpack_tiles(img, tile_rows, nkb, R, K)
    assert np.array_equal(back.view(np.uint16), x.view(np.uint16))


def test_hand_computed_offsets():
    """one element per layout, its byte offset worked out by hand from row*128 + ((chunk ^ (row & 7)) << 4)"""
    # A image, nkb = 3: element (row 130, col 77) -> tile 1, k-block 1, row 2, chunk 1 (stored at 1 ^ 2 = 3), half 5
    x = np.zeros((200, 192), np.float16); x[130, 77] = 1.0
    img = gr.pack_tiles(x, 128, 3).view(np.float16)
    off = (1 * 3 + 1) * 16384 + 2 * 128 + (3 << 4) + 5 * 2
    assert off == gr.img_offset(130, 77, 3)
    assert np.flatnonzero(img) .tolist() == [off // 2]
    # W image, BN = 80, nkb = 2: weight (n 87, k 70) -> n-tile 1, k-block 1, row 7, chunk 0 (stored at 7), half 6
    w = np.zeros((160, 128), np.float16); w[87, 70] = 1.0
    img = gr.pack_w(w, 80, 2).view(np.float16)
    off = (1 * 2 + 1) * 80 * 128 + 7 * 128 + (7 << 4) + 6 * 2
    assert np.flatnonzero(img).tolist() == [off // 2]
    # 3-term W image [hi | lo], BN = 64, nkb = 1: lo of (n 9, k 17) -> n-tile 0, k-block 1 (the lo half), row 9, chunk 2
    # (stored at 2 ^ 1 = 3), half 1
    hi = np.zeros((64, 64), np.float16); lo = np.zeros((64, 64), np.float16); lo[9, 17] = 1.0
    img = gr.pack_w_split(hi, lo, 64, 1).view(np.float16)
    off = 1 * 64 * 128 + 9 * 128 + (3 << 4) + 1 * 2
    assert np.flatnonzero(img).tolist() == [off // 2]
    # table x data: data row 200 (contraction index), channel 130 of an image with 3 column blocks -> tile 1, block 2,
    # row 72, chunk 0 (stored at 0 ^ 0 = 0), half 2
    d = np.zeros((256, 192), np.float16); d[200, 130] = 1.0
    img = gr.pack_tiles(d, 128, 3).view(np.float16)
    off = (1 * 3 + 2) * 16384 + 72 * 128 + 0 + 2 * 2
    assert np.flatnonzero(img).tolist() == [off // 2]


def test_padding_fill():
    x = np.ones((130, 60), np.float16)
    v = gr.unpack_tiles(gr.pack_tiles(x, 128, 1, row_fill=np.nan, col_fill=0.0), 128, 1, 256)
    assert np.isnan(v[130:]).all() and (v[:130, 60:] == 0).all() and (v[:130, :60] == 1).all()


def test_linear_matches_loops():
    rng = np.random.default_rng(1)
    a_hi, a_lo = gr.split16(rng.standard_normal((5, 9)))
    w_hi, w_lo = gr.split16(rng.standard_normal((4, 9)))
    pairs = gr.split_pairs(a_hi, a_lo, w_hi, w_lo)
    R, S = gr.linear(pairs)
    Rn, Sn = gr.linear_naive(pairs)
    np.testing.assert_allclose(R, Rn, rtol=1e-14, atol=1e-14)
    np.testing.assert_allclose(S, Sn, rtol=1e-14)


def test_split_and_gelu_and_remap_match_scalar_definitions():
    import math
    rng = np.random.default_rng(2)
    x = rng.standard_normal(50).astype(np.float32) * 3
    hi, lo = gr.split16(x)
    for v, h, l in zip(x, hi, lo):
        assert h == np.float16(v) and l == np.float16(np.float32(v) - np.float32(h))
    g = gr.gelu(x)
    for v, gv in zip(x, g):
        assert abs(gv - 0.5 * float(v) * (1 + math.erf(float(v) / math.sqrt(2)))) < 1e-15
    # EpiSplitRemap's forward-DFT map: (lat b, row (m, ri), channel c) -> (m, lat, ri * E + c)
    assert gr.remap_dest(3, 5, 7, bdiv=2, kmul=64, kdiv=1 << 30, rb=1, same=0) == (2, 3, 64 + 7)
    # inverse Legendre: (m b, lat r, (ro, o) c) -> (lat, 2 m + ro, o)
    assert gr.remap_dest(4, 9, 70, bdiv=1, kmul=0, kdiv=64, rb=2, same=0) == (9, 9, 6)


def test_layer_norm_and_stats_match_loops():
    rng = np.random.default_rng(3)
    R = rng.standard_normal((3, 8)); S = np.abs(R) * 2
    b, g, be, res = rng.standard_normal(8), rng.standard_normal(8), rng.standard_normal(8), rng.standard_normal((3, 8))
    out, _ = gr.layer_norm(R, S, b, g, be, res, 1e-5)
    for i in range(3):
        y = R[i] + b
        mu = sum(y) / 8
        var = sum((v - mu) ** 2 for v in y) / 8
        ref = [(y[j] - mu) / np.sqrt(var + 1e-5) * g[j] + be[j] + res[i, j] for j in range(8)]
        np.testing.assert_allclose(out[i], ref, rtol=1e-12)
    s, q, _, _ = gr.col_stats(R, S)
    np.testing.assert_allclose(s, [sum(R[:, j]) for j in range(8)], rtol=1e-14)
    np.testing.assert_allclose(q, [sum(R[:, j] ** 2) for j in range(8)], rtol=1e-14)


# ---------------------------------------------------------------------------------------------------------------------
# sensitivity: each deliberate error below must be flagged by the comparator at TAU
# ---------------------------------------------------------------------------------------------------------------------
def _w3_case(M=129, N=192, K=384, seed=0):
    rng = np.random.default_rng(seed)
    a_hi, a_lo = gr.split16(rng.uniform(-1, 1, (M, K)))
    w_hi, w_lo = gr.split16(rng.uniform(-1, 1, (N, K)) / np.sqrt(K))
    R, S = gr.linear(gr.split_pairs(a_hi, a_lo, w_hi, w_lo))
    return a_hi, a_lo, w_hi, w_lo, R, S


def _flagged(got, R, S):
    ref, bound = gr.epi_affine(R, S)
    return gr.exceed(got, ref, bound).any()


def test_exact_result_passes():
    *_, R, S = _w3_case()
    ref, bound = gr.epi_affine(R, S)
    # an fp32 result of the exact value is within the bound
    assert not _flagged(R.astype(np.float32), R, S)


def test_flags_dropped_k_block():
    a_hi, a_lo, w_hi, w_lo, R, S = _w3_case()
    sl = slice(128, 192)
    drop = [(a_hi[:, sl], w_hi[:, sl])]
    Rd = R - gr.linear(drop)[0]
    assert _flagged(Rd.astype(np.float32), R, S)


def test_flags_hi_lo_swap_in_one_k_block():
    a_hi, a_lo, w_hi, w_lo, R, S = _w3_case()
    sl = slice(64, 128)
    # in k-block 1, the lo term reads the weights' lo against A lo instead of hi against lo (and vice versa)
    Rs = R - gr.linear([(a_lo[:, sl], w_hi[:, sl]), (a_hi[:, sl], w_lo[:, sl])])[0] \
           + gr.linear([(a_hi[:, sl], w_lo[:, sl]), (a_lo[:, sl], w_lo[:, sl])])[0]
    assert _flagged(Rs.astype(np.float32), R, S)


def test_flags_row_shift():
    *_, R, S = _w3_case()
    Rs = R.copy(); Rs[40] = R[41]
    assert _flagged(Rs.astype(np.float32), R, S)


def test_flags_neighbouring_n_tile():
    *_, R, S = _w3_case(N=240)
    bn = 80
    Rs = R.copy(); Rs[:, bn:2 * bn] = R[:, 2 * bn:3 * bn]   # n-tile 1 written with n-tile 2's columns
    assert _flagged(Rs.astype(np.float32), R, S)


def test_flags_missing_triangular_element():
    """the off-by-one skip (>= for >) drops order m = 128 of degree l = 128: one missing element of the mixing output"""
    rng = np.random.default_rng(4)
    L, M, N, K = 130, 130, 64, 64
    a_hi, a_lo = gr.split16(rng.uniform(-1, 1, (L, M, K)))
    w_hi, w_lo = gr.split16(rng.uniform(-1, 1, (L, N, K)) / 8)
    R = np.empty((L, M, N)); S = np.empty((L, M, N))
    for l in range(L):
        R[l], S[l] = gr.linear(gr.split_pairs(a_hi[l], a_lo[l], w_hi[l], w_lo[l]))
    ref, bound = gr.epi_affine(R, S)
    b_hi, b_sum = gr.split_bound(ref, bound)
    hi, lo = gr.split16(R)
    got = hi.astype(np.float64) + lo
    assert not gr.exceed(got, ref, b_sum).any()
    # the skipped tile keeps the sentinel (NaN) at (l = 128, m = 128), which the bounded comparison flags
    got[128, 128] = np.nan
    bad = np.argwhere(gr.exceed(got, ref, b_sum))
    assert bad.shape[0] == N and (bad[:, :2] == [128, 128]).all()


def test_split_bound_flags_one_bit_of_lo():
    """the hi + lo check itself resolves 22 bits: for a value known to fp32 rounding, a lo off by a few of its ulps in one
    element is caught"""
    rng = np.random.default_rng(5)
    R = rng.uniform(-2, 2, 1000)
    b = gr.U32 * np.abs(R)
    hi, lo = gr.split16(R)
    _, b_sum = gr.split_bound(R, b)
    got = hi.astype(np.float64) + lo
    assert not gr.exceed(got, R, b_sum).any()
    lo2 = lo.copy(); lo2[7] = np.float16(lo[7]) + np.float16(np.abs(R[7]) * 2.0 ** -18)
    assert gr.exceed(hi.astype(np.float64) + lo2, R, b_sum)[7]


# ---------------------------------------------------------------------------------------------------------------------
# probe library: ABI mirror and host-side refusals (no device needed: validation precedes any CUDA call)
# ---------------------------------------------------------------------------------------------------------------------
def _probe():
    if not gp.PROBE_LIB_PATH.exists():
        pytest.fail(f"{gp.PROBE_LIB_PATH} is missing: __graft_entry__.build() builds it")
    return gp.lib()


def test_case_struct_matches_library():
    assert _probe().sky_probe_case_size() == C.sizeof(gp.Case)


def _good_w_case(**over):
    kw = dict(kernel=gp.W, epi=gp.EPI_F32, block_n=64, n=128, n_valid=128, batches=1, grid_sms=0, nseg=1, m=129,
              a=[0x10000], a_bytes=[2 * 2 * 16384], a_batch_stride=[0], a_nkb=[2], w=0x20000, w_bytes=2 * 2 * 64 * 128,
              num_kb=2, out=0x30000, out_bytes=129 * 128 * 4, ldo=128)
    kw.update(over)
    return gp.make_case(**kw)


@pytest.mark.parametrize("over,msg", [
    (dict(n=96), "shape"),                                               # N % BN
    (dict(num_kb=3), "k-blocks"),                                        # A holds 2 k-blocks
    (dict(nseg=7), "segments"),
    (dict(a_bytes=[2 * 2 * 16384 - 16]), "A segment 0 image too small"),
    (dict(w_bytes=100), "W image too small"),
    (dict(out_bytes=129 * 128 * 4 - 4), "fp32 output too small"),
    (dict(kernel=gp.PAIR, epi=gp.EPI_LN, block_n=192, n=192, n_valid=192, w_bytes=1 << 20), "pair"),
    (dict(block_n=48, n=96, n_valid=96, w_bytes=1 << 20), "not instantiated"),
    (dict(n_valid=126), "fp32 output layout"),
])
def test_probe_refuses_inconsistent_cases(over, msg):
    rc, err = gp.launch(_good_w_case(**over))
    assert rc != 0 and msg in err, (rc, err)


def test_probe_refuses_inconsistent_tb_cases():
    base = dict(kernel=gp.TB, epi=gp.EPI_F32, block_n=64, n=64, n_valid=64, batches=2, m=100, num_kb=6, t=0x10000,
                t_bytes=4 * 16384, t_rows=128, b_nkb_img=1, b_hi=0x20000, b_lo=0x30000, b_bytes=2 * 16384,
                b_rows_per_batch=64, out=0x40000, out_bytes=2 * 100 * 64 * 4, out_batch_stride=100 * 64, ldo=64)
    for over, msg in [(dict(b_rows_per_batch=60), "multiple of 8"), (dict(num_kb=5), "3 x"), (dict(t_rows=100), "table rows"),
                      (dict(b_bytes=16384), "data image too small"), (dict(kernel=gp.TB, block_n=64, n=96), "shape")]:
        kw = dict(base); kw.update(over)
        rc, err = gp.launch(gp.make_case(**kw))
        assert rc != 0 and msg in err, (over, rc, err)
