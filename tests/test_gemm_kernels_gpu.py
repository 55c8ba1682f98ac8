"""Kernel-level tests of the wgmma GEMM (k_gemm2 / k_gemm2_pair, gemm2.cuh; schedules SchedW, SchedW<true>, SchedTB)
against the float64 reference of oracle/gemm_ref.py, element by element.

Every case launches the kernel once through libskyrim_b200_probe.so (oracle/gemm_probe.py) with operands packed in
numpy, at the default grid and at a tiny grid (one CTA, two for the CTA pairs) so that one CTA walks many tiles:
ring phase wrap, the stg_free hand-off, the pairs' double-buffered statistics exchange.  The protocol:
  * every output buffer has a guard band on both sides and is filled, with the band, with a NaN sentinel bit pattern;
    after the launch the sentinel must be bit-for-bit intact everywhere outside the valid region and inside skipped
    tiles, and every valid element must be within its bound;
  * the padding rows of A images (rows >= M) are NaN, so a leak into a stored value or a statistic shows;
  * the data rows of the table x data schedule past the valid K are large finite values (they meet the table's zero
    K-padding);
  * epilogues without atomics are launched twice and must agree bit for bit; the fp64-atomic statistics to 1e-12.

Error bound of the linear part: |D - R| <= TAU * sum_k |a_k w_k| with TAU = 2^-18 (oracle/gemm_ref.py).  Each case prints
(pytest -s) the largest ratio |D - R| / (2^-23 sum_k |a_k w_k|) of its linear outputs.  Measured on an NVIDIA H100 80GB
HBM3 at a 700 W power limit: at most 3.1 for single fp16 products (the K = 1529 case; 1.8 and below for K <= 249), at
most 7.0 for the 3-term split (largest: the triangular mixing case; 6.1 for the batched six-segment operand, 6.0 for the
split table x data and the fp32 + statistics epilogue).  The
accumulator is fp32 but the tensor cores add each k16 product group into it with truncation, so the error of the split
grows with the count of small lo * hi additions into an accumulator that already holds the hi * hi part.  TAU = 2^-18
= 32 of these units keeps 4.6x headroom over the largest ratio seen; the model-level tests bound errors about a
thousand times coarser.
"""
from __future__ import annotations

import numpy as np
import pytest

from oracle import gemm_probe as gp
from oracle import gemm_ref as gr

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

GUARD = 16384
F32_SENT = np.uint32(0x7FBADBAD)
F16_SENT = np.uint16(0x7D5A)
F64_SENT = np.uint64(0x7FF4DEADBEEF0000)
TILE = 16384


# ---------------------------------------------------------------------------------------------------------------------
# device buffers
# ---------------------------------------------------------------------------------------------------------------------
class Dev:
    """device copy of a numpy array (an operand)"""

    def __init__(self, arr: np.ndarray):
        b = np.ascontiguousarray(arr).reshape(-1).view(np.uint8)
        self.t = torch.from_numpy(b.copy()).cuda()
        self.ptr = self.t.data_ptr()
        self.nbytes = b.size


class Guarded:
    """output buffer of `nbytes` between two guard bands, all filled with the sentinel pattern of `dtype`"""

    def __init__(self, nbytes: int, dtype, init: np.ndarray | None = None):
        self.dtype = np.dtype(dtype)
        self.nbytes = nbytes
        sent = {4: F32_SENT, 2: F16_SENT, 8: F64_SENT}[self.dtype.itemsize]
        n = (2 * GUARD + nbytes) // self.dtype.itemsize
        host = np.full(n, sent, dtype=sent.dtype)
        if init is not None:
            host.view(np.uint8)[GUARD:GUARD + init.nbytes] = np.ascontiguousarray(init).reshape(-1).view(np.uint8)
        self.t = torch.from_numpy(host.view(np.uint8)).cuda()
        self.ptr = self.t.data_ptr() + GUARD

    def fetch(self):
        """(inner region as dtype, the whole raw buffer as the sentinel's unsigned type)"""
        raw = self.t.cpu().numpy()
        inner = raw[GUARD:GUARD + self.nbytes].view(self.dtype)
        return inner, raw.view({4: np.uint32, 2: np.uint16, 8: np.uint64}[self.dtype.itemsize])

    def check_sentinel(self, written_mask: np.ndarray | None, what: str):
        """every element outside `written_mask` (over the inner region; None: nothing written) and every guard element
        still holds the sentinel"""
        _, raw = self.fetch()
        sent = raw[0]
        g = GUARD // self.dtype.itemsize
        assert np.all(raw[:g] == sent) and np.all(raw[len(raw) - g:] == sent), f"{what}: guard band overwritten"
        inner = raw[g:len(raw) - g]
        keep = np.ones(inner.size, bool) if written_mask is None else ~written_mask.reshape(-1)
        bad = np.flatnonzero(keep & (inner != sent))
        assert bad.size == 0, f"{what}: {bad.size} elements outside the valid region were written (first at {bad[:8]})"


def run(case):
    rc, msg = gp.launch(case)
    assert rc == 0, msg
    torch.cuda.synchronize()


def rnd(rng, shape, scale=1.0):
    return (rng.uniform(-1.0, 1.0, shape) * scale).astype(np.float32)


def f16(x):
    return np.asarray(x, np.float32).astype(np.float16)


def with_sentinel(values: np.ndarray, mask: np.ndarray) -> np.ndarray:
    """`values` where `mask`, the sentinel bit pattern of their dtype elsewhere"""
    u = {4: np.uint32, 2: np.uint16}[values.dtype.itemsize]
    out = np.full(values.shape, {4: F32_SENT, 2: F16_SENT}[values.dtype.itemsize], u)
    out[mask] = values.view(u)[mask]
    return out.view(values.dtype)


def mask_image(valid: np.ndarray, nkb: int) -> np.ndarray:
    """per-half mask of an A-style image: True where element (r, c) with valid[r, c] lives"""
    return gr.pack_tiles(valid.astype(np.float16), 128, nkb).view(np.float16) != 0


RATIOS = []


def record(name, got, ref, bound, S=None):
    r = gr.worst(got, ref, bound)
    lin = float((np.abs(np.asarray(got, np.float64) - ref) / (2.0 ** -23 * np.maximum(S, 1e-300))).max()) if S is not None else None
    RATIOS.append((name, r, lin))
    print(f"[gemm] {name}: max err/bound {r:.3f}" + (f", max |D-R|/(2^-23 sum|aw|) {lin:.3f}" if lin is not None else ""))
    assert r <= 1.0, f"{name}: error exceeds its bound by {r:.3f}x"


GRIDS = [0, 1]


# ---------------------------------------------------------------------------------------------------------------------
# operand builders
# ---------------------------------------------------------------------------------------------------------------------
def a_image(a16, nkb, batches=1):
    """A images of `batches` matrices [M, K] (NaN rows past M), and the batch stride"""
    imgs = [gr.pack_tiles(a16[b], 128, nkb, row_fill=np.nan) for b in range(batches)]
    return np.concatenate(imgs), imgs[0].size


# ---------------------------------------------------------------------------------------------------------------------
# SchedW x EpiF32Batched: every BLOCK_N the SFNO dispatch instantiates, M edges, several n-tiles, n_valid < N, long K
# ---------------------------------------------------------------------------------------------------------------------
F32_CASES = [
    # (BN, M, n_tiles, nkb, n_valid_drop, bias, add, accumulate, batches)
    (16, 129, 3, 2, 0, True, False, False, 1),
    (32, 127, 3, 3, 0, False, False, False, 1),
    (64, 1, 3, 2, 0, True, True, False, 1),
    (64, 128 * 5 + 1, 3, 4, 0, True, False, True, 2),
    (80, 128, 3, 3, 8, True, True, False, 1),
    (80, 257, 3, 2, 0, False, False, True, 1),
    (192, 129, 3, 24, 0, True, False, False, 1),
    (240, 300, 3, 3, 0, True, True, True, 1),
    (240, 129, 1, 2, 16, False, False, False, 2),
    (256, 128 * 3 + 1, 3, 2, 0, True, False, False, 1),
]


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("bn,M,nt,nkb,drop,use_bias,use_add,accumulate,batches", F32_CASES)
def test_w_f32(bn, M, nt, nkb, drop, use_bias, use_add, accumulate, batches, grid):
    rng = np.random.default_rng(bn * 1000 + M)
    N = bn * nt
    K = nkb * 64 - 7   # K padding: zero columns in both operands
    n_valid = N - drop
    a = f16(rnd(rng, (batches, M, K)))
    w = f16(rnd(rng, (batches, N, K), 1.0 / np.sqrt(K)))
    aimg, a_bs = a_image(a, nkb, batches)
    wimgs = [gr.pack_w(w[b], bn, nkb) for b in range(batches)]
    wimg = np.concatenate(wimgs)
    ldo = N + 8
    bstride = (M + 3) * ldo
    out_bytes = batches * bstride * 4
    bias = rnd(rng, N) if use_bias else None
    add = rnd(rng, batches * bstride) if use_add else None
    old = rnd(rng, batches * bstride) if accumulate else None
    dA, dW = Dev(aimg), Dev(wimg)
    dB = Dev(bias) if use_bias else None
    dAdd = Dev(add) if use_add else None

    def case(out):
        return gp.make_case(kernel=gp.W, epi=gp.EPI_F32_ACC if accumulate else gp.EPI_F32, block_n=bn, n=N, n_valid=n_valid,
                            batches=batches, grid_sms=grid, nseg=1, m=M, a=[dA.ptr], a_bytes=[dA.nbytes], a_batch_stride=[a_bs],
                            a_nkb=[nkb], w=dW.ptr, w_bytes=dW.nbytes, w_batch_stride=wimgs[0].size, num_kb=nkb, w_rep=0,
                            out=out.ptr, out_bytes=out_bytes, out_batch_stride=bstride, ldo=ldo,
                            bias=dB.ptr if dB else None, vec_floats=N, add=dAdd.ptr if dAdd else None,
                            add_bytes=dAdd.nbytes if dAdd else 0)

    valid = np.zeros((batches, bstride), bool)
    for b in range(batches):
        v = valid[b, : M * ldo].reshape(M, ldo)
        v[:, :n_valid] = True
    init = with_sentinel(old, valid.reshape(-1)) if accumulate else None
    outs = [Guarded(out_bytes, np.float32, init) for _ in range(2)]   # same initial contents (previous values) in both
    for o in outs:
        run(case(o))
    got, _ = outs[0].fetch()
    outs[0].check_sentinel(valid, "fp32 output")
    assert np.array_equal(outs[1].fetch()[1], outs[0].fetch()[1]), "two launches differ"
    got = got.reshape(batches, bstride)
    for b in range(batches):
        R, S = gr.linear([(a[b], w[b])])
        terms = []
        if use_bias:
            terms.append(bias[None, :])
        sl = lambda x: x.reshape(batches, bstride)[b, : M * ldo].reshape(M, ldo)[:, :N]
        if use_add:
            terms.append(sl(add))
        if accumulate:
            terms.append(sl(old))
        ref, bound = gr.epi_affine(R, S, *terms)
        g = got[b, : M * ldo].reshape(M, ldo)
        record(f"W/F32{'acc' if accumulate else ''} BN={bn} M={M} N={N} K={K} b={b} grid={grid}",
               g[:, :n_valid], ref[:, :n_valid], bound[:, :n_valid], S[:, :n_valid])


# ---------------------------------------------------------------------------------------------------------------------
# 3-term split (w_rep) with split-image / statistics epilogues; 6-segment AOperand (the decoder's concat(x, input))
# ---------------------------------------------------------------------------------------------------------------------
def split_operands(rng, M, kx, ki, N, batches=1, w_batches=1):
    """A = [x | in] (K = 64 kx + 64 ki, in's last 9 columns padding) as hi / lo [batches, M, K]; W as hi / lo
    [w_batches, N, K] (squeezed when 1)"""
    Kx, Ki = 64 * kx, 64 * ki - 9
    K = Kx + Ki
    a32 = rnd(rng, (batches, M, K))
    w32 = rnd(rng, (w_batches, N, K), 1.0 / np.sqrt(K))
    if w_batches == 1:
        w32 = w32[0]
    a_hi, a_lo = gr.split16(a32)
    w_hi, w_lo = gr.split16(w32)
    return a_hi, a_lo, w_hi, w_lo, Kx, Ki


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("epi,bn,M,nt", [
    (gp.EPI_SPLIT, 64, 129, 3), (gp.EPI_SPLIT_GELU, 192, 300, 2), (gp.EPI_SPLIT_GELU, 64, 128 * 4 + 1, 1),
    (gp.EPI_F32_STATS, 192, 257, 2), (gp.EPI_F32_STATS, 64, 127, 3),
    (gp.EPI_GELU_STATS, 64, 129, 2), (gp.EPI_GELU_STATS, 192, 128 * 3 + 1, 1),
])
def test_w_split(epi, bn, M, nt, grid):
    """A = [x | in] as six segments hi_x, hi_in, lo_x, lo_in, hi_x, hi_in with unequal k-block counts, W = [hi | lo]"""
    rng = np.random.default_rng(epi * 100 + bn + M)
    kx, ki = 2, 1
    N = bn * nt
    a_hi, a_lo, w_hi, w_lo, Kx, Ki = split_operands(rng, M, kx, ki, N)
    nkb = kx + ki
    imgs = {}
    for nm, x in (("hx", a_hi[0][:, :Kx]), ("hi", a_hi[0][:, Kx:]), ("lx", a_lo[0][:, :Kx]), ("li", a_lo[0][:, Kx:])):
        imgs[nm] = Dev(gr.pack_tiles(x, 128, kx if nm[1] == "x" else ki, row_fill=np.nan))
    segs = [imgs["hx"], imgs["hi"], imgs["lx"], imgs["li"], imgs["hx"], imgs["hi"]]
    seg_nkb = [kx, ki, kx, ki, kx, ki]
    # W = [hi | lo] with the k-blocks of x and in contiguous: [N][x | in (padded)] per half
    wpad = lambda w: np.concatenate([w, np.zeros((N, nkb * 64 - w.shape[1]), np.float16)], 1)
    dW = Dev(gr.pack_w(np.concatenate([wpad(w_hi), wpad(w_lo)], 1), bn, 2 * nkb))
    R, S = gr.linear(gr.split_pairs(a_hi[0], a_lo[0], w_hi, w_lo))
    n_valid = N
    onkb = -(-N // 64)
    img_bytes = -(-M // 128) * onkb * TILE
    bias = rnd(rng, N)
    dBias = Dev(bias)
    ld = N + 4
    add = rnd(rng, (M + 2) * ld)
    dAdd = Dev(add)
    asc, ash = rnd(rng, N) + 1.5, rnd(rng, N)
    dAsc, dAsh = Dev(asc), Dev(ash)
    stats = epi in (gp.EPI_F32_STATS, gp.EPI_GELU_STATS)
    nrep = 2
    outs = []
    for _ in range(nrep):
        hi, lo = Guarded(img_bytes, np.float16), Guarded(img_bytes, np.float16)
        out = Guarded((M + 2) * ld * 4, np.float32) if epi == gp.EPI_F32_STATS else None
        sums = Guarded(2 * 384 * 8, np.float64, np.zeros(2 * n_valid)) if stats else None
        c = gp.make_case(kernel=gp.W, epi=epi, block_n=bn, n=N, n_valid=n_valid, batches=1, grid_sms=grid, nseg=6, m=M,
                         a=[s.ptr for s in segs], a_bytes=[s.nbytes for s in segs], a_batch_stride=[0] * 6, a_nkb=seg_nkb,
                         w=dW.ptr, w_bytes=dW.nbytes, w_batch_stride=0, num_kb=3 * nkb, w_rep=nkb,
                         hi=hi.ptr, lo=lo.ptr, img_bytes=img_bytes, img_nkb=onkb, bias=dBias.ptr, vec_floats=N,
                         out=out.ptr if out else None, out_bytes=out.nbytes if out else 0, ldo=ld,
                         add=dAdd.ptr, add_bytes=dAdd.nbytes, asc=dAsc.ptr, ash=dAsh.ptr,
                         sums=sums.ptr if sums else None, sums_bytes=sums.nbytes if sums else 0, rows_per_batch=0)
        run(c)
        outs.append((hi, lo, out, sums))
    hi, lo, out, sums = outs[0]
    addm = add[: M * ld].reshape(M, ld)[:, :N]
    if epi == gp.EPI_SPLIT:
        f, fb = gr.epi_affine(R, S, bias[None, :])
    elif epi == gp.EPI_SPLIT_GELU:
        f, fb = gr.epi_gelu(*gr.epi_affine(R, S, bias[None, :]))
    elif epi == gp.EPI_F32_STATS:
        f, fb = gr.epi_affine(R, S, bias[None, :] + ash[None, :], addm * asc[None, :])
    else:
        f, fb = gr.epi_gelu(*gr.epi_affine(R, S, bias[None, :], addm))
    valid = np.ones((M, N), bool)
    wmask = mask_image(valid, onkb)
    hi.check_sentinel(wmask, "hi image"); lo.check_sentinel(wmask, "lo image")
    h = gr.unpack_tiles(hi.fetch()[0], 128, onkb, M, N).astype(np.float64)
    l = gr.unpack_tiles(lo.fetch()[0], 128, onkb, M, N).astype(np.float64)
    b_hi, b_sum = gr.split_bound(f, fb)
    name = f"W3/{['F32', 'F32acc', 'SPLIT', 'SPLIT_GELU', 'F32_STATS', 'GELU_STATS'][epi]} BN={bn} M={M} N={N} grid={grid}"
    lin_S = S if epi in (gp.EPI_SPLIT, gp.EPI_F32_STATS) else None
    record(name + " hi", h, f, b_hi)
    record(name + " hi+lo", h + l, f, b_sum, lin_S)
    if out is not None:
        vo = np.zeros((M + 2, ld), bool); vo[:M, :N] = True
        out.check_sentinel(vo, "fp32 output")
        record(name + " fp32", out.fetch()[0].reshape(M + 2, ld)[:M, :N], f, fb, lin_S)
    for first, second in zip(outs[0][:3], outs[1][:3]):
        if first is not None:
            assert np.array_equal(first.fetch()[1], second.fetch()[1]), "two launches differ"
    if sums is not None:
        vs = np.zeros(384 * 2 * 8 // 8, bool); vs[: 2 * n_valid] = True
        sums.check_sentinel(vs, "statistics")
        got = sums.fetch()[0][: 2 * n_valid]
        s, q, bs, bq = gr.col_stats(f, fb)
        record(name + " sum", got[:n_valid], s, bs)
        record(name + " sumsq", got[n_valid:], q, bq)
        got2 = outs[1][3].fetch()[0][: 2 * n_valid]
        np.testing.assert_allclose(got2, got, rtol=1e-12, atol=1e-12 * np.abs(got).max())


# ---------------------------------------------------------------------------------------------------------------------
# SchedW<true>: the triangular skip of the spectral mixing GEMM, batches (degrees) 260, rows (orders) 261
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("bn,N", [(192, 192), (64, 128)])
def test_w_tri_remap(bn, N, grid):
    rng = np.random.default_rng(bn)
    L, M = 260, 261
    K = N                      # (ri, i) -> (ro, o): square per degree
    nkb = K // 64
    a32 = rnd(rng, (L, M, K))
    w32 = rnd(rng, (L, N, K), 1.0 / np.sqrt(K))
    a_hi, a_lo = gr.split16(a32)
    w_hi, w_lo = gr.split16(w32)
    ahi_img, a_bs = a_image(a_hi, nkb, L)
    alo_img, _ = a_image(a_lo, nkb, L)
    wimgs = [gr.pack_w_split(w_hi[l], w_lo[l], bn, nkb) for l in range(L)]
    dAh, dAl, dW = Dev(ahi_img), Dev(alo_img), Dev(np.concatenate(wimgs))
    # destination: [m][l][(ro,o)] — batch' = source row m, row' = source batch l
    d_nkb = N // 64
    d_bb = -(-L // 128) * d_nkb * TILE
    img_bytes = M * d_bb
    res = []
    for _ in range(2):
        hi, lo = Guarded(img_bytes, np.float16), Guarded(img_bytes, np.float16)
        c = gp.make_case(kernel=gp.W_TRI, epi=gp.EPI_REMAP, block_n=bn, n=N, n_valid=N, batches=L, grid_sms=grid, nseg=3, m=M,
                         a=[dAh.ptr, dAl.ptr, dAh.ptr], a_bytes=[dAh.nbytes, dAl.nbytes, dAh.nbytes], a_batch_stride=[a_bs] * 3,
                         a_nkb=[nkb] * 3, w=dW.ptr, w_bytes=dW.nbytes, w_batch_stride=wimgs[0].size, num_kb=3 * nkb, w_rep=nkb,
                         hi=hi.ptr, lo=lo.ptr, img_bytes=img_bytes, img_batch_bytes=d_bb, img_nkb=d_nkb,
                         bdiv=1, kmul=0, kdiv=1 << 30, rb=1, same=0)
        run(c)
        res.append((hi, lo))
    hi, lo = res[0]
    # element (l, m) is computed iff its row tile m // 128 starts at or before row l
    l_idx, m_idx = np.meshgrid(np.arange(L), np.arange(M), indexing="ij")
    computed = (m_idx // 128) * 128 <= l_idx                       # [L, M]
    wmask = np.concatenate([mask_image(np.repeat(computed[:, m:m + 1], N, 1), d_nkb) for m in range(M)])
    hi.check_sentinel(wmask, "hi image (skipped tiles keep the sentinel)")
    lo.check_sentinel(wmask, "lo image (skipped tiles keep the sentinel)")
    assert np.array_equal(res[1][0].fetch()[1], hi.fetch()[1]) and np.array_equal(res[1][1].fetch()[1], lo.fetch()[1])
    H = hi.fetch()[0].reshape(M, -1); Lo = lo.fetch()[0].reshape(M, -1)
    got_h = np.stack([gr.unpack_tiles(H[m], 128, d_nkb, L, N) for m in range(M)], 1).astype(np.float64)   # [L, M, N]
    got_l = np.stack([gr.unpack_tiles(Lo[m], 128, d_nkb, L, N) for m in range(M)], 1).astype(np.float64)
    unwritten = np.argwhere(computed & np.isnan(got_h).all(2))
    assert unwritten.size == 0, f"computed tiles left unwritten at (l, m) = {unwritten[:4].tolist()} ..."
    Rr = np.empty((L, M, N)); Ss = np.empty((L, M, N))
    for l in range(L):
        Rr[l], Ss[l] = gr.linear(gr.split_pairs(a_hi[l], a_lo[l], w_hi[l], w_lo[l]))
    f, fb = gr.epi_affine(Rr, Ss)
    b_hi, b_sum = gr.split_bound(f, fb)
    sel = computed
    name = f"W_TRI/REMAP BN={bn} N={N} L={L} M={M} grid={grid}"
    record(name + " hi", got_h[sel], f[sel], b_hi[sel])
    record(name + " hi+lo", got_h[sel] + got_l[sel], f[sel], b_sum[sel], Ss[sel])
    # the skip boundary itself: degree 128 keeps order 128, degree 127 has no order-128 tile
    assert computed[128, 128] and not computed[127, 128] and computed[256, 256] and not computed[255, 256]


# ---------------------------------------------------------------------------------------------------------------------
# SchedTB: table x data, as the SFNO transforms use it
# ---------------------------------------------------------------------------------------------------------------------
def tb_operands(rng, M, Kv, N, batches, rows_per_batch, batch_bytes_mode, t_batched):
    """table T_b [M, Kv] (hi / lo, zero K-padding, NaN rows past M), data X_b [Kv, N] (hi / lo) as MN-major images.  Data
    rows past the last batch's valid K are large finite values."""
    nkb = -(-Kv // 64)
    Kp = nkb * 64
    tb = batches if t_batched else 1
    t32 = rnd(rng, (tb, M, Kv), 1.0 / np.sqrt(Kv))
    t_hi, t_lo = gr.split16(t32)
    t_rows = -(-M // 128) * 128
    # table rows past M are NaN (like the A padding rows of SchedW): a leak of them into a store or a statistic shows
    nan_rows = np.full((t_rows - M, Kv), np.nan, np.float16)
    timgs = [gr.pack_w_split(np.concatenate([t_hi[b], nan_rows]), np.concatenate([t_lo[b], nan_rows]), 128, nkb) for b in range(tb)]
    nkb_img = N // 64
    if batch_bytes_mode:   # one image per batch
        x32 = rnd(rng, (batches, Kv, N))
        x_hi, x_lo = gr.split16(x32)
        big = np.float16(3.0e4)
        imgs_h = [gr.pack_tiles(x_hi[b], 128, nkb_img, row_fill=big, rows_pad=Kp) for b in range(batches)]
        imgs_l = [gr.pack_tiles(x_lo[b], 128, nkb_img, row_fill=big, rows_pad=Kp) for b in range(batches)]
        bb = imgs_h[0].size
        xh_img, xl_img = np.concatenate(imgs_h), np.concatenate(imgs_l)
        xs_hi = [x_hi[b] for b in range(batches)]; xs_lo = [x_lo[b] for b in range(batches)]
        rpb = 0
    else:                  # batches inside one image, rows_per_batch apart; rows of batch b past Kv belong to b + 1
        rpb = rows_per_batch
        rows = (batches - 1) * rpb + Kv
        x32 = rnd(rng, (rows, N))
        x_hi, x_lo = gr.split16(x32)
        total = (batches - 1) * rpb + Kp
        xh_img = gr.pack_tiles(x_hi, 128, nkb_img, row_fill=np.float16(3.0e4), rows_pad=total)
        xl_img = gr.pack_tiles(x_lo, 128, nkb_img, row_fill=np.float16(3.0e4), rows_pad=total)
        bb = 0
        xs_hi = [x_hi[b * rpb:b * rpb + Kv] for b in range(batches)]
        xs_lo = [x_lo[b * rpb:b * rpb + Kv] for b in range(batches)]
    Rr, Ss = [], []
    for b in range(batches):
        th, tl = t_hi[b if t_batched else 0], t_lo[b if t_batched else 0]
        R, S = gr.linear([(th, xs_hi[b].T), (th, xs_lo[b].T), (tl, xs_hi[b].T)])
        Rr.append(R); Ss.append(S)
    dT = Dev(np.concatenate(timgs))
    dXh, dXl = Dev(xh_img), Dev(xl_img)
    kw = dict(t=dT.ptr, t_bytes=dT.nbytes, t_batch_stride=timgs[0].size if t_batched else 0, t_rows=t_rows, b_nkb_img=nkb_img,
              b_hi=dXh.ptr, b_lo=dXl.ptr, b_bytes=dXh.nbytes, b_rows_per_batch=rpb, b_batch_bytes=bb, num_kb=3 * nkb)
    return kw, (dT, dXh, dXl), np.stack(Rr), np.stack(Ss)


TB_REMAPS = {   # (bdiv, kmul, kdiv, rb, same), as forward_sht / inverse_sht build them (E = N or N / 2)
    "dft": lambda N: (2, N, 1 << 30, 1, 0),
    "legendre_to_mixing": lambda N: (1, 0, 1 << 30, 1, 0),
    "legendre_to_inverse": lambda N: (1, 0, 1 << 30, 1, 1),
    "inverse_legendre": lambda N: (1, 0, N // 2, 2, 0),
}


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("kind,bn,N,M,Kv,batches,rpb,affine", [
    ("dft", 64, 128, 74, 72, 5, 72, True),                 # rows_per_batch 72: batches start mid-tile (two-copy path)
    ("dft", 192, 192, 38, 200, 3, 200, False),
    ("legendre_to_mixing", 128, 256, 41, 130, 6, 0, False),
    ("legendre_to_inverse", 256, 512, 41, 97, 3, 0, False),
    ("inverse_legendre", 192, 384, 121, 41, 4, 0, False),
    ("inverse_legendre", 64, 128, 129, 65, 3, 0, False),
])
def test_tb_remap(kind, bn, N, M, Kv, batches, rpb, affine, grid):
    rng = np.random.default_rng(bn + N + M)
    t_batched = kind != "dft"
    kw, keep, R, S = tb_operands(rng, M, Kv, N, batches, rpb, rpb == 0, t_batched)
    bdiv, kmul, kdiv, rb, same = TB_REMAPS[kind](N)
    n_valid = N
    # destination extents
    bI, rI, cI = np.meshgrid(np.arange(batches), np.arange(M), np.arange(n_valid), indexing="ij")
    dbI, drI, dkI = gr.remap_dest(bI, rI, cI, bdiv=bdiv, kmul=kmul, kdiv=kdiv, rb=rb, same=same)
    nb, nrow, nk = int(dbI.max()) + 1, int(drI.max()) + 1, int(dkI.max()) + 1
    d_nkb = -(-nk // 64)
    d_bb = -(-nrow // 128) * d_nkb * TILE
    img_bytes = nb * d_bb
    extra = {}
    if affine:
        csc, csh = rnd(rng, N) + 1.5, rnd(rng, N)
        t1 = rnd(rng, M)
        keep = keep + (Dev(csc), Dev(csh), Dev(t1))
        extra = dict(csc=keep[-3].ptr, csh=keep[-2].ptr, t1=keep[-1].ptr, vec_floats=N, t1_floats=M)
    res = []
    for _ in range(2):
        hi, lo = Guarded(img_bytes, np.float16), Guarded(img_bytes, np.float16)
        c = gp.make_case(kernel=gp.TB, epi=gp.EPI_REMAP, block_n=bn, n=N, n_valid=n_valid, batches=batches, grid_sms=grid, m=M,
                         hi=hi.ptr, lo=lo.ptr, img_bytes=img_bytes, img_batch_bytes=d_bb, img_nkb=d_nkb,
                         bdiv=bdiv, kmul=kmul, kdiv=kdiv, rb=rb, same=same, **kw, **extra)
        run(c)
        res.append((hi, lo))
    hi, lo = res[0]
    f, fb = R, gr.TAU * S
    if affine:
        f = R * csc[None, None, :] + csh[None, None, :] * t1[None, :, None]
        fb = gr.TAU * S * np.abs(csc)[None, None, :] + 4 * gr.U32 * (np.abs(R * csc) + np.abs(csh[None, None, :] * t1[None, :, None]))
    else:
        fb = fb + 4 * gr.U32 * np.abs(R)
    # scatter the reference into destination coordinates
    ref = np.full((nb, -(-nrow // 128) * 128, d_nkb * 64), np.nan)
    bnd = np.zeros_like(ref)
    lin = np.zeros_like(ref)
    ref[dbI, drI, dkI] = f
    bnd[dbI, drI, dkI] = fb
    lin[dbI, drI, dkI] = S * (np.abs(csc)[None, None, :] if affine else 1.0)
    valid = ~np.isnan(ref)
    wmask = np.concatenate([mask_image(valid[b], d_nkb) for b in range(nb)])
    hi.check_sentinel(wmask, "hi image"); lo.check_sentinel(wmask, "lo image")
    assert np.array_equal(res[1][0].fetch()[1], hi.fetch()[1]) and np.array_equal(res[1][1].fetch()[1], lo.fetch()[1])
    H = hi.fetch()[0].reshape(nb, -1); Lo = lo.fetch()[0].reshape(nb, -1)
    gh = np.stack([gr.unpack_tiles(H[b], 128, d_nkb, ref.shape[1]) for b in range(nb)]).astype(np.float64)
    gl = np.stack([gr.unpack_tiles(Lo[b], 128, d_nkb, ref.shape[1]) for b in range(nb)]).astype(np.float64)
    b_hi, b_sum = gr.split_bound(ref[valid], bnd[valid])
    name = f"TB/REMAP {kind} BN={bn} N={N} M={M} K={Kv} batches={batches} rpb={rpb} grid={grid}"
    record(name + " hi", gh[valid], ref[valid], b_hi)
    record(name + " hi+lo", gh[valid] + gl[valid], ref[valid], b_sum, lin[valid])


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("epi,bn,N,M,Kv,batches,rpb", [
    (gp.EPI_F32, 64, 192, 200, 41, 3, 0),
    (gp.EPI_F32, 256, 512, 129, 72, 2, 0),
    (gp.EPI_GELU_STATS, 128, 256, 72, 130, 4, 0),
    (gp.EPI_GELU_STATS, 192, 192, 200, 72, 3, 72),
])
def test_tb_f32_gelu_stats(epi, bn, N, M, Kv, batches, rpb, grid):
    """inverse DFT epilogues: fp32 pixel-major field (batch = latitude, row = longitude), or GELU + statistics image"""
    rng = np.random.default_rng(epi + bn + N + M)
    kw, keep, R, S = tb_operands(rng, M, Kv, N, batches, rpb, rpb == 0, False)
    res = []
    if epi == gp.EPI_F32:
        ldo, bstride = N, M * N
        nbytes = batches * bstride * 4
        for _ in range(2):
            out = Guarded(nbytes, np.float32)
            run(gp.make_case(kernel=gp.TB, epi=epi, block_n=bn, n=N, n_valid=N, batches=batches, grid_sms=grid, m=M,
                             out=out.ptr, out_bytes=nbytes, out_batch_stride=bstride, ldo=ldo, **kw))
            res.append(out)
        res[0].check_sentinel(np.ones(batches * bstride, bool), "fp32 field")
        assert np.array_equal(res[0].fetch()[1], res[1].fetch()[1])
        got = res[0].fetch()[0].reshape(batches, M, N)
        f, fb = gr.epi_affine(R, S)
        record(f"TB/F32 BN={bn} N={N} M={M} K={Kv} batches={batches} grid={grid}", got, f, fb, S)
        return
    pixels = batches * M
    onkb = N // 64
    img_bytes = -(-pixels // 128) * onkb * TILE
    bias = rnd(rng, N)
    add = rnd(rng, pixels * N)
    dB, dAdd = Dev(bias), Dev(add)
    for _ in range(2):
        hi, lo = Guarded(img_bytes, np.float16), Guarded(img_bytes, np.float16)
        sums = Guarded(2 * 384 * 8, np.float64, np.zeros(2 * N))
        run(gp.make_case(kernel=gp.TB, epi=epi, block_n=bn, n=N, n_valid=N, batches=batches, grid_sms=grid, m=M,
                         hi=hi.ptr, lo=lo.ptr, img_bytes=img_bytes, img_nkb=onkb, bias=dB.ptr, vec_floats=N,
                         add=dAdd.ptr, add_bytes=dAdd.nbytes, ldo=N, rows_per_batch=M, sums=sums.ptr, sums_bytes=sums.nbytes, **kw))
        res.append((hi, lo, sums))
    hi, lo, sums = res[0]
    f, fb = gr.epi_gelu(*gr.epi_affine(R.reshape(pixels, N), S.reshape(pixels, N), bias[None, :], add.reshape(pixels, N)))
    wmask = mask_image(np.ones((pixels, N), bool), onkb)
    hi.check_sentinel(wmask, "hi image"); lo.check_sentinel(wmask, "lo image")
    assert np.array_equal(res[1][0].fetch()[1], hi.fetch()[1]) and np.array_equal(res[1][1].fetch()[1], lo.fetch()[1])
    h = gr.unpack_tiles(hi.fetch()[0], 128, onkb, pixels, N).astype(np.float64)
    l = gr.unpack_tiles(lo.fetch()[0], 128, onkb, pixels, N).astype(np.float64)
    b_hi, b_sum = gr.split_bound(f, fb)
    name = f"TB/GELU_STATS BN={bn} N={N} M={M} K={Kv} batches={batches} rpb={rpb} grid={grid}"
    record(name + " hi", h, f, b_hi)
    record(name + " hi+lo", h + l, f, b_sum)
    vs = np.zeros(2 * 384, bool); vs[: 2 * N] = True
    sums.check_sentinel(vs, "statistics")
    got = sums.fetch()[0][: 2 * N]
    s, q, bs, bq = gr.col_stats(f, fb)
    record(name + " sum", got[:N], s, bs)
    record(name + " sumsq", got[N:], q, bq)
    np.testing.assert_allclose(res[1][2].fetch()[0][: 2 * N], got, rtol=1e-12, atol=1e-12 * np.abs(got).max())


# ---------------------------------------------------------------------------------------------------------------------
# LayerNorm + residual (Pangu): single CTA at BN = 192, CTA pairs at 192 (N = 384)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("img_stream", [False, True])
@pytest.mark.parametrize("kernel,bn,N,M,grid", [
    (gp.W, 192, 192, 300, 0), (gp.W, 192, 192, 300, 1), (gp.W, 192, 192, 129, 1),
    (gp.PAIR, 192, 384, 128 * 5 + 17, 0), (gp.PAIR, 192, 384, 128 * 5 + 17, 2),
])
def test_layer_norm(kernel, bn, N, M, grid, img_stream):
    """in place, as the engines use it: x += LN(A W^T + b), and the fp16 image of x rewritten (or, with the fp16-only
    stream, the residual read from the image and the sum written back into it)"""
    rng = np.random.default_rng(bn + M + img_stream)
    nkb = 3
    K = nkb * 64
    a = f16(rnd(rng, (M, K)))
    w = f16(rnd(rng, (N, K), 1.0 / np.sqrt(K)))
    dA = Dev(gr.pack_tiles(a, 128, nkb, row_fill=np.nan))
    # the pair kernel takes W as two BN-row halves: the plain [N/BN][nkb][BN x 128 B] image is exactly that
    dW = Dev(gr.pack_w(w, bn, nkb))
    bias, gamma, beta = rnd(rng, N, 0.1), rnd(rng, N) + 1.0, rnd(rng, N, 0.1)
    dB, dG, dBe = Dev(bias), Dev(gamma), Dev(beta)
    onkb = N // 64
    ld = N + 4
    x0 = rnd(rng, (M, N))
    x0_16 = f16(x0)
    img0 = gr.pack_tiles(x0_16, 128, onkb)
    img_bytes = img0.size
    res = []
    for _ in range(2):
        vx = np.zeros((M + 1, ld), bool); vx[:M, :N] = True
        xfull = np.zeros((M + 1, ld), np.float32); xfull[:M, :N] = x0
        x = Guarded((M + 1) * ld * 4, np.float32, with_sentinel(xfull, vx))
        img = Guarded(img_bytes, np.float16, with_sentinel(img0.view(np.float16), mask_image(np.ones((M, N), bool), onkb)))
        run(gp.make_case(kernel=kernel, epi=gp.EPI_LN_IMG if img_stream else gp.EPI_LN, block_n=bn, n=N, n_valid=N, batches=1,
                         grid_sms=grid, nseg=1, m=M, a=[dA.ptr], a_bytes=[dA.nbytes], a_batch_stride=[0], a_nkb=[nkb],
                         w=dW.ptr, w_bytes=dW.nbytes, num_kb=nkb, out=x.ptr, out_bytes=x.nbytes, ldo=ld,
                         hi=img.ptr, img_bytes=img_bytes, img_nkb=onkb, bias=dB.ptr, gamma=dG.ptr, beta=dBe.ptr,
                         vec_floats=N, eps=1e-5))
        res.append((x, img))
    x, img = res[0]
    R, S = gr.linear([(a, w)])
    resid = x0_16.astype(np.float64) if img_stream else x0.astype(np.float64)
    ref, bound = gr.layer_norm(R, S, bias[None, :], gamma[None, :], beta[None, :], resid, 1e-5)
    name = f"{'PAIR' if kernel == gp.PAIR else 'W'}/LN{'_IMG' if img_stream else ''} BN={bn} N={N} M={M} grid={grid}"
    img.check_sentinel(mask_image(np.ones((M, N), bool), onkb), "fp16 image")
    x.check_sentinel(vx, "fp32 rows")
    if not img_stream:
        gx = x.fetch()[0].reshape(M + 1, ld)[:M, :N]
        record(name + " fp32", gx, ref, bound)
    gi = gr.unpack_tiles(img.fetch()[0], 128, onkb, M, N).astype(np.float64)
    record(name + " fp16", gi, ref, bound + 0.5 * gr.ulp16(np.abs(ref) + bound))
    assert np.array_equal(res[1][0].fetch()[1], x.fetch()[1]) and np.array_equal(res[1][1].fetch()[1], img.fetch()[1])


# ---------------------------------------------------------------------------------------------------------------------
# six-segment A operand over batches: every segment has its own batch stride (the select walk of AOperand::kblock)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("bn,M", [(64, 129), (192, 257)])
def test_w_six_segments_batched(bn, M, grid):
    rng = np.random.default_rng(bn + M + 7)
    kx, ki, B = 2, 1, 3
    N = 2 * bn
    a_hi, a_lo, w_hi, w_lo, Kx, Ki = split_operands(rng, M, kx, ki, N, batches=B, w_batches=B)
    nkb = kx + ki
    segs, strides = [], []
    for j, (src, cols, k) in enumerate(((a_hi, slice(0, Kx), kx), (a_hi, slice(Kx, None), ki), (a_lo, slice(0, Kx), kx),
                                        (a_lo, slice(Kx, None), ki))):
        imgs = [gr.pack_tiles(src[b][:, cols], 128, k, row_fill=np.nan) for b in range(B)]
        gap = np.full((j + 1) * TILE // 2, np.nan, np.float16).view(np.uint8)   # unequal strides: a NaN gap per segment
        segs.append(Dev(np.concatenate([np.concatenate([im, gap]) for im in imgs])))
        strides.append(imgs[0].size + gap.size)
    order = [0, 1, 2, 3, 0, 1]
    wpad = lambda w: np.concatenate([w, np.zeros((N, nkb * 64 - w.shape[1]), np.float16)], 1)
    wimgs = [gr.pack_w(np.concatenate([wpad(w_hi[b]), wpad(w_lo[b])], 1), bn, 2 * nkb) for b in range(B)]
    dW = Dev(np.concatenate(wimgs))
    ldo, bstride = N + 4, (M + 1) * (N + 4)
    out_bytes = B * bstride * 4
    outs = [Guarded(out_bytes, np.float32) for _ in range(2)]
    for o in outs:
        run(gp.make_case(kernel=gp.W, epi=gp.EPI_F32, block_n=bn, n=N, n_valid=N, batches=B, grid_sms=grid, nseg=6, m=M,
                         a=[segs[i].ptr for i in order], a_bytes=[segs[i].nbytes for i in order],
                         a_batch_stride=[strides[i] for i in order], a_nkb=[kx, ki, kx, ki, kx, ki],
                         w=dW.ptr, w_bytes=dW.nbytes, w_batch_stride=wimgs[0].size, num_kb=3 * nkb, w_rep=nkb,
                         out=o.ptr, out_bytes=out_bytes, out_batch_stride=bstride, ldo=ldo))
    valid = np.zeros((B, M + 1, ldo), bool); valid[:, :M, :N] = True
    outs[0].check_sentinel(valid, "fp32 output")
    assert np.array_equal(outs[0].fetch()[1], outs[1].fetch()[1]), "two launches differ"
    got = outs[0].fetch()[0].reshape(B, M + 1, ldo)
    for b in range(B):
        R, S = gr.linear(gr.split_pairs(a_hi[b], a_lo[b], w_hi[b], w_lo[b]))
        ref, bound = gr.epi_affine(R, S)
        record(f"W3/F32 6 segments BN={bn} M={M} N={N} b={b} grid={grid}", got[b, :M, :N], ref, bound, S)


# ---------------------------------------------------------------------------------------------------------------------
# fp16 epilogues: Pangu fc1 (GELU into the hidden image, BN 192) and GraphCast's node tables (row-major, BN 256)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("epi,bn,N,M", [(gp.EPI_F16_GELU_IMG, 192, 384, 300), (gp.EPI_F16_ROWS, 256, 512, 129)])
def test_w_f16(epi, bn, N, M, grid):
    rng = np.random.default_rng(epi + M)
    nkb = 3
    K = nkb * 64 - 5
    a = f16(rnd(rng, (M, K))); w = f16(rnd(rng, (N, K), 1.0 / np.sqrt(K)))
    dA, dW = Dev(gr.pack_tiles(a, 128, nkb, row_fill=np.nan)), Dev(gr.pack_w(w, bn, nkb))
    bias = rnd(rng, N); dB = Dev(bias)
    R, S = gr.linear([(a, w)])
    f, fb = gr.epi_affine(R, S, bias[None, :])
    onkb = N // 64
    if epi == gp.EPI_F16_GELU_IMG:
        f, fb = gr.epi_gelu(f, fb)
        nbytes = -(-M // 128) * onkb * TILE
        mask = mask_image(np.ones((M, N), bool), onkb)
    else:
        ldo = N + 8
        nbytes = (M + 1) * ldo * 2
        mask = np.zeros((M + 1, ldo), bool); mask[:M, :N] = True
    outs = [Guarded(nbytes, np.float16) for _ in range(2)]
    for o in outs:
        kw = dict(hi=o.ptr, img_bytes=nbytes, img_nkb=onkb) if epi == gp.EPI_F16_GELU_IMG else dict(out=o.ptr, out_bytes=nbytes, ldo=ldo)
        run(gp.make_case(kernel=gp.W, epi=epi, block_n=bn, n=N, n_valid=N, batches=1, grid_sms=grid, nseg=1, m=M, a=[dA.ptr],
                         a_bytes=[dA.nbytes], a_batch_stride=[0], a_nkb=[nkb], w=dW.ptr, w_bytes=dW.nbytes, num_kb=nkb,
                         bias=dB.ptr, vec_floats=N, **kw))
    outs[0].check_sentinel(mask, "fp16 output")
    assert np.array_equal(outs[0].fetch()[1], outs[1].fetch()[1]), "two launches differ"
    h = outs[0].fetch()[0]
    got = (gr.unpack_tiles(h, 128, onkb, M, N) if epi == gp.EPI_F16_GELU_IMG else h.reshape(M + 1, ldo)[:M, :N]).astype(np.float64)
    record(f"W/F16{'_GELU_IMG' if epi == gp.EPI_F16_GELU_IMG else '_ROWS'} BN={bn} N={N} M={M} grid={grid}", got, f, gr.f16_bound(f, fb))


# ---------------------------------------------------------------------------------------------------------------------
# GraphCast: hidden layer SiLU with 0 / 2 gathered tables (repeated and extreme indices), output head, LayerNorm pairs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("kg,M", [(0, 300), (2, 300), (2, 128 * 4 + 1)])
def test_gc_silu(kg, M, grid):
    rng = np.random.default_rng(kg + M)
    N, bn, nkb = 512, 256, 2
    K = nkb * 64
    a = f16(rnd(rng, (M, K))); w = f16(rnd(rng, (N, K), 1.0 / np.sqrt(K)))
    dA, dW = Dev(gr.pack_tiles(a, 128, nkb, row_fill=np.nan)), Dev(gr.pack_w(w, bn, nkb))
    bias = rnd(rng, N); dB = Dev(bias)
    R, S = gr.linear([(a, w)])
    terms = [bias[None, :]]
    kw = {}
    keep = []
    if kg == 2:
        # one table [rows][1024] holding both halves (sender | receiver), as the processor's edge MLP reads it
        rows = 37
        tab = f16(rnd(rng, (rows, 2 * N)))
        dT = Dev(tab)
        ia = rng.integers(0, rows, M).astype(np.int32); ib = rng.integers(0, rows, M).astype(np.int32)
        ia[:5] = 0; ia[5:10] = rows - 1; ib[:5] = rows - 1; ib[5:10] = 0; ia[-3:] = ia[0]; ib[-3:] = rows - 1   # repeats, extremes
        dIa, dIb = Dev(ia), Dev(ib)
        keep += [dT, dIa, dIb]
        terms += [tab[ia, :N].astype(np.float64), tab[ib, N:].astype(np.float64)]
        kw = dict(ta=dT.ptr, ta_bytes=dT.nbytes, ta_rows=rows, lda=2 * N, ia=dIa.ptr,
                  tb=dT.ptr + 2 * N, tb_bytes=dT.nbytes - 2 * N, tb_rows=rows, ldb=2 * N, ib=dIb.ptr)
    f, fb = gr.epi_silu(*gr.epi_affine(R, S, *terms))
    nbytes = -(-M // 128) * 8 * TILE
    outs = [Guarded(nbytes, np.float16) for _ in range(2)]
    for o in outs:
        run(gp.make_case(kernel=gp.W, epi=gp.EPI_GC_SILU2 if kg else gp.EPI_GC_SILU0, block_n=bn, n=N, n_valid=N, batches=1,
                         grid_sms=grid, nseg=1, m=M, a=[dA.ptr], a_bytes=[dA.nbytes], a_batch_stride=[0], a_nkb=[nkb],
                         w=dW.ptr, w_bytes=dW.nbytes, num_kb=nkb, hi=o.ptr, img_bytes=nbytes, img_nkb=8, bias=dB.ptr,
                         vec_floats=N, **kw))
    outs[0].check_sentinel(mask_image(np.ones((M, N), bool), 8), "hidden image")
    assert np.array_equal(outs[0].fetch()[1], outs[1].fetch()[1]), "two launches differ"
    got = gr.unpack_tiles(outs[0].fetch()[0], 128, 8, M, N).astype(np.float64)
    record(f"W/GC_SILU{kg} M={M} grid={grid}", got, f, gr.f16_bound(f, fb))


@pytest.mark.parametrize("grid", GRIDS)
def test_gc_out(grid):
    rng = np.random.default_rng(11)
    M, N, bn, nkb, nprog = 300, 128, 128, 8, 83
    K = nkb * 64
    a = f16(rnd(rng, (M, K))); w = f16(rnd(rng, (N, K), 1.0 / np.sqrt(K)))
    dA, dW = Dev(gr.pack_tiles(a, 128, nkb, row_fill=np.nan)), Dev(gr.pack_w(w, bn, nkb))
    bias, dstd = rnd(rng, N), rnd(rng, N) + 1.2
    plane = M + 5
    xin = rnd(rng, (N, plane))
    dB, dD, dX = Dev(bias), Dev(dstd), Dev(xin)
    nbytes = N * plane * 4
    outs = [Guarded(nbytes, np.float32) for _ in range(2)]
    for o in outs:
        run(gp.make_case(kernel=gp.W, epi=gp.EPI_GC_OUT, block_n=bn, n=N, n_valid=N, batches=1, grid_sms=grid, nseg=1, m=M,
                         a=[dA.ptr], a_bytes=[dA.nbytes], a_batch_stride=[0], a_nkb=[nkb], w=dW.ptr, w_bytes=dW.nbytes,
                         num_kb=nkb, out=o.ptr, out_bytes=nbytes, xin=dX.ptr, xin_bytes=dX.nbytes, bias=dB.ptr, dstd=dD.ptr,
                         vec_floats=N, plane=plane, nprog=nprog))
    valid = np.zeros((N, plane), bool); valid[:nprog, :M] = True
    outs[0].check_sentinel(valid, "output planes")
    assert np.array_equal(outs[0].fetch()[1], outs[1].fetch()[1]), "two launches differ"
    R, S = gr.linear([(a, w)])
    y = (R + bias[None, :]).T[:nprog]                                  # [channel][grid point]
    ref = xin[:nprog, :M] + dstd[:nprog, None] * y
    bound = np.abs(dstd[:nprog, None]) * (gr.TAU * S.T[:nprog] + 4 * gr.U32 * np.abs(y)) + 4 * gr.U32 * np.abs(ref)
    got = outs[0].fetch()[0].reshape(N, plane)[:nprog, :M]
    record(f"W/GC_OUT M={M} nprog={nprog} grid={grid}", got, ref, bound)


@pytest.mark.parametrize("grid", [0, 2])
@pytest.mark.parametrize("kres", [0, 1, 2])
def test_gc_layer_norm_pair(kres, grid):
    """Epi2F32Img<true, kRes> on the column-split CTA pairs (256-column halves of the 512-wide latent), in place as
    GraphCast runs it: kRes 1 with xin == xout (mesh nodes), kRes 2 with xin_img == img (grid nodes, mesh edges), kRes 0
    writing y only"""
    rng = np.random.default_rng(kres + grid + 31)
    M, N, bn, nkb = 128 * 5 + 17, 512, 256, 2
    K = nkb * 64
    a = f16(rnd(rng, (M, K))); w = f16(rnd(rng, (N, K), 1.0 / np.sqrt(K)))
    dA, dW = Dev(gr.pack_tiles(a, 128, nkb, row_fill=np.nan)), Dev(gr.pack_w(w, bn, nkb))
    bias, gamma, beta = rnd(rng, N, 0.1), rnd(rng, N) + 1.0, rnd(rng, N, 0.1)
    dB, dG, dBe = Dev(bias), Dev(gamma), Dev(beta)
    x0 = rnd(rng, (M, N)); x0_16 = f16(x0)
    img_bytes = -(-M // 128) * 8 * TILE
    vimg = mask_image(np.ones((M, N), bool), 8)
    res = []
    for _ in range(2):
        x = Guarded(M * N * 4, np.float32, x0 if kres == 1 else None)
        img = Guarded(img_bytes, np.float16, with_sentinel(gr.pack_tiles(x0_16, 128, 8).view(np.float16), vimg) if kres == 2 else None)
        yimg = Guarded(img_bytes, np.float16)
        kw = dict(out=x.ptr if kres < 2 else None, out_bytes=x.nbytes, hi=img.ptr, yimg=yimg.ptr, img_bytes=img_bytes)
        if kres == 1:
            kw.update(xin=x.ptr, xin_bytes=x.nbytes)
        if kres == 2:
            kw.update(xin_img=img.ptr, xin_bytes=img_bytes)
        run(gp.make_case(kernel=gp.PAIR, epi=[gp.EPI_GC_LN0, gp.EPI_GC_LN1, gp.EPI_GC_LN2][kres], block_n=bn, n=N, n_valid=N,
                         batches=1, grid_sms=grid, nseg=1, m=M, a=[dA.ptr], a_bytes=[dA.nbytes], a_batch_stride=[0], a_nkb=[nkb],
                         w=dW.ptr, w_bytes=dW.nbytes, num_kb=nkb, bias=dB.ptr, gamma=dG.ptr, beta=dBe.ptr, vec_floats=N,
                         eps=1e-5, **kw))
        res.append((x, img, yimg))
    x, img, yimg = res[0]
    for first, second in zip(res[0], res[1]):
        assert np.array_equal(first.fetch()[1], second.fetch()[1]), "two launches differ"
    R, S = gr.linear([(a, w)])
    resid = {0: np.zeros((M, N)), 1: x0.astype(np.float64), 2: x0_16.astype(np.float64)}[kres]
    ref, bound = gr.layer_norm(R, S, bias[None, :], gamma[None, :], beta[None, :], resid, 1e-5)
    y, yb = gr.layer_norm(R, S, bias[None, :], gamma[None, :], beta[None, :], np.zeros((M, N)), 1e-5)
    name = f"PAIR/GC_LN{kres} M={M} grid={grid}"
    img.check_sentinel(vimg, "stream image"); yimg.check_sentinel(vimg, "update image")
    if kres < 2:
        x.check_sentinel(np.ones(M * N, bool), "fp32 rows")
        record(name + " fp32", x.fetch()[0].reshape(M, N), ref, bound)
    else:
        x.check_sentinel(None, "fp32 rows (not written)")
    record(name + " img", gr.unpack_tiles(img.fetch()[0], 128, 8, M, N).astype(np.float64), ref, gr.f16_bound(ref, bound))
    record(name + " yimg", gr.unpack_tiles(yimg.fetch()[0], 128, 8, M, N).astype(np.float64), y, gr.f16_bound(y, yb))


def test_summary():
    """prints the largest ratios seen (run last by file order)"""
    if RATIOS:
        lin = [r[2] for r in RATIOS if r[2] is not None]
        print(f"[gemm] cases {len(RATIOS)}: max err/bound {max(r[1] for r in RATIOS):.3f}; "
              f"max |D-R|/(2^-23 sum|aw|) {max(lin) if lin else float('nan'):.3f}")
