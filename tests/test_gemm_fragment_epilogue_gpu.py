"""The fragment epilogue path of the wgmma GEMM (FragEpi, gemm2.cuh) against the staged path, at Pangu's shapes.

Pangu's fc1 (GELU into the fp16 hidden image) and its projection / fc2 (LayerNorm + residual on the fp16 stream image,
single CTAs at C = 192, CTA pairs at C = 384) run their epilogues on the accumulator fragments and bulk-store the output
tile.  Each case launches the same GEMM through libskyrim_b200_probe.so (oracle/gemm_probe.py) on both paths, at M = 300
(a partial second m-tile) and at the full 721 x 1440 token count of the grid (also a partial last m-tile), with one CTA
(two for a pair: one CTA walks every tile) and with the default grid:
  * fc1 must be bit for bit what the staged path writes (the same gelu_erf(v + b) and the same rounding);
  * the LayerNorm sums its statistics in another order: every value of a row sample is held to the fp64 bound of
    tests/test_gemm_kernels_gpu.py, and pytest -s prints the largest difference from the staged path;
  * the destination images sit between guard bands of fp16 NaN sentinels, and the rows past M of the last m-tile hold
    the sentinel too (as do the A image's): both must be intact afterwards, and no valid element may hold it;
  * two launches on the fragment path agree bit for bit.
"""
from __future__ import annotations

import numpy as np
import pytest

from oracle import gemm_probe as gp
from oracle import gemm_ref as gr

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

GUARD = 16384
SENT = 0x7D5A            # fp16 NaN bit pattern
TILE = 16384
BN = 192
T = {192: 8 * 181 * 360, 384: 8 * 91 * 180}   # tokens of one member on Pangu's 721 x 1440 grids
SAMPLE = 2048
# sky_probe_gemm epilogue ids of the fragment path (gemm_probe.cu): EPI_F16_GELU_IMG / EPI_LN_IMG wrapped in FragEpi
EPI_F16_GELU_IMG_FRAG, EPI_LN_IMG_FRAG = 18, 19


class Guarded:
    """`nbytes` of device memory between two guard bands of the sentinel; `init` (int16, on the device) fills the inside"""

    def __init__(self, nbytes: int, init=None):
        self.nbytes = nbytes
        self.t = torch.full(((2 * GUARD + nbytes) // 2,), SENT, dtype=torch.int16, device="cuda")
        if init is not None:
            self.inner().copy_(init)
        self.ptr = self.t.data_ptr() + GUARD

    def inner(self):
        return self.t[GUARD // 2: GUARD // 2 + self.nbytes // 2]

    def check(self, M: int, nkb: int, what: str):
        """guard bands and the rows past M are the sentinel, no row below M holds it"""
        g = GUARD // 2
        assert bool((self.t[:g] == SENT).all()) and bool((self.t[-g:] == SENT).all()), f"{what}: guard band overwritten"
        v = self.inner().view(-1, nkb, 128, 64)
        last = v[-1]
        tail = M - (v.shape[0] - 1) * 128
        assert bool((last[:, tail:] == SENT).all()), f"{what}: rows past M were written"
        assert not bool((v[:-1] == SENT).any()) and not bool((last[:, :tail] == SENT).any()), f"{what}: valid rows not written"


def run(case):
    rc, msg = gp.launch(case)
    assert rc == 0, msg
    torch.cuda.synchronize()


def image(M: int, nkb: int, seed: int, tail=SENT):
    """random fp16 tile image of M rows (uniform in [-1, 1)) as int16 on the device; rows past M hold `tail`"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    nt = -(-M // 128)
    a = (torch.rand(nt * nkb * 128 * 64, generator=gen, device="cuda") * 2 - 1).half().view(torch.int16).view(nt, nkb, 128, 64)
    a[-1, :, M - (nt - 1) * 128:] = tail
    return a.reshape(-1)


def image_rows(img, rows: np.ndarray, nkb: int) -> np.ndarray:
    """rows of a tile image on the device (int16) -> fp16 [len(rows), nkb * 64] on the host"""
    v = img.view(-1, nkb, 128, 8, 8)
    r = torch.from_numpy(np.asarray(rows, np.int64)).cuda()
    sel = v[r // 128, :, r % 128].cpu().numpy()
    idx = gr._swz_index(128)[np.asarray(rows) % 128][:, None, :, None]
    return np.take_along_axis(sel, np.broadcast_to(idx, sel.shape), axis=2).reshape(len(rows), nkb * 64).view(np.float16)


def sample_rows(M: int, seed: int) -> np.ndarray:
    """every row for small M; else the first and last m-tiles and a seeded random sample"""
    if M <= SAMPLE:
        return np.arange(M)
    rng = np.random.default_rng(seed)
    return np.unique(np.concatenate([np.arange(128), np.arange(M - 192, M), rng.choice(M, SAMPLE, replace=False)]))


def operands(C: int, N: int, K: int, M: int, seed: int):
    rng = np.random.default_rng(seed)
    nkb = K // 64
    a = image(M, nkb, seed)
    w = (rng.uniform(-1.0, 1.0, (N, K)) / np.sqrt(K)).astype(np.float16)
    dw = torch.from_numpy(gr.pack_w(w, BN, nkb).copy()).cuda()
    return a, w, dw, nkb


def case(kernel, epi, N, M, a, nkb, dw, **kw):
    return gp.make_case(kernel=kernel, epi=epi, block_n=BN, n=N, n_valid=N, batches=1, nseg=1, m=M, a=[a.data_ptr()],
                        a_bytes=[a.numel() * 2], a_batch_stride=[0], a_nkb=[nkb], w=dw.data_ptr(), w_bytes=dw.numel(),
                        num_kb=nkb, **kw)


def grids(kernel):
    return [0, 2] if kernel == gp.PAIR else [0, 1]


# ---------------------------------------------------------------------------------------------------------------------
# fc1: GELU into the hidden image, N = 4C, K = C
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid", [0, 1])
@pytest.mark.parametrize("C,M", [(192, 300), (192, T[192]), (384, 300), (384, T[384])])
def test_fc1_fragment_bitwise(C, M, grid):
    N, K = 4 * C, C
    a, _, dw, nkb = operands(C, N, K, M, C + M)
    bias = torch.from_numpy(np.random.default_rng(M).uniform(-1.0, 1.0, N).astype(np.float32)).cuda()
    onkb = N // 64
    nbytes = -(-M // 128) * onkb * TILE
    outs = {}
    for name, epi in (("staged", gp.EPI_F16_GELU_IMG), ("fragment", EPI_F16_GELU_IMG_FRAG), ("fragment again", EPI_F16_GELU_IMG_FRAG)):
        o = Guarded(nbytes)
        run(case(gp.W, epi, N, M, a, nkb, dw, grid_sms=grid, hi=o.ptr, img_bytes=nbytes, img_nkb=onkb, bias=bias.data_ptr(),
                 vec_floats=N))
        outs[name] = o
    outs["fragment"].check(M, onkb, "hidden image")
    assert torch.equal(outs["fragment"].t, outs["fragment again"].t), "two launches differ"
    diff = int((outs["fragment"].t != outs["staged"].t).sum())
    print(f"[frag] fc1 C={C} M={M} grid={grid}: {diff} fp16 values differ from the staged path")
    assert diff == 0, f"fc1: {diff} values differ from the staged path"


# ---------------------------------------------------------------------------------------------------------------------
# projection (K = C) and fc2 (K = 4C): LayerNorm + residual, in place on the fp16 stream image
# ---------------------------------------------------------------------------------------------------------------------
LN_CASES = [(192, 192, 300), (192, 768, T[192]), (384, 384, 300), (384, 1536, T[384])]


@pytest.mark.parametrize("C,K,M,grid", [(C, K, M, g) for C, K, M in LN_CASES for g in grids(gp.W if C == BN else gp.PAIR)])
def test_layer_norm_fragment(C, K, M, grid):
    kernel = gp.W if C == BN else gp.PAIR
    N, eps = C, 1e-5
    a, w, dw, nkb = operands(C, N, K, M, C + K + M)
    rng = np.random.default_rng(K + M)
    bias, gamma, beta = (rng.uniform(-0.1, 0.1, N).astype(np.float32), (rng.uniform(-1.0, 1.0, N) + 1.0).astype(np.float32),
                         rng.uniform(-0.1, 0.1, N).astype(np.float32))
    dv = [torch.from_numpy(v).cuda() for v in (bias, gamma, beta)]
    onkb = N // 64
    x0 = image(M, onkb, M + 1)
    nbytes = x0.numel() * 2
    outs = {}
    for name, epi in (("staged", gp.EPI_LN_IMG), ("fragment", EPI_LN_IMG_FRAG), ("fragment again", EPI_LN_IMG_FRAG)):
        o = Guarded(nbytes, x0)
        run(case(kernel, epi, N, M, a, nkb, dw, grid_sms=grid, hi=o.ptr, img_bytes=nbytes, img_nkb=onkb, bias=dv[0].data_ptr(),
                 gamma=dv[1].data_ptr(), beta=dv[2].data_ptr(), vec_floats=N, eps=eps))
        outs[name] = o
    got, ref_path = outs["fragment"], outs["staged"]
    got.check(M, onkb, "stream image")
    assert torch.equal(got.t, outs["fragment again"].t), "two launches differ"
    valid = got.inner().view(-1, onkb, 128, 64) != SENT
    d = (got.inner().view(torch.float16).float() - ref_path.inner().view(torch.float16).float()).abs()
    max_diff = float(d[valid.reshape(-1)].max())
    rows = sample_rows(M, K)
    R, S = gr.linear([(image_rows(a, rows, nkb), w)])
    ref, bound = gr.layer_norm(R, S, bias[None, :], gamma[None, :], beta[None, :], image_rows(x0, rows, onkb).astype(np.float64), eps)
    r = gr.worst(image_rows(got.inner(), rows, onkb).astype(np.float64), ref, bound + 0.5 * gr.ulp16(np.abs(ref) + bound))
    print(f"[frag] LN {'PAIR' if kernel == gp.PAIR else 'W'} C={C} K={K} M={M} grid={grid}: max err/bound {r:.3f} over "
          f"{len(rows)} rows, max |fragment - staged| {max_diff:.3g}")
    assert r <= 1.0, f"LayerNorm: error exceeds its bound by {r:.3f}x"
