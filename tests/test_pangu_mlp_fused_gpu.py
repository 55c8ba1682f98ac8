"""Pangu's fused MLP (mlp_fused.cuh: k_mlp_fused at C = 192, k_mlp_fused_pair at C = 384) against fc1 + fc2 of the
two-GEMM path.

The fused kernel runs fc1, GELU and fc2 per 128-row tile with the hidden activation in shared memory.  Each case launches,
through libskyrim_b200_probe.so (oracle/gemm_probe.py), the two-GEMM path as the engine runs it (fc1 with GELU into the
fp16 hidden image on the fragment path, then fc2 + LayerNorm + residual in place on the stream image) and the fused kernel
on the same fp16 operands, and requires:
  * the stream image the fused kernel writes is bit for bit the two-GEMM path's (the same fc1 sums, the same fp16
    rounding of the same GELU, the same fc2 products in the same order);
  * the image sits between guard bands of fp16 NaN sentinels and the rows past M of the last m-tile hold the sentinel
    (as they do in the input): they are intact afterwards, and no valid element holds it;
  * at one small shape, the hidden image and the result are within the fp64 per-element bounds of
    tests/test_gemm_kernels_gpu.py (oracle/gemm_ref.py).
Token counts: the C = 192 and C = 384 grids of Pangu at 41 x 96, 45 x 192 and 721 x 1440 (all but the C = 192 grid at
45 x 192 end in a partial m-tile), one and three members; grids of all SMs, 1 CTA (pair) and 7 CTAs (pairs).
"""
from __future__ import annotations

import numpy as np
import pytest

from oracle import gemm_probe as gp
from oracle import gemm_ref as gr
from oracle import pangu_kernels_ref as pk
from skyrim_b200.config import pangu_full, pangu_small

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

GUARD = 16384
SENT = 0x7D5A            # fp16 NaN bit pattern
TILE = 16384
MLP = 4                  # sky_probe_gemm kernel id of the fused MLP (gemm_probe.cu SKY_PROBE_MLP)
EPI_F16_GELU_IMG_FRAG, EPI_LN_IMG_FRAG = 18, 19   # the two-GEMM path's fragment epilogues (gemm_probe.cu)
EPS = 1e-5


def tokens(cfg, C: int) -> int:
    g = pk.grids(cfg)[0 if C == 192 else 1]
    assert g.C == C
    return g.Z * g.H * g.W


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
        g = GUARD // 2
        assert bool((self.t[:g] == SENT).all()) and bool((self.t[-g:] == SENT).all()), f"{what}: guard band overwritten"
        v = self.inner().view(-1, nkb, 128, 64)
        tail = M - (v.shape[0] - 1) * 128
        assert bool((v[-1][:, tail:] == SENT).all()), f"{what}: rows past M were written"
        assert not bool((v[:-1] == SENT).any()) and not bool((v[-1][:, :tail] == SENT).any()), f"{what}: valid rows not written"


def image(M: int, nkb: int, seed: int):
    """random fp16 tile image of M rows (uniform in [-1, 1)) as int16 on the device; rows past M hold the sentinel"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    nt = -(-M // 128)
    a = (torch.rand(nt * nkb * 128 * 64, generator=gen, device="cuda") * 2 - 1).half().view(torch.int16).view(nt, nkb, 128, 64)
    a[-1, :, M - (nt - 1) * 128:] = SENT
    return a.reshape(-1)


def image_rows(img, rows: np.ndarray, nkb: int) -> np.ndarray:
    """rows of a tile image on the device (int16) -> fp16 [len(rows), nkb * 64] on the host"""
    v = img.view(-1, nkb, 128, 8, 8)
    r = torch.from_numpy(np.asarray(rows, np.int64)).cuda()
    sel = v[r // 128, :, r % 128].cpu().numpy()
    idx = gr._swz_index(128)[np.asarray(rows) % 128][:, None, :, None]
    return np.take_along_axis(sel, np.broadcast_to(idx, sel.shape), axis=2).reshape(len(rows), nkb * 64).view(np.float16)


def run(case):
    rc, msg = gp.launch(case)
    assert rc == 0, msg
    torch.cuda.synchronize()


class Mlp:
    """one block's MLP weights (fp16 as the engine packs them) and vectors"""

    def __init__(self, seed: int, C: int):
        self.C = C
        NKB = C // 64
        rng = np.random.default_rng(seed)
        self.w1 = (rng.uniform(-1.0, 1.0, (4 * C, C)) / np.sqrt(C)).astype(np.float16)
        self.w2 = (rng.uniform(-1.0, 1.0, (C, 4 * C)) / np.sqrt(4 * C)).astype(np.float16)
        self.b1 = rng.uniform(-1.0, 1.0, 4 * C).astype(np.float32)
        self.b2, self.gamma, self.beta = (rng.uniform(-0.1, 0.1, C).astype(np.float32), (rng.uniform(-1.0, 1.0, C) + 1.0).astype(np.float32),
                                          rng.uniform(-0.1, 0.1, C).astype(np.float32))
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self.dw1_192, self.dw1_64 = dev(gr.pack_w(self.w1, 192, NKB)), dev(gr.pack_w(self.w1, 64, NKB))
        self.dw2 = dev(gr.pack_w(self.w2, 192, 4 * NKB))
        self.db1, self.db2, self.dgamma, self.dbeta = (dev(v) for v in (self.b1, self.b2, self.gamma, self.beta))

    def ln(self):
        return dict(bias=self.db2.data_ptr(), gamma=self.dgamma.data_ptr(), beta=self.dbeta.data_ptr(), vec_floats=self.C, eps=EPS)

    def two_gemm(self, x0, M: int, grid: int):
        """fc1 -> hidden image, fc2 + LayerNorm + residual in place on a copy of x0 (CTA pairs at C = 384): (stream image,
        hidden image)"""
        C, NKB = self.C, self.C // 64
        hbytes = -(-M // 128) * 4 * NKB * TILE
        hid = Guarded(hbytes)
        run(gp.make_case(kernel=gp.W, epi=EPI_F16_GELU_IMG_FRAG, block_n=192, n=4 * C, n_valid=4 * C, batches=1, grid_sms=grid, nseg=1,
                         m=M, a=[x0.data_ptr()], a_bytes=[x0.numel() * 2], a_batch_stride=[0], a_nkb=[NKB], w=self.dw1_192.data_ptr(),
                         w_bytes=self.dw1_192.numel(), num_kb=NKB, hi=hid.ptr, img_bytes=hbytes, img_nkb=4 * NKB,
                         bias=self.db1.data_ptr(), vec_floats=4 * C))
        out = Guarded(x0.numel() * 2, x0)
        run(gp.make_case(kernel=gp.W if C == 192 else gp.PAIR, epi=EPI_LN_IMG_FRAG, block_n=192, n=C, n_valid=C, batches=1, grid_sms=grid, nseg=1, m=M,
                         a=[hid.ptr], a_bytes=[hbytes], a_batch_stride=[0], a_nkb=[4 * NKB], w=self.dw2.data_ptr(),
                         w_bytes=self.dw2.numel(), num_kb=4 * NKB, hi=out.ptr, img_bytes=out.nbytes, img_nkb=NKB, **self.ln()))
        return out, hid

    def fused(self, x0, M: int, grid: int):
        C, NKB = self.C, self.C // 64
        out = Guarded(x0.numel() * 2, x0)
        run(gp.make_case(kernel=MLP, block_n=192, n=C, n_valid=C, batches=1, grid_sms=grid, m=M, hi=out.ptr, img_bytes=out.nbytes,
                         img_nkb=NKB, w=self.dw1_64.data_ptr(), w_bytes=self.dw1_64.numel(), b_hi=self.dw2.data_ptr(),
                         b_bytes=self.dw2.numel(), add=self.db1.data_ptr(), add_bytes=self.db1.numel() * 4, **self.ln()))
        return out


SHAPES = [("41x96", 1), ("45x192", 1), ("45x192", 3), ("721x1440", 1), ("721x1440", 3)]
GRIDS = {"41x96": pangu_small(41, 96), "45x192": pangu_small(45, 192), "721x1440": pangu_full()}


@pytest.mark.parametrize("grid", [0, 1, 7])   # CTAs, or CTA pairs at C = 384
@pytest.mark.parametrize("name,members", SHAPES)
@pytest.mark.parametrize("C", [192, 384])
def test_fused_mlp_bitwise(C, name, members, grid):
    if name == "721x1440" and grid:
        pytest.skip("the full grid runs on all SMs only (one CTA walks 4,073 tiles per member)")
    NKB = C // 64
    grid = grid if C == 192 else 2 * grid
    M = members * tokens(GRIDS[name], C)
    mlp = Mlp(M + grid, C)
    x0 = image(M, NKB, M)
    ref, _ = mlp.two_gemm(x0, M, grid)
    got = mlp.fused(x0, M, grid)
    got.check(M, NKB, "stream image")
    diff = int((got.t != ref.t).sum())
    print(f"[mlp] C={C} {name} x{members} M={M} grid={grid}: {diff} fp16 values differ from fc1 + fc2")
    assert diff == 0, f"fused MLP: {diff} values differ from fc1 + fc2"
    again = mlp.fused(x0, M, grid)
    assert torch.equal(got.t, again.t), "two launches differ"


def test_fused_mlp_fp64_bound():
    """41 x 96 grid, every row: the hidden image within the fp64 bound of GELU(x W1^T + b1) and the stream image within
    the bound of LN(h W2^T + b2) * gamma + beta + x, h being the hidden image the fused result is bit for bit built from"""
    C, NKB = 192, 3
    M = tokens(GRIDS["41x96"], C)
    mlp = Mlp(5, C)
    x0 = image(M, NKB, 11)
    ref, hid = mlp.two_gemm(x0, M, 0)
    got = mlp.fused(x0, M, 0)
    assert torch.equal(got.t, ref.t)
    rows = np.arange(M)
    x = image_rows(x0, rows, NKB)
    R, S = gr.linear([(x, mlp.w1)])
    f, fb = gr.epi_gelu(*gr.epi_affine(R, S, mlp.b1[None, :]))
    h = image_rows(hid.inner(), rows, 4 * NKB)
    rh = gr.worst(h.astype(np.float64), f, gr.f16_bound(f, fb))
    R2, S2 = gr.linear([(h, mlp.w2)])
    y, yb = gr.layer_norm(R2, S2, mlp.b2[None, :], mlp.gamma[None, :], mlp.beta[None, :], x.astype(np.float64), EPS)
    ry = gr.worst(image_rows(got.inner(), rows, NKB).astype(np.float64), y, yb + 0.5 * gr.ulp16(np.abs(y) + yb))
    print(f"[mlp] fp64 bound, M={M}: hidden max err/bound {rh:.3f}, result {ry:.3f}")
    assert rh <= 1.0 and ry <= 1.0, (rh, ry)
