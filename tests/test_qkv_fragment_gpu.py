"""The QKV projection's fragment epilogue (FragEpi<EpiQkvWin>) at the full 721 x 1440 token grids, through sky_probe_gemm
(epilogue id 17): the epilogue writes the fp16 window image from the accumulator registers into a shared-memory output tile,
and the loader warp bulk-stores that tile in runs of consecutive window rows.

At both grids (C = 192 and C = 384), roll 0 / 1 and one / three members (partial last m-tiles, and m-tiles that straddle two
members) it checks that
  * the window image is bit for bit the same for grids of 1 CTA, 7 CTAs and one CTA per SM: a single CTA walks every tile
    through the single-buffered output tile, and the run splitting does not depend on which CTA stores a tile;
  * the GEMM writes exactly the token rows and k_qkv_fill_pad exactly the latitude-padding rows, each row whole;
  * the guard bands around the buffer and the gaps between the q, k and v parts keep the fp16 NaN sentinel.
The values themselves are checked against the fp64 oracle by tests/test_pangu_kernels_gpu.py.
"""
from __future__ import annotations

import numpy as np
import pytest

from oracle import gemm_probe as gp
from oracle import gemm_ref as gr
from oracle import pangu_kernels_ref as pk
from skyrim_b200.config import pangu_full

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

GUARD = 16384
SENT = 0x7D5A            # fp16 NaN bit pattern
GAP = 4096               # bytes between the q, k and v parts beyond what they need
FULL = {f"721x1440-g{i + 1}": g for i, g in enumerate(pk.grids(pangu_full()))}


class Guarded:
    """`nbytes` of device memory between two guard bands, all holding the sentinel"""

    def __init__(self, nbytes: int):
        self.nbytes = nbytes
        self.t = torch.full(((2 * GUARD + nbytes) // 2,), SENT, dtype=torch.int16, device="cuda")
        self.ptr = self.t.data_ptr() + GUARD

    def guards_intact(self) -> bool:
        g = GUARD // 2
        return bool((self.t[:g] == SENT).all()) and bool((self.t[-g:] == SENT).all())


def run(launch, case):
    rc, msg = launch(case)
    assert rc == 0, msg
    torch.cuda.synchronize()


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("roll", [0, 1])
@pytest.mark.parametrize("name", list(FULL))
def test_qkv_fragment_full_grid(name, roll, B):
    g = FULL[name]
    C, nkb, M = g.C, g.C // 64, B * g.T
    assert M % 128, "a partial last m-tile (and, with B = 3, m-tiles that straddle two members)"
    tiles = B * g.nWin * g.pairs
    ps = tiles * pk.TILE_B + GAP
    img_bytes = 2 * ps + tiles * pk.TILE_B

    gen = torch.Generator(device="cuda").manual_seed(300 + 2 * B + roll)
    nt = -(-M // 128)
    a = (torch.rand(nt * nkb * 128 * 64, generator=gen, device="cuda") * 2 - 1).half().view(nt, nkb, 128, 64)
    a[-1, :, M % 128:] = float("nan")   # rows past M: a row the GEMM must not store would carry NaN
    rng = np.random.default_rng(300 + 2 * B + roll)
    w = (rng.uniform(-1, 1, (3 * C, C)) * 5 / np.sqrt(C)).astype(np.float16)
    w_img = torch.from_numpy(np.ascontiguousarray(gr.pack_w(w, 192, nkb)).reshape(-1).view(np.uint8).copy()).cuda()
    bias = torch.from_numpy(rng.uniform(-1, 1, 3 * C).astype(np.float32)).cuda()

    def gemm(buf, grid_sms):
        return gp.make_case(kernel=gp.W, epi=gp.EPI_QKV_WIN, block_n=192, n=3 * C, n_valid=3 * C, batches=1,
                            grid_sms=grid_sms, nseg=1, m=M, a=[a.data_ptr()], a_bytes=[a.numel() * 2], a_batch_stride=[0],
                            a_nkb=[nkb], w=w_img.data_ptr(), w_bytes=w_img.numel(), w_batch_stride=0, num_kb=nkb, w_rep=0,
                            hi=buf.ptr, img_bytes=img_bytes, bias=bias.data_ptr(), vec_floats=3 * C, geo=g.probe_geo(),
                            roll=roll, pairs=g.pairs, part_stride=ps)

    def fill(buf):
        return gp.make_pangu_case(op=gp.PG_FILL_PAD, geo=g.probe_geo(), roll=roll, B=B, pairs=g.pairs, n_type=g.n_type,
                                  part_stride=ps, qkv=buf.ptr, qkv_bytes=img_bytes, src=bias.data_ptr(), src_floats=3 * C)

    def rows_and_gaps(buf):
        """([3, tiles, 144] rows with any element written, [3, tiles, 144] rows with every element written, gaps intact)"""
        h = buf.t[GUARD // 2: GUARD // 2 + img_bytes // 2]
        written = torch.empty((3, tiles, pk.NTOK), dtype=torch.bool, device="cuda")
        whole = torch.empty_like(written)
        for p in range(3):
            d = h[p * ps // 2: p * ps // 2 + tiles * pk.TILE_B // 2].view(tiles, pk.NTOK, 64) != SENT
            written[p], whole[p] = d.any(-1), d.all(-1)
        gaps = all(bool((h[p * ps // 2 + tiles * pk.TILE_B // 2: (p + 1) * ps // 2] == SENT).all()) for p in range(2))
        return written, whole, gaps

    pad = torch.from_numpy(np.repeat((pk.window_tokens(g, roll, B) < 0)[:, :, None, :], g.pairs, axis=2)
                           .reshape(-1, pk.NTOK)).cuda()[None].expand(3, -1, -1)
    assert bool(pad.any()), "the full-size grids have latitude-padding rows"

    # the two writers partition the rows of the window image, each writing whole rows
    for writer, rows in (("GEMM", ~pad), ("k_qkv_fill_pad", pad)):
        buf = Guarded(img_bytes)
        if writer == "GEMM":
            run(gp.launch, gemm(buf, 0))
        else:
            run(gp.launch_pangu, fill(buf))
        written, whole, gaps = rows_and_gaps(buf)
        assert torch.equal(written, rows), f"{writer}: wrote {int(written.sum())} rows, expected {int(rows.sum())}"
        assert torch.equal(whole, rows), f"{writer}: a row partly written"
        assert gaps and buf.guards_intact(), f"{writer}: gap between parts or guard band written"
        del buf

    # the whole image, bit for bit the same whichever CTA stores a tile
    ref = None
    for grid_sms in (0, 1, 7):
        buf = Guarded(img_bytes)
        run(gp.launch, gemm(buf, grid_sms))
        run(gp.launch_pangu, fill(buf))
        if ref is None:
            written, _, gaps = rows_and_gaps(buf)
            assert bool(written.all()), "a row of the window image was not written"
            assert gaps and buf.guards_intact()
            ref = buf
        else:
            assert torch.equal(buf.t, ref.t), f"grid of {grid_sms} CTAs: window image differs from one CTA per SM"
            del buf
    print(f"[qkv fragment] {name} roll {roll} B {B}: {tiles * 3 * pk.NTOK} rows, partition and grids 1 / 7 / SMs bit-exact")

