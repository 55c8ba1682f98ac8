"""Kernel-level tests of Pangu's windowing kernels against the float64 references of oracle/pangu_kernels_ref.py,
element by element: the QKV projection's epilogue EpiQkvWin (natural tokens -> rolled, padded window image),
k_qkv_fill_pad (the latitude-padding rows), k_window_attention_tc (scores, bias gather, shift mask, softmax, P V, scatter
to the projection's operand image) and k_pack_bias_table.

Each case launches through libskyrim_b200_probe.so (sky_probe_gemm / sky_probe_pangu, oracle/gemm_probe.py) at the token
grids the engine builds: pangu_small(41, 96) (g1 H 11 -> Hp 12; g2 H 6, a single h-window row), pangu_small(33, 96)
(pad 3 / pad 1), pangu_small(45, 192) (no pad) and the full 721 x 1440 grids (g1 181 -> 186, g2 91 -> 96), at roll 0 / 1
and one or three members.  The protocol of tests/test_gemm_kernels_gpu.py:
  * output buffers have guard bands and are filled with an fp16 NaN sentinel; after the launches the sentinel must be
    intact outside the written region (the gaps between the q, k, v parts, the rows past B T of the last output tile)
    and gone inside it;
  * the A image's rows past M are NaN;
  * the separate launches are repeated and must agree bit for bit;
  * every value is within its per-element bound; pytest -s prints the largest err / bound of each case.
The attention inputs make the softmaxes peaked (oracle: attention_inputs), so that a wrong bias entry, mask, padding
row or window shows (tests/test_pangu_kernels_cpu.py checks that each such mistake leaves the bound); one case keeps the
synthetic weights' scale.  The full-size grids are checked through the chained QKV -> attention path: coverage and
sentinels over the whole buffers, values on every window of the first and last latitude rows of windows of the first
and last member, plus a seeded random sample.
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
GAP = 4096               # bytes between the q, k and v parts beyond what they need

SMALL = {f"{nlat}x{nlon}-g{i + 1}": g for nlat, nlon in [(41, 96), (33, 96), (45, 192)]
         for i, g in enumerate(pk.grids(pangu_small(nlat, nlon)))}
FULL = {f"721x1440-g{i + 1}": g for i, g in enumerate(pk.grids(pangu_full()))}
SEED = 7                 # the inputs tests/test_pangu_kernels_cpu.py's discrimination test uses


# ---------------------------------------------------------------------------------------------------------------------
# device buffers
# ---------------------------------------------------------------------------------------------------------------------
def dev(arr: np.ndarray):
    t = torch.from_numpy(np.ascontiguousarray(arr).reshape(-1).view(np.uint8).copy()).cuda()
    return t, t.data_ptr(), t.numel()


class Guarded:
    """`nbytes` of device memory between two guard bands, all holding the fp16 sentinel"""

    def __init__(self, nbytes: int):
        assert nbytes % 2 == 0
        self.nbytes = nbytes
        self.t = torch.full(((2 * GUARD + nbytes) // 2,), SENT, dtype=torch.int16, device="cuda")
        self.ptr = self.t.data_ptr() + GUARD

    def inner(self):
        return self.t[GUARD // 2: GUARD // 2 + self.nbytes // 2]

    def check_guards(self, what):
        g = GUARD // 2
        assert bool((self.t[:g] == SENT).all()) and bool((self.t[-g:] == SENT).all()), f"{what}: guard band overwritten"


def run_gemm(case):
    rc, msg = gp.launch(case)
    assert rc == 0, msg
    torch.cuda.synchronize()


def run_pangu(case):
    rc, msg = gp.launch_pangu(case)
    assert rc == 0, msg
    torch.cuda.synchronize()


def record(name, got, ref, bound):
    r = gr.worst(got, ref, bound)
    print(f"[pangu] {name}: max err/bound {r:.3f}")
    assert r <= 1.0, f"{name}: error exceeds its bound by {r:.3f}x"


def image_rows(img: "torch.Tensor", rows: np.ndarray, nkb: int) -> np.ndarray:
    """rows of a 128-row tile image on the device (int16 view) -> fp16 [len(rows), nkb * 64] on the host"""
    v = img.view(-1, nkb, 128, 8, 8)
    r = torch.from_numpy(np.asarray(rows, np.int64)).cuda()
    sel = v[r // 128, :, r % 128].cpu().numpy()                               # [n, nkb, 8 stored chunks, 8]
    idx = gr._swz_index(128)[np.asarray(rows) % 128][:, None, :, None]
    return np.take_along_axis(sel, np.broadcast_to(idx, sel.shape), axis=2).reshape(len(rows), nkb * 64).view(np.float16)


def window_geometry(g, roll, B):
    tiles = B * g.nWin * g.pairs
    ps = tiles * pk.TILE_B + GAP
    return tiles, ps, 2 * ps + tiles * pk.TILE_B


def parts_view(buf: Guarded, tiles: int, ps: int):
    """(data [3, tiles, 144, 64], gaps [2, GAP / 2]) of a window image buffer, int16 on the device"""
    h = buf.inner()
    data = torch.stack([h[p * ps // 2: p * ps // 2 + tiles * pk.TILE_B // 2] for p in range(3)]).view(3, tiles, pk.NTOK, 64)
    gaps = torch.stack([h[p * ps // 2 + tiles * pk.TILE_B // 2: (p + 1) * ps // 2] for p in range(2)])
    return data, gaps


def pad_rows_mask(g, roll, B):
    """[tiles, 144] True at the rows of latitude-padding tokens (every part, every pair)"""
    idx = pk.window_tokens(g, roll, B)                                      # [B, nWin, 144]
    return np.repeat((idx < 0)[:, :, None, :], g.pairs, axis=2).reshape(-1, pk.NTOK)


def qkv_operands(g, B, seed, device_x=False):
    """x (natural tokens, fp16 tile image with NaN rows past M), the QKV weights [3C, C] (fp16) and bias [3C] (fp32).
    Scores of the resulting q, k span several units (q, k ~ uniform with std ~1.7)."""
    rng = np.random.default_rng(seed)
    M, nkb = B * g.T, g.C // 64
    w = (rng.uniform(-1, 1, (3 * g.C, g.C)) * 5 / np.sqrt(g.C)).astype(np.float16)
    bias = rng.uniform(-1, 1, 3 * g.C).astype(np.float32)
    if device_x:   # the image itself is random fp16 (made on the device); x is whatever it holds
        gen = torch.Generator(device="cuda").manual_seed(seed)
        nt = -(-M // 128)
        a = (torch.rand(nt * nkb * 128 * 64, generator=gen, device="cuda") * 2 - 1).half().view(nt, nkb, 128, 64)
        if M % 128:
            a[-1, :, M % 128:] = float("nan")
        return a.view(torch.int16).reshape(-1), w, bias
    x = rng.uniform(-1, 1, (M, g.C)).astype(np.float16)
    return torch.from_numpy(gr.pack_tiles(x, 128, nkb, row_fill=np.nan).view(np.int16).copy()).cuda(), w, bias


def qkv_case(g, roll, B, a_img, w_dev, b_dev, buf, ps, img_bytes):
    nkb = g.C // 64
    return gp.make_case(kernel=gp.W, epi=gp.EPI_QKV_WIN, block_n=192, n=3 * g.C, n_valid=3 * g.C, batches=1, grid_sms=0, nseg=1,
                        m=B * g.T, a=[a_img.data_ptr()], a_bytes=[a_img.numel() * 2], a_batch_stride=[0], a_nkb=[nkb],
                        w=w_dev[1], w_bytes=w_dev[2], w_batch_stride=0, num_kb=nkb, w_rep=0, hi=buf.ptr, img_bytes=img_bytes,
                        bias=b_dev[1], vec_floats=3 * g.C, geo=g.probe_geo(), roll=roll, pairs=g.pairs, part_stride=ps)


def fill_case(g, roll, B, b_dev, buf, ps, img_bytes):
    return gp.make_pangu_case(op=gp.PG_FILL_PAD, geo=g.probe_geo(), roll=roll, B=B, pairs=g.pairs, n_type=g.n_type,
                              part_stride=ps, qkv=buf.ptr, qkv_bytes=img_bytes, src=b_dev[1], src_floats=3 * g.C)


def attention_case(g, roll, B, qkv_ptr, ps, img_bytes, tab_dev, out):
    sl2, ml2 = pk.sl2_mask_l2()
    return gp.make_pangu_case(op=gp.PG_ATTENTION, geo=g.probe_geo(), roll=roll, B=B, pairs=g.pairs, n_type=g.n_type,
                              att_nkb=g.C // 64, part_stride=ps, qkv=qkv_ptr, qkv_bytes=img_bytes, tab=tab_dev[1],
                              tab_bytes=tab_dev[2], out=out.ptr, out_bytes=out.nbytes, sl2=sl2, mask_l2=ml2)


def att_bytes(g, B):
    return -(-B * g.T // 128) * (g.C // 64) * TILE


def check_att_coverage(out: Guarded, g, B, what):
    """every element of rows < B T written, every row past B T of the last tile still the sentinel"""
    nkb, M = g.C // 64, B * g.T
    v = out.inner().view(-1, nkb, 128, 64)
    full, rem = divmod(M, 128)
    assert not bool((v[:full] == SENT).any()), f"{what}: a token's output was not written"
    if rem:
        assert not bool((v[full, :, :rem] == SENT).any()), f"{what}: a token's output was not written"
        assert bool((v[full, :, rem:] == SENT).all()), f"{what}: rows past B T were written"
    out.check_guards(what)


# ---------------------------------------------------------------------------------------------------------------------
# k_pack_bias_table: bit-exact
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["41x96-g1", "41x96-g2", "721x1440-g1", "721x1440-g2"])
def test_pack_bias_table(name):
    g = {**SMALL, **FULL}[name]
    rng = np.random.default_rng(1)
    # O(1) entries, and entries whose x log2 e overflows fp16 or falls into its subnormals
    table = (rng.standard_normal((pk.TABLE, g.n_type, g.heads)) * 2).astype(np.float32)
    table.reshape(-1)[:64] = np.float32(1e5) * rng.uniform(-1, 1, 64).astype(np.float32)
    table.reshape(-1)[64:128] = np.float32(1e-6) * rng.uniform(-1, 1, 64).astype(np.float32)
    want = pk.pack_bias_table(table)
    src = dev(table)
    out = Guarded(want.nbytes + 64)
    run_pangu(gp.make_pangu_case(op=gp.PG_PACK_BIAS, geo=g.probe_geo(), roll=0, B=1, pairs=g.pairs, n_type=g.n_type,
                                 src=src[1], src_floats=table.size, out=out.ptr, out_bytes=want.nbytes))
    got = out.inner().cpu().numpy()
    assert np.array_equal(got[: want.size], want.reshape(-1).view(np.int16)), "packed tables differ"
    assert (got[want.size:] == SENT).all()
    out.check_guards("bias tables")
    print(f"[pangu] pack_bias_table {name}: bit-exact over {want.size} entries")


# ---------------------------------------------------------------------------------------------------------------------
# EpiQkvWin + k_qkv_fill_pad
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("roll", [0, 1])
@pytest.mark.parametrize("name", list(SMALL))
def test_qkv_window_image(name, roll, B):
    g = SMALL[name]
    tiles, ps, img_bytes = window_geometry(g, roll, B)
    a_img, w, bias = qkv_operands(g, B, 100 + B)
    x = gr.unpack_tiles(a_img.cpu().numpy().view(np.uint8), 128, g.C // 64, B * g.T, g.C)
    w_dev, b_dev = dev(gr.pack_w(w, 192, g.C // 64)), dev(bias)
    padded = g.Hp > g.H
    pad = pad_rows_mask(g, roll, B)

    def launch(buf, epi=True, fill=True):
        if epi:
            run_gemm(qkv_case(g, roll, B, a_img, w_dev, b_dev, buf, ps, img_bytes))
        if fill and padded:
            run_pangu(fill_case(g, roll, B, b_dev, buf, ps, img_bytes))

    # the two writers partition the rows: the epilogue writes exactly the token rows, k_qkv_fill_pad the padding rows
    for epi, fill, rows_written in [(True, False, ~pad)] + ([(False, True, pad)] if padded else []):
        buf = Guarded(img_bytes)
        launch(buf, epi, fill)
        data, gaps = parts_view(buf, tiles, ps)
        d = data.cpu().numpy()
        written = (d != SENT).any(-1)                                      # [3, tiles, 144]
        untouched = (d == SENT).all(-1)
        assert (written == rows_written[None]).all() and (untouched == ~rows_written[None]).all(), \
            f"{'epilogue' if epi else 'fill-pad'}: rows written {written.sum()} (expected {3 * rows_written.sum()}), or a row partly"
        assert bool((gaps == SENT).all()), "gap between parts written"
        buf.check_guards("window image")
    bufs = [Guarded(img_bytes) for _ in range(2)]
    for b in bufs:
        launch(b)
    assert torch.equal(bufs[0].t, bufs[1].t), "two launches differ"
    data, gaps = parts_view(bufs[0], tiles, ps)
    assert not bool((data == SENT).any()), "a row of the window image was not written"
    assert bool((gaps == SENT).all())
    bufs[0].check_guards("window image")
    got = pk.unpack_window_image(bufs[0].inner().cpu().numpy().view(np.uint8), g, B, ps)
    ref_tok, bnd_tok = pk.qkv_ref(x, w, bias)
    idx = pk.window_tokens(g, roll, B)
    ref = pk.windows_from_tokens(ref_tok, bias.astype(np.float16).astype(np.float64), idx, g.heads)
    bnd = pk.windows_from_tokens(bnd_tok, np.zeros(3 * g.C), idx, g.heads)   # padding rows: fp16(bias) exactly
    record(f"qkv window image {name} roll {roll} B {B}", got, ref, bnd)


# ---------------------------------------------------------------------------------------------------------------------
# k_window_attention_tc alone, fed an oracle-packed window image
# ---------------------------------------------------------------------------------------------------------------------
ATT_CASES = [(n, r, B, False) for n in SMALL for r in (0, 1) for B in (1, 3)] + [("41x96-g1", 1, 1, True)]


@pytest.mark.parametrize("name,roll,B,synthetic", ATT_CASES)
def test_attention(name, roll, B, synthetic):
    g = SMALL[name]
    inp = pk.attention_inputs(g, B, SEED, synthetic)
    tiles, ps, img_bytes = window_geometry(g, roll, B)
    idx = pk.window_tokens(g, roll, B)
    img = pk.pack_window_image(pk.windows_from_tokens(inp.qkv_tok, inp.pad_row, idx, g.heads), ps)
    qkv_dev, tab_dev = dev(img), dev(pk.pack_bias_table(inp.table))
    outs = [Guarded(att_bytes(g, B)) for _ in range(2)]
    for o in outs:
        run_pangu(attention_case(g, roll, B, qkv_dev[1], ps, img_bytes, tab_dev, o))
    assert torch.equal(outs[0].t, outs[1].t), "two launches differ"
    check_att_coverage(outs[0], g, B, "attention output")
    got = gr.unpack_tiles(outs[0].inner().cpu().numpy().view(np.uint8), 128, g.C // 64, B * g.T, g.C)
    ref, bnd = pk.attention_tokens(g, B, roll, inp)
    record(f"attention {name} roll {roll} B {B}{' synthetic scale' if synthetic else ''}", got, ref, bnd)


# ---------------------------------------------------------------------------------------------------------------------
# QKV -> fill-pad -> attention chained: producer and consumer agree on the layout with each other and with the oracle
# ---------------------------------------------------------------------------------------------------------------------
def sample_windows(g, B, full: bool, seed: int):
    """(member, window) pairs: all of them, or every window of the first and last latitude rows of windows of the first
    and last member plus a seeded random sample"""
    if not full:
        return [(b, w) for b in range(B) for w in range(g.nWin)]
    wh = np.arange(g.nWin) // g.nWw % g.nWh
    edge = np.flatnonzero((wh == 0) | (wh == g.nWh - 1))
    s = {(b, int(w)) for b in sorted({0, B - 1}) for w in edge}
    rng = np.random.default_rng(seed)
    s |= {(int(b), int(w)) for b, w in zip(rng.integers(0, B, 32), rng.integers(0, g.nWin, 32))}
    return sorted(s)


CHAIN_CASES = [(n, 1, 3) for n in SMALL] + [(n, r, B) for n in FULL for r in (0, 1) for B in (1, 3)]


@pytest.mark.parametrize("name,roll,B", CHAIN_CASES)
def test_qkv_attention_chained(name, roll, B):
    full = name in FULL
    g = {**SMALL, **FULL}[name]
    nkb = g.C // 64
    tiles, ps, img_bytes = window_geometry(g, roll, B)
    a_img, w, bias = qkv_operands(g, B, 200 + B + roll, device_x=True)
    w_dev, b_dev = dev(gr.pack_w(w, 192, nkb)), dev(bias)
    table = (np.random.default_rng(3).uniform(-2, 2, (pk.TABLE, g.n_type, g.heads))).astype(np.float32)
    src = dev(table)
    tab = Guarded(2 * table.size)
    run_pangu(gp.make_pangu_case(op=gp.PG_PACK_BIAS, geo=g.probe_geo(), roll=0, B=1, pairs=g.pairs, n_type=g.n_type,
                                 src=src[1], src_floats=table.size, out=tab.ptr, out_bytes=tab.nbytes))
    tab16 = tab.inner().cpu().numpy().view(np.float16).reshape(g.n_type, g.heads, pk.TABLE)
    assert np.array_equal(tab16.view(np.uint16), pk.pack_bias_table(table).view(np.uint16))
    img = Guarded(img_bytes)
    run_gemm(qkv_case(g, roll, B, a_img, w_dev, b_dev, img, ps, img_bytes))
    if g.Hp > g.H:
        run_pangu(fill_case(g, roll, B, b_dev, img, ps, img_bytes))
    out = Guarded(att_bytes(g, B))
    run_pangu(attention_case(g, roll, B, img.ptr, ps, img_bytes, (None, tab.ptr, tab.nbytes), out))
    # coverage over the whole buffers
    data, gaps = parts_view(img, tiles, ps)
    assert not bool((data == SENT).any()), "a row of the window image was not written"
    assert bool((gaps == SENT).all())
    img.check_guards("window image")
    check_att_coverage(out, g, B, "attention output")
    # values on the sampled windows: the x rows they hold, read back from the A image the GEMM read
    samples = sample_windows(g, B, full, seed=5)
    idx_all = pk.window_tokens(g, roll, B)
    idx = np.stack([idx_all[b, w] for b, w in samples])                        # [n, 144]
    types = np.array([w // g.nWw for _, w in samples])
    toks = np.unique(idx[idx >= 0])
    x = image_rows(a_img, toks, nkb)
    del a_img
    ref_tok, bnd_tok = pk.qkv_ref(x, w, bias)
    local = np.where(idx >= 0, np.searchsorted(toks, np.maximum(idx, 0)), -1)
    ref_w = pk.windows_from_tokens(ref_tok, bias.astype(np.float16).astype(np.float64), local, g.heads)
    bnd_w = pk.windows_from_tokens(bnd_tok, np.zeros(3 * g.C), local, g.heads)
    tile_ids = np.array([(b * g.nWin + w) * g.pairs + p for b, w in samples for p in range(g.pairs)])
    sel = data[:, torch.from_numpy(tile_ids).cuda()].cpu().numpy()               # [3, n * pairs, 144, 64]
    got_w = pk.unpack_tiles(sel.reshape(3, len(samples), g.pairs, pk.NTOK * 64)).reshape(3, len(samples), g.heads, pk.NTOK, 32)
    record(f"chained qkv window image {name} roll {roll} B {B} ({len(samples)} windows)", got_w, ref_w, bnd_w)
    # attention from the window image exactly as the kernel read it
    sl2, ml2 = pk.sl2_mask_l2()
    mask = pk.shift_mask_types(g) if roll else None
    o, ob = pk.attention_windows(got_w[0], got_w[1], got_w[2], tab16, types, mask, ml2, sl2)
    valid = idx.reshape(-1) >= 0
    ref_o = o.transpose(0, 2, 1, 3).reshape(-1, g.C)[valid]
    bnd_o = ob.transpose(0, 2, 1, 3).reshape(-1, g.C)[valid]
    got_o = image_rows(out.inner(), idx.reshape(-1)[valid], nkb)
    record(f"chained attention {name} roll {roll} B {B} ({len(samples)} windows)", got_o, ref_o, bnd_o)
