"""CPU checks of the kernel-level test machinery of Pangu's windowing kernels (oracle/pangu_kernels_ref.py,
oracle/gemm_probe.py): the window image layout, the float64 attention reference against PanguRef, that the attention
bound separates the correct kernel from each plausible mistake at the inputs the GPU tests use, the bias-table
repacking, and that the probe refuses inconsistent cases on the host (without touching a device)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from oracle import gemm_probe as gp
from oracle import gemm_ref as gr
from oracle import pangu_kernels_ref as pk
from oracle.pangu_ref import PanguRef
from skyrim_b200.config import pangu_small

G41 = pk.grids(pangu_small(41, 96))     # g1: H 11 -> Hp 12; g2: H 6, one h-window row
DISCRIM_SEED = 7                         # the inputs of the GPU attention cases (tests/test_pangu_kernels_gpu.py SEED)


# ---------------------------------------------------------------------------------------------------------------------
# layout
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gi,B,gap", [(0, 1, 0), (1, 2, 4096)])
def test_window_image_round_trip(gi, B, gap):
    g = G41[gi]
    rng = np.random.default_rng(gi)
    x = rng.standard_normal((3, B, g.nWin, g.heads, pk.NTOK, 32)).astype(np.float16)
    ps = B * g.nWin * g.pairs * pk.TILE_B + gap
    img = pk.pack_window_image(x, ps)
    assert img.size == 2 * ps + B * g.nWin * g.pairs * pk.TILE_B
    back = pk.unpack_window_image(img, g, B, ps)
    assert np.array_equal(back.view(np.uint16), x.view(np.uint16))
    if gap:
        h = img.view(np.float16)
        assert np.isnan(h[ps // 2 - gap // 2: ps // 2]).all()


def test_window_image_hand_computed_offsets():
    """single elements, their byte offsets worked out by hand from part * part_stride + tile * 18432 + j * 128 +
    ((chunk ^ (j & 7)) << 4) + 2 * half, tile = (member * nWin + window) * pairs + pair"""
    g, B = G41[0], 2                                     # nWin 16, 3 pairs
    ps = B * g.nWin * g.pairs * pk.TILE_B
    cases = [
        # (part, b, win, head, j, d, offset): k, member 1, window 5, head 3 (pair 1, second head), row 17, dim 9 ->
        # tile (16 + 5) * 3 + 1 = 64, chunk (32 + 9) // 8 = 5 stored at 5 ^ 1 = 4, half 1
        (1, 1, 5, 3, 17, 9, ps + 64 * 18432 + 17 * 128 + (4 << 4) + 2),
        # q, member 0, window 0, head 0, row 0, dim 0 -> byte 0
        (0, 0, 0, 0, 0, 0, 0),
        # v, member 0, window 15, head 4 (pair 2, first head), row 143, dim 31 -> tile 15 * 3 + 2 = 47, chunk 3 stored at
        # 3 ^ 7 = 4, half 7
        (2, 0, 15, 4, 143, 31, 2 * ps + 47 * 18432 + 143 * 128 + (4 << 4) + 14),
    ]
    for part, b, win, head, j, d, off in cases:
        x = np.zeros((3, B, g.nWin, g.heads, pk.NTOK, 32), np.float16)
        x[part, b, win, head, j, d] = 1.0
        img = pk.pack_window_image(x, ps).view(np.float16)
        assert pk.window_image_offset(g, B, ps, part, b, win, head, j, d) == off
        assert np.flatnonzero(img).tolist() == [off // 2]


def test_window_tokens_by_hand():
    """window rows -> natural tokens, worked out from the pad-then-roll definition"""
    g = G41[0]                                            # Z 8, H 11 (Hp 12), W 24
    idx = pk.window_tokens(g, 0, 2)
    # window (wz 1, wh 1, ww 1) = 7, row (zj 1, hj 2, wj 3): z 3, h 8, w 15
    assert idx[0, 7, (1 * 6 + 2) * 12 + 3] == (3 * 11 + 8) * 24 + 15
    assert idx[1, 7, (1 * 6 + 2) * 12 + 3] == g.T + (3 * 11 + 8) * 24 + 15
    # h = 11 is padding
    assert idx[0, 7, (0 * 6 + 5) * 12 + 0] == -1
    rolled = pk.window_tokens(g, 1, 1)
    # rolled grid position (z 7, h 11, w 23) holds natural (0, 2, 5): window (3, 1, 1) = 15, row (1, 5, 11)
    assert rolled[0, 15, (1 * 6 + 5) * 12 + 11] == (0 * 11 + 2) * 24 + 5
    # rolled position (0, 8, 0) holds natural h = 11: padding
    assert rolled[0, 1 * 2 + 0, (0 * 6 + 2) * 12 + 0] == -1
    # every natural token appears exactly once; the padding rows are Z * (Hp - H) * W
    for r in (0, 1):
        i = pk.window_tokens(g, r, 2).reshape(-1)
        assert np.array_equal(np.sort(i[i >= 0]), np.arange(2 * g.T))
        assert (i < 0).sum() == 2 * g.Z * (g.Hp - g.H) * g.W


def test_seam_masks_make_up_the_shift_mask():
    for g in G41 + pk.grids(pangu_small(33, 96)):
        z, h = pk.seam_masks(g)
        assert np.array_equal(z | h, pk.shift_mask_types(g))
        assert z.any() and h.any()


# ---------------------------------------------------------------------------------------------------------------------
# the attention reference against PanguRef (float64 throughout, no fp16 rounding anywhere)
# ---------------------------------------------------------------------------------------------------------------------
def _ref_weights(g, rng, p):
    C = g.C
    return {p + "qkv.w": rng.standard_normal((3 * C, C)) / np.sqrt(C) * 2, p + "qkv.b": rng.standard_normal(3 * C),
            p + "bias_table": rng.uniform(-2, 2, (pk.TABLE, g.n_type, g.heads)),
            p + "proj.w": np.eye(C), p + "proj.b": np.zeros(C),
            p + "ln1.g": np.ones(C), p + "ln1.b": np.zeros(C)}


def _fp64_windows(g, roll, x, w, p):
    """this module's pipeline in float64: tokens -> windows -> attention -> tokens"""
    idx = pk.window_tokens(g, roll, 1)
    qkv = x.reshape(g.T, g.C) @ w[p + "qkv.w"].T + w[p + "qkv.b"]
    q, k, v = pk.windows_from_tokens(qkv, w[p + "qkv.b"], idx, g.heads)[:, 0]
    tab = w[p + "bias_table"].transpose(1, 2, 0) * pk.LOG2E
    mask = pk.shift_mask_types(g) if roll else None
    bias = pk.gathered_bias(tab, pk.window_types(g), mask, -100.0 * pk.LOG2E, round16=False)
    o, _ = pk.attention_ref(q, k, v, bias, 32 ** -0.5 * pk.LOG2E)
    return pk.tokens_from_windows(o[None], idx, g.T)


def test_attention_ref_matches_pangu_ref_attention():
    cfg = pangu_small(41, 96)
    g = G41[0]
    rng = np.random.default_rng(11)
    p = "l."
    w = _ref_weights(g, rng, p)
    ref = PanguRef(cfg, w, dtype=torch.float64)
    xw = rng.standard_normal((g.n_type, g.nWw, pk.NTOK, g.C))
    mask = ref._mask(g.Z, g.Hp, g.W)
    want = ref.attention(torch.from_numpy(xw), p, g.heads, g.n_type, mask).numpy()
    qkv = xw @ w[p + "qkv.w"].T + w[p + "qkv.b"]
    q, k, v = np.moveaxis(qkv.reshape(g.nWin, pk.NTOK, 3, g.heads, 32), 2, 0).transpose(0, 1, 3, 2, 4)
    tab = w[p + "bias_table"].transpose(1, 2, 0) * pk.LOG2E
    bias = pk.gathered_bias(tab, pk.window_types(g), pk.shift_mask_types(g), -100.0 * pk.LOG2E, round16=False)
    o, _ = pk.attention_ref(q, k, v, bias, 32 ** -0.5 * pk.LOG2E)
    got = o.transpose(0, 2, 1, 3).reshape(g.n_type, g.nWw, pk.NTOK, g.C)
    np.testing.assert_allclose(got, want, rtol=1e-11, atol=1e-11)


class _Stop(Exception):
    pass


@pytest.mark.parametrize("gi,roll", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_windowing_matches_pangu_ref_block(monkeypatch, gi, roll):
    """PanguRef.block's attention output before LayerNorm (pad, roll, window, attend, un-window, roll back, crop) equals
    this module's windows at roll 0 / 1, with a padded H (g1: 11 -> 12) and without (g2)"""
    cfg = pangu_small(41, 96)
    g = G41[gi]
    rng = np.random.default_rng(20 + gi)
    p = "l."
    w = _ref_weights(g, rng, p)
    ref = PanguRef(cfg, w, dtype=torch.float64)
    x = rng.standard_normal((g.Z, g.H, g.W, g.C))
    seen = []

    def capture(y, *a, **k):
        seen.append(y.detach().numpy().copy())
        raise _Stop

    monkeypatch.setattr(torch.nn.functional, "layer_norm", capture)
    with pytest.raises(_Stop):
        ref.block(torch.from_numpy(x), p, g.heads, roll)
    got = _fp64_windows(g, roll, x, w, p)
    np.testing.assert_allclose(got, seen[0].reshape(g.T, g.C), rtol=1e-11, atol=1e-11)


# ---------------------------------------------------------------------------------------------------------------------
# discrimination: at the GPU case's inputs, every modelled kernel mistake leaves the bound at some element
# ---------------------------------------------------------------------------------------------------------------------
def _pos_wrong_sign():
    zi, hi, wi = pk.row_position(np.arange(pk.NTOK))
    return pk.position_index() + 2 * (wi[None, :] - wi[:, None])       # wj - wi instead of wi - wj


def _mutations(g):
    z_seam, h_seam = pk.seam_masks(g)
    return {
        "relative-longitude index with the wrong sign": dict(pos=_pos_wrong_sign()),
        "query and key roles of the table index swapped": dict(pos=pk.position_index().T.copy()),
        "heads of the bias table in reverse order": dict(head_perm=np.arange(g.heads)[::-1].copy()),
        "bias window types shifted by one": dict(types=(pk.window_types(g) + 1) % g.n_type),
        "shift mask dropped": dict(mask=None),
        "shift mask dropped on the z axis": dict(mask=h_seam),
        "shift mask dropped on the latitude axis": dict(mask=z_seam),
        "padding keys zero instead of the QKV bias": dict(pad_zero=True),
        "roll in the wrong direction": dict(sign=+1),
    }


ATT_GRIDS = {f"{nlat}x{nlon}-g{i + 1}": g for nlat, nlon in [(41, 96), (33, 96), (45, 192)]
             for i, g in enumerate(pk.grids(pangu_small(nlat, nlon)))}


def _padding_visible(g, roll):
    """can any real query see a latitude-padding key?  Not when every padding row rolls into the half of the last
    h-window that the shift mask separates from the real rows (33 x 96 g1 at roll 1: pad 3 = the shift)"""
    idx = pk.window_tokens(g, roll, 1)[0]                                   # [nWin, 144]
    sep = pk.shift_mask_types(g)[pk.window_types(g)] if roll else np.zeros((g.nWin, pk.NTOK, pk.NTOK), bool)
    return bool(((idx >= 0)[:, :, None] & (idx < 0)[:, None, :] & ~sep).any())


@pytest.mark.parametrize("roll", [0, 1])
@pytest.mark.parametrize("name", list(ATT_GRIDS))
def test_bound_flags_every_mutation(name, roll):
    """at every grid and roll of the GPU attention cases, one member: each modelled mistake that can change an output
    there leaves the bound.  The mask and roll-direction mistakes exist only at roll 1; the padding-key one only where
    a real query can see a padding key (g2 of 41 x 96 has a single h-window row; 45 x 192 has no padding)."""
    g, B = ATT_GRIDS[name], 1
    inp = pk.attention_inputs(g, B, DISCRIM_SEED)
    ref, bnd = pk.attention_tokens(g, B, roll, inp)
    assert np.isfinite(ref).all() and np.isfinite(bnd).all()
    # the fp16 rounding of the exact reference is within the bound
    assert not gr.exceed(ref.astype(np.float16), ref, bnd).any()
    visible = g.Hp > g.H and _padding_visible(g, roll)
    rolled_only = {"shift mask dropped", "shift mask dropped on the z axis", "shift mask dropped on the latitude axis",
                   "roll in the wrong direction"}
    muts = {}
    for m, kw in _mutations(g).items():
        if m in rolled_only and not roll:
            continue
        got = pk.attention_tokens(g, B, roll, inp, **kw)[0]
        if kw.get("pad_zero") and not visible:
            # masked keys keep a weight of about 2^-144: far below the bound, as nothing a kernel does with them can show
            assert np.nanmax(np.abs(got - ref) / bnd) < 1e-6, "padding keys no real query sees changed an output"
            continue
        muts[m] = got
    swap = np.arange(g.C).reshape(g.pairs, 2, 32)[:, ::-1].reshape(-1)
    muts["two heads of a pair swapped"] = ref[:, swap]
    assert len(muts) == 6 + 4 * roll - (not visible)
    for m, got in muts.items():
        r = float(np.nanmax(np.abs(got - ref) / bnd))
        print(f"[pangu discrimination] {name} roll {roll} {m}: max |mutated - ref| / bound = {r:.1f}")
        # a kernel making this mistake lands within its own bound (about the same) of the mutated reference: > 2 bounds
        # away from the correct one at some element
        assert r > 3, f"{name} roll {roll} {m}: mutated reference within {r:.2f} bounds of the correct one"


def test_padding_keys_visible_at_roll_0():
    for name, g in ATT_GRIDS.items():
        if g.Hp > g.H:
            assert _padding_visible(g, 0), name
    assert not _padding_visible(ATT_GRIDS["33x96-g1"], 1)


def test_synthetic_scale_inputs_are_nearly_uniform():
    """the model-level weights' scale hides the bias: the same mutation moves the output by far less there"""
    g = G41[0]
    inp = pk.attention_inputs(g, 1, DISCRIM_SEED, synthetic=True)
    ref, bnd = pk.attention_tokens(g, 1, 1, inp)
    mut, _ = pk.attention_tokens(g, 1, 1, inp, head_perm=np.arange(g.heads)[::-1].copy())
    peaked = pk.attention_inputs(g, 1, DISCRIM_SEED)
    ref2, bnd2 = pk.attention_tokens(g, 1, 1, peaked)
    mut2, _ = pk.attention_tokens(g, 1, 1, peaked, head_perm=np.arange(g.heads)[::-1].copy())
    assert np.nanmax(np.abs(mut - ref) / bnd) * 10 < np.nanmax(np.abs(mut2 - ref2) / bnd2)


# ---------------------------------------------------------------------------------------------------------------------
# bias table repacking and the QKV reference
# ---------------------------------------------------------------------------------------------------------------------
def test_pack_bias_table_emulation():
    rng = np.random.default_rng(3)
    src = (rng.standard_normal((pk.TABLE, 4, 6)) * 3).astype(np.float32)
    out = pk.pack_bias_table(src)
    assert out.shape == (4, 6, pk.TABLE) and out.dtype == np.float16
    for l, t, h in [(0, 0, 0), (3311, 3, 5), (1000, 2, 1), (17, 1, 4)]:
        want = np.float16(np.float32(src[l, t, h]) * np.float32(1.4426950408889634))
        assert out[t, h, l].view(np.uint16) == want.view(np.uint16)
    # the fp32 product, not the exact one, is rounded: the two differ for some entry
    exact = (src.astype(np.float64) * pk.LOG2E).astype(np.float16).transpose(1, 2, 0)
    assert not np.array_equal(exact.view(np.uint16), out.view(np.uint16))


def test_qkv_ref_bound_holds_for_rounded_exact_values():
    rng = np.random.default_rng(4)
    x = rng.uniform(-1, 1, (300, 192)).astype(np.float16)
    w = (rng.uniform(-1, 1, (576, 192)) * 5 / np.sqrt(192)).astype(np.float16)
    b = rng.uniform(-1, 1, 576).astype(np.float32)
    ref, bnd = pk.qkv_ref(x, w, b)
    exact = x.astype(np.float64) @ w.astype(np.float64).T + b
    assert not gr.exceed(exact.astype(np.float16), ref, bnd).any()
    bad = exact.copy(); bad[5, 100] += 4 * gr.ulp16(exact[5, 100])
    assert gr.exceed(bad.astype(np.float16), ref, bnd)[5, 100]


# ---------------------------------------------------------------------------------------------------------------------
# probe library: ABI mirrors and host-side refusals (no device needed: validation precedes any CUDA call)
# ---------------------------------------------------------------------------------------------------------------------
def _probe():
    if not gp.PROBE_LIB_PATH.exists():
        pytest.fail(f"{gp.PROBE_LIB_PATH} is missing: __graft_entry__.build() builds it")
    return gp.lib()


def test_pangu_case_struct_matches_library():
    assert _probe().sky_probe_pangu_size() == C.sizeof(gp.PanguCase)


def _good_pangu_case(op, g=G41[0], B=1, **over):
    tiles = B * g.nWin * g.pairs
    kw = dict(op=op, geo=g.probe_geo(), roll=1, B=B, pairs=g.pairs, n_type=g.n_type, att_nkb=g.C // 64,
              part_stride=tiles * pk.TILE_B, qkv=0x10000, qkv_bytes=3 * tiles * pk.TILE_B, src=0x20000,
              src_floats=pk.TABLE * g.n_type * g.heads, tab=0x30000, tab_bytes=2 * pk.TABLE * g.n_type * g.heads,
              out=0x40000, out_bytes=-(-B * g.T // 128) * (g.C // 64) * 16384, sl2=0.25, mask_l2=-144.0)
    kw.update(over)
    geo = dict(kw.pop("geo")); geo.update(kw.pop("geo_over", {}))
    return gp.make_pangu_case(geo=geo, **kw)


@pytest.mark.parametrize("op,over,msg", [
    (gp.PG_ATTENTION, dict(geo_over=dict(Hp=11)), "Hp is not H rounded up"),
    (gp.PG_ATTENTION, dict(geo_over=dict(Z=7)), "Z is not"),
    (gp.PG_ATTENTION, dict(geo_over=dict(W=30)), "multiple of the window"),
    (gp.PG_ATTENTION, dict(geo_over=dict(T=100)), "T != Z H W"),
    (gp.PG_ATTENTION, dict(geo_over=dict(nWin=15)), "nWin"),
    (gp.PG_ATTENTION, dict(geo_over=dict(nWh=3)), "window counts"),
    (gp.PG_ATTENTION, dict(pairs=2), "heads != 2 pairs"),
    (gp.PG_ATTENTION, dict(geo_over=dict(C=160)), "C != 32 heads"),
    (gp.PG_ATTENTION, dict(qkv_bytes=3 * 48 * pk.TILE_B - 16), "window image too small"),
    (gp.PG_ATTENTION, dict(part_stride=47 * pk.TILE_B), "part stride"),
    (gp.PG_ATTENTION, dict(n_type=9), "bias window types"),
    (gp.PG_ATTENTION, dict(tab_bytes=2 * pk.TABLE * 8 * 6 - 2), "bias tables too small"),
    (gp.PG_ATTENTION, dict(att_nkb=2), "k-blocks"),
    (gp.PG_ATTENTION, dict(out_bytes=17 * 3 * 16384 - 16), "output image too small"),
    (gp.PG_ATTENTION, dict(roll=2), "roll"),
    (gp.PG_FILL_PAD, dict(src_floats=3 * 192 - 1), "QKV bias"),
    (gp.PG_FILL_PAD, dict(geo=G41[1].probe_geo(), pairs=6, n_type=4, att_nkb=6), "no latitude padding"),
    (gp.PG_PACK_BIAS, dict(out_bytes=2 * pk.TABLE * 8 * 6 - 2), "fp16 tables too small"),
    (gp.PG_PACK_BIAS, dict(src_floats=pk.TABLE * 8 * 6 - 1), "fp32 table"),
    (7, dict(), "unknown op"),
])
def test_pangu_probe_refuses_inconsistent_cases(op, over, msg):
    _probe()
    rc, err = gp.launch_pangu(_good_pangu_case(op, **over))
    assert rc != 0 and msg in err, (rc, err)


def _good_qkv_case(g=G41[0], B=1, **over):
    tiles = B * g.nWin * g.pairs
    M = B * g.T
    kw = dict(kernel=gp.W, epi=gp.EPI_QKV_WIN, block_n=192, n=3 * g.C, n_valid=3 * g.C, batches=1, grid_sms=0, nseg=1, m=M,
              a=[0x10000], a_bytes=[-(-M // 128) * 3 * 16384], a_batch_stride=[0], a_nkb=[3], w=0x20000,
              w_bytes=1 << 22, num_kb=3, hi=0x30000, img_bytes=3 * tiles * pk.TILE_B, bias=0x40000,
              vec_floats=3 * g.C, geo=g.probe_geo(), roll=0, pairs=g.pairs, part_stride=tiles * pk.TILE_B)
    kw.update(over)
    return gp.make_case(**kw)


@pytest.mark.parametrize("over,msg", [
    (dict(block_n=256, n=768, n_valid=768), "3C"),
    (dict(block_n=96, n=576, n_valid=576), "not instantiated"),
    (dict(m=2112 + 1), "members x T"),
    (dict(img_bytes=3 * 48 * pk.TILE_B - 16), "QKV window image too small"),
    (dict(part_stride=47 * pk.TILE_B), "part stride"),
    (dict(pairs=2), "heads != 2 pairs"),
    (dict(vec_floats=575), "bias"),
    (dict(roll=-1), "roll"),
])
def test_probe_refuses_inconsistent_qkv_cases(over, msg):
    _probe()
    rc, err = gp.launch(_good_qkv_case(**over))
    assert rc != 0 and msg in err, (rc, err)
