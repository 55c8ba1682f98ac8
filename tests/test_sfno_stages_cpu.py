"""The SFNO stage checker (oracle/sfno_stages_ref.py) on its own, without a GPU.

A stand-in for the engine is built from the fp64 oracle's taps (SFNORef.step(taps=...)), written in the engine's tap
formats (fp16 hi / lo tile images, fp32 and fp64 buffers).  Stage-local references fed those taps must find every stage
inside its bound; each modelled engine mistake planted into them must leave it."""
import numpy as np
import pytest
import torch

from oracle import gemm_ref as gr
from oracle import sfno_stages_ref as st
from oracle.sfno_ref import SFNORef
from skyrim_b200.config import FCNV2_CHANNELS, sfno_small
from skyrim_b200.weights import make_sfno_weights, sfno_tables, synthetic_state

SHAPES = [(49, 96, 64, 3), (49, 96, 192, 1), (49, 96, 384, 2), (385, 768, 64, 3), (433, 864, 64, 2)]


def _img(vals, alloc_bytes, batch_bytes=0):
    """fp64 values [rows, cols] or [batches, rows, cols] -> the engine's tap (hi image bytes, lo image bytes) as float32"""
    vals = np.asarray(vals)
    nkb = -(-vals.shape[-1] // 64)
    out = []
    for part in gr.split16(vals):
        if batch_bytes:
            b = np.concatenate([gr.pack_tiles(part[i], 128, nkb) for i in range(vals.shape[0])])
        else:
            b = gr.pack_tiles(part, 128, nkb)
        buf = np.zeros(alloc_bytes, np.uint8); buf[:b.size] = b
        out.append(buf)
    return np.concatenate(out).view(np.float32)


def _f32(v, n=None):
    v = np.asarray(v, np.float32).reshape(-1)
    if n is None:
        return v
    out = np.zeros(n, np.float32); out[:v.size] = v
    return out


def _fake_engine(shape):
    """taps of an engine that computes the oracle's fp64 values and rounds them like the engine stores them"""
    nlat, nlon, E, L = shape
    cfg = sfno_small(nlat, nlon, embed=E, layers=L)
    w = make_sfno_weights(cfg, 0)
    tabs = sfno_tables(cfg)
    x0 = synthetic_state(FCNV2_CHANNELS, cfg.nlat, cfg.nlon, 0)
    ref = {}
    y = SFNORef(cfg, w, torch.float64).step(x0, taps=ref)
    ref = {k: v.numpy() for k, v in ref.items()}
    sh = st.Shapes(cfg)
    nb = lambda n: sh.tap_floats(n) * 2      # bytes of one of the two images of tap n
    n2, mm, lm = 2 * E, sh.mmax, sh.lmax
    t0 = {"in_img": _img(ref["in"], nb("in_img")), "hidden_img": _img(ref["enc.hidden"], nb("hidden_img")),
          "x_img": _img(ref["enc.x"], nb("x_img")), "sums0": ref["enc.sums0"].astype(np.float64).view(np.float32)}
    if L == 1:
        t0["x"] = _f32(ref["enc.x"], sh.P1 * E)
    taps = [t0]
    for i in range(L):
        k = f"b{i}."
        Hi, Wi, Ho, Wo = sh.grids(i)
        t = {"norm0": _f32(ref[k + "norm0"]), "li": _img(ref[k + "li"], nb("li"), st.img_bytes(Hi, n2)),
             "si": _img(ref[k + "si"], nb("si"), st.img_bytes(mm, n2)), "mi": _img(ref[k + "mi"], nb("mi"), st.img_bytes(lm, n2)),
             "di": _img(ref[k + "di"], nb("di"), st.img_bytes(2 * mm, E)), "g_img": _img(ref[k + "g"], nb("g_img")),
             "sums": ref[k + "sums"].view(np.float32), "norm1": _f32(ref[k + "norm1"]), "fc1_bias": _f32(ref[k + "fc1_bias"]),
             "hidden_img": _img(ref[k + "hidden"], nb("hidden_img")), "x_img": _img(ref[k + "x"], nb("x_img"))}
        if Hi == Ho:
            t.update(f1=_f32(ref[k + "f1"], sh.P1 * E), inner_bias=_f32(ref[k + "inner_bias"]))
        else:
            t.update(mi2=_img(ref[k + "mi2"], nb("mi2"), st.img_bytes(lm, n2)), rpm=_f32(ref[k + "rpm"], sh.P1 * E))
        if i + 1 < L:
            t.update(x=_f32(ref[k + "x"], sh.P1 * E), sums0=ref[k + "sums0"].view(np.float32))
        taps.append(t)
    taps.append({"in_img": t0["in_img"], "x_img": taps[-1]["x_img"], "g_img": _img(ref["dec.hidden"], nb("g_img")),
                 "state": y.numpy().astype(np.float32)})
    return cfg, sh, w, tabs, x0, ref, taps


def _checks(sh, w, tabs, x0, taps, blocks=None):
    """every stage after the input pack (the stand-in's input image is the oracle's fp64 normalisation, not the engine's
    fused fp32 one: test_input_pack_checker covers that stage)"""
    checks = st.stage_encoder(sh, w, taps[0]["in_img"], taps[0]["hidden_img"], taps[0]["x_img"], taps[0]["sums0"], taps[0].get("x"))
    for i in range(sh.L) if blocks is None else blocks:
        t = dict(taps[1 + i]); t["_tables"] = tabs
        checks += [(f"b{i} {n}", *r) for n, *r in st.stage_block_spectral(sh, w, i, t, taps[i])]
        checks += [(f"b{i} {n}", *r) for n, *r in st.stage_block_tail(sh, w, i, t, taps[i])]
    if blocks is None:
        checks += st.stage_decoder(sh, w, taps[-1]["x_img"], taps[-1]["in_img"], taps[-1]["g_img"], taps[-1]["state"])
    return checks


_CACHE = {}


def _fake(shape):
    if shape not in _CACHE:
        _CACHE.clear()
        _CACHE[shape] = _fake_engine(shape)
    return _CACHE[shape]


@pytest.mark.parametrize("shape", SHAPES)
def test_stage_references_compose_to_the_oracle(shape):
    """every stage reference, fed the oracle's previous tap as the engine stores it, reproduces the oracle's next tap:
    the references do the oracle's arithmetic in the engine's layouts, folds and remaps.  Each stage is inside its bound,
    or, where the storage of the fed tap shows (hi + lo: 2^-22 relative, fp16 subnormal steps of small entries), within
    a per-channel relative L2 error of 1e-5"""
    cfg, sh, w, tabs, x0, ref, taps = _fake(shape)
    bad = []
    for name, got, r, bound in _checks(sh, w, tabs, x0, taps):
        got = np.asarray(got, np.float64)
        if name.endswith(" hi") or not gr.exceed(got, r, bound).any():
            continue   # hi alone is an fp16 rounding; inside the stage bound is agreement
        r = np.broadcast_to(np.asarray(r, np.float64), got.shape)
        g2, r2 = got.reshape(-1, got.shape[-1]), r.reshape(-1, got.shape[-1])
        num, den = np.sqrt(((g2 - r2) ** 2).sum(0)), np.sqrt((r2 ** 2).sum(0))
        keep = den > 1e-6 * den.max()
        e = float((num[keep] / den[keep]).max())
        if not e <= 1e-5:
            bad.append((name, e))
    assert not bad, bad


def _leaves(checks, stage):
    res = [r for r in st.evaluate(checks) if r[0].startswith(stage) or f" {stage}" in r[0]]
    assert res, stage
    return any(n for _, n, _ in res)


def test_stand_in_is_inside_the_stages_the_mistakes_are_planted_in():
    """the unmutated stand-in is inside every bound of the stages below (so that leaving one means the mistake)"""
    cfg, sh, w, tabs, x0, ref, taps = _fake((49, 96, 64, 3))
    checks = _checks(sh, w, tabs, x0, taps, blocks=[1])
    for stage in ("forward DFT", "forward Legendre", "mixing", "enc fc2+pos", "enc sums0"):
        assert not _leaves(checks, stage), stage


def _mutate_img(raw, rows, cols, fn, batches=1, batch_bytes=0):
    hi, lo = st.decode(raw, rows, cols, -(-cols // 64), batches, batch_bytes)
    v = fn(hi + lo)
    return _img(v, raw.size * 4 // 2, batch_bytes)


def test_checker_catches_modelled_mistakes():
    """each mistake planted into the stand-in's taps leaves the bound of the stage it belongs to"""
    cfg, sh, w, tabs, x0, ref, taps = _fake((49, 96, 64, 3))
    E, mm, lm = sh.E, sh.mmax, sh.lmax
    Hi, Wi, _, _ = sh.grids(1)

    def run(mutated_block1=None, mutated_enc=None):
        t = [dict(x) for x in taps]
        t[0].update(mutated_enc or {})
        t[2].update(mutated_block1 or {})
        return _checks(sh, w, tabs, x0, t, blocks=[1])

    li = taps[2]["li"]; bb = st.img_bytes(Hi, 2 * E)
    # the roll of re / im within (ri, c)
    bad = _mutate_img(li, Hi, 2 * E, lambda v: np.roll(v, E, axis=-1), mm, bb)
    assert _leaves(run({"li": bad}), "forward DFT")
    # the t1 shift fold dropped: the m = 0 real row lacks shift * t1[0]
    t1 = tabs["dft.fwd_int"].astype(np.float64).sum(1)[0]
    n0 = taps[2]["norm0"].astype(np.float64)

    def drop(v):
        v = v.copy(); v[0, :, :E] -= n0[E:] * t1
        return v
    assert _leaves(run({"li": _mutate_img(li, Hi, 2 * E, drop, mm, bb)}), "forward DFT")
    # m and l swapped in the Legendre remap
    si = ref["b1.si"]
    sw = si.copy(); n = min(lm, mm); sw[:n, :n] = si[:n, :n].transpose(1, 0, 2)
    assert _leaves(run({"si": _img(sw, taps[2]["si"].size * 2, st.img_bytes(mm, 2 * E))}), "forward Legendre")
    # the sign of Wi flipped in the mixing
    wc = w["blk1.spec.w"].astype(np.float64)
    X = si[..., :E] + 1j * si[..., E:]                                              # [l, m, i]
    Xo = np.einsum("loi,lmi->mlo", wc[..., 0] - 1j * wc[..., 1], X)
    assert _leaves(run({"mi": _img(np.concatenate([Xo.real, Xo.imag], -1), taps[2]["mi"].size * 4 // 2, st.img_bytes(lm, 2 * E))}), "mixing")
    # one split term dropped (the encoder's fc2 without lo(hidden) x hi(W))
    h_hi, h_lo = st.decode(taps[0]["hidden_img"], sh.P1, E, E // 64)
    w_hi, _ = st.wsplit(w["enc.fc2.w"])
    x_bad = ref["enc.x"] - h_lo @ w_hi.T
    assert _leaves(run(mutated_enc={"x_img": _img(x_bad, taps[0]["x_img"].size * 4 // 2)}), "enc fc2+pos")
    # statistics summed over P - 1 pixels
    d = ref["enc.x"][:-1] - w["enc.fc2.b"].astype(np.float64)
    s_bad = np.concatenate([d.sum(0), (d * d).sum(0)])
    assert _leaves(run(mutated_enc={"sums0": s_bad.view(np.float32)}), "enc sums0")


def test_checker_catches_a_lost_m_tile():
    """433x864 (lmax 144, mmax 145): the mixing's last m-tile (m >= 128) lost for the degrees l >= 128"""
    cfg, sh, w, tabs, x0, ref, taps = _fake((433, 864, 64, 2))
    E, mm, lm = sh.E, sh.mmax, sh.lmax
    mi = ref["b0.mi"].copy()                                                        # [m, l, (ro, o)]
    mi[128:, 128:] = 0.0
    t = dict(taps[1]); t["_tables"] = tabs
    t["mi"] = _img(mi, taps[1]["mi"].size * 4 // 2, st.img_bytes(lm, 2 * E))
    res = st.evaluate(st.stage_mixing(sh, w["blk0.spec.w"], w["blk0.inner.w"], t["si"], t["mi"]))
    assert any(n for _, n, _ in res), res
    t["mi"] = taps[1]["mi"]
    res = st.evaluate(st.stage_mixing(sh, w["blk0.spec.w"], w["blk0.inner.w"], t["si"], t["mi"]))
    assert not any(n for _, n, _ in res), res


def test_input_pack_checker():
    """the input stage accepts the engine's fused fp32 normalisation split into hi / lo with zero padding columns, and
    rejects an unfused one (x * (1/sigma) rounded before the shift), a 1/sigma rounded twice and a non-zero pad column"""
    cfg = sfno_small(49, 96, embed=64, layers=1)
    w = make_sfno_weights(cfg, 0)
    sh = st.Shapes(cfg)
    x0 = synthetic_state(FCNV2_CHANNELS, cfg.nlat, cfg.nlon, 0)
    std, mu = w["norm.std"].astype(np.float32), w["norm.mean"].astype(np.float32)
    sc, shf = (np.float32(1) / std).astype(np.float32), (-mu / std).astype(np.float32)
    x = x0.reshape(sh.Cin, -1).T
    fused = (x.astype(np.float64) * sc + shf).astype(np.float32)
    unfused = ((x * sc).astype(np.float32) + shf).astype(np.float32)
    pad = lambda v: np.concatenate([v, np.zeros((v.shape[0], 128 - sh.Cin))], 1)
    nbytes = sh.tap_floats("in_img") * 2
    checks, bad = st.stage_input(sh, x0, w, _img(pad(fused), nbytes))
    assert bad == 0 and not any(n for _, n, _ in st.evaluate(checks))
    _, bad = st.stage_input(sh, x0, w, _img(pad(unfused), nbytes))
    assert bad > 0
    v = pad(fused); v[7, 100] = 1.0
    checks, _ = st.stage_input(sh, x0, w, _img(v, nbytes))
    assert any(n for _, n, _ in st.evaluate(checks))
