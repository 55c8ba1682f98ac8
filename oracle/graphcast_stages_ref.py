"""ORACLE — test infrastructure, not product code.

Stage-local float64 references of the GraphCast engine (skyrim_b200/csrc/graphcast_engine.cu), for
tests/test_graphcast_stages_gpu.py (engine taps read with debug_copy after ``debug_set("stop_launch", n)``) and
tests/test_graphcast_stages_cpu.py (this module on its own).

The engine's step is written down ONCE, in program order, in ``run_program``: one call per unit (the feature kernel, every
hidden GEMM, LayerNorm GEMM, per-node table, aggregation, the output head).  A back end executes it:

  Recorder   lists the units (kind, name, outputs, rows): what a test has to read after which stop point;
  Checker    takes the ENGINE's decoded taps: every unit is recomputed in float64 from the engine's own inputs to it (the
             taps of the units before), compared per element, and the engine's output is handed on.  Errors do not
             accumulate, and a wrong unit is named by the first check that fails.  Given the checked rows of every unit,
             it takes taps as Rows (row indices, values) and computes each reference for those rows only;
  Planner    takes the rows checked in every unit and derives from the graph's index arrays which rows of which earlier
             tap each check reads: the read plan of a sampled check (full_size_rows: the rules at 721 x 1440);
  Emulator   computes the taps itself in the engine's formulation (fp16 where the engine rounds, split first layers,
             per-node tables, chunked fp32 segment sums in the engine's order), optionally with one modelled mistake.

Gathers use the GRAPH's index arrays and the raw fp32 weights, never anything the engine derived from them.  Sums and
bounds come from oracle/gemm_ref.py: |D - R| <= TAU sum |a w| + epilogue roundings, half an fp16 ulp per fp16 store.
"""
from __future__ import annotations

import math
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from oracle import gemm_ref as gr

L = 512
NKB = L // 64
FEAT_KP = 192          # GC_FEAT_KP: the feature image's three k-blocks
SEG_CHUNK = 64         # GC_SEG_CHUNK
TILE = 16384           # bytes of one 128-row x 64-column fp16 tile
TOA_REL = 2e-5         # the fp32 toa radiation against the closed form, relative to the field's maximum (test_toa_radiation_matches_oracle)
DAY_TRIG_ABS = 4e-6    # sincosf(2 pi frac(day fraction + lon / 360)) with fp32 fractions: 2 pi x 3 x 2^-24 = 1.1e-6, then sincosf
GEO_TRIG_ABS = 2e-6    # cos lat / sin lon / cos lon from fp32 angles


def pad128(n):
    return -(-n // 128) * 128


def q16(a):
    """fp32 -> fp16 -> float64: the value a tensor-core operand carries"""
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float64)


class Shapes:
    """the engine's buffer geometry for one config and graph"""

    def __init__(self, cfg, graph):
        self.cfg = cfg
        self.Ng, self.Nm = cfg.n_grid, int(graph["n_mesh"])
        self.Ngp, self.Nmp = pad128(self.Ng), pad128(self.Nm)
        self.Em, self.Eg = len(graph["mesh.senders"]), len(graph["g2m.senders"])
        self.E3 = 3 * self.Ngp
        self.Emax = max(self.E3, pad128(self.Eg))
        self.nfeat = cfg.n_features
        # rows of the k-major, tile-padded mesh2grid edge images that hold the graph's 3 n_grid edges
        self.m2g_rows = (np.arange(3)[:, None] * self.Ngp + np.arange(self.Ng)[None, :]).reshape(-1)

    def tap_floats(self, name):
        img = lambda rows, nkb=NKB: pad128(rows) // 128 * nkb * TILE // 4
        return {"feat": img(self.Ng, FEAT_KP // 64), "hid": img(self.Emax), "hid_m": img(self.Em), "vg_img": img(self.Ng),
                "tg": self.Ngp * L // 2, "yimg": img(self.Emax), "vm_img": img(self.Nm), "tm": self.Nmp * L, "em_img": img(self.Em),
                "ym_img": img(self.Em), "agg_img": img(self.Nm), "vm0_img": img(self.Nm), "e_g2m_img": img(self.Eg),
                "e_m2g_img": img(self.E3), "e_mesh_img": img(self.Em), "g2m_tr": self.Nmp * L // 2, "vm": self.Nm * L,
                "vm0": self.Nm * L}[name]

    def decode(self, name, raw, rows=None, cols=None):
        """raw tap (float32 container) -> float64 [rows, columns]; ``rows``: a count or an index array; ``cols``: the row
        length of a table (the mesh table is [W1s | W1r], 1024 wide, in the processor and 512 wide in the decoder)"""
        raw = np.ascontiguousarray(raw).reshape(-1)
        if name in ("vm", "vm0"):
            x = raw.astype(np.float64).reshape(-1, L)
        elif name in ("tg", "g2m_tr"):
            x = raw.view(np.float16).astype(np.float64).reshape(-1, L)
        elif name == "tm":
            x = raw.view(np.float16).astype(np.float64).reshape(-1, cols or 2 * L)
        else:
            nkb = FEAT_KP // 64 if name == "feat" else NKB
            b = raw.view(np.uint8)
            x = gr.unpack_tiles(b, 128, nkb, b.size // (nkb * 128)).astype(np.float64)
        if rows is None:
            return x
        return x[:rows] if np.isscalar(rows) else x[rows]

    def gather(self, name, raw, rows, kmajor=False, cols=None):
        """rows of a raw tap (the float32 torch container debug_tensor returns, on any device) -> Rows of float64 values.
        Only the rows' bytes leave the device: row r of a tile image is eight 128-byte pieces, piece kb at byte
        ((r >> 7) nkb + kb) TILE + (r & 127) 128; a table row is a row-major slice.  ``rows``: logical (k-major images:
        k n_grid + g)"""
        import torch
        rows = np.asarray(rows, np.int64)
        phys = self.m2g_rows[rows] if kmajor else rows
        if name in ("vm", "vm0"):
            v = raw.view(-1, L)[torch.from_numpy(phys).to(raw.device)].cpu().numpy()
        elif name in ("tg", "g2m_tr", "tm"):
            v = raw.view(torch.float16).view(-1, cols or L)[torch.from_numpy(phys).to(raw.device)].cpu().numpy()
        else:
            nkb = FEAT_KP // 64 if name == "feat" else NKB
            piece = ((phys >> 7)[:, None] * nkb + np.arange(nkb)[None]) * (TILE // 128) + (phys & 127)[:, None]
            b = raw.view(torch.uint8).view(-1, 128)[torch.from_numpy(piece).to(raw.device)].cpu().numpy()
            v = gr.unpack_rows(b, phys)
        return Rows(rows, v.astype(np.float64))


class Rows:
    """rows ``idx`` (sorted, unique) of a tap and their values ``val``, indexed by row number like the whole tap:
    ``t[rows]`` -> the values of those rows (each must be present), ``t[a:b]`` -> the rows in [a, b) numbered from a,
    ``t[:, cols]`` -> the same rows, those columns"""

    def __init__(self, idx, val):
        self.idx, self.val = np.asarray(idx, np.int64), val

    def __getitem__(self, key):
        if isinstance(key, tuple):
            rows, cols = key
            assert rows == slice(None)
            return Rows(self.idx, self.val[:, cols])
        if isinstance(key, slice):
            lo, hi = np.searchsorted(self.idx, [key.start, key.stop])
            return Rows(self.idx[lo:hi] - key.start, self.val[lo:hi])
        key = np.asarray(key, np.int64)
        pos = np.searchsorted(self.idx, key)
        assert (pos < len(self.idx)).all() and (self.idx[pos] == key).all(), "a row that was not read"
        return self.val[pos]


STATIC_TAPS = ("vm0", "vm0_img", "e_g2m_img", "e_m2g_img", "e_mesh_img", "g2m_tr")


# ---------------------------------------------------------------------------------------------------------------------
# the aggregation's chunk plan (load_segplan restated)
# ---------------------------------------------------------------------------------------------------------------------
def chunk_plan(ptr):
    """receiver-sorted CSR pointer -> (chunks [(node, e0, e1, part)], multi [(node, p0, p1)]): a segment of more than
    SEG_CHUNK edges is cut into ceil(deg / SEG_CHUNK) chunks that leave fp32 partial rows; any other node (degree 0
    included) is one chunk that finishes its row"""
    chunks, multi, parts = [], [], 0
    for n in range(len(ptr) - 1):
        e0, e1 = int(ptr[n]), int(ptr[n + 1])
        nc = 1 if e1 - e0 <= SEG_CHUNK else -(-(e1 - e0) // SEG_CHUNK)
        if nc == 1:
            chunks.append((n, e0, e1, -1))
            continue
        multi.append((n, parts, parts + nc))
        for c in range(nc):
            a = e0 + c * SEG_CHUNK
            chunks.append((n, a, min(a + SEG_CHUNK, e1), parts))
            parts += 1
    return chunks, multi


def segsum_f32(y, ptr, prev=None, mut=None):
    """k_gc_segsum + k_gc_segsum_fin in fp32 and in their order: per chunk four edges at a time then the e % 4 tail, the
    partial rows of a cut segment added in chunk order.  ``prev``: what the output held before (mutations only)."""
    y = np.asarray(y, np.float32)
    chunks, multi = chunk_plan(ptr)
    out = np.zeros((len(ptr) - 1, y.shape[1]), np.float32) if prev is None else np.asarray(prev, np.float32).copy()
    partial = {}
    for n, e0, e1, part in chunks:
        acc = np.zeros(y.shape[1], np.float32)
        e = e0
        while e + 4 <= e1:
            for u in range(4):
                acc = acc + y[e + u]
            e += 4
        if mut != "skip_tail":
            for k in range(e, e1):
                acc = acc + y[k]
        if part < 0:
            if not (mut == "stale_zero_degree" and e0 == e1):
                out[n] = acc
        else:
            partial[part] = acc
    for n, p0, p1 in multi:
        acc = np.zeros(y.shape[1], np.float32)
        for p in range(p0, p1 - 1 if mut == "drop_last_chunk" else p1):
            acc = acc + partial[p]
        out[n] = acc
    return out


# ---------------------------------------------------------------------------------------------------------------------
# unit references: (reference, bound) per element, from the exact operands the engine reads
# ---------------------------------------------------------------------------------------------------------------------
def _wpad(w, k):
    w = q16(w)
    return w if w.shape[1] == k else np.concatenate([w, np.zeros((w.shape[0], k - w.shape[1]))], axis=1)


def ref_hidden(parts, b1, gathers=()):
    """silu(sum_s A_s W_s^T + b1 + sum T[idx]) -> fp16.  parts: [(A [M, K_s] operand values, W [512, <= K_s] raw fp32)],
    gathers: [(table [rows, 512] values, index [M])]"""
    R, S = gr.linear([(a, _wpad(w, a.shape[1])) for a, w in parts])
    x, xb = gr.epi_affine(R, S, np.asarray(b1, np.float64)[None], *[t[np.asarray(i)] for t, i in gathers])
    f, fb = gr.epi_silu(x, xb)
    return f, gr.f16_bound(f, fb)


def ref_ln(hid, w, name, res, eps, extra=None):
    """LayerNorm GEMM: y = LN(hid W2^T + b2) gamma + beta; returns (y, sum = y + res, bound) before any fp16 store.
    ``extra``: a bound on what the operand image may differ from ``hid`` by, per accumulator element"""
    R, S = gr.linear([(hid, q16(w[name + ".w2"]))])
    if extra is not None:
        S = S + extra / gr.TAU
    f64 = lambda k: np.asarray(w[f"{name}.{k}"], np.float64)
    # every GraphCast LayerNorm runs Epi2F32Img::run on the CTA pairs at 2 x 256 columns
    y, yb = gr.layer_norm(R, S, f64("b2")[None], f64("ln.g")[None], f64("ln.b")[None], 0.0, eps, depth=gr.ln_depth(256 // 8 + 2, 2),
                          shift=gr.ln_shift(256))
    if res is None:
        return y, y, yb
    return y, y + res, yb + 4 * gr.U32 * np.abs(res)


def ref_table(a, wslices):
    """per-node table: A x [slices of the raw first-layer weight]^T -> fp16 row-major, the slices side by side"""
    out = [gr.epi_affine(*gr.linear([(a, q16(ws))])) for ws in wslices]
    f = np.concatenate([o[0] for o in out], axis=1)
    fb = np.concatenate([o[1] for o in out], axis=1)
    return f, gr.f16_bound(f, fb)


def seg_edges(ptr, nodes):
    """the incoming edge rows of ``nodes`` over the CSR pointer, node after node"""
    ptr = np.asarray(ptr, np.int64)
    nodes = np.asarray(nodes, np.int64)
    deg = ptr[nodes + 1] - ptr[nodes]
    return np.repeat(ptr[nodes] - (np.cumsum(deg) - deg), deg) + np.arange(int(deg.sum()))


def ref_agg(y, ptr, nodes):
    """fp64 sums of the update rows of each node's incoming edges (``y``: indexed by edge row), for ``nodes`` only; fp32
    accumulation bound deg 2^-24 sum |y| plus the fp16 store.  A node without edges is exactly zero (bound 0)."""
    ptr = np.asarray(ptr, np.int64)
    nodes = np.asarray(nodes, np.int64)
    deg = ptr[nodes + 1] - ptr[nodes]
    v = np.asarray(y[seg_edges(ptr, nodes)], np.float64)
    f = np.zeros((len(nodes), v.shape[1]))
    fa = np.zeros_like(f)
    has = deg > 0
    if has.any():
        start = (np.cumsum(deg) - deg)[has]
        f[has] = np.add.reduceat(v, start, axis=0)
        fa[has] = np.add.reduceat(np.abs(v), start, axis=0)
    deg = deg[:, None]
    # the fp64 sums themselves carry deg 2^-53 sum |y|
    bound = gr.f16_bound(f, deg * (gr.U32 + 2.0 ** -53) * fa)
    return f, np.where(deg == 0, 0.0, bound)


def ref_out(hid, w, x1, n_prog):
    """output head: x(t) + diff_std (hid W2^T + b2) for the prognostic channels -> [n_grid, n_prog]"""
    R, S = gr.linear([(hid, q16(w["dec.out.w2"])[:n_prog])])
    y = R + np.asarray(w["dec.out.b2"], np.float64)[None, :n_prog]
    d = np.asarray(w["norm.diff_std"], np.float64)[None, :n_prog]
    ref = x1 + d * y
    return ref, d * (gr.TAU * S + 2 * gr.U32 * np.abs(y)) + 2 * gr.U32 * (np.abs(ref) + np.abs(x1))


def ref_features(cfg, w, graph, x, t_seconds):
    """(reference [n_grid, 192], bound): the fp64 formulas of GraphCastRef.features per column, one fp16 rounding on top of
    the fp32 normalisation ((v - mean) / std: two roundings) or of the fp32 trigonometry (absolute slacks above); columns
    past n_features exactly zero"""
    import torch
    from oracle.graphcast_ref import GraphCastRef, toa_radiation
    r = GraphCastRef(cfg, w, graph, dtype=torch.float64)
    f = r.features(torch.from_numpy(np.asarray(x, np.float32)), t_seconds).numpy()
    npg, ns = cfg.n_prog, cfg.n_state
    b = 4 * gr.U32 * np.abs(f)
    c = 2 * npg
    sd = float(np.asarray(w["norm.std"], np.float64)[ns - 1])
    toa_max = float(toa_radiation(t_seconds + 3600.0 * cfg.dt_hours, r.lat, r.lon).max())
    b[:, c + 2] += TOA_REL * toa_max / sd
    c += 3
    for k in range(3):
        b[:, c + 4 * k + 2:c + 4 * k + 4] += DAY_TRIG_ABS
    c += 12 + cfg.n_static
    b[:, c:c + 3] += GEO_TRIG_ABS
    assert c + 3 == cfg.n_features
    ref = np.zeros((f.shape[0], FEAT_KP))
    bound = np.zeros_like(ref)
    ref[:, :cfg.n_features] = f
    bound[:, :cfg.n_features] = gr.f16_bound(f, b)
    return ref, bound


def ref_static(feat, w, name, eps):
    """an input-independent embedding: the whole MLP from the fp16-rounded features and the raw weights.  The hidden image
    is not kept by the engine, so its rounding (half an fp16 ulp per element) is carried through the second GEMM."""
    f, fb = ref_hidden([(q16(feat), w[name + ".w1"])], w[name + ".b1"])
    y, _, yb = ref_ln(f, w, name, None, eps, extra=fb @ np.abs(q16(w[name + ".w2"])).T)
    return f, y, yb


# ---------------------------------------------------------------------------------------------------------------------
# the step in program order
# ---------------------------------------------------------------------------------------------------------------------
def run_program(cfg, graph, be):
    """the engine's member step, one back-end call per unit.  Array arguments are what the unit READS (for the Checker:
    the engine's own taps); index arrays are the graph's."""
    g = graph
    Ng = cfg.n_grid
    st = be.statics()
    feat = be.features()
    hid = be.hidden("enc.grid_embed", [(feat, (0, cfg.n_features))], "hid", Ng)
    vg = be.ln("enc.grid_embed", hid, None, dict(img="vg_img"), Ng)["img"]
    tg = be.table("enc.g2m_edge", vg, [L], "tg", Ng)
    hid = be.hidden("enc.g2m_edge", [(st["e_g2m_img"], (0, L))], "hid", len(g["g2m.senders"]),
                    gathers=[(tg, g["g2m.senders"]), (st["g2m_tr"], g["g2m.receivers"])])
    y = be.ln("enc.g2m_edge", hid, None, dict(yimg="yimg"), len(g["g2m.senders"]))["yimg"]
    agg = be.agg("g2m", y, g["g2m.ptr"])
    hid = be.hidden("enc.g2m_mesh", [(st["vm0_img"], (0, L)), (agg, (L, 2 * L))], "hid_m", g["n_mesh"])
    o = be.ln("enc.g2m_mesh", hid, st["vm0"], dict(xout="vm", img="vm_img"), g["n_mesh"])
    vm, vm_img = o["xout"], o["img"]
    hid = be.hidden("enc.g2m_grid", [(vg, (0, L))], "hid", Ng)
    vg = be.ln("enc.g2m_grid", hid, vg, dict(img="vg_img"), Ng)["img"]
    em = st["e_mesh_img"]
    Em = len(g["mesh.senders"])
    for i in range(cfg.layers):
        tm = be.table(f"proc{i}.edge", vm_img, [L, 2 * L], "tm", g["n_mesh"])
        hid = be.hidden(f"proc{i}.edge", [(em, (0, L))], "hid_m", Em,
                        gathers=[(None if tm is None else tm[:, :L], g["mesh.senders"]),
                                 (None if tm is None else tm[:, L:], g["mesh.receivers"])])
        # the edge latents are not read after the last layer: the engine writes the update image only
        outs = dict(yimg="ym_img") if i == cfg.layers - 1 else dict(img="em_img", yimg="ym_img")
        o = be.ln(f"proc{i}.edge", hid, em, outs, Em)
        em, y = o.get("img"), o["yimg"]
        agg = be.agg(f"mesh{i}", y, g["mesh.ptr"])
        hid = be.hidden(f"proc{i}.node", [(vm_img, (0, L)), (agg, (L, 2 * L))], "hid_m", g["n_mesh"])
        o = be.ln(f"proc{i}.node", hid, vm, dict(xout="vm", img="vm_img"), g["n_mesh"])
        vm, vm_img = o["xout"], o["img"]
    tm = be.table("dec.m2g_edge", vm_img, [L], "tm", g["n_mesh"])
    tg = be.table("dec.m2g_edge", vg, [2 * L], "tg", Ng)
    hid = be.hidden("dec.m2g_edge", [(st["e_m2g_img"], (0, L))], "hid", 3 * Ng, kmajor=True,
                    gathers=[(None if tm is None else tm[:, :L], g["m2g.senders"]), (tg, g["m2g.receivers"])])
    y = be.ln("dec.m2g_edge", hid, None, dict(yimg="yimg"), 3 * Ng, kmajor=True)["yimg"]
    yk = [None if y is None else y[k * Ng:(k + 1) * Ng] for k in range(3)]
    hid = be.hidden("dec.m2g_grid", [(vg, (0, L))] + [(yk[k], (L, 2 * L)) for k in range(3)], "hid", Ng)
    vg = be.ln("dec.m2g_grid", hid, vg, dict(img="vg_img"), Ng)["img"]
    hid = be.hidden("dec.out", [(vg, (0, L))], "hid", Ng)
    be.out(hid)


class Recorder:
    """lists the units: [(kind, name, {tap: (rows, kmajor, table columns)})], unit n (1-based) = the n-th entry"""

    def __init__(self):
        self.units = []

    def _add(self, kind, name, outs, rows, kmajor=False, cols=None):
        self.units.append((kind, name, {o: (rows, kmajor, cols) for o in outs}))

    def statics(self):
        return {k: None for k in STATIC_TAPS}

    def features(self):
        self._add("features", "features", ["feat"], None)

    def hidden(self, name, parts, out, rows, gathers=(), kmajor=False):
        self._add("hidden", name, [out], rows, kmajor)

    def ln(self, name, hid, res, outs, rows, kmajor=False):
        self._add("ln", name, list(outs.values()), rows, kmajor)
        return {k: None for k in outs}

    def table(self, name, a, c0s, out, rows):
        self._add("table", name, [out], rows, cols=L * len(c0s))

    def agg(self, name, y, ptr):
        self._add("agg", name, ["agg_img"], len(ptr) - 1)

    def out(self, hid):
        self._add("out", "dec.out", ["x_out"], None)


def units(cfg, graph):
    r = Recorder()
    run_program(cfg, graph, r)
    return r.units


class _Src:
    """what Planner hands on in place of a tap: the unit that wrote it, its name, and the first row of a slice"""

    def __init__(self, n, tap, off=0):
        self.n, self.tap, self.off = n, tap, off

    def __getitem__(self, key):
        if isinstance(key, slice):
            return _Src(self.n, self.tap, self.off + key.start)
        return self            # [:, columns]: a table's rows are read whole


def every_row(kind, name, rows, kmajor):
    return np.arange(rows)


class Planner:
    """``pick(kind, name, rows, kmajor) -> the rows checked`` in a unit (``name``: the static tap's for kind "static")
    -> ``checked`` {n: rows, 0: {static tap: rows}} (Checker's ``rows``) and the read plan ``reads`` {n: {tap: [rows,
    kmajor, table columns]}}: after stop n, read these rows of these taps (0: the load-time taps).  A unit reads the
    checked rows of its A operands and residual, the sender and receiver rows of the tables it gathers, and every
    incoming edge row of a checked aggregation node; rows are logical (k-major: k n_grid + g)."""

    def __init__(self, cfg, graph, pick):
        self.cfg, self.g, self.pick = cfg, graph, pick
        self.n = 0
        self.checked, self.reads = {0: {}}, {0: {}}

    def _read(self, src, rows):
        r = self.reads[src.n][src.tap]
        r[0] = np.union1d(r[0], src.off + np.asarray(rows, np.int64))

    def _unit(self, kind, name, outs, rows, kmajor=False, cols=None):
        self.n += 1
        R = np.unique(np.asarray(self.pick(kind, name, rows, kmajor), np.int64))
        self.checked[self.n] = R
        self.reads[self.n] = {o: [R, kmajor, cols] for o in outs}
        return R

    def statics(self):
        g, Nm = self.g, int(self.g["n_mesh"])
        for tap, rows in (("vm0_img", Nm), ("e_g2m_img", len(g["g2m.senders"])), ("e_mesh_img", len(g["mesh.senders"])),
                          ("e_m2g_img", 3 * self.cfg.n_grid), ("g2m_tr", Nm)):
            R = np.unique(np.asarray(self.pick("static", tap, rows, tap == "e_m2g_img"), np.int64))
            self.checked[0][tap] = R
            self.reads[0][tap] = [R, tap == "e_m2g_img", L if tap == "g2m_tr" else None]
        self.reads[0]["vm0"] = [self.checked[0]["vm0_img"], False, None]
        self._read(_Src(0, "vm0_img"), self.checked[0]["g2m_tr"])
        return {k: _Src(0, k) for k in STATIC_TAPS}

    def features(self):
        self._unit("features", "features", ["feat"], self.cfg.n_grid)
        return _Src(self.n, "feat")

    def hidden(self, name, parts, out, rows, gathers=(), kmajor=False):
        R = self._unit("hidden", name, [out], rows, kmajor)
        for a, _ in parts:
            self._read(a, R)
        for tb, i in gathers:
            self._read(tb, np.asarray(i)[R])
        return _Src(self.n, out)

    def ln(self, name, hid, res, outs, rows, kmajor=False):
        R = self._unit("ln", name, list(outs.values()), rows, kmajor)
        self._read(hid, R)
        if res is not None:
            self._read(res, R)
        return {k: _Src(self.n, tap) for k, tap in outs.items()}

    def table(self, name, a, c0s, out, rows):
        R = self._unit("table", name, [out], rows, cols=L * len(c0s))
        self._read(a, R)
        return _Src(self.n, out)

    def agg(self, name, y, ptr):
        R = self._unit("agg", name, ["agg_img"], len(ptr) - 1)
        self._read(y, seg_edges(ptr, R))
        return _Src(self.n, "agg_img")

    def out(self, hid):
        R = self._unit("out", "dec.out", ["x_out"], self.cfg.n_grid)
        self._read(hid, R)


def plan(cfg, graph, pick=every_row):
    p = Planner(cfg, graph, pick)
    run_program(cfg, graph, p)
    return p


def row_bytes(cfg, tap, cols=None):
    """bytes of one row of a tap as the engine stores it"""
    return {"feat": 2 * FEAT_KP, "vm": 4 * L, "vm0": 4 * L, "x_out": 8 * cfg.n_state}.get(tap, 2 * (cols or L))


def full_size_rows(cfg, graph, seed=0, n_grid=4096, n_g2m_nodes=512, n_edges=16384, edge_layers=None):
    """the rows the full-size check checks, as Planner's ``pick``:
    mesh nodes   every row of every mesh-node unit (tables, node hidden and LayerNorm GEMMs, vm / vm_img, every
                 aggregation but grid2mesh's), and vm0 / vm0_img / g2m_tr;
    mesh edges   every row in layers ``edge_layers`` (default the first two and the last two), elsewhere the first and
                 the last (partial) tile and ``n_edges`` seeded rows;
    grid nodes   the first and the last (partial) tile, the first and the last latitude row, the grid points whose
                 mesh2grid rows are the tiles on either side of byte 2^31 of the k-major edge images, ``n_grid`` seeded
                 points; the mesh2grid units the three k-major rows k n_grid + g of each;
    grid2mesh    the aggregation on every node whose segment is cut into chunks, every node without edges and
                 ``n_g2m_nodes`` seeded others; the edge units on all their edges and the first and the last tile"""
    rng = np.random.default_rng(seed)
    Ng, nlon = cfg.n_grid, cfg.nlon
    ends = lambda n: np.r_[0:min(128, n), n // 128 * 128 if n % 128 else n - 128:n]
    sh = Shapes(cfg, graph)
    r31 = 2 ** 31 // (NKB * TILE) * 128                     # the first image row at or past byte 2^31
    phys = np.arange(r31 - 128, r31 + 128)
    phys = phys[(phys < sh.E3) & (phys % sh.Ngp < Ng)]
    grid = np.unique(np.concatenate([ends(Ng), np.arange(nlon), np.arange(Ng - nlon, Ng), phys % sh.Ngp,
                                     rng.choice(Ng, min(n_grid, Ng), replace=False)]))
    m2g = (np.arange(3)[:, None] * Ng + grid[None]).reshape(-1)
    ptr = np.asarray(graph["g2m.ptr"], np.int64)
    deg = np.diff(ptr)
    special = np.flatnonzero((deg > SEG_CHUNK) | (deg == 0))
    others = np.setdiff1d(np.arange(len(deg)), special)
    g2m_nodes = np.union1d(special, rng.choice(others, min(n_g2m_nodes, len(others)), replace=False))
    g2m_edges = np.union1d(seg_edges(ptr, g2m_nodes), ends(len(graph["g2m.senders"])))
    Em, Nm = len(graph["mesh.senders"]), int(graph["n_mesh"])
    full = {0, 1, cfg.layers - 2, cfg.layers - 1} if edge_layers is None else set(edge_layers)
    edges = {i: np.arange(Em) if i in full else np.union1d(ends(Em), rng.choice(Em, min(n_edges, Em), replace=False))
             for i in range(cfg.layers)}

    def pick(kind, name, rows, kmajor):
        if kind == "static":
            return {"e_g2m_img": g2m_edges, "e_m2g_img": m2g, "e_mesh_img": edges[0]}.get(name, np.arange(Nm))
        if kmajor:
            return m2g
        if name == "g2m":
            return g2m_nodes
        if name.startswith("mesh"):
            return np.arange(Nm)
        if name == "enc.g2m_edge" and kind != "table":
            return g2m_edges
        if name.startswith("proc") and name.endswith(".edge") and kind != "table":
            return edges[int(name[4:-5])]
        return np.arange(Nm) if rows == Nm else grid
    return pick


class Checker:
    """taps: {0: statics, n: {tap: decoded float64 values}} of one engine (or Emulator) step.  ``rows``: {n: the rows
    checked in unit n (its own row space; k-major units: k n_grid + g), 0: {static tap: rows}} — the taps are then Rows
    holding at least what Planner lists; a unit without an entry is checked on every row.  References are evaluated in
    blocks of BLOCK rows on up to WORKERS threads (numpy and BLAS release the GIL); each block reduces its checks to
    (n_outside, worst ratio), and the blocks merge in order."""

    def __init__(self, cfg, graph, w, x, t_seconds, taps, rows=None):
        self.cfg, self.g, self.w, self.x, self.t, self.taps = cfg, graph, w, np.asarray(x, np.float32), t_seconds, taps
        self.rows = rows or {}
        self.n = 0
        self.checks = []     # (unit, kind, name, what, n_outside, worst ratio)
        self._at = {}

    def _run(self, blocks, fn):
        """fn(R, chk) for every row block R; chk(kind, name, what, got, ref, bound) checks one quantity on the block"""
        def one(R):
            out = []
            fn(R, lambda kind, name, what, got, ref, bound: out.append((kind, name, what) + _summary(got, ref, bound)))
            return out
        if len(blocks) == 1:
            res = [one(blocks[0])]
        else:
            with ThreadPoolExecutor(min(WORKERS, len(blocks))) as ex:
                res = list(ex.map(one, blocks))
        for out in res:
            for kind, name, what, bad, wr in out:
                key = (self.n, kind, name, what)
                if key in self._at:
                    i = self._at[key]
                    self.checks[i] = key + (bad + self.checks[i][4], max(wr, self.checks[i][5]))
                else:
                    self._at[key] = len(self.checks)
                    self.checks.append(key + (bad, wr))

    def _unit(self, nrows):
        """-> (taps of the next unit, the rows it is checked on in blocks of BLOCK)"""
        self.n += 1
        R = self.rows.get(self.n)
        return self.taps[self.n], _blocks(np.arange(nrows) if R is None else R)

    def statics(self):
        cfg, g, w, t = self.cfg, self.g, self.w, self.taps[0]
        r0 = self.rows.get(0, {})
        for tap, name, feat in (("vm0_img", "enc.mesh_embed", g["mesh.node_feat"]), ("e_g2m_img", "enc.g2m_edge_embed", g["g2m.edge_feat"]),
                                ("e_mesh_img", "proc.edge_embed", g["mesh.edge_feat"]), ("e_m2g_img", "dec.m2g_edge_embed", g["m2g.edge_feat"])):
            feat = np.asarray(feat, np.float32).reshape(-1, np.asarray(feat).shape[-1])

            def block(R, chk, tap=tap, name=name, feat=feat):
                _, y, yb = ref_static(feat[R], w, name, cfg.ln_eps)
                chk("static", name, tap, t[tap][R], y, gr.f16_bound(y, yb))
                if tap == "vm0_img":
                    chk("static", name, "vm0", t["vm0"][R], y, yb)
                    chk("static", name, "vm0_img = fp16(vm0)", t["vm0_img"][R], q16(t["vm0"][R]), 0.0)
            self._run(_blocks(r0.get(tap, np.arange(len(feat)))), block)

        def block(R, chk):
            f, fb = ref_table(t["vm0_img"][R], [np.asarray(w["enc.g2m_edge.w1"])[:, 2 * L:3 * L]])
            chk("static", "enc.g2m_edge", "g2m_tr", t["g2m_tr"][R], f, fb)
        self._run(_blocks(r0.get("g2m_tr", np.arange(int(g["n_mesh"])))), block)
        return t

    def features(self):
        t, blocks = self._unit(self.cfg.n_grid)
        ref, bound = ref_features(self.cfg, self.w, self.g, self.x, self.t)
        nf = self.cfg.n_features

        def block(R, chk):
            got = t["feat"][R]
            chk("features", "features", "feat", got[:, :nf], ref[R, :nf], bound[R, :nf])
            chk("features", "features", "feat padding", got[:, nf:], 0.0, 0.0)
        self._run(blocks, block)
        return t["feat"]

    def hidden(self, name, parts, out, rows, gathers=(), kmajor=False):
        t, blocks = self._unit(rows)
        w1 = np.asarray(self.w[name + ".w1"])

        def block(R, chk):
            f, fb = ref_hidden([(a[R], w1[:, c0:c1]) for a, (c0, c1) in parts], self.w[name + ".b1"],
                               [(tb, np.asarray(i)[R]) for tb, i in gathers])
            chk("hidden", name, out, t[out][R], f, fb)
        self._run(blocks, block)
        return t[out]

    def ln(self, name, hid, res, outs, rows, kmajor=False):
        t, blocks = self._unit(rows)

        def block(R, chk):
            y, s, b = ref_ln(hid[R], self.w, name, None if res is None else res[R], self.cfg.ln_eps)
            for k, tap in outs.items():
                r = y if k == "yimg" else s
                chk("ln", name, tap, t[tap][R], r, b if k == "xout" else gr.f16_bound(r, b))
            if "xout" in outs and "img" in outs:
                chk("ln", name, f"{outs['img']} = fp16({outs['xout']})", t[outs["img"]][R], q16(t[outs["xout"]][R]), 0.0)
        self._run(blocks, block)
        return {k: t[tap] for k, tap in outs.items()}

    def table(self, name, a, c0s, out, rows):
        t, blocks = self._unit(rows)
        w1 = np.asarray(self.w[name + ".w1"])

        def block(R, chk):
            f, fb = ref_table(a[R], [w1[:, c0:c0 + L] for c0 in c0s])
            chk("table", name, out, t[out][R], f, fb)
        self._run(blocks, block)
        return t[out]

    def agg(self, name, y, ptr):
        t, blocks = self._unit(len(ptr) - 1)

        def block(R, chk):
            f, fb = ref_agg(y, ptr, R)
            chk("agg", name, "agg_img", t["agg_img"][R], f, fb)
        self._run(blocks, block)
        return t["agg_img"]

    def out(self, hid):
        cfg = self.cfg
        t, blocks = self._unit(cfg.n_grid)
        R = np.concatenate(blocks)
        ns, npg = cfg.n_state, cfg.n_prog
        x = self.x.reshape(2 * ns, -1)[:, R].astype(np.float64)
        ref, bound = ref_out(hid[R], self.w, x[ns:ns + npg].T, npg)
        # x_out: the new state [2 n_state, nlat, nlon], or Rows of grid points [n, 2 n_state]
        xo = t["x_out"][R].T if isinstance(t["x_out"], Rows) else np.asarray(t["x_out"], np.float64).reshape(2 * ns, -1)[:, R]
        # the planes the feature kernel writes: slice 0 = the old slice 1 bit for bit, the new forcing = toa(t + dt)
        from oracle.graphcast_ref import toa_radiation
        lat = np.linspace(90.0, -90.0, cfg.nlat); lon = np.arange(cfg.nlon) * (360.0 / cfg.nlon)
        toa = toa_radiation(self.t + 3600.0 * cfg.dt_hours, lat, lon).reshape(-1)

        def block(_, chk):
            chk("out", "dec.out", "x_out", xo[ns:ns + npg].T, ref, bound)
            chk("features", "features", "x_out slice 0", xo[:ns], x[ns:], 0.0)
            chk("features", "features", "x_out toa(t+dt)", xo[2 * ns - 1], toa[R], TOA_REL * toa.max())
        self._run([R], block)


BLOCK = 8192           # rows per reference evaluation: bounds each thread's temporaries at full size
WORKERS = min(8, os.cpu_count() or 1)


def _blocks(R):
    return [R[i:i + BLOCK] for i in range(0, len(R), BLOCK)] or [R]


def _summary(got, ref, bound):
    """-> (elements outside, worst |got - ref| / bound); NaN counts as outside, a bound of 0 asks for equality"""
    got = np.asarray(got, np.float64)
    ref = np.broadcast_to(np.asarray(ref, np.float64), got.shape)
    bound = np.broadcast_to(np.asarray(bound, np.float64), got.shape)
    bad = int(gr.exceed(got, ref, bound).sum())
    exact = bound == 0
    wr = gr.worst(got[~exact], ref[~exact], bound[~exact]) if (~exact).any() else 0.0
    if exact.any() and not np.array_equal(got[exact], ref[exact]):
        wr = math.inf
    return bad, wr


def check_step(cfg, graph, w, x, t_seconds, taps, rows=None):
    """-> [(unit, kind, name, what, n_outside, worst ratio)]; NaN counts as outside.  ``rows``: Checker's"""
    c = Checker(cfg, graph, w, x, t_seconds, taps, rows)
    run_program(cfg, graph, c)
    return c.checks


def by_stage(results):
    """{stage kind: worst ratio} of check_step's results"""
    d = {}
    for n, kind, name, what, bad, wr in results:
        d[kind] = max(d.get(kind, 0.0), wr)
    return d


class Emulator:
    """the engine's formulation in numpy.  ``mut``: one modelled mistake (tests/test_graphcast_stages_cpu.py)"""

    def __init__(self, cfg, graph, w, x, t_seconds, mut=None):
        self.cfg, self.g, self.w, self.x, self.t, self.mut = cfg, graph, w, np.asarray(x, np.float32), t_seconds, mut
        self.n = 0
        self.taps = {}
        self.agg_prev = None

    def _put(self, **kw):
        self.n += 1
        self.taps[self.n] = kw

    def statics(self):
        cfg, g, w = self.cfg, self.g, self.w
        t = {}
        for tap, name, feat in (("vm0_img", "enc.mesh_embed", g["mesh.node_feat"]), ("e_g2m_img", "enc.g2m_edge_embed", g["g2m.edge_feat"]),
                                ("e_mesh_img", "proc.edge_embed", g["mesh.edge_feat"]), ("e_m2g_img", "dec.m2g_edge_embed", g["m2g.edge_feat"])):
            f = q16(ref_hidden([(q16(feat), w[name + ".w1"])], w[name + ".b1"])[0])     # the hidden image the engine frees
            y = ref_ln(f, w, name, None, cfg.ln_eps)[0]
            if tap == "vm0_img":
                t["vm0"] = y.astype(np.float32).astype(np.float64)
                y = t["vm0"]
            t[tap] = q16(y)
        t["g2m_tr"] = q16(ref_table(t["vm0_img"], [np.asarray(w["enc.g2m_edge.w1"])[:, 2 * L:3 * L]])[0])
        self.taps[0] = t
        return t

    def features(self):
        f = q16(ref_features(self.cfg, self.w, self.g, self.x, self.t)[0])
        if self.mut == "swap_day_sincos":
            c = 2 * self.cfg.n_prog + 3 + 2
            f[:, [c, c + 1]] = f[:, [c + 1, c]]
        self._put(feat=f)
        return f

    def hidden(self, name, parts, out, rows, gathers=(), kmajor=False):
        w1 = np.asarray(self.w[name + ".w1"])
        if self.mut == "swap_tables" and name == "proc0.edge":
            gathers = [(gathers[1][0], gathers[0][1]), (gathers[0][0], gathers[1][1])]
        f = q16(ref_hidden([(a, w1[:, c0:c1]) for a, (c0, c1) in parts], self.w[name + ".b1"], gathers)[0])
        self._put(**{out: f})
        return f

    def ln(self, name, hid, res, outs, rows, kmajor=False):
        if self.mut == "no_residual_grid" and name == "enc.g2m_grid":
            res = None
        y, s, _ = ref_ln(hid, self.w, name, res, self.cfg.ln_eps)
        o = {}
        for k in outs:
            v = (y if k == "yimg" else s).astype(np.float32).astype(np.float64)
            o[k] = v if k == "xout" else q16(v)
        if self.mut == "shift_last_row" and name == "enc.grid_embed":
            o["img"][-1] = o["img"][-2]
        if self.mut == "scale_last_row" and name == "enc.grid_embed":
            o["img"][-1] = q16(1.1 * o["img"][-1])
        self._put(**{outs[k]: o[k] for k in outs})
        return o

    def table(self, name, a, c0s, out, rows):
        w1 = np.asarray(self.w[name + ".w1"])
        if self.mut == "w1r_from_w1s" and name == "proc0.edge":
            c0s = [c0s[0], c0s[0]]
        f = q16(ref_table(a, [w1[:, c0:c0 + L] for c0 in c0s])[0])
        self._put(**{out: f})
        return f

    def agg(self, name, y, ptr):
        prev = self.agg_prev if self.agg_prev is not None else np.ones((len(ptr) - 1, L), np.float32)
        mut = self.mut if (name == "g2m" or self.mut == "stale_zero_degree") else None
        f = q16(segsum_f32(y, ptr, prev=prev if mut == "stale_zero_degree" else None, mut=mut))
        self.agg_prev = f
        self._put(agg_img=f)
        return f

    def out(self, hid):
        cfg = self.cfg
        ns, npg = cfg.n_state, cfg.n_prog
        x2 = self.x.reshape(2 * ns, -1)
        ref, _ = ref_out(hid, self.w, x2[ns:ns + npg].T.astype(np.float64), npg)
        xo = np.zeros_like(x2)
        xo[:ns] = x2[ns:]
        xo[ns:ns + npg] = ref.T.astype(np.float32)
        from oracle.graphcast_ref import toa_radiation
        lat = np.linspace(90.0, -90.0, cfg.nlat); lon = np.arange(cfg.nlon) * (360.0 / cfg.nlon)
        xo[2 * ns - 1] = toa_radiation(self.t + 3600.0 * cfg.dt_hours, lat, lon).reshape(-1)
        self._put(x_out=xo)
        self.tendency = (ref - x2[ns:ns + npg].T) / np.asarray(self.w["norm.diff_std"], np.float64)[None, :npg]


def emulate(cfg, graph, w, x, t_seconds, mut=None):
    e = Emulator(cfg, graph, w, x, t_seconds, mut)
    run_program(cfg, graph, e)
    return e


# ---------------------------------------------------------------------------------------------------------------------
# hand-built graphs: degrees the icosahedral graphs never have
# ---------------------------------------------------------------------------------------------------------------------
G2M_DEGREES = (0, 1, 3, 4, 5, 63, 64, 65, 127, 128, 129, 256, 257, 4321)
MESH_DEGREES = (0, 1, 64, 65, 200)


def csr_edges(degrees, senders_of, n_send, rng):
    """receiver-sorted edge set with the given in-degree per receiver: (senders, receivers, ptr)"""
    recv = np.repeat(np.arange(len(degrees)), degrees).astype(np.int64)
    send = np.concatenate([senders_of(n, d) for n, d in enumerate(degrees)] + [np.zeros(0, np.int64)]).astype(np.int64)
    ptr = np.concatenate([[0], np.cumsum(degrees)]).astype(np.int64)
    assert len(send) == len(recv) == ptr[-1] and (send >= 0).all() and (send < n_send).all()
    return send, recv, ptr


def hand_graph(base, seed=0):
    """``base`` (icomesh.build_graph) with its grid2mesh and mesh edge sets replaced: grid2mesh in-degrees 0 (first and
    last node among them), 1, 3, 4, 5, 63, 64, 65, 127, 128, 129, 256, 257 and one of 4321, senders drawn with repeats and
    grid points 0 and n_grid - 1 among them; mesh in-degrees 0, 1, 64, 65 and 200 (the partial-row route no icosahedron
    takes), a self-edge and a duplicated (sender, receiver) pair.  Edge features are seeded random rows."""
    rng = np.random.default_rng(seed)
    g = type(base)(base)
    ng, nm = int(base["n_grid"]), int(base["n_mesh"])
    deg = rng.integers(2, 41, size=nm)
    deg[[0, nm - 1, nm // 2]] = 0
    slots = rng.permutation(np.arange(1, nm - 1))[:len(G2M_DEGREES) + 1]
    slots = slots[slots != nm // 2][:len(G2M_DEGREES)]
    deg[slots] = G2M_DEGREES
    s, r, p = csr_edges(deg, lambda n, d: rng.integers(0, ng, size=d), ng, rng)
    big = int(np.argmax(deg))
    s[p[big]], s[p[big] + 1], s[p[big] + 2] = 0, ng - 1, ng - 1
    g["g2m.senders"], g["g2m.receivers"], g["g2m.ptr"] = s, r, p
    g["g2m.edge_feat"] = rng.uniform(-1, 1, size=(len(s), 4)).astype(np.float32)
    deg = rng.integers(2, 9, size=nm)
    slots = rng.permutation(np.arange(1, nm - 1))[:len(MESH_DEGREES)]
    deg[slots] = MESH_DEGREES
    deg[[0, nm - 1]] = 0
    s, r, p = csr_edges(deg, lambda n, d: rng.integers(0, nm, size=d), nm, rng)
    n200 = int(slots[MESH_DEGREES.index(200)])
    s[p[n200]] = n200                                  # a self-edge
    s[p[n200] + 1] = s[p[n200] + 2]                    # a duplicated (sender, receiver) pair
    g["mesh.senders"], g["mesh.receivers"], g["mesh.ptr"] = s, r, p
    g["mesh.edge_feat"] = rng.uniform(-1, 1, size=(len(s), 4)).astype(np.float32)
    return g


# ---------------------------------------------------------------------------------------------------------------------
# chained comparison against GraphCastRef's taps
# ---------------------------------------------------------------------------------------------------------------------
def chain_pairs(cfg, graph, w, x, taps):
    """[(oracle tap name, engine values [rows, columns])]: every latent, update, aggregate and the network output, under
    the names of GraphCastRef.tendency(taps=...)"""
    at = {(kind, name): n for n, (kind, name, _) in enumerate(units(cfg, graph), 1)}
    get = lambda kind, name, tap: taps[at[(kind, name)]][tap]
    ns, npg = cfg.n_state, cfg.n_prog
    out = [("feat", get("features", "features", "feat")[:, :cfg.n_features]),
           ("grid_embed", get("ln", "enc.grid_embed", "vg_img")), ("g2m_update", get("ln", "enc.g2m_edge", "yimg")),
           ("g2m_agg", get("agg", "g2m", "agg_img")), ("enc_mesh", get("ln", "enc.g2m_mesh", "vm")),
           ("enc_grid", get("ln", "enc.g2m_grid", "vg_img"))]
    for i in range(cfg.layers):
        out += [(f"proc{i}_update", get("ln", f"proc{i}.edge", "ym_img")), (f"proc{i}_agg", get("agg", f"mesh{i}", "agg_img")),
                (f"proc{i}_mesh", get("ln", f"proc{i}.node", "vm"))]
        if i + 1 < cfg.layers:
            out.append((f"proc{i}_edges", get("ln", f"proc{i}.edge", "em_img")))
    xo = np.asarray(get("out", "dec.out", "x_out"), np.float64).reshape(2 * ns, -1)[ns:ns + npg]
    x1 = np.asarray(x, np.float64).reshape(2 * ns, -1)[ns:ns + npg]
    out += [("m2g_update", get("ln", "dec.m2g_edge", "yimg")), ("dec_grid", get("ln", "dec.m2g_grid", "vg_img")),
            ("out", ((xo - x1) / np.asarray(w["norm.diff_std"], np.float64)[:npg, None]).T)]
    return out


def row_rel(got, ref):
    """per-row relative L2 error; a row whose reference is (numerically) empty, such as the aggregate of a node without
    edges, is measured against the median row norm"""
    got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
    den = np.linalg.norm(ref, axis=1)
    return np.linalg.norm(got - ref, axis=1) / np.maximum(den, 1e-3 * np.median(den) + 1e-30)


CHAIN_FLOOR = 1e-3     # one fp16 rounding per element is 2^-11 = 4.9e-4 of a row's norm at most; twice that
CHAIN_FACTOR = 4.0     # over the largest row error of the oracle's own fp16 emulation (emulate="fp16s") of the same tap


def chain_bounds(cfg, graph, w, x, t_seconds):
    """(fp64 oracle taps, {tap: row bound}): CHAIN_FACTOR x the largest per-row error of GraphCastRef(emulate="fp16s")
    against the fp64 oracle, at least CHAIN_FLOOR"""
    import torch
    from oracle.graphcast_ref import GraphCastRef
    ref, emu = {}, {}
    GraphCastRef(cfg, w, graph, dtype=torch.float64).tendency(x, t_seconds, taps=ref)
    GraphCastRef(cfg, w, graph, dtype=torch.float64, emulate="fp16s").tendency(x, t_seconds, taps=emu)
    ref = {k: v.numpy() for k, v in ref.items()}
    tol = {k: max(CHAIN_FLOOR, CHAIN_FACTOR * float(row_rel(emu[k].numpy(), ref[k]).max())) for k in ref}
    return ref, tol
