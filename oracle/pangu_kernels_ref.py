"""ORACLE — test infrastructure, not product code.

Layouts and float64 references of Pangu's windowing kernels (skyrim_b200/csrc/attention_tc.cuh, pangu_engine.cu) at
kernel level, for tests/test_pangu_kernels_gpu.py (which launches the kernels through libskyrim_b200_probe.so) and
tests/test_pangu_kernels_cpu.py (which checks this module on its own and against oracle/pangu_ref.py).

Window image (DESIGN.md §3), packed here from that description alone, independently of the CUDA producers:
  [part q|k|v][member][window][head pair] -> one tile of 144 rows x 128 B
  row j = (zj, hj, wj) position in the (rolled) window, j = (zj * 6 + hj) * 12 + wj
  128 B = [head 2p: 32 halves | head 2p+1: 32 halves], 16-byte chunk c stored at c ^ (j & 7)
window = (wz * nWh + wh) * nWw + ww; the bias window type is wz * nWh + wh.  Windows are cut from the natural token grid
exactly as PanguRef.block does it: pad the latitude axis to Hp with zero tokens, roll by (-1, -3, -6) when shifted.

Attention bound (attention_ref).  Per element, not a norm, derived from the kernel's arithmetic (base-2 softmax):
  scores   s_j = fmaf(q.k_j, sl2, b_j): the fp32 tensor-core dot is within TAU * sum_d |q_d k_jd| (TAU of gemm_ref), the
           fmaf adds one fp32 rounding: |s_j - t_j| <= delta_j = sl2 TAU S_j + U32 |t_j|;
  exp      e_j = ex2.approx(s_j - mx): the row max mx is some s_j, so 2^(m - mx) is common to every e_j of the row and
           cancels in P V / sum (only the absolute terms below see it: c = 2^-max delta); the fp32 subtraction adds
           U32 |s_j - mx|, ex2.approx.ftz a relative 2^-21 (PTX ISA: 2 ulp) and a flush of results below 2^-126:
           e_j = c a_j (1 + r_j) with a_j = 2^(t_j - m), |r_j| <= rho_j = 2^(delta_j + U32 (m - t_j + 2 max delta)) (1 + 2^-21) - 1;
  P        rounded to fp16 for the tensor core, |p_j - e_j| <= 2^-11 e_j + 2^-25 (+ 2^-126 flushed), while the row sum
           adds the unrounded e_j in fp32 (144 terms: relative GAMMA = 143 U32 + the flushes);
  P V      fp32 tensor-core accumulation: TAU * sum_j p_j |v_j|;
  output   (P V) * (1 / sum): two fp32 roundings, then the fp16 store (half an fp16 ulp, f16_bound).
With w_j = a_j / sum a, A = sum a >= 1 and rhobar = sum w_j rho_j, first order in each term and exact in the denominator:
  |o - ref| <= [sum_j w_j |v_j| (rho_j + rhobar + 2^-11 (1 + rho_j) + GAMMA (1 + rhobar) + TAU (1 + rho_j) (1 + 2^-11))
               + (1 + TAU) sum_j (2^-25 + 2^-126) |v_j| / (c A)] / ((1 - rhobar)(1 - GAMMA)) + 2 U32 |ref|
The reference starts from the exact fp16 q, k, v and the fp16 bias entries the kernel reads, including the fp16
rounding of bias + mask (__hadd), so nothing else is left to bound.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from oracle import gemm_ref as gr

LOG2E = 1.4426950408889634
WZ, WH, WW = 2, 6, 12
SZ, SH, SW = WZ // 2, WH // 2, WW // 2
NTOK = WZ * WH * WW                      # 144 tokens per window
TILE_B = NTOK * 128                      # bytes of one (window, head pair) tile of q, k or v
TABLE = (2 * WW - 1) * WH * WH * WZ * WZ  # 3312 compact bias entries per (type, head)
EX2_REL = 2.0 ** -21                     # ex2.approx.ftz.f32: maximum relative error 2 ulp (PTX ISA)
FTZ = 2.0 ** -126                        # its flush-to-zero threshold
GAMMA = 143 * gr.U32                     # fp32 sum of 144 positive terms


# ---------------------------------------------------------------------------------------------------------------------
# geometry
# ---------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Grid:
    """one resolution level of the Pangu token grid (the engine's Geo)"""
    Z: int
    H: int
    W: int
    C: int
    heads: int

    @property
    def Hp(self):
        return -(-self.H // WH) * WH

    @property
    def nWz(self):
        return self.Z // WZ

    @property
    def nWh(self):
        return self.Hp // WH

    @property
    def nWw(self):
        return self.W // WW

    @property
    def T(self):
        return self.Z * self.H * self.W

    @property
    def nWin(self):
        return self.nWz * self.nWh * self.nWw

    @property
    def pairs(self):
        return self.heads // 2

    @property
    def n_type(self):
        return self.nWz * self.nWh

    def probe_geo(self) -> dict:
        """the fields of sky_probe_geo_t"""
        return dict(Z=self.Z, H=self.H, W=self.W, C=self.C, Hp=self.Hp, nWz=self.nWz, nWh=self.nWh, nWw=self.nWw, T=self.T,
                    nWin=self.nWin, heads=self.heads)


def grids(cfg) -> tuple[Grid, Grid]:
    """the two token grids the engine builds for a PanguConfig"""
    return (Grid(cfg.Z, cfg.H, cfg.W, cfg.dim, cfg.heads[0]), Grid(cfg.Z, cfg.H2, cfg.W2, 2 * cfg.dim, cfg.heads[1]))


def window_tokens(g: Grid, roll: int, B: int = 1, sign: int = -1) -> np.ndarray:
    """[B, nWin, 144] natural token (member * T + t) at each window row, -1 for a latitude-padding row.  Pad, then roll
    by sign * (1, 3, 6) (PanguRef.block: sign = -1; +1 only to model a roll in the wrong direction)."""
    idx = np.arange(g.T, dtype=np.int64).reshape(g.Z, g.H, g.W)
    y = np.pad(idx, ((0, 0), (0, g.Hp - g.H), (0, 0)), constant_values=-1)
    if roll:
        y = np.roll(y, (sign * SZ, sign * SH, sign * SW), axis=(0, 1, 2))
    yw = y.reshape(g.nWz, WZ, g.nWh, WH, g.nWw, WW).transpose(0, 2, 4, 1, 3, 5).reshape(g.nWin, NTOK)
    b = np.arange(B, dtype=np.int64)[:, None, None] * g.T
    return np.where(yw[None] >= 0, yw[None] + b, -1)


def window_types(g: Grid) -> np.ndarray:
    """[nWin] bias window type of each window"""
    return np.arange(g.nWin) // g.nWw


def row_position(j):
    """window row j -> (zj, hj, wj)"""
    j = np.asarray(j)
    return j // (WH * WW), (j // WW) % WH, j % WW


# ---------------------------------------------------------------------------------------------------------------------
# window image
# ---------------------------------------------------------------------------------------------------------------------
def window_image_offset(g: Grid, B: int, part_stride: int, part: int, b: int, win: int, head: int, j: int, d: int) -> int:
    """byte offset of element d of head `head` at row j of window `win`, member b, part (0 q, 1 k, 2 v)"""
    pair, hh = divmod(head, 2)
    tile = (b * g.nWin + win) * g.pairs + pair
    c, e = divmod(hh * 32 + d, 8)
    return part * part_stride + tile * TILE_B + j * 128 + ((c ^ (j & 7)) << 4) + 2 * e


def pack_window_image(qkv: np.ndarray, part_stride: int | None = None, gap_fill=np.nan) -> np.ndarray:
    """q | k | v [3, B, nWin, heads, 144, 32] -> image bytes; parts `part_stride` bytes apart, the gaps `gap_fill`"""
    qkv = np.asarray(qkv, np.float16)
    _, B, nWin, heads, n, d = qkv.shape
    assert n == NTOK and d == 32 and heads % 2 == 0
    t = qkv.reshape(3, B, nWin, heads // 2, 2, NTOK, 32).transpose(0, 1, 2, 3, 5, 4, 6).reshape(3, -1, NTOK, 8, 8)
    idx = np.broadcast_to(gr._swz_index(NTOK)[None, None, :, :, None], t.shape)
    t = np.take_along_axis(t, idx, axis=3).reshape(3, -1)
    size = t.shape[1] * 2
    ps = size if part_stride is None else part_stride
    assert ps >= size and ps % 2 == 0
    out = np.full((3, ps // 2), gap_fill, np.float16)
    out[:, : t.shape[1]] = t
    return out.reshape(-1)[: 2 * (ps // 2) + t.shape[1]].view(np.uint8)   # the last part ends with its data


def unpack_tiles(tiles: np.ndarray) -> np.ndarray:
    """window image tiles [..., 144 rows x 128 B] (any leading shape, fp16 or bytes) -> [..., 2 heads, 144, 32]"""
    h = np.asarray(tiles).view(np.float16)
    lead = h.shape[:-1] if h.shape[-1] == NTOK * 64 else h.shape[:-2]
    v = h.reshape(*lead, NTOK, 8, 8)
    idx = np.broadcast_to(gr._swz_index(NTOK).reshape((1,) * len(lead) + (NTOK, 8, 1)), v.shape)
    x = np.take_along_axis(v, idx, axis=-2).reshape(*lead, NTOK, 2, 32)
    return np.moveaxis(x, -2, -3)


def unpack_window_image(img: np.ndarray, g: Grid, B: int, part_stride: int | None = None) -> np.ndarray:
    """inverse of pack_window_image: -> [3, B, nWin, heads, 144, 32] fp16"""
    size = B * g.nWin * g.pairs * TILE_B
    ps = size if part_stride is None else part_stride
    h = np.asarray(img).reshape(-1).view(np.float16)
    parts = np.stack([h[p * ps // 2: p * ps // 2 + size // 2] for p in range(3)])
    x = unpack_tiles(parts.reshape(3, B, g.nWin, g.pairs, NTOK * 64))     # [3, B, nWin, pairs, 2, 144, 32]
    return x.reshape(3, B, g.nWin, g.heads, NTOK, 32)


def windows_from_tokens(qkv_tok: np.ndarray, pad_row: np.ndarray, idx: np.ndarray, heads: int) -> np.ndarray:
    """the window image's contents: natural-order projections [rows, 3C] and the padding tokens' row [3C] (the QKV
    bias) gathered at window rows idx [..., 144] -> [3, ..., heads, 144, 32]"""
    rows = np.where((idx >= 0)[..., None], np.asarray(qkv_tok)[np.maximum(idx, 0)], np.asarray(pad_row)[None])
    lead = idx.shape[:-1]
    x = rows.reshape(*lead, NTOK, 3, heads, 32)
    return np.moveaxis(np.moveaxis(x, -3, 0), -2, -3)


def tokens_from_windows(o: np.ndarray, idx: np.ndarray, rows: int) -> np.ndarray:
    """attention outputs [..., heads, 144, 32] at window rows idx [..., 144] -> natural tokens [rows, heads * 32] (NaN
    where no window row holds the token); padding rows are dropped"""
    heads = o.shape[-3]
    x = np.moveaxis(o, -3, -2).reshape(-1, heads * 32)
    i = idx.reshape(-1)
    out = np.full((rows, heads * 32), np.nan)
    out[i[i >= 0]] = x[i >= 0]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# bias tables and masks
# ---------------------------------------------------------------------------------------------------------------------
def pack_bias_table(src: np.ndarray) -> np.ndarray:
    """k_pack_bias_table: fp32 (3312, n_type, heads) -> fp16 (n_type, heads, 3312) of fp32(x * fp32(log2 e))"""
    src = np.asarray(src, np.float32)
    with np.errstate(over="ignore"):      # overflow rounds to inf, as __float2half_rn does
        return (src * np.float32(LOG2E)).astype(np.float16).transpose(1, 2, 0).copy()


def position_index() -> np.ndarray:
    """(144, 144) compact table index of every (query, key) pair (oracle/pangu_ref.py)"""
    from oracle.pangu_ref import position_index as pi
    return pi((WZ, WH, WW)).numpy()


def shift_mask_types(g: Grid) -> np.ndarray:
    """(n_type, 144, 144) bool: pairs the shifted-window mask separates (oracle/pangu_ref.py shift_mask)"""
    import torch
    from oracle.pangu_ref import shift_mask
    from skyrim_b200.config import PanguConfig
    return shift_mask(PanguConfig(), g.Z, g.Hp, g.W, torch.float64).numpy() != 0


def seam_masks(g: Grid) -> tuple[np.ndarray, np.ndarray]:
    """the shift mask split by axis: (n_type, 144, 144) pairs across the Z seam, and across the latitude seam.  Their union
    is shift_mask_types (checked in the CPU tests); they exist to model a kernel that drops one axis."""
    zj, hj, _ = row_position(np.arange(NTOK))
    wz, wh = np.divmod(np.arange(g.n_type), g.nWh)
    zr = (wz == g.nWz - 1)[:, None] & (zj >= WZ - SZ)[None]     # last z-window: rows from the far side of the seam
    hr = (wh == g.nWh - 1)[:, None] & (hj >= WH - SH)[None]
    return zr[:, :, None] != zr[:, None, :], hr[:, :, None] != hr[:, None, :]


def gathered_bias(tab16: np.ndarray, types: np.ndarray, mask: np.ndarray | None, mask_l2: float, pos: np.ndarray | None = None,
                  round16: bool = True) -> np.ndarray:
    """[n, heads, 144, 144] bias entry of each (window, head, query, key): the fp16 table entry, + fp16(mask_l2) rounded to
    fp16 (__hadd) where the mask separates the pair; round16=False adds in float64 (the unrounded model)"""
    pos = position_index() if pos is None else pos
    b = np.asarray(tab16)[np.asarray(types)][:, :, pos].astype(np.float64)     # [n, heads, 144, 144]
    if mask is not None:
        mt = np.asarray(mask)[np.asarray(types)][:, None]                        # [n, 1, 144, 144]
        if round16:
            m16 = float(np.float16(np.float32(mask_l2)))
            b = np.where(mt, (b + m16).astype(np.float16).astype(np.float64), b)
        else:
            b = np.where(mt, b + mask_l2, b)
    return b


# ---------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------
def attention_ref(q, k, v, bias, sl2: float, chunk: int = 32) -> tuple[np.ndarray, np.ndarray]:
    """softmax_2(sl2 q k^T + bias) v in float64, and its per-element bound (module docstring).  q, k, v [n, heads, 144, 32]
    (the fp16 values the kernel reads), bias [n, heads, 144, 144] (gathered_bias).  Returns (ref, bound), bound being
    that of the fp16 output."""
    n = q.shape[0]
    ref = np.empty(q.shape); bnd = np.empty(q.shape)
    for s in range(0, n, chunk):
        sl = slice(s, s + chunk)
        qq, kk, vv = (np.asarray(x[sl], np.float64) for x in (q, k, v))
        dot = qq @ np.swapaxes(kk, -1, -2)
        S = np.abs(qq) @ np.swapaxes(np.abs(kk), -1, -2)
        t = dot * sl2 + bias[sl]
        m = t.max(-1, keepdims=True)
        a = np.exp2(t - m)
        A = a.sum(-1, keepdims=True)
        w = a / A
        o = w @ vv
        delta = sl2 * gr.TAU * S + gr.U32 * np.abs(t)
        dmax = delta.max(-1, keepdims=True)
        rho = np.exp2(delta + gr.U32 * (m - t + 2 * dmax)) * (1 + EX2_REL) - 1
        rbar = (w * rho).sum(-1, keepdims=True)
        av = np.abs(vv)
        rel = (rho + rbar + 2.0 ** -11 * (1 + rho) + GAMMA * (1 + rbar) + gr.TAU * (1 + rho) * (1 + 2.0 ** -11))
        lin = (w * rel) @ av
        c = np.exp2(-dmax)
        absterm = (1 + gr.TAU) * (2.0 ** -25 + FTZ) * av.sum(-2, keepdims=True)     # [.., heads, 1, 32]
        b = (lin + absterm / (c * A)) / ((1 - rbar) * (1 - GAMMA)) + 2 * gr.U32 * np.abs(o)
        ref[sl] = o
        bnd[sl] = gr.f16_bound(o, b)
    return ref, bnd


def attention_windows(q, k, v, tab16, types, mask, mask_l2: float, sl2: float, pos=None, chunk: int = 32):
    """attention_ref over windows [n, heads, 144, 32] of bias window types `types` [n], the bias gathered a chunk of
    windows at a time (a full gather of many windows would not fit in memory)"""
    ref = np.empty(q.shape); bnd = np.empty(q.shape)
    for s in range(0, q.shape[0], chunk):
        sl = slice(s, s + chunk)
        ref[sl], bnd[sl] = attention_ref(q[sl], k[sl], v[sl], gathered_bias(tab16, types[sl], mask, mask_l2, pos), sl2)
    return ref, bnd


def sl2_mask_l2(mask_value: float = -100.0) -> tuple[float, float]:
    """the attention's fp32 scalars as the engine forms them: head_dim^-0.5 log2 e and mask value x log2 e"""
    l2 = np.float32(LOG2E)
    return float(np.float32(1.0 / np.sqrt(32.0)) * l2), float(np.float32(mask_value) * l2)


@dataclass
class AttnInputs:
    """natural-order q | k | v projections [B T, 3C] (fp16), the QKV bias [3C] (fp32: the padding tokens' rows are its
    fp16 rounding) and the fp32 earth-specific bias table (3312, n_type, heads)"""
    qkv_tok: np.ndarray
    bias: np.ndarray
    table: np.ndarray

    @property
    def pad_row(self):
        return self.bias.astype(np.float16)


def attention_inputs(g: Grid, B: int, seed: int, synthetic: bool = False) -> AttnInputs:
    """Inputs at which a wrong bias entry, mask, padding or window shows: q, k uniform in (-3, 3), so scores span several
    units (std ~3) and the softmaxes are peaked, and bias entries of O(1).  synthetic=True: the scale of the synthetic
    weights (q, k, v ~0.3, table std 0.02), nearly uniform softmaxes."""
    rng = np.random.default_rng(seed)
    s, ts = (0.3, 0.02) if synthetic else (3.0, 2.0)
    qkv = (rng.uniform(-1, 1, (B * g.T, 3 * g.C)) * s).astype(np.float16)
    bias = (rng.uniform(-1, 1, 3 * g.C) * s).astype(np.float32)
    table = (rng.uniform(-1, 1, (TABLE, g.n_type, g.heads)) * ts).astype(np.float32)
    return AttnInputs(qkv, bias, table)


def attention_tokens(g: Grid, B: int, roll: int, inp: AttnInputs, mask_value: float = -100.0, *, sign: int = -1, pos=None,
                     mask="shift", types=None, head_perm=None, pad_zero: bool = False):
    """Natural-token reference of window image -> attention -> output image, (ref [B T, C], bound), with the knobs that
    model a kernel's mistakes: the roll direction, the table index, the mask (None, "shift", or an (n_type, 144, 144)
    array), the window type of each window, the order of heads in the tables, zero instead of bias padding keys."""
    idx = window_tokens(g, roll, B, sign)                               # [B, nWin, 144]
    pad = np.zeros(3 * g.C, np.float16) if pad_zero else inp.pad_row
    q, k, v = windows_from_tokens(inp.qkv_tok, pad, idx, g.heads).reshape(3, B * g.nWin, g.heads, NTOK, 32)
    tab16 = pack_bias_table(inp.table)
    if head_perm is not None:
        tab16 = tab16[:, head_perm]
    sl2, ml2 = sl2_mask_l2(mask_value)
    m = (shift_mask_types(g) if isinstance(mask, str) else mask) if roll else None
    ty = np.tile(window_types(g) if types is None else types, B)
    o, b = attention_windows(q, k, v, tab16, ty, m, ml2, sl2, pos)
    return tokens_from_windows(o, idx, B * g.T), tokens_from_windows(b, idx, B * g.T)


def qkv_ref(x16: np.ndarray, w16: np.ndarray, bias: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """EpiQkvWin values: fp16(x W^T + bias) -> (reference, bound of the fp16 value), rows in natural token order"""
    R, S = gr.linear([(x16, w16)])
    ref, bnd = gr.epi_affine(R, S, np.asarray(bias, np.float32)[None])
    return ref, gr.f16_bound(ref, bnd)
