"""ORACLE — test infrastructure, not product code.

Float64 references of the units of Pangu's transformer blocks as PanguEngine::run_block_t wires them
(skyrim_b200/csrc/pangu_engine.cu), for tests/test_pangu_stages_gpu.py, which stops a real step after each unit
(debug_set "stop_launch") and reads the unit's output and its inputs, and tests/test_pangu_stages_cpu.py, which checks
this module against oracle/pangu_ref.py and shows that each modelled wiring mistake leaves the bounds.

Units of one step, in program order (units): the embedding (two GEMMs); per block QKV (the GEMM with its window-image
epilogue, and k_qkv_fill_pad where the latitude axis is padded), attention, projection + LayerNorm + residual, then the
MLP: one fused kernel with the image-only token stream at C = 192, else fc1 + GELU and fc2 + LayerNorm + residual (the
fp32 stream at C = 192, and both streams at C = 384, where projection and fc2 run on CTA pairs); the down-sample, the
up-sample (two launches each) and the recovery.

Every reference is built from the kernel-level ones: QKV from pangu_kernels_ref.qkv_ref and the window layout
(window_tokens, windows_from_tokens: padding rows are the fp16 QKV bias), attention from attention_ref with the gathered
fp16 bias table and shift mask, projection and fc2 from gemm_ref.layer_norm with the statistics model of the epilogue
that runs (ln_model), fc1 from gemm_ref.epi_gelu.  The fused MLP writes bit for bit what fc1 + fc2 write, but its fp16
hidden activation never leaves the SM: its reference multiplies the float64 GELU output, and the fp16 hidden activation
the kernel multiplies instead lies within hb = f16_bound of fc1's bound of it, which adds sum_k |w_k| hb_k to fc2's
accumulator error (passed to layer_norm as part of its tau S term).  Inputs are the engine's own: the fp16 stream image
rows (and fp32 rows with the fp32 stream), the window image, the attention output and hidden images as the unit read
them, and the packed fp16 weights (block_weights).  round16=False gives the same functions on unrounded weights and
float64 arithmetic throughout: the model (PanguRef.block), which the CPU tests check.

Knobs model one wiring mistake each: roll_flip (the roll of the wrong parity), table (the bias table of another block),
swap_pairs (head pairs 0 and 1 exchanged), pad_fill=False (padding rows of the window image left unfilled: zeros), ln
(the other LayerNorm's gamma and beta); the residual read from the wrong source is the caller's res argument.
"""
from __future__ import annotations

import numpy as np

from oracle import gemm_ref as gr
from oracle import pangu_kernels_ref as pk
from oracle import pangu_resample_ref as pr
from oracle.graphcast_stages_ref import CHAIN_FACTOR, CHAIN_FLOOR, row_rel


# ---------------------------------------------------------------------------------------------------------------------
# the unit list
# ---------------------------------------------------------------------------------------------------------------------
def level(cfg, li: int) -> pk.Grid:
    """the token grid layer li runs on"""
    g1, g2 = pk.grids(cfg)
    return g1 if li in (0, 3) else g2


def mlp_kinds(C: int, stream: str) -> tuple[str, ...]:
    """the MLP units of a block: the fused kernel with the image-only (fp16) stream at C = 192, else fc1 and fc2"""
    return ("mlp",) if stream == "fp16" and C == 192 else ("fc1", "fc2")


def units(cfg, stream: str) -> list[tuple[str, int, int, int]]:
    """(kind, layer, block, launches) of every unit of one step in program order; layer and block are -1 outside the
    transformer blocks"""
    out = [("embed", -1, -1, 2)]
    for li in range(4):
        if li in (1, 3):
            out.append(("down" if li == 1 else "up", -1, -1, 2))
        g = level(cfg, li)
        for bi in range(cfg.depths[li]):
            out += [("qkv", li, bi, 1 + (g.Hp > g.H)), ("attn", li, bi, 1), ("proj", li, bi, 1)]
            out += [(k, li, bi, 1) for k in mlp_kinds(g.C, stream)]
    out.append(("recover", -1, -1, 1))
    return out


def unit_index(cfg, stream: str) -> dict:
    """{(kind, layer, block): stop_launch value that stops the step right after the unit}"""
    return {(k, li, bi): n for n, (k, li, bi, _) in enumerate(units(cfg, stream), 1)}


# ---------------------------------------------------------------------------------------------------------------------
# weights
# ---------------------------------------------------------------------------------------------------------------------
def block_weights(w, li: int, bi: int, round16: bool = True) -> dict:
    """the GEMM weights of block bi of layer li as the engine packs them (fp16, [N, K]), its fp32 vectors and fp32 bias
    table, as float64"""
    p = f"layer{li}.block{bi}."
    out = {k: pr.packed(w[p + k + ".w"], round16) for k in ("qkv", "proj", "fc1", "fc2")}
    for k in ("qkv.b", "proj.b", "fc1.b", "fc2.b", "ln1.g", "ln1.b", "ln2.g", "ln2.b"):
        out[k] = np.asarray(w[p + k], np.float32).astype(np.float64)
    out["table"] = np.asarray(w[p + "bias_table"], np.float32)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------
def window_rows(g: pk.Grid, B: int, roll: int, wins) -> np.ndarray:
    """[len(wins), 144] natural token (member * T + t) of each row of windows wins (member * nWin + window), -1 for
    padding rows"""
    return pk.window_tokens(g, roll, B).reshape(B * g.nWin, pk.NTOK)[np.asarray(wins)]


def qkv_unit(g: pk.Grid, B: int, roll: int, wins, x, bw: dict, *, roll_flip: bool = False, pad_fill: bool = True,
             round16: bool = True):
    """EpiQkvWin + k_qkv_fill_pad: the stream x [B T, C] (the fp16 image rows the GEMM reads) -> the window image of
    windows wins, (reference, bound) [3, len(wins), heads, 144, 32]; padding rows hold fp16(bias) exactly"""
    idx = window_rows(g, B, roll ^ roll_flip, wins)
    toks = np.unique(idx[idx >= 0])
    local = np.where(idx >= 0, np.searchsorted(toks, np.maximum(idx, 0)), -1)
    xr = np.asarray(x)[toks].astype(np.float64)
    if round16:
        ref, bnd = pk.qkv_ref(xr, bw["qkv"], bw["qkv.b"])
        pad = bw["qkv.b"].astype(np.float32).astype(np.float16).astype(np.float64)
    else:
        ref, bnd = xr @ bw["qkv"].T + bw["qkv.b"][None], np.zeros((len(toks), 3 * g.C))
        pad = bw["qkv.b"]
    pad = pad if pad_fill else np.zeros(3 * g.C)
    return (pk.windows_from_tokens(ref, pad, local, g.heads), pk.windows_from_tokens(bnd, np.zeros(3 * g.C), local, g.heads))


def attention_unit(g: pk.Grid, B: int, roll: int, wins, qkv, bw: dict, mask_value: float, *, roll_flip: bool = False,
                   table=None, swap_pairs: bool = False, round16: bool = True, chunk: int = 32):
    """k_window_attention_tc on the window image values qkv [3, len(wins), heads, 144, 32] (as the kernel read them) ->
    (tokens, reference, bound): the natural tokens the windows' rows hold and their rows [n, C] of the output image"""
    r = roll ^ roll_flip
    idx = window_rows(g, B, r, wins)
    types = np.asarray(wins) % g.nWin // g.nWw
    tab = bw["table"] if table is None else np.asarray(table, np.float32)
    mask = pk.shift_mask_types(g) if r else None
    q, k, v = (np.asarray(a, np.float64) for a in qkv)
    if round16:
        sl2, ml2 = pk.sl2_mask_l2(mask_value)
        o, b = pk.attention_windows(q, k, v, pk.pack_bias_table(tab), types, mask, ml2, sl2, chunk=chunk)
    else:
        tab64 = tab.astype(np.float64).transpose(1, 2, 0) * pk.LOG2E
        o, b = np.empty(q.shape), np.empty(q.shape)
        for s in range(0, q.shape[0], chunk):
            sl = slice(s, s + chunk)
            bias = pk.gathered_bias(tab64, types[sl], mask, mask_value * pk.LOG2E, round16=False)
            o[sl], b[sl] = pk.attention_ref(q[sl], k[sl], v[sl], bias, 32 ** -0.5 * pk.LOG2E)
    if swap_pairs:
        o[:, [0, 1, 2, 3]], b[:, [0, 1, 2, 3]] = o[:, [2, 3, 0, 1]], b[:, [2, 3, 0, 1]]
    valid = idx.reshape(-1) >= 0
    rows = lambda a: np.moveaxis(a, 1, 2).reshape(-1, g.C)[valid]   # noqa: E731
    return idx.reshape(-1)[valid], rows(o), rows(b)


def ln_model(C: int, stream: str, fused: bool = False) -> dict:
    """gemm_ref.layer_norm's depth and shift of the LayerNorm epilogue that runs: the fragment path
    FragEpi<Epi2F32Img<true, 2>> with the image-only stream (and the fused MLP), Epi2F32Img<true, 1>::run with the fp32
    stream; on a CTA pair at C = 384"""
    pair = int(C == 384)
    if stream == "fp16" or fused:
        return dict(depth=gr.ln_depth(192 // 16 + 2, 2 + pair))
    return dict(depth=gr.ln_depth(192 // 8 + 2, 1 + pair), shift=gr.ln_shift(192))


def ln_unit(a, wt, bw: dict, bias: str, ln: str, res, eps: float, stream: str, *, a_bound=None, fused: bool = False,
            round16: bool = True):
    """Epi2F32Img<true, kRes>: LN(a W^T + bias) * gamma + beta + res -> (reference, bound of the fp32 value; the fp16
    image's is gr.f16_bound of it).  a_bound: a bound on the error of the A operand itself (the fused MLP's hidden)"""
    C = wt.shape[0]
    R, S = gr.linear([(a, wt)])
    if a_bound is not None:
        S = S + (np.asarray(a_bound, np.float64) @ np.abs(wt).T) / gr.TAU
    g, be = bw[ln + ".g"][None], bw[ln + ".b"][None]
    if not round16:
        y = R + bw[bias][None]
        mu, var = y.mean(1, keepdims=True), y.var(1, keepdims=True)
        return (y - mu) / np.sqrt(var + eps) * g + be + res, np.zeros_like(y)
    return gr.layer_norm(R, S, bw[bias][None], g, be, np.asarray(res, np.float64), eps, **ln_model(C, stream, fused))


def proj_unit(att, bw, res, eps, stream, *, ln: str = "ln1", round16: bool = True):
    """projection + LayerNorm (ln1) + residual from the attention output rows att [n, C]"""
    return ln_unit(att, bw["proj"], bw, "proj.b", ln, res, eps, stream, round16=round16)


def fc1_unit(x, bw, round16: bool = True):
    """fc1 + bias + GELU -> the fp16 hidden image rows [n, 4C]: (reference, bound of the fp16 value)"""
    R, S = gr.linear([(x, bw["fc1"])])
    if not round16:
        return gr.gelu(R + bw["fc1.b"][None]), np.zeros_like(R)
    f, fb = gr.epi_gelu(*gr.epi_affine(R, S, bw["fc1.b"][None]))
    return f, gr.f16_bound(f, fb)


def fc2_unit(hid, bw, res, eps, stream, *, ln: str = "ln2", round16: bool = True):
    """fc2 + LayerNorm (ln2) + residual from the hidden image rows hid [n, 4C]"""
    return ln_unit(hid, bw["fc2"], bw, "fc2.b", ln, res, eps, stream, round16=round16)


def mlp_unit(x, bw, res, eps, stream, *, ln: str = "ln2", round16: bool = True):
    """the fused MLP (mlp_fused.cuh) from the stream rows x [n, C] and residual res: fc1_unit, then fc2_unit on the
    float64 hidden activation with its fp16 bound carried into fc2's accumulator error (module docstring)"""
    h, hb = fc1_unit(x, bw, round16)
    if not round16:
        return fc2_unit(h, bw, res, eps, stream, ln=ln, round16=False)
    return ln_unit(h, bw["fc2"], bw, "fc2.b", ln, res, eps, stream, a_bound=hb, fused=True)


def block_ref(cfg, li: int, bi: int, B: int, x, bw: dict, stream: str = "fp32", round16: bool = False):
    """one whole block from the stream rows x [B T, C] by the unit references, all windows; round16=False is the
    float64 model (PanguRef.block)"""
    g = level(cfg, li)
    roll, wins = bi & 1, np.arange(B * g.nWin)
    qkv, _ = qkv_unit(g, B, roll, wins, x, bw, round16=round16)
    if round16:
        qkv = qkv.astype(np.float16)
    tok, att, _ = attention_unit(g, B, roll, wins, qkv, bw, cfg.mask_value, round16=round16)
    a = np.empty_like(att)
    a[tok] = att
    if round16:
        a = a.astype(np.float16)
    x1, _ = proj_unit(a, bw, x, cfg.ln_eps, stream, round16=round16)
    h, _ = fc1_unit(x1.astype(np.float16) if round16 else x1, bw, round16)
    return fc2_unit(h.astype(np.float16) if round16 else h, bw, x1, cfg.ln_eps, stream, round16=round16)[0]


# ---------------------------------------------------------------------------------------------------------------------
# chained: the fp64 oracle's stream after every block
# ---------------------------------------------------------------------------------------------------------------------
def block_outputs(ref, state) -> dict:
    """{(layer, block): token rows [T, C]} of PanguRef ``ref`` stepping one state"""
    import torch
    out = {}
    with torch.no_grad():
        x = ref.patch_embed(torch.as_tensor(state).to(ref.dtype))
        for li in range(4):
            if li == 1:
                x = ref.downsample(x)
            if li == 3:
                x = ref.upsample(x)
            for bi, x in enumerate(ref.blocks(x, li)):
                out[(li, bi)] = x.reshape(-1, x.shape[-1]).numpy()
    return out


def chain_bounds(cfg, w, states):
    """(fp64 oracle stream after every block for the members ``states``, {(layer, block): row bound}): CHAIN_FACTOR x
    the largest per-row relative error of PanguRef(emulate="fp16s") against the fp64 oracle at that block, at least
    CHAIN_FLOOR (graphcast_stages_ref's rule)"""
    import torch
    from oracle.pangu_ref import PanguRef
    exact, emu = PanguRef(cfg, w, dtype=torch.float64), PanguRef(cfg, w, dtype=torch.float64, emulate="fp16s")
    per = [(block_outputs(exact, s), block_outputs(emu, s)) for s in states]
    ref = {k: np.concatenate([r[k] for r, _ in per]) for k in per[0][0]}
    tol = {k: max(CHAIN_FLOOR, CHAIN_FACTOR * float(row_rel(np.concatenate([e[k] for _, e in per]), ref[k]).max())) for k in ref}
    return ref, tol
