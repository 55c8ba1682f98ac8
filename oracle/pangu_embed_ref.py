"""ORACLE — test infrastructure, not product code.

Float64 reference of Pangu's patch embedding as the engine computes it (the producers ProdEmbedUpper / ProdEmbedSurf and
the epilogue EpiStoreF32 in skyrim_b200/csrc/pangu_ops.cuh), for tests/test_pangu_embed_gpu.py.

The A operand is built bit for bit as the producer warps build it: fp32 (x - mean) * (1 / std), with 1 / std rounded to
fp32, then rounded to fp16.  The constant masks are three more surface channels, taken as they are.  Latitude padding, the
missing 14th level and the K padding of the packed weights (160 -> 192, 112 -> 128) are zeros.  W is the fp16 weight.  The
linear part is exact in float64; its bound is gemm_ref's tau * sum |a w|, and the bias add and the stores add their own
roundings.  Rows are the engine's tokens (member, z, h, w): surface at z = 0, upper-air level pair zt at z = 1 + zt.
"""
from __future__ import annotations

import numpy as np

from oracle import gemm_ref as gr
from oracle import pangu_resample_ref as pr


def a_operands(cfg, w, x: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """x: (B, n_channels, nlat, nlon) fp32 -> the A operands of the upper-air GEMM (B * (Z - 1) * H * W rows, k =
    ((v * 2 + dz) * 4 + dh) * 4 + dw) and of the surface GEMM (B * H * W rows, k = (c * 4 + dh) * 4 + dw), as fp16"""
    x = np.asarray(x, np.float32)
    B = x.shape[0]
    nu, nl, ns = cfg.n_upper_vars, cfg.n_levels, cfg.n_surface_vars
    pz, ph, pw = cfg.patch
    H, W, nzt = cfg.H, cfg.W, cfg.Z - 1
    mean = np.asarray(w["norm.mean"], np.float32)[:, None, None]
    rs = (np.float32(1.0) / np.asarray(w["norm.std"], np.float32))[:, None, None]
    xn = ((x - mean) * rs).astype(np.float16)
    masks = np.broadcast_to(np.asarray(w["const.masks"], np.float32).astype(np.float16), (B, cfg.n_const_masks) + x.shape[2:])
    lat_pad = ((0, 0), (0, 0), (0, H * ph - cfg.nlat), (0, 0))
    up = np.pad(xn[:, : nu * nl].reshape(B, nu, nl, cfg.nlat, cfg.nlon), ((0, 0), (0, 0), (0, nzt * pz - nl)) + lat_pad[2:])
    up = up.reshape(B, nu, nzt, pz, H, ph, W, pw).transpose(0, 2, 4, 6, 1, 3, 5, 7).reshape(B * nzt * H * W, nu * pz * ph * pw)
    sf = np.pad(np.concatenate([xn[:, nu * nl: nu * nl + ns], masks], axis=1), lat_pad)
    sf = sf.reshape(B, ns + cfg.n_const_masks, H, ph, W, pw).transpose(0, 2, 4, 1, 3, 5).reshape(B * H * W, -1)
    return up, sf


def embed_reference(cfg, w, x: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """(B * T, C) float64 tokens after the embedding and the per-element bound of the fp32 result (gr.f16_bound of it
    for the fp16 image)"""
    B, C = x.shape[0], cfg.dim
    up, sf = a_operands(cfg, w, x)
    out = []
    for a, name in ((up, "embed.upper"), (sf, "embed.surf")):
        wt = np.asarray(w[name + ".w"], np.float32).reshape(C, -1).astype(np.float16)
        R, S = gr.linear([(a, wt)])
        out.append(gr.epi_affine(R, S, np.asarray(w[name + ".b"], np.float32)[None, :]))
    HW = cfg.H * cfg.W
    (ru, bu), (rsf, bsf) = out
    ref = np.concatenate([rsf.reshape(B, HW, C), ru.reshape(B, -1, C)], axis=1).reshape(-1, C)
    bound = np.concatenate([bsf.reshape(B, HW, C), bu.reshape(B, -1, C)], axis=1).reshape(-1, C)
    return ref, bound


def skip_image_offset(cfg, B: int) -> int:
    """byte offset of the skip image in the engine's workspace for B members (pr.workspace_layout, the mirror of
    PanguEngine::carve)"""
    return pr.workspace_layout(cfg, B)["skiph"]
