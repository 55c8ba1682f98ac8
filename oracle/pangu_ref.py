"""ORACLE — test infrastructure, not product code.

CPU fp32 (or fp64) restatement of the Pangu-Weather 6-hour forward that the reference
reaches through ``pangu.load(registry.get_model("e2mip://pangu"))``
(/root/reference/skyrim/core/models/pangu.py:45-46) and steps through
``for k, (time, output, _) in enumerate(model(time, x))``
(/root/reference/skyrim/core/models/utils.py:34-40).

PARITY UNPINNED: the arithmetic lives in third-party code that is not vendored under
/root/reference and cannot be imported here (earth2mip @ unpinned git HEAD,
requirements.txt:2; onnxruntime + pangu_weather_6.onnx, unpinned; SURVEY.md §8(c)), and
the reference's tests hold no golden vector for this path (tests/core/test_graphcast.py:11-22
check dims and names only).  This file therefore restates the *published* architecture
(Bi et al. 2023, authors' pseudocode; SURVEY.md Appendix A) with the free choices fixed as
documented in DESIGN.md, and is the parity authority for the CUDA engine on seeded
synthetic weights (skyrim_b200/weights.py).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
may import this module.

Layout: state (69, nlat, nlon) in the reference channel order
(/root/reference/skyrim/core/models/pangu.py:6-13): 5 upper-air variables x 13 levels
(1000..50 hPa), then msl, u10m, v10m, t2m.  Token grid (Z, H, W, C) with the surface
slab at Z index 0.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from skyrim_b200.config import PanguConfig


def position_index(window) -> torch.Tensor:
    """Index into the earth-specific bias table for every (query, key) token pair of a
    window; absolute in (z, h), relative in w (Appendix A item 2)."""
    wz, wh, ww = window
    zi, hi, wi = torch.meshgrid(torch.arange(wz), torch.arange(wh), torch.arange(ww), indexing="ij")
    zi, hi, wi = zi.reshape(-1), hi.reshape(-1), wi.reshape(-1)
    idx = ((zi[:, None] + wz * zi[None, :]) * ((2 * ww - 1) * wh * wh)
           + (hi[:, None] + wh * hi[None, :]) * (2 * ww - 1)
           + (wi[:, None] - wi[None, :] + ww - 1))
    return idx  # (N, N), rows = query token, cols = key token


def shift_mask(cfg: PanguConfig, Z: int, Hp: int, W: int, dtype) -> torch.Tensor:
    """Swin-style additive mask for the rolled grid: tokens of one window that come from
    different sides of the Z / latitude seam do not attend to each other.  Longitude is
    periodic, so no mask along W.  Returns (nWz*nWh, N, N) indexed by window type."""
    wz, wh, ww = cfg.window
    sz, sh = wz // 2, wh // 2
    img = torch.zeros(Z, Hp, W)
    cnt = 0
    for zs in (slice(0, -wz), slice(-wz, -sz), slice(-sz, None)):
        for hs in (slice(0, -wh), slice(-wh, -sh), slice(-sh, None)):
            img[zs, hs, :] = cnt
            cnt += 1
    win = img.reshape(Z // wz, wz, Hp // wh, wh, W // ww, ww).permute(0, 2, 4, 1, 3, 5)
    win = win.reshape(Z // wz, Hp // wh, W // ww, wz * wh * ww)[:, :, 0]  # identical for every w-window
    diff = win[:, :, :, None] - win[:, :, None, :]
    m = torch.zeros_like(diff).masked_fill(diff != 0, cfg.mask_value)
    return m.reshape(-1, wz * wh * ww, wz * wh * ww).to(dtype)


class PanguRef:
    """Functional forward over a dict of numpy weights (skyrim_b200.weights.make_pangu_weights).

    ``emulate`` reproduces the engine's storage/operand precision so that the error budget
    can be studied on CPU: "fp16" rounds GEMM operands (activations and weights) to half,
    accumulates in fp32 — what the engine's tensor-core GEMMs do.
    """

    def __init__(self, cfg: PanguConfig, weights, dtype=torch.float32, emulate: str | None = None):
        self.cfg = cfg
        self.dtype = dtype
        self.emulate = emulate
        self.w = {k: torch.from_numpy(np.asarray(v)).to(dtype) for k, v in weights.items()}
        self.pos_idx = position_index(cfg.window)
        self._masks = {}

    # -- operand rounding hooks -----------------------------------------------------------
    def _q(self, t):
        if self.emulate in ("fp16", "fp16s"):
            return t.to(torch.float16).to(self.dtype)
        if self.emulate == "bf16":
            return t.to(torch.bfloat16).to(self.dtype)
        return t

    def _linear(self, x, w, b=None):
        y = self._q(x) @ self._q(w).t()
        return y if b is None else y + b

    # -- pieces ---------------------------------------------------------------------------
    def patch_embed(self, state):
        cfg, w = self.cfg, self.w
        pz, ph, pw = cfg.patch
        nu, nl = cfg.n_upper_vars, cfg.n_levels
        x = (state - w["norm.mean"][:, None, None]) / w["norm.std"][:, None, None]
        upper = x[: nu * nl].reshape(nu, nl, cfg.nlat, cfg.nlon)
        surf = torch.cat([x[nu * nl:], w["const.masks"]], 0)
        Zp, Hp = (cfg.Z - 1) * pz, cfg.H * ph
        upper = F.pad(upper, (0, 0, 0, Hp - cfg.nlat, 0, Zp - nl))       # zero-pad at the high-index end
        surf = F.pad(surf, (0, 0, 0, Hp - cfg.nlat))
        # non-overlapping conv == matmul over flattened patches
        up = upper.reshape(nu, cfg.Z - 1, pz, cfg.H, ph, cfg.W, pw).permute(1, 3, 5, 0, 2, 4, 6)
        up = up.reshape(cfg.Z - 1, cfg.H, cfg.W, nu * pz * ph * pw)
        tu = self._linear(up, w["embed.upper.w"].reshape(cfg.dim, -1), w["embed.upper.b"])
        sf = surf.reshape(surf.shape[0], cfg.H, ph, cfg.W, pw).permute(1, 3, 0, 2, 4).reshape(cfg.H, cfg.W, -1)
        ts = self._linear(sf, w["embed.surf.w"].reshape(cfg.dim, -1), w["embed.surf.b"])
        return torch.cat([ts[None], tu], 0)  # (Z, H, W, C), surface slab at z = 0

    def _mask(self, Z, Hp, W):
        key = (Z, Hp, W)
        if key not in self._masks:
            self._masks[key] = shift_mask(self.cfg, Z, Hp, W, self.dtype)
        return self._masks[key]

    def attention(self, xw, p, heads, n_types, mask):
        """xw: (nWz*nWh (type), nWw, N, C) windows.  Returns same shape."""
        w = self.w
        T, Ww, N, C = xw.shape
        d = C // heads
        qkv = self._linear(xw, w[p + "qkv.w"], w[p + "qkv.b"])
        qkv = self._q(qkv)  # engine stores q, k, v as half
        qkv = qkv.reshape(T, Ww, N, 3, heads, d).permute(3, 0, 1, 4, 2, 5)
        q, k, v = qkv[0], qkv[1], qkv[2]                     # (T, Ww, heads, N, d)
        att = (q @ k.transpose(-1, -2)) * (d ** -0.5)
        bias = w[p + "bias_table"][self.pos_idx.reshape(-1)]  # (N*N, n_types, heads)
        bias = bias.reshape(N, N, n_types, heads).permute(2, 3, 0, 1)
        att = att + bias[:, None]
        if mask is not None:
            att = att + mask[:, None, None]
        att = torch.softmax(att, dim=-1)
        o = self._q(att) @ v                                  # P is rounded to half for the AV product
        o = o.permute(0, 1, 3, 2, 4).reshape(T, Ww, N, C)
        return self._linear(self._q(o), w[p + "proj.w"], w[p + "proj.b"])

    def block(self, x, p, heads, roll):
        """x: (Z, H, W, C) -> same."""
        cfg, w = self.cfg, self.w
        wz, wh, ww = cfg.window
        Z, H, W, C = x.shape
        Hp = cfg.padded_h(H)
        y = F.pad(x, (0, 0, 0, 0, 0, Hp - H))
        mask = None
        if roll:
            y = torch.roll(y, shifts=(-(wz // 2), -(wh // 2), -(ww // 2)), dims=(0, 1, 2))
            mask = self._mask(Z, Hp, W)
        yw = y.reshape(Z // wz, wz, Hp // wh, wh, W // ww, ww, C).permute(0, 2, 4, 1, 3, 5, 6)
        yw = yw.reshape((Z // wz) * (Hp // wh), W // ww, wz * wh * ww, C)
        yw = self.attention(yw, p, heads, (Z // wz) * (Hp // wh), mask)
        y = yw.reshape(Z // wz, Hp // wh, W // ww, wz, wh, ww, C).permute(0, 3, 1, 4, 2, 5, 6).reshape(Z, Hp, W, C)
        if roll:
            y = torch.roll(y, shifts=(wz // 2, wh // 2, ww // 2), dims=(0, 1, 2))
        y = y[:, :H]
        # emulate="fp16s": like "fp16", and the residual stream itself is kept in half between the sub-layers (the engine
        # stores the token stream only as its fp16 operand image: sum in fp32, one rounding per residual add)
        qs = (lambda t: t.to(torch.float16).to(self.dtype)) if self.emulate == "fp16s" else (lambda t: t)
        x = qs(x + F.layer_norm(y, (C,), w[p + "ln1.g"], w[p + "ln1.b"], cfg.ln_eps))
        hdn = F.gelu(self._linear(x, w[p + "fc1.w"], w[p + "fc1.b"]))
        y = self._linear(self._q(hdn), w[p + "fc2.w"], w[p + "fc2.b"])
        x = qs(x + F.layer_norm(y, (C,), w[p + "ln2.g"], w[p + "ln2.b"], cfg.ln_eps))
        return x

    def blocks(self, x, li):
        """the token tensor after each block of layer li, in order"""
        for bi in range(self.cfg.depths[li]):
            x = self.block(x, f"layer{li}.block{bi}.", self.cfg.heads[li], roll=(bi % 2 == 1))
            yield x

    def layer(self, x, li):
        for x in self.blocks(x, li):
            pass
        return x

    def downsample(self, x):
        cfg, w = self.cfg, self.w
        Z, H, W, C = x.shape
        x = F.pad(x, (0, 0, 0, 0, 0, 2 * cfg.H2 - H))
        x = x.reshape(Z, cfg.H2, 2, cfg.W2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(Z, cfg.H2, cfg.W2, 4 * C)
        x = F.layer_norm(x, (4 * C,), w["down.ln.g"], w["down.ln.b"], cfg.ln_eps)
        return self._linear(x, w["down.w"])

    def upsample(self, x):
        cfg, w = self.cfg, self.w
        Z, H2, W2, C2 = x.shape
        C = C2 // 2
        x = self._linear(x, w["up.w1"])                      # (Z, H2, W2, 4C) as (2, 2, C)
        x = x.reshape(Z, H2, W2, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(Z, 2 * H2, 2 * W2, C)
        x = x[:, : cfg.H]
        x = F.layer_norm(x, (C,), w["up.ln.g"], w["up.ln.b"], cfg.ln_eps)
        return self._linear(x, w["up.w2"])

    def patch_recover(self, x):
        cfg, w = self.cfg, self.w
        pz, ph, pw = cfg.patch
        nu, ns, nl = cfg.n_upper_vars, cfg.n_surface_vars, cfg.n_levels
        Z, H, W, C2 = x.shape
        wu = w["recover.upper.w"].reshape(C2, -1)              # (C2, nu*pz*ph*pw)
        yu = self._q(x[1:]) @ self._q(wu)                      # (Z-1, H, W, nu*pz*ph*pw)
        yu = yu.reshape(Z - 1, H, W, nu, pz, ph, pw).permute(3, 0, 4, 1, 5, 2, 6)
        yu = yu.reshape(nu, (Z - 1) * pz, H * ph, W * pw)[:, :nl, : cfg.nlat] + w["recover.upper.b"][:, None, None, None]
        ws = w["recover.surf.w"].reshape(C2, -1)
        ys = self._q(x[0]) @ self._q(ws)
        ys = ys.reshape(H, W, ns, ph, pw).permute(2, 0, 3, 1, 4).reshape(ns, H * ph, W * pw)[:, : cfg.nlat]
        ys = ys + w["recover.surf.b"][:, None, None]
        out = torch.cat([yu.reshape(nu * nl, cfg.nlat, cfg.nlon), ys], 0)
        return out * w["norm.std"][:, None, None] + w["norm.mean"][:, None, None]

    # -- the operator ---------------------------------------------------------------------
    @torch.no_grad()
    def step(self, state) -> torch.Tensor:
        """One 6-h step: (69, nlat, nlon) -> (69, nlat, nlon), de-normalised state."""
        state = torch.as_tensor(state).to(self.dtype)
        x = self.patch_embed(state)
        x = self.layer(x, 0)
        skip = x
        x = self.downsample(x)
        x = self.layer(x, 1)
        x = self.layer(x, 2)
        x = self.upsample(x)
        x = self.layer(x, 3)
        x = torch.cat([skip, x], -1)
        return self.patch_recover(x)

    @torch.no_grad()
    def stages(self, state):
        """Intermediate tensors for kernel-level parity tests."""
        out = {}
        state = torch.as_tensor(state).to(self.dtype)
        x = self.patch_embed(state); out["embed"] = x
        x = self.layer(x, 0); out["layer0"] = x
        skip = x
        x = self.downsample(x); out["down"] = x
        x = self.layer(x, 1); out["layer1"] = x
        x = self.layer(x, 2); out["layer2"] = x
        x = self.upsample(x); out["up"] = x
        x = self.layer(x, 3); out["layer3"] = x
        out["out"] = self.patch_recover(torch.cat([skip, x], -1))
        return out


def rel_err_per_channel(y, ref) -> np.ndarray:
    """max-over-nothing: per-channel ||y - ref||_2 / ||ref||_2 (the north-star metric)."""
    y = np.asarray(y, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    num = np.sqrt(((y - ref) ** 2).sum(axis=(-1, -2)))
    den = np.sqrt((ref ** 2).sum(axis=(-1, -2)))
    return num / den


def normalised_err_per_channel(y, ref, std) -> np.ndarray:
    """RMS error in units of the channel's climatological std (stricter than rel_err for
    channels whose mean dominates their norm)."""
    y = np.asarray(y, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    return np.sqrt(((y - ref) ** 2).mean(axis=(-1, -2))) / np.asarray(std, dtype=np.float64)
