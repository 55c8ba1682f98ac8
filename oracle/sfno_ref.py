"""ORACLE — test infrastructure, not product code.

CPU fp32 / fp64 restatement of the FourCastNet-v2-small SFNO 6-hour forward that the
reference reaches through ``fcnv2_sm.load(registry.get_model("e2mip://fcnv2_sm"))``
(/root/reference/skyrim/core/models/fourcastnet_v2.py:36-37) and steps through
earth2mip's ``Inference`` wrapper (normalise, yield IC, x = model(x), de-normalise;
/root/reference/skyrim/core/models/utils.py:34-40).

PARITY UNPINNED: earth2mip (unpinned git HEAD, requirements.txt:2), modulus / makani's
sfnonet and torch-harmonics are not vendored under /root/reference and cannot be imported
here; the reference's tests hold no golden vector for this path.  The network below follows
SURVEY.md Appendix B with the hyper-parameters marked "default synthetic config" there
(E=384, L=8, scale_factor=3) and the free choices fixed in DESIGN.md (inner skip = 1x1 conv,
outer skip = identity, instance norm with affine, no spectral bias).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this module.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from skyrim_b200.config import SFNOConfig
from oracle import sht_ref


class SFNORef:
    def __init__(self, cfg: SFNOConfig, weights, dtype=torch.float32, emulate: str | None = None):
        self.cfg, self.dtype, self.emulate = cfg, dtype, emulate
        self.w = {k: torch.from_numpy(np.asarray(v)).to(dtype) for k, v in weights.items()}
        cd = torch.complex128 if dtype == torch.float64 else torch.complex64
        # Legendre / quadrature tables from the oracle's OWN builder (scipy), not the product's skyrim_b200/sht.py
        self.tabs = {}
        for tag, (nlat, nlon, grid) in (("big", (cfg.nlat, cfg.nlon, "equiangular")), ("int", (cfg.h, cfg.w, "legendre-gauss"))):
            fwd, inv, _, _ = sht_ref.tables(nlat, cfg.lmax, cfg.mmax, grid)
            self.tabs[tag] = dict(fwd=torch.from_numpy(fwd).to(dtype), inv=torch.from_numpy(inv).to(dtype), nlon=nlon, nlat=nlat)
        self.cd = cd

    def _q(self, t, tag="all"):
        """operand rounding emulation: emulate = "fp16" rounds every GEMM operand to half; a set / tuple of tags
        ("mlp", "dft", "leg", "spec") rounds only those contractions (precision-budget studies, tests/test_sfno_cpu.py)"""
        if self.emulate == "fp16" or (isinstance(self.emulate, (set, frozenset, tuple, list)) and tag in self.emulate):
            if t.is_complex():
                return torch.complex(t.real.half().to(self.dtype), t.imag.half().to(self.dtype))
            return t.half().to(self.dtype)
        return t

    # -- transforms (channel-major (C, nlat, nlon) <-> complex (C, lmax, mmax)) -----------------
    def sht(self, x, tag):
        t = self.tabs[tag]
        f = 2.0 * np.pi * torch.fft.rfft(self._q(x, "dft"), dim=-1, norm="forward")[..., : self.cfg.mmax]
        f = self._q(f, "leg")
        return torch.einsum("mlk,ckm->clm", self._q(t["fwd"], "leg").to(self.cd), f)

    def isht(self, X, tag):
        t = self.tabs[tag]
        f = torch.einsum("mkl,clm->ckm", self._q(t["inv"], "leg").to(self.cd), self._q(X, "leg"))
        return torch.fft.irfft(self._q(f, "dft"), n=t["nlon"], dim=-1, norm="forward")

    def _conv1x1(self, x, w, b=None):  # x (C, H, W)
        y = torch.einsum("oc,chw->ohw", self._q(w, "mlp"), self._q(x, "mlp"))
        return y if b is None else y + b[:, None, None]

    def _inorm(self, x, g, b):
        return F.instance_norm(x[None], weight=g, bias=b, eps=self.cfg.eps)[0]

    def _inorm_affine(self, x, g, b):
        """(scale, shift) of the instance norm with affine: norm(x) = scale * x + shift per channel (biased variance)"""
        mean = x.mean(dim=(1, 2))
        var = ((x - mean[:, None, None]) ** 2).mean(dim=(1, 2))
        sc = g / torch.sqrt(var + self.cfg.eps)
        return sc, b - mean * sc

    def block(self, x, i, taps=None):
        cfg, w = self.cfg, self.w
        p = f"blk{i}."
        tin = "big" if i == 0 else "int"
        tout = "big" if i == cfg.layers - 1 else "int"
        xn = self._inorm(x, w[p + "norm0.g"], w[p + "norm0.b"])
        X = self.sht(xn, tin)
        residual = xn if tin == tout else self.isht(X, tout)
        wc = torch.complex(w[p + "spec.w"][..., 0], w[p + "spec.w"][..., 1])  # (l, out, in)
        Xo = torch.einsum("loi,ilm->olm", self._q(wc, "spec"), self._q(X, "spec"))
        y = self.isht(Xo, tout)
        y = y + self._conv1x1(residual, w[p + "inner.w"], w[p + "inner.b"])
        y = F.gelu(y)
        g = y
        y = self._inorm(y, w[p + "norm1.g"], w[p + "norm1.b"])
        hdn = F.gelu(self._conv1x1(y, w[p + "fc1.w"], w[p + "fc1.b"]))
        y = self._conv1x1(hdn, w[p + "fc2.w"], w[p + "fc2.b"])
        out = y + residual
        if taps is not None:
            self._block_taps(taps, f"b{i}.", x, X, Xo, g, hdn, out, i, tin, tout)
        return out

    def _block_taps(self, taps, k, x, X, Xo, g, hdn, out, i, tin, tout):
        """the block's intermediates in the engine's layouts (skyrim_b200/csrc/sfno_engine.cu header): pixel-major fields
        [pixel][channel], spectra [l][m][(ri, c)] / [m][l][(ro, o)], DFT rows [m][lat][(ri, c)], [lat][(m, ro)][o]"""
        w, p = self.w, f"blk{i}."
        ri = lambda z, dim: torch.cat([z.real, z.imag], dim=dim)
        pm = lambda f: f.reshape(f.shape[0], -1).T.contiguous()
        sc, sh = self._inorm_affine(x, w[p + "norm0.g"], w[p + "norm0.b"])
        taps[k + "norm0"] = torch.cat([sc, sh])
        xn = x * sc[:, None, None] + sh[:, None, None]
        f = 2.0 * np.pi * torch.fft.rfft(xn, dim=-1, norm="forward")[..., : self.cfg.mmax]      # (c, lat, m)
        taps[k + "li"] = ri(f.permute(2, 1, 0), 2)                                               # [m][lat][(ri, c)]
        taps[k + "si"] = ri(X.permute(1, 2, 0), 2)                                               # [l][m][(ri, c)]
        if tin == tout:
            taps[k + "mi"] = ri(Xo.permute(2, 1, 0), 2)                                          # [m][l][(ro, o)]
            taps[k + "inner_bias"] = w[p + "inner.b"] + w[p + "inner.w"] @ sh
            taps[k + "f1"] = pm(self.isht(Xo, tout))
        else:   # the engine folds the inner skip into the mixing matrices: its mixing output is (W_l + V) X
            taps[k + "mi"] = ri((Xo + torch.einsum("oi,ilm->olm", w[p + "inner.w"].to(X.dtype), X)).permute(2, 1, 0), 2)
            taps[k + "mi2"] = ri(X.permute(2, 1, 0), 2)
            taps[k + "rpm"] = pm(self.isht(X, tout))
            Xo = Xo + torch.einsum("oi,ilm->olm", w[p + "inner.w"].to(X.dtype), X)
        t = self.tabs[tout]
        d = torch.einsum("mkl,clm->ckm", t["inv"].to(self.cd), Xo)                               # (o, lat, m)
        taps[k + "di"] = ri(d.permute(1, 2, 0)[:, :, None, :], 2).reshape(d.shape[1], -1, d.shape[0])  # [lat][(m, ro)][o]
        taps[k + "g"] = pm(g)
        taps[k + "sums"] = torch.cat([pm(g).sum(0), (pm(g) ** 2).sum(0)])
        n1sc, n1sh = self._inorm_affine(g, w[p + "norm1.g"], w[p + "norm1.b"])
        taps[k + "norm1"] = torch.cat([n1sc, n1sh])
        taps[k + "fc1_bias"] = w[p + "fc1.b"] + w[p + "fc1.w"] @ n1sh
        taps[k + "hidden"] = pm(hdn)
        taps[k + "x"] = pm(out)
        d = pm(out) - w[p + "fc2.b"]    # the engine gathers the statistics about the bias of the epilogue that writes x
        taps[k + "sums0"] = torch.cat([d.sum(0), (d ** 2).sum(0)])

    @torch.no_grad()
    def step(self, state, taps=None):
        """(73, nlat, nlon) de-normalised -> (73, nlat, nlon) de-normalised.  ``taps``: a dict that receives every
        intermediate the engine exposes through debug_copy, in its layouts (``_block_taps``): "in" (normalised input),
        "enc.hidden", "enc.x", "enc.sums0", "b{i}.*" per block, "dec.hidden"."""
        w = self.w
        x = torch.as_tensor(state).to(self.dtype)
        xh = (x - w["norm.mean"][:, None, None]) / w["norm.std"][:, None, None]
        y = F.gelu(self._conv1x1(xh, w["enc.fc1.w"], w["enc.fc1.b"]))
        if taps is not None:
            pm = lambda f: f.reshape(f.shape[0], -1).T.contiguous()
            taps["in"], taps["enc.hidden"] = pm(xh), pm(y)
        y = self._conv1x1(y, w["enc.fc2.w"], w["enc.fc2.b"]) + w["pos_embed"]
        if taps is not None:
            taps["enc.x"] = pm(y)
            d = pm(y) - w["enc.fc2.b"]
            taps["enc.sums0"] = torch.cat([d.sum(0), (d ** 2).sum(0)])
        for i in range(self.cfg.layers):
            y = self.block(y, i, taps)
        y = torch.cat([y, xh], 0)
        y = F.gelu(self._conv1x1(y, w["dec.fc1.w"], w["dec.fc1.b"]))
        if taps is not None:
            taps["dec.hidden"] = pm(y)
        y = self._conv1x1(y, w["dec.fc2.w"], w["dec.fc2.b"])
        return y * w["norm.std"][:, None, None] + w["norm.mean"][:, None, None]
