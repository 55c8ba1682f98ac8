"""ORACLE — test infrastructure, not product code.

CPU fp32 / fp64 restatement of one GraphCast 6-hour step: what the reference reaches through
``self.stepper.step(state)`` (/root/reference/skyrim/core/models/graphcast.py:118) after
``graphcast.load_time_loop_operational(registry.get_model("e2mip://graphcast"))`` (:51-54).

PARITY UNPINNED: earth2mip's graphcast wrapper, deepmind's ``graphcast`` package (JAX / Haiku, requirements.txt:2-4) and
its checkpoint are not vendored under /root/reference and cannot be imported here; the reference's own test checks
dimension names and the channel-name set only (tests/core/test_graphcast.py:11-22).  The network below follows the
PUBLISHED architecture (Lam et al. 2023, "Learning skillful medium-range global weather forecasting", and SURVEY.md §8(a)
A9): encoder = embed grid nodes / mesh nodes / grid2mesh edges with one-hidden-layer swish MLPs + LayerNorm, one
interaction-network step on the bipartite grid2mesh graph; processor = 16 unshared interaction-network steps on the
multimesh (edge update from [edge, sender, receiver], node update from [node, SUM of incoming updated edges], residuals);
decoder = one interaction-network step on mesh2grid and an output MLP without LayerNorm; the prediction is a residual in
units of per-channel difference standard deviations.  It is written the NAIVE way (gather, concatenate, MLP, index_add):
the engine's algebraic rewrites (first-layer weights split per input, per-node partial products gathered in the GEMM
epilogue, mesh2grid aggregation as a K-concatenation, input-independent embeddings computed once) are checked against it.

Free choices fixed for the synthetic-weight definition (documented in DESIGN.md, unverifiable offline): feature order
(`features()`), the closed-form toa radiation (`toa_radiation`), mesh nodes embedded from their three structural features
only (the published model concatenates an all-zero data block, which multiplies weights by zero), the mesh-node update of
the mesh2grid step skipped (its result is never read), the operational model's total-precipitation head dropped (the
reference's CHANNEL_MAP :29-41 has no entry for it).

Only tests/, tools/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may import this module.
"""
from __future__ import annotations

import numpy as np
import torch

from skyrim_b200.config import GraphCastConfig

SECONDS_PER_DAY = 86400.0
DAYS_PER_YEAR = 365.24219
SOLAR_CONSTANT = 1361.0


def year_progress(t_seconds: float) -> float:
    return (t_seconds / SECONDS_PER_DAY / DAYS_PER_YEAR) % 1.0


def day_progress(t_seconds: float, lon_deg: np.ndarray) -> np.ndarray:
    return ((t_seconds / SECONDS_PER_DAY) % 1.0 + lon_deg / 360.0) % 1.0


def toa_radiation(t_seconds: float, lat_deg: np.ndarray, lon_deg: np.ndarray) -> np.ndarray:
    """Top-of-atmosphere incident solar radiation accumulated over one hour [J m^-2], closed form (fp64):
    S0 (1 + 0.033 cos g) max(0, sin lat sin d + cos lat cos d cos h) x 3600, g = 2 pi year_progress,
    d = 0.4093 sin(g - 1.405), h = 2 pi day_progress(lon) - pi."""
    g = 2.0 * np.pi * year_progress(t_seconds)
    d = 0.4093 * np.sin(g - 1.405)
    h = 2.0 * np.pi * day_progress(t_seconds, lon_deg)[None, :] - np.pi
    lat = np.deg2rad(lat_deg)[:, None]
    cosz = np.sin(lat) * np.sin(d) + np.cos(lat) * np.cos(d) * np.cos(h)
    return SOLAR_CONSTANT * (1.0 + 0.033 * np.cos(g)) * np.maximum(cosz, 0.0) * 3600.0


class GraphCastRef:
    CHUNK = 1 << 17   # rows per chunk of the edge / node MLPs (bounds the concatenated inputs in host memory)

    def __init__(self, cfg: GraphCastConfig, weights, graph, dtype=torch.float32, emulate: str | None = None):
        self.cfg, self.dtype, self.emulate = cfg, dtype, emulate
        self.w = {k: torch.from_numpy(np.asarray(v)).to(dtype) for k, v in weights.items() if not k.startswith("graph.")}
        self.g = graph
        self.lat = np.linspace(90.0, -90.0, cfg.nlat)
        self.lon = np.arange(cfg.nlon) * (360.0 / cfg.nlon)
        li = lambda a: torch.from_numpy(np.asarray(a, dtype=np.int64))
        self.idx = {k: li(graph[k]) for k in ("mesh.senders", "mesh.receivers", "g2m.senders", "g2m.receivers",
                                              "m2g.senders", "m2g.receivers")}
        self._static = None

    # -- building blocks -----------------------------------------------------------------------
    def _q(self, t):
        return t.half().to(self.dtype) if self.emulate else t

    def mlp(self, name: str, parts, ln: bool = True, table_parts=()):
        """Linear -> swish -> Linear (-> LayerNorm) on the concatenation of ``parts`` along the feature axis, row chunked.
        emulate="fp16" rounds every GEMM operand to half; emulate="fp16t" additionally rounds the first-layer partial
        products of the parts listed in ``table_parts`` (the engine stores those per-node tables in fp16); emulate="fp16s"
        additionally keeps the grid-node and mesh-edge residual streams in half between layers (``tendency``), as the engine
        does (they exist only as fp16 operand images there)."""
        w1, b1, w2, b2 = (self.w[f"{name}.{k}"] for k in ("w1", "b1", "w2", "b2"))
        n = parts[0].shape[0]
        out = torch.empty(n, w2.shape[0], dtype=self.dtype)
        w1q, w2q = self._q(w1), self._q(w2)
        for r0 in range(0, n, self.CHUNK):
            sl = slice(r0, min(n, r0 + self.CHUNK))
            if self.emulate in ("fp16t", "fp16s") and table_parts:
                h, c0 = b1.clone().expand(sl.stop - sl.start, -1).clone(), 0
                for i, p in enumerate(parts):
                    pp = self._q(p[sl]) @ w1q[:, c0:c0 + p.shape[1]].T
                    h += self._q(pp) if i in table_parts else pp
                    c0 += p.shape[1]
            else:
                h = self._q(torch.cat([p[sl] for p in parts], dim=1)) @ w1q.T + b1
            h = h * torch.sigmoid(h)
            y = self._q(h) @ w2q.T + b2
            if ln:
                y = torch.nn.functional.layer_norm(y, (y.shape[1],), self.w[f"{name}.ln.g"], self.w[f"{name}.ln.b"], self.cfg.ln_eps)
            out[sl] = y
        return out

    def static_embeddings(self):
        """input-independent embeddings: mesh nodes and the three edge sets"""
        if self._static is None:
            f = lambda k: torch.from_numpy(np.asarray(self.g[k])).to(self.dtype)
            self._static = dict(
                vm=self.mlp("enc.mesh_embed", [f("mesh.node_feat")]),
                e_g2m=self.mlp("enc.g2m_edge_embed", [f("g2m.edge_feat")]),
                e_mesh=self.mlp("proc.edge_embed", [f("mesh.edge_feat")]),
                e_m2g=self.mlp("dec.m2g_edge_embed", [f("m2g.edge_feat")]))
        return self._static

    def features(self, x: torch.Tensor, t_seconds: float) -> torch.Tensor:
        """x: (2*n_state, nlat, nlon) at times (t-6h, t) -> (n_grid, n_features)"""
        cfg = self.cfg
        ns, npg = cfg.n_state, cfg.n_prog
        mean, std = self.w["norm.mean"], self.w["norm.std"]
        dt = 3600.0 * cfg.dt_hours
        xs = x.reshape(2, ns, cfg.nlat, cfg.nlon).to(self.dtype)
        xn = (xs - mean[None, :, None, None]) / std[None, :, None, None]
        toa_next = torch.from_numpy(toa_radiation(t_seconds + dt, self.lat, self.lon)).to(self.dtype)
        toa_next = (toa_next - mean[ns - 1]) / std[ns - 1]
        planes = [xn[0, :npg], xn[1, :npg], xn[0, ns - 1:ns], xn[1, ns - 1:ns], toa_next[None]]
        ones = torch.ones(cfg.nlat, cfg.nlon, dtype=self.dtype)
        for k in (-1, 0, 1):
            tk = t_seconds + k * dt
            yp = 2.0 * np.pi * year_progress(tk)
            dp = torch.from_numpy(2.0 * np.pi * day_progress(tk, self.lon)).to(self.dtype)[None, :].expand(cfg.nlat, -1)
            planes.append(torch.stack([ones * float(np.sin(yp)), ones * float(np.cos(yp)), torch.sin(dp), torch.cos(dp)]))
        planes.append(self.w["static.fields"])
        la = torch.from_numpy(np.deg2rad(self.lat)).to(self.dtype)[:, None].expand(-1, cfg.nlon)
        lo = torch.from_numpy(np.deg2rad(self.lon)).to(self.dtype)[None, :].expand(cfg.nlat, -1)
        planes.append(torch.stack([torch.cos(la), torch.sin(lo), torch.cos(lo)]))
        f = torch.cat(planes, dim=0)
        assert f.shape[0] == cfg.n_features, f.shape
        return f.reshape(cfg.n_features, -1).T.contiguous()

    # -- one step --------------------------------------------------------------------------------
    @torch.no_grad()
    def tendency(self, x, t_seconds: float, taps: dict | None = None) -> torch.Tensor:
        """network output (n_grid, n_prog): the residual in units of diff_std"""
        cfg, ix = self.cfg, self.idx
        x = torch.as_tensor(np.asarray(x))
        st = self.static_embeddings()
        nm = self.g["n_mesh"]
        tap = (lambda k, v: taps.__setitem__(k, v.clone())) if taps is not None else (lambda k, v: None)
        qs = (lambda t: t.half().to(self.dtype)) if self.emulate == "fp16s" else (lambda t: t)   # fp16-only residual streams
        # encoder
        feat = self.features(x, t_seconds)
        tap("feat", feat)
        vg = qs(self.mlp("enc.grid_embed", [feat]))
        tap("grid_embed", vg)
        vm = st["vm"]
        s, r = ix["g2m.senders"], ix["g2m.receivers"]
        e = self.mlp("enc.g2m_edge", [st["e_g2m"], vg[s], vm[r]], table_parts=(1, 2))
        agg = torch.zeros(nm, cfg.latent, dtype=self.dtype).index_add_(0, r, e)
        tap("g2m_update", e); tap("g2m_agg", agg)
        vm = vm + self.mlp("enc.g2m_mesh", [vm, agg])
        vg = qs(vg + self.mlp("enc.g2m_grid", [vg]))
        tap("enc_mesh", vm); tap("enc_grid", vg)
        # processor
        em = st["e_mesh"]
        s, r = ix["mesh.senders"], ix["mesh.receivers"]
        for i in range(cfg.layers):
            e = self.mlp(f"proc{i}.edge", [em, vm[s], vm[r]], table_parts=(1, 2))
            agg = torch.zeros(nm, cfg.latent, dtype=self.dtype).index_add_(0, r, e)
            vm_new = vm + self.mlp(f"proc{i}.node", [vm, agg])
            em = qs(em + e)
            vm = vm_new
            tap(f"proc{i}_mesh", vm); tap(f"proc{i}_update", e); tap(f"proc{i}_agg", agg); tap(f"proc{i}_edges", em)
        # decoder
        s, r = ix["m2g.senders"], ix["m2g.receivers"]
        e = self.mlp("dec.m2g_edge", [st["e_m2g"], vm[s], vg[r]], table_parts=(1, 2))
        agg = torch.zeros(cfg.n_grid, cfg.latent, dtype=self.dtype).index_add_(0, r, e)
        tap("m2g_update", e)
        del e
        vg = qs(vg + self.mlp("dec.m2g_grid", [vg, agg]))
        tap("dec_grid", vg)
        out = self.mlp("dec.out", [vg], ln=False)
        tap("out", out[:, :cfg.n_prog])
        return out[:, :cfg.n_prog]

    @torch.no_grad()
    def step(self, x, t_seconds: float, return_tendency: bool = False):
        """x: (2*n_state, nlat, nlon) fp32 at (t-6h, t) -> state at (t, t+6h)"""
        cfg = self.cfg
        ns, npg = cfg.n_state, cfg.n_prog
        x = torch.as_tensor(np.asarray(x))
        tend = self.tendency(x, t_seconds)
        xs = x.reshape(2, ns, cfg.nlat, cfg.nlon).to(self.dtype)
        new = torch.empty(ns, cfg.nlat, cfg.nlon, dtype=self.dtype)
        new[:npg] = xs[1, :npg] + self.w["norm.diff_std"][:npg, None, None] * tend.T.reshape(npg, cfg.nlat, cfg.nlon)
        new[npg] = torch.from_numpy(toa_radiation(t_seconds + 3600.0 * cfg.dt_hours, self.lat, self.lon)).to(self.dtype)
        y = torch.cat([xs[1], new], dim=0)
        return (y, tend) if return_tendency else y


def rel_err_per_channel(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """per-channel relative L2 error of a against b, both (C, nlat, nlon)"""
    a = np.asarray(a, dtype=np.float64).reshape(a.shape[0], -1)
    b = np.asarray(b, dtype=np.float64).reshape(b.shape[0], -1)
    return np.linalg.norm(a - b, axis=1) / np.maximum(np.linalg.norm(b, axis=1), 1e-30)
