"""Host-side handle on one CUDA step operator (thin Python over the C-ABI).

PyTorch tensors are used as device-memory containers only: the engine receives raw
``data_ptr()`` addresses and the current CUDA stream.
"""
from __future__ import annotations

import ctypes as C
import functools
from collections import OrderedDict

import numpy as np

from . import _ffi
from .config import GraphCastConfig, PanguConfig, SFNOConfig

ARENA_ALIGN = 64  # floats (256 B)


def pack_arena(weights: "OrderedDict[str, np.ndarray]"):
    """Flatten named fp32 tensors into one arena + manifest (name, offset, count)."""
    offs, total = [], 0
    for name, a in weights.items():
        offs.append(total)
        total += (a.size + ARENA_ALIGN - 1) // ARENA_ALIGN * ARENA_ALIGN
    arena = np.zeros(total, dtype=np.float32)
    manifest = (_ffi.ParamDesc * len(weights))()
    for i, ((name, a), off) in enumerate(zip(weights.items(), offs)):
        arena[off:off + a.size] = np.asarray(a, dtype=np.float32).reshape(-1)
        manifest[i].name = name.encode()
        manifest[i].offset = off
        manifest[i].count = a.size
    return arena, manifest


def _pangu_cfg_c(cfg: PanguConfig) -> _ffi.PanguConfigC:
    assert tuple(cfg.patch) == (2, 4, 4) and tuple(cfg.window) == (2, 6, 12)
    c = _ffi.PanguConfigC()
    c.nlat, c.nlon, c.n_levels, c.dim = cfg.nlat, cfg.nlon, cfg.n_levels, cfg.dim
    c.depths[:] = cfg.depths
    c.heads[:] = cfg.heads
    c.ln_eps, c.mask_value = cfg.ln_eps, cfg.mask_value
    return c


def _sfno_cfg_c(cfg: SFNOConfig) -> _ffi.SFNOConfigC:
    c = _ffi.SFNOConfigC()
    c.nlat, c.nlon, c.n_channels, c.embed = cfg.nlat, cfg.nlon, cfg.n_channels, cfg.embed
    c.layers, c.scale_factor, c.mlp_ratio, c.eps = cfg.layers, cfg.scale_factor, cfg.mlp_ratio, cfg.eps
    return c


def _graphcast_cfg_c(cfg: GraphCastConfig, graph) -> _ffi.GraphCastConfigC:
    c = _ffi.GraphCastConfigC()
    c.nlat, c.nlon, c.latent, c.layers = cfg.nlat, cfg.nlon, cfg.latent, cfg.layers
    c.n_mesh, c.n_mesh_edges, c.n_g2m_edges = graph["n_mesh"], len(graph["mesh.senders"]), len(graph["g2m.senders"])
    c.n_state, c.n_prog, c.n_static, c.dt_hours, c.ln_eps = cfg.n_state, cfg.n_prog, cfg.n_static, cfg.dt_hours, cfg.ln_eps
    return c


class StepEngine:
    """One 6-h step operator resident on one GPU."""

    def __init__(self, cfg, device: int = 0, graph=None):
        import torch
        if not torch.cuda.is_available():
            raise _ffi.SkyError("skyrim_b200 needs a CUDA device (sm_90a, H100); there is no CPU fallback")
        self.cfg = cfg
        self.device = device
        self.torch = torch
        L = self._L = _ffi.lib()
        if isinstance(cfg, PanguConfig):
            kind, cc = _ffi.SKY_MODEL_PANGU6, _pangu_cfg_c(cfg)
        elif isinstance(cfg, SFNOConfig):
            kind, cc = _ffi.SKY_MODEL_SFNO73, _sfno_cfg_c(cfg)
        elif isinstance(cfg, GraphCastConfig):
            # the multimesh and the grid<->mesh edge sets are built on the host once (icomesh.py) and travel in the arena
            if graph is None:
                from .icomesh import build_graph
                graph = build_graph(cfg.nlat, cfg.nlon, cfg.mesh_levels, cfg.radius_frac)
            self.graph = graph
            kind, cc = _ffi.SKY_MODEL_GRAPHCAST, _graphcast_cfg_c(cfg, graph)
        else:
            raise TypeError(cfg)
        self.n_channels = cfg.n_channels
        h = C.c_void_p()
        _ffi.check(L.sky_model_create(C.byref(h), kind, C.byref(cc), C.sizeof(cc), device), "sky_model_create", L)
        self._h = h
        self._ws = None
        self._ws_batch = 0
        self._ws_source = None

    # -- weights ---------------------------------------------------------------------------
    def load_weights(self, weights: "OrderedDict[str, np.ndarray]"):
        if isinstance(self.cfg, GraphCastConfig) and not any(k.startswith("graph.") for k in weights):
            from .icomesh import graph_arena_entries
            weights = OrderedDict(list(weights.items()) + list(graph_arena_entries(self.graph).items()))
        arena, manifest = pack_arena(weights)
        self.load_arena(arena, manifest)

    def load_arena(self, arena, manifest):
        """``arena``: host numpy fp32 array, or a CUDA torch tensor (e.g. after a broadcast)."""
        L = self._L
        torch = self.torch
        st = torch.cuda.current_stream(self.device).cuda_stream
        if isinstance(arena, np.ndarray):
            ptr, n, on_dev = arena.ctypes.data, arena.size, 0
        else:
            assert arena.is_cuda and arena.dtype == torch.float32 and arena.is_contiguous()
            ptr, n, on_dev = arena.data_ptr(), arena.numel(), 1
        _ffi.check(L.sky_model_load_weights(self._h, ptr, n, manifest, len(manifest), on_dev, st),
                   "sky_model_load_weights", L)

    # -- stepping --------------------------------------------------------------------------
    def share_workspace(self, other: "StepEngine"):
        """Step on ``other``'s workspace from now on instead of allocating one (about 2.7 GB per member for Pangu at
        721x1440).  The workspace is per-step scratch, so this is safe while both handles step in order on one stream;
        it grows to the larger batch either handle asks for."""
        if other is self or other._ws_source is not None or other.device != self.device:
            raise ValueError("share_workspace: the owner must be another handle with its own workspace on the same device")
        self._ws, self._ws_batch, self._ws_source = None, 0, other

    def _workspace(self, batch: int):
        if self._ws_source is not None:
            ws = self._ws_source._workspace(batch)
            need = self._L.sky_model_workspace_bytes(self._h, batch)
            if ws.numel() < need:
                raise _ffi.SkyError(f"shared workspace of {ws.numel()} bytes is smaller than the {need} this step needs")
            return ws
        if self._ws is None or self._ws_batch < batch:
            nbytes = self._L.sky_model_workspace_bytes(self._h, batch)
            self._ws = self.torch.empty(nbytes, dtype=self.torch.uint8, device=f"cuda:{self.device}")
            self._ws_batch = batch
        return self._ws

    def step(self, x_in, x_out=None):
        """x_in: CUDA fp32 (B, C, nlat, nlon) contiguous.  Returns x_out (allocated if None).
        Asynchronous on the current stream."""
        torch = self.torch
        assert x_in.is_cuda and x_in.dtype == torch.float32 and x_in.is_contiguous() and x_in.dim() == 4
        B = x_in.shape[0]
        assert tuple(x_in.shape[1:]) == (self.n_channels, self.cfg.nlat, self.cfg.nlon), x_in.shape
        if x_out is None:
            x_out = torch.empty_like(x_in)
        ws = self._workspace(B)
        st = torch.cuda.current_stream(self.device).cuda_stream
        _ffi.check(self._L.sky_model_step(self._h, x_in.data_ptr(), x_out.data_ptr(), B, ws.data_ptr(),
                                             ws.numel(), st), "sky_model_step", self._L)
        return x_out

    def set_clock(self, when):
        """Valid time of the LAST time slice of the state the next step starts from (datetime, numpy datetime64 or unix
        seconds).  Only operators with time-dependent forcings (GraphCast) use it; they advance it themselves per step."""
        t = unix_seconds(when)
        st = self.torch.cuda.current_stream(self.device).cuda_stream
        _ffi.check(self._L.sky_model_set_clock(self._h, t, st), "sky_model_set_clock", self._L)

    def toa_radiation(self, when, out=None):
        """(nlat, nlon) CUDA fp32: the toa-radiation forcing channel ("tp06") at time ``when``."""
        torch = self.torch
        if out is None:
            out = torch.empty((self.cfg.nlat, self.cfg.nlon), dtype=torch.float32, device=f"cuda:{self.device}")
        st = torch.cuda.current_stream(self.device).cuda_stream
        _ffi.check(self._L.sky_toa_radiation(out.data_ptr(), self.cfg.nlat, self.cfg.nlon, unix_seconds(when), st),
                   "sky_toa_radiation", self._L)
        return out

    def debug_tensor(self, what: str, shape, batch: int = 1):
        torch = self.torch
        out = torch.empty(shape, dtype=torch.float32, device=f"cuda:{self.device}")
        st = torch.cuda.current_stream(self.device).cuda_stream
        _ffi.check(self._L.sky_model_debug_copy(self._h, what.encode(), out.data_ptr(), out.numel(),
                                                   self._workspace(batch).data_ptr(), batch, st), "debug_copy", self._L)
        return out

    RANGE_SLOTS = ("token_images", "qkv", "attention_out", "resampled_images", "pixel_images", "hidden_images",
                   "spectral_images", "unused")
    FP16_LIMIT = 3.0e4

    def step_guarded(self, x_in, x_out=None, limit: float | None = None):
        """One step with the fp16-range guard on: the engine scans every fp16 operand image it produces (the tensor cores
        take 5-exponent-bit operands) and this call raises if any |value| exceeds ``limit`` (default 3e4) or is not finite.
        Meant for the FIRST step of a rollout with real checkpoints (synthetic weights keep every activation O(1)); the
        guarded step runs with plain launches and a few extra reduction kernels.  Returns (x_out, {class: max |value|})."""
        limit = self.FP16_LIMIT if limit is None else limit
        self.debug_set("range_guard", 1)
        try:
            y = self.step(x_in, x_out)
            r = self.torch.empty(8, dtype=self.torch.float32, device=f"cuda:{self.device}")
            st = self.torch.cuda.current_stream(self.device).cuda_stream
            _ffi.check(self._L.sky_model_debug_copy(self._h, b"range", r.data_ptr(), 8, self._workspace(x_in.shape[0]).data_ptr(),
                                                    x_in.shape[0], st), "debug_copy(range)", self._L)
            vals = r.cpu().tolist()
        finally:
            self.debug_set("range_guard", 0)
        ranges = {n: v for n, v in zip(self.RANGE_SLOTS, vals) if v != 0.0}
        bad = {n: v for n, v in ranges.items() if not (v <= limit)}
        if bad:
            raise _ffi.SkyError(f"fp16 operand range exceeded (limit {limit:g}): {bad}; this checkpoint needs operand scaling "
                                f"the engine does not implement")
        return y, ranges

    def debug_set(self, key: str, value: int):
        """test taps (never environment variables): e.g. ``debug_set("stop_after", 3)``"""
        _ffi.check(self._L.sky_model_debug_set(self._h, key.encode(), int(value)), "debug_set", self._L)

    # -- per-kernel-family device timing (CUDA events inside the library) -------------------
    @staticmethod
    def profile_tags():
        L = _ffi.lib()
        return [L.sky_profile_tag_name(i).decode() for i in range(L.sky_profile_tag_count())]

    def profile_begin(self, tags=None):
        names = self.profile_tags()
        mask = 0
        for i, n in enumerate(names):
            if tags is None or n in tags:
                mask |= 1 << i
        _ffi.check(self._L.sky_model_profile_begin(self._h, mask), "profile_begin", self._L)

    def profile_end(self):
        """-> {family: (total_ms, launches)} for the families that ran since profile_begin."""
        names = self.profile_tags()
        ms = (C.c_double * len(names))()
        cnt = (C.c_uint64 * len(names))()
        _ffi.check(self._L.sky_model_profile_end(self._h, ms, cnt, len(names)), "profile_end", self._L)
        return {n: (ms[i], int(cnt[i])) for i, n in enumerate(names) if cnt[i]}

    def close(self):
        if getattr(self, "_h", None):
            self._L.sky_model_destroy(self._h)
            self._h = None
            self._ws = None
            self._ws_source = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def perturb_ic(x, sigma_c, amp: float, seed: int, member0: int = 0):
    """In-place Gaussian perturbation of (M, C, nlat, nlon) CUDA fp32 members (K11)."""
    import torch
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 4
    M, Cn = x.shape[0], x.shape[1]
    plane = x.shape[2] * x.shape[3]
    assert sigma_c.is_cuda and sigma_c.numel() == Cn
    st = torch.cuda.current_stream(x.device).cuda_stream
    _ffi.check(_ffi.lib().sky_perturb_ic(x.data_ptr(), sigma_c.data_ptr(), float(amp), int(seed), int(member0), M,
                                         Cn, plane, st), "sky_perturb_ic")
    return x


def grf_spectrum(alpha: float = 2.0, tau: float = 3.0, lmax: int = 180):
    """Per-degree standard deviations of the spherical Gaussian random field, float64 [lmax + 1]:
    s_l = k (l (l + 1) + tau^2)^(-alpha / 2) for 1 <= l <= lmax, s_0 = 0 (zero mean over the sphere), with k chosen so that
    sum_l s_l^2 (2l + 1) / (4 pi) = 1 (unit pointwise variance).  Also returns the fraction of the untruncated field's
    variance that degrees <= lmax keep (alpha > 1, else the untruncated variance is infinite)."""
    if not alpha > 1.0:
        raise ValueError(f"alpha = {alpha} must exceed 1 for the field's variance to be finite")
    if lmax < 1:
        raise ValueError(f"lmax = {lmax} must be at least 1")
    l = np.arange(lmax + 1, dtype=np.float64)
    s = (l * (l + 1) + tau * tau) ** (-alpha / 2)
    s[0] = 0.0
    var = np.sum(s * s * (2 * l + 1))
    # untruncated sum: exact terms up to 2^20, then the integral of (2l + 1) u^-alpha du / dl from u(N + 1/2)
    big = np.arange(1, 1 << 20, dtype=np.float64)
    u = lambda x: x * (x + 1) + tau * tau  # noqa: E731
    total = np.sum((2 * big + 1) * u(big) ** -alpha) + u(big[-1] + 0.5) ** (1 - alpha) / (alpha - 1)
    return s / np.sqrt(var / (4 * np.pi)), float(var / total)


_GRF_TABLES: "OrderedDict[tuple, object]" = OrderedDict()


def grf_legendre_table(nlat: int, lmax: int, device):
    """Pbar_l^m(cos theta_k) on the equiangular grid (sht.legpoly), fp32 on ``device``, m-major triangle
    [m][k][l - m] (the layout sky_perturb_ic_grf reads; 47 MB at nlat 721, lmax 180).  The last four are cached."""
    import torch
    from . import sht
    key = (nlat, lmax, str(device))
    if key not in _GRF_TABLES:
        p = sht.legpoly(lmax + 1, lmax + 1, sht.clenshaw_curtis(nlat)[0])          # [m, l, k]
        tab = np.concatenate([p[m, m:].T.astype(np.float32).reshape(-1) for m in range(lmax + 1)])
        _GRF_TABLES[key] = torch.from_numpy(tab).to(device)
        while len(_GRF_TABLES) > 4:
            _GRF_TABLES.popitem(last=False)
    return _GRF_TABLES[key]


@functools.lru_cache(maxsize=16)
def _grf_spectrum_device(alpha: float, tau: float, lmax: int, device):
    import torch
    return torch.from_numpy(grf_spectrum(alpha, tau, lmax)[0].astype(np.float32)).to(device)


def perturb_ic_grf(x, sigma_c, amp: float, seed: int, member0: int = 0, alpha: float = 2.0, tau: float = 3.0,
                   lmax: int = 180):
    """In-place spherically correlated perturbation of (M, C, nlat, nlon) CUDA fp32 members on the equiangular grid:
    x[m, c] += amp sigma_c f, f a Gaussian random field with unit pointwise variance and the spectrum of
    ``grf_spectrum(alpha, tau, lmax)``, drawn per (seed, member0 + m, c) (include/skyrim_b200.h sky_perturb_ic_grf).
    Channels with sigma_c == 0 stay bit-identical.  lmax may be at most (nlat - 1) / 2, the finest degree the grid's
    latitudes resolve (360 at 0.25 degrees)."""
    import torch
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 4
    M, Cn, nlat, nlon = x.shape
    assert sigma_c.is_cuda and sigma_c.dtype == torch.float32 and sigma_c.is_contiguous() and sigma_c.numel() == Cn
    if not 1 <= lmax <= (nlat - 1) // 2:
        raise ValueError(f"lmax = {lmax} must lie in [1, {(nlat - 1) // 2}] on {nlat} latitudes")
    L = _ffi.lib()
    s = _grf_spectrum_device(float(alpha), float(tau), lmax, x.device)
    leg = grf_legendre_table(nlat, lmax, x.device)
    nbytes = L.sky_grf_workspace_bytes(M, Cn, nlat, nlon, lmax)
    if nbytes == 0:
        _ffi.check(-1, "sky_grf_workspace_bytes", L)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    st = torch.cuda.current_stream(x.device).cuda_stream
    _ffi.check(L.sky_perturb_ic_grf(x.data_ptr(), sigma_c.data_ptr(), float(amp), int(seed), int(member0), M, Cn, nlat,
                                    nlon, lmax, s.data_ptr(), leg.data_ptr(), ws.data_ptr(), nbytes, st),
               "sky_perturb_ic_grf", L)
    return x


ENS_MAX_MEMBERS, ENS_MAX_CHANNELS, ENS_MAX_QUANTILES, ENS_MAX_EVENTS = 64, 128, 8, 64
ENS_MAX_SOURCES = 4


def _c_array(ctype, values):
    """a ctypes array of ``values`` (one element even when empty, so the pointer is never null)"""
    return (ctype * max(len(values), 1))(*values)


def _check_out(t, shape, dtype, name):
    if tuple(t.shape) != shape or t.dtype != dtype or not t.is_contiguous() or not t.is_cuda:
        raise ValueError(f"{name} of shape {tuple(t.shape)} {t.dtype} on {t.device}: contiguous CUDA {dtype} {shape} "
                         "needed")


def _member_view(x, channel_offset: int = 0, name: str = "x"):
    """(M, H, W, count, member_stride, base) of ``x``, a CUDA fp32 (M, C, H, W) tensor or a view of one whose members each
    hold contiguous (C, H, W) planes, as the statistics and verification entries read it: the count = C - channel_offset
    channels from ``channel_offset`` on, member m's at the address base + 4 m member_stride"""
    import torch
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4):
        raise ValueError(f"{name} must be a CUDA fp32 (members, channels, nlat, nlon) tensor")
    M, Cn, H, W = x.shape
    plane = H * W
    if x.stride(3) != 1 or x.stride(2) != W or x.stride(1) != plane:
        raise ValueError(f"each member of {name} must hold contiguous (C, H, W) planes (strides {x.stride()})")
    if not 0 <= channel_offset < Cn:
        raise ValueError(f"channel_offset = {channel_offset} is outside [0, {Cn})")
    member_stride = x.stride(0) if M > 1 else max(x.stride(0), Cn * plane)
    return M, H, W, Cn - channel_offset, member_stride, x.data_ptr() + 4 * channel_offset * plane


def _verified_members(x, channels, channel_offset, row_weights=None, **fields):
    """``_member_view(x, channel_offset)`` and the selected channels sel (default: all), with every named field (truth,
    clim) None or a contiguous CUDA fp32 (n_sel, H, W) tensor, and ``row_weights`` None or a contiguous CUDA fp64
    (n_regions, H) tensor: (M, H, W, count, member_stride, base, sel)"""
    import torch
    M, H, W, count, member_stride, base = _member_view(x, channel_offset)
    sel = list(range(count)) if channels is None else [int(c) for c in channels]
    for name, t in fields.items():
        if t is not None and (not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous()
                              or tuple(t.shape) != (len(sel), H, W)):
            raise ValueError(f"{name} must be a contiguous CUDA fp32 {(len(sel), H, W)} tensor (got {tuple(t.shape)})")
    if row_weights is not None and not (row_weights.is_cuda and row_weights.dtype == torch.float64
                                        and row_weights.is_contiguous() and row_weights.dim() == 2
                                        and row_weights.shape[1] == H):
        raise ValueError(f"row_weights must be a contiguous CUDA fp64 (n_regions, {H}) tensor")
    return M, H, W, count, member_stride, base, sel


def ensemble_statistics(x, channels=None, quantiles=(), events=(), channel_offset: int = 0, out=None):
    """Per-point statistics over the members of a CUDA fp32 (M, C, H, W) tensor, or a view of one whose members each hold
    contiguous (C, H, W) planes (include/skyrim_b200.h sky_ensemble_stats).  Channels are counted from ``channel_offset``
    (a GraphCast state reduces its new time slice with offset 83); ``channels`` lists the reduced ones (default: all),
    ``quantiles`` the numpy-"linear" quantiles, ``events`` (i, threshold) pairs for P(x > threshold) of ``channels[i]``
    with i nondecreasing.  Returns (stats (2 + n_q, n_sel, H, W): mean, spread, quantiles; prob (n_events, H, W)), into
    ``out`` = (stats, prob) when given.  Asynchronous on the current stream."""
    import torch
    M, H, W, count, member_stride, base, sel = _verified_members(x, channels, channel_offset)
    q = [float(v) for v in quantiles]
    ev_sel, ev_thr = [int(i) for i, _ in events], [float(t) for _, t in events]
    shapes = ((2 + len(q), len(sel), H, W), (len(ev_sel), H, W))
    if out is None:
        out = tuple(torch.empty(s, dtype=torch.float32, device=x.device) for s in shapes)
    stats, prob = out
    for t, s, name in zip(out, shapes, ("stats", "prob")):
        _check_out(t, s, torch.float32, name)
    L = _ffi.lib()
    st = torch.cuda.current_stream(x.device).cuda_stream
    _ffi.check(L.sky_ensemble_stats(base, M, member_stride, H * W, count, _c_array(C.c_int32, sel), len(sel),
                                    _c_array(C.c_double, q), len(q), _c_array(C.c_int32, ev_sel),
                                    _c_array(C.c_float, ev_thr), len(ev_sel), stats.data_ptr(),
                                    prob.data_ptr() if prob.numel() else None, st), "sky_ensemble_stats", L)
    return stats, prob


def multi_model_statistics(sources, channels_per_source, quantiles=(), events=(), source_means: bool = True, out=None):
    """``ensemble_statistics`` over the members of up to four sources pooled in source-then-member order
    (include/skyrim_b200.h sky_ensemble_stats_multi).  ``sources``: CUDA fp32 (M_k, C_k, H, W) tensors or views whose
    members each hold contiguous (C_k, H, W) planes, sum of M_k at most 64 (a GraphCast state's new slice is the view
    ``state.view(M, 166, H, W)[:, 83:]``); ``channels_per_source[k]`` lists, for every selected channel, its index in
    source k; ``events`` as for ``ensemble_statistics``.  Returns (stats (2 + n_q, n_sel, H, W), prob (n_events, H, W),
    means (K, n_sel, H, W): the mean of each source's own members, or None without ``source_means``), into ``out`` =
    (stats, prob, means) when given.  Asynchronous on the current stream."""
    import torch
    K = len(sources)
    if not 1 <= K <= ENS_MAX_SOURCES or len(channels_per_source) != K:
        raise ValueError(f"{K} sources with {len(channels_per_source)} channel lists: 1 to {ENS_MAX_SOURCES} sources, one "
                         "list each")
    views = [_member_view(x, name=f"source {k}") for k, x in enumerate(sources)]
    members, nlat, nlon, counts, strides, bases = zip(*views)
    if len(set(zip(nlat, nlon))) != 1:
        raise ValueError(f"every source must lie on one grid ({list(zip(nlat, nlon))})")
    H, W = nlat[0], nlon[0]
    sel = [[int(c) for c in chans] for chans in channels_per_source]
    n_sel = len(sel[0])
    if any(len(c) != n_sel for c in sel):
        raise ValueError("every source must list the same number of channels")
    q = [float(v) for v in quantiles]
    ev_sel, ev_thr = [int(i) for i, _ in events], [float(t) for _, t in events]
    shapes = ((2 + len(q), n_sel, H, W), (len(ev_sel), H, W), (K, n_sel, H, W))
    if out is None:
        out = tuple(torch.empty(s, dtype=torch.float32, device=sources[0].device) for s in shapes)
        if not source_means:
            out = out[:2] + (None,)
    stats, prob, means = out
    for t, s, name in zip(out, shapes, ("stats", "prob", "means")):
        if t is not None:
            _check_out(t, s, torch.float32, name)
    L = _ffi.lib()
    st = torch.cuda.current_stream(sources[0].device).cuda_stream
    _ffi.check(L.sky_ensemble_stats_multi(K, _c_array(C.c_void_p, bases), _c_array(C.c_int32, members),
                                          _c_array(C.c_int64, strides), _c_array(C.c_int32, counts),
                                          _c_array(C.c_int32, [c for chans in sel for c in chans]), n_sel, H * W,
                                          _c_array(C.c_double, q), len(q), _c_array(C.c_int32, ev_sel),
                                          _c_array(C.c_float, ev_thr), len(ev_sel), stats.data_ptr(),
                                          prob.data_ptr() if prob.numel() else None,
                                          means.data_ptr() if means is not None else None, st),
               "sky_ensemble_stats_multi", L)
    return stats, prob, means


SCORES_MAX_REGIONS, SCORES_TERMS, SCORES_BLOCKS = 4, 9, 128
MAP_TERMS = 5


def forecast_scores(x, truth, row_weights, channels=None, clim=None, channel_offset: int = 0, out=None):
    """Verification sums of the members of a CUDA fp32 (M, C, H, W) tensor, or a view of one whose members each hold
    contiguous (C, H, W) planes, against ``truth`` (CUDA fp32 (n_sel, H, W)) and optionally ``clim`` (same shape), per
    region of ``row_weights`` (CUDA fp64 (n_regions, H), ``scores.region_weights``) (include/skyrim_b200.h
    sky_forecast_scores).  Channels are counted from ``channel_offset`` (a GraphCast state scores its new time slice with
    offset 83); ``channels`` lists the scored ones (default: all), in the order of the truth's planes.  Returns the CUDA
    fp64 sums (n_regions, n_sel, 9) (``scores.SUMS`` names them; ``scores.metrics_from_sums`` forms the metrics), into
    ``out`` when given.  Asynchronous on the current stream."""
    import torch
    M, H, W, count, member_stride, base, sel = _verified_members(x, channels, channel_offset, row_weights,
                                                                 truth=truth, clim=clim)
    R = row_weights.shape[0]
    shape = (R, len(sel), SCORES_TERMS)
    if out is None:
        out = torch.empty(shape, dtype=torch.float64, device=x.device)
    _check_out(out, shape, torch.float64, "out")
    ws = torch.empty(max(R * len(sel) * SCORES_TERMS * SCORES_BLOCKS, 1), dtype=torch.float64, device=x.device)
    L = _ffi.lib()
    st = torch.cuda.current_stream(x.device).cuda_stream
    _ffi.check(L.sky_forecast_scores(base, M, member_stride, H, W, count, _c_array(C.c_int32, sel), len(sel),
                                     truth.data_ptr(), None if clim is None else clim.data_ptr(), row_weights.data_ptr(),
                                     R, ws.data_ptr(), 8 * ws.numel(), out.data_ptr(), st), "sky_forecast_scores", L)
    return out


def forecast_rank_histogram(x, truth, row_weights, seed: int, date_index: int, lead_index: int, channels=None,
                            channel_offset: int = 0, out=None):
    """Rank histogram of ``truth`` (CUDA fp32 (n_sel, H, W)) among the members of x (as for ``forecast_scores``), per
    region of ``row_weights`` (include/skyrim_b200.h sky_forecast_rank_histogram): ties between the truth and members are
    broken by Philox draws keyed by (``seed``, ``date_index``) and counted by (point, channel index in x from
    ``channel_offset``, ``lead_index``).  Returns the CUDA fp64 (n_regions, n_sel, M + 1) histogram, each summing to 1,
    into ``out`` when given.  Asynchronous on the current stream."""
    import torch
    M, H, W, count, member_stride, base, sel = _verified_members(x, channels, channel_offset, row_weights, truth=truth)
    if not 0 <= int(seed) < 2 ** 32 or int(date_index) < 0 or int(lead_index) < 0:
        raise ValueError(f"seed = {seed} must lie in [0, 2^32), date_index = {date_index} and lead_index = {lead_index} "
                         "must not be negative")
    R = row_weights.shape[0]
    shape = (R, len(sel), M + 1)
    if out is None:
        out = torch.empty(shape, dtype=torch.float64, device=x.device)
    _check_out(out, shape, torch.float64, "out")
    ws = torch.empty(max(len(sel) * H * (M + 2), 1), dtype=torch.int32, device=x.device)
    L = _ffi.lib()
    st = torch.cuda.current_stream(x.device).cuda_stream
    _ffi.check(L.sky_forecast_rank_histogram(base, M, member_stride, H, W, count, _c_array(C.c_int32, sel), len(sel),
                                             truth.data_ptr(), row_weights.data_ptr(), R, int(seed), int(date_index),
                                             int(lead_index), ws.data_ptr(), 4 * ws.numel(), out.data_ptr(), st),
               "sky_forecast_rank_histogram", L)
    return out


def score_maps_accumulate(x, truth, maps, channels=None, channel_offset: int = 0):
    """Adds the per-point terms e, e^2, sum_m (x_m - x_bar)^2, mae and G of the members of x against ``truth`` (both as
    for ``forecast_scores``) to ``maps``, a CUDA fp64 (n_sel, 5, H, W) tensor of accumulators (include/skyrim_b200.h
    sky_forecast_score_maps; ``scores.map_metrics`` forms the maps).  Returns ``maps``.  Asynchronous on the current
    stream."""
    import torch
    M, H, W, count, member_stride, base, sel = _verified_members(x, channels, channel_offset, truth=truth)
    _check_out(maps, (len(sel), MAP_TERMS, H, W), torch.float64, "maps")
    L = _ffi.lib()
    st = torch.cuda.current_stream(x.device).cuda_stream
    _ffi.check(L.sky_forecast_score_maps(base, M, member_stride, H, W, count, _c_array(C.c_int32, sel), len(sel),
                                         truth.data_ptr(), maps.data_ptr(), st), "sky_forecast_score_maps", L)
    return maps


def _pooled_sources(sources, channels_per_source, truth=None, clim=None, row_weights=None):
    """the source arguments of the *_multi verification entries: (K, M, H, W, bases, members, strides, counts, flat
    channels, n_sel), with sources and their channel lists checked as ``multi_model_statistics`` checks them and truth /
    clim / row_weights as ``_verified_members`` checks them"""
    import torch
    K = len(sources)
    if not 1 <= K <= ENS_MAX_SOURCES or len(channels_per_source) != K:
        raise ValueError(f"{K} sources with {len(channels_per_source)} channel lists: 1 to {ENS_MAX_SOURCES} sources, one "
                         "list each")
    views = [_member_view(x, name=f"source {k}") for k, x in enumerate(sources)]
    members, nlat, nlon, counts, strides, bases = zip(*views)
    if len(set(zip(nlat, nlon))) != 1:
        raise ValueError(f"every source must lie on one grid ({list(zip(nlat, nlon))})")
    if len({x.device for x in sources}) != 1:
        raise ValueError(f"every source must lie on one device ({[str(x.device) for x in sources]})")
    H, W = nlat[0], nlon[0]
    sel = [[int(c) for c in chans] for chans in channels_per_source]
    n_sel = len(sel[0])
    if any(len(c) != n_sel for c in sel):
        raise ValueError("every source must list the same number of channels")
    for name, t in dict(truth=truth, clim=clim).items():
        if t is not None and (not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous()
                              or tuple(t.shape) != (n_sel, H, W)):
            raise ValueError(f"{name} must be a contiguous CUDA fp32 {(n_sel, H, W)} tensor (got {tuple(t.shape)})")
    if row_weights is not None and not (row_weights.is_cuda and row_weights.dtype == torch.float64
                                        and row_weights.is_contiguous() and row_weights.dim() == 2
                                        and row_weights.shape[1] == H):
        raise ValueError(f"row_weights must be a contiguous CUDA fp64 (n_regions, {H}) tensor")
    flat = [c for chans in sel for c in chans]
    return (K, sum(members), H, W, _c_array(C.c_void_p, bases), _c_array(C.c_int32, members),
            _c_array(C.c_int64, strides), _c_array(C.c_int32, counts), _c_array(C.c_int32, flat), n_sel)


def forecast_scores_multi(sources, channels_per_source, truth, row_weights, clim=None, out=None):
    """``forecast_scores`` of the members of up to four sources pooled in source-then-member order
    (include/skyrim_b200.h sky_forecast_scores_multi): ``sources`` and ``channels_per_source`` as for
    ``multi_model_statistics`` (a GraphCast state's new slice is a view), ``truth`` / ``clim`` CUDA fp32 (n_sel, H, W) in
    the order of the channel lists.  Bitwise the sums ``forecast_scores`` gives on the pooled members stacked into one
    tensor in source 0's channel order.  Returns the CUDA fp64 sums (n_regions, n_sel, 9), into ``out`` when given.
    Asynchronous on the current stream."""
    import torch
    K, M, H, W, bases, members, strides, counts, flat, n_sel = _pooled_sources(sources, channels_per_source, truth, clim,
                                                                               row_weights)
    dev = sources[0].device
    R = row_weights.shape[0]
    shape = (R, n_sel, SCORES_TERMS)
    if out is None:
        out = torch.empty(shape, dtype=torch.float64, device=dev)
    _check_out(out, shape, torch.float64, "out")
    ws = torch.empty(max(R * n_sel * SCORES_TERMS * SCORES_BLOCKS, 1), dtype=torch.float64, device=dev)
    L = _ffi.lib()
    st = torch.cuda.current_stream(dev).cuda_stream
    _ffi.check(L.sky_forecast_scores_multi(K, bases, members, strides, counts, flat, n_sel, H, W, truth.data_ptr(),
                                           None if clim is None else clim.data_ptr(), row_weights.data_ptr(), R,
                                           ws.data_ptr(), 8 * ws.numel(), out.data_ptr(), st),
               "sky_forecast_scores_multi", L)
    return out


def forecast_rank_histogram_multi(sources, channels_per_source, truth, row_weights, seed: int, date_index: int,
                                  lead_index: int, out=None):
    """``forecast_rank_histogram`` of the pooled members of ``sources`` (as for ``forecast_scores_multi``;
    include/skyrim_b200.h sky_forecast_rank_histogram_multi): the tie-breaking draws are counted by source 0's channel
    index.  Returns the CUDA fp64 (n_regions, n_sel, M + 1) histogram, M the pooled member count, into ``out`` when given.
    Asynchronous on the current stream."""
    import torch
    K, M, H, W, bases, members, strides, counts, flat, n_sel = _pooled_sources(sources, channels_per_source, truth, None,
                                                                               row_weights)
    if not 0 <= int(seed) < 2 ** 32 or int(date_index) < 0 or int(lead_index) < 0:
        raise ValueError(f"seed = {seed} must lie in [0, 2^32), date_index = {date_index} and lead_index = {lead_index} "
                         "must not be negative")
    dev = sources[0].device
    R = row_weights.shape[0]
    shape = (R, n_sel, M + 1)
    if out is None:
        out = torch.empty(shape, dtype=torch.float64, device=dev)
    _check_out(out, shape, torch.float64, "out")
    ws = torch.empty(max(n_sel * H * (M + 2), 1), dtype=torch.int32, device=dev)
    L = _ffi.lib()
    st = torch.cuda.current_stream(dev).cuda_stream
    _ffi.check(L.sky_forecast_rank_histogram_multi(K, bases, members, strides, counts, flat, n_sel, H, W, truth.data_ptr(),
                                                   row_weights.data_ptr(), R, int(seed), int(date_index), int(lead_index),
                                                   ws.data_ptr(), 4 * ws.numel(), out.data_ptr(), st),
               "sky_forecast_rank_histogram_multi", L)
    return out


def score_maps_accumulate_multi(sources, channels_per_source, truth, maps):
    """``score_maps_accumulate`` of the pooled members of ``sources`` (as for ``forecast_scores_multi``;
    include/skyrim_b200.h sky_forecast_score_maps_multi) into ``maps``, CUDA fp64 (n_sel, 5, H, W).  Returns ``maps``.
    Asynchronous on the current stream."""
    import torch
    K, M, H, W, bases, members, strides, counts, flat, n_sel = _pooled_sources(sources, channels_per_source, truth)
    _check_out(maps, (n_sel, MAP_TERMS, H, W), torch.float64, "maps")
    L = _ffi.lib()
    st = torch.cuda.current_stream(sources[0].device).cuda_stream
    _ffi.check(L.sky_forecast_score_maps_multi(K, bases, members, strides, counts, flat, n_sel, H, W, truth.data_ptr(),
                                               maps.data_ptr(), st), "sky_forecast_score_maps_multi", L)
    return maps


SITES_METHODS = {"bilinear": 0, "nearest": 1}
SITES_MAX, SITE_TERMS, SITES_THREADS = 1 << 20, 6, 128


class SiteTable:
    """A site table on one GPU (include/skyrim_b200.h sky_sites_create): the 4-point stencil of every site at (``lat``,
    ``lon``) degrees on the equiangular (nlat, nlon) grid, "bilinear" or "nearest", validated on the host and uploaded
    once.  ``sample_sites`` reads it; ``close`` (or garbage collection) frees it."""

    def __init__(self, lat, lon, nlat: int, nlon: int, method: str = "bilinear", device: int = 0):
        if method not in SITES_METHODS:
            raise ValueError(f"unknown site method {method!r} ({', '.join(SITES_METHODS)})")
        lat = np.ascontiguousarray(lat, dtype=np.float64).reshape(-1)
        lon = np.ascontiguousarray(lon, dtype=np.float64).reshape(-1)
        if lat.shape != lon.shape:
            raise ValueError(f"{lat.size} latitudes and {lon.size} longitudes: one of each per site")
        L = self._L = _ffi.lib()
        h = C.c_void_p()
        _ffi.check(L.sky_sites_create(C.byref(h), lat.ctypes.data_as(C.POINTER(C.c_double)),
                                      lon.ctypes.data_as(C.POINTER(C.c_double)), lat.size, int(nlat), int(nlon),
                                      SITES_METHODS[method], int(device)), "sky_sites_create", L)
        self._h = h
        self.n_sites, self.nlat, self.nlon, self.method, self.device = lat.size, int(nlat), int(nlon), method, int(device)

    def close(self):
        if getattr(self, "_h", None):
            self._L.sky_sites_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def sample_sites(x, table: SiteTable, channels=None, channel_offset: int = 0, out=None):
    """The members of a CUDA fp32 (M, C, H, W) tensor, or a view of one whose members each hold contiguous (C, H, W)
    planes, sampled at the sites of ``table`` (include/skyrim_b200.h sky_sample_sites).  Channels are counted from
    ``channel_offset`` (a GraphCast state samples its new time slice with offset 83); ``channels`` lists the sampled ones
    (default: all).  Returns CUDA fp32 (M, n_sel, 1, n_sites), into ``out`` when given: ``ensemble_statistics`` of it gives
    the site statistics.  Asynchronous on the current stream."""
    import torch
    M, H, W, count, member_stride, base, sel = _verified_members(x, channels, channel_offset)
    if (H, W) != (table.nlat, table.nlon):
        raise ValueError(f"x's grid {H} x {W} is not the site table's {table.nlat} x {table.nlon}")
    shape = (M, len(sel), 1, table.n_sites)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=x.device)
    _check_out(out, shape, torch.float32, "out")
    L = _ffi.lib()
    st = torch.cuda.current_stream(x.device).cuda_stream
    _ffi.check(L.sky_sample_sites(table._h, base, M, member_stride, count, _c_array(C.c_int32, sel), len(sel),
                                  out.data_ptr(), st), "sky_sample_sites", L)
    return out


def site_scores(values, obs, acc, out=None):
    """Adds the site terms 1, e, e^2, sum_m (x_m - x_bar)^2, mae and G of ``values`` (CUDA fp32 (M, n_sel, 1, n_sites), from
    ``sample_sites``) against ``obs`` (CUDA fp32 (n_sel, n_sites), NaN where missing) to ``acc`` (CUDA fp64 (n_sel,
    n_sites, 6)), and returns the sums of the terms over the sites with an observation, CUDA fp64 (n_sel, 6), into ``out``
    when given (include/skyrim_b200.h sky_site_scores).  Asynchronous on the current stream."""
    import torch
    if not (values.is_cuda and values.dtype == torch.float32 and values.is_contiguous() and values.dim() == 4
            and values.shape[2] == 1):
        raise ValueError("values must be a contiguous CUDA fp32 (members, n_sel, 1, n_sites) tensor")
    M, n_sel, _, n = values.shape
    _check_out(obs, (n_sel, n), torch.float32, "obs")
    _check_out(acc, (n_sel, n, SITE_TERMS), torch.float64, "acc")
    if out is None:
        out = torch.empty((n_sel, SITE_TERMS), dtype=torch.float64, device=values.device)
    _check_out(out, (n_sel, SITE_TERMS), torch.float64, "out")
    ws = torch.empty(n_sel * SITE_TERMS * ((n + SITES_THREADS - 1) // SITES_THREADS), dtype=torch.float64,
                     device=values.device)
    L = _ffi.lib()
    st = torch.cuda.current_stream(values.device).cuda_stream
    _ffi.check(L.sky_site_scores(values.data_ptr(), M, n_sel, n, obs.data_ptr(), acc.data_ptr(), ws.data_ptr(),
                                 8 * ws.numel(), out.data_ptr(), st), "sky_site_scores", L)
    return out


def unix_seconds(when) -> float:
    """datetime (naive = UTC) / numpy datetime64 / number -> unix seconds"""
    import datetime as _dt
    if isinstance(when, (int, float)):
        return float(when)
    if isinstance(when, np.datetime64):
        return float((when - np.datetime64("1970-01-01T00:00:00")) / np.timedelta64(1, "s"))
    if isinstance(when, _dt.datetime):
        if when.tzinfo is None:
            when = when.replace(tzinfo=_dt.timezone.utc)
        return when.timestamp()
    raise TypeError(type(when))


def launch_count() -> int:
    return int(_ffi.lib().sky_launch_count())
