"""Perturbed-initial-condition ensembles sharded over GPUs (SURVEY.md §8(e); new functionality —
the reference only has a sequential multi-model mean, models/ensemble.py:86-101).

One process per GPU.  Members are independent trajectories: member m lives on rank m // M
(M members per GPU, stacked along the batch of every kernel so weights and tables are read once
per step).  The only collective of the whole run is ONE broadcast of the fp32 weight arena at
init; optional mean / spread reductions happen after the step loop.
"""
from __future__ import annotations

import numpy as np


def member_range(rank: int, members_per_gpu: int):
    """global member indices owned by ``rank``"""
    return range(rank * members_per_gpu, (rank + 1) * members_per_gpu)


def broadcast_arena(weights, shapes, device, rank: int, world: int):
    """Rank 0 packs the named fp32 tensors; every rank returns (arena tensor on ``device``,
    manifest).  ``weights`` may be None on ranks != 0; ``shapes`` (name -> shape) must be known
    everywhere (it follows from the config)."""
    import torch
    import torch.distributed as dist
    from .engine import pack_arena
    if rank == 0:
        arena_h, manifest = pack_arena(weights)
        arena = torch.from_numpy(arena_h).to(device)
    else:
        arena_h, manifest = pack_arena({k: np.zeros(s, np.float32) for k, s in shapes.items()})
        arena = torch.empty(arena_h.size, dtype=torch.float32, device=device)
    if world > 1:
        dist.broadcast(arena, 0)
    return arena, manifest


class EnsembleRunner:
    """Per-rank driver: M members resident on this GPU, chained device-resident steps."""

    def __init__(self, engine, base_state, sigma_c, members_per_gpu: int, rank: int = 0, amp: float = 0.05,
                 seed: int = 0, perturbation: str = "gaussian", grf: dict | None = None):
        """``perturbation``: "gaussian" adds independent N(0, 1) amp sigma_c noise at every grid point (K11);
        "spherical_grf" adds amp sigma_c times a spherical Gaussian random field of unit pointwise variance,
        ``grf`` = keyword arguments of ``engine.perturb_ic_grf`` (alpha, tau, lmax); "none" leaves every member equal to
        ``base_state`` (one member is then the model's own unperturbed trajectory)."""
        import torch
        if perturbation not in ("gaussian", "spherical_grf", "none"):
            raise ValueError(f"unknown perturbation {perturbation!r} (gaussian, spherical_grf, none)")
        if grf and perturbation != "spherical_grf":
            raise ValueError("grf options need perturbation='spherical_grf'")
        self.engine, self.M, self.rank = engine, members_per_gpu, rank
        self.amp, self.perturbation, self.grf = amp, perturbation, grf
        dev = torch.device("cuda", engine.device)
        x = torch.as_tensor(base_state, dtype=torch.float32)[None].repeat(self.M, 1, 1, 1).to(dev).contiguous()
        self.sigma = torch.as_tensor(sigma_c, dtype=torch.float32, device=dev)
        self._perturb(x, seed)
        self.x, self.y = x, torch.empty_like(x)
        self.steps = 0

    def _perturb(self, x, seed: int):
        from .engine import perturb_ic, perturb_ic_grf
        # Philox keyed by the GLOBAL member id
        if self.perturbation == "gaussian":
            perturb_ic(x, self.sigma, self.amp, seed=seed, member0=self.rank * self.M)
        elif self.perturbation == "spherical_grf":
            perturb_ic_grf(x, self.sigma, self.amp, seed=seed, member0=self.rank * self.M, **(self.grf or {}))

    def restart(self, base_state, seed: int):
        """Starts a new forecast in the existing member tensors: every member becomes ``base_state`` perturbed with
        ``seed`` (the perturbation, amplitude and options of the constructor), bit for bit the members a new runner
        built with ``seed`` would hold.  A verification campaign restarts one runner for each start date."""
        import torch
        self.x[0].copy_(torch.as_tensor(base_state, dtype=torch.float32))
        if self.M > 1:
            self.x[1:].copy_(self.x[:1].expand(self.M - 1, *self.x.shape[1:]))
        self._perturb(self.x, seed)
        self.steps = 0

    def step(self, n: int = 1):
        for _ in range(n):
            self.engine.step(self.x, self.y)
            self.x, self.y = self.y, self.x
        self.steps += n
        return self.x

    def mean_and_spread(self, world: int = 1):
        """ensemble mean / standard deviation over ALL members (two all-reduces, outside the step loop)"""
        return mean_and_spread(self.x, world)

    def _walk(self, n_steps: int, every_slice: bool = True):
        """Yields (n, members) for the current state (n = 0) and after each of ``n_steps`` steps; the forwards of lead n
        are launched when the walk is asked for it.  ``members`` stays valid until the second next() after it.  The plain
        chain has every slice; only the hierarchical schedule reads ``every_slice``."""
        yield 0, self.x
        for n in range(1, n_steps + 1):
            yield n, self.step()

    def iter_stats(self, n_steps: int, channels=None, quantiles=(), events=(), channel_offset: int = 0):
        """Steps ``n_steps`` times and yields (n, stats, prob) for the current state (n = 0) and after each step:
        ``engine.ensemble_statistics`` of this rank's members, as pinned host tensors.  Only the statistics leave the
        device, and the device->host copy of step n runs on a copy stream while step n + 1 computes (the event pattern of
        ``timeloop._EngineTimeLoop.iter_host``, with rings of two statistics buffers on the device and on the host).  A
        yielded pair is valid until the second next() after it."""
        from .engine import ensemble_statistics
        return self._iter_on_host(self._walk(n_steps), lambda members, out=None: ensemble_statistics(
            members, channels, quantiles, events, channel_offset, out=out))

    def iter_sites(self, n_steps: int, table, channels=None, quantiles=(), events=(), channel_offset: int = 0):
        """``iter_stats`` at the sites of ``table`` (``engine.SiteTable``): yields (n, values) with one member, (n, values,
        stats, prob) with more, as pinned host tensors: ``engine.sample_sites`` of this rank's members, (M, n_sel, 1,
        n_sites), and ``engine.ensemble_statistics`` of those values, events (i, threshold) about ``channels[i]``.  Every
        slice of the walk is sampled; each slice's copy runs under the next slice's forwards."""
        from .engine import ensemble_statistics, sample_sites

        def reduce(members, out=None):
            v = sample_sites(members, table, channels, channel_offset, out=None if out is None else out[0])
            if members.shape[0] == 1:
                return (v,)
            return (v,) + ensemble_statistics(v, None, quantiles, events, out=None if out is None else out[1:])
        return self._iter_on_host(self._walk(n_steps, every_slice=True), reduce)

    def _iter_on_host(self, walk, reduce):
        """Yields (n,) + the host copies of ``reduce(members)`` (a tuple of CUDA tensors) for every (n, members) of
        ``walk``, each slice's device->host copy on a copy stream under the next slice's forwards and reduction
        (``reduce(members, out=)`` writes into a ring of two device tuples; the pinned host tuples are a ring of two)."""
        import torch
        dev = self.x.device
        main = torch.cuda.current_stream(dev)
        copy = torch.cuda.Stream(dev)
        cur = next(walk)
        ring = [reduce(cur[1])]
        ring.append(tuple(torch.empty_like(t) for t in ring[0]))
        host = [tuple(torch.empty(t.shape, dtype=t.dtype).pin_memory() for t in ring[0]) for _ in range(2)]
        done = [torch.cuda.Event() for _ in range(2)]    # reduction i % 2 is complete on the main stream
        copied = torch.cuda.Event()
        done[0].record(main)
        i = 0
        while cur is not None:
            nxt = next(walk, None)
            if nxt is not None:   # launch the next slice's forwards and reduction before waiting for the copy of this one
                reduce(nxt[1], out=ring[(i + 1) % 2])
                done[(i + 1) % 2].record(main)
            copy.wait_event(done[i % 2])
            with torch.cuda.stream(copy):
                for h, d in zip(host[i % 2], ring[i % 2]):
                    h.copy_(d, non_blocking=True)
                copied.record(copy)
            copied.synchronize()   # also orders the next reduction into ring[i % 2] (launched at i + 1) after this copy
            yield (cur[0],) + host[i % 2]
            cur, i = nxt, i + 1

    def truth_ring(self, n_sel: int):
        """``truth_ring`` for ``n_sel`` channels on this runner's device and grid.  Pinning dominates the set-up of a
        scoring call, so a campaign over many start dates makes one ring and passes it to every call."""
        return truth_ring(self.x.device, n_sel, *self.x.shape[-2:])

    def iter_scores(self, n_steps: int, truth_at, clim=None, channels=None, row_weights=None, channel_offset: int = 0,
                    hist=None, seed: int = 0, date_index: int = 0, maps=None, map_slot=None, map_channels=(), sums=None,
                    ring=None):
        """Steps ``n_steps`` times and scores this rank's members at every lead n = 0 .. n_steps against
        ``truth_at(n)`` (host fp32 (n_sel, H, W) of the selected channels), with the static climatology ``clim`` (host
        fp32 (n_sel, H, W) or None) and the regions of ``row_weights`` (fp64 (n_regions, H)): ``engine.forecast_scores``.
        Per lead the forwards are launched first and the truth is fetched on the host while they run, then uploaded by
        ``upload_truth``.  Every lead's sums stay in one device tensor that crosses to the host
        once, at the end.  Returns (leads, fp64 host tensor (n_leads, n_regions, n_sel, 9)).

        Off the same uploaded truth, optionally: ``hist`` (CUDA fp64 (n_leads, n_regions, n_sel, M + 1)) receives each
        lead's ``engine.forecast_rank_histogram`` with key (``seed``, ``date_index``) and lead index n; ``maps`` (CUDA fp64
        (n_slots, len(map_channels), 5, H, W)) accumulates ``engine.score_maps_accumulate`` of the channels at positions
        ``map_channels`` of ``channels`` at each lead n in ``map_slot`` (dict lead -> slot).  ``sums`` (CUDA fp64
        (n_leads, n_regions, n_sel, 9)) receives the sums, and is returned on the device instead of a host copy; ``ring``
        (``truth_ring``) replaces the truth buffers this call would allocate."""
        import torch
        from .engine import forecast_rank_histogram, forecast_scores, score_maps_accumulate
        dev = self.x.device
        main = torch.cuda.current_stream(dev)
        n_sel = self.x.shape[1] - channel_offset if channels is None else len(channels)
        sel = list(range(n_sel)) if channels is None else list(channels)
        rw = torch.as_tensor(np.asarray(row_weights, dtype=np.float64), device=dev).contiguous()
        kd = None if clim is None else torch.from_numpy(np.ascontiguousarray(clim, dtype=np.float32)).to(dev)
        out = sums if sums is not None else torch.empty((n_steps + 1, rw.shape[0], n_sel, 9), dtype=torch.float64,
                                                        device=dev)
        ring = ring or self.truth_ring(n_sel)
        map_slot = map_slot or {}
        leads = []
        for i, (n, members) in enumerate(self._walk(n_steps, every_slice=True)):
            y = upload_truth(ring, i, truth_at(n), main)   # the host fetch runs under the forwards just launched
            forecast_scores(members, y, rw, channels, kd, channel_offset, out=out[i])
            if hist is not None:
                forecast_rank_histogram(members, y, rw, seed, date_index, n, channels, channel_offset, out=hist[i])
            if n in map_slot:
                for j, k in enumerate(map_channels):       # one plane of the truth per map channel
                    score_maps_accumulate(members, y[k:k + 1], maps[map_slot[n], j:j + 1], [sel[k]], channel_offset)
            ring["scored"][i % 2].record(main)
            leads.append(n)
        return leads, (out if sums is not None else out.cpu())


def truth_ring(device, n_sel: int, H: int, W: int):
    """the truth buffers of a scoring loop for ``n_sel`` channels: a copy stream and two device and two pinned host
    (n_sel, H, W) fp32 buffers with their events (``upload_truth``)"""
    import torch
    return dict(copy=torch.cuda.Stream(device),
                dbuf=[torch.empty((n_sel, H, W), dtype=torch.float32, device=device) for _ in range(2)],
                hbuf=[torch.empty((n_sel, H, W), dtype=torch.float32).pin_memory() for _ in range(2)],
                uploaded=[torch.cuda.Event() for _ in range(2)],   # truth i % 2 is on the device
                scored=[torch.cuda.Event() for _ in range(2)])     # the work that read dbuf[i % 2] is done


def upload_truth(ring, i: int, y, main):
    """Uploads lead i's host truth ``y`` (fp32 (n_sel, H, W)) into ``ring`` (``truth_ring``) and returns its device buffer,
    which the work queued next on ``main`` may read.  The upload runs on the ring's copy stream through the pinned buffer
    i % 2: it waits on the host until lead i - 2's upload has left that buffer and, on the copy stream, until the work that
    read lead i - 2's device buffer is done; ``main`` waits for the upload.  The caller records ``ring["scored"][i % 2]``
    on ``main`` after the last work that reads the buffer."""
    import torch
    copy, dbuf, hbuf, uploaded, scored = (ring[k] for k in ("copy", "dbuf", "hbuf", "uploaded", "scored"))
    uploaded[i % 2].synchronize()                   # lead i - 2's upload has left hbuf[i % 2]
    np.copyto(hbuf[i % 2].numpy(), y)
    copy.wait_event(scored[i % 2])                  # lead i - 2's scoring has read dbuf[i % 2]
    with torch.cuda.stream(copy):
        dbuf[i % 2].copy_(hbuf[i % 2], non_blocking=True)
        uploaded[i % 2].record(copy)
    main.wait_event(uploaded[i % 2])
    return dbuf[i % 2]


class HierarchicalEnsembleRunner(EnsembleRunner):
    """``EnsembleRunner`` on Pangu's hierarchical schedule (schedule.py): ``engine`` is the 6-h handle, ``engine_24`` the
    24-h one on its workspace, both batched over the M members, whose anchor states sit beside their chain states in the
    plan's four buffers.  Without ``every_slice``, ``iter_stats`` yields only steps n_steps - 1 and n_steps, reached with
    the fewest forwards; ``iter_scores`` always scores every slice.  The members are perturbed exactly as
    ``EnsembleRunner`` perturbs them."""

    def __init__(self, engine, *args, engine_24, every_slice: bool = True, **kw):
        super().__init__(engine, *args, **kw)
        self.engine_24, self.every_slice = engine_24, every_slice

    def step(self, n: int = 1):
        raise NotImplementedError("a hierarchical ensemble steps through iter_stats / iter_scores, which follow the "
                                  "schedule")

    def _walk(self, n_steps: int, every_slice: bool | None = None):
        """the plan's forward walk: yields (n, buffer of slice n) once the forwards completing slice n are launched"""
        import torch
        from . import schedule
        p = schedule.plan("hierarchical", n_steps, self.every_slice if every_slice is None else every_slice)
        if getattr(self, "_spare", None) is None:   # the plan's other buffers, kept for the next walk
            self._spare = [torch.empty_like(self.x) for _ in range(schedule.N_BUFFERS - 2)]
        bufs = [self.x, self.y] + self._spare
        engines = {"6h": self.engine, "24h": self.engine_24}
        issued = 0
        for n, buf, after in p.slices:   # none for slice 0; a last-slices plan may need many before its first slice
            for op, src, dst in p.forwards[issued:after]:
                engines[op].step(bufs[src], bufs[dst])
            issued = after
            yield n, bufs[buf]
        last = p.slices[-1][1]
        self.x, self.y = bufs[last], bufs[schedule.A1 if last == schedule.A0 else schedule.A0]
        self._spare = [b for b in bufs if b is not self.x and b is not self.y]
        self.steps += n_steps


def mean_and_spread(x, world: int = 1):
    """x: this rank's members (M, C, H, W).  Two-pass: the mean is reduced first, then the sum of squared DEVIATIONS —
    E[x^2] - mean^2 in fp32 cancels catastrophically on de-normalised fields (z ~ 5e4, t ~ 280 with a spread of a few
    units), and clamping hid the negative variances it produced."""
    import torch
    import torch.distributed as dist
    n = world * x.shape[0]
    s = x.sum(0, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(s)
    mean = (s / n).to(x.dtype)
    ss = ((x - mean) ** 2).sum(0, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(ss)
    return mean, (ss / n).sqrt().to(x.dtype)
