"""Which Pangu operator runs when: the one module that knows the 6-h / 24-h hierarchy.

Pangu-Weather ships a 6-h and a 24-h operator.  earth2mip's ``PanguInference`` interleaves them ("hierarchical temporal
aggregation" in the Pangu paper), anchored at the rollout's starting state x0:

    yield x0; loop: a = P24(a); 3 x (c = P6(c); yield c); c = a; yield a

so the slice at 24 d + 6 k hours (0 <= k < 4) is P6^k(P24^d(x0)).  The "6h" schedule is the plain chain P6^n(x0).

A plan lists the forwards as (operator, source buffer, destination buffer) over four fixed device buffers, anchors
``A0`` / ``A1`` (day d's anchor lives in A[d % 2]; x0 starts in A0) and chain states ``C0`` / ``C1``, and the slices as
(n, buffer, after): slice n is complete in ``buffer`` once the first ``after`` forwards have run.  The buffers are fixed
so that the 6-h operator sees at most four (source, destination) pairs and the 24-h one two, which the engine's
per-handle CUDA-graph cache (eight entries) replays.  Two properties the TimeLoop and the ensemble runner rely on, checked by the tests:

  * a slice's buffer is not written by the forwards that complete the next slice (a host copy of slice n may run under
    them), and
  * in a last-slices plan, both slices are still in their buffers after the last forward.
"""
from __future__ import annotations

import itertools
from dataclasses import dataclass

SCHEDULES = ("6h", "hierarchical")
A0, A1, C0, C1 = 0, 1, 2, 3
N_BUFFERS = 4
_A, _C = (A0, A1), (C0, C1)


@dataclass(frozen=True)
class Plan:
    forwards: tuple   # ((op, src, dst), ...), op "6h" or "24h"
    slices: tuple     # ((n, buffer, after), ...) in increasing n


def check_schedule(schedule: str) -> str:
    if schedule not in SCHEDULES:
        raise ValueError(f"unknown Pangu schedule {schedule!r} (one of {SCHEDULES})")
    return schedule


def iter_slices(schedule: str):
    """Every slice, without end: yields (n, buffer, forwards that complete slice n) for n = 1, 2, ..."""
    check_schedule(schedule)
    for n in itertools.count(1):
        if schedule == "6h":   # the chain, ping-ponged between the two anchors
            src, dst = _A[(n - 1) % 2], _A[n % 2]
            yield n, dst, (("6h", src, dst),)
            continue
        d, k = divmod(n, 4)
        if k == 0:   # the day boundary: P24 of yesterday's anchor
            src, dst = _A[(d - 1) % 2], _A[d % 2]
            yield n, dst, (("24h", src, dst),)
        else:
            src, dst = (_A[d % 2] if k == 1 else _C[k % 2]), _C[(k - 1) % 2]
            yield n, dst, (("6h", src, dst),)


def plan(schedule: str, n_steps: int, every_slice: bool = True) -> Plan:
    """The forwards of an ``n_steps``-step rollout.  ``every_slice``: slices 0 .. n_steps in order; otherwise only slices
    n_steps - 1 and n_steps (the two a rollout returns; slice 0 alone for n_steps = 0) with the fewest forwards:
    d + k for a lead of 24 d + 6 k hours with k > 0, d + 3 for k = 0 < d."""
    check_schedule(schedule)
    if n_steps < 0:
        raise ValueError(f"n_steps = {n_steps} must not be negative")
    if every_slice or schedule == "6h" or n_steps == 0:
        fw, sl = [], [(0, A0, 0)]
        for n, buf, f in itertools.islice(iter_slices(schedule), n_steps):
            fw += f
            sl.append((n, buf, len(fw)))
        if not every_slice:
            sl = sl[-2:]
        return Plan(tuple(fw), tuple(sl))
    d, k = divmod(n_steps, 4)
    days = d if k else d - 1   # anchor the 6-h chain starts from
    fw = [("24h", _A[j % 2], _A[(j + 1) % 2]) for j in range(days)]
    chain = [_A[days % 2]]
    for j in range(k if k else 3):
        fw.append(("6h", chain[-1], _C[j % 2]))
        chain.append(_C[j % 2])
    if k:
        sl = ((n_steps - 1, chain[-2], len(fw) - 1), (n_steps, chain[-1], len(fw)))
    else:   # slice n - 1 closes yesterday's chain, slice n is today's anchor
        fw.append(("24h", _A[days % 2], _A[d % 2]))
        sl = ((n_steps - 1, chain[-1], len(fw) - 1), (n_steps, _A[d % 2], len(fw)))
    return Plan(tuple(fw), sl)
