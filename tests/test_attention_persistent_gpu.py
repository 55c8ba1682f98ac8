"""The persistent window-attention kernel (k_window_attention_tc) at chosen grid sizes.

CTA c of a G-CTA grid walks items [c items / G, (c+1) items / G) through a two-slot ring of q / k / v tiles and keeps a
bias slice per (window type, head pair) that it rebuilds when the type or pair changes.  The output must not depend on
G: each case launches the ATTENTION op through sky_probe_pangu_grid with one CTA per SM (0), one CTA, seven CTAs and
more CTAs than items, and requires the four outputs to be bitwise equal.  One CTA walks every item, so the ring wraps
many times and every (type, pair) run is entered; with seven CTAs most ranges start in the middle of a run.  Coverage
and sentinels are checked as in tests/test_pangu_kernels_gpu.py; on the small grids the values are also checked against
oracle/pangu_kernels_ref.attention_tokens.  The full-size g2 grid (5,760 items per member) is fed a random window image.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from oracle import gemm_probe as gp
from oracle import gemm_ref as gr
from oracle import pangu_kernels_ref as pk
from test_pangu_kernels_gpu import FULL, SEED, SMALL, Guarded, att_bytes, attention_case, check_att_coverage, dev, record, \
    window_geometry

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu


def launch_grid(case, grid_ctas: int):
    L = gp.lib()
    L.sky_probe_pangu_grid.restype = C.c_int
    L.sky_probe_pangu_grid.argtypes = [C.POINTER(gp.PanguCase), C.c_int32, C.c_void_p]
    rc = L.sky_probe_pangu_grid(C.byref(case), grid_ctas, None)
    assert rc == 0, (L.sky_last_error() or b"").decode()
    torch.cuda.synchronize()


def run_all_grids(g, roll, B, qkv_ptr, ps, img_bytes, tab_dev):
    """the ATTENTION op at every grid size; returns the one-CTA-per-SM output after asserting all are bitwise equal"""
    items = B * g.nWin * g.pairs
    outs = {}
    for grid in (0, 1, 7, items + 5):
        out = Guarded(att_bytes(g, B))
        launch_grid(attention_case(g, roll, B, qkv_ptr, ps, img_bytes, tab_dev, out), grid)
        check_att_coverage(out, g, B, f"attention output, {grid} CTAs")
        outs[grid] = out
    for grid, out in outs.items():
        assert torch.equal(out.t, outs[0].t), f"{grid} CTAs: output differs from one CTA per SM"
    return outs[0]


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("roll", [0, 1])
@pytest.mark.parametrize("name", ["41x96-g1", "41x96-g2", "45x192-g1"])
def test_attention_grids_small(name, roll, B):
    g = SMALL[name]
    inp = pk.attention_inputs(g, B, SEED, False)
    _, ps, img_bytes = window_geometry(g, roll, B)
    idx = pk.window_tokens(g, roll, B)
    img = pk.pack_window_image(pk.windows_from_tokens(inp.qkv_tok, inp.pad_row, idx, g.heads), ps)
    qkv_dev, tab_dev = dev(img), dev(pk.pack_bias_table(inp.table))
    out = run_all_grids(g, roll, B, qkv_dev[1], ps, img_bytes, tab_dev)
    got = gr.unpack_tiles(out.inner().cpu().numpy().view(np.uint8), 128, g.C // 64, B * g.T, g.C)
    ref, bnd = pk.attention_tokens(g, B, roll, inp)
    record(f"persistent attention {name} roll {roll} B {B}", got, ref, bnd)


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("roll", [0, 1])
def test_attention_grids_fullsize(roll, B):
    g = FULL["721x1440-g2"]
    _, ps, img_bytes = window_geometry(g, roll, B)
    gen = torch.Generator(device="cuda").manual_seed(11 + 2 * B + roll)
    # q, k, v uniform in [-2, 2) (scores span several units); every row of every tile is a finite value
    img = ((torch.rand(img_bytes // 2, generator=gen, device="cuda") * 4 - 2).half()).view(torch.int16)
    table = np.random.default_rng(3 + B).uniform(-2, 2, (pk.TABLE, g.n_type, g.heads)).astype(np.float32)
    tab_dev = dev(pk.pack_bias_table(table))
    run_all_grids(g, roll, B, img.data_ptr(), ps, img_bytes, tab_dev)
