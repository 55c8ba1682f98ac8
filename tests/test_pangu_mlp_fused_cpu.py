"""CPU checks of Pangu's fused MLP (mlp_fused.cuh) at C = 192 and, for the compiler report and the probe, C = 384: the chunk plan its loader relies on, what
ptxas made of it, and that the probe refuses inconsistent fused cases on the host (without touching a device)."""
from __future__ import annotations

import re
from pathlib import Path

import numpy as np
import pytest

from oracle import gemm_probe as gp
from oracle import gemm_ref as gr

C, NKB = 192, 3
MLP = 4   # sky_probe_gemm kernel id of the fused MLP (gemm_probe.cu SKY_PROBE_MLP)
CSRC = Path(__file__).resolve().parent.parent / "skyrim_b200" / "csrc"


def test_chunk_plan():
    """the loader copies W1's chunk j as the one contiguous 24 KB run at j * 24 KB of the BLOCK_N 64 image, and W2's
    k-block j as the 24 KB run at j * 24 KB of the BLOCK_N 192 image: those runs hold exactly W1 rows 64j .. 64j + 63 over
    all of K = C, and W2 columns 64j .. 64j + 63 of all C rows"""
    rng = np.random.default_rng(0)
    w1 = rng.standard_normal((4 * C, C)).astype(np.float16)
    w2 = rng.standard_normal((C, 4 * C)).astype(np.float16)
    img1, img2 = gr.pack_w(w1, 64, NKB), gr.pack_w(w2, 192, 4 * NKB)
    run = NKB * 64 * 128
    assert img1.size == img2.size == 4 * NKB * run
    for j in range(4 * NKB):
        sl = img1[j * run:(j + 1) * run]
        assert np.array_equal(sl, gr.pack_w(np.ascontiguousarray(w1[64 * j:64 * j + 64]), 64, NKB))
        kb = img2[j * run:(j + 1) * run]
        assert np.array_equal(kb, gr.pack_w(np.ascontiguousarray(w2[:, 64 * j:64 * j + 64]), 192, 1))


def test_ptxas_report():
    """no spills (a few in the pair kernel), and a register count that lets 288 threads (two consumer warpgroups and the
    loader) run"""
    log = CSRC / "pangu_engine.ptxas.log"
    if not log.exists():
        pytest.skip("library not built (build() writes the ptxas report next to the objects)")
    text = log.read_text()
    for name in ("_ZN3sky11k_mlp_fusedILi3EEEvNS_7MlpArgsE", "_ZN3sky16k_mlp_fused_pairILi6EEEvNS_7MlpArgsE"):
        m = re.search(r"Function properties for " + name + r"\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                      r"(\d+) bytes spill loads\s*\n.*?Used (\d+) registers", text)
        assert m, f"{name} not in the ptxas report"
        stack, st, ld, regs = map(int, m.groups())
        # the pair kernel spills about 20 loop-invariant values: at most 96 bytes
        limit = 0 if "pair" not in name else 96
        assert stack <= limit and st <= limit and ld <= limit, (name, stack, st, ld)
        assert regs <= 168, (name, regs)   # three of the nine warps share a sub-partition's 16K registers


def _good_case(**over):
    kw = dict(kernel=MLP, block_n=192, n=C, n_valid=C, batches=1, m=300, hi=0x10000, img_bytes=3 * NKB * 16384, img_nkb=NKB,
              w=0x100000, w_bytes=4 * C * C * 2, b_hi=0x200000, b_bytes=4 * C * C * 2, add=0x300000, add_bytes=4 * C * 4,
              bias=0x400000, gamma=0x410000, beta=0x420000, vec_floats=C, eps=1e-5)
    kw.update(over)
    return gp.make_case(**kw)


@pytest.mark.parametrize("over,msg", [
    (dict(n=256), "N=256"),
    (dict(add=0x300008), "fc1 bias"),
    (dict(n=384, grid_sms=1), "CTA pairs"),
    (dict(img_nkb=6), "stream image"),
    (dict(img_bytes=2 * NKB * 16384), "stream image"),
    (dict(b_hi=0), "weight images"),
    (dict(w_bytes=4 * C * C), "weight images"),
    (dict(add_bytes=C * 4), "fc1 bias"),
    (dict(vec_floats=C - 1), "bias: null, misaligned or shorter"),
    (dict(grid_sms=-1), "grid_sms"),
])
def test_probe_refuses_inconsistent_fused_cases(over, msg):
    try:
        gp.lib()
    except (RuntimeError, OSError) as e:
        pytest.skip(f"probe library not loadable: {e}")
    rc, err = gp.launch(_good_case(**over))
    assert rc != 0 and msg in err, (rc, err)
