"""CPU check of the patch-embedding reference (oracle/pangu_embed_ref.py) that tests/test_pangu_embed_gpu.py compares the
engine against: its token layout and its A operand are those of the model oracle (PanguRef.patch_embed with fp16 operands),
for every member."""
import numpy as np
import pytest
import torch

from oracle import pangu_embed_ref as pe
from oracle.pangu_ref import PanguRef
from skyrim_b200.config import PANGU_CHANNELS, pangu_small
from skyrim_b200.weights import make_pangu_weights, synthetic_state


@pytest.mark.parametrize("nlat,nlon", [(41, 96), (24, 96)])
def test_embed_reference_matches_model_oracle(nlat, nlon):
    cfg = pangu_small(nlat, nlon)
    w = make_pangu_weights(cfg, 1)
    x = np.stack([synthetic_state(PANGU_CHANNELS, nlat, nlon, s) for s in (3, 4)])
    ref, bound = pe.embed_reference(cfg, w, x)
    assert ref.shape == bound.shape == (2 * cfg.Z * cfg.H * cfg.W, cfg.dim)
    oracle = PanguRef(cfg, w, emulate="fp16")
    for m in range(2):
        want = oracle.patch_embed(torch.from_numpy(x[m])).double().numpy().reshape(-1, cfg.dim)
        got = ref.reshape(2, -1, cfg.dim)[m]
        # the oracle divides by std where the engine multiplies by its fp32 reciprocal, so a few fp16 operands differ by one
        # ulp (6e-5 of the largest token value at 41x96); a layout mistake, e.g. two members swapped, is of order 1
        assert np.abs(got - want).max() <= 5e-4 * np.abs(want).max(), m
    assert np.all(bound > 0) and bound.max() < 1e-3 * np.abs(ref).max()
