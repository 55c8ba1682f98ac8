"""Pangu's patch embedding element by element against float64 (oracle/pangu_embed_ref.py).

The two embedding GEMMs run on k_gemm2 under SchedProd: producer warps gather, normalise and round the state into the A
tiles, and EpiStoreF32 adds the bias and writes each token at its member and level.  After debug_set("stop_after", 0) the
test reads the skip image (and, in fp32_stream mode, the fp32 token rows) and checks every element against the reference
built from the same fp16 A and W.  Every grid has a partial last row tile in both GEMMs, with one and with three members.
The workspace starts as 0xFF bytes (an fp16 NaN): the rows past the last token in the skip image's last tile keep them,
and so do the fp32 token rows in the default stream mode, which keeps the tokens only as their fp16 image."""
import numpy as np
import pytest

from oracle import gemm_ref as gr
from oracle import pangu_embed_ref as pe
from oracle import pangu_resample_ref as pr

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

GRIDS = [(41, 96), (33, 96), (45, 192), (24, 96)]   # those of tests/test_pangu_gpu.py


@pytest.fixture(scope="module", params=GRIDS, ids=lambda g: f"{g[0]}x{g[1]}")
def engine(request):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from skyrim_b200.config import pangu_small
    from skyrim_b200.engine import StepEngine
    from skyrim_b200.weights import make_pangu_weights
    cfg = pangu_small(*request.param)
    w = make_pangu_weights(cfg, 1)
    eng = StepEngine(cfg, 0)
    eng.load_weights(w)
    yield cfg, w, eng
    eng.close()


@pytest.mark.parametrize("stream", ["fp16", "fp32"])
@pytest.mark.parametrize("B", [1, 3])
def test_embedding_per_element(engine, B, stream):
    from skyrim_b200.config import PANGU_CHANNELS
    from skyrim_b200.weights import synthetic_state
    cfg, w, eng = engine
    C, HW, nzt = cfg.dim, cfg.H * cfg.W, cfg.Z - 1
    R1 = B * cfg.Z * HW
    assert (B * nzt * HW) % 128 and (B * HW) % 128, "a partial last row tile in both GEMMs"
    x = np.stack([synthetic_state(PANGU_CHANNELS, cfg.nlat, cfg.nlon, 3 + m) for m in range(B)])
    eng.debug_set("fp32_stream", int(stream == "fp32"))
    eng.debug_set("stop_after", 0)
    ws = eng._workspace(B)
    ws.fill_(0xFF)
    eng.step(torch.from_numpy(x).cuda())
    got = {"skip_h": eng.debug_tensor("skip_h", (R1, C), B).cpu().numpy()}
    if stream == "fp32":
        got["tokens1"] = eng.debug_tensor("tokens1", (R1, C), B).cpu().numpy()
    raw = ws.cpu().numpy()

    ref, bound = pe.embed_reference(cfg, w, x)
    bounds = {"skip_h": gr.f16_bound(ref, bound), "tokens1": bound}
    for name, g in got.items():
        bad = gr.exceed(g, ref, bounds[name])
        print(f"{cfg.nlat}x{cfg.nlon} B={B} {stream} stream, {name}: largest |error| / bound {gr.worst(g, ref, bounds[name]):.3f}")
        assert not bad.any(), (name, int(bad.sum()), np.argwhere(bad)[:4].tolist())

    tiles = -(-R1 // 128)
    assert eng._L.sky_model_workspace_bytes(eng._h, B) == pr.workspace_layout(cfg, B)["total"]
    off = pe.skip_image_offset(cfg, B)
    img = raw[off: off + tiles * (C // 64) * 128 * 128].reshape(tiles, C // 64, 128, 128)
    assert (img[-1, :, R1 - (tiles - 1) * 128:] == 0xFF).all(), "skip image rows past the last token written"
    if stream == "fp16":
        assert (raw[: R1 * C * 4] == 0xFF).all(), "fp32 token rows written in the image-only stream mode"
