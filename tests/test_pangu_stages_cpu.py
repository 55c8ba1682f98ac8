"""oracle/pangu_stages_ref.py on the CPU: its units compose to PanguRef's block in float64, each modelled wiring mistake
leaves the bound of the unit it touches, and the unit list follows PanguEngine::run_block_t's dispatch."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

from oracle import gemm_ref as gr  # noqa: E402
from oracle import pangu_kernels_ref as pk  # noqa: E402
from oracle import pangu_stages_ref as ps  # noqa: E402
from oracle.pangu_ref import PanguRef  # noqa: E402
from skyrim_b200.config import pangu_full, pangu_small  # noqa: E402
from skyrim_b200.weights import make_pangu_weights  # noqa: E402


@pytest.fixture(scope="module")
def small():
    cfg = pangu_small(41, 96)
    return cfg, make_pangu_weights(cfg, 1)


@pytest.mark.parametrize("li,bi", [(0, 0), (0, 1), (1, 1), (3, 1)])
def test_units_compose_to_the_block_in_float64(small, li, bi):
    """qkv -> attention -> projection -> fc1 -> fc2 on unrounded weights in float64 = PanguRef(float64).block, two
    members (the second checks the member offsets of the window rows)"""
    cfg, w = small
    g = ps.level(cfg, li)
    rng = np.random.default_rng(li * 10 + bi)
    x = rng.standard_normal((2 * g.T, g.C))
    got = ps.block_ref(cfg, li, bi, 2, x, ps.block_weights(w, li, bi, round16=False))
    ref = PanguRef(cfg, w, dtype=torch.float64)
    want = np.concatenate([ref.block(torch.from_numpy(x[m * g.T:(m + 1) * g.T]).reshape(g.Z, g.H, g.W, g.C),
                                     f"layer{li}.block{bi}.", cfg.heads[li], roll=bi % 2 == 1).reshape(g.T, g.C).numpy()
                           for m in range(2)])
    assert np.abs(got - want).max() <= 1e-11 * np.abs(want).max()


def _emulated_block(cfg, w, li, bi, B, seed):
    """fp16 stream rows, the engine-rounded inputs of every unit of block (li, bi), and the correct references"""
    g = ps.level(cfg, li)
    bw = ps.block_weights(w, li, bi)
    x = np.random.default_rng(seed).uniform(-2, 2, (B * g.T, g.C)).astype(np.float16).astype(np.float64)
    wins = np.arange(B * g.nWin)
    return g, bw, x, wins


def _leaves(knob_ref, ref, bnd):
    return int(gr.exceed(knob_ref, ref, bnd).sum())


@pytest.mark.parametrize("li,bi", [(0, 1), (1, 0), (2, 1)])
def test_each_knob_leaves_the_bound(small, li, bi):
    """every modelled wiring mistake pushes at least one element of the unit it touches past that unit's bound, on the
    synthetic weights of the tests and B = 2"""
    cfg, w = small
    B = 2
    g, bw, x, wins = _emulated_block(cfg, w, li, bi, B, seed=li + bi)
    roll = bi & 1
    counts = {}
    q, qb = ps.qkv_unit(g, B, roll, wins, x, bw)
    counts["qkv: roll of the wrong parity"] = _leaves(ps.qkv_unit(g, B, roll, wins, x, bw, roll_flip=True)[0], q, qb)
    if g.Hp > g.H:
        counts["qkv: padding rows unfilled"] = _leaves(ps.qkv_unit(g, B, roll, wins, x, bw, pad_fill=False)[0], q, qb)
    q16 = q.astype(np.float16)
    tok, a, ab = ps.attention_unit(g, B, roll, wins, q16, bw, cfg.mask_value)
    order = np.argsort(tok)
    a, ab = a[order], ab[order]

    def att(**k):
        t, o, _ = ps.attention_unit(g, B, roll, wins, q16, bw, cfg.mask_value, **k)
        out = np.full_like(a, np.nan)
        out[np.searchsorted(tok[order], t)] = o
        return out
    counts["attention: roll of the wrong parity"] = _leaves(att(roll_flip=True), a, ab)
    other = (li, bi - 1) if bi else ({0: 3, 1: 2, 2: 1, 3: 0}[li], 0)   # another block on the same grid
    counts[f"attention: bias table of block {other}"] = _leaves(att(table=ps.block_weights(w, *other)["table"]), a, ab)
    counts["attention: head pairs 0 and 1 swapped"] = _leaves(att(swap_pairs=True), a, ab)
    a16 = a.astype(np.float16).astype(np.float64)
    x1, x1b = ps.proj_unit(a16, bw, x, cfg.ln_eps, "fp32")
    counts["projection: ln2 instead of ln1"] = _leaves(ps.proj_unit(a16, bw, x, cfg.ln_eps, "fp32", ln="ln2")[0], x1, x1b)
    counts["projection: fp16 stream, residual from the (unwritten) fp32 rows"] = _leaves(
        ps.proj_unit(a16, bw, np.zeros_like(x), cfg.ln_eps, "fp16")[0], x1, gr.f16_bound(x1, x1b))
    x116 = x1.astype(np.float16).astype(np.float64)
    h, hb = ps.fc1_unit(x116, bw)
    h16 = h.astype(np.float16).astype(np.float64)
    y, yb = ps.fc2_unit(h16, bw, x116, cfg.ln_eps, "fp16")
    counts["fc2: ln1 instead of ln2"] = _leaves(ps.fc2_unit(h16, bw, x116, cfg.ln_eps, "fp16", ln="ln1")[0], y, yb)
    if g.C == 192:
        m, mb = ps.mlp_unit(x116, bw, x116, cfg.ln_eps, "fp16")
        assert gr.worst(y, m, mb) <= 1.0, "fc1 + fc2 from the rounded hidden lies inside the fused MLP's bound"
        counts["fused MLP: ln1 instead of ln2"] = _leaves(ps.mlp_unit(x116, bw, x116, cfg.ln_eps, "fp16", ln="ln1")[0], m, mb)
    for k, v in counts.items():
        print(f"layer {li} block {bi}: {k}: {v} elements outside the bound")
    assert all(counts.values()), counts


def test_fp16_stream_residual_from_the_rows_is_caught_in_the_fp32_stream(small):
    """with the fp32 stream the residual is the fp32 rows: the same values rounded to fp16 (the image) leave the bound
    of the fp32 rows"""
    cfg, w = small
    g, bw, _, _ = _emulated_block(cfg, w, 0, 0, 1, seed=4)
    x32 = np.random.default_rng(4).uniform(-2, 2, (g.T, g.C)).astype(np.float32).astype(np.float64)
    a = np.random.default_rng(5).uniform(-1, 1, (g.T, g.C)).astype(np.float16).astype(np.float64)
    y, yb = ps.proj_unit(a, bw, x32, cfg.ln_eps, "fp32")
    assert _leaves(ps.proj_unit(a, bw, x32.astype(np.float16), cfg.ln_eps, "fp32")[0], y, yb)


@pytest.mark.parametrize("cfg", [pangu_small(41, 96), pangu_small(45, 192), pangu_full()], ids=["41x96", "45x192", "full"])
@pytest.mark.parametrize("stream", ["fp16", "fp32"])
def test_unit_list_follows_the_engine_dispatch(cfg, stream):
    """run_block_t: the fused MLP only with the image-only (fp16) stream at C = 192 (layers 0 and 3), fc1 + fc2 with the
    fp32 stream and at C = 384 (layers 1 and 2); a padding fill launch beside QKV where the latitude axis is padded;
    embedding, down-sample and up-sample two launches, recovery one"""
    u = ps.units(cfg, stream)
    g1, g2 = pk.grids(cfg)
    kinds = [k for k, *_ in u]
    assert kinds[0] == "embed" and kinds[-1] == "recover"
    assert kinds.index("down") == 1 + 4 * 2 + (stream == "fp32") * 2 and kinds.count("up") == 1
    for li in range(4):
        g = ps.level(cfg, li)
        for bi in range(cfg.depths[li]):
            mine = [(k, n) for k, l_, b_, n in u if (l_, b_) == (li, bi)]
            mlp = [("mlp", 1)] if stream == "fp16" and li in (0, 3) else [("fc1", 1), ("fc2", 1)]
            assert mine == [("qkv", 1 + (g.Hp > g.H)), ("attn", 1), ("proj", 1)] + mlp
    blocks = sum(cfg.depths)
    mlp_launches = sum(cfg.depths[li] * (1 if stream == "fp16" and li in (0, 3) else 2) for li in range(4))
    pad = sum(cfg.depths[li] * (ps.level(cfg, li).Hp > ps.level(cfg, li).H) for li in range(4))
    assert sum(n for *_, n in u) == 2 + 2 + 2 + 1 + 3 * blocks + pad + mlp_launches
    assert list(ps.unit_index(cfg, stream).values()) == list(range(1, len(u) + 1))
    assert (g1.C, g2.C) == (192, 384)
