"""Pangu's hierarchical 6-h / 24-h schedule without a GPU: the planner against earth2mip's generator, the two-file
importer, and the refusals."""
import itertools
import os

import numpy as np
import pytest

from skyrim_b200 import importers as I
from skyrim_b200 import schedule as S
from skyrim_b200.config import pangu_small
from skyrim_b200.weights import make_pangu_weights


def spec(n_steps):
    """earth2mip's PanguInference generator with symbolic operators: a state is the string of operators applied to x0,
    innermost first"""
    def gen():
        a = c = "x0"
        yield a
        while True:
            a = a + ".P24"
            for _ in range(3):
                c = c + ".P6"
                yield c
            c = a
            yield a
    return list(itertools.islice(gen(), n_steps + 1))


def run(p):
    """execute a plan on symbolic buffers: {slice n: state}, checking that each slice's buffer holds it when complete
    and that no forward of the next slice overwrites it (a host copy of slice n may run under them)"""
    bufs = {S.A0: "x0"}
    done, issued, prev_buf = {}, 0, None
    for n, buf, after in p.slices:
        for op, src, dst in p.forwards[issued:after]:
            assert dst != prev_buf and src != dst
            bufs[dst] = bufs[src] + (".P6" if op == "6h" else ".P24")
        issued, prev_buf = after, buf
        done[n] = bufs[buf]
    assert issued == len(p.forwards)
    return done, bufs


@pytest.mark.parametrize("n", range(41))
def test_every_slice_plan_is_earth2mips_generator(n):
    p = S.plan("hierarchical", n)
    done, _ = run(p)
    assert [done[k] for k in range(n + 1)] == spec(n)
    assert [s[0] for s in p.slices] == list(range(n + 1))
    # the generator's prefix: iter_slices (what the TimeLoop's __call__ follows) gives the same forwards
    fw = [f for _, _, fs in itertools.islice(S.iter_slices("hierarchical"), n) for f in fs]
    assert tuple(fw) == p.forwards


@pytest.mark.parametrize("hours", range(6, 241, 6))
def test_last_slices_plan_is_minimal(hours):
    n = hours // 6
    d, k = divmod(n, 4)
    p = S.plan("hierarchical", n, every_slice=False)
    done, bufs = run(p)
    want = spec(n)
    assert [s[0] for s in p.slices] == [n - 1, n]
    assert [done[n - 1], done[n]] == want[-2:]
    # both slices are still in their buffers at the end
    assert [bufs[b] for _, b, _ in p.slices] == want[-2:]
    count = 1 if n == 1 else d + k if k else d + 3
    assert len(p.forwards) == count <= len(S.plan("hierarchical", n).forwards)
    if hours == 168:
        assert len(p.forwards) == 10 and len(S.plan("hierarchical", n).forwards) == 28


def test_each_operator_sees_few_buffer_pairs():
    """the engine keeps eight CUDA graphs per handle: the plans must not cycle through more (source, destination) pairs"""
    plans = [S.plan("hierarchical", 40)] + [S.plan("hierarchical", n, every_slice=False) for n in range(41)]
    for op in ("6h", "24h"):
        pairs = {(s, d) for p in plans for o, s, d in p.forwards if o == op}
        assert len(pairs) <= 8, (op, pairs)
        assert all(0 <= b < S.N_BUFFERS for pr in pairs for b in pr)


@pytest.mark.parametrize("every_slice", [True, False])
def test_6h_plan_is_the_chain(every_slice):
    for n in range(0, 13):
        p = S.plan("6h", n, every_slice)
        assert [op for op, _, _ in p.forwards] == ["6h"] * n
        done, _ = run(p)
        assert all(done[k] == "x0" + ".P6" * k for k in done)
        assert sorted(done) == (list(range(n + 1)) if every_slice else list(range(max(n - 1, 0), n + 1)))


def test_planner_refusals():
    with pytest.raises(ValueError, match="schedule"):
        S.plan("12h", 4)
    with pytest.raises(ValueError):
        S.plan("hierarchical", -1)
    assert S.plan("hierarchical", 0, every_slice=False) == S.Plan((), ((0, S.A0, 0),))


def _export(w, path):
    """write a parameter dict as an exporter leaves it (the layout of tests/test_importers_cpu.py)"""
    idx = I.position_index((2, 6, 12)).reshape(-1)
    exported = {}
    for k, (name, a) in enumerate((n, a) for n, a in w.items() if n not in ("norm.mean", "norm.std", "const.masks")):
        if name.endswith("bias_table"):
            a = np.moveaxis(a[idx].reshape(144, 144, a.shape[1], a.shape[2]), (2, 3), (0, 1))
        elif a.ndim == 2:
            a = a.T
        exported[f"onnx::T_{k}"] = np.ascontiguousarray(a)
    exported["mean"], exported["std"], exported["masks"] = w["norm.mean"], w["norm.std"], w["const.masks"]
    I.write_onnx_initializers(path, exported)


def test_importer_loads_both_operators(tmp_path):
    cfg = pangu_small(41, 96)
    w6, w24 = make_pangu_weights(cfg, 0), make_pangu_weights(cfg, 1)
    _export(w6, str(tmp_path / "pangu_weather_6.onnx"))
    _export(w24, str(tmp_path / "pangu_weather_24.onnx"))
    got6, got24 = I.load_pangu_pair(str(tmp_path), cfg)
    for got, want in ((got6, w6), (got24, w24)):
        assert list(got) == list(want)
        for name in want:
            assert np.array_equal(got[name], want[name]), name
    with pytest.raises(ValueError, match="pangu_weather_24.onnx"):
        I.load_pangu_pair(str(tmp_path / "pangu_weather_6.onnx"), cfg)
    os.remove(tmp_path / "pangu_weather_24.onnx")
    with pytest.raises(FileNotFoundError, match="pangu_weather_24.onnx"):
        I.load_pangu_pair(str(tmp_path), cfg)


def test_model_refuses_a_lone_file_before_any_engine(tmp_path, monkeypatch):
    from skyrim_b200 import engine as E
    from skyrim_b200.core.models.pangu import PanguModel
    monkeypatch.setattr(E, "StepEngine", lambda *a, **k: pytest.fail("an engine was built"))
    monkeypatch.setenv("SKYRIM_B200_WEIGHTS", str(tmp_path / "pangu_weather_6.onnx"))
    with pytest.raises(ValueError, match="pangu_weather_24.onnx"):
        PanguModel(cfg=pangu_small(41, 96), schedule="hierarchical")


def test_model_refusals_before_any_engine(monkeypatch):
    from skyrim_b200 import engine as E
    from skyrim_b200.core.models.pangu import PanguModel
    from skyrim_b200.core.skyrim import Skyrim
    monkeypatch.setattr(E, "StepEngine", lambda *a, **k: pytest.fail("an engine was built"))
    with pytest.raises(ValueError, match="schedule"):
        PanguModel(schedule="24h")
    with pytest.raises(ValueError, match="hierarchical"):
        PanguModel(weight_seed_24=3)
    with pytest.raises(ValueError, match="hierarchical"):
        Skyrim("pangu", "graphcast", pangu=dict(schedule="hierarchical"))
    with pytest.raises(ValueError, match="hierarchical"):
        Skyrim("graphcast", "pangu", schedule="hierarchical")


def test_cli_pangu_schedule(monkeypatch):
    from click.testing import CliRunner
    from skyrim_b200 import forecast as F
    calls = []
    monkeypatch.setattr(F, "run_forecast", lambda *a, **kw: calls.append(kw) or [])
    monkeypatch.setattr(F, "run_ensemble_forecast", lambda *a, **kw: calls.append(kw) or [])
    for bad in (["--models", "pangu,graphcast", "--pangu_schedule", "hierarchical"],
                ["-m", "graphcast", "--pangu_schedule", "hierarchical"],
                ["-m", "fourcastnet_v2", "--pangu_schedule", "6h"],
                ["-m", "pangu", "--pangu_schedule", "12h"]):
        r = CliRunner().invoke(F.main, bad)
        assert r.exit_code == 2 and "pangu_schedule" in r.output, (bad, r.output)
    assert calls == []
    assert CliRunner().invoke(F.main, ["-m", "pangu", "--pangu_schedule", "hierarchical"]).exit_code == 0
    assert CliRunner().invoke(F.main, ["-m", "pangu", "--members", "3", "--pangu_schedule", "hierarchical"]).exit_code == 0
    assert CliRunner().invoke(F.main, ["-m", "pangu"]).exit_code == 0
    assert [kw.get("schedule") for kw in calls] == ["hierarchical", "hierarchical", None]
