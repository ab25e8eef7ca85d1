"""bench.py contract checks that do not need a GPU: the reference arm reports why it is unavailable
with one JSON line and exit code 0; the own arm refuses to run without CUDA with one JSON line."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(*args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *args], capture_output=True, text=True,
                          cwd=ROOT, timeout=300)


def test_reference_arm_reports_unavailable_in_one_json_line():
    r = _run("--impl", "reference", "--gpus", "1", "--steps", "2", "--warmup", "3")
    assert r.returncode == 0
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and isinstance(d["unavailable"], str) and d["unavailable"]


def test_own_arm_prints_exactly_one_json_line_without_cuda():
    import torch
    if torch.cuda.is_available():
        import pytest
        pytest.skip("CPU-only contract check")
    r = _run()
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1 and "error" in json.loads(lines[0])


def test_graft_entry_exposes_build_and_smoke():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    assert callable(g.build) and callable(g.smoke)


def _fake_run(n):
    import torch

    class Pack:
        flat = torch.arange(n, dtype=torch.float32) * 0.5

    class Run:
        pack = Pack()
        history = [{"loss": 0.25, "accuracy": 0.75}]

    return Run()


def test_dump_outputs_writes_float_arrays_of_the_last_round(tmp_path):
    import numpy as np

    sys.path.insert(0, ROOT)
    import bench

    run = _fake_run(1000)
    bench.dump_outputs(str(tmp_path), run)
    assert sorted(os.listdir(tmp_path)) == ["accuracy.npy", "global_weights.npy", "loss.npy"]
    w = np.load(tmp_path / "global_weights.npy")
    assert w.dtype == np.float32 and np.array_equal(w, run.pack.flat.numpy())
    assert np.load(tmp_path / "loss.npy").dtype == np.float64 and float(np.load(tmp_path / "loss.npy")[0]) == 0.25
    assert float(np.load(tmp_path / "accuracy.npy")[0]) == 0.75


def test_dump_outputs_samples_large_outputs_at_fixed_indices_within_64_mb(tmp_path, monkeypatch):
    import numpy as np

    sys.path.insert(0, ROOT)
    import bench

    assert bench.DUMP_MAX_ELEMS * (4 + 8) <= 64 << 20          # weights (float32) + their indices (float64)
    monkeypatch.setattr(bench, "DUMP_MAX_ELEMS", 100)
    run = _fake_run(1000)
    bench.dump_outputs(str(tmp_path / "a"), run)
    bench.dump_outputs(str(tmp_path / "b"), run)
    idx = np.load(tmp_path / "a" / "global_weights_sample_idx.npy")
    w = np.load(tmp_path / "a" / "global_weights.npy")
    assert idx.shape == (100,) and w.shape == (100,) and np.all(np.diff(idx) > 0)
    assert np.array_equal(w, run.pack.flat.numpy()[idx.astype(np.int64)])
    assert np.array_equal(idx, np.load(tmp_path / "b" / "global_weights_sample_idx.npy"))   # same sample every run
