"""bench.py's output contract, as far as it can be exercised without a GPU: the reference arm (`--impl reference`) is
the CPU restatement of the path timed on the host cores, so it runs here -- one JSON line on stdout with the keys the
driver reads -- and under torchrun only rank 0 prints.  The GPU arm's line is checked on the box (`-m gpu`)."""
from __future__ import annotations

import json
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
REQUIRED = {"impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
            "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"}


def _run(extra: list[str], env: dict[str, str] | None = None) -> list[str]:
    out = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--steps", "2", "--warmup", "1",
                          "--cpu-sample-chunks", "256", *extra], capture_output=True, text=True, timeout=300, check=True,
                         env={**os.environ, **(env or {})})
    return [ln for ln in out.stdout.splitlines() if ln.strip()]


def test_reference_arm_prints_one_contract_line():
    lines = _run([])
    assert len(lines) == 1, lines
    d = json.loads(lines[0])
    assert REQUIRED <= set(d), REQUIRED - set(d)
    assert d["impl"] == "reference" and d["n_gpus"] == 1 and d["steps"] == 2 and d["warmup"] == 1
    assert d["value"] > 0 and d["higher_is_better"] is True and d["vs_baseline"] is None
    assert d["metric"].startswith("queries/sec multi-vector MaxSim") and "workload" in d["config"]
    cb = d["cpu_baseline"]
    assert cb["kind"] in ("port", "reference") and cb["cores"] >= 1 and cb["sample"] and cb["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}


@pytest.mark.parametrize("workload", ["c2", "c3"])
def test_reference_arm_other_workloads(workload):
    d = json.loads(_run(["--workload", workload])[0])
    assert d["impl"] == "reference" and d["value"] > 0 and workload in ("c2", "c3")


@pytest.mark.parametrize("extra", [["--steps", "0"], ["--workload", "c5", "--gpus", "2", "--dump-outputs", "unused"]])
def test_bad_argument_combinations_are_rejected(extra):
    """Zero timed steps, and a c5 dump on several GPUs (each rank only holds its own pairs), stop at argument parsing."""
    out = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", *extra], capture_output=True, text=True,
                         timeout=120, check=False)
    assert out.returncode == 2 and "error:" in out.stderr and not out.stdout.strip()


def test_reference_arm_under_torchrun_only_rank0_prints():
    """N > 1: the driver launches the arm with torchrun; rank 0 alone runs and prints, the others exit 0 without work."""
    base = {"WORLD_SIZE": "2", "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": "29655"}
    assert _run(["--gpus", "2"], {**base, "RANK": "1", "LOCAL_RANK": "1"}) == []
    lines = _run(["--gpus", "2"], {**base, "RANK": "0", "LOCAL_RANK": "0"})
    assert len(lines) == 1 and json.loads(lines[0])["n_gpus"] == 2


@pytest.mark.gpu
def test_gpu_arm_line_carries_the_contract_keys():
    """The GPU arm on configs[1] (1.2 GB corpus, seconds): one JSON line with roofline / e2e / clocks / launch count and
    the oracle check of 16 queries green."""
    out = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--workload", "c2", "--steps", "4", "--warmup", "3",
                          "--no-cpu-baseline"], capture_output=True, text=True, timeout=600, check=True)
    lines = [ln for ln in out.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1, lines
    d = json.loads(lines[0])
    need = (REQUIRED - {"impl", "cpu_baseline"}) | {"roofline", "clocks", "gpu_launches", "check", "stage_ms"}
    assert need <= set(d), need - set(d)
    r = d["roofline"]
    assert r["bound"] in ("hbm", "tensor") and 0 < r["frac"] <= 1.0 and r["achieved"] > 0 and r["peak"] > 0 and "traffic" in r
    assert d["gpu_launches"] > 0 and d["steps"] == 4 and d["n_gpus"] == 1
    e = d["e2e"]
    assert e["value"] > 0 and e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0
    assert d["check"]["checked_queries"] >= 16 and d["check"]["identical_topk_sets"] == d["check"]["checked_queries"]
    assert {"sm_mhz", "sm_max_mhz", "reasons"} <= set(d["clocks"])


@pytest.mark.gpu
def test_gpu_arm_dump_outputs_are_reproducible(tmp_path):
    """``--dump-outputs``: the last timed step's results as float32 / float64 .npy files, at most 64 MB in all, and the
    same numbers from a second run with the same arguments (seeded inputs)."""
    import numpy as np

    dumps = []
    for run in ("a", "b"):
        out = tmp_path / run
        subprocess.run([sys.executable, str(ROOT / "bench.py"), "--workload", "c2", "--steps", "2", "--warmup", "1",
                        "--no-cpu-baseline", "--dump-outputs", str(out)], capture_output=True, text=True, timeout=600, check=True)
        files = sorted(out.glob("*.npy"))
        assert {f.stem for f in files} == {"hit_sim", "hit_chunk", "hit_count", "status"}
        assert sum(f.stat().st_size for f in files) <= 64 << 20
        arrays = {f.stem: np.load(f) for f in files}
        assert all(a.dtype in (np.float32, np.float64) for a in arrays.values())
        dumps.append(arrays)
    for name, a in dumps[0].items():
        assert np.array_equal(a, dumps[1][name]), name
