"""CPU: bench.py's host-side helpers and the `--impl reference` arm end to end on one synthetic clip (the arm is the
CPU restatement of the reference path, so it runs without a GPU)."""

from __future__ import annotations

import json
import os
import subprocess
import sys

from conftest import ROOT

sys.path.insert(0, str(ROOT))
import bench  # noqa: E402


def test_cpu_layout_uses_physical_cores():
    assert bench.cpu_layout(128) == (16, 4)
    assert bench.cpu_layout(8) == (2, 4)
    assert bench.cpu_layout(2) == (1, 1)
    procs, threads = bench.cpu_layout(64)
    assert procs * threads <= 64


def test_shot_flops_per_window_matches_the_architecture():
    # 2*M*N*K summed by hand for the rf=16, rl=3, rs=2 stack (DESIGN.md 5b): ~83.2 GFLOP per 100-frame window
    total = bench.shot_flops_per_window()
    assert 83.0e9 < total < 83.4e9
    assert abs(bench.shot_flops_per_window(50) * 2 - total) / total < 1e-6  # linear in the frame count


def test_steps_and_dump_outputs_arguments():
    r = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--steps", "0", "--dump-outputs", "x"], capture_output=True, text=True, cwd=str(ROOT))
    assert r.returncode == 2 and "--steps must be at least 1" in r.stderr
    assert "--dump-outputs DIR" in subprocess.run([sys.executable, str(ROOT / "bench.py"), "--help"], capture_output=True, text=True, cwd=str(ROOT)).stdout


def test_reference_arm_prints_one_contract_line():
    env = dict(os.environ, CB_REF_PROCS="1", CB_REF_THREADS=str(min(8, os.cpu_count() or 1)), OPENCV_LOG_LEVEL="ERROR")
    r = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0", "--ref-clips", "1"],
                       capture_output=True, text=True, env=env, cwd=str(ROOT), timeout=600)  # fmt: skip
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "clips_per_sec" and d["unit"] == "clips/s" and d["higher_is_better"] is True
    assert d["config"]["workload"] == bench.WORKLOAD
    assert d["value"] > 0 and d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "clips/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
