"""Static shape of the Go2 shape-specialised rollout kernel (CPU only: nvcc cross-compiles, nvdisasm reads
the cubin): like the generic star<3,6> kernel (tests/test_rollout_sass.py) it must hold one copy of
rollout_warp and must not spill within 128 registers, and its env-step loop must be smaller than the generic one's."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sections(*args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "sass_sections.py"), *args],
                       capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr
    return r.stdout


def _env_step_kb(out):
    return float(re.search(r"env-step loop .*: ([0-9.]+) KB", out).group(1))


def test_shape_kernel_has_one_rollout_warp_no_spills_and_a_shorter_step():
    out = _sections("--shape", "go2")
    assert "copies of rollout_warp: 1 " in out, out
    assert "0 bytes spill stores, 0 bytes spill loads" in out, out
    assert int(re.search(r"Used (\d+) registers", out).group(1)) <= 128, out
    assert _env_step_kb(out) < _env_step_kb(_sections("--variant", "1")), out
