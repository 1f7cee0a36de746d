"""The Go2 rollout kernel with the contact, edge, feet and frame counts fixed at compile time (CPU only: nvcc
cross-compiles, nvdisasm reads the cubin).  Its static size stays where this build put it; the expressions
pinned with __fmaf_rn in dial_device.cuh compile to the same fused/unfused mix as in the generic star<3,6>
kernel; and every stock Go2 example configuration still matches every value the kernel fixes."""
import glob
import os
import re
import subprocess
import sys

import pytest
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _script(name, *args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", name), *args],
                       capture_output=True, text=True, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stderr
    return r.stdout


def test_go2_kernel_static_size():
    out = _script("sass_sections.py", "--shape", "go2")
    assert "copies of rollout_warp: 1 " in out, out
    assert "0 bytes spill stores, 0 bytes spill loads" in out, out
    assert int(re.search(r"Used (\d+) registers", out).group(1)) <= 128, out
    # nvcc 12.9, sm_90a: 91.5 KB and 22.0 KB (109.5 KB and 27.5 KB with the counts read at run time)
    assert float(re.search(r"env-step loop .*: ([0-9.]+) KB", out).group(1)) <= 93.0, out
    assert float(re.search(r"Newton loop body .*: ([0-9.]+) KB", out).group(1)) <= 22.5, out


def test_pinned_lines_compile_alike_in_both_kernels():
    out = _script("contraction_diff.py", "--all")
    m = re.search(r"pinned lines whose mix differs between generic and go2: (\d+)", out)
    assert m and int(m.group(1)) == 0, out
    # the pins are in the env-step loop: the tool sees them in both kernels
    assert re.search(r"\| pinned \|", out), out


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(ROOT, "dial_mpc_b200", "examples", "unitree_go2_*.yaml"))),
                         ids=os.path.basename)
def test_stock_go2_examples_match_the_fixed_structure(path):
    import dial_mpc_b200.envs as E
    from dial_mpc_b200 import _capi
    from dial_mpc_b200.core.dial_config import DialConfig
    from dial_mpc_b200.modelc.shape import SHAPES, env_structure_defines, structure_defines
    from dial_mpc_b200.utils.io_utils import load_dataclass_from_dict
    cfg = yaml.safe_load(open(path))
    dc = load_dataclass_from_dict(DialConfig, cfg)
    env = E.get_environment(dc.env_name, config=load_dataclass_from_dict(E.get_config(dc.env_name), cfg,
                                                                          convert_list_to_array=True))
    pd = env.plan_desc(Nsample=8, Hsample=dc.Hsample, Hnode=dc.Hnode)
    (go2,) = [e for name, e in SHAPES if name == "go2"]
    fixed = env_structure_defines(go2)
    assert structure_defines(_capi.fill_model_desc(env.sys.model), pd) == fixed
    assert {"DIAL_SHAPE_NCON=4", "DIAL_SHAPE_NEDGE=16", "DIAL_SHAPE_NFEET=4", "DIAL_SHAPE_N_FRAMES=1"} <= set(fixed)
