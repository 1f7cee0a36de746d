"""Per-instance sampling schedules on the CPU: the schedule spec (schedule_setting) and its errors, the noise
table (schedule_table) against MBDPI.schedule of the updated config, the --instance-overrides errors, and on
the warp emulator the planner rows of a batched launch with per-instance noise rows against single-instance
launches bound to that row, and the CTA -> instance mapping the skipped instances exit by (cta_instance)."""
import ctypes as C
import dataclasses
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dial_mpc_b200 import _capi
from dial_mpc_b200.core.dial_config import DialConfig
from dial_mpc_b200.utils.spline import interp_matrix
from tests.conftest import make_pair
from tests.test_emul_batch import _instances

EMUL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
BASE = DialConfig(env_name="unitree_go2_walk", Nsample=64, Hsample=12, Hnode=4, Ndiffuse=2, Ndiffuse_init=3,
                  temp_sample=0.05, horizon_diffuse_factor=0.9, traj_diffuse_factor=0.5)


def test_schedule_setting_updates_the_sampling_fields():
    from dial_mpc_b200.core.dial_core import SCHEDULE_FIELDS, schedule_setting
    assert schedule_setting({}, BASE) == BASE
    spec = {"temp_sample": 0.1, "sigma_scale": 0, "horizon_diffuse_factor": 1, "traj_diffuse_factor": 0.3,
            "Ndiffuse": 4, "Ndiffuse_init": 64}
    assert set(spec) == set(SCHEDULE_FIELDS)
    got = schedule_setting(spec, BASE)
    assert got == dataclasses.replace(BASE, **spec)
    assert (got.Nsample, got.Hsample, got.Hnode) == (64, 12, 4)
    assert schedule_setting({"Ndiffuse": np.int64(5)}, BASE).Ndiffuse == 5


BAD_SPECS = [
    ([("temp_sample", 0.1)], r"a schedule spec maps"),
    ({"temp_sample": 0.0}, r"temp_sample must be a finite number > 0, got 0.0"),
    ({"temp_sample": -0.1}, r"temp_sample must be a finite number > 0"),
    ({"temp_sample": float("inf")}, r"temp_sample must be a finite number > 0, got inf"),
    ({"temp_sample": 1e-60}, r"temp_sample must be a finite number > 0"),       # 0 in fp32
    ({"temp_sample": "0.1"}, r"temp_sample must be a finite number"),
    ({"sigma_scale": -1.0}, r"sigma_scale must be a finite number >= 0"),
    ({"sigma_scale": float("nan")}, r"sigma_scale must be a finite number >= 0, got nan"),
    ({"horizon_diffuse_factor": 0}, r"horizon_diffuse_factor must be a finite number > 0"),
    ({"traj_diffuse_factor": True}, r"traj_diffuse_factor must be a finite number > 0, got True"),
    ({"Ndiffuse": 0}, r"Ndiffuse must be an int in 1..64, got 0"),
    ({"Ndiffuse": 65}, r"Ndiffuse must be an int in 1..64, got 65"),
    ({"Ndiffuse_init": 2.0}, r"Ndiffuse_init must be an int in 1..64, got 2.0"),
    ({"Nsample": 128}, r"Nsample is shared by every instance of the plan"),
    ({"Hnode": 3}, r"Hnode is shared by every instance"),
    ({"update_method": "mppi"}, r"update_method is shared by every instance"),
    ({"temp": 0.1}, r"unknown key 'temp'"),
]


@pytest.mark.parametrize("spec, match", BAD_SPECS)
def test_schedule_setting_names_the_bad_key_or_value(spec, match):
    from dial_mpc_b200.core.dial_core import schedule_setting
    with pytest.raises(ValueError, match=match):
        schedule_setting(spec, BASE)


@pytest.mark.parametrize("spec", [{}, {"temp_sample": 0.1}, {"Ndiffuse": 4, "traj_diffuse_factor": 0.3},
                                  {"sigma_scale": 0.7, "horizon_diffuse_factor": 1.0, "Ndiffuse_init": 10}])
def test_table_is_the_schedule_of_the_updated_config(spec):
    """schedule_table of the updated config is MBDPI.schedule of an MBDPI built with it, and the reference's
    sigma_control * traj_diffuse_factor ** arange(n) with sigma_control from that MBDPI."""
    from dial_mpc_b200.core.dial_core import MBDPI, schedule_setting, schedule_table
    from tests.emul.emul import EmulPlan
    env, _ = make_pair("unitree_go2_walk")
    cfg = schedule_setting(spec, dataclasses.replace(BASE, Nsample=8, Hsample=6))
    mb = MBDPI(cfg, env, plan_factory=EmulPlan)
    n = max(cfg.Ndiffuse, cfg.Ndiffuse_init)
    got = schedule_table(cfg, n, mb.device)
    assert got.dtype == torch.float32 and tuple(got.shape) == (n, cfg.Hnode + 1)
    assert torch.equal(got, mb.schedule(n))
    sigma = torch.as_tensor(mb.sigma_control_np.astype(np.float32))
    ref = sigma[None, :] * (cfg.traj_diffuse_factor ** torch.arange(n, dtype=torch.float32))[:, None]
    assert torch.equal(got, ref)
    # row i does not depend on the row count
    assert torch.equal(schedule_table(cfg, 1, mb.device)[0], got[0])


def _main(monkeypatch, capsys, argv):
    from dial_mpc_b200.core import dial_core
    monkeypatch.setattr(sys, "argv", ["dial_core", "--example", "unitree_go2_trot"] + argv)
    with pytest.raises(SystemExit) as e:
        dial_core.main()
    return e.value.code, capsys.readouterr().err


@pytest.mark.parametrize("entry, match", [
    ({"temp_sample": 0}, r"temp_sample must be a finite number > 0"),
    ({"Ndiffuse": 70, "default_vx": 0.5}, r"Ndiffuse must be an int in 1\.\.64, got 70"),
    ({"traj_diffuse_factor": "x"}, r"traj_diffuse_factor must be a finite number > 0"),
    ({"Nsample": 128}, r"Nsample is shared by every instance of the plan"),
    ({"Hsample": 10, "temp_sample": 0.1}, r"Hsample is shared by every instance of the plan"),
    ({"seed": 3}, r"seed is shared by every instance of the plan"),
])
def test_cli_instance_override_schedule_errors(tmp_path, monkeypatch, capsys, entry, match):
    import re
    import yaml
    ov = tmp_path / "ov.yaml"
    ov.write_text(yaml.safe_dump([{"temp_sample": 0.1}, {}, entry]))
    code, err = _main(monkeypatch, capsys, ["--instances", "3", "--instance-overrides", str(ov)])
    assert code == 2 and re.search(r"--instance-overrides entry 2: " + match, err), err


# ---- warp emulator ---------------------------------------------------------------------------------------
SCHED = np.dtype([("on", "<i4"), ("temp", "<f4"), ("n_rows", "<i4"), ("pad", "<i4"),
                  ("noise", "<f4", (_capi.DEFINES["DIAL_MAXDIFFUSE"], _capi.DEFINES["DIAL_MAXNODE"]))])


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    """g++ build of tests/emul/emul_schedule.cpp (the device code under the lock-step warp emulator)."""
    so = str(tmp_path_factory.mktemp("emul_schedule") / "libdial_emul_schedule.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", EMUL, "-shared", "-fPIC", "-o", so,
                           os.path.join(EMUL, "emul_schedule.cpp")])
    lib = C.CDLL(so)
    lib.emul_sizeof_schedule.restype = C.c_size_t
    assert lib.emul_sizeof_schedule() == SCHED.itemsize
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _rows(lib, env, desc, qpos, qvel, warm, counters, keys, Y, noise, iter_, sched, single):
    md = _capi.fill_model_desc(env.sys.model)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    qpos, qvel, warm, Y, noise = map(f32, (qpos, qvel, warm, Y, noise))
    B, rows, H = qpos.shape[0], desc.Nsample + 1, desc.Hsample + 1
    rews, q = np.zeros(B * rows, np.float32), np.zeros((B * rows, H, md.nq), np.float32)
    rc = lib.emul_rollout_schedule(C.byref(md), C.byref(desc), B * rows, H, 0 if single else rows, iter_, _p(sched),
                                   _p(qpos), _p(qvel), _p(warm), _p(np.ascontiguousarray(counters, np.int32)),
                                   _p(np.ascontiguousarray(keys, np.uint32)), _p(Y), _p(noise), _p(rews), _p(q))
    assert rc == 0
    return rews, q


def test_batched_rows_take_their_instance_noise_row(lib):
    """Instance b's planner rows at iteration i with its own table equal a single-instance launch bound to
    row i of that table; an instance whose schedule is off takes the bound row."""
    env, o = make_pair("unitree_go2_walk")
    B, N, Hs, Hn, it = 3, 4, 6, 3, 2
    nu = env.action_size
    rng = np.random.default_rng(7)
    qpos, qvel, warm, Y = _instances(o, B, nu, Hn, rng)
    counters = np.array([[5, 0], [9, 0], [0, 0]], np.int32)
    keys = np.array([[0, 7], [11, 3], [123, 456]], np.uint32)
    bound = np.float32(0.9 ** np.arange(Hn + 1)[::-1])
    desc = env.plan_desc(Nsample=N, Hsample=Hs, Hnode=Hn, temp_sample=0.05,
                         M_n2u=interp_matrix(np.linspace(0, 1, Hn + 1), np.linspace(0, 1, Hs + 1)), n_inst=B)
    sched = np.zeros(B, SCHED)
    for b, scale in ((1, 0.3), (2, 1.7)):
        sched["on"][b], sched["temp"][b], sched["n_rows"][b] = 1, 0.1, it + 1
        sched["noise"][b, :it + 1, :Hn + 1] = rng.uniform(0.1, 1.0, (it + 1, Hn + 1)) * scale
    bat = _rows(lib, env, desc, qpos, qvel, warm, counters, keys, Y, bound, it, sched, single=False)
    rows = N + 1
    for b in range(B):
        row = sched["noise"][b, it, :Hn + 1] if sched["on"][b] else bound
        one = _rows(lib, env, desc, qpos[b:b + 1], qvel[b:b + 1], warm[b:b + 1], counters[b:b + 1], keys[b:b + 1],
                    Y[b:b + 1], row, 0, None, single=True)
        sl = slice(b * rows, (b + 1) * rows)
        assert np.array_equal(bat[0][sl], one[0]) and np.array_equal(bat[1][sl], one[1]), b
    # the table row was read: instance 1 bound to the plan's row differs
    other = _rows(lib, env, desc, qpos[1:2], qvel[1:2], warm[1:2], counters[1:2], keys[1:2], Y[1:2], bound, 0, None,
                  single=True)
    assert not np.array_equal(bat[0][rows:2 * rows], other[0])


def _brute_instance(nrows, rpi, rps, models, cta, wpc):
    """The instance of each warp of CTA `cta` as rollout_kernel maps rows (the duplicated last row included)."""
    insts = set()
    for warp in range(wpc):
        if models:
            cpi = (rps + wpc - 1) // wpc
            slot = cta // cpi
            row = (cta - slot * cpi) * wpc + warp
            row = min(row, rps - 1) + slot * rps
        else:
            row = cta * wpc + warp
        row = min(row, nrows - 1)
        insts.add(row // rpi)
    return insts.pop() if len(insts) == 1 else -1


@pytest.mark.parametrize("B, K, N, wpc", [(24, 0, 100, 16), (24, 0, 100, 7), (5, 0, 128, 16), (3, 2, 64, 16),
                                          (4, 4, 20, 3), (2, 16, 8, 16)])
def test_cta_instance_mapping(lib, B, K, N, wpc):
    rows = N + 1
    rpi = max(K, 1) * rows
    nrows = B * rpi
    # straddled: the plain launch (no model slots); every CTA that holds one instance's rows names it
    grid = (nrows + wpc - 1) // wpc
    straddle = 0
    for cta in range(grid):
        want = _brute_instance(nrows, rpi, 0, False, cta, wpc)
        straddle += want < 0
        assert lib.emul_cta_instance(nrows, rpi, 0, 0, cta, wpc) == want, cta
    if K == 0 and rpi % wpc:
        assert straddle > 0
    # model layout (per-instance models, or the member slots of an ensemble: slot b K + k is instance b)
    rps = rows if K > 0 else rpi
    grid = (nrows // rps) * ((rps + wpc - 1) // wpc)
    seen = set()
    for cta in range(grid):
        want = _brute_instance(nrows, rpi, rps, True, cta, wpc)
        assert want >= 0
        assert lib.emul_cta_instance(nrows, rpi, rows if K > 0 else 0, 1, cta, wpc) == want, cta
        seen.add(want)
    assert seen == set(range(B))
    # a single-instance launch
    assert lib.emul_cta_instance(rows, 0, 0, 0, 0, wpc) == 0
