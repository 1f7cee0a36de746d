"""CPU test of per-instance tasks (dial_mpc_buffers.tasks) through the warp emulator: instance b of a
batched launch that reads its reward inputs from tasks[b] must compute bitwise what a single-instance
launch computes whose plan constants hold task b (tasks NULL).  Plus the host-side task helpers."""
import ctypes as C
import os
import subprocess
from dataclasses import replace

import numpy as np
import pytest

from dial_mpc_b200 import _capi
from dial_mpc_b200.utils.spline import interp_matrix
from tests.conftest import make_pair

EMUL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    """g++ build of tests/emul/emul_tasks.cpp (the device code under the lock-step warp emulator)."""
    so = str(tmp_path_factory.mktemp("emul_tasks") / "libdial_emul_tasks.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", EMUL, "-shared", "-fPIC", "-o", so,
                           os.path.join(EMUL, "emul_tasks.cpp")])
    return C.CDLL(so)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _desc_with_task(desc, t):
    """A copy of ``desc`` whose task fields hold ``t`` (the single-instance oracle's plan constants)."""
    d = _capi.dial_plan_desc.from_buffer_copy(desc)
    for name in _capi.TASK_FIELDS:
        v = getattr(t, name)
        if isinstance(v, C.Array):
            C.memmove(C.addressof(getattr(d, name)), C.addressof(v), C.sizeof(v))
        else:
            setattr(d, name, v)
    return d


def rollout_tasks(lib, env, desc, qpos, qvel, warm, counters, tasks=None, rng=None, us=None, Ybar=None, noise=None,
                  mode=1, H=None, us_row=0, single=False):
    """Rows as dial_mpc_step launches them (see tests/test_emul_batch.py), the reward inputs of instance
    b from tasks[b] (None: the plan's own task).  single=True: one instance as a single-instance plan."""
    md = _capi.fill_model_desc(env.sys.model)
    nq, nv, nu, nb = md.nq, md.nv, md.nu, md.nbody
    f32 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float32)
    qpos, qvel, warm, us, Ybar, noise = map(f32, (qpos, qvel, warm, us, Ybar, noise))
    B = qpos.shape[0]
    rpi = desc.Nsample + 1 if mode == 1 else 1
    nrows = B * rpi
    assert not single or B == 1
    task_arr = None if tasks is None else (_capi.dial_task * len(tasks))(*tasks)
    cin = np.ascontiguousarray(counters, dtype=np.int32)
    rng = None if rng is None else np.ascontiguousarray(rng, dtype=np.uint32)
    out = dict(rewss=np.zeros((nrows, H), np.float32), rews=np.zeros(nrows, np.float32),
               q=np.zeros((nrows, H, nq), np.float32), qd=np.zeros((nrows, H, nv), np.float32),
               xpos=np.zeros((nrows, H, nb - 1, 3), np.float32), qpos_out=np.zeros((B, nq), np.float32),
               qvel_out=np.zeros((B, nv), np.float32), warm_out=np.zeros((B, nv), np.float32),
               ctrl_out=np.zeros((B, nu), np.float32), counters=cin.copy())
    fin = mode == 0
    rc = lib.emul_rollout_tasks(C.byref(md), C.byref(desc), task_arr, rpi, mode, nrows, H, 0 if single else rpi,
                                int(us_row), _p(qpos), _p(qvel), _p(warm), _p(cin),
                                _p(out["counters"]) if fin else None, _p(rng), _p(us), _p(Ybar), _p(noise),
                                _p(out["rewss"]), _p(out["rews"]), _p(out["q"]), _p(out["qd"]), _p(out["xpos"]),
                                *(_p(out[k]) if fin else None for k in ("qpos_out", "qvel_out", "warm_out", "ctrl_out")))
    assert rc == 0
    return out


def _instances(o, B, nu, Hn, rng):
    s = o.reset()
    qpos = np.repeat(s.qpos, B, 0)
    qpos[:, 2] += rng.uniform(-0.02, 0.02, B)
    qpos[:, 7:7 + nu] += rng.normal(size=(B, nu)) * 0.05
    qvel = rng.normal(size=(B, o.m.nv)) * 0.2
    warm = rng.normal(size=(B, o.m.nv)) * 0.1
    Y = np.clip(rng.normal(size=(B, Hn + 1, nu)) * 0.4, -1, 1)
    return qpos, qvel, warm, Y


def _check_against_singles(lib, env, o, tasks, counters, N=4, Hs=6, Hn=3, seed=5):
    """Batched launches with per-instance tasks == single-instance launches on plans holding task b."""
    B = len(tasks)
    nu = env.action_size
    qpos, qvel, warm, Y = _instances(o, B, nu, Hn, np.random.default_rng(seed))
    keys = np.array([[0, 7], [11, 3], [123, 456]], np.uint32)[:B]
    noise = 0.9 ** np.arange(Hn + 1)[::-1]
    kw = dict(Nsample=N, Hsample=Hs, Hnode=Hn, temp_sample=0.05,
              M_n2u=interp_matrix(np.linspace(0, 1, Hn + 1), np.linspace(0, 1, Hs + 1)))
    desc = env.plan_desc(n_inst=B, **kw)
    single_desc = env.plan_desc(**kw)
    rows = N + 1
    # planner rows (mode 1): B (N+1) rows in one launch
    bat = rollout_tasks(lib, env, desc, qpos, qvel, warm, counters, tasks, rng=keys, Ybar=Y, noise=noise, mode=1,
                        H=Hs + 1)
    for b in range(B):
        one = rollout_tasks(lib, env, _desc_with_task(single_desc, tasks[b]), qpos[b:b + 1], qvel[b:b + 1],
                            warm[b:b + 1], counters[b:b + 1], rng=keys[b:b + 1], Ybar=Y[b:b + 1], noise=noise,
                            mode=1, H=Hs + 1, single=True)
        sl = slice(b * rows, (b + 1) * rows)
        for k in ("rewss", "rews", "q", "qd", "xpos"):
            assert np.array_equal(bat[k][sl], one[k]), (b, k)
    # env step (mode 0): one row per instance, action Y[b][0]
    us_row = (Hn + 1) * nu
    bat0 = rollout_tasks(lib, env, desc, qpos, qvel, warm, counters, tasks, us=Y, mode=0, H=1, us_row=us_row)
    for b in range(B):
        one = rollout_tasks(lib, env, _desc_with_task(single_desc, tasks[b]), qpos[b:b + 1], qvel[b:b + 1],
                            warm[b:b + 1], counters[b:b + 1], us=Y[b:b + 1, :1], mode=0, H=1, single=True)
        for k in ("qpos_out", "qvel_out", "warm_out", "ctrl_out", "counters"):
            assert np.array_equal(bat0[k][b], one[k][0]), (b, k)
        assert np.array_equal(bat0["rewss"][b], one["rewss"][0]), b
    return bat, bat0, (qpos, qvel, warm, Y, keys, noise, desc)


def test_walk_tasks_equal_single_instance_plans(lib):
    import dial_mpc_b200.envs as E
    env, o = make_pair("unitree_go2_walk")
    cfgs = [replace(env._config, default_vx=0.3, gait="trot"), replace(env._config, default_vx=-0.6, default_vyaw=0.5, gait="walk"),
            replace(env._config, default_vx=1.0, default_vy=0.2, gait="trot")]
    envs = [E.get_environment("unitree_go2_walk", config=c) for c in cfgs]
    tasks = [e.task() for e in envs]
    # instance 1 meets a randomize_tasks one-step command inside its horizon (steps 45..51)
    _capi.task_set_command(tasks[1], (48, np.array([0.9, -0.3, 0.0]), np.array([0.0, 0.0, -1.1])))
    counters = np.array([[45, 0], [45, 0], [40, 0]], np.int32)
    bat, bat0, _ = _check_against_singles(lib, env, o, tasks, counters)
    rows = 5
    # the tasks really change the rewards: instance 0 under instance 2's task differs
    assert not np.array_equal(bat["rewss"][:rows], bat["rewss"][2 * rows:])
    # and the command of step 48 is what instance 1 sees (the same row without it differs)
    t1 = _capi.dial_task.from_buffer_copy(tasks[1])
    _capi.task_set_command(t1, None)
    alt, _, _ = _check_against_singles(lib, env, o, [tasks[0], t1, tasks[2]], counters)
    assert not np.array_equal(alt["rewss"][rows:2 * rows], bat["rewss"][rows:2 * rows])
    assert np.array_equal(alt["rewss"][rows:2 * rows, :3], bat["rewss"][rows:2 * rows, :3])   # steps 45..47


def test_seq_jump_tasks_equal_single_instance_plans(lib):
    from dial_mpc_b200 import random as drandom
    env, o = make_pair("unitree_go2_seq_jump")
    tasks = []
    for k in (3, 4, 5):
        tgt, rad, pose, yaw = env.sample_command(drandom.PRNGKey(k))
        tasks.append(_capi.task_set_stages(env.task(), (pose, yaw, tgt, rad)))
    assert tasks[0].n_stage == env.N_RANDOM_STAGES + 1
    # the counters straddle the first stage boundary (the env step from step 49 enters stage 1)
    counters = np.array([[45, 0], [49, 0], [50, 1]], np.int32)
    bat, bat0, _ = _check_against_singles(lib, env, o, tasks, counters)
    assert bat0["counters"][1, 1] == 1 and bat0["counters"][0, 1] == 0


def test_own_task_for_every_instance_equals_no_tasks(lib):
    env, o = make_pair("unitree_go2_walk")
    B, N, Hs, Hn = 3, 4, 6, 3
    nu = env.action_size
    qpos, qvel, warm, Y = _instances(o, B, nu, Hn, np.random.default_rng(9))
    keys = np.array([[0, 7], [11, 3], [123, 456]], np.uint32)
    noise = 0.9 ** np.arange(Hn + 1)[::-1]
    desc = env.plan_desc(Nsample=N, Hsample=Hs, Hnode=Hn, temp_sample=0.05,
                         M_n2u=interp_matrix(np.linspace(0, 1, Hn + 1), np.linspace(0, 1, Hs + 1)), n_inst=B)
    counters = np.array([[0, 0], [17, 0], [30, 0]], np.int32)
    own = [env.task() for _ in range(B)]
    for mode, H, extra in ((1, Hs + 1, dict(rng=keys, Ybar=Y, noise=noise)), (0, 1, dict(us=Y, us_row=(Hn + 1) * nu))):
        a = rollout_tasks(lib, env, desc, qpos, qvel, warm, counters, own, mode=mode, H=H, **extra)
        b = rollout_tasks(lib, env, desc, qpos, qvel, warm, counters, None, mode=mode, H=H, **extra)
        for k in a:
            assert np.array_equal(a[k], b[k]), (mode, k)


@pytest.mark.parametrize("name", ["unitree_go2_walk", "unitree_go2_seq_jump", "unitree_h1_walk", "unitree_h1_loco",
                                  "allegro_reorient"])
def test_env_task_is_the_descriptor_task(name):
    env, _ = make_pair(name)
    d, t = env.plan_desc(), env.task()
    for field in _capi.TASK_FIELDS:
        a, b = getattr(d, field), getattr(t, field)
        assert (bytes(a) == bytes(b)) if isinstance(a, C.Array) else a == b, field
    assert t.cmd_step == -1 and 1 <= t.n_stage <= _capi.DEFINES["DIAL_MAXSTAGE"]


def test_custom_env_task_carries_user_params():
    import importlib
    import sys
    ex = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dial_mpc_b200", "examples",
                      "custom_env")
    if ex not in sys.path:
        sys.path.insert(0, ex)
    qe = importlib.import_module("quadpod_env")
    env = qe.QuadpodEnv(qe.QuadpodEnvConfig(target_vx=0.8))
    t = env.task()
    assert t.n_user == 6 and np.allclose(np.ctypeslib.as_array(t.user)[:6], env.user_params())
    assert t.n_stage == 1


def test_shared_field_check_names_the_field():
    import dial_mpc_b200.envs as E
    from dial_mpc_b200.core.dial_core import DeviceLoop
    env, _ = make_pair("unitree_go2_walk")
    ok = E.get_environment("unitree_go2_walk", config=replace(env._config, default_vx=1.2, gait="walk"))
    DeviceLoop._check_shared(env, ok)      # commands and gait are task fields
    kp = E.get_environment("unitree_go2_walk", config=replace(env._config, kp=env._config.kp * 2))
    assert _capi.first_shared_difference(env.plan_desc(), kp.plan_desc()) == "kp"
    with pytest.raises(ValueError, match="'kp'"):
        DeviceLoop._check_shared(env, kp)
    other, _ = make_pair("unitree_go2_seq_jump")
    with pytest.raises(ValueError, match="UnitreeGo2Env"):
        DeviceLoop._check_shared(env, other)


def test_task_ranges_are_checked_on_the_host():
    env, _ = make_pair("unitree_go2_walk")
    t = env.task()
    for field, bad in (("n_stage", 0), ("n_stage", _capi.DEFINES["DIAL_MAXSTAGE"] + 1), ("n_user", -1),
                       ("n_user", _capi.DEFINES["DIAL_MAXUSER"] + 1)):
        u = _capi.dial_task.from_buffer_copy(t)
        setattr(u, field, bad)
        with pytest.raises(ValueError, match=field):
            _capi.check_task(u)
    with pytest.raises(ValueError, match="stages"):
        _capi.task_set_stages(env.task(), (np.zeros((13, 3)), np.zeros(13), np.zeros((13, 4, 3)), np.zeros((13, 4))))
