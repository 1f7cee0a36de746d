"""CPU test of the rollout kernel specialised on the Go2 model's integer structure (ShapeFixed) through the
warp emulator: planner rows, env steps and batched launches with per-instance tasks must equal the generic
star<3,6> kernel's bit for bit; and the host selects the specialised kernel for the stock Go2 model only."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from dial_mpc_b200 import _capi
from dial_mpc_b200.modelc.shape import SHAPES, env_structure_defines
from dial_mpc_b200.utils.spline import interp_matrix
from tests.conftest import make_pair
from tests.emul import emul
from tests.test_emul_batch import rollout_batched
from tests.test_emul_tasks import _instances


GO2_DEFINES = tuple(env_structure_defines(*[e for name, e in SHAPES if name == "go2"]))   # the library's "go2"


@pytest.fixture(scope="module")
def lib():
    return emul.build(GO2_DEFINES)


def _rollout(specialised, env, desc, qpos, qvel, warm, counters, tasks=None, **kw):
    """One launch as dial_mpc_step issues it (tests/test_emul_batch.py) through the specialised (ShapeFixed) or
    the generic star<3,6> kernel."""
    return rollout_batched(env, desc, qpos, qvel, warm, counters, tasks, single=len(qpos) == 1,
                           kernel=5 if specialised else 1, defines=GO2_DEFINES, **kw)


def _check_equal(env, o, tasks, counters, N=4, Hs=6, Hn=3, seed=3):
    """Planner rows and env steps: the specialised kernel == the generic kernel, every output."""
    B = len(counters)
    nu = env.action_size
    qpos, qvel, warm, Y = _instances(o, B, nu, Hn, np.random.default_rng(seed))
    keys = np.array([[0, 7], [11, 3], [123, 456]], np.uint32)[:B]
    noise = 0.9 ** np.arange(Hn + 1)[::-1]
    desc = env.plan_desc(Nsample=N, Hsample=Hs, Hnode=Hn, temp_sample=0.05, n_inst=B,
                         M_n2u=interp_matrix(np.linspace(0, 1, Hn + 1), np.linspace(0, 1, Hs + 1)))
    runs = []
    for spec in (True, False):
        plan = _rollout(spec, env, desc, qpos, qvel, warm, counters, tasks, rng=keys, Ybar=Y, noise=noise,
                        mode=1, H=Hs + 1)
        step = _rollout(spec, env, desc, qpos, qvel, warm, counters, tasks, us=Y, mode=0, H=1,
                        us_row=(Hn + 1) * nu)
        runs.append((plan, step))
    for (a, b) in zip(*runs):
        for k in a:
            assert np.array_equal(a[k], b[k]), k
    assert np.isfinite(runs[0][0]["rews"]).all()
    return runs[0]


def test_walk_rows_with_a_one_step_command():
    env, o = make_pair("unitree_go2_walk")
    t = env.task()
    _capi.task_set_command(t, (48, np.array([0.9, -0.3, 0.0]), np.array([0.0, 0.0, -1.1])))
    with_cmd, _ = _check_equal(env, o, [t], np.array([[45, 0]], np.int32))
    without, _ = _check_equal(env, o, None, np.array([[45, 0]], np.int32))
    assert not np.array_equal(with_cmd["rewss"], without["rewss"])      # the command is inside the horizon


def test_seq_jump_rows_across_a_stage_boundary():
    env, o = make_pair("unitree_go2_seq_jump")
    _, step = _check_equal(env, o, None, np.array([[49, 0]], np.int32))
    assert step["counters"][0, 1] == 1


def test_batched_launch_with_tasks():
    from dial_mpc_b200 import random as drandom
    env, o = make_pair("unitree_go2_seq_jump")
    tasks = []
    for k in (3, 4, 5):
        tgt, rad, pose, yaw = env.sample_command(drandom.PRNGKey(k))
        tasks.append(_capi.task_set_stages(env.task(), (pose, yaw, tgt, rad)))
    _check_equal(env, o, tasks, np.array([[45, 0], [49, 0], [50, 1]], np.int32))
    envw, ow = make_pair("unitree_go2_walk")
    _check_equal(envw, ow, [envw.task()] * 3, np.array([[0, 0], [17, 0], [30, 0]], np.int32))


def test_selection_rule(lib):
    walk, _ = make_pair("unitree_go2_walk")
    jump, _ = make_pair("unitree_go2_seq_jump")
    sel = lambda md, pd: lib.emul_shape_selects(C.byref(md), C.byref(pd))
    md = _capi.fill_model_desc(walk.sys.model)
    # the stock Go2 model selects the kernel under both of its envs
    assert sel(md, walk.plan_desc()) == 1 and sel(md, jump.plan_desc()) == 1
    # one structural field of the model changed: the generic kernel
    for field, value in (("iterations", md.iterations + 1), ("ls_iterations", md.ls_iterations + 1)):
        m2 = _capi.dial_model_desc.from_buffer_copy(md)
        setattr(m2, field, value)
        assert sel(m2, walk.plan_desc()) == 0, field
    m2 = _capi.dial_model_desc.from_buffer_copy(md)
    m2.pair_kind[0] = 1                      # a plane-capsule pair
    assert sel(m2, walk.plan_desc()) == 0
    # a four-legged custom model (quadpod: star<3,6> too) keeps the generic kernel, under any env
    ex = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dial_mpc_b200", "examples",
                      "custom_env")
    if ex not in sys.path:
        sys.path.insert(0, ex)
    import quadpod_env
    q = quadpod_env.QuadpodEnv(quadpod_env.QuadpodEnvConfig())
    qmd = _capi.fill_model_desc(q.sys.model)
    assert sel(qmd, q.plan_desc()) == 0 and sel(qmd, walk.plan_desc()) == 0
