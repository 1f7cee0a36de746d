"""CPU test of batched launches (dial_plan_desc.n_inst > 1) through the warp emulator: instance b of a
batched launch must compute bitwise what a single-instance launch from instance b's state, counters,
rng and knots computes.  Only the base addresses of the per-instance data differ."""
import numpy as np

from dial_mpc_b200 import _capi
from dial_mpc_b200.utils.spline import interp_matrix
from tests.conftest import make_pair
from tests.emul import emul


def rollout_batched(env, plan_desc, qpos, qvel, warm, counters, tasks=None, rng=None, us=None, Ybar=None, noise=None,
                    mode=1, H=None, us_row=0, single=False, **kw):
    """Batched rows as the control-step graph launches them: instance b's state qpos[b] / qvel[b] /
    warm[b], counters[b] = {step, stage}, planner rng[b] (mode 1), knots Ybar[b] and reward inputs tasks[b]
    (None: the plan's own task); mode 1 rolls Nsample+1 rows per instance, mode 0 one row per instance (the
    env step, action = us[b][0] with rows us_row floats apart).  single=True: one instance launched as a
    single-instance plan does (rows_per_inst = 0).  ``env``: an env or a model; ``kw``: emul.launch's (models,
    wpc, kernel, defines).  Returns the per-row outputs and the per-instance final states."""
    m = env.sys.model if hasattr(env, "sys") else env
    nq, nv, nu, nb = m.nq, m.nv, m.nu, m.nbody
    f32 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float32)
    qpos, qvel, warm, us, Ybar, noise = map(f32, (qpos, qvel, warm, us, Ybar, noise))
    B = qpos.shape[0]
    rpi = plan_desc.Nsample + 1 if mode == 1 else 1
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
    fin = {k: out[k] if mode == 0 else None for k in ("qpos_out", "qvel_out", "warm_out", "ctrl_out")}
    emul.launch(env, plan_desc, mode=mode, nrows=nrows, H=H, rows_per_inst=0 if single else rpi, us_row=us_row,
                tasks=task_arr, task_rows=rpi if tasks is not None else 0, qpos0=qpos, qvel0=qvel, warm0=warm,
                counters_in=cin, counters_out=out["counters"] if mode == 0 else None, rng_dev=rng, us=us, Ybar=Ybar,
                noise=noise, rewss=out["rewss"], rews=out["rews"], q=out["q"], qd=out["qd"], xpos=out["xpos"], **fin,
                **kw)
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


def test_batched_rows_equal_single_instance_rows():
    env, o = make_pair("unitree_go2_seq_jump")
    B, N, Hs, Hn = 3, 4, 6, 3
    nu = env.action_size
    rng = np.random.default_rng(5)
    qpos, qvel, warm, Y = _instances(o, B, nu, Hn, rng)
    # counters straddle the first stage boundary of the jump sequence (the env step from step 49 enters stage 1 at dt 0.02, jump_dt 1)
    counters = np.array([[45, 0], [49, 0], [50, 1]], np.int32)
    keys = np.array([[0, 7], [11, 3], [123, 456]], np.uint32)
    noise = 0.9 ** np.arange(Hn + 1)[::-1]
    desc = env.plan_desc(Nsample=N, Hsample=Hs, Hnode=Hn, temp_sample=0.05,
                         M_n2u=interp_matrix(np.linspace(0, 1, Hn + 1), np.linspace(0, 1, Hs + 1)), n_inst=B)

    # planner rows (mode 1, native rng): B (N+1) rows in one launch
    bat = rollout_batched(env, desc, qpos, qvel, warm, counters, rng=keys, Ybar=Y, noise=noise, mode=1, H=Hs + 1)
    rows = N + 1
    for b in range(B):
        one = rollout_batched(env, desc, qpos[b:b + 1], qvel[b:b + 1], warm[b:b + 1], counters[b:b + 1],
                                   rng=keys[b:b + 1], Ybar=Y[b:b + 1], noise=noise, mode=1, H=Hs + 1, single=True)
        sl = slice(b * rows, (b + 1) * rows)
        for k in ("rewss", "rews", "q", "qd", "xpos"):
            assert np.array_equal(bat[k][sl], one[k]), (b, k)
    # the instances differ (different states, keys and knots)
    assert not np.array_equal(bat["rews"][:rows], bat["rews"][rows:2 * rows])

    # env step (mode 0): one row per instance, action Y[b][0], counters advanced per instance
    us_row = (Hn + 1) * nu
    bat = rollout_batched(env, desc, qpos, qvel, warm, counters, us=Y, mode=0, H=1, us_row=us_row)
    for b in range(B):
        one = rollout_batched(env, desc, qpos[b:b + 1], qvel[b:b + 1], warm[b:b + 1], counters[b:b + 1],
                                   us=Y[b:b + 1, :1], mode=0, H=1, single=True)
        for k in ("qpos_out", "qvel_out", "warm_out", "ctrl_out", "counters"):
            assert np.array_equal(bat[k][b], one[k][0]), (b, k)
        assert np.array_equal(bat["rewss"][b], one["rewss"][0]), b
        assert bat["counters"][b, 0] == counters[b, 0] + 1
    assert bat["counters"][1, 1] == 1 and bat["counters"][0, 1] == 0   # instance 1 crossed into stage 1
