"""Per-instance control latency (dial_plan_set_instance_delay, DeviceLoop(..., delay=...)), on the GPU at every
step of the eager, captured and replayed schedule: a predicting instance's planning state after step t is the
plant state after step t + d, bit for bit; delayed instances equal a reference built from eager env steps, a
host FIFO and single-instance loops that plan from a set state; instances without a delay equal a loop without
delays, which launches what it launched before; and the combinations with straddling CTAs, tasks, models,
schedules, ensembles, adaptation and randomize_tasks, the error paths and the CLI."""
import os

import numpy as np
import pytest
import torch
import yaml

from tests.conftest import make_pair
from tests.test_gpu_batch import _config, _instances
from tests.test_gpu_instance_models import _with_sys
from tests.test_gpu_tasks import _cli_runs, _go2_sweep

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLANT = ("qpos", "qvel", "qacc_warmstart", "counters")
OUT = ("Y", "rews", "qbar", "qdbar", "xbar", "rng")


def _loop(name, B, N=32, Hs=8, Hn=4, delay=None, envs=None, **kw):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair(name)
    args = _config(name, N, Hs, Hn)
    states, rngs, Y0 = _instances(envs[0] if envs else env, B, Hn)
    K = len(kw["ensemble"]) if kw.get("ensemble") else 0
    loop = DeviceLoop(MBDPI(args, env, n_instances=B, n_ensemble=K), states, rngs, Y0, envs=envs, delay=delay, **kw)
    return loop, env, args, states, rngs, Y0


def _record(loop, n_steps, n=1, env_step=1):
    """Plant state, planning state and outputs after each of n_steps steps (step 1 eager, 2 captured, then
    replayed)."""
    out = []
    for _ in range(n_steps):
        loop.step(n, env_step=env_step)
        ps = loop.planning_state()
        torch.cuda.synchronize()
        out.append(dict({k: loop.buf[k].clone() for k in PLANT + OUT + ("reward", "ctrl")},
                        plan={k: v.clone() for k, v in zip(PLANT, (ps["qpos"], ps["qvel"], ps["qacc_warmstart"],
                                                                      ps["counters"]))}))
    return out


DELAYS = [{"steps": 2, "predict": True}, {"steps": 5, "predict": True}, 3, 0]


@pytest.mark.parametrize("name, force_generic", [("unitree_go2_walk", False), ("unitree_go2_seq_jump", False),
                                                 ("unitree_h1_walk", False), ("allegro_reorient", False),
                                                 ("unitree_go2_walk", True)])
def test_prediction_is_the_plant_d_steps_later(built, monkeypatch, name, force_generic):
    if force_generic:
        monkeypatch.setenv("DIAL_FORCE_GENERIC_TREE", "1")
    loop, *_ = _loop(name, 4, N=16, Hs=6, Hn=3, delay=DELAYS)
    rec = _record(loop, 12)
    for b, d in ((0, 2), (1, 5)):
        for t in range(len(rec) - d):
            for k in PLANT:
                assert torch.equal(rec[t]["plan"][k][b], rec[t + d][k][b]), (name, b, t, k)
    for b in (2, 3):   # not predicting: the plant state
        for t, r in enumerate(rec):
            for k in PLANT:
                assert torch.equal(r["plan"][k][b], r[k][b]), (name, b, t, k)
    # the queue of instance 2 holds the knots of its last three steps, in application order
    pend = loop.pending_actions()
    assert pend.shape == (4, 16, loop.mbdpi.nu) and not pend[2, 3:].any() and not pend[3].any()
    assert pend[2, :3].abs().sum() > 0


def _reference(env, args, state, rng, Y0, d, predict, n_steps, n=1, plan_env=None):
    """Instance with delay d restated from parts that exist: a held plant state stepped eagerly with the front of
    a host FIFO, and a single-instance loop that plans (env_step 2) from it, or from d eager env steps on the
    planning model with the queued actions."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    loop = DeviceLoop(MBDPI(args, env), state, rng, Y0)
    fifo = [Y0[0].clone() for _ in range(d)]
    plant, out = state, []
    for _ in range(n_steps):
        fifo.append(loop.action.clone())
        a = fifo.pop(0)
        plant = env.step(plant, a)
        s = plant
        if predict:
            for u in fifo:
                s = (plan_env or env).step(s, u)
        ps = s.pipeline_state
        loop.set_state(ps.qpos, ps.qvel, ps.qacc_warmstart, step=s.info["step"])
        loop.step(n, env_step=2)
        torch.cuda.synchronize()
        pp = plant.pipeline_state
        out.append(dict({k: loop.buf[k].clone() for k in OUT}, qpos=pp.qpos.clone(), qvel=pp.qvel.clone(),
                        qacc_warmstart=pp.qacc_warmstart.clone(), reward=plant.reward, plan_qpos=ps.qpos.clone()))
    return out


@pytest.mark.parametrize("B, N", [(4, 32), (24, 100)])   # 24 x 101 rows: the plain layout straddles CTAs
def test_delayed_instances_equal_the_reference(built, B, N):
    from dial_mpc_b200.core.dial_core import delay_setting
    delays = [DELAYS[b % 4] for b in range(B)]
    loop, env, args, states, rngs, Y0 = _loop("unitree_go2_walk", B, N=N, delay=delays)
    rec = _record(loop, 8)
    for b in (0, 1, 2, 3) if B == 4 else (0, 1, 2, 3, 13, 22):
        d, predict = delay_setting(delays[b])
        ref = _reference(env, args, states[b], rngs[b], Y0[b], d, predict, len(rec))
        for t, (got, want) in enumerate(zip(rec, ref)):
            for k in OUT + ("qpos", "qvel", "qacc_warmstart"):
                assert torch.equal(got[k][b], want[k]), (b, t, k)
            assert torch.equal(got["reward"][b], torch.as_tensor(want["reward"], device="cuda").reshape(())), (b, t)
            assert torch.equal(got["plan"]["qpos"][b], want["plan_qpos"]), (b, t)


def test_undelayed_instances_and_launches(built):
    """Instances with d = 0 in a mixed batch equal a loop without delays; a loop that never set a delay launches
    env step + shift + (rollout + update + 2 bars) per iteration; the delays add the queue launch and one launch
    per prediction step; a setter that keeps the largest delays keeps the launch sequence."""
    plain, *_ = _loop("unitree_go2_walk", 3)
    mixed, *_ = _loop("unitree_go2_walk", 3, delay=[0, {"steps": 3, "predict": True}, 0])
    a, b = _record(plain, 6, n=2), _record(mixed, 6, n=2)
    for t in range(6):
        for k in OUT + PLANT:
            for i in (0, 2):
                assert torch.equal(a[t][k][i], b[t][k][i]), (t, k, i)
        assert not torch.equal(a[t]["Y"][1], b[t]["Y"][1])

    def per_step(loop, es):
        c0 = loop.plan.lib.dial_launch_count(loop.plan.handle)
        loop.step(2, env_step=es)
        return loop.plan.lib.dial_launch_count(loop.plan.handle) - c0

    for es, base in ((1, 2 + 2 * 4), (0, 2 * 4), (2, 1 + 2 * 4)):
        assert [per_step(plain, es) for _ in range(3)] == [base] * 3, es
        assert [per_step(mixed, es) for _ in range(3)] == [base + 1 + 3] * 3, es
    # instance 0's delay changes below the largest: the same launch sequence
    mixed.set_delay(0, 2)
    assert per_step(mixed, 1) == 2 + 2 * 4 + 1 + 3


def test_delay_with_tasks_models_and_schedules(built):
    """Per-instance tasks, plant models and schedules (one instance with no diffusion iterations): the
    prediction still equals the instance's plant d steps later."""
    envs = _go2_sweep()
    envs[2] = _with_sys(envs[2], {"body_mass": {"base": envs[2].sys.model.arrays["body_mass"][1] + 3.0}})
    sched = [{"Ndiffuse": 2, "temp_sample": 0.08}, None, {"Ndiffuse": 1}]
    loop, *_ = _loop("unitree_go2_walk", 3, envs=envs, schedule=sched,
                     delay=[{"steps": 2, "predict": True}, {"steps": 1, "predict": True}, {"steps": 4, "predict": True}])
    rec = []
    for t in range(10):
        if t == 4:
            loop.plan.set_instance_iterations([2, 0, 1])   # instance 1 is only env-stepped, shifted and predicted
        loop.plan.mpc_step(2, 1)
        ps = loop.planning_state()
        torch.cuda.synchronize()
        rec.append(dict({k: loop.buf[k].clone() for k in PLANT}, plan=ps))
    for b, d in enumerate((2, 1, 4)):
        for t in range(len(rec) - d):
            for k, kk in zip(PLANT, ("qpos", "qvel", "qacc_warmstart", "counters")):
                assert torch.equal(rec[t]["plan"][kk][b], rec[t + d][k][b]), (b, t, k)


def test_nominal_ensemble_prediction_error(built):
    """A K = 1 nominal ensemble planning for a heavier plant: the prediction runs on the nominal model, so it
    misses the plant d steps later, and equals d eager env steps of the nominal model from the plant state with
    the queued actions."""
    env, _ = make_pair("unitree_go2_walk")
    heavy = _with_sys(env, {"body_mass": {"base": env.sys.model.arrays["body_mass"][1] + 4.0}})
    d = 3
    loop, _, args, states, *_ = _loop("unitree_go2_walk", 2, envs=[heavy, heavy], ensemble=[env],
                                      delay={"steps": d, "predict": True})
    pred, plant = [], []
    for t in range(10):
        loop.step(1, env_step=1)
        ps = loop.planning_state()
        pend = loop.pending_actions()   # the queue the step's prediction applied, after its env step
        torch.cuda.synchronize()
        for b in range(2):
            s = loop.state(b)
            for j in range(d):
                s = env.step(s, pend[b, j].clone())
            p = s.pipeline_state
            for k, want in (("qpos", p.qpos), ("qvel", p.qvel), ("qacc_warmstart", p.qacc_warmstart)):
                assert torch.equal(ps[k][b], want), (t, b, k)
            assert int(ps["counters"][b, 0]) == s.info["step"], (t, b)
        pred.append(ps["qpos"].clone())
        plant.append(loop.buf["qpos"].clone())
    # the heavier plant d steps later is not where the nominal model predicted it
    err = torch.stack([(pred[t] - plant[t + d])[:, :3] for t in range(len(pred) - d)])
    assert err.abs().max() > 0


def test_adaptation_scores_the_applied_action(built):
    """With a delay, the members predict the env step under the action the plant applies: the member equal to
    the plant scores l = 0 exactly."""
    env, _ = make_pair("unitree_go2_walk")
    heavy = _with_sys(env, {"body_mass": {"base": env.sys.model.arrays["body_mass"][1] + 4.0}})
    loop, *_ = _loop("unitree_go2_walk", 2, envs=[heavy, heavy], ensemble=[env, heavy],
                     adapt={"sigma": 0.5}, delay=[{"steps": 3, "predict": True}, 2])
    for t in range(6):
        loop.step(1, env_step=1)
        ell = loop.member_loglik()
        torch.cuda.synchronize()
        assert torch.all(ell[:, 1] == 0), (t, ell)
        assert torch.all(ell[:, 0] < 0), (t, ell)


def test_randomize_tasks_window_reaches_the_prediction(built):
    """Batched randomize_tasks with a predicting instance whose rollouts reach step 500 from the first step on:
    its one-step command is bound then (the window grows by d), and its prediction through step 500 still
    equals its plant d steps later."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    from tests.test_gpu_tasks import _env
    env = _env("unitree_go2_walk", randomize_tasks=True)
    args = _config("unitree_go2_walk", 16, 6, 3)
    states, rngs, Y0 = _instances(env, 2, 3, start_step=488)   # instance 1 at step 489
    d = 6
    loop = DeviceLoop(MBDPI(args, env, n_instances=2), states, rngs, Y0, delay=[{"steps": d, "predict": True}, 0])
    loop.step(1, env_step=1)
    # instance 0: env step at 488, prediction 489..494, rollouts 495..501; instance 1: env step and rollouts 489..497
    assert loop._task_cmd[0] is not None and loop._task_cmd[0][0] == 500
    assert loop._task_cmd[1] is None
    rec = _record(loop, 14)
    for t in range(len(rec) - d):
        for k in PLANT:
            assert torch.equal(rec[t]["plan"][k][0], rec[t + d][k][0]), (t, k)


def test_errors(built):
    loop, *_ = _loop("unitree_go2_walk", 2)
    with pytest.raises(IndexError, match=r"instance 2 out of range"):
        loop.set_delay(2, 1)
    with pytest.raises(ValueError, match=r"steps must be an int in 0\.\.16, got 17"):
        loop.set_delay(0, 17)
    with pytest.raises(RuntimeError, match=r"dial_plan_set_instance_delay: steps 17 out of range \(0\.\.16\)"):
        loop.plan.set_instance_delay(0, 17)
    with pytest.raises(RuntimeError, match=r"dial_plan_set_instance_delay: instance -1 out of range"):
        loop.plan.set_instance_delay(-1, 1)
    with pytest.raises(RuntimeError, match=r"predict must be 0 or 1, got 2"):
        loop.plan._check(loop.plan.lib.dial_plan_set_instance_delay(loop.plan.handle, 0, 1, 2, None))
    with pytest.raises(ValueError, match=r"delay must be one delay spec or a list of 2, got a list of 3"):
        _loop("unitree_go2_walk", 2, delay=[1, 2, 3])
    # a plan without delays: empty queues
    assert not loop.pending_actions().any()


def test_cli_delay(built, tmp_path):
    base = yaml.safe_load(open(os.path.join(ROOT, "dial_mpc_b200", "examples", "unitree_go2_trot.yaml")))
    base.update(Nsample=64, Hsample=8, Hnode=4, Ndiffuse=1, Ndiffuse_init=1)
    ov = tmp_path / "ov.yaml"
    ov.write_text(yaml.safe_dump([{}, {"delay": {"steps": 2, "predict": True}}]))
    out = _cli_runs(tmp_path, {"one": (base, ["--delay", "2:predict"]),
                               "two": (base, ["--instances", "2", "--delay", "3", "--instance-overrides", str(ov)]),
                               "plain": (base, [])})
    assert len(out["one"][0]) == 1 and len(out["two"][0]) == 2
    # the delayed single run differs from the plain one
    assert not np.array_equal(np.load(out["one"][0][0]), np.load(out["plain"][0][0]))
