"""Per-instance observation (dial_plan_set_instance_observation, DeviceLoop(..., observe=...)), on the GPU at every
step of the eager, captured and replayed schedule: with zero noise an instance observes its plant min(k, t) steps
earlier and a predicting one plans from its plant d steps later, bit for bit; the noise is the oracle's restated
draw within the CPU tolerances (tests/test_instance_observation.py), and the rollouts start from the observation;
instances without a setting equal a loop without observations, which launches what it launched before; and the
combinations with straddling CTAs, tasks, models, schedules and ensembles, the error paths and the CLI."""
import os

import numpy as np
import pytest
import torch
import yaml

from dial_mpc_b200 import random as drandom
from tests.conftest import make_pair
from tests.test_gpu_batch import _config, _instances
from tests.test_gpu_instance_models import _with_sys
from tests.test_gpu_tasks import _cli_runs, _go2_sweep
from tests.test_instance_observation import EPS_ULP, QUAT_TOL, _noise_ref, _ulp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLANT = ("qpos", "qvel", "qacc_warmstart", "counters")
OUT = ("Y", "rews", "qbar", "qdbar", "xbar", "rng")


def _loop(name, B, N=32, Hs=8, Hn=4, envs=None, **kw):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair(name)
    args = _config(name, N, Hs, Hn)
    states, rngs, Y0 = _instances(envs[0] if envs else env, B, Hn)
    K = len(kw["ensemble"]) if kw.get("ensemble") else 0
    loop = DeviceLoop(MBDPI(args, env, n_instances=B, n_ensemble=K), states, rngs, Y0, envs=envs, **kw)
    return loop, env, args, states, rngs, Y0


def _record(loop, n_steps, n=1, env_step=1):
    """Plant, observed and planning state, outputs and the queue's front (the action the step applied) after
    each of n_steps steps (step 1 eager, 2 captured, then replayed)."""
    out = []
    for _ in range(n_steps):
        front = loop.pending_actions()[..., 0, :].clone()
        loop.step(n, env_step=env_step)
        ps, ob = loop.planning_state(), loop.observed_state()
        torch.cuda.synchronize()
        out.append(dict({k: loop.buf[k].clone() for k in PLANT + OUT + ("reward", "ctrl")}, front=front,
                        plan={k: v.clone() for k, v in zip(PLANT, (ps["qpos"], ps["qvel"], ps["qacc_warmstart"],
                                                                      ps["counters"]))},
                        obs={k: v.clone() for k, v in zip(PLANT + ("age",), (ob["qpos"], ob["qvel"],
                                                                            ob["qacc_warmstart"], ob["counters"],
                                                                            ob["age"]))}))
    return out


OBSERVE = [{"delay": 2}, {"delay": 5}, None, {"delay": 0}]


def _check_observed(rec, b, k):
    for t, r in enumerate(rec):
        age = min(k, t)
        assert int(r["obs"]["age"][b]) == age, (b, t)
        for key in PLANT:
            assert torch.equal(r["obs"][key][b], rec[t - age][key][b]), (b, t, key)


@pytest.mark.parametrize("name, force_generic", [("unitree_go2_walk", False), ("unitree_go2_seq_jump", False),
                                                 ("unitree_h1_walk", False), ("allegro_reorient", False),
                                                 ("unitree_go2_walk", True)])
def test_observation_is_the_plant_k_steps_earlier(built, monkeypatch, name, force_generic):
    """Zero noise, no prediction: the observed and the planning state after step t are the plant after step
    t - min(k, t)."""
    if force_generic:
        monkeypatch.setenv("DIAL_FORCE_GENERIC_TREE", "1")
    loop, *_ = _loop(name, 4, N=16, Hs=6, Hn=3, observe=OBSERVE)
    rec = _record(loop, 10)
    for b, k in enumerate((2, 5, 0, 0)):
        _check_observed(rec, b, k)
        for t, r in enumerate(rec):
            for key in PLANT:
                assert torch.equal(r["plan"][key][b], r["obs"][key][b]), (name, b, t, key)


def _check_prediction(rec, b, d):
    for t in range(len(rec) - d):
        for key in PLANT:
            assert torch.equal(rec[t]["plan"][key][b], rec[t + d][key][b]), (b, t, key)


def test_prediction_through_observation_and_action_delay(built):
    """Zero noise, observation delay k, action delay d, predicting: the planning state after step t is the plant
    after step t + d, for (k, d) = (2, 1), (3, 0), (1, 3), (4, 2), with per-instance tasks, a heavier plant model
    and schedules, and an instance that runs no diffusion iteration."""
    envs = _go2_sweep() + [_go2_sweep()[0]]
    envs[2] = _with_sys(envs[2], {"body_mass": {"base": envs[2].sys.model.arrays["body_mass"][1] + 3.0}})
    kd = [(2, 1), (3, 0), (1, 3), (4, 2)]
    loop, *_ = _loop("unitree_go2_walk", 4, envs=envs, schedule=[{"Ndiffuse": 2, "temp_sample": 0.08}, None,
                                                                  {"Ndiffuse": 1}, None],
                     delay=[{"steps": d, "predict": True} for _, d in kd], observe=[{"delay": k} for k, _ in kd])
    rec = []
    for t in range(12):
        if t == 4:
            loop.plan.set_instance_iterations([2, 0, 1, 2])   # instance 1 is only env-stepped, shifted and predicted
        rec += _record(loop, 1, n=2)
    for b, (k, d) in enumerate(kd):
        _check_prediction(rec, b, d)
        _check_observed(rec, b, k)


@pytest.mark.parametrize("B, N", [(4, 32), (24, 100)])   # 24 x 101 rows: the plain layout straddles CTAs
def test_noise_and_rollouts_from_the_observation(built, B, N):
    """The observed state is the plant record plus the noise restated from the oracle's sampler (CPU
    tolerances), with sigma-0 dofs copied; a single-instance loop set to the GPU's observed state plans (env_step
    2) the batched instance's outputs bit for bit: the rollouts start from the observation."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI, observe_setting
    spec = lambda b: {"delay": b % 3, "qpos": {"": [0.01, 0.01, 0.01, 0.05, 0.05, 0.05], "FR_thigh_joint": 0.03},
                      "qvel": 0.2 * (b % 2), "seed": b % 2}
    loop, env, args, states, rngs, Y0 = _loop("unitree_go2_walk", B, N=N, observe=[spec(b) for b in range(B)])
    rec = _record(loop, 6)
    model = env.sys.model
    for b in (0, 1, 2, 3) if B == 4 else (0, 1, 13, 22):
        k, sq, sv, key = observe_setting(spec(b), env.sys)
        subs = []
        for _ in rec:
            key, sub = drandom.split(key)
            subs.append(sub)
        ref = DeviceLoop(MBDPI(args, env), states[b], rngs[b], Y0[b])
        for t, r in enumerate(rec):
            age = min(k, t)
            plant = {"qpos": rec[t - age]["qpos"][b].cpu().numpy(), "qvel": rec[t - age]["qvel"][b].cpu().numpy()}
            q, v, quats, eps = _noise_ref(model, plant, subs[t], sq, sv)
            got_q, got_v = r["obs"]["qpos"][b].cpu().numpy(), r["obs"]["qvel"][b].cpu().numpy()
            for i in range(model.nv):
                tol = EPS_ULP * float(sv[i]) * _ulp(eps[model.nv + i]) + _ulp(v[i])
                assert abs(got_v[i] - v[i]) <= tol if sv[i] else got_v[i].tobytes() == plant["qvel"][i].tobytes()
            for i in range(model.nq):
                if 3 <= i < 7:
                    continue
                dof = i if i < 3 else i - 1
                tol = EPS_ULP * float(sq[dof]) * _ulp(eps[dof]) + _ulp(q[i])
                assert abs(got_q[i] - q[i]) <= tol if sq[dof] else got_q[i].tobytes() == plant["qpos"][i].tobytes(), (b, t, i)
            assert np.abs(got_q[3:7] - q[3:7]).max() <= QUAT_TOL, (b, t)
            assert torch.equal(r["obs"]["qacc_warmstart"][b], rec[t - age]["qacc_warmstart"][b])
            # the rollouts start from the observation
            o = r["obs"]
            ref.set_state(o["qpos"][b], o["qvel"][b], o["qacc_warmstart"][b], step=int(o["counters"][b, 0]))
            ref.step(1, env_step=2)
            torch.cuda.synchronize()
            for key_ in OUT:
                assert torch.equal(ref.buf[key_], r[key_][b]), (b, t, key_)


def test_unobserved_instances_and_launches(built):
    """Instances without a setting in a mixed batch equal a loop without observations; a loop that never set one
    launches env step + shift + (rollout + update + 2 bars) per iteration; observation adds the observe launch
    and max(k + d) prediction launches over the predicting instances; a setter that keeps that maximum keeps the
    launch sequence."""
    plain, *_ = _loop("unitree_go2_walk", 3)
    mixed, *_ = _loop("unitree_go2_walk", 3, observe=[None, {"delay": 3, "qpos": 0.02}, None])
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

    pred, *_ = _loop("unitree_go2_walk", 3, delay=[0, {"steps": 2, "predict": True}, 0],
                     observe=[None, {"delay": 3}, {"delay": 6}])
    for es, base in ((1, 2 + 2 * 4), (0, 2 * 4), (2, 1 + 2 * 4)):
        assert [per_step(plain, es) for _ in range(3)] == [base] * 3, es
        assert [per_step(mixed, es) for _ in range(3)] == [base + 1] * 3, es
        # the queue launch (steps with an env step, or while a delay predicts), observe, 3 + 2 prediction launches
        assert [per_step(pred, es) for _ in range(3)] == [base + 1 + 1 + 5] * 3, es
    # settings that keep max(k + d) over the predicting instances keep the launch sequence
    pred.set_observation(2, {"delay": 1, "qvel": 0.1})
    pred.set_observation(1, {"delay": 3, "qpos": 0.01})
    assert per_step(pred, 1) == 2 + 2 * 4 + 1 + 1 + 5
    pred.set_observation(1, {"delay": 1})
    assert per_step(pred, 1) == 2 + 2 * 4 + 1 + 1 + 3
    # removing every setting: plans from the plant again (the observe launch stays)
    mixed.set_observation(1, None)
    r = _record(mixed, 2, n=2)
    for t in range(2):
        for k in PLANT:
            assert torch.equal(r[t]["plan"][k], r[t][k]), (t, k)


def test_nominal_ensemble_prediction_error(built):
    """A K = 1 nominal ensemble planning for a plant 4 kg heavier, observing 2 steps late and acting 1 step late:
    the prediction equals eager env steps of the nominal model from the observed state with the applied actions
    since it and the queued one, and misses the plant."""
    from dial_mpc_b200.envs.base_env import PipelineState
    env, _ = make_pair("unitree_go2_walk")
    heavy = _with_sys(env, {"body_mass": {"base": env.sys.model.arrays["body_mass"][1] + 4.0}})
    k, d = 2, 1
    loop, *_ = _loop("unitree_go2_walk", 2, envs=[heavy, heavy], ensemble=[env],
                     delay={"steps": d, "predict": True}, observe={"delay": k})
    rec, err = [], []
    for t in range(10):
        rec += _record(loop, 1)
        pend = loop.pending_actions()
        torch.cuda.synchronize()
        r = rec[-1]
        for b in range(2):
            age = int(r["obs"]["age"][b])
            s = loop.state(b)
            s = s.replace(pipeline_state=PipelineState(r["obs"]["qpos"][b].clone(), r["obs"]["qvel"][b].clone(),
                                                       r["obs"]["qacc_warmstart"][b].clone(), s.pipeline_state.ctrl),
                          info=dict(s.info, step=int(r["obs"]["counters"][b, 0])))
            for u in [rec[t - age + 1 + j]["front"][b] for j in range(age)] + [pend[b, j] for j in range(d)]:
                s = env.step(s, u.clone())
            p = s.pipeline_state
            for key, want in (("qpos", p.qpos), ("qvel", p.qvel), ("qacc_warmstart", p.qacc_warmstart)):
                assert torch.equal(r["plan"][key][b], want), (t, b, key)
            assert int(r["plan"]["counters"][b, 0]) == s.info["step"], (t, b)
    for t in range(len(rec) - d):
        err.append((rec[t]["plan"]["qpos"] - rec[t + d]["qpos"])[:, :3].abs().max())
    assert max(err) > 0


def test_errors(built):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    from tests.test_gpu_tasks import _env
    loop, env, *_ = _loop("unitree_go2_walk", 2)
    nv = env.sys.nv
    with pytest.raises(IndexError, match=r"instance 2 out of range"):
        loop.set_observation(2, {"delay": 1})
    with pytest.raises(RuntimeError, match=r"dial_plan_set_instance_observation: instance -1 out of range"):
        loop.plan.set_instance_observation(-1, 1)
    with pytest.raises(ValueError, match=r"delay must be an int in 0\.\.16, got 17"):
        loop.set_observation(0, {"delay": 17})
    with pytest.raises(RuntimeError, match=r"dial_plan_set_instance_observation: delay 17 out of range \(0\.\.16\)"):
        loop.plan.set_instance_observation(0, 17)
    bad = np.zeros(nv, np.float32)
    bad[4] = np.nan
    with pytest.raises(RuntimeError, match=r"qpos_std\[4\] = nan must be finite and >= 0"):
        loop.plan.set_instance_observation(0, 1, bad)
    bad[4] = -0.5
    with pytest.raises(RuntimeError, match=r"qvel_std\[4\] = -0\.5\d* must be finite and >= 0"):
        loop.plan.set_instance_observation(0, 1, None, bad)
    # k + d > 16, from either setter order
    loop.set_delay(0, {"steps": 10, "predict": True})
    with pytest.raises(RuntimeError, match=r"delay 7 plus instance 0's action delay 10 exceeds 16"):
        loop.set_observation(0, {"delay": 7})
    loop.set_observation(1, {"delay": 9})
    with pytest.raises(RuntimeError, match=r"steps 8 plus instance 1's observation delay 9 exceeds 16"):
        loop.set_delay(1, 8)
    with pytest.raises(ValueError, match=r"observe must be one observe spec or a list of 2, got a list of 3"):
        _loop("unitree_go2_walk", 2, observe=[{}, {}, {}])
    # sharded plans
    from dial_mpc_b200.plan import Plan
    from dial_mpc_b200.utils.spline import interp_matrix
    args = _config("unitree_go2_walk", 16, 4, 2)
    desc = env.plan_desc(Nsample=16, Hsample=4, Hnode=2, temp_sample=0.05,
                         M_n2u=interp_matrix(np.linspace(0, 1, 3), np.linspace(0, 1, 5)))
    desc.Ntotal = 32
    sharded = Plan(env, desc)
    with pytest.raises(RuntimeError, match=r"sharded plans \(Ntotal != Nsample\) have no per-instance observation"):
        sharded.set_instance_observation(0, 1)
    # randomize_tasks: an observation delay is rejected, noise alone is allowed
    renv = _env("unitree_go2_walk", randomize_tasks=True)
    states, rngs, Y0 = _instances(renv, 2, 2)
    with pytest.raises(ValueError, match=r"an observation delay needs a loop without randomize_tasks"):
        DeviceLoop(MBDPI(args, renv, n_instances=2), states, rngs, Y0, observe={"delay": 1})
    ok = DeviceLoop(MBDPI(args, renv, n_instances=2), states, rngs, Y0, observe={"qvel": 0.1})
    ok.step(1)
    with pytest.raises(ValueError, match=r"an observation delay needs a loop without randomize_tasks"):
        ok.set_observation(0, {"delay": 2})
    # a plan without observations observes its plant at age 0
    fresh, *_ = _loop("unitree_go2_walk", 2)
    ob = fresh.observed_state()
    assert not ob["age"].any() and torch.equal(ob["qpos"], fresh.buf["qpos"])


def test_set_state_resets_the_history(built):
    """set_state seeds every observing instance's ring again from the new state: its observation ramps from
    age 0, and its noise restarts from its seed."""
    loop, *_ = _loop("unitree_go2_walk", 2, observe=[{"delay": 3, "qvel": 0.1}, None])
    first = _record(loop, 5)
    s0 = first[0]
    loop.set_state(s0["qpos"], s0["qvel"], s0["qacc_warmstart"], step=s0["counters"][:, 0].cpu().numpy())
    again = _record(loop, 4, env_step=0)
    for t, r in enumerate(again):
        assert int(r["obs"]["age"][0]) == 0, t       # no env step: the seed stays the only record
        assert torch.equal(r["obs"]["qvel"][0], first[0]["obs"]["qvel"][0]), t   # the same state, the first draw
        assert torch.equal(r["obs"]["qpos"][1], s0["qpos"][1]), t


def test_cli_observe(built, tmp_path):
    base = yaml.safe_load(open(os.path.join(ROOT, "dial_mpc_b200", "examples", "unitree_go2_trot.yaml")))
    base.update(Nsample=64, Hsample=8, Hnode=4, Ndiffuse=1, Ndiffuse_init=1)
    ov = tmp_path / "ov.yaml"
    ov.write_text(yaml.safe_dump([{}, {"observe": {"delay": 2, "qvel": 0.1}}]))
    out = _cli_runs(tmp_path, {"one": (base, ["--observe", "{delay: 2, qpos: 0.01}"]),
                               "two": (base, ["--instances", "2", "--observe", "{delay: 1}", "--instance-overrides",
                                              str(ov)]),
                               "plain": (base, [])})
    assert len(out["one"][0]) == 1 and len(out["two"][0]) == 2
    assert not np.array_equal(np.load(out["one"][0][0]), np.load(out["plain"][0][0]))
