"""The CUDA build's built-in rewards against fp64 on the kernel's own states (fp64_rewards in
test_reward_parity.py): the start states on the edges of each reward term on every kernel variant that
computes them, a batched DeviceLoop whose instances carry unlike tasks, and the seq-jump stage at every
stage boundary of twelve-stage tasks with jump_dt that is not a power of two.

Tolerance: REWARD_TOL = 1e-5 * (1 + |r|) per env step, the bound of the emulator test.  Largest
relative error measured on an H100 80GB HBM3 (700 W power limit), per env and kernel:
  Go2 walk       go2 1.6e-6, v1 1.6e-6, generic tree 1.9e-6
  Go2 seq-jump   go2 6.4e-8, v1 6.4e-8, generic tree 6.4e-8 (7 steps of ~25000 dropped in the fp32 band)
  H1 walk, loco  v2 / v4 9.6e-7, generic tree 9.5e-7
  Allegro        dense 2.8e-8
  batched DeviceLoop env steps: Go2 walk 2.5e-7, Go2 seq-jump 1.2e-7"""
import json

import numpy as np
import pytest
import torch

from tests.test_reward_parity import (JUMP_DT, N_STAGE, REWARD_TOL, _jump_pair, all_cases, check_case,
                                      check_jump_coverage, fp64_rewards, host_stage, last_boundary, make_pair,
                                      stage_from_reward)

pytestmark = pytest.mark.gpu
ROWS = 96          # rows spread over multi-warp CTAs

# kernel variant -> environment variables at plan creation
VARIANTS = {"default": {}, "v1": {"DIAL_FORCE_GENERIC_SHAPE": "1"}, "tree": {"DIAL_FORCE_GENERIC_TREE": "1"}}
GROUPS = [("unitree_go2_walk", "default"), ("unitree_go2_walk", "v1"), ("unitree_go2_walk", "tree"),
          ("unitree_go2_seq_jump", "default"), ("unitree_go2_seq_jump", "v1"), ("unitree_go2_seq_jump", "tree"),
          ("unitree_h1", "default"), ("unitree_h1", "tree"), ("allegro_reorient", "default")]


def _state(plan, qpos, qvel, step, stage):
    from dial_mpc_b200.envs.base_env import PipelineState, State
    ps = PipelineState(plan.f32(qpos), plan.f32(qvel), plan.f32(np.zeros(len(qvel))))
    return State(ps, None, 0.0, 0.0, {}, {"step": int(step), "contact_stage": int(stage)})


def _gpu_run(env, desc, case, us):
    """rewss, q, qd of a rollout of every row, and the ctrl of row 0's last step from an env step at that
    step's pre-state (the env-step path of the same kernel)."""
    from dial_mpc_b200.plan import Plan
    plan = Plan(env, desc)
    if case.cmd is not None:        # a plan takes its command override through dial_plan_set_command only
        plan.set_command(case.cmd)
    rewss, q, qd, _ = plan.rollout(_state(plan, case.qpos, case.qvel, case.step, case.stage), us)
    H = us.shape[1]
    q, qd = q.cpu().numpy(), qd.cpu().numpy()
    qp, vp = (case.qpos, case.qvel) if H == 1 else (q[0, H - 2], qd[0, H - 2])
    # the stage only selects reward terms: the ctrl does not depend on it
    ps, _ = plan.env_step(_state(plan, qp, vp, case.step + H - 1, 0), us[0, H - 1])
    torch.cuda.synchronize()
    return rewss.cpu().numpy(), q, qd, ps.ctrl.cpu().numpy()


@pytest.mark.parametrize("group,variant", GROUPS)
def test_rewards_match_fp64_at_term_edges(built, monkeypatch, group, variant):
    for k, v in VARIANTS[variant].items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(5)
    results = [check_case(c, _gpu_run, ROWS, rng) for c in all_cases()[group]]
    rep = dict(group=group, variant=variant, worst=max(r[0] for r in results))
    if group == "unitree_go2_seq_jump":
        rep["branches"] = check_jump_coverage(results)
        rep["dropped"] = int(sum((~r[1]).sum() for r in results))
    print("reward parity", json.dumps(rep))


def _batched_rewards(name, envs, qpos, qvel, steps, stages, n_steps=3):
    """A batched DeviceLoop, instance b on envs[b]'s task from (qpos[b], qvel[b]) at steps[b] / stages[b]:
    every env step's reward (loop.reward) against fp64 of b's own pre-state, action and task."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    from tests.test_gpu_batch import _config, _instances
    B = len(envs)
    args = _config(name, 64, 8, 4)
    states, rngs, Y0 = _instances(envs[0], B, 4)
    states = [s.replace(info=dict(s.info, step=int(steps[b]), **({"contact_stage": int(stages[b])} if "contact_stage" in s.info else {})))
              for b, s in enumerate(states)]
    loop = DeviceLoop(MBDPI(args, envs[0], n_instances=B), states, rngs, Y0, envs=envs)
    loop.set_state(np.stack(qpos), np.stack(qvel), np.zeros((B, len(qvel[0]))))
    oracles = [make_pair(name, **e._test_over)[1] for e in envs]
    worst = 0.0
    for _ in range(n_steps):
        torch.cuda.synchronize()
        q0, v0 = loop.buf["qpos"].cpu().numpy(), loop.buf["qvel"].cpu().numpy()
        cnt, act = loop.buf["counters"].cpu().numpy(), loop.action.cpu().numpy().astype(np.float64)
        loop.step(2, env_step=1)
        torch.cuda.synchronize()
        q1, v1, r = loop.buf["qpos"].cpu().numpy(), loop.buf["qvel"].cpu().numpy(), loop.reward.cpu().numpy()
        for b, o in enumerate(oracles):
            ref, *_ = fp64_rewards(o, q0[b], v0[b], int(cnt[b, 0]), int(cnt[b, 1]), act[b][None, None],
                                   q1[b][None, None], v1[b][None, None])
            err = abs(r[b] - ref[0, 0]) / (1 + abs(ref[0, 0]))
            assert err < REWARD_TOL, (name, b, int(cnt[b, 0]), float(err))
            worst = max(worst, float(err))
    return worst


def _env(name, **over):
    env, _ = make_pair(name, **over)
    env._test_over = over
    return env


def test_batched_loop_rewards_of_unlike_tasks(built):
    """Go2 walk instances with every gait and commands of either sign (ramps before and after their end),
    and seq-jump instances with their own jump sequences and jump_dt, started next to stage boundaries."""
    cases = all_cases()
    walk = [("trot", 0.8, 0.0, 0.0), ("walk", -0.9, -0.3, -0.6), ("stand", 0.2, 0.1, 0.5), ("canter", 1.2, 0.0, -1.0),
            ("gallop", -0.4, 0.3, 1.3), ("trot", -1.5, 0.5, 0.0), ("walk", 0.5, -0.2, 1.5), ("stand", -0.3, 0.0, -1.2)]
    envs = [_env("unitree_go2_walk", gait=g, default_vx=vx, default_vy=vy, default_vyaw=w) for g, vx, vy, w in walk]
    starts = cases["unitree_go2_walk"][:len(envs)]
    steps = [0, 30, 48, 49, 50, 120, 333, 498]
    w_walk = _batched_rewards("unitree_go2_walk", envs, [c.qpos for c in starts], [c.qvel for c in starts], steps,
                              [0] * len(envs))
    far = dict(pose_target_sequence=[[100.0 * j, 0.0, 0.27] for j in range(N_STAGE)], yaw_target_sequence=[0.0] * N_STAGE)
    turn = dict(pose_target_sequence=[[0, 0, 0.27], [0.3, 0.2, 0.3], [0.5, -0.1, 0.25]], yaw_target_sequence=[0.0, 0.6, -0.4])
    jumps = [({}, 48), (dict(far, jump_dt=0.3), 13), (dict(turn, jump_dt=0.55), 26), (dict(far, jump_dt=1.1), 163),
             (dict(turn, jump_dt=0.85), 83), ({"jump_dt": 0.6}, 28)]
    envs = [_env("unitree_go2_seq_jump", **over) for over, _ in jumps]
    starts = cases["unitree_go2_seq_jump"][:len(envs)]
    stg = [host_stage(e, s - 1) for e, (_, s) in zip(envs, jumps)]
    w_jump = _batched_rewards("unitree_go2_seq_jump", envs, [c.qpos for c in starts], [c.qvel for c in starts],
                              [s for _, s in jumps], stg)
    print("reward parity", json.dumps(dict(batched_walk=w_walk, batched_jump=w_jump)))


@pytest.mark.parametrize("variant", ["default", "v1"])
def test_stage_at_every_boundary(built, monkeypatch, variant):
    """Device counters after one env step of a batched DeviceLoop (one instance per boundary and side, each
    with its own jump_dt) and the stage a rollout's reward scored at the step after, against the host."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    from dial_mpc_b200.plan import Plan
    from tests.test_gpu_batch import _config, _instances
    for k, v in VARIANTS[variant].items():
        monkeypatch.setenv(k, v)
    pairs = {jd: _jump_pair(jd) for jd in JUMP_DT}
    inst = []          # (jump_dt, info["step"]): one step before each boundary, and two
    for jd in JUMP_DT:
        s = np.arange(1, last_boundary(jd) + 1)
        st = np.floor(s.astype(np.float32) * np.float32(0.02) / np.float32(jd))
        for b in s[1:][np.diff(st) > 0]:
            inst += [(jd, int(b) - 1), (jd, int(b) - 2)]
    assert len(inst) == 2 * (N_STAGE - 1) * len(JUMP_DT)
    envs = [pairs[jd][0] for jd, _ in inst]
    B = len(envs)
    states, rngs, Y0 = _instances(envs[0], 1, 2)
    states = [states[0].replace(info=dict(states[0].info, step=s, contact_stage=host_stage(envs[i], s - 1) if s else 0))
              for i, (_, s) in enumerate(inst)]
    loop = DeviceLoop(MBDPI(_config("unitree_go2_seq_jump", 8, 4, 2), envs[0], n_instances=B), states,
                      np.repeat(rngs, B, 0), Y0.repeat(B, 1, 1), envs=envs)
    loop.step(1, env_step=1)
    cnt = loop.buf["counters"].cpu().numpy()
    want = np.array([host_stage(envs[i], s) for i, (_, s) in enumerate(inst)])
    bad = [(jd, s + 1, int(c), int(w)) for (jd, s), c, w in zip(inst, cnt[:, 1], want) if c != w]
    assert np.array_equal(cnt[:, 0], [s + 1 for _, s in inst])
    assert not bad, f"(jump_dt, step + 1, device stage, host stage): {bad}"
    # the stage the rollout's reward used at the step after info["step"] = s
    bad = []
    for jd, (env, o) in pairs.items():
        plan = Plan(env, env.plan_desc())
        st0 = o.reset()
        for _, s in [x for x in inst if x[0] == jd]:
            stage0 = host_stage(env, s - 1) if s else 0
            rewss, *_ = plan.rollout(_state(plan, st0.qpos[0], st0.qvel[0], s, stage0), np.zeros((32, 2, o.nu)), want_traj=False)
            got = stage_from_reward(rewss.cpu().numpy())
            if not (got[:, 0] == stage0).all() or not (got[:, 1] == host_stage(env, s)).all():
                bad.append((jd, s + 1, np.unique(got[:, 1]).tolist(), host_stage(env, s)))
    assert not bad, f"(jump_dt, step + 1, rollout stage, host stage): {bad}"
