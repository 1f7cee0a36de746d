"""The built-in rewards of the rollout kernel (csrc/dial_device.cuh: reward_partials, reward_lane0) against
an fp64 restatement evaluated on the kernel's own states, from start states built on the edges of each
reward term; and the seq-jump stage counter of the oracle, the host env and the C port at every stage
boundary.

``fp64_rewards`` recomputes every env step of a kernel rollout from what the kernel itself produced: the
pre-state of step t is the kernel's state after step t - 1 (the start state at t = 0), its ctrl follows
from the action and that state, its kinematics and contacts from ``mo.forward`` on it, and its reward
from the oracle env with the kernel's post-state.  No dynamics lies between the two, so what differs is
the fp32 rounding of one reward evaluation, not the drift of a rollout.  This module runs the device code
through the CPU warp emulator; test_gpu_reward_parity.py holds the CUDA build to the same reference."""
from dataclasses import dataclass, field
from typing import Optional

import numpy as np
import pytest

from baseline_configs import ENV_CFG
from oracle import mjx_oracle as mo
from oracle.envs_oracle import OState, make_env

# Reward tolerance: |kernel - fp64| < REWARD_TOL * (1 + |fp64|) per env step.  The emulator's worst case
# over the cases below is 1.2e-6 (Go2 walk around the command override at step 500); 1e-5 leaves room for
# the GPU's fast-math sin / cos / atan2 and fused multiply-adds.  A rollout through contact dynamics is held
# to 2e-3 (test_gpu_parity.py); one reward on the kernel's own state needs no such slack.
REWARD_TOL = 1e-5
CTRL_TOL = 1e-4          # ctrl of the last step (torques up to 200 N m / joint targets), absolute
BAND = 1e-5              # fp32 band (m) around the seq-jump branches: rows this close to one are dropped
JUMP_DT = (0.1, 0.3, 0.55, 0.6, 0.85, 1.0, 1.1, 1.2, 1.3)
N_STAGE = 12             # DIAL_MAXSTAGE: every boundary a task can have


def f32(a):
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def make_pair(name, **over):
    """(product env, oracle env) of ENV_CFG[name] with the same overrides applied to both.  Allegro runs
    one physics step per env step (dt = timestep = 0.005), so that nothing but the reward lies between
    the kernel's states."""
    import dial_mpc_b200.envs as E
    cfg = dict(ENV_CFG[name])
    if name == "allegro_reorient":
        cfg.update(dt=0.005, timestep=0.005)
    cfg.update(over)
    cfg_t = E.get_config(name)
    env = E.get_environment(name, config=cfg_t(**{k: (np.array(v) if isinstance(v, list) else v) for k, v in cfg.items()}))
    tables = {k: np.asarray(cfg.pop(k), dtype=np.float64) for k in ("contact_targets", "contact_target_radius") if k in cfg}
    o = make_env(name, cfg)
    if tables:          # explicit disc tables (the oracle derives them from the pose sequence otherwise)
        o.contact_targets, o.contact_radius = tables["contact_targets"], tables["contact_target_radius"]
    assert env._n_frames == 1 and o.n_frames == 1
    return env, o


def rpy_quat(r, p, y):
    cr, sr, cp, sp, cy, sy = np.cos(r / 2), np.sin(r / 2), np.cos(p / 2), np.sin(p / 2), np.cos(y / 2), np.sin(y / 2)
    return np.array([cr * cp * cy + sr * sp * sy, sr * cp * cy - cr * sp * sy,
                     cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy])


@dataclass
class Case:
    env: str
    qpos: np.ndarray
    qvel: np.ndarray
    step: int
    stage: int = 0
    H: int = 2
    over: dict = field(default_factory=dict)     # env config overrides (both envs)
    cmd: Optional[tuple] = None                   # (step, vel[3], ang[3]): one-step command override
    extreme: bool = False                         # actions at +-1 (torques at their limits)
    tag: str = ""

    def pair(self):
        env, o = make_pair(self.env, **self.over)
        o.cmd_override = self.cmd
        return env, o

    def desc(self, env):
        d = env.plan_desc()
        if self.cmd is not None:
            d.cmd_step = self.cmd[0]
            d.cmd_vel[:], d.cmd_ang[:] = list(self.cmd[1]), list(self.cmd[2])
        return d

    def actions(self, rng, B, nu):
        if self.extreme:
            return np.sign(rng.uniform(-1, 1, (B, self.H, nu)))
        return f32(np.clip(rng.normal(size=(B, self.H, nu)) * 0.6, -1, 1))


def fp64_rewards(o, q0, v0, step0, stage0, us, q, qd):
    """The fp64 reward [B,H] of every env step of a kernel rollout from (q0, v0) at (step0, stage0) with
    actions us [B,H,nu], whose per-step outputs are q [B,H,nq], qd [B,H,nv]; each step is evaluated on the
    kernel's own pre-state.  Also returns the fp64 ctrl [B,nu] of the last step, the Data of each step's
    pre-state and the stage [B,H] each step used."""
    assert o.n_frames == 1
    B, H, _ = us.shape
    q, qd = np.asarray(q, dtype=np.float64), np.asarray(qd, dtype=np.float64)
    qpre = np.concatenate([np.broadcast_to(f32(q0), (B, 1, q.shape[-1])), q[:, :-1]], 1)
    vpre = np.concatenate([np.broadcast_to(f32(v0), (B, 1, qd.shape[-1])), qd[:, :-1]], 1)
    stage = np.full(B, stage0, dtype=np.int64)
    rew, stages, datas = np.zeros((B, H)), np.zeros((B, H), dtype=np.int64), []
    for t in range(H):
        qp, vp = qpre[:, t], vpre[:, t]
        ctrl = o.act2tau(us[:, t], qp, vp) if o.leg_control == "torque" else o.act2joint(us[:, t])
        d = mo.forward(o.m, qp, vp, ctrl, np.zeros_like(vp))
        s = OState(qp, vp, None, np.full(B, step0 + t, dtype=np.int64), stage)
        stages[:, t] = stage
        rew[:, t], stage = o.reward(s, q[:, t], qd[:, t], d, ctrl)
        datas.append(d)
    return rew, ctrl, datas, stages


def jump_branches(o, datas, stages):
    """The seq-jump branch margins on the kernel's pre-states (fp64): disc [B,H,4,n] = |foot xy - target xy|
    - radius of stage j, contact [B,H,4] = dist - 0.001; and the steps [B,H] none of whose margins lies in
    the fp32 band."""
    tgt = o.contact_targets.transpose(1, 0, 2)[None, :, :, :2]                  # [1,4,n,2]
    r = o.contact_radius.T[None]
    # a disc of infinite radius holds every foot: inf <= inf in fp32 as in fp64, far from any rounding
    with np.errstate(invalid="ignore"):
        disc = np.stack([np.where(np.isposinf(r), -np.inf, np.linalg.norm(d.con_pos[:, :4, None, :2] - tgt, axis=-1) - r)
                         for d in datas], 1)
    cont = np.stack([d.con_dist[:, :4] - 0.001 for d in datas], 1)
    keep = (np.abs(disc) > BAND).all((-1, -2)) & (np.abs(cont) > BAND).all(-1)
    return disc, cont, keep


def jump_coverage(disc, cont, stages, keep):
    """Per-foot counts of each side of each seq-jump branch over the kept steps."""
    inside = disc <= 0                                                          # [B,H,4,n]
    n = disc.shape[-1]
    cur = np.take_along_axis(inside, np.broadcast_to(stages[:, :, None, None], inside.shape[:3] + (1,)), -1)[..., 0]
    other = (inside & (np.arange(n) != stages[:, :, None, None])).any(-1) & ~cur
    none = ~inside.any(-1)
    touch = cont <= 0
    k = keep[:, :, None]
    return {"current disc": int((cur & k).sum()), "other disc": int((other & k).sum()), "no disc": int((none & k).sum()),
            "penalised": int((touch & none & k).sum()), "penalty cleared by a disc": int((touch & ~none & k).sum()),
            "above 0.001": int((~touch & k).sum())}


# ---- start states on the edges of each reward term ---------------------------------------------------
def _base(o, rpy=(0.0, 0.0, 0.0), dz=0.0, vel=None, joints=None):
    q = o.init_q.copy()
    q[2] += dz
    q[3:7] = rpy_quat(*rpy)
    if joints is not None:
        q[7:7 + len(joints)] = joints
    v = np.zeros(o.m.nv)
    if vel is not None:
        v[:len(vel)] = vel
    return f32(q), f32(v)


def go2_walk_cases(rng):
    o = make_env("unitree_go2_walk", ENV_CFG["unitree_go2_walk"])
    W, cases = "unitree_go2_walk", []
    jv = lambda s: np.r_[np.zeros(6), rng.normal(size=12) * s]
    for y in (np.pi - 4e-4, -np.pi + 4e-4):                                   # yaw at the wrap
        q, v = _base(o, (0.0, 0.0, y), vel=jv(0.5))
        cases.append(Case(W, q, v, 30, tag=f"yaw {y:+.4f}"))
        cases.append(Case(W, q, v, 400, over=dict(default_vyaw=0.8), tag=f"yaw {y:+.4f}, target 6.4 rad"))
    for vyaw, step, y in ((1.5, 700, 0.3), (-0.7, 200, -2.0), (1.2, 333, 2.9)):  # yaw targets wrapped several times
        q, v = _base(o, (0.05, -0.04, y), vel=jv(1.0))
        cases.append(Case(W, q, v, step, H=3, over=dict(default_vyaw=vyaw), tag=f"vyaw {vyaw} step {step}"))
    for r, p in ((20, 0), (0, -35), (45, 30), (-60, 10), (25, 55)):            # tilted base
        q, v = _base(o, (np.radians(r), np.radians(p), 0.7), dz=0.05, vel=jv(1.0))
        cases.append(Case(W, q, v, 60, tag=f"tilt {r},{p}"))
    q, v = _base(o, (0.1, -0.1, 0.4), vel=np.r_[0.7, -0.5, 0.3, 1.2, -0.8, 1.5, rng.normal(size=12) * 2])
    cases.append(Case(W, q, v, 75, over=dict(default_vyaw=0.5), tag="body velocities"))
    neg = dict(default_vx=-0.9, default_vy=-0.3, default_vyaw=-0.6)
    q, v = _base(o, (0.0, 0.05, -0.3), vel=np.r_[-0.4, 0.2, 0, 0.3, 0.2, -0.5, np.zeros(12)])
    cases.append(Case(W, q, v, 0, H=3, over=neg, tag="ramp from 0, negative commands"))
    cases.append(Case(W, q, v, 47, H=6, over=neg, tag="ramp end, negative commands"))
    cases.append(Case(W, q, v, 150, over=neg, tag="ramp 3, negative commands"))
    cases.append(Case(W, q, v, 47, H=6, over=dict(default_vy=0.4, default_vyaw=0.9), tag="ramp end"))
    for gait, H in (("stand", 3), ("walk", 50), ("trot", 25), ("canter", 13), ("gallop", 15)):   # a gait period each
        q, v = _base(o, (0.0, 0.0, 0.1), vel=jv(0.5))
        cases.append(Case(W, q, v, 20, H=H, over=dict(gait=gait), tag=f"gait {gait}"))
    q, v = _base(o, (0.02, 0.0, 0.2), vel=jv(0.5))
    cases.append(Case(W, q, v, 498, H=5, cmd=(500, (-1.2, 0.4, 0.0), (0.0, 0.0, 1.1)), tag="cmd_step 500"))
    return cases


def _feet(o, q):
    _, xpos, _, xmat, *_ = mo.kinematics(o.m, q[None])
    dist, pos, _ = mo.collision(o.m, xpos, xmat)
    return pos[0, :4, :2], dist[0, :4]


def go2_jump_cases(rng):
    """Every stage; a foot a few mm inside or outside a target disc of the current stage, of another
    stage or of none; its contact distance just below or above 0.001.  Every other case starts one step
    before a stage boundary, so its second step scores the next stage."""
    o = make_env("unitree_go2_seq_jump", ENV_CFG["unitree_go2_seq_jump"])
    J, cases = "unitree_go2_seq_jump", []
    n = o.contact_targets.shape[0]
    for j in range(n):
        for m, (where, radial, dz) in enumerate((("cur", -1, -1), ("cur", -1, 1), ("cur", 1, -1), ("other", -1, -1),
                                                 ("none", 0, -1), ("none", 0, 1))):
            q, v = _base(o, (0.02, -0.03, 0.08 * (j - 2)), vel=np.r_[rng.normal(size=6) * 0.3, rng.normal(size=12)])
            pos, dist = _feet(o, q)
            i = (j + m) % 4
            if where == "none":
                shift = np.array([0.2 + 0.4 * j, 0.45])
            else:
                k = j if where == "cur" else (j + 1) % n
                u = rng.normal(size=2)
                shift = o.contact_targets[k, i, :2] - pos[i] + (o.contact_radius[k, i] + radial * 3e-3) * u / np.linalg.norm(u)
            q[:2] += shift
            q[2] += 0.001 + dz * 3e-4 - dist[i]
            step = 50 * j + (49 if m % 2 else 20)
            cases.append(Case(J, f32(q), v, step, stage=j, tag=f"stage {j}: {where} disc, {radial * 3} mm, dz {dz:+d}"))
    # a stage whose discs accept any foot position (radius inf, centred at infinity: squared distance inf,
    # inf <= inf), and feet touching: the bonus and the cleared penalty rest on the disc test's equality
    tgt, rad = o.contact_targets.copy(), o.contact_radius.copy()
    tgt[2, :, 0], rad[2] = np.inf, np.inf
    any_pos = dict(contact_targets=tgt.tolist(), contact_target_radius=rad.tolist(),
                   pose_target_sequence=o.pose_seq.tolist(), yaw_target_sequence=o.yaw_seq.tolist())
    for stage in (2, 1):
        q, v = _base(o, (0.0, 0.0, 0.05), vel=np.r_[np.zeros(6), rng.normal(size=12) * 0.3])
        q[2] -= _feet(o, q)[1].max() + 2e-3
        cases.append(Case(J, f32(q), v, 50 * stage + 10, stage=stage, over=any_pos, tag=f"stage {stage}: disc of infinite radius"))
    return cases


def h1_cases(rng):
    cases = []
    o = make_env("unitree_h1_walk", ENV_CFG["unitree_h1_walk"])
    lo, hi = o.physical_joint_range[:, 0], o.physical_joint_range[:, 1]
    for step in (10, 100, 200):                                                 # torques at their limits
        jt = np.where(rng.uniform(size=o.nu) < 0.5, lo, hi) * 0.9 + rng.normal(size=o.nu) * 0.02
        q, v = _base(o, (0.1, -0.08, 0.3), vel=np.r_[rng.normal(size=6) * 0.5, rng.normal(size=o.nu) * 3], joints=jt)
        cases.append(Case("unitree_h1_walk", q, v, step, extreme=True, tag=f"h1 walk torque limits, step {step}"))
    o = make_env("unitree_h1_loco", ENV_CFG["unitree_h1_loco"])
    lo, hi = o.physical_joint_range[:, 0], o.physical_joint_range[:, 1]
    for step, vyaw in ((15, 0.0), (120, 0.4), (400, -0.5)):                    # tilted feet, fast joints, body rates
        jt = lo + rng.uniform(0.1, 0.9, o.nu) * (hi - lo)
        vel = np.r_[rng.normal(size=3) * 0.5, 1.5, -1.2, 0.9, rng.choice([-1, 1], o.nu) * rng.uniform(10, 40, o.nu)]
        q, v = _base(o, (0.2, -0.15, 0.5), vel=vel, joints=jt)
        cases.append(Case("unitree_h1_loco", q, v, step, over=dict(default_vyaw=vyaw),
                          extreme=step == 400, tag=f"h1 loco step {step}"))
    return cases


def allegro_cases(rng):
    cases = []
    _, o = make_pair("allegro_reorient")
    lo, hi = o.physical_joint_range[:, 0], o.physical_joint_range[:, 1]
    for k in range(3):
        q = o.init_q.copy()
        q[0:3] += rng.uniform(-0.015, 0.015, 3)                                 # ball displaced
        q[3:7] = rpy_quat(*rng.uniform(-1, 1, 3))
        q[7:] = np.clip(q[7:] + rng.uniform(-0.3, 0.3, o.nu), lo, hi)           # joints away from their offsets
        v = np.zeros(o.m.nv)
        v[0:6] = np.r_[rng.normal(size=3) * 0.1, rng.normal(size=3) * 5]       # ball spinning
        v[6:] = rng.normal(size=o.nu)
        cases.append(Case("allegro_reorient", f32(q), f32(v), 7 * k, tag=f"allegro {k}"))
    return cases


def all_cases():
    rng = np.random.default_rng(2024)
    return {"unitree_go2_walk": go2_walk_cases(rng), "unitree_go2_seq_jump": go2_jump_cases(rng),
            "unitree_h1": h1_cases(rng), "allegro_reorient": allegro_cases(rng)}


def check_case(case, run, B, rng):
    """Roll `case` on a kernel, `run(env, desc, case, us)` -> (rewss, q, qd, ctrl of row 0's last step), and
    compare with fp64.  Returns (worst relative reward error, kept [B,H] mask, branch data or None)."""
    env, o = case.pair()
    us = case.actions(rng, B, o.nu)
    rew_k, q, qd, ctrl_k = run(env, case.desc(env), case, us)
    rew, ctrl, datas, stages = fp64_rewards(o, case.qpos, case.qvel, case.step, case.stage, us, q, qd)
    keep, branches = np.ones(rew.shape, dtype=bool), None
    if case.env == "unitree_go2_seq_jump":
        disc, cont, keep = jump_branches(o, datas, stages)
        branches = (disc, cont, stages, keep)
    err = (np.abs(rew_k - rew) / (1 + np.abs(rew)))[keep]
    assert err.size == 0 or err.max() < REWARD_TOL, (case.tag, float(err.max()), np.argwhere(keep)[err.argmax()])
    if ctrl_k is not None:
        assert np.abs(ctrl_k - ctrl[0]).max() < CTRL_TOL, (case.tag, np.abs(ctrl_k - ctrl[0]).max())
    return (float(err.max()) if err.size else 0.0), keep, branches


def check_jump_coverage(results):
    """Few steps dropped for lying in the fp32 band, and every side of every branch still tested."""
    kept = np.concatenate([k.ravel() for _, k, _ in results])
    assert (~kept).sum() <= 0.05 * kept.size, f"{(~kept).sum()} of {kept.size} steps dropped"
    cov = {}
    for _, _, (disc, cont, stages, keep) in results:
        for k, v in jump_coverage(disc, cont, stages, keep).items():
            cov[k] = cov.get(k, 0) + v
    assert all(v > 0 for v in cov.values()), cov
    used = np.unique(np.concatenate([s[k] for _, k, (_, _, s, _) in results]))
    assert set(used) == set(range(5)), used
    return cov


# ---- CPU half: the device code through the warp emulator ---------------------------------------------
def _emul_run(env, desc, case, us):
    from tests.emul import emul
    out = emul.rollout(env, desc, case.qpos, case.qvel, np.zeros(len(case.qvel)), step0=case.step, stage0=case.stage, us=us)
    return out["rewss"], out["q"], out["qd"], out["ctrl_out"]


@pytest.mark.parametrize("group", ["unitree_go2_walk", "unitree_go2_seq_jump", "unitree_h1", "allegro_reorient"])
def test_emulated_rewards_match_fp64_at_term_edges(group):
    rng = np.random.default_rng(5)
    cases = all_cases()[group]
    results = [check_case(c, _emul_run, 3 if c.H <= 6 else 1, rng) for c in cases]
    if group == "unitree_go2_seq_jump":
        check_jump_coverage(results)


def test_edge_states_are_on_the_edges():
    """The start states really sit where their tags say: yaw within 1e-3 of +-pi, tilts of 20-60 degrees,
    yaw targets wrapped more than once, and each seq-jump foot margin of a few mm / 0.3 mm."""
    from oracle.envs_oracle import quat_to_euler
    cases = all_cases()
    walk = cases["unitree_go2_walk"]
    yaws = np.array([quat_to_euler(c.qpos[3:7])[2] for c in walk if c.tag.startswith("yaw")])
    assert len(yaws) == 4 and (np.pi - np.abs(yaws)).max() < 1e-3
    ups = [c.qpos[3:7] for c in walk if c.tag.startswith("tilt")]
    tilt = np.degrees([np.arccos(1 - 2 * (q[1] ** 2 + q[2] ** 2)) for q in ups])
    assert tilt.min() > 19 and tilt.max() > 59
    ramp_up = ENV_CFG["unitree_go2_walk"]["ramp_up_time"]
    wraps = [abs(min(v * c.step * 0.02 / ramp_up, v) * 0.02 * c.step) for c in walk if c.tag.startswith("vyaw")
             for v in (c.over["default_vyaw"],)]
    assert len(wraps) == 3 and min(wraps) > 2 * np.pi
    o = make_env("unitree_go2_seq_jump", ENV_CFG["unitree_go2_seq_jump"])
    for c in cases["unitree_go2_seq_jump"]:
        if "infinite" in c.tag:
            continue
        pos, dist = _feet(o, c.qpos)
        assert np.abs(dist - 0.001).min() < 3.5e-4, c.tag
        if "none" not in c.tag:
            d = np.abs(np.linalg.norm(pos[:, None] - o.contact_targets.transpose(1, 0, 2)[:, :, :2], axis=-1) - 0.1)
            assert d.min() < 3.5e-3, c.tag


# ---- the seq-jump stage: oracle, host env and C port -------------------------------------------------
def _jump_pair(jump_dt):
    """Twelve stages 100 m apart: the stage a reward used is read off its r_pos."""
    pose = [[100.0 * j, 0.0, 0.27] for j in range(N_STAGE)]
    return make_pair("unitree_go2_seq_jump", jump_dt=jump_dt, pose_target_sequence=pose, yaw_target_sequence=[0.0] * N_STAGE)


def last_boundary(jump_dt, dt=0.02):
    """The first step + 1 that reaches the last stage under the fp32 formula."""
    s = np.arange(1, 100000)
    return int(s[np.floor(s.astype(np.float32) * np.float32(dt) / np.float32(jump_dt)) >= N_STAGE - 1][0])


def host_stage(env, step):
    """The stage the host env gives the state after the env step whose info["step"] is `step`."""
    return env._next_info({"step": int(step)})["contact_stage"]


def stage_from_reward(rew):
    """Stage of a seq-jump reward with the 100 m stage table of _jump_pair (r_pos dominates every other term)."""
    return np.rint(np.sqrt(np.maximum(10.0 - np.asarray(rew, dtype=np.float64), 0.0)) / 100.0).astype(np.int64)


@pytest.fixture(scope="module")
def built_port():
    from oracle import build_oracle
    build_oracle.build()
    return True


@pytest.mark.parametrize("jump_dt", JUMP_DT)
def test_stage_oracle_host_and_c_port_agree(built_port, jump_dt):
    from oracle.c_port import CPort
    env, o = _jump_pair(jump_dt)
    last = last_boundary(jump_dt)
    steps = np.arange(last)                         # env steps from info["step"] = 0 .. last - 1
    host = np.array([host_stage(env, s) for s in steps])
    assert (np.diff(host) >= 0).all() and host[-1] == N_STAGE - 1 and host[-2] == N_STAGE - 2
    assert np.array_equal(o.next_stage(steps), host)
    # the C port from reset: its reward at step t scores the stage its step t - 1 produced
    s0 = o.reset()
    rew, *_ = CPort(o, real="double").rollout(s0, np.zeros((1, last + 1, o.nu)))
    assert np.array_equal(stage_from_reward(rew[0, 1:]), host)
    assert stage_from_reward(rew[0, :1])[0] == 0
