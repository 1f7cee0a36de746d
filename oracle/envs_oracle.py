"""ORACLE (test infrastructure, not product code) — fp64 restatement of the
reference environments' ``step`` (PD torque -> physics -> reward) for the
BASELINE configs.  PARITY UNPINNED (see mjx_oracle.py header).

Follows, line by line:
* BaseEnv.act2joint / act2tau        dial_mpc/envs/base_env.py:37-66
* UnitreeGo2Env.reset / step         dial_mpc/envs/unitree_go2_env.py:101-261
* UnitreeGo2SeqJumpEnv.reset / step  dial_mpc/envs/unitree_go2_env.py:363-521,
  generate_jumping_sequence          dial_mpc/envs/unitree_go2_env.py:559-592
* UnitreeH1WalkEnv.reset / step      dial_mpc/envs/unitree_h1_env.py:156-321
* get_foot_step, global_to_body_velocity   dial_mpc/utils/function_utils.py:7-43
* brax.math rotate / inv_rotate / quat_to_euler / euler_to_quat (third party,
  restated; SURVEY.md Appendix E)
Only non-zero-weight reward terms are evaluated (zero-weight terms multiply
finite values by 0.0 in the reference).
"""

from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Dict, Optional

import numpy as np

from . import mjx_oracle as mo

_MODELS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "dial_mpc_b200", "models")


# ---- brax.math restatements (batched over leading axes) ------------------------
def rotate(v, q):
    return mo.qrot(q, v)


def inv_rotate(v, q):
    return mo.qrot(mo.qconj(q), v)


def quat_to_euler(q):
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    ez = np.arctan2(-2 * x * y + 2 * w * z, x * x + w * w - z * z - y * y)
    ey = np.arcsin(np.clip(2 * x * z + 2 * w * y, -1.0, 1.0))
    ex = np.arctan2(-2 * y * z + 2 * w * x, z * z - y * y - x * x + w * w)
    return np.stack([ex, ey, ez], -1)


def euler_to_quat_deg(v):
    c1, c2, c3 = np.cos(v * np.pi / 360)
    s1, s2, s3 = np.sin(v * np.pi / 360)
    return np.array([c1 * c2 * c3 - s1 * s2 * s3, s1 * c2 * c3 + c1 * s2 * s3,
                     c1 * s2 * c3 - s1 * c2 * s3, c1 * c2 * s3 + s1 * s2 * c3])


def get_foot_step(duty_ratio, cadence, amplitude, phases, time):
    """function_utils.py:18-43.  ``time`` [B] -> heights [B, nfeet]."""
    t = time[..., None] * 2 * np.pi * cadence + np.pi
    footphase = 2 * np.pi * np.asarray(phases)
    angle = np.mod(t + np.pi - footphase, 2 * np.pi) - np.pi
    if duty_ratio < 1:
        angle = angle * 0.5 / (1 - duty_ratio)
    clipped = np.clip(angle, -np.pi / 2, np.pi / 2)
    value = np.cos(clipped) if duty_ratio < 1 else np.zeros_like(clipped)
    final = np.where(np.abs(value) >= 1e-6, np.abs(value), 0.0)
    return amplitude * final


@dataclass
class OState:
    """Minimal planner-visible state (batched): Brax pipeline_state + env info."""
    qpos: np.ndarray
    qvel: np.ndarray
    qacc_warmstart: np.ndarray
    step: np.ndarray           # int [B]
    stage: np.ndarray          # int [B] (seq-jump contact_stage)

    def tile(self, B):
        return OState(*(np.repeat(a[:1], B, axis=0) for a in
                        (self.qpos, self.qvel, self.qacc_warmstart, self.step, self.stage)))


class OracleEnv:
    """Common part: BaseEnv (base_env.py:13-66)."""

    model_file = ""
    init_key = "home"

    def __init__(self, dt=0.02, timestep=0.02, kp=30.0, kd=0.0, action_scale=1.0,
                 leg_control="torque", model_path=None):
        self.m = mo.OModel(model_path or os.path.join(_MODELS, self.model_file), timestep=timestep)
        self.dt, self.timestep = dt, timestep
        self.n_frames = int(dt / timestep)
        self.kp, self.kd = np.asarray(kp, dtype=np.float64), np.asarray(kd, dtype=np.float64)
        self.action_scale = action_scale
        self.leg_control = leg_control
        self.nu = self.m.nu
        self.physical_joint_range = self.m.jnt_range[1:].copy()
        self.joint_range = self.physical_joint_range.copy()
        tr = self.m.actuator_ctrlrange.copy()
        tr[self.m.actuator_ctrllimited == 0] = [-np.inf, np.inf]   # brax.io.mjcf loader behaviour
        self.joint_torque_range = tr
        self.init_q = np.array(self.m.keyframes[self.init_key]["qpos"], dtype=np.float64)

    def reset(self) -> OState:
        nv = self.m.nv
        z = np.zeros((1, nv))
        # pipeline_init runs mjx.forward: qacc_warmstart = solver result at the initial state
        d = mo.forward(self.m, self.init_q[None], z, np.zeros((1, self.nu)), z)
        return OState(d.qpos, z.copy(), d.qacc.copy(), np.zeros(1, dtype=np.int64),
                      np.zeros(1, dtype=np.int64))

    def act2joint(self, act):
        an = (act * self.action_scale + 1.0) / 2.0
        jt = self.joint_range[:, 0] + an * (self.joint_range[:, 1] - self.joint_range[:, 0])
        return np.clip(jt, self.physical_joint_range[:, 0], self.physical_joint_range[:, 1])

    def act2tau(self, act, qpos, qvel):
        jt = self.act2joint(act)
        q = qpos[:, 7:7 + self.nu]
        qd = qvel[:, 6:6 + self.nu]
        tau = self.kp * (jt - q) - self.kd * qd
        return np.clip(tau, self.joint_torque_range[:, 0], self.joint_torque_range[:, 1])

    def _physics(self, s: OState, action):
        if self.leg_control == "torque":
            ctrl = self.act2tau(action, s.qpos, s.qvel)
        else:
            ctrl = self.act2joint(action)
        qpos, qvel, warm = s.qpos, s.qvel, s.qacc_warmstart
        for _ in range(self.n_frames):
            qpos, qvel, warm, d = mo.step(self.m, qpos, qvel, ctrl, warm)
        return qpos, qvel, warm, d, ctrl

    def reward(self, s, qpos, qvel, d, ctrl):  # pragma: no cover - abstract
        raise NotImplementedError

    def step(self, s: OState, action):
        """One env step for a batch.  Returns (new_state, reward[B], aux dict)."""
        qpos, qvel, warm, d, ctrl = self._physics(s, action)
        rew, stage = self.reward(s, qpos, qvel, d, ctrl)
        ns = OState(qpos, qvel, warm, s.step + 1, stage)
        aux = dict(q=qpos, qd=qvel, xpos=d.xpos[:, 1:], ctrl=ctrl, data=d, prev=s)
        return ns, rew, aux

    # -- randomize_tasks: the one-step command of unitree_go2_env.py:141-155 --------------------
    cmd_override = None      # (step, vel[3], ang[3]) or None

    def commands(self, step):
        """(vel_cmd, ang_cmd) [B,3] used by the env step whose info["step"] is `step`."""
        B = len(step)
        vel, ang = np.tile(self.vel_cmd, (B, 1)), np.tile(self.ang_cmd, (B, 1))
        if self.cmd_override is not None:
            hit = (np.asarray(step) == self.cmd_override[0])[:, None]
            vel = np.where(hit, np.asarray(self.cmd_override[1], dtype=np.float64), vel)
            ang = np.where(hit, np.asarray(self.cmd_override[2], dtype=np.float64), ang)
        return vel, ang

    # -- observation / done of env.step (not on the sampling path) ----------------------------
    done_height = 0.18

    def info_targets(self, step):
        """state.info["vel_tar"/"ang_vel_tar"] as the state ENTERING step number `step` carries
        them: zero after reset, else ramped from the previous (pre-increment) step
        (unitree_go2_env.py:108-110,156-163)."""
        step = np.asarray(step, dtype=np.float64)
        ramp = np.maximum(step - 1.0, 0.0)[:, None] * self.dt / self.ramp_up_time
        live = (step >= 1)[:, None]
        vel_cmd, ang_cmd = self.commands(step - 1)
        return (np.where(live, np.minimum(vel_cmd * ramp, vel_cmd), 0.0),
                np.where(live, np.minimum(ang_cmd * ramp, ang_cmd), 0.0))

    def _vb_ab(self, d):
        v = mo.brax_views(self.m, d)
        rot_b = v["x_rot"][:, self.torso]
        return (inv_rotate(v["xd_vel"][:, self.torso], rot_b),
                inv_rotate(v["xd_ang"][:, self.torso] * np.pi / 180.0, rot_b), v)

    def observe(self, s: OState, qpos, qvel, d, ctrl, last_ctrl=None):
        """_get_obs(pipeline_state, state.info) of the walk envs (unitree_go2_env.py:263-286,
        unitree_h1_env.py:323-346, :850-873) for the step s -> (qpos, qvel, d)."""
        vel_tar, ang_tar = self.info_targets(s.step)
        vb, ab, _ = self._vb_ab(d)
        return np.concatenate([vel_tar, ang_tar, ctrl, qpos, vb, ab, qvel[:, 6:]], -1)

    def done(self, s: OState, qpos, qvel, d):
        """unitree_go2_env.py:241-248 / unitree_h1_env.py:300-308."""
        v = mo.brax_views(self.m, d)
        up = np.array([0.0, 0.0, 1.0])
        ja = qpos[:, 7:7 + len(self.joint_range)]
        dn = rotate(up, v["x_rot"][:, self.torso])[:, 2] < 0
        dn |= np.any(ja < self.joint_range[:, 0], -1) | np.any(ja > self.joint_range[:, 1], -1)
        dn |= v["x_pos"][:, self.torso, 2] < self.done_height
        return dn.astype(np.float64)

    def rollout(self, s0: OState, us):
        """rollout_us (dial_core.py:36-42) vmapped: us [B,H,nu] ->
        rewss [B,H], q [B,H,nq], qd [B,H,nv], xpos [B,H,nbody-1,3]."""
        B, H, _ = us.shape
        s = s0.tile(B)
        rews, qs, qds, xs = [], [], [], []
        for t in range(H):
            s, r, aux = self.step(s, us[:, t])
            rews.append(r)
            qs.append(aux["q"])
            qds.append(aux["qd"])
            xs.append(aux["xpos"])
        return (np.stack(rews, 1), np.stack(qs, 1), np.stack(qds, 1), np.stack(xs, 1))


class Go2WalkOracle(OracleEnv):
    model_file = "unitree_go2_mjx_scene_force.json"
    GAIT_PHASE = {"stand": [0, 0, 0, 0], "walk": [0.0, 0.5, 0.75, 0.25], "trot": [0.0, 0.5, 0.5, 0.0],
                  "canter": [0.0, 0.33, 0.33, 0.66], "gallop": [0.0, 0.05, 0.4, 0.35]}
    GAIT_PARAMS = {"stand": (1.0, 1.0, 0.0), "walk": (0.75, 1.0, 0.08), "trot": (0.45, 2, 0.08),
                   "canter": (0.4, 4, 0.06), "gallop": (0.3, 3.5, 0.10)}

    def __init__(self, default_vx=1.0, default_vy=0.0, default_vyaw=0.0, ramp_up_time=2.0,
                 gait="trot", **kw):
        kw.setdefault("kp", 30.0)
        kw.setdefault("kd", 0.0)
        super().__init__(**kw)
        self.vel_cmd = np.array([default_vx, default_vy, 0.0])
        self.ang_cmd = np.array([0.0, 0.0, default_vyaw])
        self.ramp_up_time = ramp_up_time
        self.gait = gait
        self.torso = self.m.names["body"].index("base") - 1
        self.feet_site = [self.m.names["site"].index(n) for n in ("FL_foot", "FR_foot", "RL_foot", "RR_foot")]
        self.joint_range = np.array([[-0.5, 0.5], [0.4, 1.4], [-2.3, -0.85]] * 2
                                    + [[-0.5, 0.5], [0.4, 1.4], [-2.3, -1.3]] * 2)
        self.pos_tar = np.array([0.282, 0.0, 0.3])

    def reward(self, s, qpos, qvel, d, ctrl):
        v = mo.brax_views(self.m, d)
        stepf = s.step.astype(np.float64)
        ramp = stepf[:, None] * self.dt / self.ramp_up_time
        vel_cmd, ang_cmd = self.commands(s.step)
        vel_tar = np.minimum(vel_cmd * ramp, vel_cmd)
        ang_tar = np.minimum(ang_cmd * ramp, ang_cmd)
        z_feet = d.site_xpos[:, self.feet_site, 2]
        duty, cad, amp = self.GAIT_PARAMS[self.gait]
        z_tar = get_foot_step(duty, cad, amp, self.GAIT_PHASE[self.gait], stepf * self.dt)
        r_gaits = -np.sum(((z_tar - z_feet) / 0.05) ** 2, -1)
        up = np.array([0.0, 0.0, 1.0])
        r_upright = -np.sum((rotate(up, v["x_rot"][:, 0]) - up) ** 2, -1)
        rot_b = v["x_rot"][:, self.torso]
        yaw_tar = 0.0 + ang_tar[:, 2] * self.dt * stepf
        dyaw = quat_to_euler(rot_b)[:, 2] - yaw_tar
        r_yaw = -np.arctan2(np.sin(dyaw), np.cos(dyaw)) ** 2
        vb = inv_rotate(v["xd_vel"][:, self.torso], rot_b)
        ab = inv_rotate(v["xd_ang"][:, self.torso] * np.pi / 180.0, rot_b)
        r_vel = -np.sum((vb[:, :2] - vel_tar[:, :2]) ** 2, -1)
        r_angvel = -(ab[:, 2] - ang_tar[:, 2]) ** 2
        r_height = -(v["x_pos"][:, self.torso, 2] - self.pos_tar[2]) ** 2
        rew = 0.1 * r_gaits + 0.5 * r_upright + 0.3 * r_yaw + r_vel + r_angvel + r_height
        return rew, s.stage


class Go2SeqJumpOracle(Go2WalkOracle):
    def __init__(self, jump_dt=1.0, pose_target_sequence=None, yaw_target_sequence=None, **kw):
        super().__init__(**kw)
        self.jump_dt = jump_dt
        pose = np.asarray(pose_target_sequence, dtype=np.float64)
        yaw = np.asarray(yaw_target_sequence, dtype=np.float64)
        n = pose.shape[0]
        offsets = np.array([[0.2, -0.135, 0.0], [0.2, 0.135, 0.0], [-0.2, -0.135, 0.0], [-0.2, 0.135, 0.0]])
        targets = []
        for i in range(n):
            R = mo.qmat(euler_to_quat_deg(np.array([0.0, 0.0, yaw[i] * 180 / np.pi])))
            targets.append(pose[i][None] + offsets @ R.T)
        self.contact_targets = np.array(targets)            # [n,4,3]
        self.contact_radius = np.full((n, 4), 0.1)
        self.pose_seq, self.yaw_seq = pose, yaw
        self.joint_range = np.array([[-0.5, 0.5], [0.4, 2.0], [-2.3, -1.3]] * 2
                                    + [[-0.5, 0.5], [0.4, 1.4], [-2.3, -1.3]] * 2)

    done_height = 0.1

    def observe(self, s, qpos, qvel, d, ctrl, last_ctrl=None):
        """unitree_go2_env.py:523-557 (vel_tar / ang_vel_tar stay zero in this env)."""
        vb, ab, v = self._vb_ab(d)
        B = qpos.shape[0]
        rpy = quat_to_euler(qpos[:, 3:7])
        dpos = v["x_pos"][:, self.torso] - self.pose_seq[s.stage]
        dyaw = rpy[:, 2] - self.yaw_seq[s.stage]
        dyaw = np.arctan2(np.sin(dyaw), np.cos(dyaw))[:, None]
        last = np.zeros((B, self.nu)) if last_ctrl is None else np.broadcast_to(last_ctrl, (B, self.nu))
        return np.concatenate([np.zeros((B, 6)), last, dpos, rpy[:, :2], dyaw, qpos[:, 7:], vb, ab, qvel[:, 6:]], -1)

    def reward(self, s, qpos, qvel, d, ctrl):
        v = mo.brax_views(self.m, d)
        stage = s.stage
        pos = v["x_pos"][:, self.torso]
        r_pos = -np.sum((pos - self.pose_seq[stage]) ** 2, -1)
        up = np.array([0.0, 0.0, 1.0])
        r_upright = -np.sum((rotate(up, v["x_rot"][:, 0]) - up) ** 2, -1)
        yaw = quat_to_euler(v["x_rot"][:, self.torso])[:, 2]
        r_yaw = -(yaw - self.yaw_seq[stage]) ** 2
        r_contact = np.zeros(qpos.shape[0])
        penalty = d.con_dist[:, :4] <= 0.001
        n = self.contact_targets.shape[0]
        for i in range(4):
            for j in range(n):
                cond = (np.sum((d.con_pos[:, i, :2] - self.contact_targets[j, i, :2]) ** 2, -1)
                        <= self.contact_radius[j, i] ** 2)
                val = (j == stage) * np.clip(d.con_dist[:, i] * -1.0 + 1.0, 0.0, 1.0)
                r_contact += np.where(cond, val, 0.0)
                penalty[:, i] &= ~cond
        pen = penalty.sum(-1)
        rew = r_pos + r_upright + 0.3 * r_yaw + 0.1 * r_contact - 0.1 * pen + 10.0
        return rew, self.next_stage(s.step)

    def next_stage(self, step):
        """Stage after the env step whose info["step"] is `step`: the reference computes the quotient in
        JAX fp32 (unitree_go2_env.py:508-515), and an fp64 one floors differently at boundaries such as
        step + 1 = 15 for jump_dt = 0.3 (fp32 0.99999994 -> stage 0)."""
        f = np.float32
        q = (np.asarray(step) + 1).astype(f) * f(self.dt) / f(self.jump_dt)
        return np.minimum(np.floor(q), self.contact_targets.shape[0] - 1).astype(np.int64)


class H1WalkOracle(OracleEnv):
    model_file = "unitree_h1_mjx_scene_h1_walk.json"
    GAIT_PHASE = {"stand": [0, 0], "slow_walk": [0.0, 0.5], "walk": [0.0, 0.5], "jog": [0.0, 0.5]}
    GAIT_PARAMS = {"stand": (1.0, 1.0, 0.0), "slow_walk": (0.6, 0.8, 0.15), "walk": (0.5, 1.0, 0.15),
                   "jog": (0.3, 2, 0.2)}
    KP = [200.0, 200.0, 200.0, 200.0, 60.0] * 2 + [200.0] + [60.0] * 8
    KD = [5.0, 5.0, 5.0, 5.0, 1.5] * 2 + [5.0] + [1.5] * 8

    def __init__(self, default_vx=1.0, default_vy=0.0, default_vyaw=0.0, ramp_up_time=2.0,
                 gait="jog", **kw):
        kw.setdefault("kp", self.KP)
        kw.setdefault("kd", self.KD)
        super().__init__(**kw)
        self.vel_cmd = np.array([default_vx, default_vy, 0.0])
        self.ang_cmd = np.array([0.0, 0.0, default_vyaw])
        self.ramp_up_time = ramp_up_time
        self.gait = gait
        self.torso = self.m.names["body"].index("torso_link") - 1
        self.joint_range = np.array(
            [[-0.3, 0.3], [-0.3, 0.3], [-1.0, 1.0], [0.0, 1.74], [-0.6, 0.4]] * 2 + [[-0.5, 0.5]]
            + [[-0.78, 0.78], [-0.3, 0.3], [-0.3, 0.3], [-0.3, 0.3]] * 2)
        self.pos_tar = np.array([0.0, 0.0, 1.3])

    def reward(self, s, qpos, qvel, d, ctrl):
        v = mo.brax_views(self.m, d)
        stepf = s.step.astype(np.float64)
        ramp = stepf[:, None] * self.dt / self.ramp_up_time
        vel_cmd, ang_cmd = self.commands(s.step)
        vel_tar = np.minimum(vel_cmd * ramp, vel_cmd)
        ang_tar = np.minimum(ang_cmd * ramp, ang_cmd)
        duty, cad, amp = self.GAIT_PARAMS[self.gait]
        z_tar = get_foot_step(duty, cad, amp, self.GAIT_PHASE[self.gait], stepf * self.dt)
        z_feet = np.stack([d.con_dist[:, 0:2].min(-1), d.con_dist[:, 2:4].min(-1)], -1)
        r_gaits = -np.sum((z_tar - z_feet) ** 2, -1)
        up = np.array([0.0, 0.0, 1.0])
        r_upright = -np.sum((rotate(up, v["x_rot"][:, 0]) - up) ** 2, -1)
        rot_b = v["x_rot"][:, self.torso]
        yaw_tar = 0.0 + ang_tar[:, 2] * self.dt * stepf
        dyaw = quat_to_euler(rot_b)[:, 2] - yaw_tar
        r_yaw = -np.arctan2(np.sin(dyaw), np.cos(dyaw)) ** 2
        vb = inv_rotate(v["xd_vel"][:, self.torso], rot_b)
        ab = inv_rotate(v["xd_ang"][:, self.torso] * np.pi / 180.0, rot_b)
        r_vel = -np.sum((vb[:, :2] - vel_tar[:, :2]) ** 2, -1)
        r_angvel = -(ab[:, 2] - ang_tar[:, 2]) ** 2
        r_height = -(v["x_pos"][:, self.torso, 2] - self.pos_tar[2]) ** 2
        r_energy = -np.sum((ctrl / self.joint_torque_range[:, 1]) ** 2, -1)
        rew = (5.0 * r_gaits + 0.5 * r_upright + 0.1 * r_yaw + r_vel + r_angvel
               + 0.5 * r_height + 0.01 * r_energy)
        return rew, s.stage


class H1LocoOracle(H1WalkOracle):
    """UnitreeH1LocoEnv.step (dial_mpc/envs/unitree_h1_env.py:686-830): 11 actuated joints (arms
    welded), two capsules per foot (8 contacts), iterations = ls_iterations = 1."""
    model_file = "unitree_h1_mjx_scene_h1_loco.json"
    GAIT_PARAMS = {"stand": (1.0, 1.0, 0.0), "slow_walk": (0.6, 0.8, 0.15), "walk": (0.5, 1.5, 0.10),
                   "jog": (0.3, 2.0, 0.2)}
    KP = [200.0, 200.0, 200.0, 200.0, 60.0] * 2 + [200.0]
    KD = [5.0, 5.0, 5.0, 5.0, 1.5] * 2 + [5.0]

    def __init__(self, **kw):
        kw.setdefault("kp", self.KP)
        kw.setdefault("kd", self.KD)
        super().__init__(**kw)
        self.joint_range = np.array([[-0.2, 0.2], [-0.2, 0.2], [-0.6, 0.6], [0.0, 1.5], [-0.6, 0.4]] * 2 + [[-0.5, 0.5]])
        self.feet_site = [self.m.names["site"].index(n) for n in ("left_foot", "right_foot")]

    def reward(self, s, qpos, qvel, d, ctrl):
        v = mo.brax_views(self.m, d)
        stepf = s.step.astype(np.float64)
        ramp = stepf[:, None] * self.dt / self.ramp_up_time
        vel_cmd, ang_cmd = self.commands(s.step)
        vel_tar = np.minimum(vel_cmd * ramp, vel_cmd)
        ang_tar = np.minimum(ang_cmd * ramp, ang_cmd)
        duty, cad, amp = self.GAIT_PARAMS[self.gait]
        z_tar = get_foot_step(duty, cad, amp, self.GAIT_PHASE[self.gait], stepf * self.dt)
        z_feet = np.stack([d.con_dist[:, 0:4].min(-1), d.con_dist[:, 4:8].min(-1)], -1)
        r_gaits = -np.sum((z_tar - z_feet) ** 2, -1)
        up = np.array([0.0, 0.0, 1.0])
        r_upright = -np.sum((rotate(up, v["x_rot"][:, 0]) - up) ** 2, -1)
        rot_b = v["x_rot"][:, self.torso]
        yaw_tar = 0.0 + ang_tar[:, 2] * self.dt * stepf
        dyaw = quat_to_euler(rot_b)[:, 2] - yaw_tar
        r_yaw = -np.arctan2(np.sin(dyaw), np.cos(dyaw)) ** 2
        vb = inv_rotate(v["xd_vel"][:, self.torso], rot_b)
        ab = inv_rotate(v["xd_ang"][:, self.torso] * np.pi / 180.0, rot_b)
        r_vel = -np.sum((vb[:, :2] - vel_tar[:, :2]) ** 2, -1)
        r_angvel = -np.sum((ab - ang_tar) ** 2, -1)
        r_height = -(v["x_pos"][:, self.torso, 2] - self.pos_tar[2]) ** 2
        r_level = 0.0
        for sid in self.feet_site:
            zc = d.xmat[:, self.m.site_bodyid[sid], :, 2]        # site frame = body frame (no site quat)
            r_level = r_level - np.sum((zc - up) ** 2, -1)
        nj = len(self.joint_range)
        r_energy = -np.sum((ctrl / self.joint_torque_range[:, 1] * qvel[:, 6:6 + nj] / 160.0) ** 2, -1)
        rew = (10.0 * r_gaits + 0.5 * r_upright + 0.5 * r_yaw + r_vel + r_angvel + 0.5 * r_height
               + 0.02 * r_level + 0.01 * r_energy)
        return rew, s.stage


class AllegroReorientOracle(OracleEnv):
    """AllegroReorientEnv (dial_mpc/envs/manipulation.py:23-115): position targets, 4 substeps."""
    model_file = "wonik_allegro_scene_left.json"
    init_key = "in_hand_reorient"

    def __init__(self, **kw):
        kw.setdefault("kp", 1.0)
        kw.setdefault("kd", 0.1)
        kw.setdefault("dt", 0.02)
        kw.setdefault("timestep", 0.005)
        kw.setdefault("leg_control", "position")
        super().__init__(**kw)
        self.obj = self.m.names["body"].index("object") - 1
        self.ang_vel_tar = np.array([0.0, 0.0, 0.5])
        self.pos_tar = np.array([0.0, 0.0, 0.13])

    def act2joint(self, act):  # manipulation.py:102-115 (adds init_q, clips to the physical range)
        an = (act * self.action_scale + 1.0) / 2.0
        jt = self.joint_range[:, 0] + self.init_q[7:] + an * (self.joint_range[:, 1] - self.joint_range[:, 0])
        return np.clip(jt, self.physical_joint_range[:, 0], self.physical_joint_range[:, 1])

    def reward(self, s, qpos, qvel, d, ctrl):
        v = mo.brax_views(self.m, d)
        w = v["xd_ang"][:, self.obj] * np.pi / 180.0
        r_ang = -np.sum((w - self.ang_vel_tar) ** 2, -1)
        r_pos = -np.sum((v["x_pos"][:, self.obj] - self.pos_tar) ** 2, -1)
        r_joint = -np.sum((qpos[:, 7:] - self.init_q[7:]) ** 2, -1)
        return r_ang + 5.0 * r_pos + 0.1 * r_joint, s.stage


class CustomRewardOracle(OracleEnv):
    """Checker for user-written envs (the reference's README.md:223-312 recipe): the physics of
    ``step`` is the common ``OracleEnv`` path, the reward a Python callable
    ``reward_fn(ctx) -> [B]`` over the batched fp64 counterparts of ``dial_reward_ctx``
    (include/dial_custom_reward.h): step, dt, qpos, qvel, ctrl, xpos, xquat, xmat, xd_vel,
    xd_ang (indexed by MuJoCo body id), contact_dist, contact_pos, site_xpos, user."""

    def __init__(self, model_path, reward_fn, user=(), joint_range=None, init_q=None, **kw):
        super().__init__(model_path=model_path, **kw)
        self.reward_fn = reward_fn
        self.user = np.asarray(user, dtype=np.float64)
        if joint_range is not None:
            self.joint_range = np.asarray(joint_range, dtype=np.float64)
        if init_q is not None:
            self.init_q = np.asarray(init_q, dtype=np.float64)

    def reward(self, s, qpos, qvel, d, ctrl):
        v = mo.brax_views(self.m, d)
        B = qpos.shape[0]
        pad = lambda a: np.concatenate([np.zeros((B, 1) + a.shape[2:]), a], 1)  # body 0 = world
        ctx = dict(step=s.step, dt=self.dt, qpos=qpos, qvel=qvel, ctrl=ctrl, xpos=d.xpos, xquat=d.xquat,
                   xmat=d.xmat, xd_vel=pad(v["xd_vel"]), xd_ang=pad(v["xd_ang"]),
                   contact_dist=d.con_dist, contact_pos=d.con_pos, site_xpos=d.site_xpos,
                   user=self.user)
        return np.asarray(self.reward_fn(ctx), dtype=np.float64), s.stage


def make_env(env_name: str, cfg: Optional[Dict] = None) -> OracleEnv:
    cfg = dict(cfg or {})
    cls = {"unitree_go2_walk": Go2WalkOracle, "unitree_go2_seq_jump": Go2SeqJumpOracle,
           "unitree_h1_walk": H1WalkOracle, "allegro_reorient": AllegroReorientOracle, "unitree_h1_loco": H1LocoOracle}[env_name]
    return cls(**cfg)
