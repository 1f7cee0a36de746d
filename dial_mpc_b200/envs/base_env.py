"""Environment base class for the CUDA sampling core.

Mirrors the surface of the reference ``BaseEnv`` (dial_mpc/envs/base_env.py:13-66), which
is a Brax ``PipelineEnv``: ``sys``, ``dt``, ``action_size``, ``physical_joint_range``,
``joint_range``, ``joint_torque_range``, ``act2joint``, ``act2tau``, ``reset``, ``step``.
The physics + reward of ``step`` run in the fused CUDA rollout kernel (csrc/) through the
C ABI (include/dial_b200.h); there is no CPU fallback.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Any, Dict

import numpy as np

from dial_mpc_b200 import _capi
from dial_mpc_b200.config.base_env_config import BaseEnvConfig
from dial_mpc_b200.modelc import CompiledModel


class System:
    """What the reference reads from ``brax.base.System`` (``self.sys``)."""

    def __init__(self, model: CompiledModel):
        self.model = model
        self.nq, self.nv, self.nu, self.nbody = model.nq, model.nv, model.nu, model.nbody
        self.jnt_range = model.jnt_range.copy()
        ctrl = model.actuator_ctrlrange.copy()
        # brax.io.mjcf.load replaces the range of un-limited actuators by +-inf
        ctrl[model.actuator_ctrllimited == 0] = [-np.inf, np.inf]
        self.actuator_ctrlrange = ctrl

    @property
    def timestep(self) -> float:
        return self.model.timestep

    def tree_replace(self, params: Dict[str, Any]) -> "System":
        """``sys.tree_replace`` of the float model fields (``CompiledModel.replace``): ``opt.timestep``,
        ``opt.gravity``, ``body_mass``, ``pair_friction``, ... as full arrays or ``{name: value}``
        mappings.  Derived constants are left as they are, as in MJX; ``sys.model.set_const()``
        recomputes them.  Structural fields raise ``KeyError``."""
        return System(self.model.replace(params))

    def keyframe(self, name: str) -> np.ndarray:
        return self.model.keyframe_qpos(name)

    def body_id(self, name: str) -> int:
        return self.model.body_id(name)

    def site_id(self, name: str) -> int:
        return self.model.site_id(name)


@dataclass
class PipelineState:
    """The slice of the Brax/MJX pipeline state the planner carries between calls
    (device tensors, fp32)."""
    qpos: Any
    qvel: Any
    qacc_warmstart: Any
    ctrl: Any = None
    kin: Any = None     # [13] torso x.pos, x.rot, body-frame xd.vel, xd.ang*pi/180 after env.step (for _get_obs)

    @property
    def q(self):
        return self.qpos

    @property
    def qd(self):
        return self.qvel


@dataclass
class State:
    pipeline_state: PipelineState
    obs: Any
    reward: Any
    done: Any
    metrics: Dict[str, Any] = field(default_factory=dict)
    info: Dict[str, Any] = field(default_factory=dict)

    def replace(self, **kw) -> "State":
        d = dict(pipeline_state=self.pipeline_state, obs=self.obs, reward=self.reward, done=self.done,
                 metrics=self.metrics, info=self.info)
        d.update(kw)
        return State(**d)


class BaseEnv:
    env_id: int = -1
    supports_randomize_tasks = False     # walk envs: one-step random command every 500 steps
    COMMAND_PERIOD = 500                 # unitree_go2_env.py:152

    def __init__(self, config: BaseEnvConfig):
        assert math.isclose(config.dt % config.timestep, 0.0, abs_tol=1e-9) or \
            math.isclose(config.dt % config.timestep, config.timestep, abs_tol=1e-9), \
            "timestep must be divisible by dt"
        if config.randomize_tasks and not self.supports_randomize_tasks:
            raise NotImplementedError(f"randomize_tasks=True is not supported by {type(self).__name__}")
        self._config = config
        self._n_frames = int(round(config.dt / config.timestep))
        self.sys = self.make_system(config)
        # joint limit definitions (base_env.py:22-25)
        self.physical_joint_range = self.sys.jnt_range[1:]
        self.joint_range = self.physical_joint_range
        self.joint_torque_range = self.sys.actuator_ctrlrange
        self._nv = self.sys.nv
        self._nq = self.sys.nq
        self._plan = None  # lazily created 1-sample plan for reset()/step()

    # -- Brax PipelineEnv surface ---------------------------------------------------------
    @property
    def sys(self) -> System:
        return self._sys

    @sys.setter
    def sys(self, value: System) -> None:
        """Assigning a new system (e.g. ``env.sys = env.sys.tree_replace({...})``) drops the cached plan:
        the next ``reset`` / ``step`` runs the new model."""
        self._sys = value
        self._plan = None

    @property
    def dt(self) -> float:
        return self._config.timestep * self._n_frames

    @property
    def action_size(self) -> int:
        return self.sys.nu

    def make_system(self, config: BaseEnvConfig) -> System:
        raise NotImplementedError

    def act2joint(self, act):
        """[-1,1] action -> joint target (base_env.py:37-50); numpy, host side."""
        act = np.asarray(act, dtype=np.float64)
        an = (act * self._config.action_scale + 1.0) / 2.0
        jt = self.joint_range[:, 0] + an * (self.joint_range[:, 1] - self.joint_range[:, 0])
        return np.clip(jt, self.physical_joint_range[:, 0], self.physical_joint_range[:, 1])

    def act2tau(self, act, pipeline_state):
        """PD torque for an action (base_env.py:52-66); numpy, host side."""
        jt = self.act2joint(act)
        q = _to_numpy(pipeline_state.qpos)[7:][: len(jt)]
        qd = _to_numpy(pipeline_state.qvel)[6:][: len(jt)]
        tau = self._kp() * (jt - q) - self._kd() * qd
        return np.clip(tau, self.joint_torque_range[:, 0], self.joint_torque_range[:, 1])

    def _kp(self):
        return np.broadcast_to(np.asarray(self._config.kp, dtype=np.float64), (self.sys.nu,))

    def _kd(self):
        return np.broadcast_to(np.asarray(self._config.kd, dtype=np.float64), (self.sys.nu,))

    # -- C descriptor -----------------------------------------------------------------------
    def _fill_reward_desc(self, d: "_capi.dial_plan_desc") -> None:
        raise NotImplementedError

    def plan_desc(self, Nsample=1, Hsample=1, Hnode=2, temp_sample=1.0, M_n2u=None,
                  Ntotal=None, shard_offset=0, n_inst=1, n_ens=0) -> "_capi.dial_plan_desc":
        """``n_inst``: independent planner instances sharing this descriptor (batched control-step
        graph, ``DeviceLoop`` on an ``MBDPI(..., n_instances=n_inst)``).  ``n_ens``: planning models per
        instance (``MBDPI(..., n_ensemble=n_ens)``; 0: the instance's own model)."""
        d = _capi.dial_plan_desc()
        d.env_id = self.env_id
        d.Nsample, d.Ntotal, d.shard_offset = int(Nsample), int(Ntotal or Nsample), int(shard_offset)
        d.Hsample, d.Hnode = int(Hsample), int(Hnode)
        if Hsample + 1 > _capi.DEFINES["DIAL_MAXH"] or Hnode + 1 > _capi.DEFINES["DIAL_MAXNODE"]:
            raise ValueError("Hsample/Hnode exceed DIAL_MAXH/DIAL_MAXNODE")
        d.n_frames = self._n_frames
        if self._config.leg_control not in ("torque", "position"):
            raise ValueError("Invalid leg control type.")
        d.leg_control_torque = int(self._config.leg_control == "torque")
        d.temp_sample = float(temp_sample)
        d.dt = float(self.dt)
        d.action_scale = float(self._config.action_scale)
        _capi._set(d.kp, self._kp())
        _capi._set(d.kd, self._kd())
        _capi._set(d.joint_range, self.joint_range)
        _capi._set(d.physical_joint_range, self.physical_joint_range)
        big = 3.0e38
        _capi._set(d.joint_torque_range, np.clip(self.joint_torque_range, -big, big))
        if M_n2u is not None:
            _capi._set(d.M_n2u, M_n2u)
        d.cmd_step = -1
        d.n_inst = int(n_inst)
        d.n_ens = int(n_ens)
        d.n_stage = 1         # one (unused) stage unless the env has a jump sequence
        self._fill_reward_desc(d)
        return d

    def task(self) -> "_capi.dial_task":
        """The reward inputs of this env's configuration that may differ between the instances of one
        plan (commands, gait, jump sequence, custom-reward user constants): the task fields of
        ``plan_desc()``, for ``DeviceLoop(..., envs=...)`` / ``DeviceLoop.set_task``."""
        return _capi.task_from_desc(self.plan_desc())

    # -- reset / step through the CUDA core ---------------------------------------------------
    def _get_plan(self):
        if self._plan is None:
            from dial_mpc_b200.plan import Plan
            self._plan = Plan(self, self.plan_desc())
        return self._plan

    def _init_info(self, rng) -> Dict[str, Any]:
        return {"rng": rng, "step": 0}

    def reset(self, rng) -> State:
        """``pipeline_init(init_q, 0)`` (mjx.forward) + fresh info (unitree_go2_env.py:101-124)."""
        from dial_mpc_b200 import random as drandom
        rng, _ = drandom.split(rng)
        ps = self._get_plan().pipeline_init(self._init_q)
        info = self._init_info(rng)
        return State(ps, self._get_obs(ps, info), 0.0, 0.0, {}, info)

    # -- randomize_tasks (unitree_go2_env.py:141-155,298-315; unitree_h1_env.py:198-212,358-375) --
    def sample_command(self, rng):
        """``sample_command(rng)`` of the walk envs: uniform vx in [-1.5, 1.5], vy in [-0.5, 0.5],
        yaw rate in [-1.5, 1.5] from keys 1..3 of ``jax.random.split(rng, 4)``."""
        from dial_mpc_b200 import random as drandom
        keys = drandom.split_n(rng, 4)
        vx = drandom.uniform1(keys[1], -1.5, 1.5)
        vy = drandom.uniform1(keys[2], -0.5, 0.5)
        wz = drandom.uniform1(keys[3], -1.5, 1.5)
        return np.array([vx, vy, 0.0], dtype=np.float32), np.array([0.0, 0.0, wz], dtype=np.float32)

    def command_override(self, info: Dict[str, Any], horizon: int):
        """(step, vel, ang) of the random command an env step within ``horizon`` steps of
        ``info["step"]`` uses, or None.  The reference draws it inside ``step`` from
        ``split(info["rng"])[1]`` whenever ``step % 500 == 0``; ``info["rng"]`` advances by one split
        per env step, so the key for a future step follows from the current one."""
        if not info.get("randomize_target", False):
            return None
        from dial_mpc_b200 import random as drandom
        s0 = int(info["step"])
        hit = -(-s0 // self.COMMAND_PERIOD) * self.COMMAND_PERIOD       # next multiple of the period >= s0
        if hit >= s0 + max(int(horizon), 1):
            return None
        cache = getattr(self, "_cmd_cache", None)
        tag = (hit, tuple(int(v) for v in np.asarray(info["rng"]).ravel()), s0)
        if cache is not None and cache[0] == tag:
            return cache[1]
        rng = np.asarray(info["rng"], dtype=np.uint32)
        for _ in range(hit - s0):
            rng, _unused = drandom.split(rng)
        vel, ang = self.sample_command(drandom.split(rng)[1])
        out = (hit, vel, ang)
        self._cmd_cache = (tag, out)
        return out

    def _next_info(self, info: Dict[str, Any]) -> Dict[str, Any]:
        new = dict(info)
        new["step"] = info["step"] + 1
        c = self._config
        if "vel_tar" in info and hasattr(c, "default_vx"):
            # commanded velocities ramped from the PRE-increment step, fp32 like the reference
            # (unitree_go2_env.py:151-163, unitree_h1_env.py:208-219)
            f = np.float32
            ramp = f(info["step"]) * f(self.dt) / f(c.ramp_up_time)
            vel = np.array([c.default_vx, c.default_vy, 0.0], dtype=f)
            ang = np.array([0.0, 0.0, c.default_vyaw], dtype=f)
            ov = self.command_override(info, 1)
            if ov is not None:
                vel, ang = ov[1], ov[2]
            new["vel_tar"] = np.minimum(vel * ramp, vel)
            new["ang_vel_tar"] = np.minimum(ang * ramp, ang)
        return new

    def step(self, state: State, action) -> State:
        from dial_mpc_b200 import random as drandom
        ps, reward = self._get_plan().env_step(state, action)
        info = self._next_info(state.info)
        info["rng"], _ = drandom.split(state.info["rng"])
        # the observation is taken before the info update (unitree_go2_env.py:139)
        return State(ps, self._get_obs(ps, state.info), reward, self._get_done(ps, state.info), state.metrics, info)

    # -- observation / termination flag (device tensors; not on the sampling path) ---------------
    _done_height = 0.18      # torso height below which the locomotion envs flag `done`

    @staticmethod
    def _dev(ps, a):
        import torch
        return torch.as_tensor(np.asarray(a, dtype=np.float32), device=ps.qpos.device)

    def _vb_ab(self, ps):
        """global_to_body_velocity of the torso's xd.vel and xd.ang*pi/180: written by the kernel
        from the kinematics of the step's forward pass (Brax x / xd are one integration behind
        qpos); zero at reset (qvel = 0)."""
        import torch
        return ps.kin[7:13] if ps.kin is not None else torch.zeros(6, device=ps.qpos.device)

    def _ctrl(self, ps):
        import torch
        return ps.ctrl if ps.ctrl is not None else torch.zeros(self.sys.nu, device=ps.qpos.device)

    def _get_obs(self, pipeline_state: PipelineState, info: Dict[str, Any]):
        """``_get_obs`` of the walk envs (unitree_go2_env.py:263-286, unitree_h1_env.py:323-346):
        [vel_tar, ang_vel_tar, ctrl, qpos, vb, ab, qvel[6:]]."""
        import torch
        ps = pipeline_state
        return torch.cat([self._dev(ps, info.get("vel_tar", np.zeros(3))), self._dev(ps, info.get("ang_vel_tar", np.zeros(3))),
                          self._ctrl(ps), ps.qpos, self._vb_ab(ps), ps.qvel[6:]])

    def _get_done(self, pipeline_state: PipelineState, info: Dict[str, Any]):
        """Termination flag of the locomotion envs (unitree_go2_env.py:241-248, :498-505,
        unitree_h1_env.py:300-308): torso upside down, a joint outside ``joint_range``, or the torso
        below ``_done_height``.  The planner never reads it (``reward_alive`` has weight 0)."""
        import torch
        ps = pipeline_state
        if ps.kin is None:
            return torch.zeros((), device=ps.qpos.device)
        jr = self._dev(ps, self.joint_range)
        ja = ps.qpos[7:7 + jr.shape[0]]
        up_z = 1.0 - 2.0 * (ps.kin[4] ** 2 + ps.kin[5] ** 2)      # dot(rotate(up, rot), up)
        done = (up_z < 0) | (ja < jr[:, 0]).any() | (ja > jr[:, 1]).any() | (ps.kin[2] < self._done_height)
        return done.to(torch.float32)


def _to_numpy(x):
    if hasattr(x, "detach"):
        return x.detach().cpu().numpy().astype(np.float64)
    return np.asarray(x, dtype=np.float64)
