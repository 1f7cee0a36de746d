"""Thin Python wrapper over the C-ABI plan handle (include/dial_b200.h).

PyTorch is used only for device memory and streams; every compute call goes to the
hand-written kernels in ``csrc/libdial_b200.so``."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np
import torch

from dial_mpc_b200 import _capi


def _ptr(t: Optional[torch.Tensor]):
    if t is None:
        return None
    assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous(), "need contiguous fp32 CUDA tensor"
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _key(key):
    if key is None:
        return None
    k = np.ascontiguousarray(key, dtype=np.uint32)
    return (C.c_uint32 * 2)(int(k[0]), int(k[1]))


class Plan:
    def __init__(self, env, desc: "_capi.dial_plan_desc", device: Optional[torch.device] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("dial_mpc_b200 needs a CUDA device (H100); there is no CPU fallback")
        # custom-reward envs carry their own build of the library (dial_mpc_b200.custom)
        self.lib = _capi.lib(getattr(env, "library_path", None))
        self.env = env
        self.desc = desc
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.mdesc = _capi.fill_model_desc(env.sys.model)
        with torch.cuda.device(self.device):
            self.handle = self.lib.dial_plan_create(C.byref(self.mdesc), C.byref(desc))
        if not self.handle:
            raise RuntimeError(f"dial_plan_create failed: {self.lib.dial_last_error().decode()}")
        m = self.mdesc
        self.nq, self.nv, self.nu, self.nbody = m.nq, m.nv, m.nu, m.nbody
        self.N, self.Ntotal = desc.Nsample, desc.Ntotal
        self.Hs, self.Hn = desc.Hsample, desc.Hnode
        self.exchange_on = False
        self._cmd = None          # last command override uploaded (randomize_tasks)
        self._stages = None       # identity of the last stage tables uploaded (seq-jump randomize_tasks)

    def set_command(self, override) -> None:
        """``override`` = (step, vel[3], ang[3]) or None: the one-step random command of
        ``randomize_tasks`` (envs' ``command_override``); uploaded only when it changes."""
        key = None if override is None else (int(override[0]), tuple(np.float32(override[1]).tolist()),
                                             tuple(np.float32(override[2]).tolist()))
        if key == self._cmd:
            return
        if key is None:
            self._check(self.lib.dial_plan_set_command(self.handle, -1, None, None, _stream()))
        else:
            v, a = (C.c_float * 3)(*key[1]), (C.c_float * 3)(*key[2])
            self._check(self.lib.dial_plan_set_command(self.handle, key[0], v, a, _stream()))
        self._cmd = key

    def set_stages(self, tables) -> None:
        """``tables`` = (pose [n,3], yaw [n], contact_targets [n,4,3], contact_radius [n,4]): the jump
        sequence of the state a launch starts from (seq-jump ``randomize_tasks``: drawn at reset);
        uploaded only when it differs from what the plan holds."""
        pose, yaw, tgt, rad = (np.ascontiguousarray(t, dtype=np.float32) for t in tables)
        key = (pose.tobytes(), yaw.tobytes(), tgt.tobytes(), rad.tobytes())
        if key == self._stages:
            return
        n = int(pose.shape[0])
        assert yaw.shape == (n,) and tgt.shape == (n, 4, 3) and rad.shape == (n, 4)
        F = C.POINTER(C.c_float)
        self._check(self.lib.dial_plan_set_stages(self.handle, n, pose.ctypes.data_as(F), yaw.ctypes.data_as(F),
                                                  tgt.ctypes.data_as(F), rad.ctypes.data_as(F), _stream()))
        self._stages = key

    def set_instance_model(self, b: int, model) -> None:
        """Instance b's own physical model (a ``CompiledModel`` or ``System`` with the plan model's
        structure, timestep, joint ranges and control ranges) for every later ``mpc_step``; a
        stream-ordered copy on the current stream (``dial_plan_set_instance_model``)."""
        model = getattr(model, "model", model)
        md = _capi.fill_model_desc(model)
        self._check(self.lib.dial_plan_set_instance_model(self.handle, int(b), C.byref(md), _stream()))

    def set_ensemble_model(self, b: int, k: int, model) -> None:
        """Member k of instance b's planning ensemble (a plan with ``n_ens`` >= 1): the model its rollout
        rows run in every later ``mpc_step``; the same checks and stream-ordered copy as
        ``set_instance_model`` (``dial_plan_set_ensemble_model``)."""
        model = getattr(model, "model", model)
        md = _capi.fill_model_desc(model)
        self._check(self.lib.dial_plan_set_ensemble_model(self.handle, int(b), int(k), C.byref(md), _stream()))

    def set_ensemble_risk(self, b: int, mode: int, alpha: float = 1.0) -> None:
        """Instance b's risk measure over its members' rewards (``_capi.DEFINES["DIAL_ENS_MEAN"]`` or
        ``["DIAL_ENS_CVAR"]`` with ``alpha`` in (0, 1]) from the next ``mpc_step`` on; a stream-ordered copy
        on the current stream that keeps the captured graphs (``dial_plan_set_ensemble_risk``)."""
        self._check(self.lib.dial_plan_set_ensemble_risk(self.handle, int(b), int(mode), float(alpha), _stream()))

    def member_rewards(self, out: torch.Tensor) -> torch.Tensor:
        """Copy the member rewards of the last reverse_once of ``mpc_step`` into ``out``
        [n_inst * n_ens * (Nsample+1)] elements, instance-, then member-major (``dial_plan_member_rewards``)."""
        n = max(self.desc.n_inst, 1) * self.desc.n_ens * (self.N + 1)
        assert self.desc.n_ens < 1 or out.numel() == n, f"need {n} elements, got {tuple(out.shape)}"
        self._check(self.lib.dial_plan_member_rewards(self.handle, _ptr(out), _stream()))
        return out

    def set_ensemble_adapt(self, b: int, on: bool, forget: float = 1.0, prune: float = 0.0, sigma=None) -> None:
        """Instance b adapts its belief over its members to the plant at every env step (``on``), with
        ``forget`` in (0, 1], ``prune`` in [0, 1/K) and ``sigma`` [nv] > 0; or stops (the belief is kept).
        A stream-ordered copy on the current stream; the first call that turns adaptation on in a plan
        changes the launch sequence, so the next steps capture their graphs again; later calls keep them
        (``dial_plan_set_ensemble_adapt``)."""
        s = None
        if sigma is not None:
            a = np.ascontiguousarray(sigma, dtype=np.float32).ravel()
            assert a.size == self.nv, f"sigma needs {self.nv} values, got {a.size}"
            s = (C.c_float * len(a))(*a.tolist())
        self._check(self.lib.dial_plan_set_ensemble_adapt(self.handle, int(b), int(bool(on)), float(forget),
                                                          float(prune), s, _stream()))

    def set_ensemble_belief(self, b: int, w) -> None:
        """Instance b's belief from K weights >= 0 with a positive sum, normalised in fp64 on the host
        (``dial_plan_set_ensemble_belief``)."""
        a = np.ascontiguousarray(w, dtype=np.float32).ravel()
        assert self.desc.n_ens < 2 or a.size == self.desc.n_ens, f"need {self.desc.n_ens} weights, got {a.size}"
        self._check(self.lib.dial_plan_set_ensemble_belief(self.handle, int(b), (C.c_float * a.size)(*a.tolist()),
                                                           _stream()))

    def ensemble_belief(self, w: Optional[torch.Tensor], loglik: Optional[torch.Tensor] = None) -> None:
        """Copy the belief [n_inst * n_ens] and the last update's log-likelihoods into ``w`` / ``loglik``
        (either may be None; ``dial_plan_ensemble_belief``)."""
        n = max(self.desc.n_inst, 1) * self.desc.n_ens
        for t in (w, loglik):
            assert t is None or t.numel() == n, f"need {n} elements, got {tuple(t.shape)}"
        self._check(self.lib.dial_plan_ensemble_belief(self.handle, _ptr(w), _ptr(loglik), _stream()))

    def set_instance_schedule(self, b: int, temp: float = 1.0, noise=None) -> None:
        """Instance b's sampling schedule from the next ``mpc_step`` on: softmax temperature ``temp`` and
        noise rows ``noise`` [n_rows, Hnode+1] (fp32, n_rows in 1..64); ``noise=None`` returns it to the
        plan's temp_sample and the bound noise.  A stream-ordered copy on the current stream; the first
        call on a plan changes the launch sequence, so the next steps capture their graphs again; later calls
        keep them (``dial_plan_set_instance_schedule``)."""
        if noise is None:
            self._check(self.lib.dial_plan_set_instance_schedule(self.handle, int(b), float(temp), 0, None, _stream()))
            return
        a = np.ascontiguousarray(noise.cpu().numpy() if isinstance(noise, torch.Tensor) else noise, dtype=np.float32)
        assert a.ndim == 2 and a.shape[1] == self.Hn + 1, f"noise must be [n_rows, {self.Hn + 1}], got {a.shape}"
        self._check(self.lib.dial_plan_set_instance_schedule(self.handle, int(b), float(temp), int(a.shape[0]),
                                                             a.ctypes.data_as(C.POINTER(C.c_float)), _stream()))

    def set_instance_iterations(self, n_iter) -> None:
        """Each instance's iteration limit (one int in 0..64 per instance) from the next ``mpc_step`` on: instance
        b runs min(n_diffuse, n_iter[b]) diffusion iterations (``dial_plan_set_instance_iterations``)."""
        a = np.ascontiguousarray(n_iter, dtype=np.int32).ravel()
        assert a.size == max(self.desc.n_inst, 1), f"need {max(self.desc.n_inst, 1)} limits, got {a.size}"
        self._check(self.lib.dial_plan_set_instance_iterations(self.handle, a.ctypes.data_as(C.POINTER(C.c_int32)),
                                                               _stream()))

    def set_instance_delay(self, b: int, steps: int, predict: bool = False) -> None:
        """Instance b's control latency from the next ``mpc_step`` on: the action planned at step t reaches the
        plant at step t + ``steps`` (0..16), and with ``predict`` the instance plans from the state predicted
        through its queued actions.  Refills b's queue with ``steps`` copies of its current Y[0]; a stream-ordered
        copy on the current stream (``dial_plan_set_instance_delay``)."""
        self._check(self.lib.dial_plan_set_instance_delay(self.handle, int(b), int(steps), int(bool(predict)), _stream()))

    def pending_actions(self, out: torch.Tensor) -> torch.Tensor:
        """Copy each instance's queued actions in application order into ``out`` [n_inst * 16 * nu] elements,
        rows past the instance's delay zero (``dial_plan_pending_actions``)."""
        n = max(self.desc.n_inst, 1) * _capi.DEFINES["DIAL_MAXDELAY"] * self.nu
        assert out.numel() == n, f"need {n} elements, got {tuple(out.shape)}"
        self._check(self.lib.dial_plan_pending_actions(self.handle, _ptr(out), _stream()))
        return out

    def planning_state(self, qpos: Optional[torch.Tensor], qvel: Optional[torch.Tensor] = None,
                       warm: Optional[torch.Tensor] = None, counters: Optional[torch.Tensor] = None) -> None:
        """Copy the state the last planning rollouts started from (each output may be None; ``counters`` int32
        [n_inst * 2]) (``dial_plan_planning_state``)."""
        B = max(self.desc.n_inst, 1)
        for t, n in ((qpos, B * self.nq), (qvel, B * self.nv), (warm, B * self.nv)):
            assert t is None or t.numel() == n, f"need {n} elements, got {tuple(t.shape)}"
        cnt = None
        if counters is not None:
            assert counters.is_cuda and counters.dtype == torch.int32 and counters.is_contiguous() and counters.numel() == 2 * B
            cnt = C.c_void_p(counters.data_ptr())
        self._check(self.lib.dial_plan_planning_state(self.handle, _ptr(qpos), _ptr(qvel), _ptr(warm), cnt, _stream()))

    def set_instance_observation(self, b: int, delay: int, qpos_std=None, qvel_std=None, key=None) -> None:
        """Instance b plans from an observation of its plant from the next ``mpc_step`` on: the record ``delay``
        (0..16) env steps old, with Gaussian noise of standard deviations ``qpos_std`` [nv] (tangent space) and
        ``qvel_std`` [nv] (None: zero) drawn from ``key`` (uint32 [2], None: {0, 0}).  Resets b's history; a
        stream-ordered copy on the current stream (``dial_plan_set_instance_observation``)."""
        arrs = []
        for a in (qpos_std, qvel_std):
            if a is None:
                arrs.append(None)
                continue
            a = np.ascontiguousarray(a, dtype=np.float32)
            assert a.shape == (self.nv,), f"need {self.nv} standard deviations, got shape {a.shape}"
            arrs.append(a)
        ptr = [None if a is None else a.ctypes.data_as(C.c_void_p) for a in arrs]
        self._check(self.lib.dial_plan_set_instance_observation(self.handle, int(b), int(delay), ptr[0], ptr[1],
                                                                _key(key), _stream()))

    def observed_state(self, qpos: Optional[torch.Tensor], qvel: Optional[torch.Tensor] = None,
                       warm: Optional[torch.Tensor] = None, counters: Optional[torch.Tensor] = None,
                       age: Optional[torch.Tensor] = None) -> None:
        """Copy the observation of the last ``mpc_step``, before the prediction (each output may be None;
        ``counters`` int32 [n_inst * 2], ``age`` int32 [n_inst]) (``dial_plan_observed_state``)."""
        B = max(self.desc.n_inst, 1)
        for t, n in ((qpos, B * self.nq), (qvel, B * self.nv), (warm, B * self.nv)):
            assert t is None or t.numel() == n, f"need {n} elements, got {tuple(t.shape)}"
        ints = []
        for t, n in ((counters, 2 * B), (age, B)):
            if t is not None:
                assert t.is_cuda and t.dtype == torch.int32 and t.is_contiguous() and t.numel() == n
            ints.append(None if t is None else C.c_void_p(t.data_ptr()))
        self._check(self.lib.dial_plan_observed_state(self.handle, _ptr(qpos), _ptr(qvel), _ptr(warm), ints[0], ints[1],
                                                      _stream()))

    def set_instance_pushes(self, b: int, pushes) -> None:
        """Instance b's push table from the next ``mpc_step`` on: a sequence of at most 16 ``_capi.dial_push``
        (empty: no pushes).  A stream-ordered copy on the current stream (``dial_plan_set_instance_pushes``)."""
        pushes = list(pushes)
        arr = (_capi.dial_push * max(len(pushes), 1))(*pushes)
        self._check(self.lib.dial_plan_set_instance_pushes(self.handle, int(b), len(pushes), arr, _stream()))

    def set_instance_plant(self, b: int, plant) -> None:
        """Instance b's plant fidelity from the next ``mpc_step`` on: a ``_capi.dial_plant`` (None: the plan's own).
        Stream-ordered on the current stream (``dial_plan_set_instance_plant``)."""
        self._check(self.lib.dial_plan_set_instance_plant(self.handle, int(b), None if plant is None else C.byref(plant),
                                                          _stream()))

    def set_instance_terrain(self, b: int, side: int, terrain) -> None:
        """Instance b's terrain on ``side`` (``terrain.PLANT`` or ``terrain.PLANNER``) from the next ``mpc_step`` on:
        a ``terrain.Terrain`` (None: the flat floor).  The heights are copied into plan-owned device memory,
        stream-ordered on the current stream (``dial_plan_set_instance_terrain``)."""
        t = None if terrain is None else terrain.c_struct()
        self._check(self.lib.dial_plan_set_instance_terrain(self.handle, int(b), int(side),
                                                            None if t is None else C.byref(t), _stream()))

    def _check(self, rc: int) -> None:
        if rc != 0:
            raise RuntimeError(f"dial_b200: {self.lib.dial_last_error().decode()} (rc={rc})")

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                self.lib.dial_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    # -- helpers ------------------------------------------------------------------------------
    def f32(self, x, shape=None) -> torch.Tensor:
        if isinstance(x, torch.Tensor):
            t = x.to(device=self.device, dtype=torch.float32).contiguous()
        else:
            t = torch.as_tensor(np.asarray(x, dtype=np.float32), device=self.device).contiguous()
        if shape is not None:
            assert tuple(t.shape) == tuple(shape), f"expected shape {shape}, got {tuple(t.shape)}"
        return t

    def empty(self, *shape) -> torch.Tensor:
        return torch.empty(shape, dtype=torch.float32, device=self.device)

    def _state(self, state, horizon: int = 1) -> Tuple["_capi.dial_state", tuple]:
        ps = state.pipeline_state
        qpos, qvel, warm = self.f32(ps.qpos, (self.nq,)), self.f32(ps.qvel, (self.nv,)), self.f32(ps.qacc_warmstart, (self.nv,))
        s = _capi.dial_state()
        s.qpos, s.qvel, s.qacc_warmstart = qpos.data_ptr(), qvel.data_ptr(), warm.data_ptr()
        s.step = int(state.info.get("step", 0))
        s.stage = int(state.info.get("contact_stage", 0))
        if state.info.get("randomize_target", False):
            # every launch that starts from `state` sees the random command its horizon may reach
            self.set_command(self.env.command_override(state.info, horizon))
            if hasattr(self.env, "stage_tables"):
                self.set_stages(self.env.stage_tables(state.info))
        return s, (qpos, qvel, warm)

    @property
    def launches(self) -> int:
        return int(self.lib.dial_launch_count(self.handle))

    # -- API ------------------------------------------------------------------------------------
    def pipeline_init(self, qpos):
        from dial_mpc_b200.envs.base_env import PipelineState
        q = self.f32(qpos, (self.nq,))
        qv = torch.zeros(self.nv, dtype=torch.float32, device=self.device)
        qo, wo = self.empty(self.nq), self.empty(self.nv)
        self._check(self.lib.dial_pipeline_init(self.handle, _ptr(q), _ptr(qv), _ptr(qo), _ptr(wo), _stream()))
        return PipelineState(qo, qv, wo, torch.zeros(self.nu, dtype=torch.float32, device=self.device))

    def env_step(self, state, action):
        from dial_mpc_b200.envs.base_env import PipelineState
        s, keep = self._state(state, 1)
        a = self.f32(action, (self.nu,))
        qo, vo, wo, r, c = self.empty(self.nq), self.empty(self.nv), self.empty(self.nv), self.empty(1), self.empty(self.nu)
        kin = self.empty(13)
        self._check(self.lib.dial_env_step_kin(self.handle, C.byref(s), _ptr(a), _ptr(qo), _ptr(vo), _ptr(wo), _ptr(r),
                                               _ptr(c), _ptr(kin), _stream()))
        ps = PipelineState(qo, vo, wo, c)
        ps.kin = kin      # torso x.pos, x.rot, body-frame velocities (what _get_obs reads of x / xd)
        return ps, r[0]

    def rollout(self, state, us, want_traj=True):
        s, keep = self._state(state, int(np.shape(us)[1]))
        us = self.f32(us)
        B, H, nu = us.shape
        assert nu == self.nu
        rewss = self.empty(B, H)
        q = self.empty(B, H, self.nq) if want_traj else None
        qd = self.empty(B, H, self.nv) if want_traj else None
        x = self.empty(B, H, self.nbody - 1, 3) if want_traj else None
        self._check(self.lib.dial_rollout(self.handle, C.byref(s), _ptr(us), B, H, _ptr(rewss), _ptr(q), _ptr(qd),
                                          _ptr(x), _stream()))
        return rewss, q, qd, x

    def reverse_rollout(self, state, eps, key, Ybar, noise_scale, rews_local):
        s, keep = self._state(state, self.Hs + 1)
        self._check(self.lib.dial_reverse_rollout(self.handle, C.byref(s), _ptr(eps), _key(key), _ptr(Ybar),
                                                  _ptr(noise_scale), _ptr(rews_local), _stream()))

    def reverse_update(self, eps, key, Ybar, noise_scale, rews_all, Ybar_out, weights=None, rews_gathered=None):
        """``rews_all=None``: the rewards come from this rank's exchange mailbox (sharded plans with a
        connected exchange); ``rews_gathered`` then receives a compact copy of all Ntotal+1 rewards."""
        self._check(self.lib.dial_reverse_update_x(self.handle, _ptr(eps), _key(key), _ptr(Ybar), _ptr(noise_scale),
                                                   _ptr(rews_all), _ptr(Ybar_out), _ptr(weights), _ptr(rews_gathered),
                                                   _stream()))

    def reverse_update_fused(self, rews, rng, Ybar, noise_scale, Ybar_out, weights):
        """The control-step graph's update (one fused kernel launch for every instance of the plan) on
        caller buffers: rews [B,Ntotal+1], rng [B,2] int32 (the uint32 key bits; advanced in place to
        ``split(rng)[0]``), Ybar / Ybar_out [B,Hn+1,nu], noise_scale [Hn+1], weights [B,Ntotal+1] out.
        A single-instance plan takes the same tensors without the leading B."""
        assert rng.is_cuda and rng.dtype == torch.int32 and rng.is_contiguous(), "rng: contiguous int32 CUDA tensor"
        self._check(self.lib.dial_reverse_update_fused(self.handle, _ptr(rews), C.c_void_p(rng.data_ptr()), _ptr(Ybar),
                                                       _ptr(noise_scale), _ptr(Ybar_out), _ptr(weights), _stream()))

    # -- multi-GPU exchange over NVLink peer memory (include/dial_b200.h: dial_exchange_*) -------------
    def exchange_setup(self, rank: int, world: int, group=None) -> None:
        """Create this rank's mailbox, all-gather the CUDA IPC handles over ``torch.distributed`` and
        map the peers' mailboxes.  Raises if peer memory cannot be mapped (the caller then keeps NCCL)."""
        import torch.distributed as dist
        nb = _capi.DEFINES["DIAL_IPC_HANDLE_BYTES"]
        h = (C.c_ubyte * nb)()
        with torch.cuda.device(self.device):
            self._check(self.lib.dial_exchange_create(self.handle, int(rank), int(world), h))
            mine = torch.tensor(list(bytes(h)), dtype=torch.uint8, device=self.device)
            allh = torch.empty(world * nb, dtype=torch.uint8, device=self.device)
            dist.all_gather_into_tensor(allh, mine, group=group)
            buf = (C.c_ubyte * (world * nb)).from_buffer_copy(bytes(allh.cpu().numpy().tobytes()))
            self._check(self.lib.dial_exchange_connect(self.handle, buf))
            torch.cuda.synchronize()
            dist.barrier(group=group)      # every rank has mapped every mailbox before anyone writes
        self.exchange_on = True

    def exchange_status(self) -> dict:
        out = (C.c_uint32 * 6)()
        self._check(self.lib.dial_exchange_status(self.handle, out))
        return dict(seq=int(out[0]), done=int(out[1]), error=int(out[2]), bars_seq=int(out[3]),
                    update_wait_ns=int(out[4]), bars_wait_ns=int(out[5]))

    def reverse_trajbar(self, weights, rank, qbar, qdbar, xbar):
        self._check(self.lib.dial_reverse_trajbar(self.handle, _ptr(weights), int(rank), _ptr(qbar), _ptr(qdbar),
                                                  _ptr(xbar), _stream()))

    def reverse_trajectories(self):
        """q, qd, x.pos [Nsample+1,Hs+1,*] of the last reverse_rollout (copies)."""
        H = self.Hs + 1
        q, qd, x = self.empty(self.N + 1, H, self.nq), self.empty(self.N + 1, H, self.nv), self.empty(self.N + 1, H, self.nbody - 1, 3)
        self._check(self.lib.dial_reverse_trajectories(self.handle, _ptr(q), _ptr(qd), _ptr(x), _stream()))
        return q, qd, x

    # -- device-resident MPC loop (one CUDA graph per control step) ---------------------------------
    def mpc_bind(self, bufs: dict, M_shift) -> None:
        """``bufs``: name -> CUDA tensor for every field of ``dial_mpc_buffers`` (qbar/qdbar/xbar may be
        None; ``tasks``, [B, sizeof(dial_task)] bytes, may be None or absent).  The tensors must stay alive
        and in place while bound (kept on ``self``)."""
        b = _capi.dial_mpc_buffers()
        want = {"counters": torch.int32, "rng": torch.int32, "tasks": torch.uint8}
        for name, _ in _capi.dial_mpc_buffers._fields_:
            t = bufs.get(name)
            if t is None:
                setattr(b, name, None)
                continue
            assert t.is_cuda and t.is_contiguous() and t.dtype == want.get(name, torch.float32), name
            setattr(b, name, t.data_ptr())
        M = np.ascontiguousarray(M_shift, dtype=np.float32)
        assert M.shape == (self.Hn + 1, self.Hn + 1)
        self._mpc_keep = (dict(bufs), b, M)
        self._check(self.lib.dial_mpc_bind(self.handle, C.byref(b), M.ctypes.data_as(C.c_void_p)))

    def mpc_step(self, n_diffuse: int, env_step=True) -> None:
        """env_step: True / 1 env step + shift, False / 0 plan only, 2 shift + plan (state untouched)."""
        self._check(self.lib.dial_mpc_step(self.handle, int(n_diffuse), int(env_step), _stream()))
