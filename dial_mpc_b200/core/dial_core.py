"""DIAL-MPC planner on the H100 sampling core.

Same class and method surface as the reference ``MBDPI`` (dial_mpc/core/dial_core.py:51-172)
and the same synchronous MPC loop as its ``main()`` (:175-268).  The shift-and-anneal loop
stays in Python; ``reverse_once`` is two kernel stages (rollout, update) reached through the
C ABI, with one NCCL allgather of the per-sample rewards between them when the samples are
sharded over several GPUs (one process per GPU).
"""
from __future__ import annotations

import argparse
import collections
import dataclasses
import importlib
import math
import os
import sys
import time
import types
from typing import Any, Dict, Optional

import numpy as np
import torch
import yaml

import dial_mpc_b200.envs as dial_envs
from dial_mpc_b200 import _capi
from dial_mpc_b200 import random as drandom
from dial_mpc_b200.core.dial_config import DialConfig
from dial_mpc_b200.plan import Plan
from dial_mpc_b200.terrain import PLANNER as TERRAIN_PLANNER, PLANT as TERRAIN_PLANT, terrain_setting, terrains
from dial_mpc_b200.utils.io_utils import get_example_path, load_dataclass_from_dict
from dial_mpc_b200.utils.spline import interp_matrix


def rollout_us(step_env, state, us):
    """Reference semantics of ``rollout_us`` (dial_core.py:36-42) for a *single* action
    sequence, expressed with the env's own ``step`` (used by tests / custom callers)."""
    rews, pipeline_states = [], []
    for u in us:
        state = step_env(state, u)
        rews.append(state.reward)
        pipeline_states.append(state.pipeline_state)
    return torch.stack([torch.as_tensor(r) for r in rews]), pipeline_states


def softmax_update(weights, Y0s, sigma, mu_0t):
    """``softmax_update`` (dial_core.py:45-48) on torch tensors (API parity; the planner's
    own update runs in ``ybar_kernel``)."""
    return torch.einsum("n,nij->ij", weights, Y0s), sigma


def schedule_table(args: DialConfig, n: int, device) -> torch.Tensor:
    """The annealing schedule [n, Hnode+1] of ``args`` (dial_core.py:259-261): the control sigma
    ``horizon_diffuse_factor ** arange(Hnode+1)[::-1] * sigma_scale`` in fp64, rounded to fp32, times
    ``traj_diffuse_factor ** arange(n)`` computed on ``device``.  Every table a plan uses is built here on
    the plan's device: torch's CUDA and CPU ``pow`` may differ in the last bit."""
    sigma = (args.horizon_diffuse_factor ** np.arange(args.Hnode + 1)[::-1]) * args.sigma_scale
    sigma = torch.as_tensor(np.asarray(sigma, dtype=np.float32), device=device)
    f = args.traj_diffuse_factor ** torch.arange(n, device=device, dtype=torch.float32)
    return sigma[None, :] * f[:, None]


class MBDPI:
    def __init__(self, args: DialConfig, env, rank: int = 0, world_size: int = 1, process_group=None,
                 compute_bars: bool = True, plan_factory=None, n_instances: int = 1, n_ensemble: int = 0):
        """``n_instances`` > 1: one plan holds that many independent planner instances (same model,
        config and annealing schedule; own state, rng and knots), advanced together by ``DeviceLoop``.
        ``n_ensemble`` = K >= 1: every instance plans against K member models (``DeviceLoop(...,
        ensemble=...)``) and scores each sample by its reward averaged over them, while its env step runs
        its own model (the plant).  K = 1 with the nominal member is the plain mismatch experiment."""
        self.args = args
        self.env = env
        self.nu = env.action_size
        if args.update_method != "mppi":
            raise KeyError(args.update_method)
        self.update_fn = softmax_update
        self.rank, self.world_size, self.pg = rank, world_size, process_group
        self.compute_bars = compute_bars
        if args.Nsample % world_size != 0:
            raise ValueError("Nsample must be divisible by the number of ranks")
        self.Nlocal = args.Nsample // world_size
        self.n_instances = int(n_instances)
        if self.n_instances < 1:
            raise ValueError("n_instances must be >= 1")
        self.n_ensemble = int(n_ensemble)
        if not 0 <= self.n_ensemble <= _capi.DEFINES["DIAL_MAXENS"]:
            raise ValueError(f"n_ensemble must be in 0..{_capi.DEFINES['DIAL_MAXENS']}, got {self.n_ensemble}")

        sigma_control = args.horizon_diffuse_factor ** np.arange(args.Hnode + 1)[::-1]
        self.sigma_control_np = (sigma_control * args.sigma_scale).astype(np.float64)

        # node to u (dial_core.py:73-77; ctrl_dt is hard-coded to 0.02 there)
        self.ctrl_dt = 0.02
        self.step_us_np = np.linspace(0, self.ctrl_dt * args.Hsample, args.Hsample + 1)
        self.step_nodes_np = np.linspace(0, self.ctrl_dt * args.Hsample, args.Hnode + 1)
        self.node_dt = self.ctrl_dt * (args.Hsample) / (args.Hnode)
        self.M_n2u_np = interp_matrix(self.step_nodes_np, self.step_us_np)
        self.M_u2n_np = interp_matrix(self.step_us_np, self.step_nodes_np)

        desc = env.plan_desc(Nsample=self.Nlocal, Ntotal=args.Nsample, shard_offset=rank * self.Nlocal,
                             Hsample=args.Hsample, Hnode=args.Hnode, temp_sample=args.temp_sample,
                             M_n2u=self.M_n2u_np, n_inst=self.n_instances, n_ens=self.n_ensemble)
        # plan_factory exists for the CPU test harness (tests/emul); the product path is Plan
        self.plan = (plan_factory or Plan)(env, desc)
        dev = self.plan.device
        self.device = dev
        f = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float32), device=dev)
        self.sigma_control = f(self.sigma_control_np)
        self.step_us, self.step_nodes = f(self.step_us_np), f(self.step_nodes_np)
        self.M_n2u, self.M_u2n = f(self.M_n2u_np), f(self.M_u2n_np)
        Hs1 = args.Hsample + 1
        P = np.zeros((Hs1, Hs1))
        P[np.arange(Hs1 - 1), np.arange(1, Hs1)] = 1.0  # roll(-1) with the last row zeroed
        self.M_shift = f(self.M_u2n_np @ P @ self.M_n2u_np)
        # persistent buffers
        N, Nl = args.Nsample, self.Nlocal
        self._rews_local = torch.empty(Nl + 1, dtype=torch.float32, device=dev)
        self._rews_all = torch.empty(N + 1, dtype=torch.float32, device=dev)
        self._weights = torch.empty(N + 1, dtype=torch.float32, device=dev)
        m = env.sys
        self._bars = torch.empty(Hs1 * (m.nq + m.nv + 3 * (m.nbody - 1)), dtype=torch.float32, device=dev)
        # the info-only bars (+ their allreduce) run on a side stream and overlap the next rollout
        self._side = torch.cuda.Stream(device=dev) if dev.type == "cuda" else None
        self._bar_events = []
        # sharded plans: rewards (and bars) are exchanged through NVLink peer memory by the kernels
        # themselves (dial_exchange_*).  DIAL_EXCHANGE=nccl keeps the host-issued NCCL collectives;
        # they are also the fallback when CUDA IPC cannot map the peers (different nodes / no P2P).
        self.xch = False
        self.xch_error = None
        if world_size > 1 and dev.type == "cuda" and hasattr(self.plan, "exchange_setup") \
                and os.environ.get("DIAL_EXCHANGE", "p2p") != "nccl":
            try:
                self.plan.exchange_setup(rank, world_size, process_group)
                self.xch = True
            except Exception as e:  # noqa: BLE001  (kept: reported through exchange_name / bench line)
                self.xch_error = str(e)

    # -- spline maps (dial_core.py:82-101) -------------------------------------------------------
    def node2u(self, nodes):
        return self.M_n2u @ self._t(nodes)

    def u2node(self, us):
        return self.M_u2n @ self._t(us)

    def node2u_vmap(self, Y):      # (horizon, node)
        return self.M_n2u @ self._t(Y)

    def u2node_vmap(self, u):
        return self.M_u2n @ self._t(u)

    def node2u_vvmap(self, Ys):    # (batch, horizon, node)
        return torch.einsum("tk,bka->bta", self.M_n2u, self._t(Ys))

    def u2node_vvmap(self, us):
        return torch.einsum("kt,bta->bka", self.M_u2n, self._t(us))

    def _t(self, x):
        return self.plan.f32(x)

    # -- batched rollout (dial_core.py:80-81) ------------------------------------------------------
    def rollout_us_vmap(self, state, us):
        """-> (rewss [B,H], (q [B,H,nq], qd [B,H,nv], x_pos [B,H,nbody-1,3]))."""
        rewss, q, qd, x = self.plan.rollout(state, us)
        return rewss, (q, qd, x)

    # -- the hot path (dial_core.py:103-145) ----------------------------------------------------------
    def reverse_once(self, state, rng, Ybar_i, noise_scale, eps=None, _sync_bars=True):
        """One annealing iteration.  ``eps`` (optional, [Nsample,Hnode+1,nu]) injects the noise;
        otherwise it is drawn in-kernel from the Threefry stream keyed by ``split(rng)[1]``."""
        self._single("reverse_once")
        rng, Y0s_rng = drandom.split(rng)
        Ybar_i = self._t(Ybar_i)
        noise_scale = self._t(noise_scale)
        if eps is not None:
            eps = self.plan.f32(eps, (self.args.Nsample, self.args.Hnode + 1, self.nu))
        key = None if eps is not None else Y0s_rng
        N, Nl = self.args.Nsample, self.Nlocal
        if self._side is not None and len(self._bar_events) >= 2:
            # the trajectory buffer about to be overwritten was read by the bars two iterations ago
            torch.cuda.current_stream().wait_event(self._bar_events.pop(0))
        Ybar = torch.empty_like(Ybar_i)
        weights = torch.empty_like(self._weights)
        if self.world_size == 1:
            rews = torch.empty_like(self._rews_local)      # fresh output (functional API), written by the kernel
            self.plan.reverse_rollout(state, eps, key, Ybar_i, noise_scale, rews)
            self.plan.reverse_update(eps, key, Ybar_i, noise_scale, rews, Ybar, weights)
        elif self.xch:
            # the rollout epilogue stores the rewards into every rank's mailbox; the weights kernel waits
            rews = torch.empty_like(self._rews_all)
            self.plan.reverse_rollout(state, eps, key, Ybar_i, noise_scale, self._rews_local)
            self.plan.reverse_update(eps, key, Ybar_i, noise_scale, None, Ybar, weights, rews_gathered=rews)
        else:
            import torch.distributed as dist
            self.plan.reverse_rollout(state, eps, key, Ybar_i, noise_scale, self._rews_local)
            dist.all_gather_into_tensor(self._rews_all[:N], self._rews_local[:Nl], group=self.pg)
            self._rews_all[N:].copy_(self._rews_local[Nl:])
            rews = self._rews_all.clone()
            self.plan.reverse_update(eps, key, Ybar_i, noise_scale, rews, Ybar, weights)
        info: Dict[str, Any] = {"rews": rews, "new_noise_scale": noise_scale, "weights": weights}
        if self.compute_bars:
            m = self.env.sys
            Hs1 = self.args.Hsample + 1
            n1, n2 = Hs1 * m.nq, Hs1 * m.nv
            bars = torch.empty_like(self._bars)
            qbar, qdbar, xbar = bars[:n1], bars[n1:n1 + n2], bars[n1 + n2:]
            main = torch.cuda.current_stream() if self._side is not None else None
            if self._side is not None:
                self._side.wait_stream(main)
                ctx = torch.cuda.stream(self._side)
            else:
                import contextlib
                ctx = contextlib.nullcontext()
            with ctx:
                self.plan.reverse_trajbar(weights, self.rank, qbar, qdbar, xbar)   # exchange on: already the all-rank sum
                if self.world_size > 1 and not self.xch:
                    import torch.distributed as dist
                    dist.all_reduce(bars, group=self.pg)
                if self._side is not None:
                    ev = torch.cuda.Event()
                    ev.record(self._side)
                    self._bar_events.append(ev)
                    for t in (bars, weights):
                        t.record_stream(self._side)
            if self._side is not None and _sync_bars:
                main.wait_stream(self._side)
            info["qbar"] = qbar.view(Hs1, m.nq)
            info["qdbar"] = qdbar.view(Hs1, m.nv)
            info["xbar"] = xbar.view(Hs1, m.nbody - 1, 3)
        return rng, Ybar, info

    def _single(self, what: str) -> None:
        if self.n_instances > 1:
            raise RuntimeError(f"MBDPI.{what} plans one instance; a plan of {self.n_instances} instances runs "
                               "through DeviceLoop (one CUDA graph per control step for all instances)")
        if self.n_ensemble > 0:
            raise RuntimeError(f"MBDPI.{what} plans on the plan's own model; an ensemble plan (n_ensemble = "
                               f"{self.n_ensemble}) runs through DeviceLoop, which rolls every member")

    @property
    def exchange_name(self) -> str:
        if self.world_size == 1:
            return "no exchange (single GPU)"
        return ("one peer-memory exchange fused into the rollout epilogue / weights prologue (NVLink stores + flags)"
                if self.xch else "one NCCL allgather" + (f" (peer exchange unavailable: {self.xch_error})" if self.xch_error else ""))

    def phase_times(self, state, key, Ybar_i, noise_scale, reps: int = 10) -> Dict[str, float]:
        """Device time (microseconds, CUDA events on the current stream) of the stages of one
        ``reverse_once``: rollout | rewards exchange | weights + Ybar | bars (+ their allreduce).
        Measurement aid for bench.py; the stages run back to back on one stream here."""
        self._single("phase_times")
        Ybar_i, noise_scale = self._t(Ybar_i), self._t(noise_scale)
        N, Nl = self.args.Nsample, self.Nlocal
        m = self.env.sys
        Hs1 = self.args.Hsample + 1
        n1, n2 = Hs1 * m.nq, Hs1 * m.nv
        bars = torch.empty_like(self._bars)
        Ybar = torch.empty_like(Ybar_i)
        acc = {"rollout": 0.0, "exchange": 0.0, "update": 0.0, "bars": 0.0}
        for rep in range(reps + 2):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
            ev[0].record()
            self.plan.reverse_rollout(state, None, key, Ybar_i, noise_scale, self._rews_local)
            ev[1].record()
            if self.world_size > 1 and not self.xch:
                import torch.distributed as dist
                dist.all_gather_into_tensor(self._rews_all[:N], self._rews_local[:Nl], group=self.pg)
                self._rews_all[N:].copy_(self._rews_local[Nl:])
                rews_all = self._rews_all
            else:
                rews_all = None if self.xch else self._rews_local   # exchange: the wait is inside the update stage
            ev[2].record()
            self.plan.reverse_update(None, key, Ybar_i, noise_scale, rews_all, Ybar, self._weights)
            ev[3].record()
            self.plan.reverse_trajbar(self._weights, self.rank, bars[:n1], bars[n1:n1 + n2], bars[n1 + n2:])
            if self.world_size > 1 and not self.xch:
                dist.all_reduce(bars, group=self.pg)
            ev[4].record()
            torch.cuda.synchronize()
            if rep >= 2:
                for i, k in enumerate(acc):
                    acc[k] += ev[i].elapsed_time(ev[i + 1]) * 1e3 / reps
        return acc

    def reverse_scan(self, state, rng, Y0, factors):
        """``lax.scan(reverse_scan, (rng, Y0, state), factors)`` of dial_core.py:177-180,262-264."""
        self._single("reverse_scan")
        info = None
        n = factors.shape[0]
        for i in range(n):
            rng, Y0, info = self.reverse_once(state, rng, Y0, factors[i], _sync_bars=(i == n - 1))
        return rng, Y0, info

    def schedule(self, n_diffuse: int) -> torch.Tensor:
        """``sigma_control * traj_diffuse_factor ** arange(n_diffuse)[:, None]`` (dial_core.py:259-261)."""
        return schedule_table(self.args, n_diffuse, self.device)

    # -- shift (dial_core.py:160-172) -------------------------------------------------------------------
    def shift(self, Y):
        return self.M_shift @ self._t(Y)

    def shift_Y_from_u(self, u, n_step):
        u = self._t(u)
        u = torch.roll(u, -n_step, dims=0)
        u[-n_step:] = 0.0
        return self.u2node_vmap(u)


class DeviceLoop:
    """Device-resident synchronous MPC loop: the reference's per-step sequence
    (dial_core.py:242-268) — ``state = step_env(state, Y0[0]); Y0 = shift(Y0); Y0 = reverse_scan(...)``
    — replayed as ONE CUDA graph per control step (C ABI ``dial_mpc_bind`` / ``dial_mpc_step``).
    State, step counters, rng and control knots live in device tensors owned by this object; the
    host only launches the graph and reads back what it needs (e.g. ``action``).  Equals the
    eager ``env.step`` + ``MBDPI.shift`` + ``MBDPI.reverse_scan`` sequence (tests/test_gpu_parity.py).
    Sharded plans replay the same graph on every rank (one process per GPU): the rewards cross
    the GPUs inside the kernels (peer-memory exchange), so no host collective sits in the step."""

    def __init__(self, mbdpi: "MBDPI", state, rng, Y0=None, n_diffuse_max: Optional[int] = None,
                 compute_bars: bool = True, noise=None, envs=None, ensemble=None, risk=None, adapt=None, prior=None,
                 schedule=None, delay=None, observe=None, pushes=None, plant=None, terrain=None):
        """``noise`` [>= n_diffuse_max, Hnode+1]: annealing schedule, default ``mbdpi.schedule`` (the
        deploy planner passes its own, dial_plan.py:199-209).

        Batched ``mbdpi`` (``n_instances`` = B > 1): ``state`` is a sequence of B States, ``rng`` [B,2]
        uint32 and ``Y0`` [B,Hnode+1,nu] or None.  Every per-instance buffer, ``Y``, ``action``,
        ``reward``, ``info()`` and ``set_state`` gain a leading [B]; ``state(b)`` materialises
        instance b.  Instance b computes bitwise what a single-instance loop from its state, rng and
        knots computes.

        ``envs``: B env objects of ``mbdpi.env``'s class, one task per instance (commands, gait, jump
        sequence, custom-reward user constants; ``BaseEnv.task``).  Every other field of their plan
        descriptors must equal ``mbdpi.env``'s: the plan shares it.  Instance b then computes bitwise
        what a single-instance loop on ``envs[b]`` computes.  An env whose ``sys.model`` differs from
        ``mbdpi.env``'s also gives its instance that physical model (``dial_plan_set_instance_model``:
        the same structure, timestep, joint and control ranges; masses, friction, damping, gravity, ...
        may differ).  A batched loop whose states all carry
        ``randomize_target`` binds per-instance tasks as well: each instance draws its own commands
        (and seq-jump its own jump sequence, from its state's info).

        ``ensemble`` (an ``mbdpi`` with ``n_ensemble`` = K >= 1): the planning models, either one list of K
        envs, ``System``s or ``CompiledModel``s shared by every instance, or B such lists (one per
        instance).  ``envs[b]``'s model stays instance b's plant (the env step); the rollouts of member k
        run ``ensemble[k]`` (or ``ensemble[b][k]``), and ``rews`` receives each sample's reward averaged
        over the members.  A member whose model equals ``mbdpi.env``'s needs no upload; None: every
        member is ``mbdpi.env``'s model.

        ``risk`` (an ensemble ``mbdpi``): how each sample's member rewards become its score, one risk spec
        for every instance or a list of B (``risk_setting``: ``{"aggregate": "mean"}``, the default,
        ``{"aggregate": "worst"}`` or ``{"aggregate": "cvar", "alpha": a}``).

        ``adapt`` (an ensemble ``mbdpi`` with K >= 2): instances that adapt their belief over the members to
        their plant at every env step and score samples by the belief-weighted risk measure, one adapt spec
        for every instance or a list of B specs or None (``adapt_setting``: ``{"sigma": s, "forget": 1.0,
        "prune": 0.0}``).  ``prior``: the starting belief, K weights >= 0 with a positive sum for every
        instance or B such lists (default uniform; ``set_belief``).

        ``schedule``: each instance's own sampling schedule, one schedule spec for every instance or a list of
        B specs or None (the plan's; ``schedule_setting``: any of ``temp_sample``, ``sigma_scale``,
        ``horizon_diffuse_factor``, ``traj_diffuse_factor``, ``Ndiffuse``, ``Ndiffuse_init``).  Instance b then
        computes bitwise what a single-instance loop on an MBDPI with b's updated DialConfig computes
        (``set_schedule``, ``step``).

        ``delay``: each instance's control latency, one delay spec for every instance or a list of B specs or
        None (``delay_setting``: an int d, or ``{"steps": d, "predict": True}``).  The action planned at step t
        reaches the plant at step t + d; a predicting instance plans from the plant state predicted d steps
        ahead through its queued actions on its planning model (``set_delay``, ``pending_actions``,
        ``planning_state``).

        ``observe``: each instance's view of its plant, one observe spec for every instance or a list of B specs
        or None (``observe_setting``: ``{"delay": k, "qpos": S, "qvel": S, "seed": s}``).  Instance b's
        rollouts start from the plant record min(k, records - 1) env steps old plus Gaussian noise drawn once
        per env step; a predicting instance (its delay spec's ``predict``) first takes the actions applied since
        that record and its queued ones.  The plant, its reward and adaptation keep the plant state
        (``set_observation``, ``observed_state``, ``planning_state``).

        ``pushes``: each instance's pushes, one push spec for every instance or a list of B specs or None
        (``push_setting``: a list of ``{"step": s, "steps": n, "body": name, "pos": p, "force": f, "torque": t}``).
        After each env step whose post-step counter lies in [s, s + n), the plant's qvel takes the impulse of
        the force at the point p of the body and of the torque, held over that env step.  The planner is not
        told; the trigger moves with the counter (``set_state(step=...)``) (``set_pushes``).

        ``plant``: each instance's plant fidelity, one plant spec for every instance or a list of B specs (or
        Nones) or None (``plant_setting``: a mapping of ``substeps`` or ``sim_dt``, ``iterations``,
        ``ls_iterations`` and ``tolerance``, each defaulting to the planner's own).  With a spec, the instance's
        env step makes substeps x n_frames physics steps of timestep / substeps on its plant model with those
        solver settings, the control held across them; the planner, the members and the predictions keep the
        plan's discretisation (``set_plant``).

        ``terrain``: each instance's ground, one terrain spec for every instance or a list of B specs (or Nones) or
        None (``terrain.terrain_setting``: ``{"kind": "rough", "amplitude": a, "wavelength": w, "seed": s}``,
        ``{"kind": "slope", "angle": deg}`` or ``{"kind": "grid", "heights": ..., "spacing": s}``, with
        ``"planner": True`` for a planner that plans on the same ground).  The heightfield replaces the floor
        plane in the instance's env steps, and the built-in rewards measure heights above it (``set_terrain``)."""
        if mbdpi.world_size != 1 and not mbdpi.xch:
            raise RuntimeError("DeviceLoop on a sharded plan needs the peer-memory exchange (dial_exchange_*); "
                               f"it is off: {mbdpi.xch_error or 'DIAL_EXCHANGE=nccl'}")
        self.mbdpi, self.plan = mbdpi, mbdpi.plan
        a, pl, dev = mbdpi.args, mbdpi.plan, mbdpi.device
        nmax = int(n_diffuse_max or max(a.Ndiffuse, a.Ndiffuse_init))
        f, e = pl.f32, pl.empty
        Hs1 = a.Hsample + 1
        m = mbdpi.env.sys
        B = self.n_instances = mbdpi.n_instances
        states = list(state) if B > 1 else [state]
        if len(states) != B:
            raise ValueError(f"a plan of {B} instances needs {B} states, got {len(states)}")
        rand = [bool(s.info.get("randomize_target", False)) for s in states]
        if any(rand) and not all(rand):
            raise RuntimeError("randomize_tasks draws per-instance commands: in a batched DeviceLoop either every "
                               "state carries randomize_target or none does")
        settings = resolve_settings(B, mbdpi.n_ensemble, mbdpi.env, a, mbdpi.world_size, rand[0], envs=envs,
                                    ensemble=ensemble, risk=risk, prior=prior, adapt=adapt, schedule=schedule,
                                    delay=delay, observe=observe, pushes=pushes, plant=plant, terrain=terrain)
        envs = [spec for spec, _ in settings["envs"]] if "envs" in settings else None
        lead = (B,) if B > 1 else ()
        key = np.ascontiguousarray(rng, dtype=np.uint32)
        if key.shape != lead + (2,):
            raise ValueError(f"rng must have shape {lead + (2,)}, got {key.shape}")
        if Y0 is not None and tuple(np.shape(Y0)) != lead + (a.Hnode + 1, mbdpi.nu):
            raise ValueError(f"Y0 must have shape {lead + (a.Hnode + 1, mbdpi.nu)}, got {tuple(np.shape(Y0))}")
        # each instance's DialConfig, whether it has a table of its own, and the iteration limits last
        # uploaded (None: no limits, every instance runs every iteration of a step)
        self._cfg, self._own, self._lims = [a] * B, [False] * B, None
        # each instance's (steps, predict) as last set, and its observation setting (None: none)
        self._delay = [(0, False)] * B
        self._observe = [None] * B
        ps = [s.pipeline_state for s in states]
        per = (lambda t: t[0]) if B == 1 else torch.stack   # one instance: the buffers keep their plain shapes
        counters = [[int(s.info.get("step", 0)), int(s.info.get("contact_stage", 0))] for s in states]
        self.info0 = dict(state.info) if B == 1 else [dict(s.info) for s in states]
        self.buf = dict(
            qpos=per([f(p.qpos) for p in ps]).clone(), qvel=per([f(p.qvel) for p in ps]).clone(),
            qacc_warmstart=per([f(p.qacc_warmstart) for p in ps]).clone(),
            counters=torch.tensor(counters[0] if B == 1 else counters, dtype=torch.int32, device=dev),
            rng=torch.as_tensor(key.view(np.int32).copy(), device=dev),
            Y=(torch.zeros(*lead, a.Hnode + 1, mbdpi.nu, device=dev) if Y0 is None else f(Y0).clone()),
            ctrl=torch.zeros(*lead, mbdpi.nu, device=dev), reward=torch.zeros(B, device=dev),
            rews=torch.zeros(*lead, mbdpi.Nlocal + 1, device=dev),
            rews_all=(torch.zeros(a.Nsample + 1, device=dev) if mbdpi.world_size > 1 else None),
            qbar=e(*lead, Hs1, m.nq) if compute_bars else None, qdbar=e(*lead, Hs1, m.nv) if compute_bars else None,
            xbar=e(*lead, Hs1, m.nbody - 1, 3) if compute_bars else None,
            noise=(mbdpi.schedule(nmax) if noise is None else f(noise)).contiguous())
        assert tuple(self.buf["noise"].shape) == (nmax, a.Hnode + 1) or self.buf["noise"].shape[0] >= nmax
        self.n_diffuse_max = nmax
        # randomize_tasks: per instance, a host mirror of info["step"] / info["rng"] (the env's key chain),
        # from which the one-step random command the horizon may reach is computed ahead
        # (BaseEnv.command_override)
        self._rand = rand[0]
        self._env_info = [{"randomize_target": self._rand, "step": int(s.info.get("step", 0)),
                           "rng": np.asarray(s.info.get("rng", np.zeros(2)), dtype=np.uint32).copy()} for s in states]
        # per-instance tasks: an explicit env per instance, or per-instance random commands
        self._envs = envs if envs is not None else [mbdpi.env] * B
        self._tasks_host = None
        if envs is not None or (B > 1 and self._rand):
            self._tasks_host = [e.task() for e in self._envs]
            if self._rand and hasattr(mbdpi.env, "stage_tables"):
                # seq-jump: the jump sequence drawn at reset is constant afterwards
                for b, s in enumerate(states):
                    _capi.task_set_stages(self._tasks_host[b], self._envs[b].stage_tables(s.info))
            self._task_cmd = [()] * B       # command override last uploaded per instance (() = none yet)
            self.buf["tasks"] = torch.from_numpy(
                np.stack([np.frombuffer(bytes(t), np.uint8) for t in self._tasks_host])).to(dev)
        elif self._rand and hasattr(mbdpi.env, "stage_tables"):
            # seq-jump: the jump sequence drawn at reset is constant afterwards; one upload at bind time
            pl.set_stages(mbdpi.env.stage_tables(states[0].info))
        pl.mpc_bind(self.buf, mbdpi.M_shift.cpu().numpy())
        # a setting that changes nothing is not applied: the plan then allocates nothing for it and keeps its launches
        for s in SETTINGS:
            for b, (spec, setting) in enumerate(settings.get(s.key, ())):
                if not s.identity(setting):
                    s.apply(self, b, spec, setting)

    def _instance(self, b) -> int:
        b = int(b)
        if not 0 <= b < self.n_instances:
            raise IndexError(f"instance {b} out of range (0..{self.n_instances - 1})")
        return b

    def _need_ensemble(self, what: str, k: int) -> None:
        if self.mbdpi.n_ensemble < k:
            raise RuntimeError(f"{what} needs an MBDPI built with n_ensemble >= {k}")

    @staticmethod
    def _check_shared(ref_env, env) -> None:
        """``env`` may give an instance of ``ref_env``'s plan its task: same class, and the same plan
        descriptor outside the task fields."""
        if type(env) is not type(ref_env):
            raise ValueError(f"every instance's env must be a {type(ref_env).__name__}, got {type(env).__name__}")
        diff = _capi.first_shared_difference(ref_env.plan_desc(), env.plan_desc())
        if diff is not None:
            raise ValueError(f"plan descriptor field '{diff}' differs between the instances' envs; it is shared "
                             "by every instance of a plan (only the dial_task fields may differ)")

    def _upload_task(self, b: int) -> None:
        """Stream-ordered copy of instance b's host task into the bound tasks (no host synchronisation)."""
        t = self._tasks_host[b]
        src = torch.from_numpy(np.frombuffer(bytes(t), np.uint8).copy())
        self.buf["tasks"][b].copy_(src, non_blocking=True)

    def set_task(self, b: int, env_or_task) -> None:
        """Replace instance b's task before the next ``step``: an env of ``mbdpi.env``'s class (its
        ``task()``; the shared fields must match) or a ``_capi.dial_task``.  A stream-ordered copy on
        the current stream, no host synchronisation.  Needs a loop with per-instance tasks bound
        (``envs=`` or batched ``randomize_tasks``); randomize_tasks loops keep applying each instance's
        one-step random command on top."""
        if self._tasks_host is None:
            raise RuntimeError("set_task needs per-instance tasks: build the DeviceLoop with envs=[...]")
        b = self._instance(b)
        if isinstance(env_or_task, _capi.dial_task):
            t = _capi.check_task(_capi.dial_task.from_buffer_copy(env_or_task))
        else:
            self._check_shared(self.mbdpi.env, env_or_task)
            t = env_or_task.task()
        self._tasks_host[b] = t
        self._task_cmd[b] = ()
        self._upload_task(b)

    def set_model(self, b: int, env_or_sys) -> None:
        """Replace instance b's physical model before the next ``step``: an env (its ``sys``), a
        ``System`` or a ``CompiledModel`` with the structure, timestep, joint and control ranges of
        ``mbdpi.env``'s model.  A stream-ordered copy on the current stream.  The first per-instance
        model of a loop makes the next steps capture their graphs again."""
        self.plan.set_instance_model(self._instance(b), getattr(env_or_sys, "sys", env_or_sys))

    def set_ensemble_model(self, b: int, k: int, env_or_sys) -> None:
        """Replace member k of instance b's planning ensemble before the next ``step``: an env, a ``System``
        or a ``CompiledModel`` (``Plan.set_ensemble_model``).  The first member set on a loop makes the next
        steps capture their graphs again."""
        self._need_ensemble("set_ensemble_model", 1)
        b, k = self._instance(b), int(k)
        if not 0 <= k < self.mbdpi.n_ensemble:
            raise IndexError(f"member {k} out of range (0..{self.mbdpi.n_ensemble - 1})")
        self.plan.set_ensemble_model(b, k, _model(env_or_sys))

    def set_risk(self, b: int, spec) -> None:
        """Instance b's risk measure over its members' rewards from the next ``step`` on (a risk spec,
        ``risk_setting``).  A stream-ordered copy on the current stream; the captured graphs are kept."""
        self._need_ensemble("set_risk", 1)
        self.plan.set_ensemble_risk(self._instance(b), *risk_setting(spec, self.mbdpi.n_ensemble))

    def set_adapt(self, b: int, spec) -> None:
        """Instance b adapts its belief to its plant from the next env step on (an adapt spec,
        ``adapt_setting``), or stops adapting (None; the belief is kept).  A stream-ordered copy on the
        current stream; the first instance of a loop to adapt makes the next steps capture their graphs
        again, later calls keep them."""
        self._need_ensemble("set_adapt", 2)
        b = self._instance(b)
        if spec is None:
            self.plan.set_ensemble_adapt(b, False)
        else:
            self.plan.set_ensemble_adapt(b, True, *adapt_setting(spec, self.mbdpi.n_ensemble, self.mbdpi.env.sys.nv))

    def set_belief(self, b: int, w) -> None:
        """Instance b's belief from K weights >= 0 with a positive sum (``prior_setting``), e.g. from an
        outside estimator; a stream-ordered copy that keeps the captured graphs."""
        self._need_ensemble("set_belief", 2)
        self.plan.set_ensemble_belief(self._instance(b), prior_setting(w, self.mbdpi.n_ensemble))

    def _belief(self, which: int) -> torch.Tensor:
        self._need_ensemble(("belief", "member_loglik")[which], 2)
        out = self.plan.empty(*((self.n_instances,) if self.n_instances > 1 else ()), self.mbdpi.n_ensemble)
        self.plan.ensemble_belief(*((out, None) if which == 0 else (None, out)))
        return out

    def belief(self) -> torch.Tensor:
        """The belief over the members after the steps launched so far, a new tensor [B, K] ([K] for one
        instance).  Asynchronous on the current stream."""
        return self._belief(0)

    def member_loglik(self) -> torch.Tensor:
        """The members' log-likelihoods l of each instance's last belief update, [B, K] ([K] for one
        instance; 0 before the first).  Asynchronous on the current stream."""
        return self._belief(1)

    def member_rewards(self) -> torch.Tensor:
        """The member rewards of the last diffusion iteration of the steps launched so far, a new tensor
        [B, K, Nsample+1] ([K, Nsample+1] for one instance): the rewards each sample's score reduces
        (``Plan.member_rewards``).  Asynchronous on the current stream."""
        self._need_ensemble("member_rewards", 1)
        lead = (self.n_instances,) if self.n_instances > 1 else ()
        return self.plan.member_rewards(self.plan.empty(*lead, self.mbdpi.n_ensemble, self.mbdpi.Nlocal + 1))

    def set_schedule(self, b: int, spec) -> None:
        """Instance b's sampling schedule from the next ``step`` on: a schedule spec (``schedule_setting``),
        or None for the plan's own.  Its noise table (``schedule_table`` of the updated DialConfig, max(Ndiffuse,
        Ndiffuse_init) rows, on the plan's device) and temperature go to the plan with a stream-ordered copy on
        the current stream.  The first schedule of a loop makes the next steps capture their graphs again,
        later calls keep them."""
        b = self._instance(b)
        if spec is None:
            if self._own[b]:
                self.plan.set_instance_schedule(b, noise=None)
            self._cfg[b], self._own[b] = self.mbdpi.args, False
            return
        cfg = schedule_setting(spec, self.mbdpi.args)
        table = schedule_table(cfg, max(cfg.Ndiffuse, cfg.Ndiffuse_init), self.mbdpi.device)
        self.plan.set_instance_schedule(b, float(np.float32(cfg.temp_sample)), table)
        self._cfg[b], self._own[b] = cfg, True

    def set_delay(self, b: int, spec) -> None:
        """Instance b's control latency from the next ``step`` on (a delay spec, ``delay_setting``).  Refills its
        queue with d copies of its current ``Y[0]``: until then the plant applies the plan it holds.  A
        stream-ordered copy on the current stream.  The first delay of a loop, and a call that changes the
        number of prediction launches or whether any instance predicts through its delay, change the launch
        sequence: the next steps capture their graphs again.  Other calls keep them."""
        b = self._instance(b)
        steps, predict = delay_setting(spec)
        self.plan.set_instance_delay(b, steps, predict)
        self._delay[b] = (steps, predict)

    _RAND_OBSERVE = ("an observation delay needs a loop without randomize_tasks: its rollouts would start before "
                     "the current command window (noise alone is allowed)")

    @staticmethod
    def _observing(setting) -> bool:
        return setting[0] > 0 or bool(setting[1].any()) or bool(setting[2].any())

    def _set_observation(self, b: int, setting) -> None:
        self.plan.set_instance_observation(b, *setting)
        self._observe[b] = setting if self._observing(setting) else None

    def set_observation(self, b: int, spec) -> None:
        """Instance b plans from an observation of its plant from the next ``step`` on (an observe spec,
        ``observe_setting``), or from its plant state again (None).  Resets its history: the next step seeds it
        from the plant, and its noise restarts from the spec's seed.  A stream-ordered copy on the current
        stream.  The first observation of a loop, and a call that changes the number of prediction launches
        (max(k + d) over the predicting instances), change the launch sequence: the next steps capture their
        graphs again.  Other calls keep them."""
        b = self._instance(b)
        if spec is None:
            if self._observe[b] is not None:
                nv = self.mbdpi.env.sys.nv
                self._set_observation(b, (0, np.zeros(nv, np.float32), np.zeros(nv, np.float32), np.zeros(2, np.uint32)))
            return
        setting = observe_setting(spec, self.mbdpi.env.sys)
        if self._rand and setting[0] > 0:
            raise ValueError(self._RAND_OBSERVE)
        self._set_observation(b, setting)

    def set_pushes(self, b: int, spec) -> None:
        """Instance b's push table from the next ``step`` on (a push spec, ``push_setting``; None or [] clears
        it).  A stream-ordered copy on the current stream.  The first table of a loop changes the launch sequence:
        the next steps capture their graphs again.  Later calls keep them."""
        self.plan.set_instance_pushes(self._instance(b), push_setting(spec, self.mbdpi.env.sys))

    def set_plant(self, b: int, spec) -> None:
        """Instance b's plant fidelity from the next ``step`` on (a plant spec, ``plant_setting``; None clears it:
        the plant then steps like the planner).  Stream-ordered on the current stream.  The first setting of a
        loop, and any later one that changes the set of distinct substep counts in use, changes the launch
        sequence: the next steps capture their graphs again.  Other calls keep them."""
        self.plan.set_instance_plant(self._instance(b), plant_setting(spec, self.mbdpi.env.sys))

    def set_terrain(self, b: int, spec) -> None:
        """Instance b's terrain from the next ``step`` on (a terrain spec, ``terrain.terrain_setting``; None: the
        flat floor on both sides).  Stream-ordered on the current stream.  The first terrain on a side, and a grid
        larger than the instance's earlier ones, change the launch sequence: the next steps capture their graphs
        again.  Other calls keep them."""
        _set_terrain(self, self._instance(b), None if spec is None else terrain_setting(spec, self.mbdpi.env.sys))

    def observed_state(self) -> Dict[str, torch.Tensor]:
        """The observation the last step planned from, before any prediction: new tensors ``qpos``, ``qvel``,
        ``qacc_warmstart``, ``counters`` (int32 {step, contact_stage}) and ``age`` (int32, how many env steps
        old the observed record is), with a leading [B] on a batched loop; the plant state at age 0 for an
        instance without an observation.  Asynchronous on the current stream."""
        lead = (self.n_instances,) if self.n_instances > 1 else ()
        m = self.mbdpi.env.sys
        i32 = dict(dtype=torch.int32, device=self.mbdpi.device)
        out = dict(qpos=self.plan.empty(*lead, m.nq), qvel=self.plan.empty(*lead, m.nv),
                   qacc_warmstart=self.plan.empty(*lead, m.nv), counters=torch.empty(*lead, 2, **i32),
                   age=torch.empty(*lead, **i32) if lead else torch.empty(1, **i32))
        self.plan.observed_state(out["qpos"], out["qvel"], out["qacc_warmstart"], out["counters"], out["age"])
        if not lead:
            out["age"] = out["age"][0]
        return out

    def pending_actions(self) -> torch.Tensor:
        """Each instance's queued actions in the order the next env steps apply them, a new tensor [B, 16, nu]
        ([16, nu] for one instance; rows past the instance's delay are zero).  Asynchronous on the current
        stream."""
        lead = (self.n_instances,) if self.n_instances > 1 else ()
        return self.plan.pending_actions(self.plan.empty(*lead, _capi.DEFINES["DIAL_MAXDELAY"], self.mbdpi.nu))

    def planning_state(self) -> Dict[str, torch.Tensor]:
        """The state the last step's planning rollouts started from, new tensors ``qpos``, ``qvel``,
        ``qacc_warmstart`` and ``counters`` (int32 {step, contact_stage}) with a leading [B] on a batched loop:
        the predicted state of a predicting instance, the observation of an observing one, the plant state of
        any other.  Asynchronous on the current stream."""
        lead = (self.n_instances,) if self.n_instances > 1 else ()
        m = self.mbdpi.env.sys
        out = dict(qpos=self.plan.empty(*lead, m.nq), qvel=self.plan.empty(*lead, m.nv),
                   qacc_warmstart=self.plan.empty(*lead, m.nv),
                   counters=torch.empty(*lead, 2, dtype=torch.int32, device=self.mbdpi.device))
        self.plan.planning_state(out["qpos"], out["qvel"], out["qacc_warmstart"], out["counters"])
        return out

    def step(self, n_diffuse: Optional[int] = None, env_step=True, initial: bool = False) -> None:
        """One control step (asynchronous on the current stream).  env_step: True = env step + shift
        + plan (the reference's main loop), False = plan only, 2 = shift + plan (state untouched).
        ``n_diffuse`` None: each instance runs its own ``Ndiffuse`` (``Ndiffuse_init`` with ``initial``); an
        int: every instance runs that many iterations, each with its own table and temperature.  The step's
        graph runs the largest count; instances with fewer skip the rest (iteration limits, uploaded when the
        counts need other limits than those the plan holds)."""
        if n_diffuse is None:
            counts = [c.Ndiffuse_init if initial else c.Ndiffuse for c in self._cfg]
        else:
            counts = [int(n_diffuse)] * self.n_instances
        n = max(counts)
        if any(c > self.n_diffuse_max for c, own in zip(counts, self._own) if not own):
            raise ValueError("n_diffuse exceeds the bound noise schedule")
        lim = self._lims or [n] * self.n_instances    # no limits: every instance runs all n iterations
        if any(min(n, l) != c for l, c in zip(lim, counts)):
            self.plan.set_instance_iterations(counts)
            self._lims = list(counts)
        stepping = env_step is True or env_step == 1
        if self._rand:
            # the env step (if any) runs at info["step"], the rollouts cover the Hsample+1 steps after it; a
            # predicting instance's prediction steps and rollouts reach d steps further
            ahead = [d if p else 0 for d, p in self._delay]
            horizon = self.mbdpi.args.Hsample + (2 if stepping else 1)
            if self._tasks_host is None:
                self.plan.set_command(self.mbdpi.env.command_override(self._env_info[0], horizon + max(ahead)))
            else:
                for b, info in enumerate(self._env_info):
                    ov = self._envs[b].command_override(info, horizon + ahead[b])
                    key = _capi.task_set_command(self._tasks_host[b], ov)
                    if key != self._task_cmd[b]:      # upload only the instances whose command changed
                        self._upload_task(b)
                        self._task_cmd[b] = key
        self.plan.mpc_step(n, env_step)
        if stepping:
            for info in self._env_info:
                info["step"] += 1
                if self._rand:
                    info["rng"] = drandom.split(info["rng"])[0]

    def rng_host(self) -> np.ndarray:
        """The planner rng after the steps launched so far (synchronises)."""
        return self.buf["rng"].cpu().numpy().view(np.uint32).copy()

    def set_state(self, qpos, qvel, qacc_warmstart=None, step: Optional[int] = None) -> None:
        """Overwrite the planning state (deploy: the state comes from the robot / simulator).  ``step``
        sets ``info["step"]`` only, like the reference's ``update_mjx_state`` (dial_plan.py:149-155):
        a seq-jump ``contact_stage`` is whatever the bound state carries.  Batched loops: [B,...]
        arrays and ``step`` an int or [B].  Each observing instance starts its history again from the new
        state, and its noise from its seed, as ``set_observation`` does."""
        self.buf["qpos"].copy_(self.plan.f32(qpos))
        self.buf["qvel"].copy_(self.plan.f32(qvel))
        if qacc_warmstart is not None:
            self.buf["qacc_warmstart"].copy_(self.plan.f32(qacc_warmstart))
        if step is not None and self.n_instances > 1:
            steps = np.broadcast_to(np.asarray(step, dtype=np.int32), (self.n_instances,))
            self.buf["counters"][:, 0] = torch.as_tensor(steps.copy(), device=self.buf["counters"].device)
            for info, s in zip(self._env_info, steps):
                info["step"] = int(s)
        elif step is not None:
            self.buf["counters"][0] = int(step)
            self._env_info[0]["step"] = int(step)
        # the observing instances start their history again from the new state (and their noise from the seed)
        for b, setting in enumerate(self._observe):
            if setting is not None:
                self.plan.set_instance_observation(b, *setting)

    @property
    def action(self) -> torch.Tensor:
        """``Y0[0]``: the action the next env step applies (device view; batched: [B,nu]).  With a delay it is
        the action the next env step puts at the back of the instance's queue; the env step applies the
        queue's front (``pending_actions()[..., 0, :]``)."""
        return self.buf["Y"][:, 0] if self.n_instances > 1 else self.buf["Y"][0]

    @property
    def Y(self) -> torch.Tensor:
        return self.buf["Y"]

    @property
    def reward(self) -> torch.Tensor:
        return self.buf["reward"] if self.n_instances > 1 else self.buf["reward"][0]

    def info(self) -> Dict[str, Any]:
        b = self.buf
        d = {"rews": b["rews_all"] if b["rews_all"] is not None else b["rews"]}
        if b["qbar"] is not None:
            d.update(qbar=b["qbar"], qdbar=b["qdbar"], xbar=b["xbar"])
        return d

    def state(self, i: Optional[int] = None):
        """Materialise the env ``State`` (synchronises: reads the counters); batched loops: that of
        instance ``i``."""
        from dial_mpc_b200.envs.base_env import PipelineState, State
        if self.n_instances > 1:
            if i is None:
                raise ValueError("a batched DeviceLoop materialises one instance: state(i)")
            b = {k: (t[i] if t is not None and k != "noise" else t) for k, t in self.buf.items()}
            info0, r = self.info0[i], b["reward"]
        else:
            b, info0, r = self.buf, self.info0, self.buf["reward"][0]
        c = b["counters"].cpu().numpy()
        info = dict(info0)
        info["step"] = int(c[0])
        if "contact_stage" in info:
            info["contact_stage"] = int(c[1])
        info["rng"] = b["rng"].cpu().numpy().view(np.uint32).copy()
        ps = PipelineState(b["qpos"].clone(), b["qvel"].clone(), b["qacc_warmstart"].clone(), b["ctrl"].clone())
        return State(ps, None, r.clone(), 0.0, {}, info)


def save_run(output_dir, rollout, infos, timestamp=None):
    """End-of-run dumps of the reference (dial_core.py:305-323): ``*_states.npy`` rows
    ``[i, qpos, qvel, ctrl]`` and ``*_predictions.npy`` = per control step the ``xbar`` of the LAST
    diffusion iteration, shape [n_steps, Hsample+1, nbody-1, 3] (``infos[i]["xbar"][-1]`` there:
    ``lax.scan`` stacks the iterations, ``[-1]`` picks the last one, not the last horizon step)."""
    os.makedirs(output_dir, exist_ok=True)
    timestamp = timestamp or time.strftime("%Y%m%d-%H%M%S")
    states = torch.stack([torch.as_tensor(r) for r in rollout]).cpu().numpy()
    preds = torch.stack([torch.as_tensor(x) for x in infos]).cpu().numpy()
    assert preds.ndim == 4 and preds.shape[-1] == 3, preds.shape
    np.save(os.path.join(output_dir, f"{timestamp}_states"), states)
    np.save(os.path.join(output_dir, f"{timestamp}_predictions"), preds)
    return states, preds


def _model(env_or_sys):
    """The ``CompiledModel`` of an env, a ``System`` or a ``CompiledModel``."""
    m = getattr(env_or_sys, "sys", env_or_sys)
    return getattr(m, "model", m)


def _mapping(spec, keys, not_mapping: str, takes: str, at: str = "") -> dict:
    """``spec`` if it is a mapping of some of ``keys``; else ValueError '<at><not_mapping><spec>' or '<at>unknown key
    'k' (<takes>)'."""
    if not isinstance(spec, dict):
        raise ValueError(f"{at}{not_mapping}{spec!r}")
    extra = sorted(set(spec) - set(keys), key=str)
    if extra:
        raise ValueError(f"{at}unknown key {extra[0]!r} ({takes})")
    return spec


def _num(v) -> bool:
    """A finite real number: a Python or NumPy int or float, not a bool."""
    return not isinstance(v, bool) and isinstance(v, (int, float, np.integer, np.floating)) and math.isfinite(v)


def _int(v, lo: int, hi: int, error: str) -> int:
    """A Python or NumPy int (not a bool) in lo..hi; else ValueError '<error>, got <v>'."""
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not lo <= v <= hi:
        raise ValueError(f"{error}, got {v!r}")
    return int(v)


RISK_AGGREGATES = ("mean", "worst", "cvar")


def risk_setting(spec, K: int):
    """A risk spec -> (mode, alpha) of ``dial_plan_set_ensemble_risk`` for K members.  ``{"aggregate":
    "mean"}``: the member mean (the default); ``{"aggregate": "worst"}``: the minimum, CVaR with alpha = 1/K;
    ``{"aggregate": "cvar", "alpha": a}``: the mean of the worst fraction a in (0, 1] of the members.
    Raises ValueError naming the bad key or value."""
    _mapping(spec, ("aggregate", "alpha"), f"a risk spec maps 'aggregate' ({', '.join(RISK_AGGREGATES)}) and, for "
             "cvar, 'alpha'; got ", "a risk spec takes 'aggregate' and, for cvar, 'alpha'")
    agg = spec.get("aggregate")
    if agg not in RISK_AGGREGATES:
        raise ValueError(f"aggregate must be one of {', '.join(RISK_AGGREGATES)}, got {agg!r}")
    mean, cvar = _capi.DEFINES["DIAL_ENS_MEAN"], _capi.DEFINES["DIAL_ENS_CVAR"]
    if agg != "cvar":
        if "alpha" in spec:
            raise ValueError(f"alpha applies to aggregate cvar only, not {agg}")
        return (mean, 1.0) if agg == "mean" else (cvar, 1.0 / max(int(K), 1))
    if "alpha" not in spec:
        raise ValueError("aggregate cvar needs alpha, the fraction of the members it averages, in (0, 1]")
    a = spec["alpha"]
    if not (_num(a) and 0 < a <= 1 and np.float32(a) > 0):
        raise ValueError(f"alpha must be a finite number in (0, 1], got {a!r}")
    return cvar, float(a)


def adapt_setting(spec, K: int, nv: int):
    """An adapt spec -> (forget, prune, sigma [nv] fp32) of ``dial_plan_set_ensemble_adapt`` for K members
    and nv dofs.  ``sigma`` (required): the scale of each qvel residual, one number for every dof or nv
    numbers, each finite and > 0; ``forget`` (default 1.0): in (0, 1], how much of the old log-belief each
    env step keeps; ``prune`` (default 0.0): in [0, 1/K), members with a smaller weight are left out of
    the score.  Raises ValueError naming the bad key or value."""
    _mapping(spec, ("sigma", "forget", "prune"), "an adapt spec maps 'sigma' and optionally 'forget' and 'prune'; got ",
             "an adapt spec takes 'sigma', 'forget' and 'prune'")
    if "sigma" not in spec:
        raise ValueError("adapt needs sigma, the scale of the qvel residuals: one number or one per dof")
    s = spec["sigma"]
    if isinstance(s, (list, tuple)):
        if len(s) != nv:
            raise ValueError(f"sigma must be one number or a list of {nv} (one per dof), got a list of {len(s)}")
        bad = [x for x in s if not (_num(x) and np.float32(x) > 0)]
        if bad:
            raise ValueError(f"sigma must be finite and > 0, got {bad[0]!r}")
        sigma = np.asarray(s, np.float32)
    elif _num(s) and np.float32(s) > 0:
        sigma = np.full(nv, s, np.float32)
    else:
        raise ValueError(f"sigma must be a finite number > 0 or a list of {nv}, got {s!r}")
    forget = spec.get("forget", 1.0)
    if not (_num(forget) and 0 < np.float32(forget) <= 1):
        raise ValueError(f"forget must be a finite number in (0, 1], got {forget!r}")
    prune = spec.get("prune", 0.0)
    if not (_num(prune) and 0 <= np.float32(prune) and float(np.float32(prune)) < 1.0 / K):
        raise ValueError(f"prune must be a number in [0, 1/K) = [0, {1.0 / K:g}), got {prune!r}")
    return float(forget), float(prune), sigma


def prior_setting(w, K: int):
    """A belief given as K weights, each finite and >= 0 with a positive sum -> fp32 [K].  Raises ValueError
    naming the bad value."""
    if isinstance(w, torch.Tensor):
        w = w.detach().cpu().tolist()
    w = list(w) if isinstance(w, (list, tuple, np.ndarray)) else w
    if not isinstance(w, list) or len(w) != K:
        raise ValueError(f"a belief is a list of {K} weights (one per member), got {w!r}")
    for x in w:
        if not (_num(x) and np.float32(x) >= 0):
            raise ValueError(f"every weight must be finite and >= 0, got {x!r}")
    a = np.asarray(w, np.float32)
    if not a.astype(np.float64).sum() > 0:
        raise ValueError("the weights must have a positive sum")
    return a


SCHEDULE_FIELDS = ("temp_sample", "sigma_scale", "horizon_diffuse_factor", "traj_diffuse_factor", "Ndiffuse",
                   "Ndiffuse_init")


def schedule_setting(spec, args: DialConfig) -> DialConfig:
    """A schedule spec -> ``args`` with the spec's sampling fields replaced: a mapping of any of
    ``SCHEDULE_FIELDS``; missing keys keep ``args``'s values.  ``temp_sample``, ``horizon_diffuse_factor`` and
    ``traj_diffuse_factor`` are finite numbers > 0, ``sigma_scale`` a finite number >= 0, ``Ndiffuse`` and
    ``Ndiffuse_init`` ints in 1..64.  Raises ValueError naming the bad key or value; the other DialConfig
    fields (Nsample, Hsample, Hnode, update_method, ...) are shared by every instance of a plan."""
    if not isinstance(spec, dict):
        raise ValueError(f"a schedule spec maps any of {', '.join(SCHEDULE_FIELDS)}; got {spec!r}")
    shared = {f.name for f in dataclasses.fields(DialConfig)} - set(SCHEDULE_FIELDS)
    for key in spec:
        if key in shared:
            raise ValueError(f"{key} is shared by every instance of the plan; a schedule sets only "
                             f"{', '.join(SCHEDULE_FIELDS)}")
        if key not in SCHEDULE_FIELDS:
            raise ValueError(f"unknown key {key!r} (a schedule takes {', '.join(SCHEDULE_FIELDS)})")
    out = {}
    for key, v in spec.items():
        if key.startswith("Ndiffuse"):
            v = _int(v, 1, _capi.DEFINES["DIAL_MAXDIFFUSE"], f"{key} must be an int in 1..{_capi.DEFINES['DIAL_MAXDIFFUSE']}")
        elif not (_num(v) and (v >= 0 if key == "sigma_scale" else (v > 0 and np.float32(v) > 0))):
            raise ValueError(f"{key} must be a finite number {'>= 0' if key == 'sigma_scale' else '> 0'}, got {v!r}")
        out[key] = v
    return dataclasses.replace(args, **out)


def delay_setting(spec):
    """A delay spec -> (steps, predict) of ``dial_plan_set_instance_delay``: an int ``d`` (the action planned at
    step t reaches the plant at step t + d, planned from the plant state) or ``{"steps": d, "predict": p}``
    (``predict``, default False: plan from the state predicted through the d queued actions), d in 0..16.
    Raises ValueError naming the bad key or value."""
    steps = lambda v: _int(v, 0, _capi.DEFINES["DIAL_MAXDELAY"], f"steps must be an int in 0..{_capi.DEFINES['DIAL_MAXDELAY']}")
    if isinstance(spec, dict):
        _mapping(spec, ("steps", "predict"), "", "a delay spec takes 'steps' and 'predict'")
        if "steps" not in spec:
            raise ValueError("a delay spec mapping needs steps, the delay in control steps")
        p = spec.get("predict", False)
        if not isinstance(p, (bool, np.bool_)):
            raise ValueError(f"predict must be true or false, got {p!r}")
        return steps(spec["steps"]), bool(p)
    if isinstance(spec, bool) or not isinstance(spec, (int, np.integer)):
        raise ValueError(f"a delay spec is an int (control steps) or a mapping of 'steps' and 'predict', got {spec!r}")
    return steps(spec), False


def delay_spec(text: str) -> dict:
    """The delay spec of a ``STEPS[:predict]`` command-line value.  Raises ValueError for any other text; the
    steps themselves are checked by ``delay_setting``."""
    steps, sep, mode = text.partition(":")
    if sep and mode != "predict":
        raise ValueError(f"the suffix must be ':predict', got {text!r}")
    if not steps.strip().lstrip("-").isdigit():
        raise ValueError(f"STEPS must be an int, got {steps!r}")
    return {"steps": int(steps), "predict": bool(sep)}


OBSERVE_KEYS = ("delay", "qpos", "qvel", "seed")


def observe_setting(spec, sys):
    """An observe spec -> (delay, qpos_std [nv], qvel_std [nv], key) of ``dial_plan_set_instance_observation``
    for the model of ``sys`` (a ``System``, an env or a ``CompiledModel``).  The spec maps any of ``delay`` (the
    observation delay in control steps, 0..16, default 0), ``qpos`` and ``qvel`` (noise standard deviations,
    default 0: one number for every dof, a list of nv, or ``{joint_name: value}`` resolved as
    ``System.tree_replace`` resolves a dof field by joint name; a free joint takes one number or 6, 3 position
    and 3 rotation) and ``seed`` (the noise key is ``PRNGKey(seed)``, default 0: instances with other
    standard deviations see the same draws, scaled).  Raises ValueError naming the bad key or value."""
    model = _model(sys)
    nv = model.nv
    dmax = _capi.DEFINES["DIAL_MAXDELAY"]
    _mapping(spec, OBSERVE_KEYS, f"an observe spec is a mapping of {', '.join(OBSERVE_KEYS)}, got ",
             f"an observe spec takes {', '.join(map(repr, OBSERVE_KEYS))}")

    def std(name, v):
        if not (_num(v) and v >= 0):
            raise ValueError(f"{name} must be a finite number >= 0, got {v!r}")
        return float(v)

    def stds(name, S):
        out = np.zeros(nv, np.float32)
        if isinstance(S, dict):
            for joint, v in S.items():
                try:
                    rows = model._entries("joint", joint, name)
                except KeyError:
                    raise ValueError(f"{name}: unknown joint {joint!r} (known: {model.names.get('joint', [])})") from None
                n = len(range(nv)[rows]) if isinstance(rows, slice) else 1
                vals = v if isinstance(v, (list, tuple, np.ndarray)) else [v] * n
                if len(vals) != n:
                    raise ValueError(f"{name}: joint {joint!r} has {n} dofs: give one number or {n}, got {list(vals)!r}")
                out[rows] = [std(f"{name}: {joint}", x) for x in vals]
            return out
        if isinstance(S, (list, tuple, np.ndarray)):
            if len(S) != nv:
                raise ValueError(f"{name} must be one number, a list of nv = {nv} or a mapping of joint names, "
                                 f"got a list of {len(S)}")
            out[:] = [std(f"{name}[{i}]", x) for i, x in enumerate(S)]
            return out
        out[:] = std(name, S)
        return out

    delay = _int(spec.get("delay", 0), 0, dmax, f"delay must be an int in 0..{dmax}")
    q, v = stds("qpos", spec.get("qpos", 0.0)), stds("qvel", spec.get("qvel", 0.0))
    key = drandom.PRNGKey(_int(spec.get("seed", 0), 0, 0xFFFFFFFF, f"seed must be an int in 0..{0xFFFFFFFF}"))
    return delay, q, v, np.asarray(key, np.uint32)


PUSH_KEYS = ("step", "steps", "body", "pos", "force", "torque")


def push_setting(spec, sys) -> list:
    """A push spec -> the push table of ``dial_plan_set_instance_pushes`` (a list of ``_capi.dial_push``) for the
    model of ``sys`` (a ``System``, an env or a ``CompiledModel``).  The spec is a list of at most 16 mappings of
    ``step`` (the first post-step counter ``info["step"]`` the push fires at, >= 1), ``steps`` (the env steps it
    fires in, >= 1, default 1), ``body`` (a body name other than the world), ``pos`` (the point of application
    in the body's frame, default its origin), ``force`` [N] and ``torque`` [N m] (world frame, default zero).
    After each env step it fires in, the plant's qvel takes the impulse of the force and torque held over that
    step.  An empty list (or None) is no pushes.  Raises ValueError naming the entry and the bad key or value."""
    model = _model(sys)
    pmax = _capi.DEFINES["DIAL_MAXPUSH"]
    if spec is None:
        return []
    if not isinstance(spec, (list, tuple)):
        raise ValueError(f"a push spec is a list of mappings of {', '.join(PUSH_KEYS)}, got {spec!r}")
    if len(spec) > pmax:
        raise ValueError(f"a push spec has at most {pmax} entries, got {len(spec)}")
    bodies = model.names.get("body", [])
    fmax = float(np.finfo(np.float32).max)
    out = []
    for i, e in enumerate(spec):
        at = f"push {i}: "
        _mapping(e, PUSH_KEYS, f"an entry is a mapping of {', '.join(PUSH_KEYS)}, got ",
                 f"an entry takes {', '.join(map(repr, PUSH_KEYS))}", at)
        if "step" not in e:
            raise ValueError(f"{at}needs step, the post-step counter it fires at")
        if "body" not in e:
            raise ValueError(f"{at}needs body, the name of the body pushed")
        body = e["body"]
        if not isinstance(body, str) or body not in bodies[1:]:
            raise ValueError(f"{at}unknown body {body!r} (known: {bodies[1:]})")
        p = _capi.dial_push()
        p.step, p.n_steps = (_int(e.get(k, 1), 1, 0x7FFFFFFF, f"{at}{k} must be an int >= 1") for k in ("step", "steps"))
        p.body = bodies.index(body)
        for name in ("pos", "force", "torque"):
            v = e.get(name, [0.0, 0.0, 0.0])
            if not (isinstance(v, (list, tuple, np.ndarray)) and len(v) == 3 and
                    all(_num(x) and abs(float(x)) <= fmax for x in v)):
                raise ValueError(f"{at}{name} must be a list of 3 finite numbers, got {v!r}")
            getattr(p, name)[:] = [float(x) for x in v]
        out.append(p)
    return out


PLANT_KEYS = ("substeps", "sim_dt", "iterations", "ls_iterations", "tolerance")


def plant_setting(spec, sys):
    """A plant spec -> the ``_capi.dial_plant`` of ``dial_plan_set_instance_plant`` for the model of ``sys`` (a
    ``System``, an env or a ``CompiledModel``: the planner's model), or None for a None spec (no setting).  The
    spec maps any of ``substeps`` (physics substeps per planner physics step, 1..16, default 1) or ``sim_dt``
    (the plant's physics step in seconds; timestep / sim_dt must be an integer, the substeps, so that the env
    step's dt / sim_dt is an integer too), ``iterations`` (Newton iterations, 1..100), ``ls_iterations`` (line
    search iterations, 1..50) and ``tolerance`` (finite, >= 0).  The solver settings default to the model's own;
    MuJoCo's defaults are 100, 50 and 1e-8.  An empty mapping is the identity setting: the plant steps like the
    planner.  Raises ValueError naming the bad key or value."""
    model = _model(sys)
    if spec is None:
        return None
    _mapping(spec, PLANT_KEYS, f"a plant spec is a mapping of {', '.join(PLANT_KEYS)}, got ",
             f"a plant spec takes {', '.join(map(repr, PLANT_KEYS))}")
    if "substeps" in spec and "sim_dt" in spec:
        raise ValueError("a plant spec takes substeps or sim_dt, not both")
    kmax = _capi.DEFINES["DIAL_MAXSUBSTEPS"]
    ts = float(model.timestep)
    if "sim_dt" in spec:
        s = spec["sim_dt"]
        if not (_num(s) and s > 0):
            raise ValueError(f"sim_dt must be a finite number > 0, got {s!r}")
        k = round(ts / float(s))
        if k < 1 or abs(ts / float(s) - k) > 1e-6 * k:
            raise ValueError(f"sim_dt {s!r} must divide the model's timestep {ts:g} into an integer number of substeps")
        if k > kmax:
            raise ValueError(f"sim_dt {s!r} gives {k} substeps of the model's timestep {ts:g}, at most {kmax}")
    else:
        k = _int(spec.get("substeps", 1), 1, kmax, f"substeps must be an int in 1..{kmax}")
    f = _capi.dial_plant()
    f.substeps = k
    f.iterations = _int(spec.get("iterations", int(model.iterations)), 1, 100, "iterations must be an int in 1..100")
    f.ls_iterations = _int(spec.get("ls_iterations", int(model.ls_iterations)), 1, 50,
                           "ls_iterations must be an int in 1..50")
    tol = spec.get("tolerance", float(model.tolerance))
    if not (_num(tol) and tol >= 0 and abs(float(tol)) <= float(np.finfo(np.float32).max)):
        raise ValueError(f"tolerance must be a finite number >= 0, got {tol!r}")
    f.tolerance = float(tol)
    return f


def _set_terrain(loop, b, setting):
    """Instance b's plant and planner terrains from a ``TerrainSetting`` (None: flat on both sides)."""
    plant, planner = terrains(setting)
    loop.plan.set_instance_terrain(b, TERRAIN_PLANT, plant)
    loop.plan.set_instance_terrain(b, TERRAIN_PLANNER, planner)


def _each(parse):
    """A per-spec parser as a parser of the B specs of a setting; a None spec stays None."""
    return lambda specs, c: [None if spec is None else parse(spec, c) for spec in specs]


def _plant_model(env, c):
    """An instance's env, checked against the planner's: its ``sys`` when its model differs, else None."""
    DeviceLoop._check_shared(c.env, env)
    return env.sys if bytes(_capi.fill_model_desc(env.sys.model)) != c.base else None


def _members(rows, c):
    """Every instance's K members: each a ``System`` or ``CompiledModel``, None where it is the planner's model."""
    if any(len(r) != c.K for r in rows):
        raise ValueError(f"ensemble must be a list of {c.K} models or {c.B} such lists, got {[len(r) for r in rows]}")
    return [[None if bytes(_capi.fill_model_desc(_model(m))) == c.base else m for m in r] for r in rows]


def _observation(spec, c):
    o = observe_setting(spec, c.env)
    if c.rand and o[0] > 0:
        raise ValueError(DeviceLoop._RAND_OBSERVE)
    return o


def _lists(v):
    return isinstance(v, (list, tuple))


_Setting = collections.namedtuple("_Setting", "key flag shape per parse identity apply ens unsharded seq",
                                  defaults=(0, False, False))

# DeviceLoop's per-instance settings in their order of application (a plant slot copies its instance's model the
# first time it is set, the planning models copy member (b, 0)).  key: the DeviceLoop keyword; flag: the
# command-line flag and --instance-overrides key; shape: the error for a list of other than B specs; per(value):
# the value is B specs (else one spec for every instance; seq: list(value) first); parse(specs, c): the B
# settings, checked; identity(setting): a setting that changes nothing, not applied at bind, so that a loop
# without it keeps the plan's launches; apply(loop, b, spec, setting); ens: needs an ensemble of at least that
# many members; unsharded: needs world_size 1.
SETTINGS = (
    _Setting("envs", None, "a plan of {B} instances needs {B} envs, got {n}", lambda v: True,
             lambda envs, c: [_plant_model(e, c) for e in envs], lambda s: s is None,
             lambda loop, b, spec, s: loop.set_model(b, spec), seq=True),
    _Setting("ensemble", None, "ensemble must be a list of {K} models or {B} such lists, got a list of {n}",
             lambda e: len(e) > 0 and all(_lists(r) for r in e), _members, lambda s: not any(m is not None for m in s),
             lambda loop, b, spec, s: [loop.set_ensemble_model(b, k, m) for k, m in enumerate(s) if m is not None],
             ens=1, seq=True),
    _Setting("risk", None, "risk must be one risk spec or a list of {B}, got a list of {n}", _lists,
             lambda specs, c: [risk_setting(spec, c.K) for spec in specs], lambda s: False,
             lambda loop, b, spec, s: loop.set_risk(b, spec), ens=1),
    _Setting("prior", None, "prior must be K weights or a list of {B} such lists, got a list of {n}",
             lambda p: len(p) > 0 and all(isinstance(r, (list, tuple, np.ndarray)) for r in p),
             lambda specs, c: [prior_setting(w, c.K) for w in specs], lambda s: False,
             lambda loop, b, spec, s: loop.set_belief(b, s), ens=2, seq=True),
    _Setting("adapt", None, "adapt must be one adapt spec or a list of {B}, got a list of {n}", _lists,
             _each(lambda spec, c: adapt_setting(spec, c.K, c.nv)), lambda s: s is None,
             lambda loop, b, spec, s: loop.set_adapt(b, spec), ens=2),
    _Setting("schedule", None, "schedule must be one schedule spec or a list of {B}, got a list of {n}", _lists,
             _each(lambda spec, c: schedule_setting(spec, c.cfg)), lambda s: s is None,
             lambda loop, b, spec, s: loop.set_schedule(b, spec)),
    _Setting("delay", "delay", "delay must be one delay spec or a list of {B}, got a list of {n}", _lists,
             lambda specs, c: [(0, False) if spec is None else delay_setting(spec) for spec in specs],
             lambda s: s == (0, False), lambda loop, b, spec, s: loop.set_delay(b, spec), unsharded=True),
    _Setting("observe", "observe", "observe must be one observe spec or a list of {B}, got a list of {n}", _lists,
             _each(_observation), lambda s: s is None or not DeviceLoop._observing(s),
             lambda loop, b, spec, s: loop._set_observation(b, s), unsharded=True),
    # a list of B lists (or Nones) is per instance; a list of mappings is one spec for every instance
    _Setting("pushes", "push", "pushes must be one push spec or a list of {B}, got a list of {n}",
             lambda v: _lists(v) and len(v) > 0 and all(x is None or _lists(x) for x in v),
             lambda specs, c: [push_setting(spec, c.env) for spec in specs], lambda s: not s,
             lambda loop, b, spec, s: loop.plan.set_instance_pushes(b, s), unsharded=True),
    _Setting("plant", "plant", "plant must be one plant spec or a list of {B}, got a list of {n}", _lists,
             lambda specs, c: [plant_setting(spec, c.env) for spec in specs], lambda s: s is None,
             lambda loop, b, spec, s: loop.plan.set_instance_plant(b, s), unsharded=True),
    _Setting("terrain", "terrain", "terrain must be one terrain spec or a list of {B}, got a list of {n}", _lists,
             _each(lambda spec, c: terrain_setting(spec, c.env.sys)), lambda s: s is None,
             lambda loop, b, spec, s: _set_terrain(loop, b, s), unsharded=True),
)


def _context(B: int, K: int, env, cfg: DialConfig, rand: bool):
    """What the parsers of ``SETTINGS`` check a spec against."""
    return types.SimpleNamespace(B=B, K=K, env=env, nv=env.sys.nv, cfg=cfg, rand=rand,
                                 base=bytes(_capi.fill_model_desc(_model(env))))


def resolve_settings(B: int, K: int, env, cfg: DialConfig, world_size: int = 1, rand: bool = False, **given) -> dict:
    """DeviceLoop's per-instance keywords (``SETTINGS``: envs, ensemble, risk, prior, adapt, schedule, delay,
    observe, pushes, plant, terrain; None or missing: not set) for a plan of B instances and K ensemble members on ``env``'s
    model and ``cfg``, sharded over ``world_size`` GPUs, with per-instance random tasks (``rand``) or not ->
    ``{key: [(spec, setting)] * B}`` for every keyword given, each spec checked and parsed.  A keyword is one spec
    for every instance or a list of B specs.  Raises ValueError naming the keyword, the spec or the value."""
    c = _context(B, K, env, cfg, rand)
    out = {}
    for s in SETTINGS:
        value = given.pop(s.key, None)
        if value is None:
            continue
        if K < s.ens:
            raise ValueError(f"{s.key}= needs an MBDPI built with n_ensemble >= {s.ens}")
        if s.unsharded and world_size != 1:
            raise ValueError(f"{s.key}= needs an unsharded plan (world_size 1)")
        value = list(value) if s.seq else value
        specs = list(value) if s.per(value) else [value] * B
        if len(specs) != B:
            raise ValueError(s.shape.format(B=B, K=K, n=len(specs)))
        out[s.key] = list(zip(specs, s.parse(specs, c)))
    if given:
        raise TypeError(f"unknown per-instance setting {sorted(given)[0]!r}")
    return out


def load_setting(spec, key: str, K: int, nv: Optional[int] = None):
    """The ``risk``, ``adapt`` or ``prior`` entry ``key`` of an ``--ensemble`` file or an
    ``--instance-overrides`` mapping, checked for K members and nv dofs (``risk_setting``,
    ``adapt_setting``, ``prior_setting``), or None when ``spec`` has no such entry.  Raises ValueError
    starting with '<key>: '."""
    if not isinstance(spec, dict) or spec.get(key) is None:
        return None
    try:
        if key == "risk":
            risk_setting(spec[key], K)
        elif K < 2:
            raise ValueError(f"needs an ensemble of at least 2 members, got {K}")
        elif key == "adapt":
            adapt_setting(spec[key], K, nv)
        else:
            prior_setting(spec[key], K)
    except ValueError as e:
        raise ValueError(f"{key}: {e}") from None
    return spec[key]


def load_ensemble(spec, env):
    """The ``--ensemble`` file's mapping -> (K member ``System``s, the plant's ``sys`` mapping or None).
    ``members``: a list of K ``System.tree_replace`` mappings of ``env``'s model (``{}``: the nominal
    model); ``plant`` (optional): one such mapping for every instance's plant; ``risk`` (optional): the
    risk spec of every instance; ``adapt`` / ``prior`` (optional): adaptation to the plant; the last three
    are read by ``load_setting``.  Raises ValueError naming the entry that is malformed."""
    if not isinstance(spec, dict) or set(spec) - {"members", "plant", "risk", "adapt", "prior"} or "members" not in spec:
        raise ValueError("must map 'members' (a list of sys mappings) and optionally 'plant' (one sys mapping), "
                         "'risk' (a risk spec), 'adapt' (an adapt spec) and 'prior' (K weights), got "
                         f"{sorted(spec) if isinstance(spec, dict) else spec!r}")
    members, plant = spec["members"], spec.get("plant")
    kmax = _capi.DEFINES["DIAL_MAXENS"]
    if not isinstance(members, list) or not 1 <= len(members) <= kmax:
        raise ValueError(f"members must be a list of 1..{kmax} sys mappings, got "
                         f"{len(members) if isinstance(members, list) else type(members).__name__}")
    out = []
    for k, ov in enumerate(members):
        ov = {} if ov is None else ov
        if not isinstance(ov, dict):
            raise ValueError(f"members[{k}] must map model fields, got {ov!r}")
        try:
            out.append(env.sys.tree_replace(ov))
        except (KeyError, ValueError) as e:
            raise ValueError(f"members[{k}]: {e}") from None
    if plant is not None:
        if not isinstance(plant, dict):
            raise ValueError(f"plant must map model fields, got {plant!r}")
        try:
            env.sys.tree_replace(plant)
        except (KeyError, ValueError) as e:
            raise ValueError(f"plant: {e}") from None
    return out, plant


def run_instances(dial_config, env, B, Nstep, **settings):
    """``B`` closed loops of ``main`` advanced by one CUDA graph per control step; instance b is the
    plain run with seed ``dial_config.seed + b`` (on ``envs[b]``, its own task and plant, when given).  With
    ``randomize_tasks`` each instance draws its own commands or jump sequence from its reset key.
    ``settings``: DeviceLoop's per-instance keywords (``envs``, ``ensemble``, ``risk``, ``prior``, ``adapt``,
    ``schedule``, ``delay``, ``observe``, ``pushes``, ``plant``); with ``ensemble``, K planning models shared by
    every instance; each instance runs its own Ndiffuse_init, then Ndiffuse."""
    envs = settings.get("envs")
    mbdpi = MBDPI(dial_config, env, n_instances=B, n_ensemble=len(settings.get("ensemble") or ()))
    states, rngs = [], []
    for b in range(B):
        rng, rng_reset = drandom.split(drandom.PRNGKey(seed=dial_config.seed + b))
        states.append((envs[b] if envs is not None else env).reset(rng_reset))
        rngs.append(drandom.split(rng)[1])
    loop = DeviceLoop(mbdpi, states, np.stack(rngs), **settings)
    buf = loop.buf
    rews, rollout, infos = [], [], []
    t0, tlast = time.time(), -1
    for t in range(Nstep):
        loop.step(initial=(t == 0))
        tt = torch.full((B, 1), float(t), device=mbdpi.device)
        rollout.append(torch.cat([tt, buf["qpos"], buf["qvel"], buf["ctrl"]], 1))
        rews.append(buf["reward"].clone())
        infos.append(buf["xbar"].clone())
        if t % 10 == 0:
            r = rews[-1].cpu().numpy()   # synchronises
            print(f"step {t}: rew={r.mean():.3e} (min {r.min():.3e}, max {r.max():.3e} over {B} instances) "
                  f"freq={(t - tlast) / (time.time() - t0):.1f} Hz")
            t0, tlast = time.time(), t
    rew = torch.stack(rews).mean(0).cpu().numpy()
    print("mean reward per instance = " + " ".join(f"{r:.2e}" for r in rew))
    _print_belief(loop)
    timestamp = time.strftime("%Y%m%d-%H%M%S")
    for b in range(B):
        save_run(dial_config.output_dir, [r[b] for r in rollout], [x[b] for x in infos], timestamp=f"{timestamp}_inst{b}")


def _spec_from_text(flag: str, text: str):
    """The spec of a per-instance setting's command-line value: ``STEPS[:predict]`` for --delay, YAML otherwise."""
    if flag == "delay":
        return delay_spec(text)
    try:
        return yaml.safe_load(text)
    except yaml.YAMLError as e:
        raise ValueError(f"not a YAML {'list' if flag == 'push' else 'mapping'}: {e}") from None


def _print_belief(loop) -> None:
    """The final belief over the members of each instance of an ensemble loop (K >= 2)."""
    if loop.mbdpi.n_ensemble < 2:
        return
    w = loop.belief().cpu().numpy().reshape(loop.n_instances, -1)
    for b, row in enumerate(w):
        print(f"belief instance {b} = " + " ".join(f"{x:.3f}" for x in row))


def main():
    """Synchronous MPC loop — dial_core.py:175-268 without the rendering / flask tail."""
    parser = argparse.ArgumentParser()
    g = parser.add_mutually_exclusive_group(required=True)
    g.add_argument("--config", type=str, default=None)
    g.add_argument("--example", type=str, default=None)
    g.add_argument("--list-examples", action="store_true")
    parser.add_argument("--custom-env", type=str, default=None, help="Custom environment to import dynamically")
    parser.add_argument("--n-steps", type=int, default=None)
    parser.add_argument("--eager", action="store_true",
                        help="per-call launches (env.step / reverse_scan) instead of the CUDA-graph loop")
    parser.add_argument("--instances", type=int, default=1,
                        help="run this many independent closed loops in one CUDA graph per control step; instance b "
                             "resets from PRNGKey(seed + b) and writes its output files under the prefix <time>_inst<b>")
    parser.add_argument("--instance-overrides", type=str, default=None, metavar="FILE.yaml",
                        help="a YAML list of one mapping of env-config fields per instance (--instances of them): "
                             "instance b runs the config updated by mapping b (its own commands, gait, targets, ...); "
                             "a mapping may also set the instance's sampling schedule: temp_sample, sigma_scale, "
                             "horizon_diffuse_factor, traj_diffuse_factor, Ndiffuse, Ndiffuse_init")
    parser.add_argument("--ensemble", type=str, default=None, metavar="FILE.yaml",
                        help="plan against an ensemble of models: a YAML mapping with 'members', a list of K sys "
                             "mappings ({} = the nominal model), optionally 'plant', one sys mapping applied to "
                             "every instance's simulated robot before its own --instance-overrides sys, and "
                             "optionally 'risk', how a sample's member rewards become its score: {aggregate: mean} "
                             "(default), {aggregate: worst} or {aggregate: cvar, alpha: A}; an --instance-overrides "
                             "mapping may carry its own 'risk'; optionally 'adapt', {sigma: S, forget: F, prune: P}: "
                             "weight the members by how well they predict each env step's qvel (S: one scale or one "
                             "per dof), from 'prior', K weights (default uniform); an --instance-overrides mapping "
                             "may carry its own 'adapt'")
    parser.add_argument("--delay", type=str, default=None, metavar="STEPS[:predict]",
                        help="control latency of every instance: the action planned at step t reaches the simulated "
                             "robot at step t + STEPS (0..16); ':predict' plans from the state predicted STEPS steps "
                             "ahead through the queued actions; an --instance-overrides mapping may carry its own "
                             "'delay' (an int or {steps: d, predict: true})")
    parser.add_argument("--observe", type=str, default=None, metavar="SPEC",
                        help="every instance plans from an observation of its simulated robot: a YAML flow mapping "
                             "such as '{delay: 2, qpos: 0.01, qvel: 0.1, seed: 0}', the record 'delay' control "
                             "steps old (0..16) with Gaussian noise of standard deviation 'qpos' / 'qvel' (one number, "
                             "nv numbers or a mapping of joint names); an --instance-overrides mapping may carry its "
                             "own 'observe'")
    parser.add_argument("--push", type=str, default=None, metavar="SPEC",
                        help="push every instance's simulated robot: a YAML flow list such as "
                             "'[{step: 50, body: base, force: [60, 0, 0], steps: 5}]'; after each env step whose "
                             "counter lies in [step, step + steps) the robot takes the impulse of 'force' [N] at 'pos' "
                             "(body frame, default the body's origin) and 'torque' [N m] (world frame) held over that "
                             "step; the planner is not told; an --instance-overrides mapping may carry its own 'push'")
    parser.add_argument("--plant", type=str, default=None, metavar="SPEC",
                        help="step every instance's simulated robot at its own physics fidelity: a YAML flow mapping "
                             "such as '{sim_dt: 0.005, iterations: 100, ls_iterations: 50, tolerance: 1e-8}' or "
                             "'{substeps: 4}'; each env step makes 'substeps' (or timestep / sim_dt) physics steps per "
                             "planner physics step with the control held, solved with the given settings (default: "
                             "the planner's); the planner keeps its model; an --instance-overrides mapping may carry "
                             "its own 'plant'")
    parser.add_argument("--terrain", type=str, default=None, metavar="SPEC",
                        help="give every instance's simulated robot its own ground: a YAML flow mapping such as "
                             "'{kind: rough, amplitude: 0.03, wavelength: 0.3, seed: 1}', '{kind: slope, angle: 10}' "
                             "or '{kind: grid, heights: ground.npy, spacing: 0.05}'; 'planner: true' lets the planner "
                             "plan on the same ground (default: it plans on the flat floor); an --instance-overrides "
                             "mapping may carry its own 'terrain'")
    args = parser.parse_args()
    from dial_mpc_b200.examples import examples
    if args.list_examples:
        print("Examples:")
        for example in examples:
            print(f"  {example}")
        return
    if args.custom_env is not None:
        sys.path.append(os.getcwd())
        importlib.import_module(args.custom_env)
    if args.example is not None:
        config_dict = yaml.safe_load(open(get_example_path(args.example + ".yaml")))
    else:
        config_dict = yaml.safe_load(open(args.config))
    dial_config = load_dataclass_from_dict(DialConfig, config_dict)
    if args.instances < 1:
        parser.error("--instances must be at least 1")
    if args.instances > 1 and args.eager:
        parser.error("--instances runs on the CUDA-graph loop; it excludes --eager")
    flagged = [s for s in SETTINGS if s.flag]
    given = {s.key: None for s in flagged}     # DeviceLoop keyword -> the spec of its flag
    for s in flagged:
        text = getattr(args, s.flag)
        if text is None:
            continue
        if args.eager:
            parser.error(f"--{s.flag} runs on the CUDA-graph loop; it excludes --eager")
        try:
            given[s.key] = _spec_from_text(s.flag, text)
        except ValueError as e:
            parser.error(f"--{s.flag}: {e}")
    rng = drandom.PRNGKey(seed=dial_config.seed)
    env_config_type = dial_envs.get_config(dial_config.env_name)
    env_config = load_dataclass_from_dict(env_config_type, config_dict, convert_list_to_array=True)
    env = dial_envs.get_environment(dial_config.env_name, config=env_config)
    # a flag or an override key holds one spec: it is checked by the setting's parser, not split into B
    ctx = _context(args.instances, 0, env, dial_config, bool(getattr(env_config, "randomize_tasks", False)))
    for s in flagged:
        if given[s.key] is not None:
            try:
                s.parse([given[s.key]], ctx)
            except ValueError as e:
                parser.error(f"--{s.flag}: {e}")
    envs = None
    members, plant, risk, adapt, prior = None, None, None, None, None
    if args.ensemble is not None:
        if args.eager:
            parser.error("--ensemble runs on the CUDA-graph loop; it excludes --eager")
        try:
            ens_spec = yaml.safe_load(open(args.ensemble))
            members, plant = load_ensemble(ens_spec, env)
            risk, adapt, prior = (load_setting(ens_spec, key, len(members), env.sys.nv)
                                  for key in ("risk", "adapt", "prior"))
        except (ValueError, yaml.YAMLError) as e:
            parser.error(f"--ensemble {args.ensemble}: {e}")
    if args.instance_overrides is not None:
        if args.instances < 2:
            parser.error("--instance-overrides needs --instances B with B >= 2")
        overrides = yaml.safe_load(open(args.instance_overrides))
        if not isinstance(overrides, list) or len(overrides) != args.instances:
            parser.error(f"--instance-overrides must hold a list of {args.instances} mappings (one per instance), "
                         f"got {len(overrides) if isinstance(overrides, list) else type(overrides).__name__}")
        env_fields = {f.name for f in dataclasses.fields(env_config_type)}
        # DialConfig fields: the sampling schedule (SCHEDULE_FIELDS), or fields shared by the plan, which
        # schedule_setting rejects by name
        dial_fields = {f.name for f in dataclasses.fields(DialConfig)} - env_fields
        known = env_fields | dial_fields | {"sys", "risk", "adapt", "delay", "observe", "push", "plant", "terrain"}
        envs = []
        settings = {"risk": [risk] * args.instances, "adapt": [adapt] * args.instances}
        uses = {"risk": "it scores the members' rewards", "adapt": "it weights the members"}
        schedule = [None] * args.instances
        per = {s.key: [given[s.key]] * args.instances for s in flagged}
        for b, ov in enumerate(overrides):
            ov = ov or {}
            if not isinstance(ov, dict) or set(ov) - known:
                parser.error(f"--instance-overrides entry {b} must map {env_config_type.__name__} fields, sys, risk, adapt, delay, observe, push, plant "
                             f"or the sampling fields {', '.join(SCHEDULE_FIELDS)}, got "
                             f"{sorted(set(ov) - known) if isinstance(ov, dict) else ov!r}")
            ov = dict(ov)
            spec = {k: ov.pop(k) for k in list(ov) if k in dial_fields}
            if spec:
                try:
                    schedule_setting(spec, dial_config)
                except ValueError as e:
                    parser.error(f"--instance-overrides entry {b}: {e}")
                schedule[b] = spec
            sys_ov = ov.pop("sys", None)
            for s in flagged:
                spec = ov.pop(s.flag, None)
                if spec is not None:
                    try:
                        s.parse([spec], ctx)
                    except ValueError as e:
                        parser.error(f"--instance-overrides entry {b}: {s.flag}: {e}")
                    per[s.key][b] = spec
            for key in ("risk", "adapt"):
                if ov.get(key) is not None:
                    if members is None:
                        parser.error(f"--instance-overrides entry {b}: {key} needs --ensemble ({uses[key]})")
                    try:
                        settings[key][b] = load_setting(ov, key, len(members), env.sys.nv)
                    except ValueError as e:
                        parser.error(f"--instance-overrides entry {b}: {e}")
                ov.pop(key, None)
            cfg_b = load_dataclass_from_dict(env_config_type, dict(config_dict, **ov), convert_list_to_array=True)
            envs.append(dial_envs.get_environment(dial_config.env_name, config=cfg_b))
            try:
                if plant is not None:
                    envs[-1].sys = envs[-1].sys.tree_replace(plant)
                if sys_ov is not None:
                    # sys: {field: value}: the instance's own physical model (System.tree_replace)
                    if not isinstance(sys_ov, dict):
                        raise ValueError(f"sys must map model fields, got {sys_ov!r}")
                    envs[-1].sys = envs[-1].sys.tree_replace(sys_ov)
                DeviceLoop._check_shared(env, envs[-1])
            except (ValueError, KeyError) as e:
                parser.error(f"--instance-overrides entry {b}: {e}")
    plant_env = env
    if plant is not None and envs is None:
        # one plant for every instance: the env the loop steps (and resets) with the plant's model
        plant_env = dial_envs.get_environment(dial_config.env_name, config=env_config)
        plant_env.sys = env.sys.tree_replace(plant)
        if args.instances > 1:
            envs = [plant_env] * args.instances
    if given["terrain"] is None:
        del given["terrain"]   # (passed only when some instance has a terrain)
    if args.instances > 1:
        if args.instance_overrides is not None and any(r is not None for r in settings["risk"]):
            risk = [r or {"aggregate": "mean"} for r in settings["risk"]]
        if args.instance_overrides is not None and any(a is not None for a in settings["adapt"]):
            adapt = settings["adapt"]
        for key, specs in (per.items() if args.instance_overrides is not None else ()):
            if any(spec is not None for spec in specs):
                given[key] = specs
        run_instances(dial_config, env, args.instances, args.n_steps or dial_config.n_steps, envs=envs,
                      ensemble=members, risk=risk, adapt=adapt, prior=prior,
                      schedule=schedule if args.instance_overrides is not None and any(schedule) else None, **given)
        return
    mbdpi = MBDPI(dial_config, env, n_ensemble=len(members) if members else 0)
    rng, rng_reset = drandom.split(rng)
    state = plant_env.reset(rng_reset)
    Y0 = torch.zeros(dial_config.Hnode + 1, mbdpi.nu, device=mbdpi.device)
    rng_exp, rng = drandom.split(rng)
    Nstep = args.n_steps or dial_config.n_steps
    rews, rollout, infos = [], [], []
    if not args.eager:
        # one CUDA graph per control step; the host launches it and logs
        loop = DeviceLoop(mbdpi, state, rng, Y0, envs=[plant_env] if members else None, ensemble=members, risk=risk,
                          adapt=adapt, prior=prior, **given)
        b = loop.buf
        t0, tlast = time.time(), -1
        for t in range(Nstep):
            loop.step(dial_config.Ndiffuse_init if t == 0 else dial_config.Ndiffuse)
            rollout.append(torch.cat([torch.tensor([float(t)], device=mbdpi.device), b["qpos"], b["qvel"], b["ctrl"]]))
            rews.append(b["reward"][0].clone())
            infos.append(b["xbar"].clone())   # = infos[i]["xbar"][-1] of the reference: last diffusion iteration, full horizon
            if t % 10 == 0:
                r = float(rews[-1])  # synchronises: the rate below is whole control steps per second
                print(f"step {t}: rew={r:.3e} freq={(t - tlast) / (time.time() - t0):.1f} Hz")
                t0, tlast = time.time(), t
    else:
        for t in range(Nstep):
            state = env.step(state, Y0[0])
            ps = state.pipeline_state
            rollout.append(torch.cat([torch.tensor([float(t)], device=mbdpi.device), ps.qpos, ps.qvel, ps.ctrl]))
            rews.append(state.reward)
            Y0 = mbdpi.shift(Y0)
            n_diffuse = dial_config.Ndiffuse_init if t == 0 else dial_config.Ndiffuse
            t0 = time.time()
            rng, Y0, info = mbdpi.reverse_scan(state, rng, Y0, mbdpi.schedule(n_diffuse))
            torch.cuda.synchronize()
            freq = 1 / (time.time() - t0)
            infos.append(info["xbar"])
            if t % 10 == 0:
                print(f"step {t}: rew={float(state.reward):.3e} freq={freq:.1f} Hz")
    rew = torch.stack([torch.as_tensor(r) for r in rews]).mean()
    print(f"mean reward = {float(rew):.2e}")
    if not args.eager:
        _print_belief(loop)
    save_run(dial_config.output_dir, rollout, infos)


if __name__ == "__main__":
    main()
