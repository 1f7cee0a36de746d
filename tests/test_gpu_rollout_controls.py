"""The controls the sampled rollouts of the control-step graph apply, read out of the kernel exactly and
compared with an fp64 restatement (tests/ctrl_probe.py: the probe envs, the reference and the derivation
of the tolerances; tests/test_rollout_controls.py runs the same checks in the CPU warp emulator).

The prologue of rollout_warp in sampled mode turns each row into the controls of its physics steps: the
row's sample (gidx = shard_offset + row % rows_per_model), the instance's key and this iteration's noise,
clip, node 0 pinned, the mean row unnoised, the spline row of the step, the action map.  The probe reward
makes each row's mean reward the control of one actuator at one step, so one launch reads one control of
every row; a batched plan whose instances probe different (step, actuator) pairs reads several.  Cases:
  a. the sampler element by element (Hs = Hn: the spline is the identity), every row of N = 2047;
  b. spline and horizon: Hn in {2, 3, 5, 7}, Hs in {Hn, 16, 25, 63} on the three solver variants;
  c. row layouts: N in {1, 31, 255, 2047} with unlike instances, DIAL_WPC = 1 and 16, the unfused update's
     key path; per-instance models; an ensemble (every member rolls the same samples); the rank-1 shard of
     a two-rank plan and injected eps;
  d. iterations of DeviceLoop.step(n): iteration i uses noise[i], instance b its own schedule's, eager,
     captured and replayed;
  e. the action map at its edges: clipped knots, targets beyond the physical range, saturated torques,
     action_scale 1.7;
  f. the update kernel's knots of a sample (one-hot weights) give the controls the rollout applied to it.
Torque-mode controls depend on the state: they are compared on single-instance plans, with q and qd read
from the GPU's own stored trajectories.  The batched layouts run position control.  The fixtures' nu is
even, so ntot is even here; the odd layout is test_gpu_update.py's (H1, nu = 19)."""
import functools

import numpy as np
import pytest
import torch

from tests import ctrl_probe as cp

pytestmark = pytest.mark.gpu

TEMP = 0.05
WORST = {}      # group -> worst |err| / tol, printed by each test


def _note(group, r):
    WORST[group] = max(WORST.get(group, 0.0), r)
    print(f"{group}: worst {WORST[group]:.3f} of the tolerance")


@functools.lru_cache(maxsize=None)
def _pair(name, scale=1.0):
    env, o = cp.make_probe(name, action_scale=scale)
    assert env.library_path      # one build per solver variant; the probed copies share it
    return env, o


def _mb(env, N, Hs, Hn, B=1, K=0, nd=4, **kw):
    from dial_mpc_b200.core.dial_config import DialConfig
    from dial_mpc_b200.core.dial_core import MBDPI
    cfg = DialConfig(env_name="ctrl_probe", Nsample=N, Hsample=Hs, Hnode=Hn, Ndiffuse=nd, Ndiffuse_init=nd,
                     temp_sample=TEMP)
    return MBDPI(cfg, env, n_instances=B, n_ensemble=K, **kw)


def _inputs(B, Hn, nu, seed, edges=False):
    """rng [B, 2], Ybar [B, Hn+1, nu].  ``edges``: every actuator has knots beyond +1 and below -1, some at +-1."""
    g = np.random.default_rng(seed)
    rngs = g.integers(0, 2 ** 32, size=(B, 2), dtype=np.uint64).astype(np.uint32)
    Y = g.standard_normal((B, Hn + 1, nu)) * 0.4
    if edges:
        Y = np.broadcast_to(1.3 * (-1.0) ** np.add.outer(np.arange(Hn + 1), np.arange(nu)), Y.shape).copy()
        Y[:, 1, 0], Y[:, 2, 1], Y[:, 3, 2] = 1.0, -1.0, 1.0
    return rngs, Y.astype(np.float32)


def _np(t):
    return t.detach().cpu().numpy().astype(np.float64)


def _restart(loop, Y, rng):
    loop.buf["Y"].copy_(torch.as_tensor(Y, device=loop.buf["Y"].device))
    loop.buf["rng"].copy_(torch.as_tensor(np.ascontiguousarray(rng, np.uint32).view(np.int32), device=loop.buf["rng"].device))


# ---- single-instance plans (torque mode: the state comes from the stored trajectories) ---------------------
def _single(name, N, Hs, Hn, pairs, seed=0, edges=False, scale=1.0, group=None):
    """Every row of a one-instance DeviceLoop, one probe (t, a) per step; returns {(t, a): ctrl [N+1]}."""
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import DeviceLoop
    env, o = _pair(name, scale)
    nu = env.action_size
    rngs, Ys = _inputs(1, Hn, nu, seed, edges)
    state = env.reset(drandom.PRNGKey(seed))
    mb = _mb(env, N, Hs, Hn)
    loop = DeviceLoop(mb, state, rngs[0], Ys[0], envs=[env])
    noise = _np(loop.buf["noise"][0])
    M = cp.spline64(Hs, Hn)
    Y, e = cp.knots64(cp.eps_xla(cp.sample_key(rngs[0]), N, Hn, nu), np.arange(N + 1), N, 0, Ys[0], noise)
    st0 = tuple(np.repeat(_np(x)[None], N + 1, 0) for x in (state.pipeline_state.qpos, state.pipeline_state.qvel))
    got = {}
    for t, a in pairs:
        loop.set_task(0, env.probed(t, a))
        _restart(loop, Ys[0], rngs[0])
        loop.step(1, env_step=False)
        torch.cuda.synchronize()
        ctrl = _np(loop.info()["rews"]) * (Hs + 1)
        if t == 0:
            st = st0
        else:
            q, qd, _ = mb.plan.reverse_trajectories()
            st = (_np(q[:, t - 1]), _np(qd[:, t - 1]))
        ref = cp.ctrl64(o, M, Y, t, a, st)
        tol = cp.ctrl_tol(o, M, Y, e, noise, t, a, ctrl, st)
        _note(group or name, cp.check(ctrl, ref, tol, f"{name} N={N} Hs={Hs} Hn={Hn} t={t} a={a}"))
        got[t, a] = ctrl
    return got, o


@pytest.mark.parametrize("name,Hn", [("quadpod", 4), ("slidepod", 7)])
def test_sampler_elements_match_restatement(built, name, Hn):
    """Case a: every knot of every actuator of every row of N = 2047 (rows 0 and N - 1, both halves of the
    legacy layout, the erfinv tail rows), against XLA's float32 algorithm."""
    nu = _pair(name)[0].action_size
    _single(name, 2047, Hn, Hn, [(t, a) for t in range(1, Hn + 1) for a in range(nu)], group="a. sampler")


SPLINES = [("quadpod", 16, 2), ("quadpod", 25, 3), ("branchpod", 16, 5), ("pincher", 25, 5), ("slidepod", 63, 7),
           ("quadpod", 63, 7), ("branchpod", 63, 7)]


@pytest.mark.parametrize("name,Hs,Hn", SPLINES, ids=[f"{n}-Hs{s}-Hn{k}" for n, s, k in SPLINES])
def test_spline_and_horizon_match_fp64(built, name, Hs, Hn):
    """Case b: t = 0, a step between knots, a step on a knot (or next to it when Hs is not a multiple of Hn)
    and the last step, every actuator."""
    env, _ = _pair(name)
    on = round(Hs / Hn * (Hn // 2))
    steps = (0, max(1, Hs // (2 * Hn)), on, Hs)
    _single(name, 255, Hs, Hn, [(t, a) for t in steps for a in range(env.action_size)], seed=Hs, group="b. spline")


@pytest.mark.parametrize("name", ["quadpod", "quadpod_pos", "pincher"])
def test_action_map_edges_match_fp64(built, name):
    """Case e: action_scale 1.7, Ybar at and beyond +-1: clipped knots, targets beyond physical_joint_range,
    PD torques saturating joint_torque_range; the bounds are reached on most actuators."""
    got, o = _single(name, 255, 4, 4, [(t, a) for t in (0, 2, 4) for a in range(_pair(name)[0].action_size)],
                     edges=True, scale=1.7, group="e. action map")
    rng = o.joint_torque_range if o.leg_control == "torque" else o.physical_joint_range
    at = lambda c, b: (np.abs(c - np.float32(b)) <= 4 * np.spacing(np.float32(abs(b)))).any()
    clipped = [a for a in range(o.nu) if any(at(got[t, a], rng[a][0]) or at(got[t, a], rng[a][1]) for t in (0, 2, 4))]
    assert len(clipped) >= o.nu // 2, clipped


def test_shard_and_injected_eps_match_fp64(built, monkeypatch):
    """Case c: the rank-1 shard of MBDPI(rank=1, world_size=2) on one GPU: local row j draws sample
    Ntotal / 2 + j from the Ntotal-sample stream, its mean row is unnoised; then the caller's eps."""
    from dial_mpc_b200 import random as drandom
    monkeypatch.setenv("DIAL_EXCHANGE", "nccl")     # one process: the shard's kernels run without a peer
    env, o = _pair("quadpod")
    N, Hs, Hn, nu = 512, 16, 4, 8
    rngs, Ys = _inputs(1, Hn, nu, 11)
    state = env.reset(drandom.PRNGKey(0))
    M = cp.spline64(Hs, Hn)
    noise = (0.9 ** np.arange(Hn + 1)[::-1]).astype(np.float32)
    key = cp.sample_key(rngs[0])
    eps_in = np.random.default_rng(12).standard_normal((N, Hn + 1, nu)).astype(np.float32)
    for t, a in ((3, 1), (8, 6), (16, 2)):
        mb = _mb(env.probed(t, a), N, Hs, Hn, rank=1, world_size=2)
        assert mb.plan.desc.shard_offset == N // 2 and mb.Nlocal == N // 2
        for inject in (False, True):
            eps = eps_in if inject else cp.eps_xla(key, N, Hn, nu)
            Y, e = cp.knots64(eps.astype(np.float64), np.arange(N // 2 + 1), N // 2, N // 2, Ys[0], noise)
            rews = torch.empty(N // 2 + 1, device="cuda")
            mb.plan.reverse_rollout(state, mb.plan.f32(eps_in) if inject else None, None if inject else key,
                                    mb.plan.f32(Ys[0]), mb.plan.f32(noise), rews)
            torch.cuda.synchronize()
            ctrl = _np(rews) * (Hs + 1)
            q, qd, _ = mb.plan.reverse_trajectories()
            st = (_np(q[:, t - 1]), _np(qd[:, t - 1]))
            tol = cp.ctrl_tol(o, M, Y, e * (not inject), noise, t, a, ctrl, st)
            _note("c. shard / eps", cp.check(ctrl, cp.ctrl64(o, M, Y, t, a, st), tol, f"shard t={t} a={a} inject={inject}"))


# ---- batched plans (position mode: the controls do not depend on the state) ---------------------------------
def _heavy(env, m):
    return env.sys.tree_replace({"body_mass": {"torso": m}})


def _batched(N, Hs, Hn, probes, seed, K=0, ensemble=None, models=None, schedule=None, n=1, update_rows=()):
    """A batched DeviceLoop on quadpod in position mode whose instance b probes probes[b]; unlike rng and
    Ybar per instance.  Runs step(n, env_step=False) eager, captured and replayed, each from the same
    start; the controls of iteration n - 1 of every row of every instance (every member) against fp64."""
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import DeviceLoop, schedule_setting, schedule_table
    env, o = _pair("quadpod_pos")
    B, nu = len(probes), env.action_size
    rngs, Ys = _inputs(B, Hn, nu, seed)
    states = [env.reset(drandom.PRNGKey(b)) for b in range(B)]
    envs = [env.probed(t, a) for t, a in probes]
    for b, m in enumerate(models or ()):
        if m is not None:
            envs[b].sys = m

    def make():
        return DeviceLoop(_mb(env, N, Hs, Hn, B=B, K=K), states, rngs, Ys, envs=envs, ensemble=ensemble,
                          schedule=schedule)
    loop1, loop2 = make(), (make() if n > 1 else None)
    dev = loop1.buf["noise"].device
    tables = [_np(schedule_table(schedule_setting(s, loop1.mbdpi.args), 4, dev)) if s else _np(loop1.buf["noise"])
              for s in (schedule or [None] * B)]
    M = cp.spline64(Hs, Hn)
    first = None
    for rep in range(3):                      # eager, capture, replay
        _restart(loop1, Ys, rngs)
        if n > 1:
            _restart(loop2, Ys, rngs)
            loop2.step(n - 1, env_step=False)
        loop1.step(n, env_step=False)
        torch.cuda.synchronize()
        Yin = _np(loop2.buf["Y"]) if n > 1 else Ys.astype(np.float64)
        rin = loop2.rng_host() if n > 1 else rngs
        r = _np(loop1.member_rewards()) if K else _np(loop1.info()["rews"])[:, None]
        if first is None:
            first = r
        assert np.array_equal(r, first), rep      # capture and replay compute what the eager step computed
        for b, (t, a) in enumerate(probes):
            noise = tables[b][n - 1]
            Y, e = cp.knots64(cp.eps_xla(cp.sample_key(rin[b]), N, Hn, nu), np.arange(N + 1), N, 0, Yin[b], noise)
            ref = cp.ctrl64(o, M, Y, t, a)
            for k in range(r.shape[1]):
                ctrl = r[b, k] * (Hs + 1)
                tol = cp.ctrl_tol(o, M, Y, e, noise, t, a, ctrl)
                _note("c/d. layouts", cp.check(ctrl, ref, tol, f"N={N} n={n} rep={rep} instance {b} member {k} t={t} a={a}"))
            if rep == 0:
                _update_agrees(env, o, N, Hs, Hn, M, Yin[b], rin[b], noise, t, a, r[b, 0] * (Hs + 1), e, update_rows)


def _update_agrees(env, o, N, Hs, Hn, M, Ybar, rng, noise, t, a, ctrl, e, rows):
    """Case f: one-hot weights make update_kernel's Ybar_out the knots it regenerates for sample j; the
    controls they give are those the rollout applied to row j."""
    from dial_mpc_b200.plan import Plan
    if not rows:
        return
    plan = Plan(env, env.plan_desc(Nsample=N, Hsample=Hs, Hnode=Hn, temp_sample=TEMP))
    for j in rows:
        r = np.full(N + 1, -np.inf, np.float32)
        r[j] = 0.0
        if j < N:
            r[N] = np.nan
        k = torch.as_tensor(np.ascontiguousarray(rng, np.uint32).view(np.int32).copy(), device="cuda")
        Yo, w = torch.empty(Hn + 1, env.action_size, device="cuda"), torch.empty(N + 1, device="cuda")
        plan.reverse_update_fused(torch.as_tensor(r, device="cuda"), k, plan.f32(Ybar), plan.f32(noise), Yo, w)
        torch.cuda.synchronize()
        assert float(w[j]) == 1.0
        Yu = _np(Yo)[None]
        ref = cp.ctrl64(o, M, Yu, t, a)
        tol = cp.ctrl_tol(o, M, Yu, e[j:j + 1], noise, t, a, ctrl[j:j + 1])
        _note("f. update agrees", cp.check(ctrl[j:j + 1], ref, tol, f"update knots of sample {j}, t={t} a={a}"))


# each actuator once, at steps on and between the knots of Hs = 16, Hn = 4
PROBES = list(zip((1, 5, 8, 10, 13, 16, 3, 15), range(8)))
LAYOUTS = [(1, None), (31, "16"), (255, "1"), (255, "16"), (2047, None)]


@pytest.mark.parametrize("N,wpc", LAYOUTS, ids=[f"N{n}-wpc{w or 'auto'}" for n, w in LAYOUTS])
def test_batched_rows_match_fp64(built, monkeypatch, N, wpc):
    """Case c/f: eight unlike instances, every row; DIAL_WPC sets the warps per CTA (rows straddle CTAs, the
    last lock-step CTA is padded)."""
    if wpc:
        monkeypatch.setenv("DIAL_WPC", wpc)
    _batched(N, 16, 4, PROBES, seed=N, update_rows=(0, N // 2, N - 1, N) if N == 255 else ())


def test_unfused_key_path_matches_fp64(built, monkeypatch):
    """Case c: without the fused update (a one-instance plan) a separate kernel splits the rng and the
    rollout reads the key it wrote (key_dev), not the rng (rng_dev)."""
    monkeypatch.setenv("DIAL_NO_FUSED_UPDATE", "1")
    _single("quadpod", 255, 16, 4, [(t, a) for t in (0, 5, 8) for a in range(8)], seed=21, group="c/d. layouts")


def test_instance_models_rows_match_fp64(built):
    """Case c: instances with their own physical model (set_instance_model) next to instances on the plan's."""
    env, _ = _pair("quadpod_pos")
    _batched(255, 16, 4, PROBES[:5], seed=3, models=[None, _heavy(env, 6.0), None, _heavy(env, 3.0), None])


def test_ensemble_members_roll_the_same_samples(built):
    """Case c: every member of an ensemble rolls the same samples (member_rewards, per member)."""
    env, _ = _pair("quadpod_pos")
    _batched(255, 16, 4, PROBES[2:5], seed=4, K=3, ensemble=[env.sys, _heavy(env, 6.0), _heavy(env, 2.5)])


@pytest.mark.parametrize("n", [1, 2, 4])
def test_iterations_use_their_noise_row(built, n):
    """Case d: the last iteration of step(n) rolls with noise[n - 1]; instance 1 with its own schedule's."""
    spec = {"sigma_scale": 0.6, "traj_diffuse_factor": 0.7, "horizon_diffuse_factor": 0.8}
    _batched(255, 16, 4, PROBES[:3], seed=5 + n, schedule=[None, spec, None], n=n)
