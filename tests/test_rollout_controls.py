"""The controls the sampled rollout applies, read out of the device code in the CPU warp emulator and
compared with an fp64 restatement (tests/ctrl_probe.py, whose docstring derives the tolerances).

The emulator runs the prologue of rollout_warp in sampled mode (mode 1: in-kernel Threefry + erfinv
knots, clip, node 0 pinned, mean row unnoised, spline, action map) on every row of a launch; the probe
reward makes each row's mean reward the control of one actuator at one step.  The launch is cut after
the probed step (H = t + 1): the control at step t does not depend on later steps.  Cases:
  a. the sampler element by element (Hs = Hn: the spline is the identity), tail rows of the erfinv;
  b. spline and horizon, Hn in {2, 3, 5, 7} with Hs up to 63 = DIAL_MAXH - 1;
  c. the rank-1 shard of a two-rank plan (gidx = shard_offset + row) and the mean row;
  d. injected eps against native sampling.
The same checks run on an H100 in tests/test_gpu_rollout_controls.py."""
import numpy as np
import pytest

from dial_mpc_b200.utils.spline import interp_matrix
from tests import ctrl_probe as cp

RNG = np.uint32([0xD9C2825F, 0xA30FEBCF])     # N = 15, Hn = 4, nu = 8: erfinv tail elements in rows 0, 3, 6, 8, 10, 11


def _desc(env, t, a, N, Hs, Hn, Ntotal=None, shard_offset=0):
    T = cp.CTRL_DT * Hs
    M = interp_matrix(np.linspace(0, T, Hn + 1), np.linspace(0, T, Hs + 1))
    return env.probed(t, a).plan_desc(Nsample=N, Ntotal=Ntotal or N, shard_offset=shard_offset, Hsample=Hs,
                                      Hnode=Hn, M_n2u=M)


def _state(env, seed):
    """Initial state: the env's init_q, a nonzero velocity (the PD's kd term acts from step 0)."""
    g = np.random.default_rng(seed)
    nv = env.sys.nv
    return np.asarray(env._init_q, np.float32), (0.3 * g.standard_normal(nv)).astype(np.float32), np.zeros(nv, np.float32)


def _inputs(Hn, nu, seed, edges=False):
    """Ybar, noise.  ``edges``: Ybar at and beyond +-1 (knots that clip), the noise scaled up."""
    g = np.random.default_rng(seed)
    Ybar = (g.standard_normal((Hn + 1, nu)) * (1.2 if edges else 0.4)).astype(np.float32)
    if edges:       # every actuator has knots beyond +1 and below -1, and some at exactly +-1
        Ybar = (1.3 * (-1.0) ** np.add.outer(np.arange(Hn + 1), np.arange(nu))).astype(np.float32)
        Ybar[1, 0], Ybar[2, 1], Ybar[3, 2] = 1.0, -1.0, 1.0
    noise = (0.9 ** np.arange(Hn + 1)[::-1] * (0.9 if edges else 0.6)).astype(np.float32)
    return Ybar, noise


def _emul_ctrl(env, desc, s0, t, Ybar, noise, key=None, eps=None):
    """(ctrl [N+1] at step t of every row, (q, qd) [N+1, *] the step started from)."""
    from tests.emul import emul
    q0, v0, w0 = s0
    nrows = desc.Nsample + 1
    out = emul.rollout(env, desc, q0, v0, w0, mode=1, eps=eps, Ybar=Ybar, noise=noise,
                       key=key or (0, 0), nrows=nrows, H=t + 1)
    ctrl = out["rews"].astype(np.float64) * (t + 1)
    if t == 0:
        st = (np.repeat(q0[None], nrows, 0).astype(np.float64), np.repeat(v0[None], nrows, 0).astype(np.float64))
    else:
        st = (out["q"][:, t - 1].astype(np.float64), out["qd"][:, t - 1].astype(np.float64))
    return ctrl, st


def _run(name, N, Hs, Hn, steps, acts=None, seed=0, Ntotal=None, shard_offset=0, inject=False, edges=False, **cfg):
    """Every row of a plan, the probed (t, a) pairs, against the reference; returns the worst err / tol and
    the controls read, {(t, a): ctrl [N+1]}."""
    env, o = cp.make_probe(name, **cfg)
    nu = env.action_size
    Ntotal = Ntotal or N
    Ybar, noise = _inputs(Hn, nu, seed, edges)
    s0 = _state(env, seed)
    key = cp.sample_key(RNG)
    eps = cp.eps_xla(key, Ntotal, Hn, nu)
    M = cp.spline64(Hs, Hn)
    rows = np.arange(N + 1)
    Y, e = cp.knots64(eps, rows, N, shard_offset, Ybar, noise)
    inj = None
    if inject:      # the caller's eps [Ntotal, Hn+1, nu] (every rank's): the kernel reads it instead of sampling
        inj = np.random.default_rng(seed + 1).standard_normal(eps.shape).astype(np.float32)
        Y, e = cp.knots64(inj.astype(np.float64), rows, N, shard_offset, Ybar, noise)
        e = e * 0.0     # injected eps are exact: no sampler error in the tolerance
    worst, got = 0.0, {}
    for t in steps:
        for a in (range(nu) if acts is None else acts):
            desc = _desc(env, t, a, N, Hs, Hn, Ntotal, shard_offset)
            ctrl, st = _emul_ctrl(env, desc, s0, t, Ybar, noise, key=None if inject else key, eps=inj)
            ref = cp.ctrl64(o, M, Y, t, a, st)
            tol = cp.ctrl_tol(o, M, Y, e, noise, t, a, ctrl, st)
            worst = max(worst, cp.check(ctrl, ref, tol, f"{name} N={N} Hs={Hs} Hn={Hn} t={t} a={a}"))
            got[t, a] = ctrl
    return worst, got


def test_probe_reads_the_applied_control():
    """The probe returns ctrl at its step only: a rollout of known actions (mode 0) gives back act2tau."""
    from tests.emul import emul
    env, o = cp.make_probe("quadpod")
    q0, v0, w0 = _state(env, 1)
    us = np.random.default_rng(1).uniform(-1, 1, (1, 3, env.action_size))
    for t, a in ((0, 0), (2, 5)):
        out = emul.rollout(env, env.probed(t, a).plan_desc(), q0, v0, w0, us=us)
        r = out["rewss"][0]
        assert (r[np.arange(3) != t] == 0).all()
        st = (q0[None], v0[None]) if t == 0 else (out["q"][:, t - 1], out["qd"][:, t - 1])
        ref = o.act2tau(us[:, t], *[np.asarray(x, np.float64) for x in st])[0, a]
        assert abs(r[t] - ref) <= 1e-5 * (1 + abs(ref)), (t, a, r[t], ref)


def test_sampler_elements_match_restatement():
    """Case a: Hs = Hn = 4, every actuator at every knot of every row of N = 15: rows 0 and N - 1, row 7 that
    holds the legacy layout's halfway point (element 300 of 600), at least three erfinv tail rows."""
    from oracle.planner_oracle import erfinv_tail_indices
    N, Hn, nu = 15, 4, 8
    ne = (Hn + 1) * nu
    tail = [i for i in erfinv_tail_indices(cp.sample_key(RNG), N * ne) if (i % ne) // nu >= 1]
    assert len({i // ne for i in tail}) >= 3
    worst, _ = _run("quadpod", N, Hn, Hn, range(1, Hn + 1))
    print(f"sampler elements: worst {worst:.3f} of the tolerance")


@pytest.mark.parametrize("name,Hs,Hn,steps,acts", [
    ("quadpod", 16, 2, (0, 5, 8), None),          # t = 0, between knots, on a knot; every actuator
    ("quadpod", 25, 3, (9, 25), (2, 7)),          # Hs not a multiple of Hn: no step on the inner knots; the last step
    ("branchpod", 16, 5, (7,), (0, 5, 11)),       # the generic tree solver
    ("quadpod", 63, 7, (63,), (6,)),              # the longest horizon, the most knots, the last step
], ids=["Hs16-Hn2", "Hs25-Hn3", "branchpod-Hs16-Hn5", "Hs63-Hn7"])
def test_spline_and_horizon_match_fp64(name, Hs, Hn, steps, acts):
    worst, _ = _run(name, 7, Hs, Hn, steps, acts)
    print(f"{name} Hs={Hs} Hn={Hn}: worst {worst:.3f} of the tolerance")


@pytest.mark.parametrize("name", ["quadpod", "quadpod_pos"])
def test_action_map_edges_match_fp64(name):
    """Case e: action_scale 1.7 and Ybar at and beyond +-1: knots that clip, targets beyond the physical
    joint range and (torque mode) PD torques that saturate the torque range, on most actuators."""
    env, o = cp.make_probe(name, action_scale=1.7)
    worst, got = _run(name, 7, 4, 4, (0, 2, 4), edges=True, action_scale=1.7)
    print(f"{name} edges: worst {worst:.3f} of the tolerance")
    rng = o.joint_torque_range if name == "quadpod" else o.physical_joint_range
    at = lambda c, b: (np.abs(c - np.float32(b)) <= 4 * np.spacing(np.float32(abs(b)))).any()
    clipped = [a for a in range(env.action_size)
               if any(at(got[t, a], rng[a][0]) or at(got[t, a], rng[a][1]) for t in (0, 2, 4))]
    assert len(clipped) >= env.action_size // 2, clipped


def test_shard_and_mean_row_match_fp64():
    """Case c: rank 1 of a two-rank plan: local row j draws sample Ntotal / 2 + j, its mean row is unnoised."""
    worst, _ = _run("quadpod", 8, 8, 4, (3, 8), (1, 6), Ntotal=16, shard_offset=8)
    print(f"shard: worst {worst:.3f} of the tolerance")


def test_injected_eps_match_fp64():
    worst, _ = _run("quadpod", 8, 8, 4, (5,), (0, 3), Ntotal=16, shard_offset=8, inject=True)
    print(f"injected eps: worst {worst:.3f} of the tolerance")


@pytest.mark.parametrize("perturb", ["spline_row", "eps_key", "shard_offset", "noise_row"])
def test_reference_perturbations_fail(perturb):
    """The checks have teeth: each of these errors in the reference fails them by far."""
    env, o = cp.make_probe("quadpod")
    N, Hs, Hn, t, a = 7, 8, 4, 3, 1
    nu = env.action_size
    Ybar, noise = _inputs(Hn, nu, 0)
    s0 = _state(env, 0)
    key = cp.sample_key(RNG)
    ctrl, st = _emul_ctrl(env, _desc(env, t, a, N, Hs, Hn, 2 * N, N), s0, t, Ybar, noise, key=key)
    M = cp.spline64(Hs, Hn)
    bad_key = tuple(int(v) for v in cp.split(RNG)[0]) if perturb == "eps_key" else key
    eps = cp.eps_xla(bad_key, 2 * N, Hn, nu)
    off = 0 if perturb == "shard_offset" else N
    nz = noise[::-1].copy() if perturb == "noise_row" else noise
    Y, e = cp.knots64(eps, np.arange(N + 1), N, off, Ybar, nz)
    tt = t + 1 if perturb == "spline_row" else t
    ref = cp.ctrl64(o, M, Y, tt, a, st)
    tol = cp.ctrl_tol(o, M, Y, e, nz, tt, a, ctrl, st)
    err = np.abs(ctrl - ref)
    assert (err[:N] > 100 * tol[:N]).mean() > 0.5, (perturb, float(np.median(err[:N] / tol[:N])))
