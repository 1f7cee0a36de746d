"""TEST-ONLY probe envs that read the controls a sampled rollout applies, and their fp64 reference.

The probe reward (tests/probes/ctrl_probe_reward.cuh) returns ctrl[a] at env step t and 0 at every other
step, (t, a) = the env's ``probe`` (its user constants).  A row's mean reward is then ctrl / H exactly up
to the final division, so ``rews * H`` is the control row j applied at step t of its rollout.  The
probe envs are the fixtures the suite already builds, with that reward: one custom build per solver
variant (star<3,6>: quadpod and slidepod; generic tree: branchpod; dense nv = 10: pincher).

The reference restates the rollout prologue from the oracle alone (planner_oracle's Threefry + erfinv
and scipy-checked spline, the oracle env's act2joint / act2tau), not from the product's host code:
  Y0s = clip(Ybar + eps * noise, +-1), node 0 and the mean row not noised, eps keyed by split(rng)[1];
  u = spline_matrix(step_nodes, step_us) @ Y0s;  ctrl = act2joint(u), or act2tau(u, q, qd).

Tolerance of one control (``ctrl_tol``), from the fp32 arithmetic, with e = 2^-24:
  u       10 e sum_k |M_tk| (|Y_k| + 1)            fp32 spline entries and products, a sum of <= 8 terms
          + sum_k |M_tk| noise_k EPS_ULP ulp(eps_k)  the kernel's eps against XLA's float32 algorithm
  target  g tol_u + 4 ulp(max(|jr0|, |jr1|, jr1 - jr0))   g = action_scale (jr1 - jr0) / 2
  torque  kp tol_target + kp ulp(max(|jt|, |q|)) + kd ulp(|qd|)
  + 4 ulp(|ctrl|): rews * H recovers ctrl from the mean reward to 4 ulp (the library divides with
    -use_fast_math, <= 2 ulp of the quotient).
A wrong row -> sample map, key, noise iteration or spline row moves a control by O(noise x joint range),
above 1e-2, while these tolerances are below 1e-5."""
import copy
import functools
import os
import sys
import tempfile

import numpy as np

from tests.conftest import ROOT

PROBE = os.path.join(ROOT, "tests", "probes", "ctrl_probe_reward.cuh")
EX = os.path.join(ROOT, "dial_mpc_b200", "examples", "custom_env")
E32 = 2.0 ** -24
EPS_ULP = 4          # the sampler's eps against jax_normal_legacy_xla (tests/test_gpu_update.py, test e)
CTRL_DT = 0.02       # MBDPI's knot grid: linspace(0, 0.02 Hs, ...)


class _Probe:
    """Mixin: the probe reward, ``probe`` = (env step, actuator) as the reward's user constants."""
    reward_source = PROBE
    probe = (0, 0)

    def user_params(self):
        return np.array(self.probe, dtype=np.float32)

    def probed(self, t, a):
        """A copy of this env (same model and build) that probes actuator a at env step t."""
        e = copy.copy(self)
        e.probe = (int(t), int(a))
        return e


def _classes():
    if EX not in sys.path:
        sys.path.insert(0, EX)
    import pincher_env
    import quadpod_env
    from tests import tree_envs

    class QuadpodProbe(_Probe, quadpod_env.QuadpodEnv):
        pass

    class SlidepodProbe(_Probe, tree_envs.SlidepodEnv):
        pass

    class BranchpodProbe(_Probe, tree_envs.BranchpodEnv):
        pass

    class PincherProbe(_Probe, pincher_env.PincherEnv):
        pass

    # name -> (class, config class, configuration)
    return {
        "quadpod": (QuadpodProbe, quadpod_env.QuadpodEnvConfig, {}),                         # star<3,6>, torque
        "quadpod_pos": (QuadpodProbe, quadpod_env.QuadpodEnvConfig, dict(leg_control="position")),
        "slidepod": (SlidepodProbe, tree_envs.TreeEnvConfig, tree_envs.FIXTURES["slidepod"][1]),  # per-joint kp/kd
        "branchpod": (BranchpodProbe, tree_envs.TreeEnvConfig, tree_envs.FIXTURES["branchpod"][1]),  # generic tree
        "pincher": (PincherProbe, pincher_env.PincherEnvConfig, {}),                         # dense nv = 10, position
    }


_CLASSES = None


def make_probe(name, **overrides):
    """(probe env, oracle env) of a fixture; ``overrides`` go into the env configuration."""
    global _CLASSES
    from oracle.envs_oracle import CustomRewardOracle
    if _CLASSES is None:
        _CLASSES = _classes()
    cls, cfg_cls, kw = _CLASSES[name]
    cfg = cfg_cls(**dict(kw, **overrides))
    env = cls(cfg)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, name + ".json")
        env.sys.model.save(path)
        o = CustomRewardOracle(path, lambda ctx: 0.0, joint_range=env.joint_range, kp=env._kp(), kd=env._kd(),
                               dt=cfg.dt, timestep=cfg.timestep, action_scale=cfg.action_scale,
                               leg_control=cfg.leg_control)
    return env, o


# ---- the fp64 reference -----------------------------------------------------------------------------
def split(rng):
    from oracle.planner_oracle import jax_split_legacy
    return jax_split_legacy(tuple(int(v) for v in np.asarray(rng, dtype=np.uint32)))


def sample_key(rng):
    """The key the rollout of an iteration draws its noise with: split(planner rng)[1]."""
    return tuple(int(v) for v in split(rng)[1])


def spline64(Hs, Hn):
    """[Hs+1, Hn+1]: the quadratic spline from MBDPI's knot grid to its step grid (oracle, scipy)."""
    from oracle.planner_oracle import spline_matrix
    T = CTRL_DT * Hs
    return spline_matrix(np.linspace(0, T, Hn + 1), np.linspace(0, T, Hs + 1))


@functools.lru_cache(maxsize=64)
def eps_xla(key, Ntotal, Hn, nu):
    """jax.random.normal(key, (Ntotal, Hn+1, nu)) by XLA's float32 erfinv algorithm (read-only: cached)."""
    from oracle.planner_oracle import jax_normal_legacy_xla
    return jax_normal_legacy_xla(key, (Ntotal, Hn + 1, nu))


def knots64(eps, rows, Nlocal, shard_offset, Ybar, noise):
    """(Y0s [R, Hn+1, nu], the eps each knot was drawn with) of local rows ``rows`` of a plan with Nlocal
    samples at ``shard_offset``: row Nlocal is the mean row (Ybar); sample j has eps[shard_offset + j]."""
    rows = np.asarray(rows)
    Ybar, noise = np.asarray(Ybar, np.float64), np.asarray(noise, np.float64)
    e = np.zeros((len(rows),) + Ybar.shape)
    smp = rows < Nlocal
    e[smp] = eps[shard_offset + rows[smp]]
    e[:, 0] = 0.0                                   # node 0 is pinned to Ybar[0]
    return np.clip(Ybar[None] + e * noise[None, :, None], -1.0, 1.0), e


def ctrl64(o, M, Y, t, a, state=None):
    """Control of actuator a at step t of rows with knots Y [R, Hn+1, nu]; ``state`` = (q [R, nq], qd [R, nv]),
    the state the step starts from (torque mode)."""
    u = np.einsum("k,rka->ra", M[t], Y)
    if o.leg_control == "torque":
        return o.act2tau(u, *state)[:, a]
    return o.act2joint(u)[:, a]


def ctrl_tol(o, M, Y, e, noise, t, a, ctrl, state=None):
    """Per-row tolerance of ctrl[row, t, a] (module docstring); ``e``: the eps of ``knots64``."""
    sp = lambda x: np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)
    Mt = np.abs(M[t])
    tol_u = (Mt[None] * (10 * E32 * (np.abs(Y[:, :, a]) + 1)
                         + np.asarray(noise, np.float64)[None] * EPS_ULP * sp(e[:, :, a]) * (e[:, :, a] != 0))).sum(1)
    jr0, jr1 = o.joint_range[a]
    g = o.action_scale * (jr1 - jr0) / 2
    tol = g * tol_u + 4 * sp(max(abs(jr0), abs(jr1), jr1 - jr0))
    if o.leg_control == "torque":
        u = np.einsum("k,rk->r", M[t], Y[:, :, a])
        jt = o.act2joint(np.repeat(u[:, None], o.nu, 1))[:, a]
        kp, kd = np.broadcast_to(o.kp, (o.nu,))[a], np.broadcast_to(o.kd, (o.nu,))[a]
        qa, qda = state[0][:, 7 + a], state[1][:, 6 + a]
        tol = kp * tol + kp * sp(np.maximum(np.abs(jt), np.abs(qa))) + kd * sp(qda)
    return tol + 4 * sp(ctrl)


def check(got, ref, tol, what):
    """Assert |got - ref| <= tol elementwise; returns the worst |got - ref| / tol."""
    err = np.abs(np.asarray(got, np.float64) - ref)
    ratio = err / tol
    i = int(np.argmax(ratio))
    assert np.isfinite(got).all() and ratio.max() <= 1.0, \
        f"{what}: element {i}: got {np.ravel(got)[i]!r}, fp64 {np.ravel(ref)[i]!r}, tol {np.ravel(tol)[i]:.3g}"
    return float(ratio.max())
