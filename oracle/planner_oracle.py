"""ORACLE (test infrastructure, not product code) — fp64 restatement of the
reference planner maths.  PARITY UNPINNED (see mjx_oracle.py header).

Follows dial_mpc/core/dial_core.py:
* MBDPI.__init__ (sigma_control, time grids)            :51-89
* node2u / u2node (jax_cosmo InterpolatedUnivariateSpline k=2 == scipy's)  :91-101
* reverse_once                                          :103-145
* shift / shift_Y_from_u                                :160-172
* the annealing schedule of main()                      :253-264
The noise ``eps`` is injected (the JAX PRNG stream layout is version dependent,
SURVEY.md Appendix E); :func:`threefry2x32` / :func:`jax_normal_legacy` restate the
Threefry-2x32 generator and the legacy (non-partitionable) counter layout.
"""

from __future__ import annotations

from typing import Dict, Tuple

import numpy as np
from scipy.interpolate import InterpolatedUnivariateSpline
from scipy.special import erfinv

from .envs_oracle import OracleEnv, OState


def spline_matrix(x_from: np.ndarray, x_to: np.ndarray) -> np.ndarray:
    """Matrix of the (linear) map y(x_from) -> spline(x_to), quadratic interpolating spline."""
    n = len(x_from)
    M = np.zeros((len(x_to), n))
    for i in range(n):
        e = np.zeros(n)
        e[i] = 1.0
        M[:, i] = InterpolatedUnivariateSpline(x_from, e, k=2)(x_to)
    return M


def make_Y0s(eps, Ybar, noise_scale):
    """Y0s = eps * noise + Ybar with node 0 pinned, the mean row Ybar appended, clipped to [-1, 1]
    (dial_core.py:107-116)."""
    Y0s = eps * noise_scale[None, :, None] + Ybar
    Y0s[:, 0] = Ybar[0]
    Y0s = np.concatenate([Y0s, Ybar[None]], 0)
    return np.clip(Y0s, -1.0, 1.0)


def softmax_weights_fp64(rews, temp):
    """The update's weights softmax((rews - rews[-1]) / std(rews) / temp) (dial_core.py:125-128) in
    fp64, with the guards of the CUDA kernels (the reference has none):
    * non-finite rewards get weight 0 and are left out of the statistics;
    * softmax is shift-invariant, so a non-finite mean-row reward rews[-1] changes nothing (the
      logits are taken relative to the largest finite reward);
    * flat finite rewards (std 0) give uniform weights over the finite samples;
    * no finite reward at all puts the whole weight on the mean row."""
    r = np.asarray(rews, dtype=np.float64)
    fin = np.isfinite(r)
    w = np.zeros_like(r)
    if not fin.any():
        w[-1] = 1.0
        return w
    rf = r[fin]
    sd = rf.std()                      # two-pass (mean first): no cancellation
    e = np.exp((rf - rf.max()) / sd / temp) if sd > 0 else np.ones_like(rf)
    w[fin] = e / e.sum()
    return w


def reverse_update_fp64(rews, temp, eps, Ybar, noise_scale):
    """Weights and Ybar_new = sum_n w_n Y0s_n of one reverse_once update in fp64: the reference for
    the CUDA update kernels on given rewards.  eps [N, Hn+1, nu], rews [N+1] (mean row last)."""
    w = softmax_weights_fp64(rews, temp)
    Y0s = make_Y0s(np.asarray(eps, np.float64), np.asarray(Ybar, np.float64), np.asarray(noise_scale, np.float64))
    return w, np.einsum("n,nij->ij", w, Y0s)


class PlannerOracle:
    def __init__(self, env: OracleEnv, Nsample, Hsample, Hnode, temp_sample,
                 horizon_diffuse_factor, traj_diffuse_factor, sigma_scale=1.0):
        self.env = env
        self.N, self.Hs, self.Hn = Nsample, Hsample, Hnode
        self.temp = temp_sample
        self.tdf = traj_diffuse_factor
        self.nu = env.nu
        self.sigma_control = horizon_diffuse_factor ** np.arange(Hnode + 1)[::-1] * sigma_scale
        self.ctrl_dt = 0.02
        self.step_us = np.linspace(0, self.ctrl_dt * Hsample, Hsample + 1)
        self.step_nodes = np.linspace(0, self.ctrl_dt * Hsample, Hnode + 1)
        self.M_n2u = spline_matrix(self.step_nodes, self.step_us)
        self.M_u2n = spline_matrix(self.step_us, self.step_nodes)

    def node2u(self, Y):        # [..., Hn+1, nu] -> [..., Hs+1, nu]
        return np.einsum("tk,...ka->...ta", self.M_n2u, Y)

    def u2node(self, u):
        return np.einsum("kt,...ta->...ka", self.M_u2n, u)

    def shift(self, Y):
        u = self.node2u(Y)
        u = np.roll(u, -1, axis=0)
        u[-1] = 0.0
        return self.u2node(u)

    def make_Y0s(self, eps, Ybar, noise_scale):
        return make_Y0s(eps, Ybar, noise_scale)

    def reverse_once(self, state: OState, eps, Ybar, noise_scale) -> Tuple[np.ndarray, Dict]:
        Y0s = self.make_Y0s(eps, Ybar, noise_scale)
        us = self.node2u(Y0s)
        rewss, qs, qds, xs = self.env.rollout(state, us)
        rews = rewss.mean(-1)
        rew_Ybar = rewss[-1].mean()
        logp0 = (rews - rew_Ybar) / rews.std() / self.temp
        w = np.exp(logp0 - logp0.max())
        w = w / w.sum()
        Ybar_new = np.einsum("n,nij->ij", w, Y0s)
        info = dict(rews=rews, rewss=rewss, weights=w, Y0s=Y0s, us=us,
                    qbar=np.einsum("n,nij->ij", w, qs), qdbar=np.einsum("n,nij->ij", w, qds),
                    xbar=np.einsum("n,nijk->ijk", w, xs), new_noise_scale=noise_scale)
        return Ybar_new, info

    def schedule(self, n_diffuse):
        return self.sigma_control[None] * self.tdf ** np.arange(n_diffuse)[:, None]


# ---------------------------------------------------------------------------
# Threefry-2x32 (Random123 / JAX) and the JAX legacy normal sampler
# ---------------------------------------------------------------------------
def _rotl(x, r):
    return ((x << np.uint32(r)) | (x >> np.uint32(32 - r))).astype(np.uint32)


def threefry2x32(key, x0, x1):
    """20-round Threefry-2x32.  key: (k0,k1) uint32; x0,x1: uint32 arrays."""
    k0, k1 = np.uint32(key[0]), np.uint32(key[1])
    ks = [k0, k1, np.uint32(k0 ^ k1 ^ np.uint32(0x1BD11BDA))]
    rot = [[13, 15, 26, 6], [17, 29, 16, 24]]
    x0 = (np.asarray(x0, dtype=np.uint32) + ks[0]).astype(np.uint32)
    x1 = (np.asarray(x1, dtype=np.uint32) + ks[1]).astype(np.uint32)
    with np.errstate(over="ignore"):
        for i in range(5):
            for r in rot[i % 2]:
                x0 = (x0 + x1).astype(np.uint32)
                x1 = _rotl(x1, r)
                x1 = x1 ^ x0
            x0 = (x0 + ks[(i + 1) % 3]).astype(np.uint32)
            x1 = (x1 + ks[(i + 2) % 3] + np.uint32(i + 1)).astype(np.uint32)
    return x0, x1


def jax_random_bits_legacy(key, n):
    """jax.random bits, threefry_partitionable=False: counters 0..n-1 split in halves (an odd
    count is padded with one ZERO counter, jax._src.prng.threefry_2x32)."""
    odd = n % 2
    cnt = np.concatenate([np.arange(n, dtype=np.uint32), np.zeros(odd, dtype=np.uint32)])
    half = (n + odd) // 2
    a, b = threefry2x32(key, cnt[:half], cnt[half:])
    return np.concatenate([a, b])[:n]


def jax_split_legacy(key, num=2):
    bits = jax_random_bits_legacy(key, 2 * num)
    return bits.reshape(num, 2)


def jax_uniform_legacy(key, shape, minval, maxval):
    """jax.random.uniform(key, shape, float32, minval, maxval): mantissa bits -> [1,2) - 1, scaled,
    clamped from below (jax._src.random._uniform)."""
    n = int(np.prod(shape))
    bits = jax_random_bits_legacy(key, n)
    f = ((bits >> np.uint32(9)) | np.uint32(0x3F800000)).view(np.float32) - np.float32(1.0)
    lo, hi = np.float32(minval), np.float32(maxval)
    return np.maximum(lo, f * (hi - lo) + lo).astype(np.float32).reshape(shape)


def sample_command_oracle(rng):
    """sample_command of the walk envs (unitree_go2_env.py:298-315, unitree_h1_env.py:358-375)."""
    _, k1, k2, k3 = jax_split_legacy(rng, 4)
    vx = jax_uniform_legacy(k1, (1,), -1.5, 1.5)[0]
    vy = jax_uniform_legacy(k2, (1,), -0.5, 0.5)[0]
    wz = jax_uniform_legacy(k3, (1,), -1.5, 1.5)[0]
    return np.array([vx, vy, 0.0]), np.array([0.0, 0.0, wz])


def sample_jump_sequence_oracle(rng, n_steps=10):
    """UnitreeGo2SeqJumpEnv.sample_command (unitree_go2_env.py:594-631): 2 n_steps keys from
    jax.random.split; the COM target walks by uniform(+-0.65) in x, y and the heading by
    uniform(+-0.5), both as fp32 running sums (lax.scan carries float32).  Returns (com_pos
    [n_steps+1, 3], com_yaw [n_steps+1]) — the inputs of generate_jumping_sequence."""
    keys = jax_split_legacy(rng, 2 * n_steps)
    pos = [np.array([0.0, 0.0, 0.27], dtype=np.float32)]
    yaw = [np.float32(0.0)]
    for i in range(n_steps):
        nxt = pos[-1].copy()
        nxt[:2] = nxt[:2] + jax_uniform_legacy(keys[i], (2,), -0.65, 0.65)
        pos.append(nxt)
        yaw.append(np.float32(yaw[-1] + jax_uniform_legacy(keys[n_steps + i], (1,), -0.5, 0.5)[0]))
    return np.array(pos), np.array(yaw)


def _normal_uniform_legacy(key, n):
    """The fp32 uniform in (-1, 1) that jax.random.normal feeds to erfinv (legacy layout)."""
    bits = jax_random_bits_legacy(key, n)
    f = ((bits >> np.uint32(9)) | np.uint32(0x3F800000)).view(np.float32) - np.float32(1.0)
    lo = np.nextafter(np.float32(-1.0), np.float32(0.0))
    return np.maximum(lo, f * (np.float32(1.0) - lo) + lo).astype(np.float32)


def jax_normal_legacy(key, shape):
    """jax.random.normal(key, shape, float32): sqrt(2)*erfinv(uniform(-1+ulp, 1))."""
    u = _normal_uniform_legacy(key, int(np.prod(shape)))
    return (np.sqrt(2.0) * erfinv(u.astype(np.float64))).reshape(shape)


ERFINV_TAIL_W = 5.0


def erfinv_xla(u):
    """XLA's single-precision erfinv (Giles' polynomials: the algorithm jax.random.normal runs in
    float32, and the kernels' erfinv_f32) in fp64, except for u * u, which is rounded to fp32 before
    log1p as in float32.  Near |u| = 1 that one rounding is amplified by 1 / (1 - u^2): at |u| = 0.9999
    it moves eps by about 50 fp32 ulp away from the exact sqrt(2) erfinv(u).  Elsewhere the polynomials
    are within about 2 ulp of the exact function."""
    x = np.asarray(u, dtype=np.float32)
    w = -np.log1p(-(x * x).astype(np.float64))
    x = x.astype(np.float64)
    lo = w < ERFINV_TAIL_W
    t = np.where(lo, w - 2.5, np.sqrt(w) - 3.0)
    p = np.where(lo, 2.81022636e-08, -0.000200214257)
    for a, b in zip((3.43273939e-07, -3.5233877e-06, -4.39150654e-06, 0.00021858087, -0.00125372503, -0.00417768164,
                     0.246640727, 1.50140941),
                    (0.000100950558, 0.00134934322, -0.00367342844, 0.00573950773, -0.0076224613, 0.00943887047,
                     1.00167406, 2.83297682)):
        p = np.where(lo, a, b) + p * t
    return p * x


def jax_normal_legacy_xla(key, shape):
    """jax_normal_legacy with XLA's float32 erfinv algorithm (:func:`erfinv_xla`) instead of the exact
    erfinv: what the kernels' sampler computes, up to the fp32 rounding of the remaining steps."""
    u = _normal_uniform_legacy(key, int(np.prod(shape)))
    return (np.sqrt(2.0) * erfinv_xla(u)).reshape(shape)


def erfinv_tail_indices(key, n):
    """Flat indices i < n of jax.random.normal(key, (n,)) (legacy layout) whose uniform u takes the
    tail branch of XLA's single-precision erfinv, w = -log(1 - u^2) >= 5: |u| > 0.9966, |eps| > 2.93
    (about 0.37 % of the elements).  The kernels' sampler evaluates that branch only there."""
    u = _normal_uniform_legacy(key, n).astype(np.float64)
    return np.flatnonzero(-np.log1p(-u * u) >= ERFINV_TAIL_W)
