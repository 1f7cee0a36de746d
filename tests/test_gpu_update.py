"""The update stage of the control-step graph against a plain fp64 reference on known inputs.

Every reverse_once of dial_mpc_step runs update_kernel (reward statistics, softmax, Ybar = sum_n
w_n Y0s_n with the noise regenerated in-kernel from Threefry + erfinv, rng advance), then
mpc_shift_kernel between control steps and the bars kernels on a side branch.  Here each of them is
compared with oracle/planner_oracle.py in fp64 on given rewards, so nothing chaotic sits between the
kernel and its reference:
  a. the fused update on caller buffers (dial_reverse_update_fused) across sample counts and knot
     shapes, odd element counts included;
  b. its guards (non-finite rewards, NaN mean row, flat rewards, no finite reward);
  c. ill-conditioned reward statistics, on the eager weights kernel and the fused kernel;
  d. one launch over a batch of unlike instances;
  e. the in-kernel sampler element by element (one-hot weights make Ybar_out one sample's knots);
  f. the shift of the control-step graph;
  g. the graph end to end: the last iteration recomputed from the GPU's own rewards.

Tolerances: weights |w - w64| <= 1e-4 max(w64); Ybar 2e-5 absolute (fp32 sums of |Y0s| <= 1 with
weights summing to 1); rng integer-exact."""
import functools
import math

import numpy as np
import pytest
import torch

from tests.conftest import make_pair

pytestmark = pytest.mark.gpu

TEMP = 0.05
W_TOL = 1e-4      # x max(w64)
Y_TOL = 2e-5
GO2, H1, ALLEGRO = "unitree_go2_walk", "unitree_h1_walk", "allegro_reorient"


@functools.lru_cache(maxsize=None)
def _env(name):
    return make_pair(name)[0]


def _plan(name, N, Hn, B=1, Hs=8):
    from dial_mpc_b200.plan import Plan
    env = _env(name)
    return Plan(env, env.plan_desc(Nsample=N, Hsample=max(Hs, Hn), Hnode=Hn, temp_sample=TEMP, n_inst=B))


def _split(rng):
    from oracle.planner_oracle import jax_split_legacy
    return jax_split_legacy(tuple(int(v) for v in np.asarray(rng, dtype=np.uint32)))


def _eps64(rng, N, Hn, nu):
    """The noise the kernels draw in a reverse_once from planner rng `rng`: key = split(rng)[1]."""
    from oracle.planner_oracle import jax_normal_legacy
    return jax_normal_legacy(tuple(int(v) for v in _split(rng)[1]), (N, Hn + 1, nu))


def _inputs(N, Hn, nu, seed):
    g = np.random.default_rng(seed)
    rews = (g.normal(size=N + 1) * 0.3 - 1.0).astype(np.float32)
    rng = g.integers(0, 2 ** 32, size=2, dtype=np.uint64).astype(np.uint32)
    Ybar = (g.standard_normal((Hn + 1, nu)) * 0.4).astype(np.float32)      # some Y0s clip at +-1
    noise = (0.9 ** np.arange(Hn + 1)[::-1]).astype(np.float32)
    return rews, rng, Ybar, noise


def _fused(plan, rews, rng, Ybar, noise):
    """One dial_reverse_update_fused launch on host arrays -> (weights, Ybar_out, rng after)."""
    dev = plan.device
    r = torch.as_tensor(np.ascontiguousarray(rews, np.float32), device=dev)
    k = torch.as_tensor(np.ascontiguousarray(rng, np.uint32).view(np.int32).copy(), device=dev)
    Y = torch.as_tensor(np.ascontiguousarray(Ybar, np.float32), device=dev)
    out, w = torch.empty_like(Y), torch.empty_like(r)
    plan.reverse_update_fused(r, k, Y, torch.as_tensor(np.float32(noise), device=dev), out, w)
    torch.cuda.synchronize()
    return w.cpu().numpy(), out.cpu().numpy(), k.cpu().numpy().view(np.uint32)


def _eager(plan, rews, rng, Ybar, noise):
    """The eager update (weights_kernel + ybar_kernel), noise keyed by split(rng)[1]."""
    dev = plan.device
    r = torch.as_tensor(np.ascontiguousarray(rews, np.float32), device=dev)
    Y = torch.as_tensor(np.ascontiguousarray(Ybar, np.float32), device=dev)
    out, w = torch.empty_like(Y), torch.empty_like(r)
    plan.reverse_update(None, _split(rng)[1], Y, torch.as_tensor(np.float32(noise), device=dev), r, out, w)
    torch.cuda.synchronize()
    return w.cpu().numpy(), out.cpu().numpy()


def _check(w, Y, w64, Y64, what=""):
    werr = float(np.abs(w - w64).max() / w64.max())
    yerr = float(np.abs(Y - Y64).max())
    assert werr <= W_TOL and yerr <= Y_TOL, f"{what}: weights off by {werr:.3g} x max(w64), Ybar by {yerr:.3g}"
    assert np.isfinite(w).all() and np.isfinite(Y).all()


# ---- a. fused update across shapes ------------------------------------------------------------------
# ne = (Hn+1) nu: Go2 24 / 60 / 96, H1 95 (odd) / 152 (one sample slot per CTA), Allegro 128
SHAPES = [(GO2, 1), (GO2, 4), (GO2, 7), (H1, 4), (H1, 7), (ALLEGRO, 7)]
NS = [1, 2, 31, 255, 256, 2047, 2048, 131071]      # 131071: n = Ntotal + 1 = 2^17, the largest


@pytest.mark.parametrize("name,Hn", SHAPES, ids=[f"{n.split('_')[-2]}-Hn{h}" for n, h in SHAPES])
@pytest.mark.parametrize("N", NS)
def test_fused_update_matches_fp64(built, name, Hn, N):
    from oracle.planner_oracle import reverse_update_fp64
    plan = _plan(name, N, Hn)
    nu = plan.nu
    rews, rng, Ybar, noise = _inputs(N, Hn, nu, seed=N * 31 + Hn)
    w, Y, rng_out = _fused(plan, rews, rng, Ybar, noise)
    w64, Y64 = reverse_update_fp64(rews, TEMP, _eps64(rng, N, Hn, nu), Ybar, noise)
    _check(w, Y, w64, Y64, f"N={N} ne={(Hn + 1) * nu}")
    assert np.array_equal(rng_out, _split(rng)[0])
    assert abs(float(w.sum()) - 1) < 1e-5


# ---- b. guards -----------------------------------------------------------------------------------------
def _last_cta_row(N, ne):
    """First sample row of the fused update's last CTA (grid rule of dial_plan_create)."""
    slots = 256 // ne
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ybar_grid = min(max(math.ceil((N + 1) / slots), 1), 2 * sms)
    upd_grid = min(max(math.ceil((N + 1) / (slots * 8)), 1), ybar_grid)
    assert upd_grid > 1
    return (upd_grid - 1) * slots


def _guard_rewards(case, rews, N, ne):
    r = rews.copy()
    if case == "nan_inf":
        r[5], r[7] = np.nan, np.inf
    elif case == "nan_mean_row":
        r[-1] = np.nan
    elif case == "no_finite_reward":
        r[:] = np.nan
        r[3] = -np.inf
    elif case == "flat":
        r[:] = -1.25
    elif case == "flat_nan_mean_row":
        r[:] = -1.25
        r[-1] = np.nan
    elif case == "last_cta":
        r[_last_cta_row(N, ne)], r[N - 1] = np.nan, -np.inf
    return r


GUARDS = ["nan_inf", "nan_mean_row", "no_finite_reward", "flat", "flat_nan_mean_row", "last_cta"]


@pytest.mark.parametrize("kernel", ["fused", "eager"])
@pytest.mark.parametrize("case", GUARDS)
def test_update_guards_match_fp64(built, case, kernel):
    from oracle.planner_oracle import reverse_update_fp64
    N, Hn = 1000, 4
    plan = _plan(GO2, N, Hn)
    rews, rng, Ybar, noise = _inputs(N, Hn, 12, seed=7)
    r = _guard_rewards(case, rews, N, (Hn + 1) * 12)
    if kernel == "fused":
        w, Y, rng_out = _fused(plan, r, rng, Ybar, noise)
        assert np.array_equal(rng_out, _split(rng)[0])
    else:
        w, Y = _eager(plan, r, rng, Ybar, noise)
    w64, Y64 = reverse_update_fp64(r, TEMP, _eps64(rng, N, Hn, 12), Ybar, noise)
    _check(w, Y, w64, Y64, case)
    assert (w[:-1][~np.isfinite(r[:-1])] == 0).all()
    if case == "no_finite_reward":      # the mean sample keeps the whole weight: Ybar is kept (clipped)
        assert w[-1] == 1.0 and not w[:-1].any()
        assert np.abs(Y - np.clip(Ybar, -1, 1)).max() < 1e-6
    if case.startswith("flat"):         # uniform over the finite samples
        fin = np.isfinite(r)
        assert np.abs(w[fin] * fin.sum() - 1).max() < 1e-5


# ---- c. ill-conditioned reward statistics ----------------------------------------------------------------
def _ill_rewards(case, N, seed=13):
    """Rewards `centre +- spread` (uniform with that standard deviation: the softmax then spreads its
    weight over tens of samples, so an error in the std shows in the weights).  The comments give what
    the fp32 one-pass statistics (shifted by rbar, or by 0 for a NaN mean row) computed on these."""
    g = np.random.default_rng(seed)
    z = g.uniform(-np.sqrt(3.0), np.sqrt(3.0), N + 1)
    if case == "nan_mean_row_-8+-0.003":        # std exactly 0: uniform weights
        r = -8.0 + 0.003 * z
        r[-1] = np.nan
    elif case == "nan_mean_row_-30+-0.01":      # std 21 % low
        r = -30.0 + 0.01 * z
        r[-1] = np.nan
    elif case == "mean_row_1e4_spreads_below":  # std 1 % off at 2^17 rewards (the error grows with their count)
        r = -1.0 + 0.3 * z
        r[-1] = -1.0 - 1e4 * 0.3
    elif case == "nan_mean_row_+1e4+-1":        # std 0
        r = 1e4 + z
        r[-1] = np.nan
    elif case == "nan_mean_row_-1e4+-1":        # std 0
        r = -1e4 + z
        r[-1] = np.nan
    elif case == "finite_outlier_-1e20":        # fp32: d^2 overflows, std = inf, every weight equal
        r = -1.0 + 0.3 * z
        r[-1] = -1.0
        r[17] = -1e20
    return r.astype(np.float32)


ILL = ["nan_mean_row_-8+-0.003", "nan_mean_row_-30+-0.01", "mean_row_1e4_spreads_below", "nan_mean_row_+1e4+-1",
       "nan_mean_row_-1e4+-1", "finite_outlier_-1e20"]
ILL_N = {"mean_row_1e4_spreads_below": 131071}


@pytest.mark.parametrize("kernel", ["fused", "eager"])
@pytest.mark.parametrize("case", ILL)
def test_ill_conditioned_statistics_match_fp64(built, case, kernel):
    from oracle.planner_oracle import reverse_update_fp64
    N, Hn = ILL_N.get(case, 2048), 4
    plan = _plan(GO2, N, Hn)
    _, rng, Ybar, noise = _inputs(N, Hn, 12, seed=13)
    r = _ill_rewards(case, N)
    w64, Y64 = reverse_update_fp64(r, TEMP, _eps64(rng, N, Hn, 12), Ybar, noise)
    assert np.ptp(w64[np.isfinite(r)]) > 0.1 * w64.max() or case == "finite_outlier_-1e20"   # not flat
    w, Y = _fused(plan, r, rng, Ybar, noise)[:2] if kernel == "fused" else _eager(plan, r, rng, Ybar, noise)
    _check(w, Y, w64, Y64, case)
    if case == "finite_outlier_-1e20":
        assert w64[17] == 0 and w[17] == 0


# ---- d. one launch over unlike instances --------------------------------------------------------------------
def test_mixed_batch_matches_fp64_and_single_launches(built):
    from oracle.planner_oracle import reverse_update_fp64
    N, Hn, B = 2048, 4, 3
    ne = (Hn + 1) * 12
    rews, rngs, Ybars = [], [], []
    for b in range(B):
        r, k, Y, noise = _inputs(N, Hn, 12, seed=100 + b)
        if b == 1:                                   # diverged samples, a NaN mean row, one in the last CTA
            r = _guard_rewards("last_cta", r, N, ne)
            r[5], r[-1] = np.inf, np.nan
        if b == 2:
            r[:] = -0.75                             # flat
        rews.append(r); rngs.append(k); Ybars.append(Y)
    rews, rngs, Ybars = np.stack(rews), np.stack(rngs), np.stack(Ybars)
    w, Y, rng_out = _fused(_plan(GO2, N, Hn, B=B), rews, rngs, Ybars, noise)
    single = _plan(GO2, N, Hn)
    for b in range(B):
        w64, Y64 = reverse_update_fp64(rews[b], TEMP, _eps64(rngs[b], N, Hn, 12), Ybars[b], noise)
        _check(w[b], Y[b], w64, Y64, f"instance {b}")
        assert np.array_equal(rng_out[b], _split(rngs[b])[0])
        w1, Y1, k1 = _fused(single, rews[b], rngs[b], Ybars[b], noise)
        assert np.array_equal(w1, w[b]) and np.array_equal(Y1, Y[b]) and np.array_equal(k1, rng_out[b]), b


# ---- e. the sampler element by element ---------------------------------------------------------------------
# Row j's reward 0, every other -inf, the mean row NaN: one finite reward, std 0, so the flat guard puts
# the whole weight on row j.  With Ybar = 0 and noise 2^-3 on nodes > 0 (a power of two: the scaling is
# exact and |Y0s| < 1 never clips), Ybar_out * 8 is the device's eps of row j.  It is compared with the
# restatement of XLA's float32 algorithm (jax_normal_legacy_xla) to EPS_ULP fp32 ulp, and with the exact
# fp64 erfinv (jax_normal_legacy) to EPS_ULP ulp beyond the float32 algorithm's own distance from it
# (near |u| = 1 the fp32 rounding of u * u moves eps by up to ~50 ulp: tail rows, test_update_reference.py).
EPS_ULP = 4       # measured on an H100 80GB HBM3: at most 2.2 ulp


@pytest.mark.parametrize("name,Hn,N", [(GO2, 4, 2047), (H1, 4, 2047), (H1, 4, 2048)],
                         ids=["go2-ntot-even", "h1-ntot-odd", "h1-ntot-even"])
def test_sampler_rows_match_restatement(built, name, Hn, N):
    from oracle.planner_oracle import erfinv_tail_indices, jax_normal_legacy_xla
    plan = _plan(name, N, Hn)
    nu = plan.nu
    ne = (Hn + 1) * nu
    ntot = N * ne
    rng = np.uint32([0x2545F491, 0x4F6CDD1D])
    eps64 = _eps64(rng, N, Hn, nu)
    eps_xla = jax_normal_legacy_xla(tuple(int(v) for v in _split(rng)[1]), (N, Hn + 1, nu))
    half = (ntot + 1) // 2                               # the legacy layout's halves; odd ntot pads at half - 1
    tail = [i for i in erfinv_tail_indices(tuple(int(v) for v in _split(rng)[1]), ntot) if (i % ne) // nu >= 1]
    tail_rows = sorted({i // ne for i in tail})[:3]
    rows = sorted({0, N - 1, (half - 1) // ne, half // ne} | set(tail_rows))
    assert len(tail_rows) == 3
    noise = np.full(Hn + 1, 0.125, np.float32)
    noise[0] = 0.0
    worst, worst_exact = 0.0, 0.0
    for j in rows:
        r = np.full(N + 1, -np.inf, np.float32)
        r[j], r[N] = 0.0, np.nan
        w, Y, _ = _fused(plan, r, rng, np.zeros((Hn + 1, nu), np.float32), noise)
        assert w[j] == 1.0 and np.count_nonzero(w) == 1
        e_dev = Y[1:].astype(np.float64) * 8.0
        e_ref, e_xla = eps64[j, 1:], eps_xla[j, 1:]
        ulp = np.spacing(np.abs(e_ref).astype(np.float32)).astype(np.float64)
        worst = max(worst, float((np.abs(e_dev - e_xla) / ulp).max()))
        worst_exact = max(worst_exact, float(((np.abs(e_dev - e_ref) - np.abs(e_xla - e_ref)) / ulp).max()))
    print(f"sampler rows {rows}: max {worst:.2f} fp32 ulp from XLA's float32 algorithm, "
          f"{worst_exact:.2f} ulp beyond its distance from the exact erfinv")
    assert worst <= EPS_ULP and worst_exact <= EPS_ULP, (worst, worst_exact)
    for i in tail:
        if i // ne in tail_rows:
            assert abs(eps64.reshape(-1)[i]) > 2.93


# ---- f. the shift ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("Hn", [2, 3, 4, 5, 6, 7])      # Hn = 1 has no quadratic spline (3 knots at least)
def test_graph_shift_matches_fp64(built, Hn, B):
    import types
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_config import DialConfig
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    from oracle.planner_oracle import PlannerOracle
    Hs = 16
    env = _env(GO2)
    mb = MBDPI(DialConfig(env_name=GO2, Nsample=16, Hsample=Hs, Hnode=Hn, temp_sample=TEMP), env, n_instances=B)
    states = [env.reset(drandom.PRNGKey(b)) for b in range(B)]
    lead = (B,) if B > 1 else ()
    Y0 = np.random.default_rng(Hn).uniform(-1, 1, size=lead + (Hn + 1, 12)).astype(np.float32)
    rng = np.stack([drandom.PRNGKey(10 + b) for b in range(B)]) if B > 1 else drandom.PRNGKey(10)
    loop = DeviceLoop(mb, states if B > 1 else states[0], rng, Y0)
    po = PlannerOracle(types.SimpleNamespace(nu=12), 16, Hs, Hn, TEMP, 0.9, 0.5)
    for _ in range(3):                    # eager, capture, replay
        Yp = loop.Y.cpu().numpy().astype(np.float64).reshape(-1, Hn + 1, 12)
        loop.step(0, env_step=2)
        torch.cuda.synchronize()
        Yn = loop.Y.cpu().numpy().reshape(-1, Hn + 1, 12)
        for b in range(B):
            err = float(np.abs(Yn[b] - po.shift(Yp[b])).max())
            assert err <= 2e-6, (b, err)


# ---- g. the graph end to end ---------------------------------------------------------------------------------
def test_graph_last_iteration_matches_fp64(built):
    """loop1 runs step(n, env_step=False); loop2, on its own plan, starts each call from loop1's knots and
    rng and runs the first n - 1 iterations, which are bitwise those of loop1.  Its knots and rng are the
    input of loop1's last iteration, whose update (and bars) are recomputed in fp64 from loop1's rewards."""
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_config import DialConfig
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    from oracle.planner_oracle import reverse_update_fp64
    N, Hs, Hn = 2048, 25, 5
    env = _env(GO2)
    cfg = DialConfig(env_name=GO2, Nsample=N, Hsample=Hs, Hnode=Hn, Ndiffuse=4, Ndiffuse_init=4, temp_sample=TEMP)
    mb1, mb2 = MBDPI(cfg, env), MBDPI(cfg, env)
    state = env.reset(drandom.PRNGKey(0))
    rng = drandom.PRNGKey(4)
    loop1, loop2 = DeviceLoop(mb1, state, rng), DeviceLoop(mb2, state, rng)
    noise = loop1.buf["noise"].cpu().numpy()
    for n in (1, 2, 3, 4):
        for rep in range(3):              # eager, capture, replay of the shape
            loop2.buf["Y"].copy_(loop1.buf["Y"])
            loop2.buf["rng"].copy_(loop1.buf["rng"])
            if n > 1:
                loop2.step(n - 1, env_step=False)
            loop1.step(n, env_step=False)
            torch.cuda.synchronize()
            Yprev = loop2.Y.cpu().numpy()
            rprev = loop2.rng_host()
            rews = loop1.info()["rews"].cpu().numpy()
            assert np.isfinite(rews).all()
            w64, Y64 = reverse_update_fp64(rews, TEMP, _eps64(rprev, N, Hn, 12), Yprev, noise[n - 1])
            err = float(np.abs(loop1.Y.cpu().numpy() - Y64).max())
            assert err <= Y_TOL, (n, rep, err)
            assert np.array_equal(loop1.rng_host(), _split(rprev)[0]), (n, rep)
            q, qd, x = (t.cpu().numpy().astype(np.float64) for t in mb1.plan.reverse_trajectories())
            info = loop1.info()
            for key, t in (("qbar", q), ("qdbar", qd), ("xbar", x)):
                nz = w64 > 0
                ref = np.tensordot(w64[nz], t[nz], axes=1)
                got = info[key].cpu().numpy()
                tol = 1e-5 * (1 + np.abs(t[nz]).max())
                assert np.abs(got - ref).max() <= tol, (key, n, rep, float(np.abs(got - ref).max()), tol)
