"""The generic tree solver (variant 0) and slide joints on the GPU: the real custom builds of the tree
fixtures (tests/tree_envs.py; variant 0 for branchpod, hexapod and longchain, the quadpod example's
star<3,6> build for slidepod) against the fp64 oracle.

* single physics steps from >= 120 mid-rollout oracle states per fixture, with the Go2 tolerances
  (tests/test_tree_models.py calibrates them on the emulator);
* explicit-action rollouts through the default launch policy at a size with several CTAs and a padded
  last CTA, and at a two-wave size, with the budgets and the shadowing check of tests/test_gpu_at_size.py;
  the same rows bitwise equal under DIAL_WPC=1 and DIAL_WPC=16;
* a batched DeviceLoop of three hexapod instances, one with a heavier torso, bitwise equal to single loops;
* one reverse_once on branchpod against the oracle planner fed the same Threefry noise.
The measured errors are written as tree_*.json reports by tests/test_gpu_at_size.py's _report."""
import os

import numpy as np
import pytest
import torch

from tests.test_gpu_at_size import YARD, _report
from tests.test_tree_models import NAMES, SINGLE_TOL, pair, single_step_errors, single_step_states

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", NAMES)
def test_gpu_single_steps_match_oracle(built, name):
    from dial_mpc_b200.envs.base_env import PipelineState, State
    env, o, (Q, V, W, A), ns, con, lim = single_step_states(name, 12, 10, 3)
    assert len(Q) >= 120 and con.any(-1).sum() >= 60 and lim.sum() >= 1
    plan = env._get_plan()
    rows = []
    for i in range(len(Q)):
        st = State(PipelineState(plan.f32(Q[i]), plan.f32(V[i]), plan.f32(W[i])), None, 0.0, 0.0, {}, {"step": 0})
        ps, _ = plan.env_step(st, A[i])
        rows.append(tuple(t.cpu().numpy().astype(np.float64) for t in (ps.qpos, ps.qvel, ps.qacc_warmstart)))
    rep, ok = single_step_errors(rows, ns)
    rep.update(env=name, in_contact=int(con.any(-1).sum()), at_limit=int(lim.sum()), tolerances=SINGLE_TOL)
    _report(f"tree_single_step_{name}", rep)
    assert ok, rep


def _oracle_rows(o, q0, v0, w0, step, us, rng, K=3, scale=1e-5):
    """The oracle's rollout of the rows of ``us`` from one state (rewss, q, qd, xpos, warm-start per step)
    and its own sensitivity to fp32-sized noise: the max over K re-runs with the actions perturbed by
    ``scale``*N(0,1) (tests/oracle_pool.py's yardstick without the C port, which knows no custom reward)."""
    from oracle.envs_oracle import OState
    n = us.shape[0]
    stack = np.concatenate([us] + [us + scale * rng.standard_normal(us.shape) for _ in range(K)], 0)
    s = OState(q0[None], v0[None], w0[None], np.array([step]), np.array([0])).tile(len(stack))
    out = [[] for _ in range(5)]
    for t in range(us.shape[1]):
        s, r, aux = o.step(s, stack[:, t])
        for lst, a in zip(out, (r, aux["q"], aux["qd"], aux["xpos"], s.qacc_warmstart.copy())):
            lst.append(a)
    out = [np.stack(a, 1) for a in out]
    nom = tuple(a[:n] for a in out)
    sens = tuple(np.max([np.abs(a[(k + 1) * n:(k + 2) * n] - a[:n]) for k in range(K)], 0) for a in out[:4])
    return nom, sens


def _start_state(env):
    """reset, then 5 env steps with zero action (the GPU's own state)."""
    from dial_mpc_b200 import random as drandom
    st = env.reset(drandom.PRNGKey(0))
    for _ in range(5):
        st = env.step(st, torch.zeros(env.action_size, device="cuda"))
    return st


def _launch(plan, st, us, wpc=None):
    old = os.environ.get("DIAL_WPC")
    if wpc is not None:
        os.environ["DIAL_WPC"] = str(wpc)
    try:
        out = plan.rollout(st, us)
        torch.cuda.synchronize()
    finally:
        if wpc is not None:
            if old is None:
                del os.environ["DIAL_WPC"]
            else:
                os.environ["DIAL_WPC"] = old
    return out


# rows of the launch: 301 = several CTAs with a padded last one; 4001 = more rows than one wave holds
@pytest.mark.parametrize("nrows", [301, 4001])
@pytest.mark.parametrize("name", NAMES)
def test_gpu_rollouts_at_size(built, name, nrows):
    from dial_mpc_b200.core.dial_config import DialConfig
    from dial_mpc_b200.core.dial_core import MBDPI
    from dial_mpc_b200.envs.base_env import PipelineState, State
    env, o = pair(name)
    Hs = 8
    mb = MBDPI(DialConfig(env_name="tree_" + name, Nsample=nrows - 1, Hsample=Hs, Hnode=4, temp_sample=0.05), env)
    plan = mb.plan
    st = _start_state(env)
    rng = np.random.default_rng(20 + nrows)
    us = np.clip(rng.normal(size=(nrows, Hs + 1, env.action_size)) * 0.6, -1, 1).astype(np.float32)
    got = [t.cpu().numpy() for t in _launch(plan, st, us)]
    # launch-shape independence: one warp per CTA, 16 warps per CTA (16 of the hexapod's 14 KB slabs exceed shared memory:
    # 16 is refused, the refusal must not fail the next launch, and the widest width of the launch policy is used)
    wpc = plan.lib.dial_rollout_wpc(plan.handle, nrows)
    if nrows == 301:
        widths = (1, 16)
        if name == "hexapod":
            with pytest.raises(RuntimeError, match="invalid argument"):
                _launch(plan, st, us, wpc=16)
            widths = (1, plan.lib.dial_rollout_wpc(plan.handle, 10 ** 6))
            assert widths[1] >= 12, widths
        for w in widths:
            other = [t.cpu().numpy() for t in _launch(plan, st, us, wpc=w)]
            assert all(np.array_equal(a, b) for a, b in zip(got, other)), (w, wpc)
    else:
        assert nrows > wpc * torch.cuda.get_device_properties(0).multi_processor_count   # two waves
    assert nrows % wpc != 0                                                              # a padded last CTA
    rg, qg, qdg, xg = (a.astype(np.float64) for a in got)
    assert np.isfinite(rg).all()
    last_cta = np.arange((nrows // wpc) * wpc, nrows)
    rows = np.unique(np.concatenate([rng.choice(nrows, 40, replace=False), [0, nrows - 2, nrows - 1], last_cta]))
    ps = st.pipeline_state
    sq, sv, sw = (t.cpu().numpy().astype(np.float64) for t in (ps.qpos, ps.qvel, ps.qacc_warmstart))
    step = int(st.info["step"])
    u = us[rows].astype(np.float64)
    (ro, qo, qdo, xo, wo), (rs, qs, qds, xs) = _oracle_rows(o, sq, sv, sw, step, u, rng)
    n = len(rows)
    rep = dict(env=name, rows_launched=nrows, wpc=wpc, rows_checked=n)
    over_rows, first_over, tight = np.zeros(n, bool), np.full(n, 10 ** 6), np.ones(n, bool)
    for key, g, on, op, tol, rel in (("rewss", rg[rows], ro, rs, 2e-3, True), ("q", qg[rows], qo, qs, 2e-4, False),
                                      ("qd", qdg[rows], qdo, qds, 1e-2, False), ("xpos", xg[rows], xo, xs, 2e-4, False)):
        base = tol * (1 + np.abs(on)) if rel else tol
        e = np.abs(g - on)
        over = (e > base + YARD * op).reshape(n, e.shape[1], -1).any(-1)
        tight &= ~(e > base).reshape(n, -1).any(-1)
        over_rows |= over.any(1)
        first_over = np.minimum(first_over, np.where(over.any(1), np.argmax(over, 1), 10 ** 6))
        rep[key] = dict(err_max=float(e.max()), frac_within_tolerance=float((e <= base).mean()), rows_over_budget=int(over.any(1).sum()))
    # shadowing: a row over its budget restarts from the oracle's own state one step before it left the budget
    shadow = []
    for i in np.nonzero(over_rows)[0]:
        t = int(first_over[i])
        q0, v0, w0 = (sq, sv, sw) if t == 0 else (qo[i, t - 1], qdo[i, t - 1], wo[i, t - 1])
        st0 = State(PipelineState(plan.f32(q0), plan.f32(v0), plan.f32(w0)), None, 0.0, 0.0, {}, {"step": step + t})
        ps1, r1 = plan.env_step(st0, u[i, t])
        eq1 = float(np.abs(ps1.qpos.cpu().numpy() - qo[i, t]).max())
        ev1 = float((np.abs(ps1.qvel.cpu().numpy() - qdo[i, t]) / (1 + np.abs(qdo[i, t]))).max())
        er1 = float(abs(float(r1) - ro[i, t]) / (1 + abs(ro[i, t])))
        shadow.append(dict(row=int(rows[i]), step=t, q_err=eq1, qvel_relerr=ev1, rew_relerr=er1,
                           ok=bool(eq1 < 5e-5 and ev1 < 1e-3 and er1 < 1e-3)))
    rep.update(rows_within_tolerance=float(tight.mean()), shadowing=shadow)
    _report(f"tree_rollout_{name}_{nrows}", rep)
    assert all(s["ok"] for s in shadow), rep
    assert tight.mean() >= 0.95, rep


def test_gpu_batched_hexapod_instances(built):
    """Per-instance models on the generic tree solver: a batched loop of three hexapods, the second with a
    torso 1.5 kg heavier, == single loops on each model at every step of SCHEDULE."""
    from tests.test_gpu_instance_models import _check_models, _with_sys
    env, _ = pair("hexapod")
    heavy = _with_sys(env, {"body_mass": {"torso": env.sys.model.arrays["body_mass"][1] + 1.5}})
    _, refs, _ = _check_models("tree_hexapod", [env, heavy, env], 64, 8, 4, base=env)
    assert not torch.equal(refs[1][-1]["Y"], refs[0][-1]["Y"])          # the heavier torso was read


def test_gpu_planner_matches_oracle_on_branchpod(built):
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_config import DialConfig
    from dial_mpc_b200.core.dial_core import MBDPI
    from oracle.planner_oracle import PlannerOracle, jax_normal_legacy
    env, o = pair("branchpod")
    s = o.reset()
    state = env.reset(drandom.PRNGKey(0))
    np.testing.assert_allclose(state.pipeline_state.qpos.cpu().numpy(), s.qpos[0], atol=1e-6)
    N, Hs, Hn = 64, 12, 4
    args = DialConfig(env_name="tree_branchpod", Nsample=N, Hsample=Hs, Hnode=Hn, Ndiffuse=1, temp_sample=0.05,
                      horizon_diffuse_factor=0.9, traj_diffuse_factor=0.5)
    mb = MBDPI(args, env)
    assert mb.plan.lib.dial_plan_rollout_kernel(mb.plan.handle) == b"v0"
    pl = PlannerOracle(o, N, Hs, Hn, 0.05, 0.9, 0.5)
    key = drandom.PRNGKey(7)
    _, k2 = drandom.split(key)
    eps = jax_normal_legacy(tuple(int(v) for v in k2), (N, Hn + 1, env.action_size))
    Yo, info_o = pl.reverse_once(s, eps, np.zeros((Hn + 1, env.action_size)), pl.sigma_control)
    _, Y, info = mb.reverse_once(state, key, torch.zeros(Hn + 1, env.action_size, device="cuda"),
                                 torch.as_tensor(pl.sigma_control, dtype=torch.float32, device="cuda"))
    r = info["rews"].cpu().numpy()
    ok = np.abs(r - info_o["rews"]) < 2e-3 * (1 + np.abs(info_o["rews"]))
    assert ok.mean() > 0.97, (ok.mean(), np.abs(r - info_o["rews"]).max())
    assert np.abs(Y.cpu().numpy() - Yo).max() < 5e-3
