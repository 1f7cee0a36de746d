"""The physics state a custom reward sees (include/dial_custom_reward.h), read out of the rollout kernel
exactly through the probe reward and compared with fp64 recomputed from the kernel's own stored states
(tests/state_probe.py: the probe envs on every solver variant and pair kind, the element order, the
reference and the derivation of the tolerances, here with the SFU's sin / cos error;
tests/test_state_probe.py runs the same checks in the CPU warp emulator).

Explicit-action rollouts through the default launch policy, H steps per launch:
  a. from the initial pose, ROWS = 301 rows: several warps per CTA and a padded last CTA (asserted), user[0]
     swept so that every element is read on every row;
  b. from a mid-rollout state (MID steps of random actions), MID_ROWS = 133 rows (two warps per CTA, the last
     CTA padded), user[1] a stride coprime with E, so every element is read again, at other steps;
  c. from a lifted, tilted pose (feet far above the ground), MID_ROWS rows, a quarter of the launches of (a);
  d. constructed edge states (tests/state_probe.py: edge_states, touching, pitched, coincident spheres,
     Allegro's straight fingers), read at t = 0 on 6 rows of 4-warp CTAs (DIAL_WPC = 4, the second CTA padded).
At the envs' real n_frames (Allegro, pincher: 4 substeps) the reward's qpos / qvel equal the stored state bit
for bit.

Largest |err| / tol per field measured on an H100 80GB HBM3 (the ``state probe`` lines):
  env        variant        kinematics (xpos xquat xmat)   velocities (xd_ang xd_vel)   contacts (dist pos)   sites
  go2        v1 star<3,6>   0.115 0.109 0.131              0.146 0.063                  0.027 0.022           0.215
  quadpod    v1             0.112 0.111 0.124              0.160 0.088                  0.040 0.033           0.168
  slidepod   v1             0.116 0.113 0.138              0.127 0.094                  0.075 0.045           0.118
  h1_walk    v2 star<5,7>   0.105 0.110 0.134              0.132 0.105                  0.041 0.033           0.062
  h1_loco    v4 star<5,6>   0.105 0.111 0.141              0.120 0.060                  0.042 0.036           0.052
  allegro    v3 dense 22    0.088 0.087 0.134              0.128 0.099                  0.142 0.054           -
  pincher    v3 dense 10    0.069 0.120 0.135              0.147 0.028                  0.130 0.192           -
  spheres    v3 dense 10    0.062 0.116 0.138              0.144 0.025                  0.099 0.062           0.056
  branchpod  v0 tree        0.119 0.110 0.143              0.117 0.101                  0.070 0.044           0.142
  hexapod    v0 tree        0.118 0.117 0.135              0.123 0.077                  0.060 0.040           0.124
  longchain  v0 tree        0.110 0.105 0.131              0.117 0.098                  0.047 0.039           0.145
qpos / qvel: bitwise everywhere."""
import json

import numpy as np
import pytest
import torch

from tests import state_probe as sp

pytestmark = pytest.mark.gpu
ROWS, MID_ROWS, H, MID = 301, 133, 32, 160
EDGE_ROWS, EDGE_WPC = 6, 4


def _launcher(env, check_rows=None):
    """launch(q0, qd0, us, u0, u1) -> (rewss, q, qd) of one Plan.rollout; ``check_rows``: assert that a launch of
    that many rows has several warps per CTA and a padded last CTA under the launch policy."""
    from dial_mpc_b200.envs.base_env import PipelineState, State
    from dial_mpc_b200.plan import Plan

    def launch(q0, qd0, us, u0, u1):
        e = env.probed(u0, u1)
        plan = Plan(e, e.plan_desc())
        n = us.shape[0]
        if n == check_rows:
            wpc = plan.lib.dial_rollout_wpc(plan.handle, n)
            assert wpc > 1 and n % wpc != 0, (n, wpc)
        ps = PipelineState(plan.f32(q0), plan.f32(qd0), plan.f32(np.zeros(len(qd0))))
        rewss, q, qd, _ = plan.rollout(State(ps, None, 0.0, 0.0, {}, {"step": 0}), us)
        torch.cuda.synchronize()
        return rewss.cpu().numpy(), q.cpu().numpy(), qd.cpu().numpy()
    return launch


@pytest.mark.parametrize("name", sp.NAMES)
def test_every_element_matches_fp64(built, monkeypatch, name):
    env, om = sp.make_probe(name)
    assert env.library_path
    E = sp.n_elements(om)
    q0, qd0 = np.asarray(env._init_q, np.float32), np.zeros(om.nv, np.float32)
    # a. every element on every row of a multi-warp launch with a padded last CTA
    worst, seen = sp.run_checks(om, _launcher(env, ROWS), q0, qd0, sp.actions(env, ROWS, H, 1), sp.sweep_starts(E, H),
                                True, f"{name} reset")
    assert seen == set(range(E))
    # b. every element again from a mid-rollout state, at other steps
    qm, qdm = sp.preroll(_launcher(env), env, q0, qd0, MID, 5)
    u1 = sp.sweep_stride(E, (7,))
    _, seen = sp.run_checks(om, _launcher(env, MID_ROWS), qm, qdm, sp.actions(env, MID_ROWS, H, 6),
                            sp.sweep_starts(E, H, u1), True, f"{name} mid-rollout", worst, u1=u1)
    assert seen == set(range(E))
    # c. feet far above the ground
    ql, qdl = sp.lifted(env, 0.4, 2)
    sp.run_checks(om, _launcher(env, MID_ROWS), ql, qdl, sp.actions(env, MID_ROWS, H, 2), sp.sweep_starts(E, H)[::4],
                  True, f"{name} lifted", worst)
    assert set(worst) == sp.fields_of(om)
    # d. edge states at t = 0, on multi-warp CTAs
    monkeypatch.setenv("DIAL_WPC", str(EDGE_WPC))
    assert EDGE_ROWS % EDGE_WPC != 0
    rng = np.random.default_rng(7)
    states = sp.edge_states(name, env, om)
    for kind in (0, 1):
        for depth in (0.0, 0.03):
            q = sp.touching(env, om, kind, depth)
            if q is not None:
                states.append((f"{sp.PAIR_NAMES[kind]} at depth {depth}", q, np.zeros(om.nv)))
    if sp.pitched(env) is not None:
        states.append(("root pitched 90 deg", sp.pitched(env), np.zeros(om.nv)))
    if name == "spheres":
        states.append(("coincident centres", sp.coincident_spheres(env), np.zeros(om.nv)))
    if name == "allegro":
        q = np.asarray(env._init_q, np.float64).copy()
        q[7:] = 0.0
        states.append(("fingers straight", q, np.zeros(om.nv)))
        assert sp.cc_conditioning(om, np.stack([s[1] for s in states])) < 1e-3
    for label, q, qd in states:
        sp.run_checks(om, _launcher(env), np.asarray(q, np.float32), np.asarray(qd, np.float32),
                      sp.actions(env, EDGE_ROWS, 2, 3), sp.edge_elements(om, rng, 40), True, f"{name} {label}", worst)
    print("state probe", json.dumps(dict(env=name, variant=sp.variant_of(name)[0],
                                         worst={k: round(v, 4) for k, v in sorted(worst.items())})))


@pytest.mark.parametrize("name", ["allegro", "pincher", "quadpod"])
def test_reward_state_is_the_stored_state_at_real_n_frames(built, name):
    """dt = 0.02 (Allegro, pincher: four physics substeps): every qpos / qvel element the reward reads equals
    the stored q[t] / qd[t] bit for bit."""
    env, om = sp.make_probe(name, **({} if name == "quadpod" else dict(dt=0.02)))
    assert env._n_frames == (1 if name == "quadpod" else 4)
    n = om.nq + om.nv
    launch = _launcher(env)
    q0, qd0 = np.asarray(env._init_q, np.float32), np.zeros(om.nv, np.float32)
    for u0 in range(0, n, 8):
        rewss, q, qd = launch(q0, qd0, sp.actions(env, ROWS, 8, 4), u0, 1)
        post = np.concatenate([q, qd], -1)
        for t in range(8):
            e = (u0 + t) % sp.n_elements(om)
            if e < n:
                assert np.array_equal(rewss[:, t], post[:, t, e]), (name, t, e)
