"""The physics state a custom reward sees (include/dial_custom_reward.h), read out of the device code in
the CPU warp emulator through the probe reward and compared with fp64 recomputed from the emulator's own
stored states (tests/state_probe.py: the probe envs, the element order, the reference and the derivation
of the tolerances).  Every element of every probe env is read: on random-action rollouts from the initial
pose and from a lifted, tilted pose (feet far above the ground), and at t = 0 of constructed edge states:
free-joint quaternions at identity, 180 degrees and unnormalised, hinges at and beyond their ranges and
wound past 2 pi, spheres touching and penetrating the plane, capsules standing on their axis, Allegro's
fingers near parallel, coincident sphere centres.  The same checks run on an H100 in
tests/test_gpu_state_probe.py."""
import numpy as np
import pytest

from tests import state_probe as sp

H = 24


def _launcher(env):
    return lambda q0, qd0, us, u0, u1: sp.emul_launch(env, q0, qd0, us, u0, u1)


def _start(env):
    return np.asarray(env._init_q, np.float32), np.zeros(env.sys.nv, np.float32)


def test_probe_envs_cover_every_pair_kind_and_variant():
    """Every contact pair kind the kernel implements (its PAIR_* enum, the same as the oracle's) is in some probe
    env; each stock model picks the solver variant its stock plan launches."""
    from dial_mpc_b200 import _capi, custom
    kinds = set()
    for name in sp.NAMES:
        env, om = sp.make_probe(name)
        kinds |= set(int(k) for k in om.pair_kind)
        v, nvd = sp.variant_of(name)
        assert custom.solver_variant(env.sys.model) == v, name
        assert custom.dense_nv(env.sys.model) == nvd, name
        if name in ("go2", "h1_walk", "h1_loco", "allegro"):     # the stock library's own pick
            assert _capi.lib().dial_solver_variant(_capi.fill_model_desc(env.sys.model)) == v, name
    assert sp.kernel_pair_kinds() == {v: k for k, v in sp.PAIR_NAMES.items()}
    assert kinds == set(sp.kernel_pair_kinds().values()), kinds


def test_layout_matches_probe_order():
    """The Python layout has E elements, the world body first among the bodies."""
    env, om = sp.make_probe("quadpod")
    lay = sp.layout(om)
    assert len(lay) == sp.n_elements(om)
    assert lay[om.nq + om.nv] == ("xpos", 0, 0)
    assert lay[-1] == ("site_xpos", om.nsite - 1, 2)


@pytest.mark.parametrize("name", sp.NAMES)
def test_every_element_matches_fp64(name):
    """Every element, read once on a random-action rollout from the initial pose, and a third of them from a lifted
    pose; each field of the contract the model has is compared."""
    env, om = sp.make_probe(name)
    E = sp.n_elements(om)
    launch = _launcher(env)
    q0, qd0 = _start(env)
    worst, seen = sp.run_checks(om, launch, q0, qd0, sp.actions(env, 1, H, 1), sp.sweep_starts(E, H, 1), False,
                                f"{name} reset")
    assert seen == set(range(E))
    ql, qdl = sp.lifted(env, 0.4, 2)
    _, seen2 = sp.run_checks(om, launch, ql, qdl, sp.actions(env, 1, H, 2), sp.sweep_starts(E, H, 1)[::3], False,
                             f"{name} lifted", worst)
    assert set(worst) == sp.fields_of(om), set(worst) ^ sp.fields_of(om)
    print(name, {k: round(v, 4) for k, v in sorted(worst.items())})


def _edge_run(name, states, worst, elems=None):
    env, om = sp.make_probe(name)
    launch = _launcher(env)
    rng = np.random.default_rng(7)
    for label, q, qd in states:
        us = sp.actions(env, 1, 2, 3)
        el = elems if elems is not None else sp.edge_elements(om, rng)
        sp.run_checks(om, launch, np.asarray(q, np.float32), np.asarray(qd, np.float32), us, el, False,
                      f"{name} {label}", worst)


@pytest.mark.parametrize("name", ["go2", "quadpod", "h1_walk", "h1_loco", "allegro", "pincher", "spheres", "hexapod",
                                  "longchain"])
def test_edge_states_match_fp64(name):
    env, om = sp.make_probe(name)
    states = sp.edge_states(name, env, om)
    z = np.zeros(om.nv)
    for kind in (0, 1):
        for depth in (0.0, 0.03):
            q = sp.touching(env, om, kind, depth)
            if q is not None:
                states.append((f"{sp.PAIR_NAMES[kind]} at depth {depth}", q, z))
    p = sp.pitched(env)
    if p is not None:
        states.append(("root pitched 90 deg", p, z))
    if name == "allegro":       # the emulator's dense nv = 22 step is slow: the near-parallel fingers only
        q = np.asarray(env._init_q, np.float64).copy()
        q[7:] = 0.0
        states = [("fingers straight", q, z), ("initial pose", np.asarray(env._init_q, np.float64), z)]
        assert sp.cc_conditioning(om, np.stack([s[1] for s in states])) < 1e-3
    worst = {}
    _edge_run(name, states, worst)
    print(name, "edges", {k: round(v, 4) for k, v in sorted(worst.items())})


def test_coincident_sphere_centres_take_the_fallback_normal():
    """spheres.xml: the ball centred on a tip sphere (|q2 - q1| = 0 exactly): the contact takes the fallback
    normal (1, 0, 0), so contact_pos = q1 + (r1 - r2) / 2 x, and every contact element matches fp64."""
    env, om = sp.make_probe("spheres")
    q = sp.coincident_spheres(env)
    lay = sp.layout(om)
    el = [i for i, f in enumerate(lay) if f[0] in ("contact_dist", "contact_pos")]
    worst = {}
    _edge_run("spheres", [("coincident centres", q, np.zeros(om.nv))], worst, el)
    from oracle import mjx_oracle as mo
    d, pos, _ = mo.collision(om, *mo.kinematics(om, q[None])[1:4:2])
    k = [c for c in range(om.ncon) if om.pair_kind[om.con_pair[c]] == mo.PAIR_SPHERE_SPHERE and d[0, c] == -0.0325]
    assert k and np.allclose(pos[0, k[0]] - q[:3], [0.00375, 0, 0])
    print("coincident", worst)
