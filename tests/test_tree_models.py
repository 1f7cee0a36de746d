"""The generic tree solver (variant 0, the level-scheduled compact Cholesky) and slide joints on models
that are not stars: CPU tests.

Fixtures (tests/models/trees/, envs in tests/tree_envs.py):
  branchpod  a knee dof with two child dofs (a hinge toe and a slide toe)      variant 0
  hexapod    six leaves + a neck; nu = DIAL_MAXU, 32 pyramid edges, 8 geoms  variant 0
  longchain  a 12-dof ancestor chain (DIAL_MAXCHAIN, 12 levels), a slide     variant 0
  slidepod   slide knees on the star<3,6> path                               variant 1

The fp64 oracle is first checked for self-consistency on each of them (it is the yardstick), then the
device code, compiled by g++ and run by the warp emulator, against the oracle; then the structural
rejections of modelc and of the host model derivation, and the nvcc cross-compile of the variant-0
custom build."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.emul import emul
from tests.tree_envs import FIXTURES, REWARD, make_tree_pair
from tests import test_oracle_physics as oph

NAMES = list(FIXTURES)
GENERIC = ["branchpod", "hexapod", "longchain"]
EXPECT = {   # nv, nu, ncon, ngeom, nbody, (variant, s_on, sb_on)
    "branchpod": (18, 12, 6, 7, 14, (0, 0, 0)),
    "hexapod": (26, 20, 8, 8, 22, (0, 0, 0)),
    "longchain": (20, 14, 5, 6, 16, (0, 0, 0)),
    "slidepod": (14, 8, 4, 5, 10, (1, 1, 1)),
}
JNT_SLIDE = 2
_PAIRS = {}


def pair(name):
    if name not in _PAIRS:
        _PAIRS[name] = make_tree_pair(name)
    return _PAIRS[name]


def _flags(model):
    from dial_mpc_b200 import _capi
    out = (C.c_int * 4)()
    assert emul.build().emul_model_flags(C.byref(_capi.fill_model_desc(model)), out) == 0
    return tuple(out[:3])


def _chain_len(model, d):
    p, n = model.arrays["dof_parentid"], 0
    while d >= 0:
        d, n = int(p[d]), n + 1
    return n


@pytest.mark.parametrize("name", NAMES)
def test_fixture_structure(name, built):
    """The fixtures keep the shapes they are there to cover, and their solver variant: a change to the
    star selection cannot move them silently off the generic solver."""
    from dial_mpc_b200 import _capi
    env, o = pair(name)
    m = env.sys.model
    nv, nu, ncon, ngeom, nbody, flags = EXPECT[name]
    assert (m.nv, m.nu, m.ncon, m.ngeom, m.nbody) == (nv, nu, ncon, ngeom, nbody)
    assert _flags(m) == flags
    assert _capi.lib().dial_solver_variant(_capi.fill_model_desc(m)) == flags[0]
    assert env.action_size == nu and o.m.ncon == ncon and not o.m.elliptic
    A = m.arrays
    slide = A["jnt_type"] == JNT_SLIDE
    kids = np.bincount(A["dof_parentid"][A["dof_parentid"] >= 0], minlength=nv)
    longest = max(_chain_len(m, d) for d in range(nv))
    if name == "branchpod":
        assert slide.sum() == 2 and kids[6:].max() == 2            # a knee dof with two child dofs
    elif name == "hexapod":
        D = _capi.DEFINES
        leaves = int((kids == 0).sum())
        assert leaves == 7 and nu == D["DIAL_MAXU"] and ngeom == D["DIAL_MAXG"] and 4 * ncon == 32
        from dial_mpc_b200.modelc.mjcf import PAIR_PLANE_CAPSULE
        assert (A["pair_kind"] == PAIR_PLANE_CAPSULE).sum() == 1 and A["pair_ncon"].max() == 2     # the belly
    elif name == "longchain":
        assert slide.sum() == 1 and longest == 12                  # DIAL_MAXCHAIN: 12 dofs, 12 elimination levels
        assert _chain_len(m, nv - 1) == 12 and A["jnt_type"][A["dof_jntid"][nv - 4]] == JNT_SLIDE
    else:
        assert slide.sum() == 4 and longest == 8


# ---------------------------------------------------------------------------------------------
# the oracle on these trees: the invariants of tests/test_oracle_physics.py
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model_json(tmp_path_factory):
    """name -> (model file, the same model without joint limits)"""
    d = tmp_path_factory.mktemp("trees")
    paths = {}
    for n in NAMES:
        m = pair(n)[0].sys.model
        paths[n] = (str(d / (n + ".json")), str(d / (n + "_free.json")))
        m.save(paths[n][0])
        free = m.replace({})
        free.arrays["jnt_limited"] = np.zeros_like(m.arrays["jnt_limited"])
        free.save(paths[n][1])
    return paths


@pytest.mark.parametrize("check", ["test_crb_mass_matrix_equals_jacobian_form", "test_free_fall_and_momentum",
                                   "test_energy_conservation_without_dissipation", "test_gravity_bias_is_potential_gradient",
                                   "test_contact_jacobian_matches_finite_difference"])
@pytest.mark.parametrize("name", NAMES)
def test_oracle_physics_invariants(name, check, model_json):
    """CRB M(q) = the Jacobian form, free fall of the COM, energy without dissipation, gravity bias =
    dV/dq and contact Jacobian = finite differences: slide joints and branching trees included.  The
    free-fall and energy checks run without joint limits: their random postures (0.2 rad of noise) put the
    short slide ranges out of limit, and the soft limit rows then dissipate energy and, through their
    large accelerations over one step, bend the finite-difference COM velocity."""
    plain, free = model_json[name]
    no_limits = check in ("test_free_fall_and_momentum", "test_energy_conservation_without_dissipation")
    getattr(oph, check)(free if no_limits else plain)       # an absolute path: os.path.join keeps it


# ---------------------------------------------------------------------------------------------
# the device code (warp emulator) against the oracle
# ---------------------------------------------------------------------------------------------
def _active(o, d, qpos):
    """(contacts active [B, ncon], joint limits active [B]) of oracle data after a step."""
    r = o.m.jnt_range[1:]
    lim = o.m.jnt_limited[1:].astype(bool)
    q = qpos[:, 7:]
    return d.con_dist < 0, (((q < r[:, 0]) | (q > r[:, 1])) & lim).any(-1)


@pytest.mark.parametrize("name", NAMES)
def test_emulated_rollout_matches_oracle(name):
    env, o = pair(name)
    s = o.reset()
    s.step[:] = 20
    rng = np.random.default_rng(3)
    us = np.clip(rng.normal(size=(3, 12, env.action_size)) * 0.6, -1, 1)
    rew, q, qd, x = o.rollout(s, us)
    out = emul.rollout(env, env.plan_desc(), s.qpos[0], s.qvel[0], s.qacc_warmstart[0], us=us, step0=20)
    assert np.abs(out["q"] - q).max() < 1e-4
    assert np.abs(out["qd"] - qd).max() < 5e-3
    assert np.abs(out["xpos"] - x).max() < 1e-4
    assert np.abs(out["rewss"] - rew).max() < 1e-3 * (1 + np.abs(rew).max())
    assert np.abs(rew).max() > 1e-3


def _random_state(o, s0, rng, dz):
    nv, nu = o.m.nv, o.m.nu
    q = s0.qpos[0].copy()
    q[2] += dz
    ax = rng.normal(size=3)
    ax /= np.linalg.norm(ax)
    ang = rng.uniform(0, 0.4)
    q[3:7] = [np.cos(ang / 2), *(np.sin(ang / 2) * ax)]
    lo, hi = o.physical_joint_range[:, 0], o.physical_joint_range[:, 1]
    over = np.where(hi - lo > 0.5, 0.05, 0.005)
    q[7:7 + nu] = np.clip(q[7:7 + nu] + rng.normal(size=nu) * 0.4 * (hi - lo), lo - over, hi + over)
    v = rng.normal(size=nv) * np.r_[np.ones(3) * 0.5, np.ones(3), np.ones(nv - 6) * 3.0]
    return q, v


@pytest.mark.parametrize("name", NAMES)
def test_emulated_random_states_match_oracle(name):
    """Tilted base, heights in and out of contact, joints beyond their limits (0.05 rad on hinges,
    5 mm on the short slide ranges), joint rates of tens of rad/s."""
    from oracle.envs_oracle import OState
    env, o = pair(name)
    s0 = o.reset()
    rng = np.random.default_rng(11)
    n_act, n_lim, all_con = 0, 0, False
    for k in range(6):
        q, v = _random_state(o, s0, rng, dz=[-0.04, -0.02, -0.01, 0.0, 0.03, 0.1][k])
        if k == 0:      # level and 4 cm into the floor, joints at home: every contact
            q[3:] = s0.qpos[0][3:]
        st = OState(q[None], v[None], np.zeros((1, o.m.nv)), np.array([17]), np.array([0]))
        us = np.clip(rng.normal(size=(1, 3, o.nu)), -1, 1)
        ns, _, aux = o.step(st, us[:, 0])
        con, lim = _active(o, aux["data"], q[None])
        n_act, n_lim, all_con = n_act + con.any(), n_lim + lim.sum(), all_con or con.all()
        rew, qq, qd, x = o.rollout(st, us)
        out = emul.rollout(env, env.plan_desc(), q, v, np.zeros(o.m.nv), us=us, step0=17)
        assert np.abs(out["q"] - qq).max() < 5e-5
        assert np.abs(out["qd"] - qd).max() < 2e-3 * (1 + np.abs(qd).max() / 10)
        assert np.abs(out["rewss"] - rew).max() < 1e-4 * (1 + np.abs(rew).max())
    assert n_act >= 3 and n_lim >= 3, (n_act, n_lim)      # contact rows and limit rows were exercised
    if name == "hexapod":
        assert all_con                                      # all 8 contacts (32 edge rows) at once


def single_step_states(name, n_traj, n_step, seed):
    """Mid-rollout oracle states under random actions, and the oracle's step from each:
    (env, oracle, (Q, V, W, A), next state, contacts active [n, ncon], limits active [n]).  Half the
    rollouts start from home, half from random states (joints beyond their limits, rates)."""
    from oracle.envs_oracle import OState
    env, o = pair(name)
    rng = np.random.default_rng(seed)
    s = o.reset().tile(n_traj)
    for i in range(n_traj // 2, n_traj):
        s.qpos[i], s.qvel[i] = _random_state(o, o.reset(), rng, dz=rng.uniform(-0.01, 0.03))
    Q, V, W, A = [], [], [], []
    for _ in range(n_step):
        a = np.clip(rng.normal(size=(n_traj, o.nu)) * 0.7, -1, 1)
        Q.append(s.qpos.copy()); V.append(s.qvel.copy()); W.append(s.qacc_warmstart.copy()); A.append(a)
        s, _, _ = o.step(s, a)
    Q, V, W, A = (np.concatenate(x, 0) for x in (Q, V, W, A))
    ns, _, aux = o.step(OState(Q, V, W, np.zeros(len(Q), dtype=np.int64), np.zeros(len(Q), dtype=np.int64)), A)
    con, lim = _active(o, aux["data"], ns.qpos)
    return env, o, (Q, V, W, A), ns, con, lim


# One mjx.step from identical (qpos, qvel, ctrl, qacc_warmstart): the tolerances of the Go2 single-step
# test (tests/test_gpu_at_size.py), qacc relative to 1 + |qacc|.
SINGLE_TOL = dict(q=2e-5, v=3e-4, a=2e-3, frac_1e4=0.8)


def single_step_errors(rows, ns):
    """rows: (qpos, qvel, qacc) after one step per state -> (report, pass)."""
    eq = np.array([np.abs(r[0] - ns.qpos[i]) for i, r in enumerate(rows)])
    ev = np.array([np.abs(r[1] - ns.qvel[i]) / (1 + np.abs(ns.qvel[i])) for i, r in enumerate(rows)])
    ea = np.array([np.abs(r[2] - ns.qacc_warmstart[i]) / (1 + np.abs(ns.qacc_warmstart[i])) for i, r in enumerate(rows)])
    rep = dict(states=len(rows), qpos_err_max=float(eq.max()), qvel_relerr_max=float(ev.max()),
               qacc_relerr_max=float(ea.max()), qacc_within_1e4=float((ea.max(1) <= 1e-4).mean()),
               qacc_abs_max=float(np.abs(ns.qacc_warmstart).max()))
    t = SINGLE_TOL
    ok = eq.max() < t["q"] and ev.max() < t["v"] and ea.max() < t["a"] and rep["qacc_within_1e4"] >= t["frac_1e4"]
    return rep, ok


@pytest.mark.parametrize("name", NAMES)
def test_emulated_single_steps_match_oracle(name):
    env, o, (Q, V, W, A), ns, con, lim = single_step_states(name, 6, 8, 5)
    assert len(Q) >= 48 and con.any(-1).sum() >= 24 and lim.sum() >= 1, (con.any(-1).sum(), lim.sum())
    rows = []
    for i in range(len(Q)):
        out = emul.rollout(env, env.plan_desc(), Q[i], V[i], W[i], us=A[i][None, None, :])
        rows.append((out["qpos_out"], out["qvel_out"], out["warm_out"]))
    rep, ok = single_step_errors(rows, ns)
    assert ok, rep


def test_generic_solver_equals_star_solver_on_slide_knees():
    """slidepod runs star<3,6>; forced onto the generic tree solver it must compute the same steps up to
    fp32 rounding (the two solvers sum in different orders)."""
    env, o = pair("slidepod")
    s = o.reset()
    rng = np.random.default_rng(8)
    us = np.clip(rng.normal(size=(3, 8, env.action_size)) * 0.6, -1, 1)
    star = emul.rollout(env, env.plan_desc(), s.qpos[0], s.qvel[0], s.qacc_warmstart[0], us=us)
    gen = emul.rollout(env, env.plan_desc(), s.qpos[0], s.qvel[0], s.qacc_warmstart[0], us=us, kernel=0)
    assert not np.array_equal(gen["q"], star["q"])         # the other solver did run
    assert np.abs(gen["q"] - star["q"]).max() < 1e-5
    assert np.abs(gen["qd"] - star["qd"]).max() < 1e-3
    assert np.abs(gen["rewss"] - star["rewss"]).max() < 1e-5 * (1 + np.abs(star["rewss"]).max())


# ---------------------------------------------------------------------------------------------
# structural rejections: modelc, fill_model_desc, the host model derivation (derive_model)
# ---------------------------------------------------------------------------------------------
def _xml(name):
    from tests.tree_envs import MODELS
    return open(os.path.join(MODELS, name + ".xml")).read()


def _compile(tmp_path, text):
    from dial_mpc_b200.modelc import compile_mjcf
    p = tmp_path / "m.xml"
    p.write_text(text)
    return compile_mjcf(str(p))


def _derive_error(md):
    from dial_mpc_b200 import _capi
    lib = _capi.lib()
    assert lib.dial_solver_variant(C.byref(md)) < 0
    return lib.dial_last_error().decode()


def _edit(text, old, new):
    assert text.count(old) >= 1, old
    return text.replace(old, new, 1)


def test_rejects_chain_longer_than_maxchain(tmp_path, built):
    """A 7th tail joint: the tip's chain is 13 dofs."""
    from dial_mpc_b200 import _capi
    t = _xml("longchain")
    t = _edit(t, '<geom name="tip" class="foot"', '<body name="t7" pos="-0.03 0 -0.032"><joint name="t7" range="-0.6 0.6"/>'
              '<inertial pos="0 0 0" mass="0.05" diaginertia="0.0001 0.0001 0.0001"/></body><geom name="tip" class="foot"')
    t = _edit(t, '<motor name="t6" joint="t6"/>', '<motor name="t6" joint="t6"/><motor name="t7" joint="t7"/>')
    m = _compile(tmp_path, t)
    assert m.nv == 21
    assert "dof ancestor chain longer than DIAL_MAXCHAIN" in _derive_error(_capi.fill_model_desc(m))


def test_rejects_ninth_geom(tmp_path, built):
    """A 9th collision geom does not fit the descriptor (DIAL_MAXG = 8); derive_model's own capacity check
    is behind it (reached with the count edited in a filled descriptor)."""
    from dial_mpc_b200 import _capi
    t = _edit(_xml("hexapod"), '<site name="head"', '<geom name="nose" type="sphere" size="0.02" pos="0.2 0 -0.05" conaffinity="1"/><site name="head"')
    m = _compile(tmp_path, t)
    assert m.ngeom == 9
    with pytest.raises(ValueError, match=r"exceeds capacity \(8,\)"):
        _capi.fill_model_desc(m)
    md = _capi.fill_model_desc(pair("hexapod")[0].sys.model)
    md.ngeom = 9
    assert "exceeds the fixed device capacities" in _derive_error(md)


def test_rejects_too_many_pyramid_edges(tmp_path, built):
    """A capsule foot on the hexapod: 9 contacts = 36 edges > DIAL_MAXE = 32 (geoms still 8)."""
    from dial_mpc_b200 import _capi
    t = _edit(_xml("hexapod"), '<geom name="L1" class="foot" pos="0 0 -0.12"/>',
              '<geom name="L1" class="foot" type="capsule" fromto="0 -0.02 -0.12 0 0.02 -0.12"/>')
    m = _compile(tmp_path, t)
    assert (m.ngeom, m.ncon) == (8, 9)
    assert "too many pyramidal contact edges" in _derive_error(_capi.fill_model_desc(m))


def test_rejects_sphere_sphere_pair_on_tree_path(tmp_path, built):
    """A colliding sphere on the torso touches the feet: a sphere-sphere pair, which only the dense
    (elliptic) path handles."""
    from dial_mpc_b200 import _capi
    t = _edit(_xml("slidepod"), '<site name="head"', '<geom name="bumper" type="sphere" size="0.03" contype="1"/><site name="head"')
    m = _compile(tmp_path, t)
    from dial_mpc_b200.modelc.mjcf import PAIR_SPHERE_SPHERE
    assert PAIR_SPHERE_SPHERE in m.arrays["pair_kind"]
    assert "unsupported contact pair kind on the tree (pyramidal) path" in _derive_error(_capi.fill_model_desc(m))


def test_rejects_moving_moving_pair(tmp_path, built):
    """A plane carried by the torso touches the feet: a plane-sphere pair whose plane moves."""
    from dial_mpc_b200 import _capi
    t = _edit(_xml("slidepod"), '<site name="head"', '<geom name="deck" type="plane" size="0 0 0.05" contype="1"/><site name="head"')
    m = _compile(tmp_path, t)
    assert "pyramidal contact pairs must be (static geom, moving geom)" in _derive_error(_capi.fill_model_desc(m))


def test_rejects_contact_body_dofs_off_one_chain(built):
    """modelc gives every body at most one joint whose dofs follow the body tree, so a contact body's dofs
    always form one chain: this message cannot be reached from MJCF.  It is checked on a filled
    descriptor whose last dof (RR knee, the RR foot's body) is re-parented onto the root, skipping the hip."""
    from dial_mpc_b200 import _capi
    md = _capi.fill_model_desc(pair("branchpod")[0].sys.model)
    assert md.dof_parentid[md.nv - 1] == md.nv - 2
    md.dof_parentid[md.nv - 1] = 5
    assert "contact body dofs do not form one chain" in _derive_error(md)


@pytest.mark.parametrize("what,old,new,msg", [
    ("ball joint", '<joint name="FL_hip" range="-1.2 1.2"/>', '<joint name="FL_hip" type="ball"/>', "ball joints are not supported"),
    ("two joints in one body", '<joint name="FL_hip" range="-1.2 1.2"/>',
     '<joint name="FL_hip" range="-1.2 1.2"/><joint name="FL_roll" axis="1 0 0" range="-0.3 0.3"/>',
     "more than one joint per body is not supported"),
    ("motor on the free joint", '<motor name="FL_hip" joint="FL_hip"/>', '<motor name="FL_hip" joint="FL_hip"/><motor name="push" joint="root"/>',
     "actuators on free joints are not supported"),
])
def test_modelc_rejections(tmp_path, what, old, new, msg):
    with pytest.raises(NotImplementedError, match=msg):
        _compile(tmp_path, _edit(_xml("branchpod"), old, new))


# ---------------------------------------------------------------------------------------------
# the variant-0 custom build
# ---------------------------------------------------------------------------------------------
def test_generic_custom_library_builds_and_exports(built):
    """nvcc cross-compiles the generic-tree custom build without a GPU; the tree fixtures share it."""
    from dial_mpc_b200 import _capi, custom
    paths = {n: pair(n)[0].library_path for n in GENERIC}
    path = paths["branchpod"]
    assert set(paths.values()) == {path} and "_v0_" in path and os.path.exists(path)
    assert custom.build_library(REWARD, variant=0) == path          # cached
    lib = _capi.lib(path)
    assert lib.dial_custom_reward_id().decode() == custom.reward_id(REWARD, 0)
    for sym in _capi.EXPORTS:
        assert hasattr(lib, sym)
    for n in GENERIC:
        assert lib.dial_solver_variant(_capi.fill_model_desc(pair(n)[0].sys.model)) == 0
    assert "_v1_" in pair("slidepod")[0].library_path
