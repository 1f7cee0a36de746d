"""Per-instance terrain on the CPU: the generators and ``height``; the oracle's terrain contacts against MJX's own
plane semantics (a flat terrain is the floor moved to its height, a uniform slope is a tilted plane geom); one env
step of the terrain build in the warp emulator against the oracle's env step on the same terrain (tests/
terrain_oracle.py), at the emulator's parity bounds (tests/test_instance_plant.py); a flat terrain at z = 0
bitwise equal to no terrain; ``dial_terrain_height``; the spec and CLI errors; the struct layout."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from dial_mpc_b200 import _capi
from dial_mpc_b200 import terrain as T
from tests.conftest import make_pair
from tests.terrain_oracle import collision, floor_pairs, on_terrain
from tests.test_instance_plant import emul_env_step, mid_run_states

import oracle.mjx_oracle as mo

EMUL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


# ---- generators and the surface --------------------------------------------------------------------------------
def test_generators_shape_seed_and_flat_patch():
    a = T.rough(0.04, 0.3, seed=1, size=4.0, spacing=0.05, flat_radius=0.5)
    assert a.heights.shape == (81, 81) and a.heights.dtype == np.float32 and a.origin == (-2.0, -2.0)
    assert np.array_equal(a.heights, T.rough(0.04, 0.3, seed=1, size=4.0, spacing=0.05, flat_radius=0.5).heights)
    assert not np.array_equal(a.heights, T.rough(0.04, 0.3, seed=2, size=4.0, spacing=0.05, flat_radius=0.5).heights)
    assert np.abs(a.heights).max() <= 0.04 and np.abs(a.heights).max() > 0.01
    xs = a.origin[0] + a.spacing * np.arange(81)
    X, Y = np.meshgrid(xs, xs)
    assert np.all(a.heights[np.hypot(X, Y) <= 0.5] == 0)
    s = T.slope(10.0, 90.0, size=4.0, spacing=0.1, flat_radius=0.5)
    assert np.all(s.heights[np.abs(Y[::2, ::2]) < 0.5 - 1e-9] == 0)
    far = np.abs(Y[::2, ::2]) > 0.6
    assert np.allclose(s.heights[far], np.tan(np.deg2rad(10)) * (Y[::2, ::2] - np.sign(Y[::2, ::2]) * 0.5)[far], atol=1e-6)
    g = T.grid([[0, 1], [2, 3]], 0.5, (1.0, -1.0))
    assert g.heights.shape == (2, 2) and g.origin == (1.0, -1.0)


def test_height_is_the_piecewise_linear_surface():
    rng = np.random.default_rng(0)
    t = T.grid(rng.normal(size=(7, 9)) * 0.1, 0.25, (-1.0, 0.5))
    ny, nx = t.heights.shape
    i, j = np.meshgrid(np.arange(nx), np.arange(ny))
    # the vertices
    assert np.allclose(T.height(t, t.origin[0] + i * t.spacing, t.origin[1] + j * t.spacing), t.heights, atol=1e-12)
    # linear within each triangle: H at a point = its barycentric mix of the triangle's vertex heights
    u, v = rng.uniform(0, nx - 1, 4000), rng.uniform(0, ny - 1, 4000)
    ci, cj = np.minimum(u.astype(int), nx - 2), np.minimum(v.astype(int), ny - 2)
    fu, fv = u - ci, v - cj
    h = t.heights.astype(np.float64)
    low = fu >= fv
    want = np.where(low, (1 - fu) * h[cj, ci] + (fu - fv) * h[cj, ci + 1] + fv * h[cj + 1, ci + 1],
                    (1 - fv) * h[cj, ci] + (fv - fu) * h[cj + 1, ci] + fu * h[cj + 1, ci + 1])
    got, sx, sy = T.plane(t, t.origin[0] + u * t.spacing, t.origin[1] + v * t.spacing)
    assert np.allclose(got, want, atol=1e-12)
    # outside: clamped, horizontal
    H, sx, sy = T.plane(t, np.array([-5.0, 10.0]), np.array([0.7, 100.0]))
    assert np.allclose(H, [T.height(t, -1.0, 0.7), h[-1, -1]]) and np.all(sx == 0) and np.all(sy == 0)


# ---- the oracle against MJX's plane semantics -------------------------------------------------------------------
def _states(o, n, seed, spread):
    """Kinematics of n random poses of o's robot: the reset pose moved in x, y, turned in yaw, joints perturbed."""
    rng = np.random.default_rng(seed)
    q = np.tile(o.reset().qpos, (n, 1))
    q[:, :2] += rng.uniform(-spread, spread, (n, 2))
    q[:, 2] += rng.uniform(-0.05, 0.1, n)
    yaw = rng.uniform(-np.pi, np.pi, n)
    q[:, 3:7] = np.stack([np.cos(yaw / 2), 0 * yaw, 0 * yaw, np.sin(yaw / 2)], -1)
    q[:, 7:] += rng.normal(size=(n, q.shape[1] - 7)) * 0.2
    _, xpos, _, xmat, *_ = mo.kinematics(o.m, q)
    return xpos, xmat


def _floor_geom(m):
    return {int(m.pair_geom1[k]) for _, k, _ in floor_pairs(m)}.pop()


@pytest.mark.parametrize("name", ["unitree_go2_walk", "unitree_h1_loco"])
def test_flat_terrain_is_the_floor_moved_to_its_height(name):
    _, o = make_pair(name)
    xpos, xmat = _states(o, 64, 1, 2.0)
    c = 0.137
    t = T.Terrain(np.full((5, 5), c), 0.5, (-1.0, -1.0))   # feet inside and beyond the grid
    m = o.m
    g = _floor_geom(m)
    saved = m.geom_pos.copy()
    try:
        m.geom_pos = m.geom_pos.copy()
        m.geom_pos[g, 2] += c
        want = mo.collision(m, xpos, xmat)
    finally:
        m.geom_pos = saved
    for a, b in zip(collision(m, xpos, xmat, t), want):
        assert np.abs(a - b).max() < 1e-12


@pytest.mark.parametrize("name", ["unitree_go2_walk", "unitree_h1_loco"])
def test_uniform_slope_is_a_tilted_plane_geom(name):
    """A uniform-slope terrain (flat_radius 0, fp64 heights) gives the contacts of the floor geom tilted to the
    slope; beyond the grid, those of the floor moved to the height of the clamped point."""
    _, o = make_pair(name)
    m = o.m
    g = _floor_geom(m)
    for angle, heading in [(8.0, 0.0), (15.0, 120.0), (5.0, -40.0)]:
        a, psi = np.deg2rad(angle), np.deg2rad(heading)
        xs = -3.0 + 0.25 * np.arange(25)
        X, Y = np.meshgrid(xs, xs)
        t = T.Terrain(np.tan(a) * (X * np.cos(psi) + Y * np.sin(psi)), 0.25, (-3.0, -3.0))
        xpos, xmat = _states(o, 96, int(angle), 4.0)
        axis = np.array([np.sin(psi), -np.cos(psi), 0.0])   # tilts +z away from the heading: rises along it
        quat = np.concatenate([[np.cos(a / 2)], np.sin(a / 2) * axis])
        saved = (m.geom_quat.copy(), m.geom_pos.copy())
        try:
            m.geom_quat = m.geom_quat.copy()
            m.geom_quat[g] = mo.qmul(quat, m.geom_quat[g])
            tilted = mo.collision(m, xpos, xmat)
        finally:
            m.geom_quat = saved[0]
        got = collision(m, xpos, xmat, t)
        # which contacts are inside the grid: those whose sphere centre is
        inside = np.zeros(got[0].shape, bool)
        for c, k, sgn in floor_pairs(m):
            g2 = int(m.pair_geom2[k]); b2 = int(m.geom_bodyid[g2])
            p2 = xpos[:, b2] + np.einsum("nij,j->ni", xmat[:, b2], m.geom_pos[g2])
            cc = p2 + sgn * np.einsum("nij,jk->nik", xmat[:, b2], mo.qmat(m.geom_quat[g2]))[:, :, 2] * m.geom_size[g2, 1]
            inside[:, c] = (np.abs(cc[:, 0]) <= 3.0) & (np.abs(cc[:, 1]) <= 3.0)
        floor_slots = [c for c, _, _ in floor_pairs(m)]
        ins = inside[:, floor_slots]
        assert ins.any() and (~ins).any()
        for a_, b_ in zip(got, tilted):
            err = np.abs(a_ - b_)[:, floor_slots]
            err = err.reshape(err.shape[0], err.shape[1], -1).max(-1)
            assert err[ins].max() < 1e-12, (angle, err[ins].max())
        # beyond the grid: a horizontal plane at the slope's height at the clamped point
        for c, k, sgn in floor_pairs(m):
            out = ~inside[:, c]
            n = got[2][out, c, 0]
            assert np.allclose(n, [0, 0, 1], atol=0)
            g2 = int(m.pair_geom2[k]); b2 = int(m.geom_bodyid[g2])
            p2 = xpos[:, b2] + np.einsum("nij,j->ni", xmat[:, b2], m.geom_pos[g2])
            cc = p2 + sgn * np.einsum("nij,jk->nik", xmat[:, b2], mo.qmat(m.geom_quat[g2]))[:, :, 2] * m.geom_size[g2, 1]
            hc = np.tan(a) * (np.clip(cc[:, 0], -3, 3) * np.cos(psi) + np.clip(cc[:, 1], -3, 3) * np.sin(psi))
            assert np.abs(got[0][out, c] - (cc[out, 2] - hc[out] - m.geom_size[g2, 0])).max() < 1e-12


# ---- the emulator's terrain build ------------------------------------------------------------------------------
_LIBS = {}


def _lib(reward_source=None):
    key = reward_source or ""
    if key not in _LIBS:
        so = os.path.join(EMUL, f"libdial_emul_terrain{'_' + os.path.basename(key).split('.')[0] if key else ''}.so")
        extra = [f'-DDIAL_CUSTOM_REWARD_FILE="{os.path.abspath(reward_source)}"'] if reward_source else []
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", EMUL, "-shared", "-fPIC"] + extra +
                              ["-o", so, os.path.join(EMUL, "emul_terrain.cpp")])
        lib = C.CDLL(so)
        lib.emul_terrain_height.restype = C.c_float
        lib.emul_terrain_height.argtypes = [C.c_void_p, C.c_float, C.c_float]
        _LIBS[key] = lib
    return _LIBS[key]


def emul_terrain_step(env, t, q, v, w, a, step0):
    lib = _lib(getattr(env, "reward_source", None) or None)
    md, desc = _capi.fill_model_desc(env.sys.model), env.plan_desc()
    f32 = lambda x: np.ascontiguousarray(x, dtype=np.float32)
    q, v, w, us = f32(q), f32(v), f32(w), f32(np.asarray(a).reshape(1, 1, md.nu))
    out = dict(rewss=np.zeros((1, 1), np.float32), q=np.zeros((1, 1, md.nq), np.float32),
               qd=np.zeros((1, 1, md.nv), np.float32), qpos_out=np.zeros(md.nq, np.float32),
               qvel_out=np.zeros(md.nv, np.float32), warm_out=np.zeros(md.nv, np.float32),
               ctrl_out=np.zeros(md.nu, np.float32))
    ct = None if t is None else t.c_struct()
    rc = lib.emul_rollout_terrain(C.byref(md), C.byref(desc), None if ct is None else C.byref(ct), 0, 1, 1, int(step0),
                                  _p(q), _p(v), _p(w), _p(us), _p(out["rewss"]), _p(out["q"]), _p(out["qd"]),
                                  _p(out["qpos_out"]), _p(out["qvel_out"]), _p(out["warm_out"]), _p(out["ctrl_out"]))
    assert rc == 0
    return out


def _pair(name):
    if name == "branchpod":
        from tests.tree_envs import make_tree_pair
        return make_tree_pair(name)
    return make_pair(name)


def on_ground(o, t, s, shift):
    """State s moved by `shift` in x, y and lifted so that its lowest floor contact just touches terrain t."""
    from oracle.envs_oracle import OState
    q = s.qpos.copy()
    q[:, :2] += shift
    _, xpos, _, xmat, *_ = mo.kinematics(o.m, q)
    d = collision(o.m, xpos, xmat, t)[0][:, [c for c, _, _ in floor_pairs(o.m)]]
    q[:, 2] -= d.min() - 0.002
    return OState(q, s.qvel, s.qacc_warmstart, s.step, s.stage)


TERRAINS = {"rough": lambda: T.rough(0.03, 0.3, seed=3, size=4.0, spacing=0.05, flat_radius=0.0),
            "slope": lambda: T.slope(12.0, 30.0, size=3.0, spacing=0.1, flat_radius=0.2)}


@pytest.mark.parametrize("name", ["unitree_go2_walk", "unitree_h1_loco", "branchpod"])
@pytest.mark.parametrize("kind", list(TERRAINS))
def test_emulated_env_step_on_terrain_equals_the_oracle(name, kind):
    env, o = _pair(name)
    t = TERRAINS[kind]()
    half = (t.heights.shape[1] - 1) * t.spacing / 2
    # inside the grid (feet in both halves of cells) and straddling its edge
    shifts = [(0.37, -0.21), (-0.64, 0.45), (half - 0.05, 0.1), (0.2, -half + 0.02)]
    moved = 0.0
    for i, (s0, a) in enumerate(mid_run_states(o, 4, 11)):
        s = on_ground(o, t, s0, np.array(shifts[i]))
        step0 = int(s.step[0])
        out = emul_terrain_step(env, t, s.qpos[0], s.qvel[0], s.qacc_warmstart[0], a[0], step0)
        with on_terrain(o, t):
            ns, r, aux = o.step(s, a)
        assert np.abs(out["qpos_out"] - ns.qpos[0]).max() < 1e-4, (i, np.abs(out["qpos_out"] - ns.qpos[0]).max())
        assert np.abs(out["qvel_out"] - ns.qvel[0]).max() < 5e-3 * (1 + np.abs(ns.qvel[0]).max() / 10), i
        assert abs(out["rewss"][0, 0] - r[0]) < 1e-3 * (1 + abs(r[0])), (i, out["rewss"][0, 0], r[0])
        flat, _, _ = o.step(s, a)
        moved = max(moved, float(np.abs(flat.qpos[0] - ns.qpos[0]).max()))
    assert moved > 1e-4   # the terrain changed the step


@pytest.mark.parametrize("name", ["unitree_go2_walk", "unitree_h1_loco", "branchpod"])
def test_flat_terrain_at_zero_is_bitwise_no_terrain(name):
    from tests.emul import emul
    env, o = _pair(name)
    t = T.grid(np.zeros((4, 6)), 0.4, (-1.0, -0.6))
    for i, (s, a) in enumerate(mid_run_states(o, 2, 5)):
        step0 = int(s.step[0])
        got = emul_terrain_step(env, t, s.qpos[0], s.qvel[0], s.qacc_warmstart[0], a[0], step0)
        none = emul_terrain_step(env, None, s.qpos[0], s.qvel[0], s.qacc_warmstart[0], a[0], step0)
        md = _capi.fill_model_desc(env.sys.model)
        ref = emul_env_step(env, md, env.plan_desc(), s.qpos[0], s.qvel[0], s.qacc_warmstart[0], a[0], step0)
        for k in ("qpos_out", "qvel_out", "warm_out", "ctrl_out"):
            assert np.array_equal(got[k], ref[k]) and np.array_equal(none[k], ref[k]), (i, k)
        assert np.array_equal(got["rewss"], ref["rewss"])


def test_oracle_surface_equals_the_library_definition():
    """tests/terrain_oracle.plane (restated from the definition) and terrain.plane agree, inside and beyond the grid."""
    from tests.terrain_oracle import plane as oracle_plane
    rng = np.random.default_rng(9)
    t = T.grid(rng.normal(size=(9, 6)) * 0.3, 0.2, (0.3, -1.1))
    x, y = rng.uniform(-0.5, 1.8, 3000), rng.uniform(-1.8, 1.0, 3000)
    for a, b in zip(oracle_plane(t, x, y), T.plane(t, x, y)):
        assert np.abs(a - b).max() < 1e-12


NO_FLOOR = """<mujoco><worldbody>
  <geom name="post" type="sphere" size="0.1" pos="0 0 0"/>
  <body name="ball" pos="0 0 0.5"><freejoint/><geom name="b" type="sphere" size="0.1" mass="1"/></body>
</worldbody></mujoco>"""


def test_no_floor_pair_is_rejected(tmp_path):
    from dial_mpc_b200.modelc import compile_mjcf
    path = tmp_path / "no_floor.xml"
    path.write_text(NO_FLOOR)
    model = compile_mjcf(str(path))
    assert not T.has_floor(model)
    with pytest.raises(ValueError, match=r"the model has no floor pair"):
        T.terrain_setting({"kind": "slope", "angle": 3}, model)


def test_custom_reward_terrain_height():
    lib = _lib()
    rng = np.random.default_rng(4)
    t = T.grid(rng.normal(size=(6, 8)) * 0.2, 0.3, (-1.0, -0.5))
    ct = t.c_struct()
    x, y = rng.uniform(-2, 2, 500), rng.uniform(-1.5, 2, 500)
    got = np.array([lib.emul_terrain_height(C.byref(ct), float(a), float(b)) for a, b in zip(x, y)])
    assert np.abs(got - T.height(t, x.astype(np.float32), y.astype(np.float32))).max() < 2e-6
    assert lib.emul_terrain_height(None, 0.3, 0.2) == 0.0


# ---- specs, the command line and the C ABI -------------------------------------------------------------------
def test_terrain_setting_errors():
    import dial_mpc_b200.envs as E
    env = E.get_environment("unitree_go2_walk", config=E.UnitreeGo2EnvConfig())
    s = T.terrain_setting({"kind": "slope", "angle": 5, "planner": True}, env.sys)
    assert s.planner and T.terrains(s) == (s.terrain, s.terrain)
    assert T.terrains(T.terrain_setting({"kind": "slope", "angle": 5}))[1] is None
    for spec, msg in [({"kind": "bumps"}, r"kind rough \| slope \| grid"), (3, r"a terrain spec is a mapping"),
                      ({"kind": "rough", "amplitude": 0.1}, r"needs 'wavelength'"),
                      ({"kind": "rough", "amplitude": 0.1, "wavelength": 0.3, "colour": 1}, r"got 'colour'"),
                      ({"kind": "rough", "amplitude": -1, "wavelength": 0.3}, r"amplitude must be finite and >= 0"),
                      ({"kind": "rough", "amplitude": 0.1, "wavelength": 0.3, "seed": 1.5}, r"seed must be an int"),
                      ({"kind": "slope", "angle": "x"}, r"angle_deg must be a number"),
                      ({"kind": "slope", "angle": 5, "planner": 1}, r"planner must be true or false"),
                      ({"kind": "slope", "angle": 5, "spacing": 0.001}, r"out of range \(2\.\.1024\)"),
                      ({"kind": "grid", "heights": [[0, float("nan")], [0, 0]], "spacing": 0.1}, r"heights must be finite"),
                      ({"kind": "grid", "heights": [[0, 1]], "spacing": 0.1}, r"\[ny, nx\] grid"),
                      ({"kind": "grid", "heights": [[0, 1], [0, 1]], "spacing": 0}, r"spacing must be a finite number > 0")]:
        with pytest.raises(ValueError, match=msg):
            T.terrain_setting(spec, env.sys)


def test_cli_errors(tmp_path, monkeypatch, capsys):
    from tests.test_instance_settings import run_main
    r = run_main(tmp_path, monkeypatch, capsys, ["--terrain", "{kind: slope}"], {})
    assert r[0] == "error" and r[1] == 2 and "--terrain: a slope terrain needs 'angle'" in r[2], r
    r = run_main(tmp_path, monkeypatch, capsys, ["--terrain", "{kind: slope, angle: 5}", "--eager"], {})
    assert r[:2] == ["error", 2] and "--terrain runs on the CUDA-graph loop; it excludes --eager" in r[2], r
    r = run_main(tmp_path, monkeypatch, capsys, ["--instances", "2", "--instance-overrides", "@ov"],
                 {"ov": [{}, {"terrain": {"kind": "rough", "amplitude": 0.02}}]})
    assert r[:2] == ["error", 2] and "--instance-overrides entry 1: terrain: a rough terrain needs 'wavelength'" in r[2], r
    r = run_main(tmp_path, monkeypatch, capsys, ["--instances", "2", "--instance-overrides", "@ov"],
                 {"ov": [{}, {"terrain": {"kind": "slope", "angle": 5}}]})
    assert r[0] == "call" and r[1]["run_instances"]["kwargs"]["terrain"] == [None, {"kind": "slope", "angle": 5}], r
    r = run_main(tmp_path, monkeypatch, capsys, ["--terrain", "{kind: slope, angle: 5, planner: true}"], {})
    assert r[0] == "call" and r[1]["DeviceLoop"]["kwargs"]["terrain"] == {"kind": "slope", "angle": 5, "planner": True}
    r = run_main(tmp_path, monkeypatch, capsys, [], {})
    assert r[0] == "call" and "terrain" not in r[1]["DeviceLoop"]["kwargs"]


def test_struct_layout_and_symbol():
    lib = _capi.lib()
    assert lib.dial_sizeof(7) == C.sizeof(_capi.dial_terrain) == 32
    assert [f for f, _ in _capi.dial_terrain._fields_] == ["nx", "ny", "x0", "y0", "spacing", "heights"]
    assert "dial_plan_set_instance_terrain" in _capi.EXPORTS and hasattr(lib, "dial_plan_set_instance_terrain")
    out = subprocess.run(["nm", "-D", "--defined-only", _capi.LIB_PATH], capture_output=True, text=True).stdout
    assert " dial_plan_set_instance_terrain" in out
    assert (_capi.DEFINES["DIAL_MAXTERRAIN"], T.PLANT, T.PLANNER) == (1024, 0, 1)
