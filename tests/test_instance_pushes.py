"""Per-instance pushes on the CPU: the push spec (push_setting) and its errors, the CLI errors of --push and of the
push key of --instance-overrides, the struct layout, and the push step the kernel runs (push_kinematics,
push_rows, push_solve, on the warp emulator) against the fp64 oracle: Delta qvel = solve(M, J^T [torque; force]
dt) with M from the oracle's kinematics, com_pos and crb_mass_matrix, on Go2, H1, the four generic tree models
and Allegro's ball, at many states, for points off the COM and torque-only impulses; on floating bases the
spatial momentum of the pushed tree changes by exactly the spatial impulse; a zero impulse leaves qvel bit for
bit; and the firing window of an entry."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from dial_mpc_b200 import _capi
from tests.conftest import make_pair

EMUL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
PMAX = _capi.DEFINES["DIAL_MAXPUSH"]
MODELS = ["unitree_go2_walk", "unitree_h1_walk", "branchpod", "hexapod", "longchain", "slidepod", "allegro_reorient"]
# Delta qvel of the emulator (fp64 throughout) against the oracle's np.linalg.solve: both fp64, in other
# orders; relative to the largest component
TOL = 1e-9


def _go2():
    env, _ = make_pair("unitree_go2_walk")
    return env


_ENVS = {}


def _env(name):
    if name not in _ENVS:
        if name in ("branchpod", "hexapod", "longchain", "slidepod"):
            from tests.tree_envs import make_tree_pair
            _ENVS[name] = make_tree_pair(name)[0]
        else:
            _ENVS[name] = make_pair(name)[0]
    return _ENVS[name]


# ---- push_setting and the CLI -------------------------------------------------------------------------
def test_push_setting_forms():
    from dial_mpc_b200.core.dial_core import push_setting
    env = _go2()
    assert push_setting(None, env.sys) == [] and push_setting([], env) == []
    t = push_setting([{"step": 5, "body": "base", "force": [10, 0, -2.5]},
                      {"step": 9, "steps": 3, "body": "FL_calf", "pos": [0, 0, -0.1], "torque": [0, 1, 0]}], env.sys)
    assert len(t) == 2 and all(isinstance(p, _capi.dial_push) for p in t)
    assert (t[0].step, t[0].n_steps, t[0].body) == (5, 1, 1)
    assert list(t[0].force) == [10.0, 0.0, -2.5] and not any(t[0].pos) and not any(t[0].torque)
    assert (t[1].step, t[1].n_steps, t[1].body) == (9, 3, env.sys.model.names["body"].index("FL_calf"))
    assert list(t[1].pos) == [0.0, 0.0, np.float32(-0.1)] and list(t[1].torque) == [0.0, 1.0, 0.0]
    assert len(push_setting([{"step": 1, "body": "base"}] * PMAX, env.sys)) == PMAX
    assert C.sizeof(_capi.dial_push) == 48


@pytest.mark.parametrize("spec, match", [
    ({"step": 1}, r"a push spec is a list of mappings"),
    ([{"step": 1, "body": "base"}] * (PMAX + 1), r"a push spec has at most 16 entries, got 17"),
    ([3], r"push 0: an entry is a mapping"),
    ([{"step": 1, "body": "base"}, {"body": "base"}], r"push 1: needs step"),
    ([{"step": 1}], r"push 0: needs body"),
    ([{"step": 1, "body": "world"}], r"push 0: unknown body 'world'"),
    ([{"step": 1, "body": "trunk"}], r"push 0: unknown body 'trunk' \(known: \['base'"),
    ([{"step": 0, "body": "base"}], r"push 0: step must be an int >= 1, got 0"),
    ([{"step": 1.5, "body": "base"}], r"push 0: step must be an int >= 1, got 1\.5"),
    ([{"step": True, "body": "base"}], r"push 0: step must be an int >= 1"),
    ([{"step": 1, "steps": 0, "body": "base"}], r"push 0: steps must be an int >= 1, got 0"),
    ([{"step": 1, "body": "base", "force": [1, 2]}], r"push 0: force must be a list of 3 finite numbers"),
    ([{"step": 1, "body": "base", "torque": [1, float("nan"), 0]}], r"push 0: torque must be a list of 3 finite"),
    ([{"step": 1, "body": "base", "pos": [1e39, 0, 0]}], r"push 0: pos must be a list of 3 finite numbers"),
    ([{"step": 1, "body": "base", "impulse": 1}], r"push 0: unknown key 'impulse'"),
])
def test_push_setting_names_the_bad_entry(spec, match):
    from dial_mpc_b200.core.dial_core import push_setting
    with pytest.raises(ValueError, match=match):
        push_setting(spec, _go2().sys)


def _main(monkeypatch, capsys, argv):
    from dial_mpc_b200.core import dial_core
    monkeypatch.setattr(sys, "argv", ["dial_core", "--example", "unitree_go2_trot"] + argv)
    with pytest.raises(SystemExit) as e:
        dial_core.main()
    return e.value.code, capsys.readouterr().err


@pytest.mark.parametrize("value, match", [
    ("[{step: 0, body: base}]", r"--push: push 0: step must be an int >= 1, got 0"),
    ("[{step: 3, body: head}]", r"--push: push 0: unknown body 'head'"),
    ("{step: 3, body: base}", r"--push: a push spec is a list"),
    ("[{step: 3", r"--push: not a YAML list"),
    ("[{step: 3, body: base, force: [1, 2, x]}]", r"--push: push 0: force must be a list of 3 finite numbers"),
])
def test_cli_push_errors(monkeypatch, capsys, value, match):
    code, err = _main(monkeypatch, capsys, ["--push", value])
    assert code == 2 and re.search(match, err), err


def test_cli_push_excludes_eager(monkeypatch, capsys):
    code, err = _main(monkeypatch, capsys, ["--push", "[{step: 3, body: base}]", "--eager"])
    assert code == 2 and "--push runs on the CUDA-graph loop; it excludes --eager" in err, err


@pytest.mark.parametrize("entry, match", [
    ({"push": [{"step": -1, "body": "base"}]}, r"push: push 0: step must be an int >= 1, got -1"),
    ({"push": [{"step": 2, "body": "base"}, {"step": 2, "body": "FR_foot"}]}, r"push: push 1: unknown body 'FR_foot'"),
    ({"push": {"step": 2}}, r"push: a push spec is a list"),
])
def test_cli_instance_override_push_errors(tmp_path, monkeypatch, capsys, entry, match):
    import yaml
    ov = tmp_path / "ov.yaml"
    ov.write_text(yaml.safe_dump([{"push": [{"step": 2, "body": "base"}]}, {}, entry]))
    code, err = _main(monkeypatch, capsys, ["--instances", "3", "--instance-overrides", str(ov)])
    assert code == 2 and re.search(r"--instance-overrides entry 2: " + match, err), err


def test_library_struct_layout(built):
    lib = _capi.lib()
    assert lib.dial_sizeof(5) == C.sizeof(_capi.dial_push) == 48
    assert _capi.DEFINES["DIAL_MAXPUSH"] == 16


# ---- warp emulator against the oracle -------------------------------------------------------------------
class PushTable(C.Structure):
    _fields_ = [("n", C.c_int32), ("pad", C.c_int32 * 3), ("e", _capi.dial_push * PMAX)]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    """g++ build of tests/emul/emul_push.cpp (the device code under the emulator)."""
    so = str(tmp_path_factory.mktemp("emul_push") / "libdial_emul_push.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", EMUL, "-shared", "-fPIC", "-o", so,
                           os.path.join(EMUL, "emul_push.cpp")])
    lib = C.CDLL(so)
    lib.emul_sizeof_push.restype = C.c_size_t
    assert lib.emul_sizeof_push(0) == C.sizeof(_capi.dial_push) and lib.emul_sizeof_push(1) == C.sizeof(PushTable)
    lib.emul_push_step.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double] + [C.c_void_p] * 4 + [C.c_int]
    return lib


def oracle_model(model, path):
    """The oracle's model of a compiled model (saved to `path`), with the parameters the device model holds:
    fp32 roundings of the compiled values."""
    from oracle.mjx_oracle import OModel
    model.save(path)
    o = OModel(path)
    for k, v in list(vars(o).items()):
        if isinstance(v, np.ndarray) and v.dtype.kind == "f":
            setattr(o, k, v.astype(np.float32).astype(np.float64))
    return o


@pytest.fixture(scope="module")
def omodels(tmp_path_factory):
    """(model, tag) -> oracle_model of it."""
    d = tmp_path_factory.mktemp("push_models")
    return lambda model, tag: oracle_model(model, str(d / (tag + ".json")))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _table(entries):
    T = PushTable()
    T.n = len(entries)
    for i, e in enumerate(entries):
        T.e[i] = e
    return T


def _push(step, body, pos=(0, 0, 0), force=(0, 0, 0), torque=(0, 0, 0), n_steps=1):
    p = _capi.dial_push()
    p.step, p.n_steps, p.body = step, n_steps, body
    p.pos[:], p.force[:], p.torque[:] = [float(x) for x in pos], [float(x) for x in force], [float(x) for x in torque]
    return p


def emul_push(lib, model, entries, step, dt, qpos, qvel, lanes=32):
    md = _capi.fill_model_desc(model)
    T = _table(entries)
    nv = model.nv
    q = np.ascontiguousarray(qpos, np.float32)
    v = np.ascontiguousarray(qvel, np.float32).copy()
    dq, M = np.full(nv, np.nan), np.full((nv, nv), np.nan)
    fired = lib.emul_push_step(C.byref(md), C.byref(T), int(step), float(dt), _p(q), _p(v), _p(dq), _p(M), lanes)
    assert fired in (0, 1)
    return bool(fired), v, dq, M


def oracle_push(o, entries, step, dt, qpos):
    """Delta qvel = solve(M, J^T [torque; force] dt) in fp64: M from crb_mass_matrix, J of the point's world
    position from the oracle's cdof (rotational rows cdof[:3], translational cdof[3:] + cdof[:3] x (p - c), c the
    root COM of the body's tree), summed over the entries firing at `step`; also M, the spatial impulse at each
    tree root's COM, and the oracle's COM-frame quantities."""
    from oracle.mjx_oracle import com_pos, crb_mass_matrix, kinematics
    q = np.asarray(qpos, np.float64)[None]
    _, xpos, xquat, xmat, xipos, ximat, xanchor, xaxis = kinematics(o, q)
    root_com, cinert, cdof = com_pos(o, xpos, xmat, xipos, ximat, xanchor, xaxis)
    M = crb_mass_matrix(o, cinert, cdof)[0]
    g = np.zeros(o.nv)
    imp = {}   # tree root -> spatial impulse [torque; force] dt at its COM
    for e in entries:
        if not e.step <= step < e.step + e.n_steps:
            continue
        b = e.body
        p = xpos[0, b] + xmat[0, b] @ np.asarray(e.pos, np.float64)
        c = root_com[0, b]
        f, tq = np.asarray(e.force, np.float64), np.asarray(e.torque, np.float64)
        Jr = cdof[0, :, :3]
        Jp = cdof[0, :, 3:] + np.cross(cdof[0, :, :3], p - c)
        g += o.body_dofmask[b] * (Jr @ tq + Jp @ f)
        r = int(o.body_rootid[b])
        imp[r] = imp.get(r, np.zeros(6)) + np.concatenate([tq + np.cross(p - c, f), f]) * dt
    return np.linalg.solve(M, g * dt), M, imp, (cinert[0], cdof[0], root_com[0])


def _random_state(model, rng):
    """A state the robot could be in: hinge and slide joints near qpos0, free joints anywhere with any
    orientation (an unnormalised quaternion: the kinematics normalise it), random velocities."""
    A = model.arrays
    qpos = np.array(A["qpos0"], np.float64)
    for j, t in enumerate(A["jnt_type"]):
        a = int(A["jnt_qposadr"][j])
        if t == 0:
            qpos[a:a + 3] = rng.uniform(-1, 1, 3) + [0, 0, 0.4]
            qpos[a + 3:a + 7] = rng.normal(size=4) * rng.uniform(0.5, 2.0)
        else:
            qpos[a] += rng.uniform(-0.6, 0.6) * (0.1 if t == 2 else 1.0)
    return qpos.astype(np.float32), rng.normal(size=model.nv).astype(np.float32)


def _random_entries(model, rng, n, step, torque_only=False):
    nb = model.nbody
    out = []
    for _ in range(n):
        body = int(rng.integers(1, nb))
        pos = np.zeros(3) if torque_only else rng.uniform(-0.15, 0.15, 3)
        force = np.zeros(3) if torque_only else rng.normal(size=3) * 40
        out.append(_push(step, body, pos, force, rng.normal(size=3) * 3))
    return out


def _dt(env):
    return float(env.plan_desc().n_frames) * float(np.float32(env.sys.model.timestep))


@pytest.mark.parametrize("name", MODELS)
def test_emulated_push_equals_oracle(lib, omodels, name):
    """At 12 random states, 1..4 entries on random bodies with points off the COM, or torque-only: the emulator's
    M equals the oracle's crb_mass_matrix and its Delta qvel the oracle's solve(M, J^T p dt) within fp64
    rounding; qvel takes it with one rounding; 1 and 32 lanes give the same bits."""
    env = _env(name)
    model = env.sys.model
    o = omodels(model, name)
    rng = np.random.default_rng(7)
    dt = _dt(env)
    nv = model.nv
    for t in range(12):
        qpos, qvel = _random_state(model, rng)
        step = int(rng.integers(1, 500))
        entries = _random_entries(model, rng, 1 + t % 4, step, torque_only=t % 3 == 2)
        fired, v, dq, M = emul_push(lib, model, entries, step, dt, qpos, qvel)
        ref, Mref, _, _ = oracle_push(o, entries, step, dt, qpos)
        assert fired
        np.testing.assert_allclose(M, Mref, rtol=0, atol=1e-12 * np.abs(Mref).max())
        scale = np.abs(ref).max()
        assert scale > 0
        assert np.abs(dq - ref).max() <= TOL * scale, (name, t, np.abs(dq - ref).max() / scale)
        assert np.array_equal(v, (qvel.astype(np.float64) + dq).astype(np.float32))
        _, v1, dq1, _ = emul_push(lib, model, entries, step, dt, qpos, qvel, lanes=1)
        assert np.array_equal(dq1, dq) and np.array_equal(v1, v)
    assert nv == o.nv


def test_allegro_ball_push_moves_the_ball_only(lib, omodels):
    """Allegro (the dense solver's model): a push on the ball (body 'object', its own free tree) moves the ball's
    six dofs only; a push on a fingertip moves its finger's dofs only."""
    env = _env("allegro_reorient")
    model = env.sys.model
    o = omodels(model, "allegro_reorient")
    names = model.names["body"]
    rng = np.random.default_rng(11)
    qpos, qvel = _random_state(model, rng)
    ball = _push(4, names.index("object"), (0.01, -0.02, 0.0), (0.5, 0.2, -0.3), (0.0, 0.01, 0.0))
    _, _, dq, _ = emul_push(lib, model, [ball], 4, _dt(env), qpos, qvel)
    ref, *_ = oracle_push(o, [ball], 4, _dt(env), qpos)
    assert np.abs(dq[:6]).min() > 0 and not dq[6:].any()
    assert np.abs(dq - ref).max() <= TOL * np.abs(ref).max()
    tip = _push(4, names.index("ff_tip"), force=(0.0, 0.0, 1.0))
    _, _, dq, _ = emul_push(lib, model, [tip], 4, _dt(env), qpos, qvel)
    assert not dq[:6].any() and np.count_nonzero(dq) == 4


@pytest.mark.parametrize("name", ["unitree_go2_walk", "unitree_h1_walk", "branchpod", "hexapod", "longchain",
                                  "slidepod", "allegro_reorient"])
def test_momentum_changes_by_the_impulse(lib, omodels, name):
    """Floating-base trees (no armature on their free joint): the spatial momentum of the pushed tree about its
    COM, sum_b cinert_b cvel_b, changes by exactly the spatial impulse [torque + (p - c) x force; force] dt."""
    from oracle.mjx_oracle import com_vel, inert_mul
    env = _env(name)
    model = env.sys.model
    o = omodels(model, name)
    A = model.arrays
    free = [j for j, t in enumerate(A["jnt_type"]) if t == 0]
    assert free
    rng = np.random.default_rng(5)
    dt = _dt(env)
    for t in range(6):
        qpos, qvel = _random_state(model, rng)
        j = free[t % len(free)]
        root = int(A["jnt_bodyid"][j]) if "jnt_bodyid" in A else int(np.flatnonzero(A["body_jntadr"] == j)[0])
        d0 = int(A["jnt_dofadr"][j])
        assert not A["dof_armature"][d0:d0 + 6].any()
        tree = [b for b in range(model.nbody) if int(A["body_rootid"][b]) == root]
        entries = [_push(3, int(rng.choice(tree)), rng.uniform(-0.1, 0.1, 3), rng.normal(size=3) * 30,
                         rng.normal(size=3)) for _ in range(2)]
        _, _, dq, _ = emul_push(lib, model, entries, 3, dt, qpos, qvel)
        _, _, imp, (cinert, cdof, _) = oracle_push(o, entries, 3, dt, qpos)
        dv = np.asarray(dq)[None]
        dcvel, _ = com_vel(o, cdof[None], dv)
        dh = inert_mul(cinert[tree], dcvel[0, tree]).sum(0)
        assert np.abs(dh - imp[root]).max() <= 1e-9 * np.abs(imp[root]).max(), (name, t, dh, imp[root])


@pytest.mark.parametrize("name", ["unitree_go2_walk", "allegro_reorient", "slidepod"])
def test_zero_impulse_leaves_qvel(lib, name):
    """An entry that fires with zero force and torque leaves qvel bit for bit (-0 and denormals included); an
    entry that does not fire is not a push at all."""
    env = _env(name)
    model = env.sys.model
    rng = np.random.default_rng(9)
    qpos, qvel = _random_state(model, rng)
    qvel[0], qvel[1] = -0.0, np.float32(1e-40)
    zero = [_push(10, b, rng.uniform(-1, 1, 3)) for b in range(1, model.nbody)][:PMAX]
    fired, v, dq, _ = emul_push(lib, model, zero, 10, _dt(env), qpos, qvel)
    assert fired and not dq.any() and v.tobytes() == qvel.tobytes()
    fired, v, dq, _ = emul_push(lib, model, [_push(11, 1, force=(5, 0, 0))], 10, _dt(env), qpos, qvel)
    assert not fired and v.tobytes() == qvel.tobytes() and np.isnan(dq).all()


def test_heavier_model_takes_a_smaller_push(lib, omodels):
    """Per-instance models: the push is computed on the model it is given; a base 3 kg heavier takes the oracle's
    Delta qvel of that model, whose linear base velocity change is smaller."""
    env = _env("unitree_go2_walk")
    heavy = env.sys.tree_replace({"body_mass": {"base": env.sys.model.arrays["body_mass"][1] + 3.0}}).model
    rng = np.random.default_rng(2)
    qpos, qvel = _random_state(env.sys.model, rng)
    e = [_push(2, 1, (0.05, 0, 0), (80, 0, 0))]
    _, _, dq, _ = emul_push(lib, env.sys.model, e, 2, _dt(env), qpos, qvel)
    _, _, dqh, _ = emul_push(lib, heavy, e, 2, _dt(env), qpos, qvel)
    ref, *_ = oracle_push(omodels(heavy, "go2_heavy"), e, 2, _dt(env), qpos)
    assert np.abs(dqh - ref).max() <= TOL * np.abs(ref).max()
    assert np.linalg.norm(dqh[:3]) < np.linalg.norm(dq[:3])


def test_firing_window_and_sums(lib):
    """An entry fires at post-step counters step .. step + n_steps - 1 only; entries that fire together add up
    (the sum of their separate Delta qvel, within fp64 rounding)."""
    env = _env("unitree_go2_walk")
    model = env.sys.model
    rng = np.random.default_rng(4)
    qpos, qvel = _random_state(model, rng)
    a = _push(5, 1, (0.1, 0, 0), (30, 0, 0), n_steps=3)
    b = _push(7, 4, (0, 0, -0.1), (0, 10, 0), (1, 0, 0))
    fires = [s for s in range(0, 12) if emul_push(lib, model, [a, b], s, _dt(env), qpos, qvel)[0]]
    assert fires == [5, 6, 7]
    big = _push(2**31 - 2, 1, n_steps=2**31 - 1, force=(1, 0, 0))
    assert emul_push(lib, model, [big], 2**31 - 1, _dt(env), qpos, qvel)[0]
    assert not emul_push(lib, model, [big], 2**31 - 3, _dt(env), qpos, qvel)[0]
    _, _, both, _ = emul_push(lib, model, [a, b], 7, _dt(env), qpos, qvel)
    _, _, da, _ = emul_push(lib, model, [a], 7, _dt(env), qpos, qvel)
    _, _, db, _ = emul_push(lib, model, [b], 7, _dt(env), qpos, qvel)
    assert np.abs(both - (da + db)).max() <= 1e-12 * np.abs(both).max()
