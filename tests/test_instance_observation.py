"""Per-instance observation on the CPU: the observe spec (observe_setting) and its errors, the CLI errors of
--observe and of the observe key of --instance-overrides, a NumPy restatement of the ring, the age ramp, the
reset and the prediction's actions against the observe step the kernel runs (observe_advance, observe_record,
observe_emit, on the warp emulator), the noise against a restatement built from the oracle's sampler, and the
prediction launches of lengths age + d against chains of single-row env steps."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from dial_mpc_b200 import _capi
from dial_mpc_b200 import random as drandom
from dial_mpc_b200.utils.spline import interp_matrix
from tests.conftest import make_pair
from tests.test_emul_batch import _instances
from tests.test_instance_delay import Queue

EMUL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
DMAX = _capi.DEFINES["DIAL_MAXDELAY"]
R = DMAX + 1                      # records of one ring (ages 0..16)
MAXV = _capi.DEFINES["DIAL_MAXV"]
# Tolerances of the noise against the oracle's restatement x + sigma eps (fp64, then rounded):
# hinge, slide and velocity dofs: EPS_ULP ulp of sigma eps (the kernels' sampler against XLA's float32
# erfinv, tests/test_gpu_update.py) plus 1 ulp of the result (one rounding of the fused multiply-add);
# the free joint's quaternion: QUAT_TOL per component (the SFU sine and cosine of axisangle, 4e-7, and the
# fast-math square root and reciprocals of the rotation axis and the normalisation).
EPS_ULP = 4
QUAT_TOL = 4e-6


def _go2():
    env, _ = make_pair("unitree_go2_walk")
    return env


def _slidepod():
    from dial_mpc_b200.modelc import compile_mjcf
    return compile_mjcf(os.path.join(os.path.dirname(os.path.abspath(__file__)), "models", "trees", "slidepod.xml"))


# ---- observe_setting and the CLI ----------------------------------------------------------------------
def test_observe_setting_forms():
    from dial_mpc_b200.core.dial_core import observe_setting
    env = _go2()
    nv = env.sys.nv
    k, q, v, key = observe_setting({}, env.sys)
    assert k == 0 and not q.any() and not v.any() and tuple(key) == (0, 0)
    k, q, v, key = observe_setting({"delay": 3, "qpos": 0.01, "qvel": [0.1] * nv, "seed": 7}, env)
    assert k == 3 and q.dtype == np.float32 and np.all(q == np.float32(0.01)) and np.all(v == np.float32(0.1))
    assert tuple(key) == tuple(drandom.PRNGKey(7))
    # joint names: the free joint of Go2 is unnamed (''): one number, or 3 position and 3 rotation
    _, q, v, _ = observe_setting({"qpos": {"": [0.0, 0.0, 0.01, 0.02, 0.02, 0.03], "FR_calf_joint": 0.05},
                                  "qvel": {"": 0.2, "RL_hip_joint": 0.5}}, env.sys)
    want = np.zeros(nv, np.float32)
    want[2:6] = [0.01, 0.02, 0.02, 0.03]
    want[8] = 0.05
    assert np.array_equal(q, want)
    want = np.zeros(nv, np.float32)
    want[:6] = 0.2
    want[15] = 0.5
    assert np.array_equal(v, want)
    # the same resolution as tree_replace's dof fields
    m = env.sys.tree_replace({"dof_damping": {"FR_calf_joint": 9.0}}).model
    assert np.flatnonzero(m.arrays["dof_damping"] == 9.0).tolist() == [8]
    # slide joints
    sp = _slidepod()
    _, q, _, _ = observe_setting({"qpos": {"FL_knee": 0.002}}, sp)
    assert q[sp.arrays["jnt_dofadr"][sp.names["joint"].index("FL_knee")]] == np.float32(0.002) and q.sum() == np.float32(0.002)


@pytest.mark.parametrize("spec, match", [
    (3, r"an observe spec is a mapping"),
    ({"delay": 17}, r"delay must be an int in 0\.\.16, got 17"),
    ({"delay": -1}, r"delay must be an int in 0\.\.16, got -1"),
    ({"delay": 1.0}, r"delay must be an int in 0\.\.16, got 1\.0"),
    ({"delay": True}, r"delay must be an int"),
    ({"lag": 1}, r"unknown key 'lag'"),
    ({"qpos": -0.1}, r"qpos must be a finite number >= 0, got -0\.1"),
    ({"qvel": float("nan")}, r"qvel must be a finite number >= 0, got nan"),
    ({"qpos": [0.1] * 5}, r"qpos must be one number, a list of nv = 18 .* got a list of 5"),
    ({"qpos": [0.1] * 17 + [-1]}, r"qpos\[17\] must be a finite number >= 0, got -1"),
    ({"qpos": {"knee": 0.1}}, r"qpos: unknown joint 'knee'"),
    ({"qpos": {"": [0.1, 0.2]}}, r"qpos: joint '' has 6 dofs: give one number or 6"),
    ({"qvel": {"FR_hip_joint": [0.1, 0.1]}}, r"qvel: joint 'FR_hip_joint' has 1 dofs"),
    ({"qvel": {"FR_hip_joint": "x"}}, r"qvel: FR_hip_joint must be a finite number"),
    ({"seed": -2}, r"seed must be an int in 0\.\.4294967295, got -2"),
    ({"seed": "a"}, r"seed must be an int"),
])
def test_observe_setting_names_the_bad_key_or_value(spec, match):
    from dial_mpc_b200.core.dial_core import observe_setting
    with pytest.raises(ValueError, match=match):
        observe_setting(spec, _go2().sys)


def _main(monkeypatch, capsys, argv):
    from dial_mpc_b200.core import dial_core
    monkeypatch.setattr(sys, "argv", ["dial_core", "--example", "unitree_go2_trot"] + argv)
    with pytest.raises(SystemExit) as e:
        dial_core.main()
    return e.value.code, capsys.readouterr().err


@pytest.mark.parametrize("value, match", [
    ("{delay: 20}", r"--observe: delay must be an int in 0\.\.16, got 20"),
    ("{qpos: -1}", r"--observe: qpos must be a finite number >= 0"),
    ("[1, 2]", r"--observe: an observe spec is a mapping"),
    ("{delay: 1", r"--observe: not a YAML mapping"),
    ("{qvel: {foot: 1}}", r"--observe: qvel: unknown joint 'foot'"),
])
def test_cli_observe_errors(monkeypatch, capsys, value, match):
    code, err = _main(monkeypatch, capsys, ["--observe", value])
    assert code == 2 and re.search(match, err), err


def test_cli_observe_excludes_eager(monkeypatch, capsys):
    code, err = _main(monkeypatch, capsys, ["--observe", "{delay: 1}", "--eager"])
    assert code == 2 and "--observe runs on the CUDA-graph loop; it excludes --eager" in err, err


@pytest.mark.parametrize("entry, match", [
    ({"observe": {"delay": 30}}, r"observe: delay must be an int in 0\.\.16, got 30"),
    ({"observe": {"qpos": "x"}}, r"observe: qpos must be a finite number"),
    ({"observe": 2}, r"observe: an observe spec is a mapping"),
    ({"observe": {"sigma": 1}}, r"observe: unknown key 'sigma'"),
])
def test_cli_instance_override_observe_errors(tmp_path, monkeypatch, capsys, entry, match):
    import yaml
    ov = tmp_path / "ov.yaml"
    ov.write_text(yaml.safe_dump([{"observe": {"delay": 1}}, {}, entry]))
    code, err = _main(monkeypatch, capsys, ["--instances", "3", "--instance-overrides", str(ov)])
    assert code == 2 and re.search(r"--instance-overrides entry 2: " + match, err), err


def test_cli_observe_delay_rejects_randomize_tasks(tmp_path, monkeypatch, capsys):
    import yaml
    from dial_mpc_b200.utils.io_utils import get_example_path
    cfg = yaml.safe_load(open(get_example_path("unitree_go2_trot.yaml")))
    cfg["randomize_tasks"] = True
    path = tmp_path / "rand.yaml"
    path.write_text(yaml.safe_dump(cfg))
    from dial_mpc_b200.core import dial_core
    monkeypatch.setattr(sys, "argv", ["dial_core", "--config", str(path), "--observe", "{delay: 2}"])
    with pytest.raises(SystemExit) as e:
        dial_core.main()
    err = capsys.readouterr().err
    assert e.value.code == 2 and "--observe: an observation delay needs a loop without randomize_tasks" in err, err


# ---- warp emulator -----------------------------------------------------------------------------------
class ObsSetting(C.Structure):
    _fields_ = [("k", C.c_int32), ("on", C.c_int32), ("key", C.c_uint32 * 2), ("sigma", C.c_float * (2 * MAXV))]


class ObsRing(C.Structure):
    _fields_ = [("head", C.c_int32), ("count", C.c_int32), ("key", C.c_uint32 * 2), ("sub", C.c_uint32 * 2)]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    """g++ build of tests/emul/emul_observe.cpp (the device code under the emulator)."""
    so = str(tmp_path_factory.mktemp("emul_observe") / "libdial_emul_observe.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", EMUL, "-shared", "-fPIC", "-o", so,
                           os.path.join(EMUL, "emul_observe.cpp")])
    lib = C.CDLL(so)
    lib.emul_sizeof_obs.restype = C.c_size_t
    assert lib.emul_sizeof_obs(0) == C.sizeof(ObsSetting) and lib.emul_sizeof_obs(1) == C.sizeof(ObsRing)
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _setting(k, q=None, v=None, key=(0, 0), nv=None):
    """The setting dial_plan_set_instance_observation stores."""
    s = ObsSetting()
    s.k = k
    q = np.zeros(nv, np.float32) if q is None else np.asarray(q, np.float32)
    v = np.zeros(nv, np.float32) if v is None else np.asarray(v, np.float32)
    s.on = int(k > 0 or q.any() or v.any())
    s.key[0], s.key[1] = int(key[0]), int(key[1])
    for i in range(len(q)):
        s.sigma[i] = q[i]
        s.sigma[len(q) + i] = v[i]
    return s


class Device:
    """One instance's ring and outputs, stepped by the emulator's observe step."""

    def __init__(self, lib, md, setting):
        self.lib, self.md = lib, md
        nq, nv, nu = md.nq, md.nv, md.nu
        self.rq, self.rv, self.rw = (np.zeros((R, n), np.float32) for n in (nq, nv, nv))
        self.ra, self.rc = np.zeros((R, nu), np.float32), np.zeros((R, 2), np.int32)
        self.reset(setting)

    def reset(self, setting):
        """dial_plan_set_instance_observation: the setting, and the ring emptied with the setting's key."""
        self.s = setting
        self.r = ObsRing()
        self.r.key[0], self.r.key[1] = setting.key[0], setting.key[1]

    def step(self, plant, act, env_step, d=0, predict=False, pending=None, threads=3):
        md = self.md
        nq, nv, nu = md.nq, md.nv, md.nu
        out = dict(oq=np.full(nq, np.nan, np.float32), ov=np.full(nv, np.nan, np.float32),
                   ow=np.full(nv, np.nan, np.float32), oc=np.full(2, -7, np.int32),
                   pq=np.full(nq, np.nan, np.float32), pv=np.full(nv, np.nan, np.float32),
                   pw=np.full(nv, np.nan, np.float32), pc=np.full(2, -7, np.int32),
                   seq=np.full((DMAX, nu), np.nan, np.float32))
        age, ln = C.c_int32(-1), C.c_int32(-1)
        pend = None if pending is None else np.ascontiguousarray(pending, np.float32)
        a = None if act is None else np.ascontiguousarray(act, np.float32)
        assert self.lib.emul_observe_step(
            C.byref(md), C.byref(self.s), C.byref(self.r), int(env_step), d, int(predict), _p(pend),
            _p(plant["qpos"]), _p(plant["qvel"]), _p(plant["warm"]), _p(plant["cnt"]), _p(a),
            _p(self.rq), _p(self.rv), _p(self.rw), _p(self.ra), _p(self.rc),
            _p(out["oq"]), _p(out["ov"]), _p(out["ow"]), _p(out["oc"]), _p(out["pq"]), _p(out["pv"]),
            _p(out["pw"]), _p(out["pc"]), _p(out["seq"]), C.byref(age), C.byref(ln), threads) == 0
        for x, y in (("oq", "pq"), ("ov", "pv"), ("ow", "pw"), ("oc", "pc")):
            assert np.array_equal(out[x], out[y], equal_nan=False), x   # the planning state starts as the observation
        out.update(age=age.value, len=ln.value)
        return out


class History:
    """The semantics of include/dial_b200.h restated: records since the reset, each with its noise key."""

    def __init__(self, k, key, nu):
        self.k, self.key, self.nu, self.rec = k, np.array(key, np.uint32), nu, []

    def push(self, plant, act):
        self.key, sub = drandom.split(self.key)
        self.rec.append(dict({n: plant[n].copy() for n in plant}, act=None if act is None else act.copy(), sub=sub))

    def observe(self, plant, act, env_step, d, pending):
        if not self.rec or env_step:
            self.push(plant, act if env_step else None)
        age = min(self.k, len(self.rec) - 1)
        obs = self.rec[-1 - age]
        seq = np.zeros((DMAX, self.nu), np.float32)
        for j in range(age):
            seq[j] = self.rec[-age + j]["act"]
        for j in range(d):
            seq[age + j] = pending[j]
        return obs, age, seq, self.rec[-1]["sub"]


def _plant(rng, md, step):
    return dict(qpos=rng.normal(size=md.nq).astype(np.float32), qvel=rng.normal(size=md.nv).astype(np.float32),
                warm=rng.normal(size=md.nv).astype(np.float32), cnt=np.array([step, step // 7], np.int32))


@pytest.mark.parametrize("k, d", [(0, 0), (1, 0), (3, 0), (5, 2), (DMAX, 0), (4, DMAX - 4)])
def test_ring_equals_restatement(lib, k, d):
    """Zero noise: the observation is the record min(k, c - 1) pushes back, bit for bit, with its counters; the
    prediction's actions are the actions applied since it, oldest first, then the d pending rows, and the
    length age + d when predicting.  Steps without an env step (env_step 0 or 2) observe the same record; a
    reset (a new setting or set_state) seeds the ring again."""
    env = _go2()
    md = _capi.fill_model_desc(env.sys.model)
    nu = md.nu
    rng = np.random.default_rng(100 * k + d)
    y0 = rng.uniform(-1, 1, nu).astype(np.float32)
    Q = Queue(d, y0)
    dev = Device(lib, md, _setting(k, nv=md.nv))
    ref = History(k, (0, 0), nu)
    step = 40
    plant = _plant(rng, md, step)
    for t in range(3 * DMAX + 8):
        env_step = t % 6 not in (2, 4)          # env_step 0 / 2 now and then: no record
        if t == 2 * DMAX:                       # set_state: a new plant state, the ring reset
            plant = _plant(rng, md, 7)
            dev.reset(_setting(k, nv=md.nv))
            ref = History(k, (0, 0), nu)
        y = rng.uniform(-1, 1, nu).astype(np.float32)
        act, pend = Q.step(y, env_step)
        if env_step:
            step += 1
            plant = _plant(rng, md, step)
        got = dev.step(plant, act, env_step, d, True, pend, threads=1 + t % 4)
        obs, age, seq, _ = ref.observe(plant, act, env_step, d, pend)
        assert got["age"] == age == min(k, len(ref.rec) - 1), t
        assert got["len"] == age + d, t
        for a, b in (("oq", "qpos"), ("ov", "qvel"), ("ow", "warm"), ("oc", "cnt")):
            assert np.array_equal(got[a], obs[b]), (t, a)
        assert np.array_equal(got["seq"], seq), t
        if k == 0:
            assert np.array_equal(got["oq"], plant["qpos"]) and np.array_equal(got["ov"], plant["qvel"])
    assert len(ref.rec) > k    # past the ramp


def test_change_of_delay_resets(lib):
    """A new k: the ring is seeded again, so the ramp starts over at age 0."""
    env = _go2()
    md = _capi.fill_model_desc(env.sys.model)
    rng = np.random.default_rng(3)
    dev = Device(lib, md, _setting(4, nv=md.nv))
    ages = []
    for t in range(14):
        if t == 7:
            dev.reset(_setting(2, nv=md.nv))
        ages.append(dev.step(_plant(rng, md, t), rng.normal(size=md.nu), True)["age"])
    assert ages == [0, 1, 2, 3, 4, 4, 4, 0, 1, 2, 2, 2, 2, 2]


def test_no_setting_copies_the_plant(lib):
    """An instance without a setting (k = 0, every sigma 0) plans from its plant state; its prediction is its
    queue."""
    env = _go2()
    md = _capi.fill_model_desc(env.sys.model)
    rng = np.random.default_rng(4)
    dev = Device(lib, md, _setting(0, nv=md.nv))
    pend = rng.normal(size=(DMAX, md.nu)).astype(np.float32)
    for t in range(3):
        p = _plant(rng, md, t)
        got = dev.step(p, None, t % 2, d=3, predict=True, pending=pend)
        assert np.array_equal(got["oq"], p["qpos"]) and np.array_equal(got["ov"], p["qvel"])
        assert np.array_equal(got["oc"], p["cnt"]) and got["age"] == 0 and got["len"] == 3
        assert np.array_equal(got["seq"][:3], pend[:3]) and not got["seq"][3:].any()
    assert dev.r.count == 0


def _noise_ref(model, rec, sub, sq, sv):
    """The observation of record `rec` restated from the oracle: eps = jax_normal_legacy_xla(sub, 2 nv) in fp64;
    returns (qpos, qvel) in fp64 and, per free joint, its qpos address of the quaternion and the fp64
    quaternion."""
    from oracle.planner_oracle import jax_normal_legacy_xla
    from scipy.spatial.transform import Rotation
    nv = model.nv
    eps = jax_normal_legacy_xla(np.asarray(sub, np.uint32), (2 * nv,)).astype(np.float32).astype(np.float64)
    q = rec["qpos"].astype(np.float64)
    v = rec["qvel"].astype(np.float64) + sv.astype(np.float64) * eps[nv:]
    quats = []
    for j, t in enumerate(model.arrays["jnt_type"]):
        qa, dd = int(model.arrays["jnt_qposadr"][j]), int(model.arrays["jnt_dofadr"][j])
        if t == 0:
            q[qa:qa + 3] += sq[dd:dd + 3] * eps[dd:dd + 3]
            w = sq[dd + 3:dd + 6].astype(np.float64) * eps[dd + 3:dd + 6]
            q0 = rec["qpos"][qa + 3:qa + 7].astype(np.float64)
            if w.any():
                r = Rotation.from_quat(np.r_[q0[1:], q0[0]]) * Rotation.from_rotvec(w)
                x = r.as_quat()
                x = np.r_[x[3], x[:3]]
                x *= np.sign(x @ q0)     # the hemisphere of q (the kernel does not canonicalise)
                q[qa + 3:qa + 7] = x
            quats.append(qa + 3)
        else:
            q[qa] += sq[dd] * eps[dd]
    return q, v, quats, eps


def _ulp(x):
    return np.spacing(np.abs(np.float32(x))).astype(np.float64)


@pytest.mark.parametrize("name", ["go2", "slidepod"])
def test_noise_equals_oracle_restatement(lib, name):
    """The noise over a run with pushes, steps without one and a reset, against the key chain of
    dial_mpc_b200.random.split and the oracle's jax_normal_legacy_xla: hinge, slide and velocity dofs within
    EPS_ULP ulp of sigma eps + 1 ulp, the free joint's quaternion within QUAT_TOL and of unit norm; dofs whose
    sigma is 0 (and the quaternion whose rotation sigma are 0) copied bit for bit."""
    model = _go2().sys.model if name == "go2" else _slidepod()
    md = _capi.fill_model_desc(model)
    nv = md.nv
    rng = np.random.default_rng(9)
    sq = rng.uniform(0.0, 0.1, nv).astype(np.float32)
    sv = rng.uniform(0.0, 0.5, nv).astype(np.float32)
    sq[1] = sq[7] = sq[nv - 1] = 0.0   # a position, a joint and the last dof exactly
    sv[0] = sv[9] = 0.0
    key = drandom.PRNGKey(5)
    dev = Device(lib, md, _setting(2, sq, sv, key, nv))
    ref = History(2, key, md.nu)
    worst = 0.0
    for t in range(12):
        if t == 8:
            dev.reset(_setting(2, sq, sv, key, nv))
            ref = History(2, key, md.nu)
        env_step = t % 4 != 3
        p = _plant(rng, md, t)
        for j, typ in enumerate(model.arrays["jnt_type"]):
            if typ == 0:
                qa = model.arrays["jnt_qposadr"][j] + 3
                p["qpos"][qa:qa + 4] = (p["qpos"][qa:qa + 4] * 1.01).astype(np.float32)   # not quite unit
        a = rng.normal(size=md.nu).astype(np.float32)
        got = dev.step(p, a, env_step)
        rec, age, _, sub = ref.observe(p, a, env_step, 0, None)
        assert got["age"] == age
        q, v, quats, eps = _noise_ref(model, rec, sub, sq, sv)
        qmask = np.ones(md.nq, bool)
        for qa in quats:
            qmask[qa:qa + 4] = False
        # tangent dofs of qpos: positions of free joints, hinges and slides
        dof_of_q = np.full(md.nq, -1)
        for j, typ in enumerate(model.arrays["jnt_type"]):
            qa, dd = int(model.arrays["jnt_qposadr"][j]), int(model.arrays["jnt_dofadr"][j])
            for i in range(3 if typ == 0 else 1):
                dof_of_q[qa + i] = dd + i
        for i in np.flatnonzero(qmask):
            dd = dof_of_q[i]
            if sq[dd] == 0:
                assert got["oq"][i].tobytes() == rec["qpos"][i].tobytes(), (t, i)
                continue
            tol = EPS_ULP * float(sq[dd]) * _ulp(eps[dd]) + _ulp(q[i])
            assert abs(got["oq"][i] - q[i]) <= tol, (t, i, got["oq"][i], q[i], tol)
            worst = max(worst, abs(got["oq"][i] - q[i]) / tol)
        for i in range(nv):
            if sv[i] == 0:
                assert got["ov"][i].tobytes() == rec["qvel"][i].tobytes(), (t, i)
                continue
            tol = EPS_ULP * float(sv[i]) * _ulp(eps[nv + i]) + _ulp(v[i])
            assert abs(got["ov"][i] - v[i]) <= tol, (t, i, got["ov"][i], v[i], tol)
            worst = max(worst, abs(got["ov"][i] - v[i]) / tol)
        for qa in quats:
            assert np.abs(got["oq"][qa:qa + 4] - q[qa:qa + 4]).max() <= QUAT_TOL, (t, got["oq"][qa:qa + 4], q[qa:qa + 4])
            assert abs(np.linalg.norm(got["oq"][qa:qa + 4].astype(np.float64)) - 1) < 1e-6
        assert np.array_equal(got["ow"], rec["warm"]) and np.array_equal(got["oc"], rec["cnt"])
    assert worst <= 1.0


def test_zero_rotation_sigma_keeps_the_quaternion(lib):
    """A free joint whose three rotation sigma are 0 keeps its (unnormalised) quaternion bit for bit, and an
    observation with every sigma 0 equals its record."""
    model = _go2().sys.model
    md = _capi.fill_model_desc(model)
    rng = np.random.default_rng(2)
    sq = np.zeros(md.nv, np.float32)
    sq[:3] = 0.05
    dev = Device(lib, md, _setting(1, sq, None, (0, 3), md.nv))
    zero = Device(lib, md, _setting(1, None, None, (0, 3), md.nv))
    for t in range(4):
        p = _plant(rng, md, t)
        a = rng.normal(size=md.nu).astype(np.float32)
        g, z = dev.step(p, a, True), zero.step(p, a, True)
        assert g["oq"][3:7].tobytes() == z["oq"][3:7].tobytes()
        assert not np.array_equal(g["oq"][:3], z["oq"][:3])
        if t > 0:
            assert np.array_equal(z["oq"], zero.rq[(zero.r.head - 1) % R])


@pytest.fixture(scope="module")
def delay_lib(tmp_path_factory):
    """g++ build of tests/emul/emul_delay.cpp (its env-step launch)."""
    so = str(tmp_path_factory.mktemp("emul_delay") / "libdial_emul_delay.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", EMUL, "-shared", "-fPIC", "-o", so,
                           os.path.join(EMUL, "emul_delay.cpp")])
    return C.CDLL(so)


def test_prediction_launches_over_history_and_queue(delay_lib):
    """The prediction launches of an observing step: instance b starts from its observed record and takes
    age_b + d_b single-row env steps with its sequence (history rows, then pending rows).  Three Go2 seq-jump
    instances with (age, d) = (0, 0), (2, 1), (3, 2) equal, bit for bit, chains of single-instance env steps,
    across the first stage boundary of the jump sequence (the step from 49)."""
    dl = delay_lib
    env, o = make_pair("unitree_go2_seq_jump")
    B, Hn = 3, 3
    nu = env.action_size
    rng = np.random.default_rng(12)
    qpos, qvel, warm, _ = _instances(o, B, nu, Hn, rng)
    qpos, qvel, warm = (np.ascontiguousarray(a, np.float32) for a in (qpos, qvel, warm))
    counters = np.array([[49, 0], [47, 0], [46, 0]], np.int32)
    lens = np.array([0, 3, 5], np.int32)
    seq = np.zeros((B, DMAX, nu), np.float32)
    for b in range(B):
        seq[b, :lens[b]] = rng.uniform(-1, 1, (lens[b], nu))
    desc = env.plan_desc(Nsample=4, Hsample=6, Hnode=Hn, temp_sample=0.05,
                         M_n2u=interp_matrix(np.linspace(0, 1, Hn + 1), np.linspace(0, 1, 7)), n_inst=B)
    md = _capi.fill_model_desc(env.sys.model)
    bat = dict(qpos=qpos.copy(), qvel=qvel.copy(), warm=warm.copy(), cnt=counters.copy())
    rew = np.zeros(B, np.float32)
    for j in range(int(lens.max())):
        assert dl.emul_env_launch(C.byref(md), C.byref(desc), B, 1, _p(seq[:, j:]), DMAX * nu, _p(lens), j,
                                  _p(bat["qpos"]), _p(bat["qvel"]), _p(bat["warm"]), _p(bat["cnt"]), _p(rew)) == 0
    for b in range(B):
        one = dict(qpos=qpos[b:b + 1].copy(), qvel=qvel[b:b + 1].copy(), warm=warm[b:b + 1].copy(),
                   cnt=counters[b:b + 1].copy())
        r1 = np.zeros(1, np.float32)
        for j in range(lens[b]):
            act = np.ascontiguousarray(seq[b, j][None])
            assert dl.emul_env_launch(C.byref(md), C.byref(desc), 1, 0, _p(act), 0, None, 0, _p(one["qpos"]),
                                      _p(one["qvel"]), _p(one["warm"]), _p(one["cnt"]), _p(r1)) == 0
        for k in ("qpos", "qvel", "warm", "cnt"):
            assert np.array_equal(bat[k][b], one[k][0]), (b, k)
        assert bat["cnt"][b, 0] == counters[b, 0] + lens[b]
    assert bat["cnt"][1, 1] == 1 and bat["cnt"][2, 1] == 1
