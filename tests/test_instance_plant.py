"""CPU tests of per-instance plant fidelity (dial_plan_set_instance_plant): one env step of the plant, run by the
warp emulator on the plant's model and plan descriptor (timestep / k, n_frames * k, the setting's solver
settings) against the fp64 oracle's env step with the same settings; the plant spec parser; the struct layout."""
import ctypes as C
import re
import sys

import numpy as np
import pytest

from dial_mpc_b200 import _capi
from dial_mpc_b200.core.dial_core import plant_setting
from tests.conftest import make_pair
from tests.emul import emul

KMAX = _capi.DEFINES["DIAL_MAXSUBSTEPS"]


def plant_descs(env, k, iterations=None, ls_iterations=None, tolerance=None):
    """The plant's model and plan descriptors as the library derives them: the model's timestep / k in fp32 and
    the given solver settings, n_frames * k; everything else the plan's."""
    md = _capi.fill_model_desc(env.sys.model)
    md.timestep = float(np.float32(md.timestep) / np.float32(k))
    if iterations is not None:
        md.iterations, md.ls_iterations, md.tolerance = iterations, ls_iterations, tolerance
    desc = env.plan_desc()
    desc.n_frames = desc.n_frames * k
    return md, desc


def emul_env_step(env, md, desc, q, v, w, a, step0, **kw):
    """One env step (mode 0, one row, H = 1) of the device code on the descriptors given; ``kw``: emul.launch's."""
    nq, nv, nu, nb = md.nq, md.nv, md.nu, md.nbody
    f32 = lambda x: np.ascontiguousarray(x, dtype=np.float32)
    out = dict(rewss=np.zeros((1, 1), np.float32), rews=np.zeros(1, np.float32), q=np.zeros((1, 1, nq), np.float32),
               qd=np.zeros((1, 1, nv), np.float32), xpos=np.zeros((1, 1, nb - 1, 3), np.float32),
               qpos_out=np.zeros(nq, np.float32), qvel_out=np.zeros(nv, np.float32), warm_out=np.zeros(nv, np.float32),
               ctrl_out=np.zeros(nu, np.float32))
    emul.launch(md, desc, reward_source=getattr(env, "reward_source", None) or None, mode=0, nrows=1, H=1, step0=step0,
                qpos0=f32(q), qvel0=f32(v), warm0=f32(w), us=f32(np.asarray(a).reshape(1, 1, nu)), **out, **kw)
    return out


class fine_oracle:
    """The oracle env with its env step made of n_frames * k physics steps of timestep / k under the given solver
    settings (restored on exit)."""

    def __init__(self, o, k, iterations=None, ls_iterations=None, tolerance=None):
        self.o, self.k, self.solver = o, k, (iterations, ls_iterations, tolerance)

    def __enter__(self):
        o, m = self.o, self.o.m
        self.saved = (o.n_frames, m.timestep, m.iterations, m.ls_iterations, m.tolerance)
        o.n_frames, m.timestep = o.n_frames * self.k, m.timestep / self.k
        if self.solver[0] is not None:
            m.iterations, m.ls_iterations, m.tolerance = self.solver
        return o

    def __exit__(self, *exc):
        o, m = self.o, self.o.m
        o.n_frames, m.timestep, m.iterations, m.ls_iterations, m.tolerance = self.saved


def mid_run_states(o, n, seed, scale=0.6):
    """Oracle states after a few env steps under random actions (contacts active), with the next action."""
    rng = np.random.default_rng(seed)
    s = o.reset()
    out = []
    for i in range(n):
        for _ in range(3):
            s, _, _ = o.step(s, np.clip(rng.normal(size=(1, o.nu)) * scale, -1, 1))
        out.append((s, np.clip(rng.normal(size=(1, o.nu)) * scale, -1, 1)))
    return out


def check_plant_step(env, o, ks, solver=(None, None, None), n=2, seed=0, scale=0.6):
    """For each k: the emulated plant env step equals the oracle's fine env step from the same states; returns
    {k: [qpos_out per state]}."""
    states = mid_run_states(o, n, seed, scale)
    got = {}
    for k in ks:
        md, desc = plant_descs(env, k, *solver)
        got[k] = []
        for s, a in states:
            step0 = int(s.step[0])
            out = emul_env_step(env, md, desc, s.qpos[0], s.qvel[0], s.qacc_warmstart[0], a[0], step0)
            with fine_oracle(o, k, *solver):
                ns, r, aux = o.step(s, a)
            # the tolerances of the emulator's rollout parity tests (tests/test_emul_parity.py)
            assert np.abs(out["qpos_out"] - ns.qpos[0]).max() < 1e-4, k
            assert np.abs(out["qvel_out"] - ns.qvel[0]).max() < 5e-3 * (1 + np.abs(ns.qvel[0]).max() / 10), k
            assert np.abs(out["rewss"][0, 0] - r[0]) < 1e-3 * (1 + abs(r[0])), k
            # the control is computed once, from the pre-step state, and held
            assert np.abs(out["ctrl_out"] - aux["ctrl"][0]).max() < 1e-4 * (1 + np.abs(aux["ctrl"][0]).max()), k
            got[k].append(out["qpos_out"])
    return got


def finer_differs(got, k=4, thr=1e-3):
    return max(np.abs(a - b).max() for a, b in zip(got[k], got[1])) > thr


@pytest.mark.parametrize("solver", [(None, None, None), (100, 50, 1e-8)], ids=["plan_solver", "mujoco_solver"])
def test_go2_plant_step_matches_fine_oracle(solver):
    env, o = make_pair("unitree_go2_walk")
    ks = (1, 2, 4) if solver[0] is None else (4,)
    got = check_plant_step(env, o, ks, solver)
    if solver[0] is None:
        assert finer_differs(got)   # four substeps are not one: the comparison can fail


def test_h1_plant_step_matches_fine_oracle():
    """star<5,7>; the plan's iterations = 1 never reaches the tolerance exit, iterations = 4 does."""
    env, o = make_pair("unitree_h1_loco")
    assert env.sys.model.iterations == 1
    got = check_plant_step(env, o, (1, 2, 4), (4, 6, 1e-4))
    assert finer_differs(got)


@pytest.mark.parametrize("name", ["branchpod", "hexapod"])
def test_tree_plant_step_matches_fine_oracle(name):
    from tests.tree_envs import make_tree_pair
    env, o = make_tree_pair(name)
    got = check_plant_step(env, o, (1, 2, 4), (3, 8, 1e-6))
    assert finer_differs(got)


def test_allegro_plant_step_matches_fine_oracle():
    env, o = make_pair("allegro_reorient")
    got = check_plant_step(env, o, (1, 2), scale=0.4)
    assert max(np.abs(a - b).max() for a, b in zip(got[2], got[1])) > 1e-5


def test_identity_setting_is_the_plan():
    """substeps 1 with the plan's solver settings: the plant descriptors are the plan's, bit for bit."""
    for name in ("unitree_go2_walk", "unitree_h1_loco", "allegro_reorient"):
        env, _ = make_pair(name)
        f = plant_setting({}, env.sys)
        md, desc = plant_descs(env, f.substeps, f.iterations, f.ls_iterations, f.tolerance)
        assert bytes(md) == bytes(_capi.fill_model_desc(env.sys.model)) and bytes(desc) == bytes(env.plan_desc())


# ---- plant_setting ------------------------------------------------------------------------------------
def test_plant_setting_defaults_and_sim_dt():
    env, _ = make_pair("unitree_go2_walk")
    m = env.sys.model
    assert plant_setting(None, env.sys) is None
    f = plant_setting({}, env.sys)
    assert (f.substeps, f.iterations, f.ls_iterations) == (1, m.iterations, m.ls_iterations)
    assert f.tolerance == np.float32(m.tolerance)
    f = plant_setting({"sim_dt": 0.005, "iterations": 100, "ls_iterations": 50, "tolerance": 1e-8}, env)
    assert (f.substeps, f.iterations, f.ls_iterations) == (4, 100, 50) and f.tolerance == np.float32(1e-8)
    assert plant_setting({"substeps": 16}, env.sys.model).substeps == 16
    a, _ = make_pair("allegro_reorient")    # timestep 0.005, dt 0.02: sim_dt 0.0025 is 2 substeps
    assert plant_setting({"sim_dt": 0.0025}, a.sys).substeps == 2


@pytest.mark.parametrize("spec, match", [
    ([4], r"a plant spec is a mapping"),
    ({"substep": 4}, r"unknown key 'substep'"),
    ({"substeps": 2, "sim_dt": 0.01}, r"substeps or sim_dt, not both"),
    ({"substeps": 0}, r"substeps must be an int in 1\.\.16, got 0"),
    ({"substeps": 17}, r"substeps must be an int in 1\.\.16, got 17"),
    ({"substeps": 2.0}, r"substeps must be an int"),
    ({"substeps": True}, r"substeps must be an int"),
    ({"sim_dt": 0.003}, r"sim_dt 0\.003 must divide the model's timestep 0\.02"),
    ({"sim_dt": 0.04}, r"sim_dt 0\.04 must divide"),
    ({"sim_dt": 0.001}, r"sim_dt 0\.001 gives 20 substeps of the model's timestep 0\.02, at most 16"),
    ({"sim_dt": -0.005}, r"sim_dt must be a finite number > 0"),
    ({"sim_dt": float("nan")}, r"sim_dt must be a finite number > 0"),
    ({"iterations": 0}, r"iterations must be an int in 1\.\.100, got 0"),
    ({"iterations": 101}, r"iterations must be an int in 1\.\.100, got 101"),
    ({"ls_iterations": 51}, r"ls_iterations must be an int in 1\.\.50, got 51"),
    ({"tolerance": -1e-8}, r"tolerance must be a finite number >= 0"),
    ({"tolerance": float("inf")}, r"tolerance must be a finite number >= 0"),
    ({"tolerance": "1e-8"}, r"tolerance must be a finite number >= 0"),
])
def test_plant_setting_rejections(spec, match):
    env, _ = make_pair("unitree_go2_walk")
    with pytest.raises(ValueError, match=match):
        plant_setting(spec, env.sys)


# ---- CLI ------------------------------------------------------------------------------------------------
def _main(monkeypatch, capsys, argv):
    from dial_mpc_b200.core import dial_core
    monkeypatch.setattr(sys, "argv", ["dial_core", "--example", "unitree_go2_trot"] + argv)
    with pytest.raises(SystemExit) as e:
        dial_core.main()
    return e.value.code, capsys.readouterr().err


@pytest.mark.parametrize("value, match", [
    ("{substeps: 0}", r"--plant: substeps must be an int in 1\.\.16"),
    ("{sim_dt: 0.003}", r"--plant: sim_dt 0\.003 must divide"),
    ("[4]", r"--plant: a plant spec is a mapping"),
    ("{a: [", r"--plant: not a YAML mapping"),
])
def test_cli_plant_errors(monkeypatch, capsys, value, match):
    code, err = _main(monkeypatch, capsys, ["--plant", value])
    assert code == 2 and re.search(match, err), err


def test_cli_plant_excludes_eager(monkeypatch, capsys):
    code, err = _main(monkeypatch, capsys, ["--plant", "{substeps: 4}", "--eager"])
    assert code == 2 and "--plant runs on the CUDA-graph loop; it excludes --eager" in err, err


def test_cli_instance_override_plant_errors(tmp_path, monkeypatch, capsys):
    import yaml
    ov = tmp_path / "ov.yaml"
    ov.write_text(yaml.safe_dump([{"plant": {"substeps": 4}}, {}, {"plant": {"iterations": 500}}]))
    code, err = _main(monkeypatch, capsys, ["--instances", "3", "--instance-overrides", str(ov)])
    assert code == 2 and re.search(r"--instance-overrides entry 2: plant: iterations must be an int in 1\.\.100", err), err


# ---- C ABI ----------------------------------------------------------------------------------------------
def test_plant_struct_layout():
    assert C.sizeof(_capi.dial_plant) == 16
    assert [f for f, _ in _capi.dial_plant._fields_] == ["substeps", "iterations", "ls_iterations", "tolerance"]
    assert KMAX == 16


def test_library_struct_layout_and_symbol(built):
    lib = _capi.lib()
    assert lib.dial_sizeof(6) == C.sizeof(_capi.dial_plant) == 16
    assert hasattr(lib, "dial_plan_set_instance_plant") and "dial_plan_set_instance_plant" in _capi.EXPORTS
    assert lib.dial_abi_version() == 14
