"""CPU tests of per-instance models: ``System.tree_replace`` / ``CompiledModel.set_const``, the check of
``dial_plan_set_instance_model`` and, through the warp emulator, batched launches whose instances run their
own models (bitwise equal to single-instance launches on each model)."""
import ctypes as C
import os
import xml.etree.ElementTree as ET

import numpy as np
import pytest

from dial_mpc_b200 import _capi
from dial_mpc_b200.modelc.mjcf import compile_mjcf
from dial_mpc_b200.utils.spline import interp_matrix
from tests.conftest import make_pair
from tests.emul import emul
from tests.test_emul_batch import rollout_batched

HERE = os.path.dirname(os.path.abspath(__file__))
GO2_XML = os.path.join(HERE, "golden", "unitree_go2")
FEET = ("FR", "FL", "RR", "RL")
DERIVED = ("body_invweight0", "dof_invweight0")


def _go2():
    import dial_mpc_b200.envs as E
    return E.get_environment("unitree_go2_walk", config=E.get_config("unitree_go2_walk")())


# ---- tree_replace / set_const --------------------------------------------------------------------------
def test_tree_replace_changes_exactly_the_named_entries():
    sys0 = _go2().sys
    m0 = sys0.model
    ref = {k: v.copy() for k, v in m0.arrays.items()}
    fr = [0.4, 0.4, 0.02, 0.01, 0.01]
    s = sys0.tree_replace({"body_mass": {"base": 10.921}, "pair_friction": {"RR": fr},
                           "dof_damping": {"FL_calf_joint": 1.3, "": [0, 0, 0, 0.1, 0.2, 0.3]},
                           "actuator_gear": {"FR_thigh": 2.0}, "opt.gravity": [0, 0, -3.7], "opt.timestep": 0.004})
    m = s.model
    want = {k: v.copy() for k, v in ref.items()}
    want["body_mass"][m0.body_id("base")] = 10.921
    want["pair_friction"][[m0.names["geom"][g] for g in m0.arrays["pair_geom2"]].index("RR")] = fr
    want["dof_damping"][m0.arrays["jnt_dofadr"][m0.names["joint"].index("FL_calf_joint")]] = 1.3
    want["dof_damping"][:6] = [0, 0, 0, 0.1, 0.2, 0.3]               # the free joint (name "") has 6 dofs
    want["actuator_gear"][m0.names["actuator"].index("FR_thigh")] = 2.0
    assert set(m.arrays) == set(want)
    for k in want:
        assert np.array_equal(m.arrays[k], want[k]), k
    assert np.array_equal(m.gravity, [0, 0, -3.7]) and m.timestep == 0.004
    # the original model is untouched
    for k in ref:
        assert np.array_equal(m0.arrays[k], ref[k]), k
    assert np.array_equal(m0.gravity, [0, 0, -9.81]) and m0.timestep == _go2().sys.model.timestep != 0.004
    # a full array replaces the whole field
    full = np.arange(m0.nbody, dtype=np.float64)
    assert np.array_equal(sys0.tree_replace({"body_mass": full}).model.arrays["body_mass"], full)


def test_tree_replace_leaves_derived_constants():
    m0 = _go2().sys.model
    m = _go2().sys.tree_replace({"body_mass": {"base": 1.0}, "body_inertia": {"base": [0.1, 0.2, 0.3]}}).model
    for k in DERIVED:
        assert np.array_equal(m.arrays[k], m0.arrays[k]), k
    assert m.meaninertia == m0.meaninertia
    m.set_const()
    assert not np.array_equal(m.arrays["body_invweight0"], m0.arrays["body_invweight0"])
    assert m.meaninertia != m0.meaninertia


def test_tree_replace_with_set_const_matches_compile_of_an_edited_xml(tmp_path):
    for f in os.listdir(GO2_XML):
        tree = ET.parse(os.path.join(GO2_XML, f))
        for body in tree.getroot().iter("body"):
            if body.get("name") == "base":
                body.find("inertial").set("mass", "1e-12")
        tree.write(tmp_path / f)
    edited = compile_mjcf(str(tmp_path / "mjx_scene_force.xml"))
    m = _go2().sys.tree_replace({"body_mass": {"base": 1e-12}}).model.set_const()
    assert set(m.arrays) == set(edited.arrays)
    for k in m.arrays:
        np.testing.assert_allclose(m.arrays[k], edited.arrays[k], rtol=1e-12, atol=0, err_msg=k)
    np.testing.assert_allclose(m.meaninertia, edited.meaninertia, rtol=1e-12)
    assert edited.arrays["body_mass"][1] == 1e-12


@pytest.mark.parametrize("key", ["body_parentid", "pair_kind", "jnt_range", "actuator_ctrlrange", "nq", "opt.cone",
                                 "body_invweight0", "no_such_field"])
def test_tree_replace_rejects_structural_and_unknown_keys(key):
    with pytest.raises(KeyError, match="not a replaceable"):
        _go2().sys.tree_replace({key: 1})


def test_tree_replace_rejects_unknown_names_and_shapes():
    s = _go2().sys
    with pytest.raises(KeyError, match="body 'torso'"):
        s.tree_replace({"body_mass": {"torso": 1.0}})
    with pytest.raises(KeyError, match="moving geom is 'floor'"):
        s.tree_replace({"pair_friction": {"floor": [1, 1, 0, 0, 0]}})
    with pytest.raises(ValueError, match="shape"):
        s.tree_replace({"body_mass": np.ones(3)})


def test_assigning_sys_drops_the_cached_plan():
    env = _go2()
    env._plan = object()
    env.sys = env.sys.tree_replace({"body_mass": {"base": 10.0}})
    assert env._plan is None and env.sys.model.arrays["body_mass"][1] == 10.0


# ---- emulator: the set_instance_model check and batched launches ---------------------------------------
@pytest.fixture(scope="module")
def lib():
    return emul.build()


def _difference(lib, a, b):
    out = C.create_string_buffer(256)
    rc = lib.emul_instance_model_difference(C.byref(a), C.byref(b), out, 256)
    return None if rc == 0 else out.value.decode()


def test_instance_model_check_names_the_field(lib):
    m0 = _go2().sys.model
    d0 = _capi.fill_model_desc(m0)
    ok = _go2().sys.tree_replace({"body_mass": {"base": 10.9}, "pair_friction": {f: [0.4, 0.4, 0.02, 0.01, 0.01] for f in FEET},
                                  "dof_damping": m0.arrays["dof_damping"] * 2, "actuator_gear": {"FR_hip": 0.8},
                                  "opt.gravity": [0.1, 0, -9.7]}).model.set_const()
    assert _difference(lib, d0, _capi.fill_model_desc(ok)) is None
    three = _capi.dial_model_desc.from_buffer_copy(d0)            # one foot contact fewer
    three.npair, three.ncon = 3, 3
    assert _difference(lib, d0, three) == "ncon"
    dt = _capi.fill_model_desc(_go2().sys.tree_replace({"opt.timestep": 0.004}).model)
    assert _difference(lib, d0, dt) == "timestep"
    jr = _capi.dial_model_desc.from_buffer_copy(d0)
    jr.jnt_range[3][1] += 0.1
    assert _difference(lib, d0, jr) == "jnt_range"
    cr = _capi.dial_model_desc.from_buffer_copy(d0)
    cr.actuator_ctrlrange[0][0] -= 1.0
    assert _difference(lib, d0, cr) == "actuator_ctrlrange"
    par = _capi.dial_model_desc.from_buffer_copy(d0)
    par.pair_geom2[0], par.pair_geom2[1] = par.pair_geom2[1], par.pair_geom2[0]
    assert _difference(lib, d0, par) == "pair_geom2"


def rollout_models(base_model, models, desc, wpc, *args, **kw):
    """Rows as dial_mpc_step launches them (tests/test_emul_batch.py), instance b on models[b] (None: the plan's
    model), in CTAs of ``wpc`` warps."""
    return rollout_batched(base_model, desc, *args, models=models, wpc=wpc, **kw)


def test_seq_jump_instance_models_equal_single_instance_plans():
    env, o = make_pair("unitree_go2_seq_jump")
    m0 = env.sys.model
    fr = [0.4, 0.4, 0.02, 0.01, 0.01]
    models = [env.sys.tree_replace({"body_mass": {"base": m0.arrays["body_mass"][1] + 3.0}}).model,
              env.sys.tree_replace({"pair_friction": {f: fr for f in FEET}}).model,
              env.sys.tree_replace({"dof_damping": m0.arrays["dof_damping"] * 2}).model]
    B, N, Hs, Hn = 3, 4, 6, 3
    nu = env.action_size
    rng = np.random.default_rng(3)
    s = o.reset()
    qpos = np.repeat(s.qpos[None] if s.qpos.ndim == 1 else s.qpos, B, 0)
    qpos[:, 2] += rng.uniform(-0.02, 0.02, B)
    qpos[:, 7:7 + nu] += rng.normal(size=(B, nu)) * 0.05
    qvel = rng.normal(size=(B, m0.nv)) * 0.2
    warm = rng.normal(size=(B, m0.nv)) * 0.1
    Y = np.clip(rng.normal(size=(B, Hn + 1, nu)) * 0.4, -1, 1)
    keys = np.array([[0, 7], [11, 3], [123, 456]], np.uint32)
    noise = 0.9 ** np.arange(Hn + 1)[::-1]
    kw = dict(Nsample=N, Hsample=Hs, Hnode=Hn, temp_sample=0.05,
              M_n2u=interp_matrix(np.linspace(0, 1, Hn + 1), np.linspace(0, 1, Hs + 1)))
    desc, single = env.plan_desc(n_inst=B, **kw), env.plan_desc(**kw)
    # the counters straddle the first stage boundary (the env step from step 49 enters stage 1)
    counters = np.array([[45, 0], [49, 0], [50, 1]], np.int32)
    rows = N + 1
    plain = rollout_models(m0, None, desc, 4, qpos, qvel, warm, counters, rng=keys, Ybar=Y, noise=noise, H=Hs + 1)
    # 3 warps per CTA: two CTAs per instance, the second repeats the instance's last row; 5: one each
    for wpc in (3, 5):
        bat = rollout_models(m0, models, desc, wpc, qpos, qvel, warm, counters, rng=keys, Ybar=Y, noise=noise,
                             H=Hs + 1)
        for b in range(B):
            one = rollout_models(models[b], None, single, 1, qpos[b:b + 1], qvel[b:b + 1], warm[b:b + 1],
                                 counters[b:b + 1], rng=keys[b:b + 1], Ybar=Y[b:b + 1], noise=noise, H=Hs + 1,
                                 single=True)
            sl = slice(b * rows, (b + 1) * rows)
            for k in ("rewss", "rews", "q", "qd", "xpos"):
                assert np.array_equal(bat[k][sl], one[k]), (wpc, b, k)
        # the models were read: every instance's rewards differ from the plan's model
        for b in range(B):
            assert not np.array_equal(bat["rewss"][b * rows:(b + 1) * rows], plain["rewss"][b * rows:(b + 1) * rows]), b
    # env step (mode 0): one row per instance, action Y[b][0], one CTA of one warp per instance
    us_row = (Hn + 1) * nu
    bat0 = rollout_models(m0, models, desc, 1, qpos, qvel, warm, counters, us=Y, mode=0, H=1, us_row=us_row)
    for b in range(B):
        one = rollout_models(models[b], None, single, 1, qpos[b:b + 1], qvel[b:b + 1], warm[b:b + 1],
                             counters[b:b + 1], us=Y[b:b + 1, :1], mode=0, H=1, single=True)
        for k in ("qpos_out", "qvel_out", "warm_out", "ctrl_out", "counters"):
            assert np.array_equal(bat0[k][b], one[k][0]), (b, k)
        assert np.array_equal(bat0["rewss"][b], one["rewss"][0]), b
    assert bat0["counters"][1, 1] == 1 and bat0["counters"][0, 1] == 0
