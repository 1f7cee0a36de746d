"""CPU tests of ensemble planning (dial_plan_desc.n_ens): the descriptor and plan-creation checks, the
``--ensemble`` file, and, through the warp emulator, ensemble rollout launches whose member rows are bitwise
single-instance launches on each member's model."""
import ctypes as C
import sys

import numpy as np
import pytest
import yaml

from dial_mpc_b200 import _capi
from dial_mpc_b200 import random as drandom
from dial_mpc_b200.utils.spline import interp_matrix
from tests.conftest import make_pair
from tests.emul import emul

FEET = ("FR", "FL", "RR", "RL")


def _go2():
    import dial_mpc_b200.envs as E
    return E.get_environment("unitree_go2_walk", config=E.get_config("unitree_go2_walk")())


# ---- descriptor and plan creation ----------------------------------------------------------------------
def test_descriptor_field_follows_n_inst_and_matches_the_library():
    names = [n for n, _ in _capi.dial_plan_desc._fields_]
    assert names[-2:] == ["n_inst", "n_ens"]
    assert _capi.DEFINES["DIAL_MAXENS"] == 16
    lib = _capi.lib()
    assert lib.dial_sizeof(1) == C.sizeof(_capi.dial_plan_desc)
    assert lib.dial_abi_version() == _capi.DEFINES["DIAL_ABI_VERSION"] == 14
    env = _go2()
    assert env.plan_desc().n_ens == 0 and env.plan_desc(n_ens=3).n_ens == 3


@pytest.mark.parametrize("n_ens, Ntotal, match", [(-1, None, "n_ens out of range"), (17, None, "n_ens out of range"),
                                                  (1, 16, "ensemble plan .* cannot be sharded")])
def test_plan_create_rejects_bad_n_ens(n_ens, Ntotal, match):
    # the descriptor is checked before any device allocation, so this runs without a GPU
    env = _go2()
    lib = _capi.lib()
    md = _capi.fill_model_desc(env.sys.model)
    desc = env.plan_desc(Nsample=8, Ntotal=Ntotal, Hsample=4, Hnode=2, n_ens=n_ens)
    assert not lib.dial_plan_create(C.byref(md), C.byref(desc))
    import re
    assert re.search(match, lib.dial_last_error().decode())


# ---- the --ensemble file -------------------------------------------------------------------------------
def test_load_ensemble_builds_members_and_checks_the_plant():
    from dial_mpc_b200.core.dial_core import load_ensemble
    env = _go2()
    m0 = env.sys.model
    members, plant = load_ensemble(yaml.safe_load("""
members:
  - {}
  - {body_mass: {base: 9.0}}
  - {pair_friction: {FR: [0.4, 0.4, 0.02, 0.01, 0.01]}}
plant: {dof_damping: {FL_calf_joint: 1.3}}
"""), env)
    assert len(members) == 3 and plant == {"dof_damping": {"FL_calf_joint": 1.3}}
    assert bytes(_capi.fill_model_desc(members[0].model)) == bytes(_capi.fill_model_desc(m0))
    assert members[1].model.arrays["body_mass"][m0.body_id("base")] == 9.0
    members, plant = load_ensemble({"members": [None]}, env)
    assert len(members) == 1 and plant is None


@pytest.mark.parametrize("spec, match", [
    ([{}], "must map 'members'"),
    ({"plant": {}}, "must map 'members'"),
    ({"members": [{}], "other": 1}, r"must map 'members'.*other"),
    ({"members": {}}, "members must be a list of 1..16"),
    ({"members": []}, "members must be a list of 1..16"),
    ({"members": [{}] * 17}, "members must be a list of 1..16"),
    ({"members": [{}, 3]}, r"members\[1\] must map model fields"),
    ({"members": [{"body_parentid": 1}]}, r"members\[0\]: .*not a replaceable"),
    ({"members": [{"body_mass": {"torso": 1.0}}]}, r"members\[0\]: .*body 'torso'"),
    ({"members": [{}], "plant": [1]}, "plant must map model fields"),
    ({"members": [{}], "plant": {"nq": 3}}, "plant: .*not a replaceable"),
])
def test_load_ensemble_names_the_bad_entry(spec, match):
    from dial_mpc_b200.core.dial_core import load_ensemble
    with pytest.raises(ValueError, match=match):
        load_ensemble(spec, _go2())


@pytest.mark.parametrize("text, extra, match", [
    ("members: [{}, {nq: 1}]\n", [], r"--ensemble .*members\[1\]"),
    ("members: [{}\n", [], "--ensemble"),
    ("members: [{}]\n", ["--eager"], "excludes --eager"),
])
def test_cli_reports_ensemble_errors(tmp_path, monkeypatch, capsys, text, extra, match):
    from dial_mpc_b200.core import dial_core
    f = tmp_path / "ens.yaml"
    f.write_text(text)
    monkeypatch.setattr(sys, "argv", ["dial_core", "--example", "unitree_go2_trot", "--ensemble", str(f)] + extra)
    with pytest.raises(SystemExit) as e:
        dial_core.main()
    assert e.value.code == 2
    import re
    assert re.search(match, capsys.readouterr().err)


# ---- emulator: ensemble launches -----------------------------------------------------------------------
def _desc_with_task(desc, t):
    d = _capi.dial_plan_desc.from_buffer_copy(desc)
    for name in _capi.TASK_FIELDS:
        v = getattr(t, name)
        if isinstance(v, C.Array):
            C.memmove(C.addressof(getattr(d, name)), C.addressof(v), C.sizeof(v))
        else:
            setattr(d, name, v)
    return d


def rollout(base_model, models, desc, wpc, nrows, rows_per_inst, rows_per_model, tasks, task_rows, qpos, qvel, warm,
            counters, rng, Ybar, noise, H):
    md = _capi.fill_model_desc(base_model)
    nq, nv, nb = md.nq, md.nv, md.nbody
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    out = dict(rewss=np.zeros((nrows, H), np.float32), rews=np.zeros(nrows, np.float32),
               q=np.zeros((nrows, H, nq), np.float32), qd=np.zeros((nrows, H, nv), np.float32),
               xpos=np.zeros((nrows, H, nb - 1, 3), np.float32))
    emul.launch(md, desc, wpc=wpc, models=models, mode=1, nrows=nrows, H=H, rows_per_inst=rows_per_inst,
                rows_per_model=rows_per_model, tasks=None if tasks is None else (_capi.dial_task * len(tasks))(*tasks),
                task_rows=task_rows, qpos0=f32(qpos), qvel0=f32(qvel), warm0=f32(warm),
                counters_in=np.ascontiguousarray(counters, dtype=np.int32),
                rng_dev=np.ascontiguousarray(rng, dtype=np.uint32), Ybar=f32(Ybar), noise=f32(noise), **out)
    return out


def member_mean(r):
    """The reduction of ensemble_mean_kernel restated: r [B,K,n1] -> fp32 sum in member order, then / K."""
    r = np.asarray(r, np.float32)
    s = r[:, 0].copy()
    for k in range(1, r.shape[1]):
        s = (s + r[:, k]).astype(np.float32)
    return (s / np.float32(r.shape[1])).astype(np.float32)


def test_seq_jump_ensemble_rows_equal_single_instance_launches():
    env, o = make_pair("unitree_go2_seq_jump")
    m0 = env.sys.model
    fr = [0.4, 0.4, 0.02, 0.01, 0.01]
    members = [env.sys.tree_replace({"body_mass": {"base": m0.arrays["body_mass"][1] + 3.0}}).model,
               env.sys.tree_replace({"pair_friction": {f: fr for f in FEET}}).model,
               env.sys.tree_replace({"dof_damping": m0.arrays["dof_damping"] * 2}).model]
    B, K, N, Hs, Hn = 2, 3, 4, 6, 3
    nu, n1, H = env.action_size, N + 1, Hs + 1
    rng = np.random.default_rng(11)
    s = o.reset()
    qpos = np.repeat(s.qpos[None] if s.qpos.ndim == 1 else s.qpos, B, 0)
    qpos[:, 2] += rng.uniform(-0.02, 0.02, B)
    qpos[:, 7:7 + nu] += rng.normal(size=(B, nu)) * 0.05
    qvel = rng.normal(size=(B, m0.nv)) * 0.2
    warm = rng.normal(size=(B, m0.nv)) * 0.1
    Y = np.clip(rng.normal(size=(B, Hn + 1, nu)) * 0.4, -1, 1)
    keys = np.array([[0, 7], [11, 3]], np.uint32)
    noise = 0.9 ** np.arange(Hn + 1)[::-1]
    tasks = []
    for seed in (3, 4):      # per-instance tasks: each instance its own random jump sequence
        tgt, rad, pose, yaw = env.sample_command(drandom.PRNGKey(seed))
        tasks.append(_capi.task_set_stages(env.task(), (pose, yaw, tgt, rad)))
    kw = dict(Nsample=N, Hsample=Hs, Hnode=Hn, temp_sample=0.05,
              M_n2u=interp_matrix(np.linspace(0, 1, Hn + 1), np.linspace(0, 1, Hs + 1)))
    desc, single = env.plan_desc(n_inst=B, n_ens=K, **kw), env.plan_desc(**kw)
    # the counters straddle the first stage boundary (the horizon from step 45 enters stage 1 at step 50)
    counters = np.array([[45, 0], [49, 0]], np.int32)
    slots = [members[k] for b in range(B) for k in range(K)]          # member (b, k) at slot b K + k
    # mpc_enqueue's launch: rows ((b K) + k)(N+1) + i, tasks per instance
    outs = {wpc: rollout(m0, slots, desc, wpc, B * K * n1, K * n1, n1, tasks, K * n1, qpos, qvel, warm, counters,
                         keys, Y, noise, H) for wpc in (2, 5)}   # 2 warps: three CTAs per member, the last repeats a row
    for wpc, ens in outs.items():
        for b in range(B):
            for k in range(K):
                one = rollout(members[k], None, _desc_with_task(single, tasks[b]), 1, n1, 0, 0, None, 0,
                              qpos[b:b + 1], qvel[b:b + 1], warm[b:b + 1], counters[b:b + 1], keys[b:b + 1],
                              Y[b:b + 1], noise, H)
                sl = slice((b * K + k) * n1, (b * K + k + 1) * n1)
                for f in ("rewss", "rews", "q", "qd", "xpos"):
                    assert np.array_equal(ens[f][sl], one[f]), (wpc, b, k, f)
        # the members were read: their rewards differ from one another
        r = ens["rews"].reshape(B, K, n1)
        for b in range(B):
            assert not np.array_equal(r[b, 0], r[b, 1]) and not np.array_equal(r[b, 0], r[b, 2]), b
    # the stage boundary was crossed: the rewards of one row differ between the two tasks
    assert not np.array_equal(outs[2]["rewss"][:n1], outs[2]["rewss"][K * n1:(K + 1) * n1])
    # the reduction restated: sum in member order, then / K
    r = outs[2]["rews"].reshape(B, K, n1).astype(np.float32)
    rbar = member_mean(r)
    assert rbar.dtype == np.float32 and rbar.shape == (B, n1)
    assert np.array_equal(rbar, ((r[:, 0] + r[:, 1]) + r[:, 2]) / np.float32(3))
    np.testing.assert_allclose(rbar, r.astype(np.float64).mean(1), rtol=1e-6)


def test_one_member_with_the_plan_model_equals_no_ensemble():
    env, o = make_pair("unitree_go2_walk")
    m0 = env.sys.model
    B, N, Hs, Hn = 2, 4, 6, 3
    nu, n1, H = env.action_size, N + 1, Hs + 1
    rng = np.random.default_rng(2)
    s = o.reset()
    qpos = np.repeat(s.qpos[None] if s.qpos.ndim == 1 else s.qpos, B, 0)
    qpos[:, 7:7 + nu] += rng.normal(size=(B, nu)) * 0.05
    qvel = rng.normal(size=(B, m0.nv)) * 0.2
    warm = rng.normal(size=(B, m0.nv)) * 0.1
    Y = np.clip(rng.normal(size=(B, Hn + 1, nu)) * 0.4, -1, 1)
    keys = np.array([[5, 6], [7, 8]], np.uint32)
    noise = 0.9 ** np.arange(Hn + 1)[::-1]
    kw = dict(Nsample=N, Hsample=Hs, Hnode=Hn, temp_sample=0.05,
              M_n2u=interp_matrix(np.linspace(0, 1, Hn + 1), np.linspace(0, 1, Hs + 1)))
    counters = np.array([[0, 0], [17, 0]], np.int32)
    plain = rollout(m0, None, env.plan_desc(n_inst=B, **kw), 4, B * n1, n1, 0, None, 0, qpos, qvel, warm, counters,
                    keys, Y, noise, H)
    desc = env.plan_desc(n_inst=B, n_ens=1, **kw)
    for models in (None, [m0] * B):    # no member set, and every member set to the plan's model
        one = rollout(m0, models, desc, 4, B * n1, n1, n1, None, 0, qpos, qvel, warm, counters, keys, Y, noise, H)
        for f in plain:
            assert np.array_equal(one[f], plain[f]), f
