"""Per-instance physical models of a batched plan (dial_plan_set_instance_model, DeviceLoop(..., envs=...)
with envs whose ``sys`` differs, DeviceLoop.set_model): instance b must compute bitwise what a
single-instance DeviceLoop on instance b's env (a plan created from its model) computes, at every step
(eager first uses and graph replays, env_step 1, 0 and 2)."""
import os
from dataclasses import replace

import pytest
import torch
import yaml

from tests.conftest import make_pair
from tests.test_gpu_batch import KEYS, SCHEDULE, _config, _instances, _trace
from tests.test_gpu_tasks import _cli_runs, _compare, _run, _same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FEET = ("FR", "FL", "RR", "RL")
LOW_FRICTION = [0.4, 0.4, 0.02, 0.01, 0.01]


def _with_sys(env, params):
    """A fresh env of ``env``'s class and configuration whose model is ``env.sys.tree_replace(params)``."""
    e = type(env)(env._config)
    e.sys = e.sys.tree_replace(params)
    return e


def _go2_models(env):
    m = env.sys.model
    return [env,
            _with_sys(env, {"body_mass": {"base": m.arrays["body_mass"][1] + 3.0}}),
            _with_sys(env, {"pair_friction": {f: LOW_FRICTION for f in FEET}}),
            _with_sys(env, {"dof_damping": m.arrays["dof_damping"] * 2, "actuator_gear": m.arrays["actuator_gear"] * 0.8,
                            "opt.gravity": [0.3, 0.0, -9.6]})]


def _check_models(name, envs, N, Hs, Hn, start_step=None, base=None):
    """A batched loop on base's plan with envs[b]'s model (and task) per instance == single loops on envs[b]."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    B = len(envs)
    base = base or envs[0]
    args = _config(name, N, Hs, Hn)
    states, rngs, Y0 = _instances(base, B, Hn, start_step)
    lead = (states, rngs, Y0) if B > 1 else (states[0], rngs[0], Y0[0])   # a B = 1 loop takes one state
    batched = _trace(DeviceLoop(MBDPI(args, base, n_instances=B), *lead, envs=envs))
    if B == 1:
        batched = [{k: (v[None] if k != "reward" else v) for k, v in st.items()} for st in batched]
    refs = [_trace(DeviceLoop(MBDPI(args, envs[b]), states[b], rngs[b], Y0[b])) for b in range(B)]
    _compare(batched, refs)
    return batched, refs, (args, states, rngs, Y0)


@pytest.mark.parametrize("generic", [False, True])
def test_go2_trot_configs0_size(built, monkeypatch, generic):
    from baseline_configs import BASELINE
    if generic:
        monkeypatch.setenv("DIAL_FORCE_GENERIC_SHAPE", "1")
    env, _ = make_pair("unitree_go2_walk")
    b = BASELINE[0]
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    batched, refs, (args, states, rngs, Y0) = _check_models("unitree_go2_walk", _go2_models(env), b["N"], b["Hs"], b["Hn"])
    # the models were read: every instance on the plan's own model plans something else
    for i in range(1, 4):
        plain = _trace(DeviceLoop(MBDPI(args, env), states[i], rngs[i], Y0[i]))
        assert not torch.equal(plain[0]["rews"], refs[i][0]["rews"]), i


def test_go2_kernel_name(built):
    from dial_mpc_b200.core.dial_core import MBDPI
    env, _ = make_pair("unitree_go2_walk")
    mb = MBDPI(_config("unitree_go2_walk", 16, 6, 2), env, n_instances=2)
    assert mb.plan.lib.dial_plan_rollout_kernel(mb.plan.handle) == b"go2"


def test_h1_walk_models(built):      # star <5,7>
    env, _ = make_pair("unitree_h1_walk")
    m = env.sys.model
    envs = [_with_sys(env, {"body_mass": {"pelvis": m.arrays["body_mass"][1] + 5.0}}),
            env,
            _with_sys(env, {"dof_damping": m.arrays["dof_damping"] * 2, "actuator_gear": m.arrays["actuator_gear"] * 0.9})]
    _check_models("unitree_h1_walk", envs, 64, 10, 4, base=env)


def test_allegro_models(built):      # dense solver path
    env, _ = make_pair("allegro_reorient")
    m = env.sys.model
    envs = [_with_sys(env, {"body_mass": {"object": m.arrays["body_mass"][1] * 2}}),
            _with_sys(env, {"pair_friction": m.arrays["pair_friction"] * 0.5}),
            env]
    _check_models("allegro_reorient", envs, 16, 4, 2, base=env)


def test_many_instances_n100(built):
    env, _ = make_pair("unitree_go2_walk")
    m = env.sys.model
    envs = [_with_sys(env, {"body_mass": {"base": m.arrays["body_mass"][1] + 0.25 * b},
                            "pair_friction": m.arrays["pair_friction"] * (1.0 - 0.02 * b)}) for b in range(24)]
    _check_models("unitree_go2_walk", envs, 100, 8, 4, base=env)


def test_one_sample(built):
    env, _ = make_pair("unitree_go2_walk")
    _check_models("unitree_go2_walk", _go2_models(env)[1:], 1, 8, 4, base=env)


def test_single_instance_plan(built):
    env, _ = make_pair("unitree_go2_seq_jump")
    heavy = _go2_models(env)[1]
    _check_models("unitree_go2_seq_jump", [heavy], 64, 12, 4, start_step=48, base=env)


def test_tasks_and_models_together(built):
    import dial_mpc_b200.envs as E
    env, _ = make_pair("unitree_go2_walk")
    envs = []
    for b, e in enumerate(_go2_models(env)):
        t = E.get_environment("unitree_go2_walk", config=replace(env._config, default_vx=0.3 * b, gait="walk" if b % 2 else "trot"))
        t.sys = e.sys
        envs.append(t)
    _check_models("unitree_go2_walk", envs, 64, 12, 4, base=env)


def test_set_model_mid_run(built):
    """set_model on instance 1 of a batched loop == a B = 1 loop that switches its model at the same
    step; instance 0 is untouched."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    heavy, slippery = _go2_models(env)[1:3]
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 2, 4)

    def run(loop, inst):
        out = []
        for t, (nd, es) in enumerate(SCHEDULE):
            if t == 5:
                loop.set_model(inst, slippery)
            loop.step(nd, env_step=es)
            torch.cuda.synchronize()
            out.append({k: loop.buf[k].clone() for k in KEYS})
        return out
    batched = run(DeviceLoop(MBDPI(args, env, n_instances=2), states, rngs, Y0, envs=[env, heavy]), 1)
    ref0 = _trace(DeviceLoop(MBDPI(args, env), states[0], rngs[0], Y0[0]))
    ref1 = run(DeviceLoop(MBDPI(args, env), states[1], rngs[1], Y0[1], envs=[heavy]), 0)
    _compare(batched, [ref0, ref1])
    # the B = 1 reference switches models: a loop that keeps the heavy model diverges after step 5
    keep = _trace(DeviceLoop(MBDPI(args, heavy), states[1], rngs[1], Y0[1]))
    assert torch.equal(keep[4]["Y"], ref1[4]["Y"]) and not torch.equal(keep[-1]["Y"], ref1[-1]["Y"])


def test_model_error_paths(built):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    args = _config("unitree_go2_walk", 16, 6, 2)
    mb = MBDPI(args, env, n_instances=2)
    states, rngs, Y0 = _instances(env, 2, 2)
    loop = DeviceLoop(mb, states, rngs, Y0)
    with pytest.raises(RuntimeError, match="'timestep'"):
        loop.set_model(1, env.sys.tree_replace({"opt.timestep": 0.01}))
    m = env.sys.model
    jr = env.sys.model.replace({})
    jr.arrays["jnt_range"] = m.arrays["jnt_range"] * 0.5
    with pytest.raises(RuntimeError, match="'jnt_range'"):
        loop.set_model(0, jr)
    with pytest.raises(IndexError):
        loop.set_model(2, env)
    with pytest.raises(RuntimeError, match="out of range"):
        mb.plan.set_instance_model(5, env.sys)


def test_cli_sys_overrides(built, tmp_path):
    base = yaml.safe_load(open(os.path.join(ROOT, "dial_mpc_b200", "examples", "unitree_go2_trot.yaml")))
    ov = [{}, {"sys": {"body_mass": {"base": 10.92}}},
          {"sys": {"pair_friction": {f: LOW_FRICTION for f in FEET}}}]
    f = tmp_path / "ov.yaml"
    f.write_text(yaml.safe_dump(ov))
    out = _cli_runs(tmp_path, {"batched": (base, ["--instances", "3", "--instance-overrides", str(f)]),
                               "plain0": (dict(base), [])})
    s, p = out["batched"]
    assert len(s) == 3
    assert _same(s[0], out["plain0"][0][0]) and _same(p[0], out["plain0"][1][0])
    assert not _same(s[1], s[0]) and not _same(s[2], s[0])
    # a structural field is rejected
    (tmp_path / "cfg.yaml").write_text(yaml.safe_dump(base))
    f.write_text(yaml.safe_dump([{}, {"sys": {"pair_kind": [0, 0, 0, 0]}}]))
    r = _run(["--config", "cfg.yaml", "--instances", "2", "--instance-overrides", str(f)], tmp_path)
    assert r.returncode != 0 and "pair_kind" in r.stderr
