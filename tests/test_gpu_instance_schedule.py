"""Per-instance sampling schedules (dial_plan_set_instance_schedule / _iterations, DeviceLoop(...,
schedule=...)): instance b of a batched loop computes bitwise what a single-instance loop on an MBDPI with
b's updated DialConfig computes, at every step (the initial step, then env_step 1, 0 and 2: eager, captured
and replayed), also with per-instance tasks and models and with an ensemble; specs equal to the plan's
config reproduce the loop without schedules; set_schedule between replays needs no new capture; an
instance with no iterations is only shifted; the error paths and the CLI sweep."""
import os

import numpy as np
import pytest
import torch
import yaml

from tests.conftest import make_pair
from tests.test_gpu_batch import KEYS, _config, _instances, _trace
from tests.test_gpu_ensemble import _equal_traces, _load, _snapshot
from tests.test_gpu_instance_models import FEET, LOW_FRICTION, _with_sys
from tests.test_gpu_tasks import _cli_runs, _go2_sweep, _run, _same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (initial, env_step) per control step: the initial step, then every env_step shape eager, captured, replayed
STEPS = [(True, 1), (False, 1), (False, 1), (False, 1), (False, 0), (False, 0), (False, 0), (False, 2), (False, 2),
         (False, 2)]
# distinct temperatures, factors and iteration counts; None keeps the plan's (Ndiffuse 2, Ndiffuse_init 3)
SPECS = [None,
         {"temp_sample": 0.1, "traj_diffuse_factor": 0.3, "Ndiffuse": 3, "Ndiffuse_init": 1},
         {"temp_sample": 0.04, "horizon_diffuse_factor": 1.0, "sigma_scale": 0.8, "Ndiffuse": 1, "Ndiffuse_init": 4}]


def _steps(loop, cfg=None):
    """The STEPS of a batched loop (cfg None: each instance's own counts) or of a single loop on cfg."""
    out = []
    for initial, es in STEPS:
        if cfg is None:
            loop.step(env_step=es, initial=initial)
        else:
            loop.step(cfg.Ndiffuse_init if initial else cfg.Ndiffuse, env_step=es)
        torch.cuda.synchronize()
        out.append({k: loop.buf[k].clone() for k in KEYS})
    return out


def _compare(batched, b, ref, what):
    for t, (got, want) in enumerate(zip(batched, ref)):
        for k in KEYS:
            g = got[k][b:b + 1] if k == "reward" else got[k][b]
            assert torch.equal(g, want[k]), (what, b, t, STEPS[t], k)


def _check(name, N, Hs, Hn, B, envs=None, ensemble=None, risk=None):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI, schedule_setting
    env, _ = make_pair(name)
    args = _config(name, N, Hs, Hn)
    specs = [SPECS[b % len(SPECS)] for b in range(B)]
    states, rngs, Y0 = _instances(envs[0] if envs else env, B, Hn)
    K = len(ensemble) if ensemble else 0
    loop = DeviceLoop(MBDPI(args, env, n_instances=B, n_ensemble=K), states, rngs, Y0, envs=envs, ensemble=ensemble,
                      risk=risk, schedule=specs)
    batched = _steps(loop)
    for b in range(B):
        cfg = schedule_setting(specs[b] or {}, args)
        env_b = envs[b] if envs else env
        ref = DeviceLoop(MBDPI(cfg, env_b, n_ensemble=K), states[b], rngs[b], Y0[b], ensemble=ensemble, risk=risk)
        _compare(batched, b, _steps(ref, cfg), name)
    assert not torch.equal(batched[-1]["Y"][0], batched[-1]["Y"][1])
    return loop


@pytest.mark.parametrize("name, N, Hs, Hn, B", [
    ("unitree_go2_walk", 64, 12, 4, 3),
    ("allegro_reorient", 16, 4, 2, 3),            # dense solver path, lock-step level 3
    ("unitree_go2_walk", 100, 8, 4, 24),           # the plain layout straddles CTAs
])
def test_batched_schedules_equal_single_loops(built, name, N, Hs, Hn, B):
    _check(name, N, Hs, Hn, B)


def test_batched_schedules_generic_tree(built, monkeypatch):
    monkeypatch.setenv("DIAL_FORCE_GENERIC_TREE", "1")
    _check("unitree_go2_walk", 64, 10, 4, 3)


def test_schedules_with_tasks_and_models(built):
    envs = _go2_sweep()
    envs[1] = _with_sys(envs[1], {"pair_friction": {f: LOW_FRICTION for f in FEET}})
    envs[2] = _with_sys(envs[2], {"body_mass": {"base": envs[2].sys.model.arrays["body_mass"][1] + 3.0}})
    _check("unitree_go2_walk", 64, 12, 4, 3, envs=envs)


def test_schedules_with_a_worst_case_ensemble(built):
    env, _ = make_pair("unitree_go2_walk")
    members = [env, _with_sys(env, {"dof_damping": env.sys.model.arrays["dof_damping"] * 2})]
    _check("unitree_go2_walk", 64, 12, 4, 3, ensemble=members, risk={"aggregate": "worst"})


def test_specs_of_the_plan_config_equal_no_schedule(built):
    from dial_mpc_b200.core.dial_core import SCHEDULE_FIELDS, DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 2, 4)
    plain = _trace(DeviceLoop(MBDPI(args, env, n_instances=2), states, rngs, Y0))
    own = {k: getattr(args, k) for k in SCHEDULE_FIELDS}
    _equal_traces(_trace(DeviceLoop(MBDPI(args, env, n_instances=2), states, rngs, Y0, schedule=own)), plain)


def test_set_schedule_between_replays(built):
    """Instance 1's schedule changes after the graph of (2, env_step 1) has been captured and replayed: from
    the next step on it plans with the new one, instance 0 is unchanged, and a step launches what it did."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 2, 4)
    old, new = {"Ndiffuse": 1, "temp_sample": 0.08}, {"Ndiffuse": 2, "temp_sample": 0.1, "traj_diffuse_factor": 0.3}
    loop = DeviceLoop(MBDPI(args, env, n_instances=2), states, rngs, Y0, schedule=[None, old])
    refs = [DeviceLoop(MBDPI(args, env), states[0], rngs[0], Y0[0]),
            DeviceLoop(MBDPI(args, env), states[1], rngs[1], Y0[1], schedule=old)]
    per_step = []
    for t in range(8):
        if t == 5:
            loop.set_schedule(1, new)
            refs[1].set_schedule(0, new)
        l0 = loop.plan.launches
        loop.step()
        per_step.append(loop.plan.launches - l0)
        for r in refs:
            r.step()
        torch.cuda.synchronize()
        for b, r in enumerate(refs):
            for k in KEYS:
                g = loop.buf[k][b:b + 1] if k == "reward" else loop.buf[k][b]
                assert torch.equal(g, r.buf[k]), (t, b, k)
    assert len(set(per_step)) == 1, per_step


def test_an_instance_without_iterations_is_only_shifted(built):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 2, 4)
    loop = DeviceLoop(MBDPI(args, env, n_instances=2), states, rngs, Y0)
    ref = DeviceLoop(MBDPI(args, env, n_instances=2), states, rngs, Y0)
    shifter = DeviceLoop(MBDPI(args, env, n_instances=2), states, rngs, Y0)
    for _ in range(2):
        loop.step()
        ref.step()
    loop.plan.set_instance_iterations([2, 0])
    for t in range(3):   # eager, captured, replayed
        torch.cuda.synchronize()
        pre = _snapshot(loop)
        bars = {k: loop.buf[k][1].clone() for k in ("rews", "qbar", "qdbar", "xbar")}
        loop.plan.mpc_step(2, 1)
        ref.step(2)
        _load(shifter, pre)
        shifter.step(0, env_step=1)
        torch.cuda.synchronize()
        for k in KEYS:
            g = loop.buf[k][0:1] if k == "reward" else loop.buf[k][0]
            assert torch.equal(g, ref.buf[k][0:1] if k == "reward" else ref.buf[k][0]), (t, k)
        assert torch.equal(loop.buf["Y"][1], shifter.buf["Y"][1]), t
        for k in ("qpos", "qvel", "qacc_warmstart", "ctrl", "counters"):
            assert torch.equal(loop.buf[k][1], shifter.buf[k][1]), (t, k)
        assert torch.equal(loop.buf["rng"][1], pre["rng"][1]), t
        for k, v in bars.items():
            assert torch.equal(loop.buf[k][1], v), (t, k)


def test_schedule_error_paths(built, monkeypatch):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 2, 4)
    loop = DeviceLoop(MBDPI(args, env, n_instances=2), states, rngs, Y0,
                      schedule=[{"Ndiffuse_init": 5}, {"Ndiffuse": 3}])
    pl = loop.plan
    table = np.full((3, 5), 0.5, np.float32)
    with pytest.raises(RuntimeError, match=r"instance 2 out of range"):
        pl.set_instance_schedule(2, 0.1, table)
    with pytest.raises(IndexError, match=r"instance -1 out of range"):
        loop.set_schedule(-1, {})
    for temp in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(RuntimeError, match=r"temp must be finite and > 0"):
            pl.set_instance_schedule(0, temp, table)
    with pytest.raises(RuntimeError, match=r"n_rows 65 out of range \(1\.\.64\)"):
        pl.set_instance_schedule(0, 0.1, np.full((65, 5), 0.5, np.float32))
    bad = table.copy()
    bad[1, 2] = np.nan
    with pytest.raises(RuntimeError, match=r"noise\[1\]\[2\] is not finite"):
        pl.set_instance_schedule(0, 0.1, bad)
    with pytest.raises(RuntimeError, match=r"n_iter\[1\] = 65 out of range \(0\.\.64\)"):
        pl.set_instance_iterations([1, 65])
    with pytest.raises(RuntimeError, match=r"n_iter\[0\] = -1 out of range"):
        pl.set_instance_iterations([-1, 1])
    with pytest.raises(ValueError, match=r"Ndiffuse must be an int in 1\.\.64"):
        loop.set_schedule(0, {"Ndiffuse": 0})
    # instance 0's table has 5 rows, instance 1's max(3, 3) = 3: an explicit count of 4 is refused, naming 1
    with pytest.raises(RuntimeError, match=r"instance 1 runs 4 diffusion iterations, its schedule has 3 rows"):
        loop.step(4)
    loop.step(3)
    monkeypatch.setenv("DIAL_NO_FUSED_UPDATE", "1")
    one = DeviceLoop(MBDPI(args, env), states[0], rngs[0], Y0[0], schedule={"temp_sample": 0.1})
    with pytest.raises(RuntimeError, match=r"need the fused update"):
        one.step()


def test_cli_schedule_sweep(built, tmp_path):
    """The README sweep: instance 0 is the plain run, instance 2 the plain run of a config with its fields."""
    base = yaml.safe_load(open(os.path.join(ROOT, "dial_mpc_b200", "examples", "unitree_go2_trot.yaml")))
    ov = [{}, {"temp_sample": 0.1}, {"Ndiffuse": 4, "traj_diffuse_factor": 0.3}]
    f = tmp_path / "sweep.yaml"
    f.write_text(yaml.safe_dump(ov))
    out = _cli_runs(tmp_path, {"batched": (base, ["--instances", "3", "--instance-overrides", str(f)]),
                               "plain0": (base, []),
                               "plain2": (dict(base, seed=base["seed"] + 2, **ov[2]), [])})
    s, p = out["batched"]
    assert len(s) == 3 and len(p) == 3
    for b in (0, 2):
        assert _same(s[b], out[f"plain{b}"][0][0]) and _same(p[b], out[f"plain{b}"][1][0]), b
    (tmp_path / "cfg.yaml").write_text(yaml.safe_dump(base))
    f.write_text(yaml.safe_dump([{}, {"Hnode": 3}, {}]))
    r = _run(["--config", "cfg.yaml", "--instances", "3", "--instance-overrides", str(f)], tmp_path)
    assert r.returncode == 2 and "--instance-overrides entry 1: Hnode is shared by every instance" in r.stderr
