"""Per-instance tasks of a batched plan (dial_mpc_buffers.tasks, DeviceLoop(..., envs=...), batched
randomize_tasks): instance b must compute bitwise what a single-instance DeviceLoop on instance b's env
(its own commands, gait, jump sequence or user constants) computes, at every step (eager first uses and
graph replays, env_step 1, 0 and 2)."""
import glob
import importlib
import os
import subprocess
import sys
from dataclasses import replace

import numpy as np
import pytest
import torch
import yaml

from tests.conftest import make_pair
from tests.test_gpu_batch import KEYS, SCHEDULE, _config, _instances, _trace

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EX = os.path.join(ROOT, "dial_mpc_b200", "examples", "custom_env")


def _env(name, **kw):
    import dial_mpc_b200.envs as E
    env, _ = make_pair(name)
    return E.get_environment(name, config=replace(env._config, **kw))


def _compare(batched, refs):
    for b, ref in enumerate(refs):
        for t, (got, want) in enumerate(zip(batched, ref)):
            for k in KEYS:
                g = got[k][b:b + 1] if k == "reward" else got[k][b]
                assert torch.equal(g, want[k]), (b, t, SCHEDULE[t], k)


def _check_tasks(name, envs, N, Hs, Hn, start_step=None):
    """A batched loop with envs[b]'s task per instance == single loops on envs[b]."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    B = len(envs)
    args = _config(name, N, Hs, Hn)
    states, rngs, Y0 = _instances(envs[0], B, Hn, start_step)
    batched = _trace(DeviceLoop(MBDPI(args, envs[0], n_instances=B), states, rngs, Y0, envs=envs))
    refs = [_trace(DeviceLoop(MBDPI(args, envs[b]), states[b], rngs[b], Y0[b])) for b in range(B)]
    _compare(batched, refs)
    return batched


def _go2_sweep():
    return [_env("unitree_go2_walk", default_vx=0.2), _env("unitree_go2_walk", default_vx=0.6, default_vyaw=0.4),
            _env("unitree_go2_walk", default_vx=1.0, gait="walk")]


def test_go2_walk_vx_sweep_and_gaits(built):
    tr = _check_tasks("unitree_go2_walk", _go2_sweep(), 64, 12, 4)
    # the same states and keys under another task plan something else
    assert not torch.equal(tr[-1]["Y"][0], tr[-1]["Y"][1])


def test_h1_walk_tasks(built):      # star <5,7>
    envs = [_env("unitree_h1_walk", default_vx=v) for v in (0.5, 1.2, 2.0)]
    _check_tasks("unitree_h1_walk", envs, 64, 10, 4)


def test_allegro_tasks(built):      # dense solver path
    envs = []
    for b in range(3):
        e = _env("allegro_reorient")
        e._ang_vel_tar = np.array([0.0, 0.0, 1.0]) * (b - 1)
        e._pos_tar = np.array([0.0, 0.005 * b, 0.13])
        envs.append(e)
    _check_tasks("allegro_reorient", envs, 16, 4, 2)


def test_generic_tree_tasks(built, monkeypatch):
    monkeypatch.setenv("DIAL_FORCE_GENERIC_TREE", "1")
    _check_tasks("unitree_go2_walk", _go2_sweep(), 64, 10, 4)


def test_many_instances_straddling_ctas(built):
    envs = [_env("unitree_go2_walk", default_vx=-1.0 + 0.09 * b, default_vyaw=0.05 * (b % 5)) for b in range(24)]
    _check_tasks("unitree_go2_walk", envs, 100, 8, 4)


def test_randomize_walk_per_instance_commands(built):
    """Batched randomize_tasks: each instance's one-step random command (step 500) lies inside its horizon
    and differs; the oracle is the single-instance randomize loop (dial_plan_set_command)."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env = _env("unitree_go2_walk", randomize_tasks=True)
    B, N, Hs, Hn = 3, 64, 12, 4
    args = _config("unitree_go2_walk", N, Hs, Hn)
    states, rngs, Y0 = _instances(env, B, Hn, start_step=493)
    assert all(s.info["randomize_target"] for s in states)
    cmds = [env.command_override(s.info, Hs + 2) for s in states]
    assert all(c is not None and c[0] == 500 for c in cmds)
    assert not np.array_equal(cmds[0][1], cmds[1][1])
    loop = DeviceLoop(MBDPI(args, env, n_instances=B), states, rngs, Y0)
    assert "tasks" in loop.buf
    batched = _trace(loop)
    refs = [_trace(DeviceLoop(MBDPI(args, env), states[b], rngs[b], Y0[b])) for b in range(B)]
    _compare(batched, refs)


def test_randomize_seq_jump_per_instance_sequences(built):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env = _env("unitree_go2_seq_jump", randomize_tasks=True)
    B, N, Hs, Hn = 3, 64, 12, 4
    args = _config("unitree_go2_seq_jump", N, Hs, Hn)
    states, rngs, Y0 = _instances(env, B, Hn, start_step=48)
    assert not np.array_equal(states[0].info["pose_target_sequence"], states[1].info["pose_target_sequence"])
    batched = _trace(DeviceLoop(MBDPI(args, env, n_instances=B), states, rngs, Y0))
    refs = [_trace(DeviceLoop(MBDPI(args, env), states[b], rngs[b], Y0[b])) for b in range(B)]
    _compare(batched, refs)
    stages = torch.stack([s["counters"][:, 1] for s in batched])
    assert (stages == 0).any() and (stages == 1).any()


def test_custom_env_user_params(built):
    if EX not in sys.path:
        sys.path.insert(0, EX)
    qe = importlib.import_module("quadpod_env")
    import dial_mpc_b200.envs as E
    envs = [E.get_environment("quadpod_walk", config=qe.QuadpodEnvConfig(target_vx=v, target_height=h))
            for v, h in ((0.2, 0.33), (0.5, 0.30), (0.9, 0.35))]
    _check_tasks("quadpod_walk", envs, 32, 8, 4)


def test_set_task_mid_run(built):
    """set_task on instance 1 of a batched loop == a B = 1 loop with tasks bound that switches at the
    same step; instance 0 is untouched."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    a, b, c = _go2_sweep()
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(a, 2, 4)

    def run(loop, inst):
        out = []
        for t, (nd, es) in enumerate(SCHEDULE):
            if t == 5:
                loop.set_task(inst, c)
            loop.step(nd, env_step=es)
            torch.cuda.synchronize()
            out.append({k: loop.buf[k].clone() for k in KEYS})
        return out
    batched = run(DeviceLoop(MBDPI(args, a, n_instances=2), states, rngs, Y0, envs=[a, b]), 1)
    ref0 = _trace(DeviceLoop(MBDPI(args, a), states[0], rngs[0], Y0[0]))
    ref1 = run(DeviceLoop(MBDPI(args, a), states[1], rngs[1], Y0[1], envs=[b]), 0)
    _compare(batched, [ref0, ref1])
    # the switch changed instance 1's plan: a loop that keeps task b diverges after step 5
    keep = _trace(DeviceLoop(MBDPI(args, a), states[1], rngs[1], Y0[1], envs=[b]))
    assert torch.equal(keep[4]["Y"], ref1[4]["Y"]) and not torch.equal(keep[-1]["Y"], ref1[-1]["Y"])


def test_one_instance_own_task_equals_plain_loop(built):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_seq_jump")
    args = _config("unitree_go2_seq_jump", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 1, 4, 48)
    a = _trace(DeviceLoop(MBDPI(args, env), states[0], rngs[0], Y0[0], envs=[env]))
    b = _trace(DeviceLoop(MBDPI(args, env), states[0], rngs[0], Y0[0]))
    for x, y in zip(a, b):
        for k in KEYS:
            assert torch.equal(x[k], y[k]), k


def test_task_error_paths(built):
    from dial_mpc_b200 import _capi
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    args = _config("unitree_go2_walk", 16, 6, 2)
    mb = MBDPI(args, env, n_instances=2)
    states, rngs, Y0 = _instances(env, 2, 2)
    kp = _env("unitree_go2_walk", kp=env._config.kp * 2)
    with pytest.raises(ValueError, match="'kp'"):
        DeviceLoop(mb, states, rngs, Y0, envs=[env, kp])
    with pytest.raises(ValueError, match="2 envs"):
        DeviceLoop(mb, states, rngs, Y0, envs=[env])
    plain = DeviceLoop(mb, states, rngs, Y0)
    with pytest.raises(RuntimeError, match="envs="):
        plain.set_task(0, env)
    loop = DeviceLoop(mb, states, rngs, Y0, envs=[env, env])
    bad = env.task()
    bad.n_stage = _capi.DEFINES["DIAL_MAXSTAGE"] + 1
    with pytest.raises(ValueError, match="n_stage"):
        loop.set_task(1, bad)
    with pytest.raises(ValueError, match="'kp'"):
        loop.set_task(1, kp)
    # the plan's own task through the C ABI
    import ctypes as C
    t = _capi.dial_task()
    _capi.check(mb.plan.lib.dial_plan_get_task(mb.plan.handle, C.byref(t)))
    assert bytes(t) == bytes(env.task())


def _run(cmd, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    return subprocess.run([sys.executable, "-m", "dial_mpc_b200.core.dial_core"] + cmd, cwd=cwd, env=env,
                          capture_output=True, text=True, timeout=900)


def _cli_runs(tmp_path, runs):
    """runs: name -> (config dict, extra CLI args); returns name -> (states files, predictions files)."""
    out = {}
    for name, (cfg, extra) in runs.items():
        d = tmp_path / name
        d.mkdir()
        (d / "cfg.yaml").write_text(yaml.safe_dump(cfg))
        r = _run(["--config", "cfg.yaml", "--n-steps", "3"] + extra, d)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        out[name] = (sorted(glob.glob(str(d / cfg["output_dir"] / "*_states.npy"))),
                     sorted(glob.glob(str(d / cfg["output_dir"] / "*_predictions.npy"))))
    return out


def _same(a, b):
    return np.array_equal(np.load(a), np.load(b))


def test_cli_randomize_instances_are_the_plain_runs(built, tmp_path):
    base = yaml.safe_load(open(os.path.join(ROOT, "dial_mpc_b200", "examples", "unitree_go2_trot.yaml")))
    base["randomize_tasks"] = True
    out = _cli_runs(tmp_path, {"batched": (base, ["--instances", "2"]),
                               "seed0": (dict(base, seed=base["seed"]), []),
                               "seed1": (dict(base, seed=base["seed"] + 1), [])})
    s, p = out["batched"]
    assert len(s) == 2 and len(p) == 2
    for b in range(2):
        assert "_inst%d_" % b in s[b]
        assert _same(s[b], out[f"seed{b}"][0][0]) and _same(p[b], out[f"seed{b}"][1][0]), b
    assert not _same(s[0], s[1])


def test_cli_instance_overrides(built, tmp_path):
    base = yaml.safe_load(open(os.path.join(ROOT, "dial_mpc_b200", "examples", "unitree_go2_trot.yaml")))
    ov = [{"default_vx": 0.2}, {"default_vx": 0.9, "gait": "walk"}]
    f = tmp_path / "ov.yaml"
    f.write_text(yaml.safe_dump(ov))
    out = _cli_runs(tmp_path, {"batched": (base, ["--instances", "2", "--instance-overrides", str(f)]),
                               "plain0": (dict(base, **ov[0]), []),
                               "plain1": (dict(base, seed=base["seed"] + 1, **ov[1]), [])})
    s, p = out["batched"]
    for b in range(2):
        assert _same(s[b], out[f"plain{b}"][0][0]) and _same(p[b], out[f"plain{b}"][1][0]), b
    # a list of the wrong length and a mapping that changes a shared field are rejected
    (tmp_path / "cfg.yaml").write_text(yaml.safe_dump(base))
    f.write_text(yaml.safe_dump(ov[:1]))
    r = _run(["--config", "cfg.yaml", "--instances", "2", "--instance-overrides", str(f)], tmp_path)
    assert r.returncode != 0 and "list of 2 mappings" in r.stderr
    f.write_text(yaml.safe_dump([{}, {"kp": 80.0}]))
    r = _run(["--config", "cfg.yaml", "--instances", "2", "--instance-overrides", str(f)], tmp_path)
    assert r.returncode != 0 and "'kp'" in r.stderr
