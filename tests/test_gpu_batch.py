"""Batched planner instances (dial_plan_desc.n_inst > 1, DeviceLoop on MBDPI(..., n_instances=B)):
instance b of a batched control-step graph must compute bitwise what a single-instance DeviceLoop
started from instance b's state, rng and knots computes, at every step (eager first uses and graph
replays, env_step 1, 0 and 2)."""
import glob
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.conftest import make_pair

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (n_diffuse, env_step) per control step: every shape runs eagerly, is captured, then replayed
SCHEDULE = [(3, 1), (2, 1), (2, 1), (2, 1), (2, 0), (2, 0), (2, 0), (2, 2), (2, 2), (2, 2)]
KEYS = ("Y", "rews", "reward", "qpos", "qvel", "qacc_warmstart", "ctrl", "counters", "rng", "qbar", "qdbar", "xbar")


def _config(name, N, Hs, Hn):
    from dial_mpc_b200.core.dial_config import DialConfig
    return DialConfig(env_name=name, Nsample=N, Hsample=Hs, Hnode=Hn, Ndiffuse=2, Ndiffuse_init=3, temp_sample=0.05,
                      horizon_diffuse_factor=0.9, traj_diffuse_factor=0.5)


def _instances(env, B, Hn, start_step=None):
    """B distinct states (reset keys + a few random env steps), rngs and knots."""
    from dial_mpc_b200 import random as drandom
    g = torch.Generator(device="cuda").manual_seed(0)
    states = []
    for b in range(B):
        _, r0 = drandom.split(drandom.PRNGKey(10 + b))
        st = env.reset(r0)
        for _ in range(1 + b % 3):
            st = env.step(st, (torch.rand(env.action_size, device="cuda", generator=g) * 2 - 1) * 0.5)
        if start_step is not None:
            st.info["step"] = start_step + b % 2
            if "contact_stage" in st.info:
                st.info["contact_stage"] = 0
        states.append(st)
    rngs = np.stack([drandom.PRNGKey(100 + 7 * b) for b in range(B)])
    Y0 = ((torch.rand(B, Hn + 1, env.action_size, device="cuda", generator=g) * 2 - 1) * 0.6).contiguous()
    return states, rngs, Y0


def _trace(loop):
    out = []
    for nd, es in SCHEDULE:
        loop.step(nd, env_step=es)
        torch.cuda.synchronize()
        out.append({k: loop.buf[k].clone() for k in KEYS})
    return out


def _check_batched_equals_singles(name, N, Hs, Hn, B, start_step=None):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair(name)
    args = _config(name, N, Hs, Hn)
    states, rngs, Y0 = _instances(env, B, Hn, start_step)
    batched = _trace(DeviceLoop(MBDPI(args, env, n_instances=B), states, rngs, Y0))
    single = MBDPI(args, env)
    for b in range(B):
        ref = _trace(DeviceLoop(single, states[b], rngs[b], Y0[b]))
        for t, (got, want) in enumerate(zip(batched, ref)):
            for k in KEYS:
                g = got[k][b:b + 1] if k == "reward" else got[k][b]
                assert torch.equal(g, want[k]), (name, b, t, SCHEDULE[t], k)
    # the instances really differ
    assert not torch.equal(batched[-1]["Y"][0], batched[-1]["Y"][1])
    return batched


@pytest.mark.parametrize("name,N,Hs,Hn,B,start", [
    ("unitree_go2_walk", 64, 12, 4, 3, None),
    ("unitree_go2_seq_jump", 64, 12, 4, 3, 48),     # the stage changes during the run
    ("unitree_h1_walk", 64, 10, 4, 3, None),         # star <5,7>
    ("allegro_reorient", 16, 4, 2, 3, None),         # dense solver path
    ("unitree_go2_walk", 100, 8, 4, 24, None),       # CTAs straddle instances, rows need two waves
])
def test_batched_loop_equals_single_loops(built, name, N, Hs, Hn, B, start):
    tr = _check_batched_equals_singles(name, N, Hs, Hn, B, start)
    if start is not None:
        stages = torch.stack([s["counters"][:, 1] for s in tr])
        assert (stages == 0).any() and (stages == 1).any()


def test_batched_loop_generic_tree(built, monkeypatch):
    monkeypatch.setenv("DIAL_FORCE_GENERIC_TREE", "1")
    _check_batched_equals_singles("unitree_go2_walk", 64, 10, 4, 3)


def test_one_instance_equals_unbatched_descriptor(built):
    """n_inst = 1 and the zero a caller unaware of the field leaves there are the same plan."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    from dial_mpc_b200.plan import Plan
    env, _ = make_pair("unitree_go2_seq_jump")
    args = _config("unitree_go2_seq_jump", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 1, 4, 48)

    def zero_inst(env_, desc):
        desc.n_inst = 0
        return Plan(env_, desc)
    one = MBDPI(args, env, n_instances=1)
    assert one.plan.desc.n_inst == 1
    a = _trace(DeviceLoop(one, states[0], rngs[0], Y0[0]))
    b = _trace(DeviceLoop(MBDPI(args, env, plan_factory=zero_inst), states[0], rngs[0], Y0[0]))
    for x, y in zip(a, b):
        for k in KEYS:
            assert torch.equal(x[k], y[k]), k


def test_batched_error_paths(built, monkeypatch):
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    from dial_mpc_b200.plan import Plan
    env, _ = make_pair("unitree_go2_walk")
    with pytest.raises(RuntimeError, match="cannot be sharded"):
        Plan(env, env.plan_desc(Nsample=8, Ntotal=16, Hsample=4, Hnode=2, n_inst=2))
    with pytest.raises(RuntimeError, match="131072"):
        Plan(env, env.plan_desc(Nsample=1 << 17, Hsample=4, Hnode=2, n_inst=2))
    with pytest.raises(RuntimeError, match="n_inst too large"):
        Plan(env, env.plan_desc(Nsample=8, Hsample=4, Hnode=2, n_inst=30000))
    args = _config("unitree_go2_walk", 16, 6, 2)
    mb = MBDPI(args, env, n_instances=2)
    states, rngs, Y0 = _instances(env, 2, 2)
    st = states[0]
    with pytest.raises(RuntimeError, match="DeviceLoop"):
        mb.reverse_once(st, rngs[0], Y0[0], mb.sigma_control)
    with pytest.raises(RuntimeError, match="DeviceLoop"):
        mb.reverse_scan(st, rngs[0], Y0[0], mb.schedule(2))
    rews = torch.empty(args.Nsample + 1, device="cuda")
    with pytest.raises(RuntimeError, match="batched plans run through dial_mpc_step"):
        mb.plan.reverse_rollout(st, None, drandom.PRNGKey(0), Y0[0], mb.sigma_control, rews)
    with pytest.raises(RuntimeError, match="batched plans run through dial_mpc_step"):
        mb.plan.reverse_update(None, drandom.PRNGKey(0), Y0[0], mb.sigma_control, rews, torch.empty_like(Y0[0]))
    with pytest.raises(RuntimeError, match="batched plans run through dial_mpc_step"):
        mb.plan.reverse_trajectories()
    with pytest.raises(ValueError, match="2 states"):
        DeviceLoop(mb, states[:1], rngs, Y0)
    rand = [states[0], states[1].replace(info=dict(states[1].info, randomize_target=True))]
    with pytest.raises(RuntimeError, match="randomize_tasks"):
        DeviceLoop(mb, rand, rngs, Y0)
    loop = DeviceLoop(mb, states, rngs, Y0)
    monkeypatch.setenv("DIAL_NO_FUSED_UPDATE", "1")
    with pytest.raises(RuntimeError, match="fused update"):
        loop.step(2, env_step=1)


def test_cli_instance_zero_is_the_plain_run(built, tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    base = [sys.executable, "-m", "dial_mpc_b200.core.dial_core", "--example", "unitree_go2_trot", "--n-steps", "3"]
    for sub, extra in (("plain", []), ("batched", ["--instances", "4"])):
        d = tmp_path / sub
        d.mkdir()
        r = subprocess.run(base + extra, cwd=d, env=env, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    out = lambda sub, pat: sorted(glob.glob(str(tmp_path / sub / "unitree_go2_trot" / pat)))
    plain_s, plain_p = out("plain", "*_states.npy"), out("plain", "*_predictions.npy")
    assert len(plain_s) == 1 and len(plain_p) == 1
    assert len(out("batched", "*_inst*_states.npy")) == 4 and len(out("batched", "*_inst*_predictions.npy")) == 4
    s0, p0 = out("batched", "*_inst0_states.npy"), out("batched", "*_inst0_predictions.npy")
    assert np.array_equal(np.load(s0[0]), np.load(plain_s[0]))
    assert np.array_equal(np.load(p0[0]), np.load(plain_p[0]))
    s1 = np.load(out("batched", "*_inst1_states.npy")[0])
    assert s1.shape == np.load(plain_s[0]).shape and not np.array_equal(s1, np.load(plain_s[0]))
