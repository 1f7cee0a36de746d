"""Ensemble planning (dial_plan_desc.n_ens, dial_plan_set_ensemble_model, DeviceLoop(..., ensemble=...)):
n_ens = 1 with no member set is bitwise the plain loop; with a plant model the env step is the plant's and the
plan the nominal model's; with K distinct members the rewards are the member-order fp32 means of what the
members compute, and Y and the bars follow from them bitwise."""
import os

import numpy as np
import pytest
import torch
import yaml

from tests.conftest import make_pair
from tests.test_gpu_batch import KEYS, SCHEDULE, _config, _instances, _trace
from tests.test_gpu_instance_models import FEET, LOW_FRICTION, _with_sys
from tests.test_gpu_tasks import _cli_runs, _env, _run, _same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATE = ("qpos", "qvel", "qacc_warmstart", "counters", "rng", "Y", "ctrl", "reward")


def _lead(B, states, rngs, Y0):
    return (states, rngs, Y0) if B > 1 else (states[0], rngs[0], Y0[0])


def _equal_traces(a, b):
    for t, (x, y) in enumerate(zip(a, b)):
        for k in KEYS:
            assert torch.equal(x[k], y[k]), (t, SCHEDULE[t], k)


@pytest.mark.parametrize("name, generic, B, N, Hs, Hn", [
    ("unitree_go2_walk", False, 2, 64, 12, 4),       # the go2 kernel
    ("unitree_go2_walk", True, 1, 64, 12, 4),        # generic star <3,6>, single-instance plan
    ("unitree_h1_walk", False, 2, 32, 10, 4),        # star <5,7>
    ("allegro_reorient", False, 2, 16, 4, 2),        # dense solver path
])
def test_one_member_without_members_equals_no_ensemble(built, monkeypatch, name, generic, B, N, Hs, Hn):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    if generic:
        monkeypatch.setenv("DIAL_FORCE_GENERIC_SHAPE", "1")
    env, _ = make_pair(name)
    args = _config(name, N, Hs, Hn)
    states, rngs, Y0 = _instances(env, B, Hn)
    plain = _trace(DeviceLoop(MBDPI(args, env, n_instances=B), *_lead(B, states, rngs, Y0)))
    ens = _trace(DeviceLoop(MBDPI(args, env, n_instances=B, n_ensemble=1), *_lead(B, states, rngs, Y0)))
    _equal_traces(ens, plain)


def test_two_nominal_members_with_random_seq_jump_tasks_equal_no_ensemble(built):
    """K = 2 members that are both the plan's model, bound as member slots: (r + r) / 2 == r, so the
    member rows, the reduction and member 0's bars reproduce the plain loop bitwise."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env = _env("unitree_go2_seq_jump", randomize_tasks=True)
    args = _config("unitree_go2_seq_jump", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 2, 4, start_step=48)
    for s in states:
        assert s.info.get("randomize_target", False)
    plain = _trace(DeviceLoop(MBDPI(args, env, n_instances=2), states, rngs, Y0))
    loop = DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=2), states, rngs, Y0)
    for b in range(2):
        for k in range(2):
            loop.plan.set_ensemble_model(b, k, env.sys)
    _equal_traces(_trace(loop), plain)


def _snapshot(loop):
    return {k: loop.buf[k].clone() for k in STATE}


def _load(loop, snap, b=None):
    for k in STATE:
        loop.buf[k].copy_(snap[k] if b is None else snap[k][b])


def test_plant_differs_from_the_nominal_plan(built):
    """K = 1, member = nominal, plant = base + 3 kg: every env step is the plant model's step from the same
    state and action, every plan the nominal model's plan from the state it reached."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    heavy = _with_sys(env, {"body_mass": {"base": env.sys.model.arrays["body_mass"][1] + 3.0}})
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 1, 4)
    loop = DeviceLoop(MBDPI(args, env, n_ensemble=1), states[0], rngs[0], Y0[0], envs=[heavy])
    stepper = DeviceLoop(MBDPI(args, heavy), states[0], rngs[0], Y0[0])     # env step + shift, no planning
    planner = DeviceLoop(MBDPI(args, env), states[0], rngs[0], Y0[0])       # nominal plan only
    informed = None
    for t, (nd, es) in enumerate(SCHEDULE):
        pre = _snapshot(loop)
        loop.step(nd, env_step=es)
        _load(stepper, pre)
        stepper.step(0, env_step=es)
        _load(planner, _snapshot(stepper))
        planner.step(nd, env_step=0)
        torch.cuda.synchronize()
        for k in ("qpos", "qvel", "qacc_warmstart", "counters"):
            assert torch.equal(loop.buf[k], stepper.buf[k]), (t, k)
        if es == 1:
            for k in ("ctrl", "reward"):
                assert torch.equal(loop.buf[k], stepper.buf[k]), (t, k)
        for k in ("Y", "rng", "rews", "qbar", "qdbar", "xbar"):
            assert torch.equal(loop.buf[k], planner.buf[k]), (t, k)
        if informed is None:
            # a planner that knows the plant plans something else from the same state
            informed = DeviceLoop(MBDPI(args, heavy), states[0], rngs[0], Y0[0])
            _load(informed, _snapshot(stepper))
            informed.step(nd, env_step=0)
            assert not torch.equal(informed.buf["rews"], loop.buf["rews"])


def test_distinct_members_average_the_member_rewards(built):
    """B = 2, K = 3 distinct members: at every step, from the loop's own state, rews is the member-order
    fp32 mean of the rewards a K-instance plan computes with the members as instance models, Y is the fused
    update on those means, and the bars are member 0's under the resulting weights."""
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    from dial_mpc_b200.envs.base_env import PipelineState, State
    from tests.test_ensemble import member_mean
    env, _ = make_pair("unitree_go2_walk")
    m = env.sys.model
    members = [_with_sys(env, {"body_mass": {"base": m.arrays["body_mass"][1] + 3.0}}),
               _with_sys(env, {"pair_friction": {f: LOW_FRICTION for f in FEET}}),
               _with_sys(env, {"dof_damping": m.arrays["dof_damping"] * 2})]
    B, K, N, Hs, Hn = 2, 3, 64, 12, 4
    args = _config("unitree_go2_walk", N, Hs, Hn)
    states, rngs, Y0 = _instances(env, B, Hn)
    loop = DeviceLoop(MBDPI(args, env, n_instances=B, n_ensemble=K), states, rngs, Y0, ensemble=members)
    schedule = loop.buf["noise"]
    shifter = DeviceLoop(MBDPI(args, env, n_instances=B), states, rngs, Y0)
    # the members as the instance models of a K-instance plan; its buffers are overwritten before every use
    ref = DeviceLoop(MBDPI(args, env, n_instances=K), [states[0]] * K, np.stack([rngs[0]] * K),
                     torch.stack([Y0[0]] * K), envs=members)
    upd = MBDPI(args, env)          # the fused update on a single-instance plan
    traj0 = MBDPI(args, members[0])  # member 0's trajectories (eager rollout)
    for t, (nd, es) in enumerate(SCHEDULE):
        pre = _snapshot(loop)
        loop.step(nd, env_step=es)
        torch.cuda.synchronize()
        Ystart = pre["Y"]
        if es in (1, 2):
            _load(shifter, pre)
            shifter.step(0, env_step=2)
            Ystart = shifter.buf["Y"].clone()
        for b in range(B):
            st = {k: loop.buf[k][b] for k in ("qpos", "qvel", "qacc_warmstart", "counters")}
            rng, Y = pre["rng"][b].clone(), Ystart[b].clone()
            for i in range(nd):
                for k in range(K):
                    for name, v in st.items():
                        ref.buf[name][k].copy_(v)
                    ref.buf["rng"][k].copy_(rng)
                    ref.buf["Y"][k].copy_(Y)
                ref.buf["noise"][0].copy_(schedule[i])
                ref.step(1, env_step=0)
                rbar = torch.as_tensor(member_mean(ref.buf["rews"].cpu().numpy()[None])[0], device="cuda")
                rng_in, Y_in = rng.clone(), Y.clone()
                Yout, w = torch.empty_like(Y), torch.empty(N + 1, device="cuda")
                upd.plan.reverse_update_fused(rbar, rng, Y, schedule[i].contiguous(), Yout, w)
                Y = Yout
            assert torch.equal(loop.buf["rews"][b], rbar), (t, b)
            assert torch.equal(loop.buf["Y"][b], Y), (t, b)
            assert torch.equal(loop.buf["rng"][b], rng), (t, b)
            # member 0's bars under the ensemble weights of the last iteration
            c = st["counters"].cpu().numpy()
            s = State(PipelineState(st["qpos"], st["qvel"], st["qacc_warmstart"], None), None, 0.0, 0.0, {},
                      {"step": int(c[0]), "contact_stage": int(c[1])})
            key = drandom.split(rng_in.cpu().numpy().view(np.uint32))[1]
            traj0.plan.reverse_rollout(s, None, key, Y_in, schedule[nd - 1].contiguous(), torch.empty(N + 1, device="cuda"))
            bars = [torch.empty_like(loop.buf[k][b]) for k in ("qbar", "qdbar", "xbar")]
            traj0.plan.reverse_trajbar(w, 0, *bars)
            for k, v in zip(("qbar", "qdbar", "xbar"), bars):
                assert torch.equal(loop.buf[k][b], v), (t, b, k)


def test_set_ensemble_model_between_steps(built):
    """Setting a member mid-run == a loop built with that member, from the same buffers on."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    heavy = _with_sys(env, {"body_mass": {"base": env.sys.model.arrays["body_mass"][1] + 3.0}})
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 2, 4)
    loop = DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=2), states, rngs, Y0)
    for nd, es in SCHEDULE[:4]:
        loop.step(nd, env_step=es)
    loop.set_ensemble_model(1, 1, heavy)
    other = DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=2), states, rngs, Y0,
                       ensemble=[[env, env], [env, heavy]])
    _load(other, _snapshot(loop))
    launches = loop.plan.launches
    for nd, es in SCHEDULE[4:]:
        loop.step(nd, env_step=es)
        other.step(nd, env_step=es)
        torch.cuda.synchronize()
        for k in KEYS:
            assert torch.equal(loop.buf[k], other.buf[k]), (nd, es, k)
    assert loop.plan.launches > launches
    # the member was read: instance 0 (nominal members) and instance 1 now plan differently from a loop without it
    plain = DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=2), states, rngs, Y0)
    _load(plain, _snapshot(other))
    plain.step(2, env_step=0)
    other.step(2, env_step=0)
    torch.cuda.synchronize()
    assert torch.equal(plain.buf["rews"][0], other.buf["rews"][0])
    assert not torch.equal(plain.buf["rews"][1], other.buf["rews"][1])


def test_ensemble_error_paths(built):
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    from dial_mpc_b200.plan import Plan
    env, _ = make_pair("unitree_go2_walk")
    args = _config("unitree_go2_walk", 16, 6, 2)
    with pytest.raises(RuntimeError, match="cannot be sharded"):
        Plan(env, env.plan_desc(Nsample=8, Ntotal=16, Hsample=4, Hnode=2, n_ens=1))
    with pytest.raises(RuntimeError, match="n_ens out of range"):
        Plan(env, env.plan_desc(Nsample=8, Hsample=4, Hnode=2, n_ens=17))
    with pytest.raises(ValueError, match="n_ensemble"):
        MBDPI(args, env, n_ensemble=17)
    mb = MBDPI(args, env, n_ensemble=2)
    state = env.reset(drandom.PRNGKey(0))
    Y = torch.zeros(args.Hnode + 1, mb.nu, device="cuda")
    for call in (lambda: mb.reverse_once(state, drandom.PRNGKey(1), Y, mb.sigma_control),
                 lambda: mb.reverse_scan(state, drandom.PRNGKey(1), Y, mb.schedule(2)),
                 lambda: mb.phase_times(state, drandom.PRNGKey(1), Y, mb.sigma_control)):
        with pytest.raises(RuntimeError, match="ensemble plan"):
            call()
    loop = DeviceLoop(mb, state, drandom.PRNGKey(1))
    with pytest.raises(RuntimeError, match="'timestep'"):
        loop.set_ensemble_model(0, 1, env.sys.tree_replace({"opt.timestep": 0.01}))
    with pytest.raises(IndexError):
        loop.set_ensemble_model(0, 2, env)
    with pytest.raises(IndexError):
        loop.set_ensemble_model(1, 0, env)
    with pytest.raises(RuntimeError, match="member 2 out of range"):
        mb.plan.set_ensemble_model(0, 2, env.sys)
    with pytest.raises(RuntimeError, match="instance 1 out of range"):
        mb.plan.set_ensemble_model(1, 0, env.sys)
    with pytest.raises(ValueError, match="list of 2 models"):
        DeviceLoop(mb, state, drandom.PRNGKey(1), ensemble=[env])
    plain = MBDPI(args, env)
    with pytest.raises(RuntimeError, match="no ensemble"):
        plain.plan.set_ensemble_model(0, 0, env.sys)
    with pytest.raises(RuntimeError, match="n_ensemble >= 1"):
        DeviceLoop(plain, state, drandom.PRNGKey(1)).set_ensemble_model(0, 0, env)
    with pytest.raises(ValueError, match="n_ensemble >= 1"):
        DeviceLoop(plain, state, drandom.PRNGKey(1), ensemble=[env])


def test_cli_ensemble(built, tmp_path):
    base = yaml.safe_load(open(os.path.join(ROOT, "dial_mpc_b200", "examples", "unitree_go2_trot.yaml")))
    nominal, planted = tmp_path / "nominal.yaml", tmp_path / "planted.yaml"
    nominal.write_text(yaml.safe_dump({"members": [{}]}))
    planted.write_text(yaml.safe_dump({"members": [{}, {"body_mass": {"base": 9.0}}],
                                       "plant": {"body_mass": {"base": 9.9}}}))
    out = _cli_runs(tmp_path, {"plain": (dict(base), []),
                               "nominal": (dict(base), ["--ensemble", str(nominal)]),
                               "planted": (dict(base), ["--ensemble", str(planted)]),
                               "planted2": (dict(base), ["--instances", "2", "--ensemble", str(planted)])})
    # one nominal member and no plant: the plain run, bitwise
    assert _same(out["nominal"][0][0], out["plain"][0][0]) and _same(out["nominal"][1][0], out["plain"][1][0])
    assert len(out["planted"][0]) == 1 and not _same(out["planted"][0][0], out["plain"][0][0])
    # instance 0 of a two-instance run is the single run with the same file
    assert len(out["planted2"][0]) == 2 and _same(out["planted2"][0][0], out["planted"][0][0])
    bad = tmp_path / "bad.yaml"
    bad.write_text(yaml.safe_dump({"members": [{"pair_kind": [0, 0, 0, 0]}]}))
    (tmp_path / "cfg.yaml").write_text(yaml.safe_dump(base))
    r = _run(["--config", "cfg.yaml", "--ensemble", str(bad)], tmp_path)
    assert r.returncode != 0 and "members[0]" in r.stderr
