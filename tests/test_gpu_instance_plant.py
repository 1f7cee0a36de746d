"""Per-instance plant fidelity (dial_plan_set_instance_plant, DeviceLoop(..., plant=...)) on the GPU, at every step of
the eager, captured and replayed schedule.  An instance with the identity setting is bit-identical to one without,
on a Go2 plan that runs the shape-specialised kernel (the plant then runs the generic star<3,6> kernel).  A fidelity
instance runs beside a shadow instance that is given its state, knots and rng before every step: its planner's
outputs equal the shadow's bit for bit, and its env step equals the fp64 oracle's fine env step (n_frames * k
physics steps of timestep / k with the setting's solver settings) from the shared pre-step state and action, within
the emulator's bounds (tests/test_instance_plant.py), on Go2, H1, a tree model and Allegro, in plans whose instances
mix k = 1, 2, 3, 4.  Also: instance models after a setting, ensembles with adaptation, pushes, delay and
observation, the launch sequence, the graph key, the error paths and the CLI."""
import os

import numpy as np
import pytest
import torch
import yaml

from tests.conftest import make_pair
from tests.test_gpu_batch import _config, _instances
from tests.test_gpu_instance_models import _with_sys
from tests.test_gpu_tasks import _cli_runs
from tests.test_instance_plant import fine_oracle

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLANT = ("qpos", "qvel", "qacc_warmstart", "counters")
OUT = ("Y", "rews", "qbar", "qdbar", "xbar", "rng")
ALL = PLANT + OUT + ("reward", "ctrl")
# fidelity instances 1, 3, 5, 7 of a mixed plan: substeps and solver settings (None: the plan's own)
MIXED = [{"substeps": 1, "iterations": 4, "ls_iterations": 10, "tolerance": 1e-6}, {"substeps": 2},
         {"substeps": 3, "iterations": 100, "ls_iterations": 50, "tolerance": 1e-8}, {"substeps": 4}]


def _pair(name):
    if name == "branchpod":
        from tests.tree_envs import make_tree_pair
        env, o = make_tree_pair(name)
        return env, o, "tree_" + name
    env, o = make_pair(name)
    return env, o, name


def _loop(env, cfg_name, B, N=16, Hs=6, Hn=3, twins=False, envs=None, **kw):
    """A batched loop on env; twins: instance 2i + 1 starts as a copy of instance 2i."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    args = _config(cfg_name, N, Hs, Hn)
    states, rngs, Y0 = _instances(env, B, Hn)
    if twins:
        states = [states[b - b % 2] for b in range(B)]
        rngs, Y0 = rngs[[b - b % 2 for b in range(B)]], Y0[[b - b % 2 for b in range(B)]]
    K = len(kw["ensemble"]) if kw.get("ensemble") else 0
    if B == 1:   # one instance: the loop takes a plain state, rng and knots
        states, rngs, Y0 = states[0], rngs[0], Y0[0]
    return DeviceLoop(MBDPI(args, env, n_instances=B, n_ensemble=K), states, rngs, Y0, envs=envs, **kw)


def _shadow(loop, pairs):
    """Give each shadow instance s the state, knots and rng of its fidelity instance p (pairs of (s, p))."""
    for s, p in pairs:
        for k in PLANT + ("Y", "rng"):
            loop.buf[k][s].copy_(loop.buf[k][p])


def _step(loop, n=1, env_step=1):
    loop.step(n, env_step=env_step)
    torch.cuda.synchronize()
    return {k: loop.buf[k].clone() for k in ALL}


def _oracle_step(o, spec, pre, action):
    """The oracle's fine env step of a plant spec from the GPU's pre-step state of one instance."""
    from oracle.envs_oracle import OState
    f = spec
    s = OState(pre["qpos"].double().cpu().numpy()[None], pre["qvel"].double().cpu().numpy()[None],
               pre["qacc_warmstart"].double().cpu().numpy()[None], np.array([int(pre["counters"][0])]),
               np.array([int(pre["counters"][1])]))
    with fine_oracle(o, f.substeps, f.iterations, f.ls_iterations, f.tolerance):
        ns, r, aux = o.step(s, action.double().cpu().numpy()[None])
    return ns, r[0], aux["ctrl"][0]


def _check_fine(o, spec, pre, action, r, p):
    ns, rew, ctrl = _oracle_step(o, spec, pre, action)
    q, v = r["qpos"][p].double().cpu().numpy(), r["qvel"][p].double().cpu().numpy()
    # the bounds of the emulator's parity tests (tests/test_instance_plant.py)
    assert np.abs(q - ns.qpos[0]).max() < 1e-4, np.abs(q - ns.qpos[0]).max()
    assert np.abs(v - ns.qvel[0]).max() < 5e-3 * (1 + np.abs(ns.qvel[0]).max() / 10), np.abs(v - ns.qvel[0]).max()
    assert abs(float(r["reward"][p]) - rew) < 1e-3 * (1 + abs(rew))
    assert np.abs(r["ctrl"][p].double().cpu().numpy() - ctrl).max() < 1e-4 * (1 + np.abs(ctrl).max())
    assert int(r["counters"][p, 0]) == int(pre["counters"][0]) + 1
    return q


def test_identity_setting_equals_no_setting_through_the_generic_kernel(built):
    """Go2 on the shape kernel: a loop whose instance 1 has the identity setting (its plant steps on the generic
    star<3,6> kernel) equals a loop without settings bit for bit, and so does instance 0 without a setting."""
    from dial_mpc_b200 import _capi
    env, _, cfg = _pair("unitree_go2_walk")
    plain = _loop(env, cfg, 2)
    ident = _loop(env, cfg, 2, plant=[None, {}])
    assert _capi.lib().dial_plan_rollout_kernel(plain.plan.handle) == b"go2"
    for t in range(7):
        es = (1, 1, 1, 0, 2, 1, 1)[t]
        a, b = _step(plain, 2, es), _step(ident, 2, es)
        for k in ALL:
            assert torch.equal(a[k], b[k]), (t, k)


@pytest.mark.parametrize("name", ["unitree_go2_walk", "unitree_h1_loco", "branchpod", "allegro_reorient"])
def test_fidelity_instances_equal_the_fine_oracle(built, name):
    """Four pairs (shadow 2i, fidelity 2i + 1) with k = 1 (other solver settings), 2, 3 (MuJoCo's solver) and 4: a
    plan-only step from shared states gives the pair bit-identical planner outputs; an env step from shared states
    moves the fidelity instance as the oracle's fine env step does, and k = 4 away from its shadow."""
    from dial_mpc_b200.core.dial_core import plant_setting
    env, o, cfg = _pair(name)
    loop = _loop(env, cfg, 8, twins=True, plant=[None, MIXED[0], None, MIXED[1], None, MIXED[2], None, MIXED[3]])
    specs = [plant_setting(s, env.sys) for s in MIXED]
    pairs = [(2 * i, 2 * i + 1) for i in range(4)]
    moved = 0.0
    for t in range(4):
        _shadow(loop, pairs)
        r = _step(loop, 1, env_step=0)
        for s, p in pairs:
            for k in PLANT + OUT:     # (reward and ctrl are the last env step's)
                assert torch.equal(r[k][s], r[k][p]), (t, k, p)
        _shadow(loop, pairs)
        pre = {k: loop.buf[k].clone() for k in PLANT}
        act = loop.buf["Y"][:, 0].clone()
        r = _step(loop, 1, env_step=1)
        for i, (s, p) in enumerate(pairs):
            q = _check_fine(o, specs[i], {k: v[p] for k, v in pre.items()}, act[p], r, p)
            if i == 3:
                moved = max(moved, float(np.abs(q - r["qpos"][s].double().cpu().numpy()).max()))
    assert moved > (1e-5 if name == "allegro_reorient" else 1e-4), moved


def test_instance_model_after_the_setting(built):
    """set_model(b) after set_plant(b): the plant steps the new model at its fidelity, the planner plans with the
    new model at the plan's fidelity."""
    from dial_mpc_b200.core.dial_core import plant_setting
    env, o, cfg = _pair("unitree_go2_walk")
    m = env.sys.model
    heavy = _with_sys(env, {"body_mass": {"base": m.arrays["body_mass"][1] + 3.0}})
    loop = _loop(env, cfg, 2, twins=True)
    loop.set_plant(1, {"substeps": 4})
    loop.set_model(0, heavy)
    loop.set_model(1, heavy)
    o.m.body_mass = o.m.body_mass.copy()
    o.m.body_mass[1] = float(np.float32(m.arrays["body_mass"][1] + 3.0))
    spec = plant_setting({"substeps": 4}, env.sys)
    for t in range(4):
        _shadow(loop, [(0, 1)])
        r = _step(loop, 1, env_step=0)
        for k in PLANT + OUT:
            assert torch.equal(r[k][0], r[k][1]), (t, k)
        _shadow(loop, [(0, 1)])
        pre = {k: loop.buf[k][1].clone() for k in PLANT}
        act = loop.buf["Y"][1, 0].clone()
        r = _step(loop, 1, env_step=1)
        _check_fine(o, spec, pre, act, r, 1)
    # the planner's model is the heavy one: a plan-only step differs from a loop planning with the nominal model
    plain = _loop(env, cfg, 2, twins=True)
    plain.set_plant(1, {"substeps": 4})
    for k in PLANT + ("Y", "rng"):
        plain.buf[k].copy_(loop.buf[k])
    a, b = _step(plain, 1, env_step=0), _step(loop, 1, env_step=0)
    assert not torch.equal(a["Y"][1], b["Y"][1])


def test_ensemble_adaptation_scores_coarse_members_against_the_fine_plant(built):
    """Members keep the plan's discretisation: without a setting the member equal to the plant predicts it exactly
    (l = 0); with k = 4 it does not, and the belief moves."""
    env, _, cfg = _pair("unitree_go2_walk")
    heavy = _with_sys(env, {"body_mass": {"base": env.sys.model.arrays["body_mass"][1] + 4.0}})
    loop = _loop(env, cfg, 2, ensemble=[env, heavy], adapt={"sigma": 0.1}, plant=[None, {"substeps": 4}])
    w0 = loop.belief().clone()
    for t in range(4):
        _step(loop)
        ell = loop.member_loglik()
        torch.cuda.synchronize()
        assert float(ell[0, 0]) == 0.0 and float(ell[1, 0]) < 0.0, t
    assert not torch.equal(loop.belief()[1], w0[1])


def test_pushes_delay_and_observation_as_without_a_setting(built):
    """Identity settings on every instance change nothing with pushes, a predicting delay and an observation."""
    env, _, cfg = _pair("unitree_go2_walk")
    kw = dict(pushes=[[{"step": 3, "steps": 2, "body": "base", "force": [60, 0, 0]}], None, None],
              delay=[0, {"steps": 1, "predict": True}, 0], observe=[None, None, {"delay": 1, "qpos": 0.01}])
    a_loop, b_loop = _loop(env, cfg, 3, **kw), _loop(env, cfg, 3, plant={}, **kw)
    for t in range(6):
        a, b = _step(a_loop, 2), _step(b_loop, 2)
        for k in ALL:
            assert torch.equal(a[k], b[k]), (t, k)


def test_launches_and_graph_key(built, monkeypatch):
    """No setting: the stock launch count; settings: one plant launch per distinct k; a captured loop equals an
    eager one across settings that change the group set (recapture) and settings that keep it (restage)."""
    env, _, cfg = _pair("unitree_go2_walk")

    def per_step(loop, es):
        c0 = loop.plan.lib.dial_launch_count(loop.plan.handle)
        loop.step(2, env_step=es)
        return loop.plan.lib.dial_launch_count(loop.plan.handle) - c0

    plain = _loop(env, cfg, 3)
    base = 2 + 2 * 4
    assert [per_step(plain, 1) for _ in range(3)] == [base] * 3
    groups = _loop(env, cfg, 3, plant=[{"substeps": 4}, None, {"substeps": 2}])
    assert [per_step(groups, 1) for _ in range(3)] == [base + 2] * 3
    assert [per_step(groups, 0) for _ in range(3)] == [2 * 4] * 3
    one = _loop(env, cfg, 1, plant={"substeps": 3})
    assert [per_step(one, 1) for _ in range(3)] == [base] * 3

    graph, eager = _loop(env, cfg, 4), _loop(env, cfg, 4)
    script = [lambda l: l.set_plant(1, {"substeps": 4}),                      # first: plant, groups {1, 4}
              lambda l: l.set_plant(2, {"substeps": 4, "iterations": 20}),    # same groups
              lambda l: l.set_plant(1, {"substeps": 2}),                      # groups {1, 2, 4}
              lambda l: l.set_plant(0, {"iterations": 6}),                    # same groups
              lambda l: l.set_plant(2, None),                                 # groups {1, 2}
              lambda l: l.set_plant(1, None)]                                 # groups {1}
    for i, call in enumerate([None] + script):
        if call is not None:
            call(graph)
            call(eager)
        for n, es in [(2, 1), (2, 0), (2, 1), (2, 1)]:
            graph.step(n, env_step=es)
            monkeypatch.setenv("DIAL_NO_GRAPH", "1")
            eager.step(n, env_step=es)
            monkeypatch.delenv("DIAL_NO_GRAPH")
            torch.cuda.synchronize()
            for k in ALL:
                assert torch.equal(graph.buf[k], eager.buf[k]), (i, n, es, k)
            assert graph.plan.launches == eager.plan.launches


def test_errors(built):
    from dial_mpc_b200 import _capi
    from dial_mpc_b200.plan import Plan
    from dial_mpc_b200.utils.spline import interp_matrix
    env, _, cfg = _pair("unitree_go2_walk")
    loop = _loop(env, cfg, 2)
    pl = loop.plan

    def plant(k=1, it=2, ls=5, tol=1e-6):
        f = _capi.dial_plant()
        f.substeps, f.iterations, f.ls_iterations, f.tolerance = k, it, ls, tol
        return f

    with pytest.raises(IndexError, match=r"instance 2 out of range"):
        loop.set_plant(2, {})
    with pytest.raises(RuntimeError, match=r"dial_plan_set_instance_plant: instance -1 out of range"):
        pl.set_instance_plant(-1, plant())
    for f, msg in [(plant(k=0), r"substeps 0 out of range \(1\.\.16\)"), (plant(k=17), r"substeps 17 out of range"),
                   (plant(it=0), r"iterations 0 out of range \(1\.\.100\)"), (plant(it=101), r"iterations 101"),
                   (plant(ls=0), r"ls_iterations 0 out of range \(1\.\.50\)"), (plant(ls=51), r"ls_iterations 51"),
                   (plant(tol=-1.0), r"tolerance must be finite and >= 0, got -1"),
                   (plant(tol=float("nan")), r"tolerance must be finite and >= 0, got nan"),
                   (plant(tol=float("inf")), r"tolerance must be finite and >= 0, got inf")]:
        with pytest.raises(RuntimeError, match=r"dial_plan_set_instance_plant: " + msg):
            pl.set_instance_plant(0, f)
    with pytest.raises(ValueError, match=r"plant must be one plant spec or a list of 2, got a list of 3"):
        _loop(env, cfg, 2, plant=[{}, {}, {}])
    pl.set_instance_plant(0, None)   # clearing without any setting: nothing to do
    desc = env.plan_desc(Nsample=16, Hsample=4, Hnode=2, temp_sample=0.05,
                         M_n2u=interp_matrix(np.linspace(0, 1, 3), np.linspace(0, 1, 5)))
    with pytest.raises(RuntimeError, match=r"dial_plan_set_instance_plant: call dial_mpc_bind first"):
        Plan(env, desc).set_instance_plant(0, plant())
    desc.Ntotal = 32
    with pytest.raises(RuntimeError, match=r"sharded plans \(Ntotal != Nsample\) have no per-instance plant"):
        Plan(env, desc).set_instance_plant(0, plant())
    assert _capi.lib().dial_sizeof(6) == 16


def test_cli_plant(built, tmp_path):
    base = yaml.safe_load(open(os.path.join(ROOT, "dial_mpc_b200", "examples", "unitree_go2_trot.yaml")))
    base.update(Nsample=64, Hsample=8, Hnode=4, Ndiffuse=1, Ndiffuse_init=1)
    ov = tmp_path / "ov.yaml"
    ov.write_text(yaml.safe_dump([{}, {"plant": {"sim_dt": 0.005, "iterations": 100, "ls_iterations": 50}}]))
    out = _cli_runs(tmp_path, {"one": (base, ["--plant", "{sim_dt: 0.005}"]),
                               "ident": (base, ["--plant", "{}"]),
                               "two": (base, ["--instances", "2", "--instance-overrides", str(ov)]),
                               "plain": (base, [])})
    assert len(out["one"][0]) == 1 and len(out["two"][0]) == 2
    plain = np.load(out["plain"][0][0])
    assert np.array_equal(np.load(out["ident"][0][0]), plain)
    assert not np.array_equal(np.load(out["one"][0][0]), plain)
    assert np.array_equal(np.load(out["two"][0][0]), plain)            # instance 0: no setting
    assert not np.array_equal(np.load(out["two"][0][1]), plain)
