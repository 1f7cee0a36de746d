"""Per-instance terrain (dial_plan_set_instance_terrain, DeviceLoop(..., terrain=...)) on the GPU, at the eager,
captured and replayed steps of the control-step graph.  Instances without a terrain beside terrain instances are
bit-identical to a plan without terrain, on a Go2 plan that ran the shape kernel before; a flat terrain at z = 0 on
both sides is bit-identical to no terrain.  With a plant-only terrain, the plant's env step equals the fp64
oracle's env step on that terrain (tests/terrain_oracle.py) within the emulator's bounds, and the planner's
outputs equal a shadow instance's bit for bit.  With a planner-side terrain, sampled rows of the planner's rollouts
equal the oracle's rollouts on that terrain, and adaptation's member steps and the prediction launches read it.
Also: the error paths, and restaged and larger tables."""
import numpy as np
import pytest
import torch

from tests.test_gpu_instance_plant import ALL, OUT, PLANT, _loop, _shadow, _step
from tests.test_gpu_instance_plant import _pair as _stock_pair
from tests.test_instance_plant import fine_oracle
from tests.terrain_oracle import on_terrain

pytestmark = pytest.mark.gpu

ROUGH = {"kind": "rough", "amplitude": 0.015, "wavelength": 0.25, "seed": 2, "size": 4.0, "spacing": 0.05,
         "flat_radius": 0.0}
SLOPE = {"kind": "slope", "angle": 6.0, "heading": 20.0, "size": 4.0, "spacing": 0.1, "flat_radius": 0.1}
FLAT = {"kind": "grid", "heights": np.zeros((8, 8)).tolist(), "spacing": 0.5, "origin": [-2.0, -2.0], "planner": True}


def _pair(name):
    """The stock pairs; the tree model with its custom reward compiled with the terrain branch."""
    if name == "branchpod":
        from tests.tree_envs import make_tree_pair
        env, o = make_tree_pair(name)
        env.build_defines = ("DIAL_TERRAIN",)
        return env, o, "tree_" + name
    return _stock_pair(name)


@pytest.mark.parametrize("name", ["unitree_go2_walk", "unitree_h1_walk", "unitree_h1_loco", "branchpod"])
def test_instances_without_terrain_and_flat_terrain_are_bitwise_unchanged(built, name):
    """On every variant with a terrain build (star<3,6> from the Go2 shape kernel, star<5,7>, star<5,6>, the tree
    with a custom reward compiled with and without the terrain branch): the instances without a terrain, and a
    flat terrain at z = 0, compute bitwise what a plan without terrain computes."""
    from dial_mpc_b200 import _capi
    env, _, cfg = _pair(name)
    plain = _loop(_stock_pair(name)[0], cfg, 3)
    mixed = _loop(env, cfg, 3)
    flat = _loop(_pair(name)[0], cfg, 3, terrain=FLAT)
    want = {"unitree_go2_walk": b"go2", "unitree_h1_walk": b"v2", "unitree_h1_loco": b"v4", "branchpod": b"v0"}[name]
    assert plain.plan.lib.dial_plan_rollout_kernel(plain.plan.handle) == want
    for t in range(8):
        if t == 2:   # the shape kernel ran first; the terrain arrives later
            mixed.set_terrain(1, dict(ROUGH, planner=True))
        es = (1, 1, 1, 0, 1, 2, 1, 1)[t]
        a, b, c = _step(plain, 2, es), _step(mixed, 2, es), _step(flat, 2, es)
        for k in ALL:
            assert torch.equal(a[k], c[k]), (t, k)
            for i in (0, 2):
                assert torch.equal(a[k][i], b[k][i]), (t, k, i)
        if t >= 3:
            assert not torch.equal(a["qpos"][1], b["qpos"][1])


def _rollout_rows(name, spec, Hs, rows, N=32, Hn=4):
    """A one-instance loop planning on ``spec``'s terrain: the GPU's rollout q and mean rewards of ``rows`` and the
    fp64 oracle's rollouts of the same rows on that terrain (knots from the oracle's restatement of the sampler,
    tests/ctrl_probe.py)."""
    from dial_mpc_b200.terrain import terrain_setting
    from oracle.envs_oracle import OState
    from tests import ctrl_probe as cp
    env, o, cfg = _pair(name)
    loop = _loop(env, cfg, 1, N=N, Hs=Hs, Hn=Hn, terrain=dict(spec, planner=True))
    loop.buf["Y"].copy_(torch.randn(loop.buf["Y"].shape, generator=torch.Generator().manual_seed(7)).mul(0.4).to(loop.buf["Y"]))
    torch.cuda.synchronize()
    npy = lambda t: t.detach().cpu().numpy()
    rng = npy(loop.buf["rng"]).view(np.uint32)
    Ybar, noise = npy(loop.buf["Y"]).astype(np.float64), npy(loop.buf["noise"][0]).astype(np.float64)
    pre = {k: npy(loop.buf[k]) for k in PLANT}
    loop.step(1, env_step=0)
    torch.cuda.synchronize()
    rews = npy(loop.info()["rews"]).astype(np.float64)
    q, _, _ = loop.plan.reverse_trajectories()
    q = npy(q).astype(np.float64)
    nu = env.action_size
    Y, _ = cp.knots64(cp.eps_xla(cp.sample_key(rng), N, Hn, nu), rows, N, 0, Ybar, noise)
    us = np.einsum("tk,rka->rta", cp.spline64(Hs, Hn), Y)
    s = OState(pre["qpos"][None].astype(np.float64), pre["qvel"][None].astype(np.float64),
               pre["qacc_warmstart"][None].astype(np.float64), np.array([int(pre["counters"][0])]),
               np.array([int(pre["counters"][1])]))
    with on_terrain(o, terrain_setting(spec).terrain):
        rew_o, q_o, _, _ = o.rollout(s, us)
    _, q_flat, _, _ = o.rollout(s, us)
    return q[rows], rews[rows], q_o, rew_o, q_flat


@pytest.mark.parametrize("name,Hs", [("unitree_go2_walk", 16), ("unitree_h1_loco", 20)])
@pytest.mark.parametrize("ground", ["rough", "slope"])
def test_planner_rollouts_on_terrain_equal_the_oracle(built, name, Hs, ground):
    """Planner-side terrain: sampled rows of the planner's rollout (and the mean row) match the fp64 oracle's
    rollouts of the same knots on the same terrain, states and per-row mean rewards at test_gpu_parity's bounds
    (q 2e-4, mean rewards 1e-3 (1 + |r|)); the terrain moves the rollouts beyond those bounds."""
    rows = np.array([0, 3, 8, 13, 21, 31, 32])
    qg, rg, q_o, rew_o, q_flat = _rollout_rows(name, ROUGH if ground == "rough" else SLOPE, Hs, rows)
    assert np.abs(qg - q_o).max() < 2e-4, np.abs(qg - q_o).max()
    r = rew_o.mean(1)
    assert (np.abs(rg - r) < 1e-3 * (1 + np.abs(r))).all(), np.abs(rg - r).max()
    assert np.abs(q_flat - q_o).max() > 1e-3


def test_adaptation_members_read_the_planner_terrain(built):
    """Adaptation's member steps run on the planner's terrain: with the same terrain on both sides the member equal
    to the plant predicts it exactly (l = 0); with a blind planner on the same ground it does not."""
    from tests.test_gpu_instance_models import _with_sys
    env, _, cfg = _pair("unitree_go2_walk")
    heavy = _with_sys(env, {"body_mass": {"base": env.sys.model.arrays["body_mass"][1] + 4.0}})
    loop = _loop(env, cfg, 2, ensemble=[env, heavy], adapt={"sigma": 0.1},
                 terrain=[dict(SLOPE, planner=True), SLOPE])
    for t in range(4):
        _step(loop)
        ell = loop.member_loglik()
        torch.cuda.synchronize()
        assert float(ell[0, 0]) == 0.0 and float(ell[1, 0]) < 0.0, (t, ell)


def _check(o, spec, pre, action, r, p, substeps=1):
    from dial_mpc_b200.terrain import terrain_setting
    from oracle.envs_oracle import OState
    t = terrain_setting(spec).terrain
    s = OState(pre["qpos"].double().cpu().numpy()[None], pre["qvel"].double().cpu().numpy()[None],
               pre["qacc_warmstart"].double().cpu().numpy()[None], np.array([int(pre["counters"][0])]),
               np.array([int(pre["counters"][1])]))
    with on_terrain(o, t), fine_oracle(o, substeps):
        ns, rew, aux = o.step(s, action.double().cpu().numpy()[None])
    q, v = r["qpos"][p].double().cpu().numpy(), r["qvel"][p].double().cpu().numpy()
    assert np.abs(q - ns.qpos[0]).max() < 1e-4, np.abs(q - ns.qpos[0]).max()
    assert np.abs(v - ns.qvel[0]).max() < 5e-3 * (1 + np.abs(ns.qvel[0]).max() / 10), np.abs(v - ns.qvel[0]).max()
    assert abs(float(r["reward"][p]) - rew[0]) < 1e-3 * (1 + abs(rew[0])), (float(r["reward"][p]), rew[0])


@pytest.mark.parametrize("name,substeps", [("unitree_go2_walk", 1), ("unitree_go2_walk", 4), ("unitree_h1_loco", 1),
                                           ("branchpod", 1)])
def test_plant_terrain_equals_the_oracle(built, name, substeps):
    """Pairs (shadow 2i, terrain 2i + 1) on rough ground and a slope, the planner blind: a plan-only step from shared
    states gives the pair bit-identical planner outputs; the env step of the terrain instance is the oracle's."""
    env, o, cfg = _pair(name)
    specs = [ROUGH, SLOPE]
    kw = {"plant": {"substeps": substeps}} if substeps > 1 else {}
    loop = _loop(env, cfg, 4, twins=True, terrain=[None, ROUGH, None, SLOPE], **kw)
    pairs = [(0, 1), (2, 3)]
    for t in range(4):
        _shadow(loop, pairs)
        r = _step(loop, 1, env_step=0)
        for s, p in pairs:
            for k in PLANT + OUT:
                assert torch.equal(r[k][s], r[k][p]), (t, k, p)
        _shadow(loop, pairs)
        pre = {k: loop.buf[k].clone() for k in PLANT}
        act = loop.buf["Y"][:, 0].clone()
        r = _step(loop, 1, env_step=1)
        for i, (s, p) in enumerate(pairs):
            _check(o, specs[i], {k: v[p] for k, v in pre.items()}, act[p], r, p, substeps)


def test_restage_and_larger_tables(built, monkeypatch):
    """A captured loop equals an eager one across the first terrain, same-size restages, a larger grid, a flat
    side and the planner side."""
    env, _, cfg = _pair("unitree_go2_walk")
    graph, eager = _loop(env, cfg, 3), _loop(env, cfg, 3)
    script = [lambda l: l.set_terrain(1, ROUGH),
              lambda l: l.set_terrain(1, dict(ROUGH, seed=5)),
              lambda l: l.set_terrain(1, dict(ROUGH, size=6.0)),
              lambda l: l.set_terrain(2, dict(SLOPE, planner=True)),
              lambda l: l.set_terrain(1, None)]
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


def test_errors(built):
    from dial_mpc_b200 import _capi
    from dial_mpc_b200.plan import Plan
    from dial_mpc_b200.terrain import Terrain, grid
    from dial_mpc_b200.utils.spline import interp_matrix
    env, _, cfg = _pair("unitree_go2_walk")
    loop = _loop(env, cfg, 2)
    pl = loop.plan
    ok = grid(np.zeros((3, 3)), 0.1)
    with pytest.raises(RuntimeError, match=r"dial_plan_set_instance_terrain: instance 2 out of range"):
        pl.set_instance_terrain(2, 0, ok)
    with pytest.raises(RuntimeError, match=r"side 2 out of range \(0 plant, 1 planner\)"):
        pl.set_instance_terrain(0, 2, ok)
    for t, msg in [(Terrain(np.zeros((1, 3), np.float32), 0.1, (0.0, 0.0)), r"grid 3 x 1 out of range \(2\.\.1024 per side\)"),
                   (Terrain(np.zeros((2, 1025), np.float32), 0.1, (0.0, 0.0)), r"grid 1025 x 2 out of range"),
                   (Terrain(np.zeros((2, 2), np.float32), 0.0, (0.0, 0.0)), r"spacing must be finite and > 0, got 0"),
                   (Terrain(np.zeros((2, 2), np.float32), float("inf"), (0.0, 0.0)), r"spacing must be finite"),
                   (Terrain(np.array([[0, 0], [0, np.nan]], np.float32), 0.1, (0.0, 0.0)), r"heights\[1\]\[1\] is not finite")]:
        with pytest.raises(RuntimeError, match=r"dial_plan_set_instance_terrain: " + msg):
            pl.set_instance_terrain(0, 0, t)
    pl.set_instance_terrain(0, 1, None)   # flat without any terrain: nothing to do
    desc = env.plan_desc(Nsample=16, Hsample=4, Hnode=2, temp_sample=0.05,
                         M_n2u=interp_matrix(np.linspace(0, 1, 3), np.linspace(0, 1, 5)))
    with pytest.raises(RuntimeError, match=r"dial_plan_set_instance_terrain: call dial_mpc_bind first"):
        Plan(env, desc).set_instance_terrain(0, 0, ok)
    desc.Ntotal = 32
    with pytest.raises(RuntimeError, match=r"sharded plans \(Ntotal != Nsample\) have no per-instance terrain"):
        Plan(env, desc).set_instance_terrain(0, 0, ok)
    aenv, _, acfg = _pair("allegro_reorient")
    with pytest.raises(RuntimeError, match=r"dial_plan_set_instance_terrain: the dense solver path has no terrain build"):
        _loop(aenv, acfg, 2, terrain={"kind": "slope", "angle": 3})
    tenv, _, tcfg = _stock_pair("branchpod")   # a custom build without the terrain branch
    with pytest.raises(RuntimeError, match=r"this custom build has no terrain kernel \(compile it with DIAL_TERRAIN\)"):
        _loop(tenv, tcfg, 2, terrain={"kind": "slope", "angle": 3})
    assert _capi.lib().dial_sizeof(7) == 32


def test_prediction_reads_the_planner_terrain(built):
    """delay {steps: 2, predict: true} and the same terrain on both sides: the planning state recorded after step t
    equals the plant state after step t + 2 bit for bit (the prediction launches read the planner's terrain)."""
    env, _, cfg = _pair("unitree_go2_walk")
    loop = _loop(env, cfg, 2, delay={"steps": 2, "predict": True}, terrain=[None, dict(SLOPE, planner=True)])
    planned, plant = [], []
    for t in range(8):
        loop.step(1)
        torch.cuda.synchronize()
        planned.append({k: v.clone() for k, v in loop.planning_state().items()})
        plant.append({k: loop.buf[k].clone() for k in PLANT})
    for t in range(6):
        for k in PLANT:
            assert torch.equal(planned[t][k], plant[t + 2][k]), (t, k)
