"""Per-instance pushes (dial_plan_set_instance_pushes, DeviceLoop(..., pushes=...)) on the GPU, at every step of the
eager, captured and replayed schedule.  A pushed instance runs beside a shadow instance that is given the pushed
instance's state, knots and rng before every step: the two are bit-identical after every step at which no entry
fires, and at a firing step their qvel difference is the fp64 oracle's solve(M, J^T [torque; force] dt) on the
shared post-step qpos (tests/test_instance_pushes.py), on Go2 (star and generic tree solvers), H1, the four tree
models and Allegro's ball, with per-instance models.  Also: entries that never fire, the stock launch sequence,
trains, the interactions with adaptation, observation and delay prediction, the error paths and the CLI."""
import os

import numpy as np
import pytest
import torch
import yaml

from tests.conftest import make_pair
from tests.test_gpu_batch import _config, _instances
from tests.test_gpu_instance_models import _with_sys
from tests.test_gpu_tasks import _cli_runs
from tests.test_instance_pushes import _dt, _push, oracle_push

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLANT = ("qpos", "qvel", "qacc_warmstart", "counters")
OUT = ("Y", "rews", "qbar", "qdbar", "xbar", "rng")
TREES = ("branchpod", "hexapod", "longchain", "slidepod")


def _env(name):
    if name in TREES:
        from tests.tree_envs import make_tree_pair
        return make_tree_pair(name)[0], "tree_" + name
    return make_pair(name)[0], name


def _loop(env, cfg_name, B, N=16, Hs=6, Hn=3, twins=False, envs=None, **kw):
    """A batched loop on env; twins: instance 2i + 1 starts as a copy of instance 2i."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    args = _config(cfg_name, N, Hs, Hn)
    states, rngs, Y0 = _instances(env, B, Hn)
    if twins:
        states = [states[b - b % 2] for b in range(B)]
        rngs, Y0 = rngs[[b - b % 2 for b in range(B)]], Y0[[b - b % 2 for b in range(B)]]
    K = len(kw["ensemble"]) if kw.get("ensemble") else 0
    return DeviceLoop(MBDPI(args, env, n_instances=B, n_ensemble=K), states, rngs, Y0, envs=envs, **kw)


def _shadow(loop, pairs):
    """Give each shadow instance s the state, knots and rng of its pushed instance p (pairs of (s, p))."""
    for s, p in pairs:
        for k in PLANT + ("Y", "rng"):
            loop.buf[k][s].copy_(loop.buf[k][p])


def _step(loop, n=1, env_step=1):
    loop.step(n, env_step=env_step)
    torch.cuda.synchronize()
    return {k: loop.buf[k].clone() for k in PLANT + OUT + ("reward", "ctrl")}


def _ulp(x):
    return np.spacing(np.abs(np.float32(x))).astype(np.float64)


def _check_push(o, entries, step, dt, r, s, p):
    """Instance p is instance s plus the pushes firing at `step`: the same qpos, and a qvel difference equal to the
    oracle's Delta qvel within one rounding into fp32 and fp64 rounding."""
    assert torch.equal(r["qpos"][s], r["qpos"][p])
    q = r["qpos"][p].double().cpu().numpy()
    v0, v1 = r["qvel"][s].cpu().numpy(), r["qvel"][p].cpu().numpy()
    ref, *_ = oracle_push(o, entries, step, dt, q)
    got = v1.astype(np.float64) - v0.astype(np.float64)
    tol = _ulp(np.maximum(np.abs(v0), np.abs(v1))) + 1e-8 * np.abs(ref).max()
    assert np.all(np.abs(got - ref) <= tol), (step, np.abs(got - ref).max(), tol.max())
    assert np.abs(ref).max() > 0
    # the reward of the step at which the push fires does not see it
    assert torch.equal(r["reward"][s], r["reward"][p])


def _omodel(tmp_path, model, tag):
    from tests.test_instance_pushes import oracle_model
    return oracle_model(model, str(tmp_path / (tag + ".json")))


@pytest.mark.parametrize("name, force_generic", [("unitree_go2_walk", False), ("unitree_go2_walk", True),
                                                 ("unitree_h1_walk", False), ("allegro_reorient", False),
                                                 ("branchpod", False), ("hexapod", False), ("longchain", False),
                                                 ("slidepod", False)])
def test_push_equals_oracle(built, monkeypatch, tmp_path, name, force_generic):
    """A 4-step train on the root body (a point off its COM) and a one-step torque on another body, firing at the
    eager, the captured and replayed steps: bit-identical to the shadow where nothing fires, the oracle's Delta
    qvel where something does, exactly 5 firing steps; Go2 also with per-instance models (a heavier base)."""
    if force_generic:
        monkeypatch.setenv("DIAL_FORCE_GENERIC_TREE", "1")
    env, cfg = _env(name)
    model = env.sys.model
    names = model.names["body"]
    envs = None
    if name == "unitree_go2_walk" and not force_generic:
        heavy = _with_sys(env, {"body_mass": {"base": model.arrays["body_mass"][1] + 3.0}})
        envs = [env, env, heavy, heavy]
    B = 4 if envs else 2
    loop = _loop(env, cfg, B, twins=True, envs=envs)
    root = names.index("object") if name == "allegro_reorient" else 1
    scale = 0.02 if name == "allegro_reorient" else 1.0
    other = names.index("ff_tip") if name == "allegro_reorient" else model.nbody - 1
    pushed = list(range(1, B, 2))
    tables = {}
    for p in pushed:          # each from its own counter
        s0 = int(loop.buf["counters"][p, 0])
        tables[p] = [_push(s0 + 1, root, (0.03, -0.02, 0.01), (40 * scale, -25 * scale, 10 * scale), n_steps=4),
                     _push(s0 + 5, other, (0.0, 0.01, -0.02), torque=(0.5 * scale, 0.2 * scale, -0.3 * scale))]
        loop.set_pushes(p, [{"step": e.step, "steps": e.n_steps, "body": names[e.body], "pos": list(e.pos),
                             "force": list(e.force), "torque": list(e.torque)} for e in tables[p]])
    oms = {p: _omodel(tmp_path, (envs[p] if envs else env).sys.model, f"{name}_{p}") for p in pushed}
    fired = {p: [] for p in pushed}
    for t in range(8):
        _shadow(loop, [(p - 1, p) for p in pushed])
        r = _step(loop)
        for p in pushed:      # each pair at its own counter
            step = int(r["counters"][p, 0])
            if any(e.step <= step < e.step + e.n_steps for e in tables[p]):
                fired[p].append(t)
                _check_push(oms[p], tables[p], step, _dt(env), r, p - 1, p)
            else:
                for k in PLANT + OUT + ("reward", "ctrl"):
                    assert torch.equal(r[k][p - 1], r[k][p]), (t, k, p)
    assert all(f == [0, 1, 2, 3, 4] for f in fired.values())   # from the eager step on


def test_entries_that_never_fire_and_launches(built):
    """A table whose entries never fire leaves its instance bit-identical to an instance without one, and to a
    loop without pushes; a loop without pushes launches env step + shift + (rollout + update + 2 bars) per
    iteration, and pushes add one launch to a step with an env step only."""
    env, cfg = _env("unitree_go2_walk")
    plain = _loop(env, cfg, 3)
    late = [{"step": 10**6, "steps": 5, "body": "base", "force": [100, 0, 0]},
            {"step": 1, "steps": 1, "body": "FR_calf", "force": [0, 50, 0]}]       # fired long before the start
    mixed = _loop(env, cfg, 3, pushes=[None, late, None])
    for t in range(6):
        a, b = _step(plain, 2), _step(mixed, 2)
        for k in PLANT + OUT + ("reward", "ctrl"):
            assert torch.equal(a[k], b[k]), (t, k)

    def per_step(loop, es):
        c0 = loop.plan.lib.dial_launch_count(loop.plan.handle)
        loop.step(2, env_step=es)
        return loop.plan.lib.dial_launch_count(loop.plan.handle) - c0

    for es, base in ((1, 2 + 2 * 4), (0, 2 * 4), (2, 1 + 2 * 4)):
        assert [per_step(plain, es) for _ in range(3)] == [base] * 3, es
        assert [per_step(mixed, es) for _ in range(3)] == [base + (es == 1)] * 3, es
    # later tables keep the launch sequence and take effect at the next replay; clearing keeps the launch
    mixed.set_pushes(0, [{"step": 1, "body": "base"}])
    mixed.set_pushes(2, None)
    assert per_step(mixed, 1) == 2 + 2 * 4 + 1


def test_set_state_moves_the_trigger(built):
    """The trigger is the plant's counter: set_state(step=...) back before a push fires it again."""
    env, cfg = _env("unitree_go2_walk")
    loop = _loop(env, cfg, 2, twins=True)
    s0 = int(loop.buf["counters"][1, 0])
    loop.set_pushes(1, [{"step": s0 + 2, "body": "base", "force": [0, 60, 0]}])
    start = {k: loop.buf[k].clone() for k in PLANT}
    diffs = []
    for rnd in range(2):
        for t in range(3):
            _shadow(loop, [(0, 1)])
            r = _step(loop)
            diffs.append(not torch.equal(r["qvel"][0], r["qvel"][1]))
        loop.set_state(start["qpos"], start["qvel"], start["qacc_warmstart"], step=s0)
    assert diffs == [False, True, False] * 2


def test_adaptation_observation_and_prediction_see_the_push(built):
    """With adaptation on, the member equal to the plant keeps l = 0 at the push step (it scores the unpushed
    qvel); an observation of zero noise records the pushed plant; a predicting instance starts from the pushed
    state, so its prediction equals the next plant state unless the next step pushes."""
    env, cfg = _env("unitree_go2_walk")
    model = env.sys.model
    heavy = _with_sys(env, {"body_mass": {"base": model.arrays["body_mass"][1] + 4.0}})
    # adaptation: member 0 is the plant's model
    loop = _loop(env, cfg, 2, ensemble=[env, heavy], adapt={"sigma": 0.1})
    s0 = int(loop.buf["counters"][0, 0])
    push = [{"step": s0 + 1, "steps": 3, "body": "base", "pos": [0.1, 0, 0], "force": [50, 20, 0]}]
    loop.set_pushes(1, push)
    for t in range(5):
        _step(loop)
        ell = loop.member_loglik()
        torch.cuda.synchronize()
        assert float(ell[1, 0]) == 0.0 and float(ell[0, 0]) == 0.0, t
        assert float(ell[1, 1]) < 0.0
    # observation delay 2, zero noise; prediction through a delay of 1
    k = 2
    loop = _loop(env, cfg, 2, observe=[{"delay": k}, None], delay=[0, {"steps": 1, "predict": True}])
    s0 = int(loop.buf["counters"][0, 0])
    loop.set_pushes(0, [{"step": s0 + 2, "body": "base", "force": [0, 80, 0]},
                        {"step": s0 + 5, "body": "base", "torque": [3, 0, 0]}])
    loop.set_pushes(1, [{"step": s0 + 3, "body": "base", "force": [70, 0, 0]},
                        {"step": s0 + 6, "body": "FL_thigh", "force": [0, 0, 40]}])
    rec = []
    for t in range(8):
        r = _step(loop)
        ob, ps = loop.observed_state(), loop.planning_state()
        torch.cuda.synchronize()
        rec.append(dict(r, obs={k_: v.clone() for k_, v in ob.items()}, plan={k_: v.clone() for k_, v in ps.items()}))
    for t, r in enumerate(rec):
        age = min(k, t)
        for key in PLANT:
            assert torch.equal(r["obs"][key][0], rec[t - age][key][0]), (t, key)
    pushed_next = {s0 + 3, s0 + 6}
    for t in range(len(rec) - 1):
        nxt = int(rec[t + 1]["counters"][1, 0])
        same = all(torch.equal(rec[t]["plan"][key][1], rec[t + 1][key][1]) for key in ("qpos", "qvel"))
        assert same == (nxt not in pushed_next), (t, nxt)


def test_errors(built):
    from dial_mpc_b200 import _capi
    from dial_mpc_b200.plan import Plan
    from dial_mpc_b200.utils.spline import interp_matrix
    env, cfg = _env("unitree_go2_walk")
    loop = _loop(env, cfg, 2)
    pl = loop.plan
    nb = env.sys.model.nbody
    ok = _push(3, 1, force=(1, 0, 0))
    with pytest.raises(IndexError, match=r"instance 2 out of range"):
        loop.set_pushes(2, [{"step": 1, "body": "base"}])
    with pytest.raises(RuntimeError, match=r"dial_plan_set_instance_pushes: instance -1 out of range"):
        pl.set_instance_pushes(-1, [ok])
    with pytest.raises(RuntimeError, match=r"dial_plan_set_instance_pushes: n 17 out of range \(0\.\.16\)"):
        pl.set_instance_pushes(0, [ok] * 17)
    with pytest.raises(RuntimeError, match=r"pushes\[1\]\.body 0 is the world \(1\.\.13\)"):
        pl.set_instance_pushes(0, [ok, _push(3, 0)])
    with pytest.raises(RuntimeError, match=rf"pushes\[0\]\.body {nb} out of range"):
        pl.set_instance_pushes(0, [_push(3, nb)])
    with pytest.raises(RuntimeError, match=r"pushes\[0\]\.step must be >= 1, got 0"):
        pl.set_instance_pushes(0, [_push(0, 1)])
    with pytest.raises(RuntimeError, match=r"pushes\[0\]\.n_steps must be >= 1, got 0"):
        pl.set_instance_pushes(0, [_push(1, 1, n_steps=0)])
    with pytest.raises(RuntimeError, match=r"pushes\[0\]\.torque\[2\] is not finite, got inf"):
        pl.set_instance_pushes(0, [_push(1, 1, torque=(0, 0, np.inf))])
    with pytest.raises(RuntimeError, match=r"pushes\[0\]\.pos\[1\] is not finite, got nan"):
        pl.set_instance_pushes(0, [_push(1, 1, pos=(0, np.nan, 0))])
    with pytest.raises(ValueError, match=r"pushes must be one push spec or a list of 2, got a list of 3"):
        _loop(env, cfg, 2, pushes=[[], [], []])
    desc = env.plan_desc(Nsample=16, Hsample=4, Hnode=2, temp_sample=0.05,
                         M_n2u=interp_matrix(np.linspace(0, 1, 3), np.linspace(0, 1, 5)))
    with pytest.raises(RuntimeError, match=r"dial_plan_set_instance_pushes: call dial_mpc_bind first"):
        Plan(env, desc).set_instance_pushes(0, [ok])
    desc.Ntotal = 32
    with pytest.raises(RuntimeError, match=r"sharded plans \(Ntotal != Nsample\) have no per-instance pushes"):
        Plan(env, desc).set_instance_pushes(0, [ok])
    assert _capi.lib().dial_sizeof(5) == 48


def test_cli_push(built, tmp_path):
    base = yaml.safe_load(open(os.path.join(ROOT, "dial_mpc_b200", "examples", "unitree_go2_trot.yaml")))
    base.update(Nsample=64, Hsample=8, Hnode=4, Ndiffuse=1, Ndiffuse_init=1)
    ov = tmp_path / "ov.yaml"
    ov.write_text(yaml.safe_dump([{}, {"push": [{"step": 2, "body": "base", "force": [0, 90, 0]}]}]))
    out = _cli_runs(tmp_path, {"one": (base, ["--push", "[{step: 2, body: base, force: [90, 0, 0], steps: 2}]"]),
                               "two": (base, ["--instances", "2", "--instance-overrides", str(ov)]),
                               "plain": (base, [])})
    assert len(out["one"][0]) == 1 and len(out["two"][0]) == 2
    plain = np.load(out["plain"][0][0])
    assert not np.array_equal(np.load(out["one"][0][0]), plain)
    assert np.array_equal(np.load(out["two"][0][0]), plain)            # instance 0: no push
    assert not np.array_equal(np.load(out["two"][0][1]), np.load(out["two"][0][0]))
