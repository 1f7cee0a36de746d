"""Risk measures of ensemble plans (dial_plan_set_ensemble_risk, dial_plan_member_rewards, DeviceLoop(...,
risk=...)): the scores are the fp32 restatement (tests/test_ensemble_risk.py) of the member rewards the
GPU computed, bit for bit; the member rewards are what the members compute as instance models; Y, rng and
the bars follow from the scores; the mean setting is the plan without a setting; a setting changed
between two replays of a captured graph takes effect without a new capture."""
import os

import numpy as np
import pytest
import torch
import yaml

from tests.conftest import make_pair
from tests.test_ensemble_risk import CVAR, MEAN, risk_reduce
from tests.test_gpu_batch import KEYS, SCHEDULE, _config, _instances, _trace
from tests.test_gpu_ensemble import _equal_traces, _load, _snapshot
from tests.test_gpu_instance_models import FEET, LOW_FRICTION, _with_sys
from tests.test_gpu_tasks import _cli_runs, _run, _same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORST, CVAR_HALF, MEAN_SPEC = {"aggregate": "worst"}, {"aggregate": "cvar", "alpha": 0.5}, {"aggregate": "mean"}


def _members(env):
    m = env.sys.model
    return [_with_sys(env, {"body_mass": {"base": m.arrays["body_mass"][1] + 3.0}}),
            _with_sys(env, {"pair_friction": {f: LOW_FRICTION for f in FEET}}),
            _with_sys(env, {"dof_damping": m.arrays["dof_damping"] * 2})]


def _scores(mr, settings):
    """The restated reduction of member rewards mr [B,K,N+1] under (mode, alpha) per instance."""
    mr = mr.cpu().numpy()
    return torch.as_tensor(np.stack([risk_reduce(mr[b], *s) for b, s in enumerate(settings)]), device="cuda")


def test_cvar_and_worst_instances_score_the_member_rewards(built):
    """B = 2, K = 3 distinct members, instance 0 CVaR 0.5 and instance 1 the worst case: at every step rews is
    the restatement on member_rewards(), which a K-instance plan with the members as instance models
    reproduces; Y and rng are the fused update on those scores and the bars are member 0's under them."""
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI, risk_setting
    from dial_mpc_b200.envs.base_env import PipelineState, State
    env, _ = make_pair("unitree_go2_walk")
    members = _members(env)
    B, K, N, Hs, Hn = 2, 3, 64, 12, 4
    settings = [risk_setting(CVAR_HALF, K), risk_setting(WORST, K)]
    assert settings == [(CVAR, 0.5), (CVAR, 1 / 3)]
    args = _config("unitree_go2_walk", N, Hs, Hn)
    states, rngs, Y0 = _instances(env, B, Hn)
    loop = DeviceLoop(MBDPI(args, env, n_instances=B, n_ensemble=K), states, rngs, Y0, ensemble=members,
                      risk=[CVAR_HALF, WORST])
    schedule = loop.buf["noise"]
    shifter = DeviceLoop(MBDPI(args, env, n_instances=B), states, rngs, Y0)
    ref = DeviceLoop(MBDPI(args, env, n_instances=K), [states[0]] * K, np.stack([rngs[0]] * K),
                     torch.stack([Y0[0]] * K), envs=members)
    upd = MBDPI(args, env)
    traj0 = MBDPI(args, members[0])
    differs = [False, False]
    for t, (nd, es) in enumerate(SCHEDULE):
        pre = _snapshot(loop)
        loop.step(nd, env_step=es)
        mr = loop.member_rewards()
        torch.cuda.synchronize()
        assert mr.shape == (B, K, N + 1)
        assert torch.equal(loop.buf["rews"], _scores(mr, settings)), t
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
                score = _scores(ref.buf["rews"][None], [settings[b]])[0]
                rng_in, Y_in = rng.clone(), Y.clone()
                Yout, w = torch.empty_like(Y), torch.empty(N + 1, device="cuda")
                upd.plan.reverse_update_fused(score, rng, Y, schedule[i].contiguous(), Yout, w)
                Y = Yout
            assert torch.equal(mr[b], ref.buf["rews"]), (t, b)
            assert torch.equal(loop.buf["rews"][b], score), (t, b)
            assert torch.equal(loop.buf["Y"][b], Y), (t, b)
            assert torch.equal(loop.buf["rng"][b], rng), (t, b)
            mean = torch.as_tensor(risk_reduce(mr[b].cpu().numpy(), MEAN, 0), device="cuda")
            differs[b] |= not torch.equal(score, mean)
            c = st["counters"].cpu().numpy()
            s = State(PipelineState(st["qpos"], st["qvel"], st["qacc_warmstart"], None), None, 0.0, 0.0, {},
                      {"step": int(c[0]), "contact_stage": int(c[1])})
            key = drandom.split(rng_in.cpu().numpy().view(np.uint32))[1]
            traj0.plan.reverse_rollout(s, None, key, Y_in, schedule[nd - 1].contiguous(), torch.empty(N + 1, device="cuda"))
            bars = [torch.empty_like(loop.buf[k][b]) for k in ("qbar", "qdbar", "xbar")]
            traj0.plan.reverse_trajbar(w, 0, *bars)
            for k, v in zip(("qbar", "qdbar", "xbar"), bars):
                assert torch.equal(loop.buf[k][b], v), (t, b, k)
    assert all(differs)     # the settings were read: neither instance scored by the mean


@pytest.mark.parametrize("generic", [False, True])   # the go2 kernel and the generic star <3,6> kernel
def test_explicit_mean_equals_no_setting(built, monkeypatch, generic):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    if generic:
        monkeypatch.setenv("DIAL_FORCE_GENERIC_SHAPE", "1")
    env, _ = make_pair("unitree_go2_walk")
    members = _members(env)[:2]
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 2, 4)
    mb = MBDPI(args, env, n_instances=2, n_ensemble=2)
    assert mb.plan.lib.dial_plan_rollout_kernel(mb.plan.handle) == (b"v1" if generic else b"go2")
    plain = _trace(DeviceLoop(mb, states, rngs, Y0, ensemble=members))
    mean = _trace(DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=2), states, rngs, Y0, ensemble=members,
                             risk=MEAN_SPEC))
    _equal_traces(mean, plain)
    worst = _trace(DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=2), states, rngs, Y0, ensemble=members,
                              risk=WORST))
    assert not torch.equal(worst[0]["rews"], plain[0]["rews"])


def test_cvar_on_one_member_equals_the_plain_loop(built):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 2, 4)
    plain = _trace(DeviceLoop(MBDPI(args, env, n_instances=2), states, rngs, Y0))
    loop = DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=1), states, rngs, Y0, risk=[CVAR_HALF, WORST])
    one = _trace(loop)
    _equal_traces(one, plain)
    # K = 1: the member rewards are rews itself
    assert torch.equal(loop.member_rewards()[:, 0], loop.buf["rews"])


def test_exact_ties(built):
    """Two nominal members and one distinct member: members 0 and 1 tie on every sample."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI, risk_setting
    env, _ = make_pair("unitree_go2_walk")
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 2, 4)
    specs = [{"aggregate": "cvar", "alpha": 0.5}, WORST]
    loop = DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=3), states, rngs, Y0,
                      ensemble=[env, env, _members(env)[1]], risk=specs)
    settings = [risk_setting(s, 3) for s in specs]
    for t, (nd, es) in enumerate(SCHEDULE):
        loop.step(nd, env_step=es)
        mr = loop.member_rewards()
        torch.cuda.synchronize()
        assert torch.equal(mr[:, 0], mr[:, 1]) and not torch.equal(mr[:, 0], mr[:, 2]), t
        assert torch.equal(loop.buf["rews"], _scores(mr, settings)), t


def test_set_risk_between_replays_keeps_the_graph(built, monkeypatch):
    """set_risk after the (2, 1) graph is captured and replayed: the next replay equals a fresh loop built with
    the new setting from the same buffers, and it is a replay: with DIAL_WPC=99 any new enqueue of the step
    (eager or capture) is refused by the rollout launch, a replay enqueues nothing."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    members = _members(env)
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 2, 4)
    loop = DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=3), states, rngs, Y0, ensemble=members)
    for nd, es in SCHEDULE[:4]:       # (3, 1) eager, (2, 1) eager, captured, replayed
        loop.step(nd, env_step=es)
    torch.cuda.synchronize()
    snap = _snapshot(loop)
    loop.set_risk(1, WORST)
    monkeypatch.setenv("DIAL_WPC", "99")
    launches = loop.plan.launches
    loop.step(2, env_step=1)
    torch.cuda.synchronize()
    assert loop.plan.launches > launches
    with pytest.raises(RuntimeError, match="launch_rollout_any"):
        loop.step(3, env_step=0)       # a shape not captured yet must enqueue, and cannot
    monkeypatch.delenv("DIAL_WPC")
    other = DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=3), states, rngs, Y0, ensemble=members,
                       risk=[MEAN_SPEC, WORST])
    _load(other, snap)
    other.step(2, env_step=1)
    torch.cuda.synchronize()
    for k in KEYS:
        assert torch.equal(loop.buf[k], other.buf[k]), k
    base = DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=3), states, rngs, Y0, ensemble=members)
    _load(base, snap)
    base.step(2, env_step=1)
    torch.cuda.synchronize()
    assert torch.equal(base.buf["rews"][0], other.buf["rews"][0])
    assert not torch.equal(base.buf["rews"][1], other.buf["rews"][1])


def test_set_risk_twice_before_a_replay_takes_the_second(built):
    """Two settings of instance 1 written back to back into one staging slot, with no synchronisation
    between them, before a replay of the captured (2, 1) graph: the replay scores instance 1 by the second
    setting, bit for bit the restatement on its member rewards, and instance 0 computes what it computes
    without either call."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI, risk_setting
    env, _ = make_pair("unitree_go2_walk")
    members = _members(env)
    K = len(members)
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 2, 4)
    loop = DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=K), states, rngs, Y0, ensemble=members)
    for nd, es in SCHEDULE[:4]:       # (3, 1) eager, (2, 1) eager, captured, replayed
        loop.step(nd, env_step=es)
    torch.cuda.synchronize()
    snap = _snapshot(loop)
    loop.set_risk(1, WORST)
    loop.set_risk(1, CVAR_HALF)
    loop.step(2, env_step=1)
    mr = loop.member_rewards()
    torch.cuda.synchronize()
    assert torch.equal(loop.buf["rews"], _scores(mr, [risk_setting(MEAN_SPEC, K), risk_setting(CVAR_HALF, K)]))
    assert not torch.equal(loop.buf["rews"][1], _scores(mr[1:], [risk_setting(WORST, K)])[0])
    base = DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=K), states, rngs, Y0, ensemble=members)
    _load(base, snap)
    base.step(2, env_step=1)
    torch.cuda.synchronize()
    for k in KEYS:
        assert torch.equal(loop.buf[k][0], base.buf[k][0]), k


def test_risk_error_paths(built):
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    args = _config("unitree_go2_walk", 16, 6, 2)
    mb = MBDPI(args, env, n_instances=2, n_ensemble=2)
    with pytest.raises(RuntimeError, match="dial_mpc_bind first"):
        mb.plan.member_rewards(torch.empty(2 * 2 * 17, device="cuda"))
    states, rngs, Y0 = _instances(env, 2, 2)
    loop = DeviceLoop(mb, states, rngs, Y0)
    for b, mode, alpha, match in [(2, CVAR, 0.5, "instance 2 out of range"), (-1, MEAN, 1.0, "instance -1 out of range"),
                                  (0, 2, 0.5, "mode 2 is neither"), (0, CVAR, 0.0, "alpha must be finite and in"),
                                  (0, CVAR, 1.5, "got 1.5"), (0, CVAR, float("nan"), "got nan"),
                                  (0, CVAR, float("inf"), "got inf")]:
        with pytest.raises(RuntimeError, match=match):
            mb.plan.set_ensemble_risk(b, mode, alpha)
    mb.plan.set_ensemble_risk(0, MEAN, float("nan"))      # alpha is ignored for the mean
    with pytest.raises(IndexError):
        loop.set_risk(2, WORST)
    with pytest.raises(ValueError, match="aggregate must be one of"):
        loop.set_risk(0, {"aggregate": "median"})
    with pytest.raises(ValueError, match="list of 2"):
        DeviceLoop(mb, states, rngs, Y0, risk=[WORST])
    plain = MBDPI(args, env)
    state = env.reset(drandom.PRNGKey(0))
    with pytest.raises(RuntimeError, match="no ensemble"):
        plain.plan.set_ensemble_risk(0, MEAN, 1.0)
    pl = DeviceLoop(plain, state, drandom.PRNGKey(1))
    with pytest.raises(RuntimeError, match="no ensemble"):
        plain.plan.member_rewards(torch.empty(17, device="cuda"))
    with pytest.raises(RuntimeError, match="n_ensemble >= 1"):
        pl.set_risk(0, WORST)
    with pytest.raises(RuntimeError, match="n_ensemble >= 1"):
        pl.member_rewards()
    with pytest.raises(ValueError, match="n_ensemble >= 1"):
        DeviceLoop(plain, state, drandom.PRNGKey(1), risk=WORST)


def test_cli_risk(built, tmp_path):
    base = yaml.safe_load(open(os.path.join(ROOT, "dial_mpc_b200", "examples", "unitree_go2_trot.yaml")))
    members = [{}, {"body_mass": {"base": 9.0}}, {"pair_friction": {f: LOW_FRICTION for f in FEET}}]
    files = {}
    for name, extra in (("mean", {}), ("explicit", {"risk": MEAN_SPEC}), ("worst", {"risk": WORST})):
        files[name] = tmp_path / f"{name}.yaml"
        files[name].write_text(yaml.safe_dump(dict({"members": members}, **extra)))
    ov = tmp_path / "ov.yaml"
    ov.write_text(yaml.safe_dump([{"risk": WORST}, {}]))
    out = _cli_runs(tmp_path, {"mean": (dict(base), ["--ensemble", str(files["mean"])]),
                               "explicit": (dict(base), ["--ensemble", str(files["explicit"])]),
                               "worst": (dict(base), ["--ensemble", str(files["worst"])]),
                               "per_instance": (dict(base), ["--instances", "2", "--ensemble", str(files["mean"]),
                                                             "--instance-overrides", str(ov)])})
    assert _same(out["explicit"][0][0], out["mean"][0][0]) and _same(out["explicit"][1][0], out["mean"][1][0])
    assert not _same(out["worst"][1][0], out["mean"][1][0])
    # instance 0 of the two-instance run takes its own risk: the single worst-case run
    assert _same(out["per_instance"][0][0], out["worst"][0][0]) and _same(out["per_instance"][1][0], out["worst"][1][0])
    (tmp_path / "cfg.yaml").write_text(yaml.safe_dump(base))
    bad = tmp_path / "bad.yaml"
    bad.write_text(yaml.safe_dump({"members": members, "risk": {"aggregate": "cvar", "alpha": 2}}))
    r = _run(["--config", "cfg.yaml", "--ensemble", str(bad)], tmp_path)
    assert r.returncode == 2 and "risk: alpha must be" in r.stderr
