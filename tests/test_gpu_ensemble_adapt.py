"""Adapting ensemble plans to their plant (dial_plan_set_ensemble_adapt / _belief, dial_plan_ensemble_belief,
DeviceLoop(..., adapt=..., prior=...)): the members' predictions are eager env steps on each member's model,
the log-likelihoods their fp64 restatement bit for bit, the belief the restated update within fp32 rounding,
the scores the weighted restatement (tests/test_ensemble_adapt.py) of the GPU's member rewards under the
GPU's belief bit for bit; an instance that does not adapt is untouched, and the belief identifies the plant."""
import math
import os

import numpy as np
import pytest
import torch
import yaml

from tests.conftest import make_pair
from tests.test_ensemble_adapt import belief_update, member_loglik, weighted_reduce
from tests.test_gpu_batch import KEYS, SCHEDULE, _config, _instances
from tests.test_gpu_ensemble import _snapshot
from tests.test_gpu_instance_models import FEET, LOW_FRICTION, _with_sys
from tests.test_gpu_tasks import _run

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORST, CVAR_HALF, MEAN_SPEC = {"aggregate": "worst"}, {"aggregate": "cvar", "alpha": 0.5}, {"aggregate": "mean"}
FLT_MIN = np.finfo(np.float32).tiny
# the GPU's fp64 exp / log may differ from the C library's in the last bit, and w is rounded to fp32 from
# there: w is compared with the restatement to 1e-6 relative (a few fp32 ulps); weights below FLT_MIN are
# flushed to 0 on the GPU (-use_fast_math)
W_RTOL, W_ATOL = 1e-6, 2 * FLT_MIN


def _ftz(w):
    w = np.asarray(w, np.float32)
    return np.where(np.abs(w) < FLT_MIN, np.float32(0), w)


def _members(env):
    """The nominal model (the plant of the tests below), +3 kg on the base, low foot friction."""
    m = env.sys.model
    return [env, _with_sys(env, {"body_mass": {"base": m.arrays["body_mass"][1] + 3.0}}),
            _with_sys(env, {"pair_friction": {f: LOW_FRICTION for f in FEET}})]


def _eager_qvel(env, st, action):
    """qvel after one eager dial_env_step on a single-instance plan of ``env``'s model."""
    from dial_mpc_b200.envs.base_env import PipelineState, State
    c = st["counters"].cpu().numpy()
    s = State(PipelineState(st["qpos"], st["qvel"], st["qacc_warmstart"], None), None, 0.0, 0.0, {},
              {"step": int(c[0]), "contact_stage": int(c[1])})
    ps, _ = env._get_plan().env_step(s, action)
    return ps.qvel.cpu().numpy()


def test_predictions_belief_and_scores(built):
    """B = 3 adapting instances (mean, CVaR 0.5, worst) over K = 3 members, member 0 equal to the plant: at
    every step of the eager, captured and replayed schedule, l is the restatement from eager env steps of
    each member (member 0: exactly 0), the belief the restated update (unchanged by env_step 0 and 2), and
    rews the weighted restatement of member_rewards() under belief()."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI, adapt_setting, risk_setting
    env, _ = make_pair("unitree_go2_walk")
    members = _members(env)
    B, K, N, Hs, Hn = 3, 3, 64, 12, 4
    risks = [MEAN_SPEC, CVAR_HALF, WORST]
    adapts = [{"sigma": 0.05, "forget": 1.0}, {"sigma": 0.1, "forget": 0.8, "prune": 0.1}, {"sigma": 0.2, "prune": 0.3}]
    args = _config("unitree_go2_walk", N, Hs, Hn)
    states, rngs, Y0 = _instances(env, B, Hn)
    loop = DeviceLoop(MBDPI(args, env, n_instances=B, n_ensemble=K), states, rngs, Y0, ensemble=members,
                      risk=risks, adapt=adapts)
    nv = env.sys.nv
    settings = [risk_setting(r, K) for r in risks]
    ad = [adapt_setting(a, K, nv) for a in adapts]
    L = [[math.log(1.0 / K)] * K for _ in range(B)]
    w = loop.belief()
    torch.cuda.synchronize()
    np.testing.assert_array_equal(w.cpu().numpy(), np.float32(math.exp(math.log(1.0 / K))))
    moved = False
    for t, (nd, es) in enumerate(SCHEDULE):
        pre = _snapshot(loop)
        ll_pre = loop.member_loglik()
        loop.step(nd, env_step=es)
        w, ll, mr = loop.belief(), loop.member_loglik(), loop.member_rewards()
        torch.cuda.synchronize()
        w, ll = w.cpu().numpy(), ll.cpu().numpy()
        for b in range(B):
            forget, prune, sigma = ad[b]
            if es == 1:
                st = {k: pre[k][b] for k in ("qpos", "qvel", "qacc_warmstart", "counters")}
                v = loop.buf["qvel"][b].cpu().numpy()
                ell = [member_loglik(_eager_qvel(members[k], st, pre["Y"][b][0]), v, sigma) for k in range(K)]
                assert ell[0] == 0 and ll[b][0] == 0, (t, b)
                assert np.array_equal(ll[b], np.array(ell, np.float32)), (t, b, ll[b], ell)
                L[b], want = belief_update(L[b], ell, forget)
                np.testing.assert_allclose(w[b], want, rtol=W_RTOL, atol=W_ATOL, err_msg=f"{t} {b}")
            else:   # no env step: the belief and the last l stay as they are
                np.testing.assert_allclose(w[b], _ftz(np.exp(L[b])), rtol=W_RTOL, atol=W_ATOL, err_msg=f"{t} {b}")
                assert torch.equal(loop.member_loglik()[b], ll_pre[b]), (t, b)
            score = weighted_reduce(mr[b].cpu().numpy(), *settings[b], _ftz(w[b]), prune)
            assert torch.equal(loop.buf["rews"][b], torch.as_tensor(score, device="cuda")), (t, b)
        moved |= bool((np.abs(w - 1.0 / K) > 1e-3).any())
    assert moved


def test_instance_without_adaptation_is_untouched(built):
    """Instance 0 adapts, instance 1 does not: instance 1's trace equals that of a loop that never enabled
    adaptation bit for bit; only the env steps of the adapting loop add launches (gather, prediction,
    belief), and a loop that only turns adaptation off launches what the plain loop launches."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    members = _members(env)
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 2, 4)

    def counted(loop):
        out, counts = [], []
        for nd, es in SCHEDULE:
            l0 = loop.plan.launches
            loop.step(nd, env_step=es)
            torch.cuda.synchronize()
            counts.append(loop.plan.launches - l0)
            out.append({k: loop.buf[k].clone() for k in KEYS})
        return out, counts

    plain, n_plain = counted(DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=3), states, rngs, Y0,
                                        ensemble=members, risk=[CVAR_HALF, WORST]))
    off = DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=3), states, rngs, Y0, ensemble=members,
                     risk=[CVAR_HALF, WORST])
    off.set_adapt(0, None)
    off_trace, n_off = counted(off)
    assert n_off == n_plain
    for t in range(len(SCHEDULE)):
        for k in KEYS:
            assert torch.equal(off_trace[t][k], plain[t][k]), (t, k)
    loop = DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=3), states, rngs, Y0, ensemble=members,
                      risk=[CVAR_HALF, WORST], adapt=[{"sigma": 0.05}, None])
    trace, n_adapt = counted(loop)
    assert [a - p for a, p in zip(n_adapt, n_plain)] == [3 if es == 1 else 0 for _, es in SCHEDULE]
    for t in range(len(SCHEDULE)):
        for k in KEYS:
            assert torch.equal(trace[t][k][1], plain[t][k][1]), (t, k)
    assert not torch.equal(trace[-1]["rews"][0], plain[-1]["rews"][0])
    w = loop.belief().cpu().numpy()
    assert np.array_equal(w[1], np.full(3, np.float32(math.exp(math.log(1 / 3))))) and not np.array_equal(w[0], w[1])


def test_identification(built):
    """K = 4 members +0 / +2 / +4 / +6 kg on the base, the plant member 2: member 2 is the argmax after every
    env step and its weight passes 0.9; after set_model switches the plant to member 0 (forget 0.9) the
    argmax moves to member 0."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    base = env.sys.model.arrays["body_mass"][1]
    members = [_with_sys(env, {"body_mass": {"base": base + dm}}) for dm in (0.0, 2.0, 4.0, 6.0)]
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 1, 4)
    sigma = 0.02
    loop = DeviceLoop(MBDPI(args, env, n_ensemble=4), states[0], rngs[0], Y0[0], envs=[members[2]], ensemble=members,
                      adapt={"sigma": sigma})
    history = []
    for t in range(20):
        loop.step(2, env_step=1)
        w = loop.belief().cpu().numpy()
        history.append(w.copy())
        assert int(np.argmax(w)) == 2, (t, w)
    n_id = next(t for t, w in enumerate(history) if w[2] > 0.9) + 1
    print(f"identification: sigma {sigma}: w[2] > 0.9 after {n_id} env steps; final {history[-1]}")
    assert n_id <= 10
    loop.set_model(0, members[0])
    loop.set_adapt(0, {"sigma": sigma, "forget": 0.9})
    moved = None
    for t in range(40):
        loop.step(2, env_step=1)
        w = loop.belief().cpu().numpy()
        if int(np.argmax(w)) == 0:
            moved = t + 1
            break
    print(f"identification: after the switch the argmax is member 0 after {moved} env steps; {w}")
    assert moved is not None and moved <= 30


def test_set_belief_and_set_adapt_between_replays_keep_the_graph(built, monkeypatch):
    """After the (2, 1) graph is captured and replayed, set_belief(1, w) and set_adapt(1, spec) take effect at
    the next replay without a capture: with DIAL_WPC=99 any new enqueue of the step is refused by the
    planner's rollout launch, a replay enqueues nothing.  Instance 1's belief is then one restated update
    of the belief it was given, by the l the replay computed."""
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    members = _members(env)
    args = _config("unitree_go2_walk", 64, 12, 4)
    states, rngs, Y0 = _instances(env, 2, 4)
    loop = DeviceLoop(MBDPI(args, env, n_instances=2, n_ensemble=3), states, rngs, Y0, ensemble=members,
                      adapt=[{"sigma": 0.05}, None])
    for nd, es in SCHEDULE[:4]:       # (3, 1) eager, (2, 1) eager, captured, replayed
        loop.step(nd, env_step=es)
    torch.cuda.synchronize()
    assert (loop.member_loglik()[1] == 0).all() and (loop.member_loglik()[0] != 0).any()
    prior = [0.2, 0.5, 0.3]
    loop.set_belief(1, prior)
    loop.set_adapt(1, {"sigma": 0.1, "forget": 0.5})
    assert np.allclose(loop.belief()[1].cpu().numpy(), prior, rtol=1e-6)
    monkeypatch.setenv("DIAL_WPC", "99")
    launches = loop.plan.launches
    loop.step(2, env_step=1)
    torch.cuda.synchronize()
    assert loop.plan.launches > launches
    with pytest.raises(RuntimeError, match="launch_rollout_any"):
        loop.step(3, env_step=0)       # a shape not captured yet must enqueue, and cannot
    monkeypatch.delenv("DIAL_WPC")
    ell = loop.member_loglik()[1].cpu().numpy().astype(np.float64)
    assert ell[0] == 0 and (ell[1:] < 0).all()
    # l is fp64 on the GPU and read back in fp32: the restated update from it agrees to fp32 rounding
    L0 = [math.log(np.float32(x) / sum(float(np.float32(y)) for y in prior)) for x in prior]
    _, want = belief_update(L0, list(ell), 0.5)
    np.testing.assert_allclose(loop.belief()[1].cpu().numpy(), want, rtol=1e-4, atol=1e-6)


def test_adapt_error_paths(built):
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    args = _config("unitree_go2_walk", 16, 6, 2)
    nv = env.sys.nv
    mb = MBDPI(args, env, n_instances=2, n_ensemble=4)
    states, rngs, Y0 = _instances(env, 2, 2)
    loop = DeviceLoop(mb, states, rngs, Y0)
    s = np.full(nv, 0.1, np.float32)
    for b, forget, prune, sigma, match in [
            (2, 1.0, 0.0, s, "instance 2 out of range"), (-1, 1.0, 0.0, s, "instance -1 out of range"),
            (0, 0.0, 0.0, s, "forget must be in \\(0, 1\\], got 0"), (0, 1.5, 0.0, s, "forget .* got 1.5"),
            (0, float("nan"), 0.0, s, "forget .* got nan"), (0, 1.0, 0.25, s, "prune must be in \\[0, 1/K\\) = \\[0, 0.25\\)"),
            (0, 1.0, -0.1, s, "prune .* got -0.1"), (0, 1.0, 0.0, np.r_[s[:-1], -1.0], "sigma\\[17\\] must be finite and > 0"),
            (0, 1.0, 0.0, np.r_[s[:-1], np.inf], "sigma\\[17\\] .* got inf")]:
        with pytest.raises(RuntimeError, match=match):
            mb.plan.set_ensemble_adapt(b, True, forget, prune, sigma)
    for w, match in [([1, 1, 1, -1], "w\\[3\\] must be finite and >= 0"), ([0, 0, 0, 0], "positive sum"),
                     ([1, float("nan"), 0, 0], "w\\[1\\] .* got nan")]:
        with pytest.raises(RuntimeError, match=match):
            mb.plan.set_ensemble_belief(0, w)
    with pytest.raises(IndexError):
        loop.set_adapt(2, {"sigma": 0.1})
    with pytest.raises(ValueError, match="adapt needs sigma"):
        loop.set_adapt(0, {"forget": 0.5})
    with pytest.raises(ValueError, match="positive sum"):
        loop.set_belief(0, [0, 0, 0, 0])
    with pytest.raises(ValueError, match="list of 2"):
        DeviceLoop(mb, states, rngs, Y0, adapt=[{"sigma": 0.1}])
    # K = 1 and no ensemble are rejected
    one = MBDPI(args, env, n_instances=2, n_ensemble=1)
    with pytest.raises(RuntimeError, match="n_ens >= 2 members, it has 1"):
        one.plan.set_ensemble_adapt(0, True, 1.0, 0.0, s)
    with pytest.raises(RuntimeError, match="n_ens >= 2 members, it has 1"):
        one.plan.set_ensemble_belief(0, [1.0])
    with pytest.raises(ValueError, match="n_ensemble >= 2"):
        DeviceLoop(one, states, rngs, Y0, adapt={"sigma": 0.1})
    plain = MBDPI(args, env)
    with pytest.raises(RuntimeError, match="it has 0"):
        plain.plan.set_ensemble_adapt(0, True, 1.0, 0.0, s)
    with pytest.raises(RuntimeError, match="it has 0"):
        plain.plan.ensemble_belief(None, None)
    state = env.reset(drandom.PRNGKey(0))
    pl = DeviceLoop(plain, state, drandom.PRNGKey(1))
    for call in (lambda: pl.set_adapt(0, {"sigma": 0.1}), lambda: pl.set_belief(0, [1]), pl.belief, pl.member_loglik):
        with pytest.raises(RuntimeError, match="n_ensemble >= 2"):
            call()
    with pytest.raises(ValueError, match="n_ensemble >= 2"):
        DeviceLoop(plain, state, drandom.PRNGKey(1), prior=[1, 1])


def test_cli_adapt(built, tmp_path):
    base = yaml.safe_load(open(os.path.join(ROOT, "dial_mpc_b200", "examples", "unitree_go2_trot.yaml")))
    ens = tmp_path / "ens.yaml"
    ens.write_text(yaml.safe_dump({"members": [{}, {"body_mass": {"base": 9.0}}, {"pair_friction": {f: LOW_FRICTION for f in FEET}}],
                                   "plant": {"body_mass": {"base": 9.0}}, "risk": WORST,
                                   "adapt": {"sigma": 0.05, "forget": 0.95}, "prior": [1, 1, 2]}))
    ov = tmp_path / "ov.yaml"
    ov.write_text(yaml.safe_dump([{"adapt": {"sigma": 0.1, "prune": 0.1}}, {}]))
    (tmp_path / "cfg.yaml").write_text(yaml.safe_dump(base))
    for extra, n in (([], 1), (["--instances", "2", "--instance-overrides", str(ov)], 2)):
        r = _run(["--config", "cfg.yaml", "--n-steps", "4", "--ensemble", str(ens)] + extra, tmp_path)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        lines = [ln for ln in r.stdout.splitlines() if ln.startswith("belief instance")]
        assert len(lines) == n, r.stdout[-2000:]
        for ln in lines:
            w = [float(x) for x in ln.split("=")[1].split()]
            assert len(w) == 3 and abs(sum(w) - 1) < 2e-3 and w != [0.25, 0.25, 0.5]   # moved from the prior
