"""The control-step graphs replay what an eager step would launch, across every per-instance setter: a batched
ensemble loop that captures and replays its graphs equals, bit for bit at every step, a loop driven by the same
setter calls whose steps all run eagerly (DIAL_NO_GRAPH=1).  The setter calls come after the graphs were
captured and cover each feature's first setting and the delay and observation calls that change the number of
prediction launches, or whether any instance predicts through its delay, and calls that keep both."""
import pytest
import torch

from tests.conftest import make_pair
from tests.test_gpu_batch import _config, _instances
from tests.test_gpu_instance_models import FEET, LOW_FRICTION, _with_sys

pytestmark = pytest.mark.gpu
B, K = 4, 2
OUT = ("Y", "rews", "rng", "qbar", "qdbar", "xbar", "qpos", "qvel", "qacc_warmstart", "counters", "reward", "ctrl")
SHAPES = [(2, 1), (2, 0), (2, 2)] * 3     # after each call: every shape eager, captured, then replayed


def _script(env):
    """(what, call) pairs, each call applied to a loop; the comment names the key change it makes, if any."""
    heavy = _with_sys(env, {"body_mass": {"base": env.sys.model.arrays["body_mass"][1] + 3.0}})
    slippery = _with_sys(env, {"pair_friction": {f: LOW_FRICTION for f in FEET}})
    return [
        ("instance model", lambda l: l.set_model(1, heavy)),                                   # first: models
        ("member model", lambda l: l.set_ensemble_model(2, 1, slippery)),                      # first: members
        ("risk", lambda l: l.set_risk(0, {"aggregate": "worst"})),                             # none
        ("adaptation on", lambda l: l.set_adapt(0, {"sigma": 0.05})),                          # first: adapt
        ("belief", lambda l: l.set_belief(3, [0.3, 0.7])),                                     # none
        ("schedule", lambda l: l.set_schedule(2, {"Ndiffuse": 2, "temp_sample": 0.08})),       # first: sched
        ("iterations", lambda l: l.plan.set_instance_iterations([2, 1, 2, 0])),                # first: lims
        ("delay, not predicting", lambda l: l.set_delay(1, {"steps": 2, "predict": False})),   # first: delay
        ("delay, predicting", lambda l: l.set_delay(0, {"steps": 3, "predict": True})),        # predicts, 3 launches
        ("delay, shorter prediction", lambda l: l.set_delay(2, {"steps": 1, "predict": True})),   # none
        ("delay, non-predicting only", lambda l: l.set_delay(1, {"steps": 5, "predict": False})),  # none
        ("observation, not predicting", lambda l: l.set_observation(3, {"delay": 2})),         # first: obs
        ("observation, predicting", lambda l: l.set_observation(0, {"delay": 2, "qpos": 0.01})),  # 5 launches
        ("observation, shorter prediction", lambda l: l.set_observation(2, {"delay": 1})),     # none
        ("delay 0, predicting", lambda l: l.set_delay(0, {"steps": 0, "predict": True})),      # 2 launches
        ("delay 0, not predicting", lambda l: l.set_delay(2, {"steps": 0, "predict": False})),  # not predicts
        ("adaptation off", lambda l: l.set_adapt(0, None)),                                    # none
        ("observation removed", lambda l: l.set_observation(0, None)),                         # 0 launches
        ("schedule removed", lambda l: l.set_schedule(2, None)),                               # none
        ("instance model again", lambda l: l.set_model(1, env)),                               # none
    ]


def _snapshot(loop):
    ps, ob = loop.planning_state(), loop.observed_state()
    torch.cuda.synchronize()
    out = {k: loop.buf[k].clone() for k in OUT}
    out.update({"plan." + k: v.clone() for k, v in ps.items()})
    out.update({"obs." + k: v.clone() for k, v in ob.items()})
    return out


def test_captured_graphs_equal_eager_steps_across_setters(built, monkeypatch):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    env, _ = make_pair("unitree_go2_walk")
    args = _config("unitree_go2_walk", 32, 8, 4)
    states, rngs, Y0 = _instances(env, B, 4)
    graph, eager = (DeviceLoop(MBDPI(args, env, n_instances=B, n_ensemble=K), states, rngs, Y0) for _ in range(2))

    def step(n, es, where):
        graph.step(n, env_step=es)
        monkeypatch.setenv("DIAL_NO_GRAPH", "1")
        eager.step(n, env_step=es)
        monkeypatch.delenv("DIAL_NO_GRAPH")
        a, b = _snapshot(graph), _snapshot(eager)
        for k in a:
            assert torch.equal(a[k], b[k]), (where, n, es, k)
        assert graph.plan.launches == eager.plan.launches, (where, n, es)

    for n, es in SHAPES:
        step(n, es, "before the setters")
    for what, call in _script(env):
        call(graph)
        call(eager)
        for n, es in SHAPES:
            step(n, es, what)
