"""The rollout kernel specialised on the Go2 model's integer structure (ShapeFixed, "go2") must compute
bitwise what the generic star<3,6> kernel computes (DIAL_FORCE_GENERIC_SHAPE=1):
rewards, trajectories and bars, the final state and the counters of DeviceLoop control steps (eager first
uses and graph replays, env_step 1, 0 and 2), single and batched plans, at configs[0] and configs[1] size."""
import numpy as np
import pytest
import torch

from tests.conftest import make_pair
from tests.test_gpu_batch import KEYS, _instances, _trace

pytestmark = pytest.mark.gpu


def _config(name, N, Hs, Hn, Nd):
    from dial_mpc_b200.core.dial_config import DialConfig
    return DialConfig(env_name=name, Nsample=N, Hsample=Hs, Hnode=Hn, Ndiffuse=Nd, Ndiffuse_init=Nd + 1,
                      temp_sample=0.05, horizon_diffuse_factor=0.9, traj_diffuse_factor=0.5)


def _loop(name, N, Hs, Hn, Nd, B, start, generic, monkeypatch):
    from dial_mpc_b200.core.dial_core import DeviceLoop, MBDPI
    if generic:
        monkeypatch.setenv("DIAL_FORCE_GENERIC_SHAPE", "1")
    else:
        monkeypatch.delenv("DIAL_FORCE_GENERIC_SHAPE", raising=False)
    env, _ = make_pair(name)
    mb = MBDPI(_config(name, N, Hs, Hn, Nd), env, n_instances=B)
    kernel = mb.plan.lib.dial_plan_rollout_kernel(mb.plan.handle).decode()
    states, rngs, Y0 = _instances(env, B, Hn, start)
    loop = DeviceLoop(mb, states, rngs, Y0) if B > 1 else DeviceLoop(mb, states[0], rngs[0], Y0[0])
    return kernel, _trace(loop)


@pytest.mark.parametrize("name,N,Hs,Hn,Nd,B,start", [
    ("unitree_go2_walk", 128, 16, 4, 2, 1, None),            # configs[0]
    ("unitree_go2_seq_jump", 2048, 25, 5, 4, 1, 46),         # configs[1], across the first stage boundary
    ("unitree_go2_walk", 64, 12, 4, 2, 3, None),             # batched
    ("unitree_go2_seq_jump", 100, 8, 4, 2, 24, 48),          # batched, rows in two waves
])
def test_specialised_kernel_equals_generic(built, monkeypatch, name, N, Hs, Hn, Nd, B, start):
    k_spec, spec = _loop(name, N, Hs, Hn, Nd, B, start, False, monkeypatch)
    k_gen, gen = _loop(name, N, Hs, Hn, Nd, B, start, True, monkeypatch)
    assert (k_spec, k_gen) == ("go2", "v1")
    for t, (a, b) in enumerate(zip(spec, gen)):
        for k in KEYS:
            assert torch.equal(a[k], b[k]), (name, t, k)
    if start is not None:
        stages = torch.stack([s["counters"].reshape(-1, 2)[:, 1] for s in spec])
        assert (stages == 0).any() and (stages == 1).any()
    assert np.isfinite(spec[-1]["rews"].cpu().numpy()).all()


def test_other_models_keep_the_generic_kernel(built):
    from dial_mpc_b200.core.dial_core import MBDPI
    env, _ = make_pair("unitree_h1_walk")
    mb = MBDPI(_config("unitree_h1_walk", 16, 4, 2, 1), env)
    assert mb.plan.lib.dial_plan_rollout_kernel(mb.plan.handle).decode() == "v2"
