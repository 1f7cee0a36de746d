"""TEST-ONLY custom environments on the tree-shaped fixture models of tests/models/trees/.

They all use the quadpod example's reward (examples/custom_env/quadpod_reward.cuh; its NumPy twin is
tests/test_custom_env.py::_reward_np), so one custom build per solver variant serves them all: the
generic tree solver (variant 0) for branchpod, hexapod and longchain, the quadpod example's star<3,6>
build (variant 1) for slidepod.

Not covered yet: a second kinematic tree on the tree path (e.g. a free object beside the robot).  The
device code takes up to four roots, but BaseEnv reads the joint ranges as jnt_range[1:], assuming every
joint after the root is actuated, so such a model needs host changes before it can be a custom env."""
import os
import tempfile
from dataclasses import dataclass

import numpy as np

import dial_mpc_b200.envs as dial_envs
from dial_mpc_b200.config.base_env_config import BaseEnvConfig
from dial_mpc_b200.envs.base_env import System
from dial_mpc_b200.envs.custom_env import CustomRewardEnv
from dial_mpc_b200.modelc import compile_mjcf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = os.path.join(ROOT, "tests", "models", "trees")
REWARD = os.path.join(ROOT, "dial_mpc_b200", "examples", "custom_env", "quadpod_reward.cuh")


@dataclass
class TreeEnvConfig(BaseEnvConfig):
    kp: object = 20.0
    kd: object = 0.5
    target_vx: float = 0.5
    ramp_up_time: float = 1.0
    target_height: float = 0.3
    energy_weight: float = 0.01
    feet_weight: float = 2.0


class TreeEnv(CustomRewardEnv):
    reward_source = REWARD
    model_file = ""

    def __init__(self, config: TreeEnvConfig):
        super().__init__(config)
        # joint targets are sampled over each joint's whole range: the PD drives joints into their limits
        self.joint_range = self.physical_joint_range.copy()

    def make_system(self, config: TreeEnvConfig) -> System:
        sys = System(compile_mjcf(os.path.join(MODELS, self.model_file)))
        return sys.tree_replace({"opt.timestep": config.timestep})

    def user_params(self):
        c = self._config
        return np.array([c.target_vx, c.ramp_up_time, c.target_height, c.energy_weight, c.feet_weight, 12.0],
                        dtype=np.float32)


class BranchpodEnv(TreeEnv):
    model_file = "branchpod.xml"


class HexapodEnv(TreeEnv):
    model_file = "hexapod.xml"


class LongchainEnv(TreeEnv):
    model_file = "longchain.xml"


class SlidepodEnv(TreeEnv):
    model_file = "slidepod.xml"


# per fixture: env class, configuration (stiff PD on the slide knees of slidepod: they carry the torso)
FIXTURES = {
    "branchpod": (BranchpodEnv, dict(target_height=0.34)),
    "hexapod": (HexapodEnv, dict(target_height=0.14, target_vx=0.3)),
    "longchain": (LongchainEnv, dict(target_height=0.22)),
    "slidepod": (SlidepodEnv, dict(target_height=0.30, kp=[20.0, 400.0] * 4, kd=[0.5, 4.0] * 4)),
}
for _name, (_cls, _) in FIXTURES.items():
    dial_envs.register_environment("tree_" + _name, _cls)
    dial_envs.register_config("tree_" + _name, TreeEnvConfig)


def make_tree_pair(name, **overrides):
    """(product env, oracle env) of a fixture with identical configuration; ``overrides`` go into
    the env configuration (e.g. dt / timestep)."""
    from oracle.envs_oracle import CustomRewardOracle
    from tests.test_custom_env import _reward_np
    cls, kw = FIXTURES[name]
    cfg = TreeEnvConfig(**dict(kw, **overrides))
    env = cls(cfg)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, name + ".json")
        env.sys.model.save(path)
        o = CustomRewardOracle(path, _reward_np, user=env.user_params(), joint_range=env.joint_range,
                               kp=env._kp(), kd=env._kd(), dt=cfg.dt, timestep=cfg.timestep)
    return env, o
