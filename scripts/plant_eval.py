"""How the closed loop does against a plant that is finer than the planner's model.

    python scripts/plant_eval.py --steps 200 --delay 2:predict --ensemble payload.yaml --push '[{step: 60, body: base, force: [80, 0, 0], steps: 5}]'

Go2 trot at BASELINE configs[0] size and H1 loco (its example's planner settings).  One control-step graph per
robot runs one instance per plant (DeviceLoop(..., plant=...)): the planner's own discretisation (substeps 1, the
model's solver settings), 4 substeps with the model's solver settings, and 4 substeps with MuJoCo's default solver
(100 iterations, 50 line-search iterations, tolerance 1e-8), the setting of the reference's sim-to-sim deploy
(sim_dt 0.005 under a 0.02 s planner step).  Every instance starts from the same reset state with the same planner
rng, so the instances differ by their plant only.  --delay, --ensemble (dial_core's --ensemble file) and --push (a
push spec) apply to every instance.  Prints per robot and plant the mean env-step reward, the mean absolute error of
the base's world-frame forward velocity against the commanded one over the second half of the run, the minimum base
height and whether the base fell below --fall-height, then one JSON line.  Each number is one run on one seed, not
a mean over seeds."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_instances import gpu_info  # noqa: E402

PLANTS = [("k=1, plan solver", {}), ("k=4, plan solver", {"substeps": 4}),
          ("k=4, 100/50/1e-8", {"substeps": 4, "iterations": 100, "ls_iterations": 50, "tolerance": 1e-8})]
FALL = {"unitree_go2_walk": 0.15, "unitree_h1_loco": 0.5}


def robots():
    """(label, DialConfig, env, commanded forward velocity) of each robot."""
    import yaml
    from baseline_configs import dial_config, product_env
    import dial_mpc_b200.envs as E
    from dial_mpc_b200.core.dial_config import DialConfig
    from dial_mpc_b200.utils.io_utils import get_example_path, load_dataclass_from_dict
    go2 = product_env("unitree_go2_walk")
    out = [("Go2 trot, configs[0] size", dial_config(0, world=1), go2, float(go2._config.default_vx))]
    d = yaml.safe_load(open(get_example_path("unitree_h1_loco.yaml")))
    cfg = load_dataclass_from_dict(DialConfig, d)
    env = E.get_environment(cfg.env_name, config=load_dataclass_from_dict(E.get_config(cfg.env_name), d,
                                                                          convert_list_to_array=True))
    out.append(("H1 loco, example size", cfg, env, float(env._config.default_vx)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--seed", type=int, default=None, help="the run's seed (default: the config's)")
    ap.add_argument("--delay", default=None, metavar="STEPS[:predict]")
    ap.add_argument("--ensemble", default=None, metavar="FILE.yaml")
    ap.add_argument("--push", default=None, metavar="SPEC", help="a push spec (YAML flow list) for every instance")
    ap.add_argument("--robots", nargs="+", default=None, help="env names to run (default: unitree_go2_walk unitree_h1_loco)")
    args = ap.parse_args()
    import numpy as np
    import torch
    import yaml
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import MBDPI, DeviceLoop, delay_spec, load_ensemble, load_setting

    delay = None
    if args.delay is not None:
        try:
            delay = delay_spec(args.delay)
        except ValueError as e:
            ap.error(f"--delay: {e}")
    push = yaml.safe_load(args.push) if args.push is not None else None
    B = len(PLANTS)
    results = []
    for label, cfg, env, vx in robots():
        if args.robots and cfg.env_name not in args.robots:
            continue
        if args.seed is not None:
            cfg.seed = args.seed
        members, plant, kw = None, None, {}
        if args.ensemble is not None:
            spec = yaml.safe_load(open(args.ensemble))
            members, plant = load_ensemble(spec, env)
            for key in ("risk", "adapt", "prior"):
                kw[key] = load_setting(spec, key, len(members), env.sys.nv)
        plant_env = env
        if plant is not None:
            plant_env = type(env)(env._config)
            plant_env.sys = env.sys.tree_replace(plant)
        mb = MBDPI(cfg, env, n_instances=B, n_ensemble=len(members) if members else 0)
        _, rng_reset = drandom.split(drandom.PRNGKey(cfg.seed))
        states = [plant_env.reset(rng_reset) for _ in range(B)]
        rngs = np.stack([drandom.split(drandom.PRNGKey(cfg.seed))[1]] * B)
        loop = DeviceLoop(mb, states, rngs, envs=[plant_env] * B if members else None, ensemble=members, delay=delay,
                          pushes=push, plant=[p for _, p in PLANTS], **{k: v for k, v in kw.items() if v is not None})
        rew, z, vel = [], [], []
        for t in range(args.steps):
            loop.step(initial=(t == 0))
            rew.append(loop.buf["reward"].clone())
            z.append(loop.buf["qpos"][:, 2].clone())
            vel.append(loop.buf["qvel"][:, 0].clone())
        rew, z, vel = (torch.stack(x).cpu().numpy() for x in (rew, z, vel))
        half = args.steps // 2
        rows = [dict(robot=cfg.env_name, plant=name, spec=p, mean_reward=float(rew[:, b].mean()),
                     vel_err=float(np.abs(vel[half:, b] - vx).mean()), min_height=float(z[:, b].min()),
                     fell=bool(z[:, b].min() < FALL.get(cfg.env_name, 0.0))) for b, (name, p) in enumerate(PLANTS)]
        extra = ", ".join(x for x in (f"delay {args.delay}" if args.delay else "",
                                      f"ensemble {os.path.basename(args.ensemble)}" if args.ensemble else "",
                                      f"push {args.push}" if args.push else "") if x) or "no delay, ensemble or push"
        print(f"{label} (N={cfg.Nsample}, H={cfg.Hsample}, Ndiffuse={cfg.Ndiffuse}), {args.steps} steps, seed {cfg.seed} "
              f"(one run), {extra}; commanded forward velocity {vx:g} m/s")
        print("| plant | mean reward | forward-velocity error [m/s] | min base height [m] | fell |")
        print("|---|---|---|---|---|")
        for r in rows:
            print(f"| {r['plant']} | {r['mean_reward']:.4f} | {r['vel_err']:.3f} | {r['min_height']:.3f} | "
                  f"{'yes' if r['fell'] else 'no'} |")
        results += rows
    print(json.dumps(dict(steps=args.steps, delay=args.delay, ensemble=args.ensemble, push=args.push,
                          results=results, gpu=gpu_info())))


if __name__ == "__main__":
    main()
