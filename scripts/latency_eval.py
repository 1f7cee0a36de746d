"""Closed-loop cost of control latency, and what predicting through it recovers.

    python scripts/latency_eval.py --max-delay 6 --steps 200 [--payload 4 | --plant '{body_mass: {base: 10.0}}']

Go2 trot at BASELINE configs[0] size.  One control-step graph runs 2 D + 1 instances: delay 0, and every
delay d = 1..D (--max-delay) once planning from the plant state and once planning from the state predicted d
steps ahead through the queued actions (DeviceLoop(..., delay=...)).  Every instance starts from the same
reset state with the same planner rng, so the instances differ by their latency only.  At Go2 trot's 20 ms
control step a delay of d steps is 20 d ms.  --plant (a System.tree_replace mapping, as YAML) or --payload KG
(kg added to the base) gives every instance a plant that differs from the planner's model; the planner then
runs a K = 1 ensemble of the nominal model, so the prediction runs on the wrong model too.  Prints per
instance the mean env-step reward, the minimum base height, whether the robot fell (base height below
--fall-height at any step) and the RMS error of the planning state's base position against the plant's d
steps later (for a planner without prediction: how far the state it plans from lags behind), then one JSON
line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_instances import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-delay", type=int, default=6)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--fall-height", type=float, default=0.15)
    g = ap.add_mutually_exclusive_group()
    g.add_argument("--plant", default=None, metavar="YAML",
                   help="the plant's model as a System.tree_replace mapping of the nominal one")
    g.add_argument("--payload", type=float, default=None, metavar="KG", help="the plant carries KG on its base")
    args = ap.parse_args()
    import yaml
    from dial_mpc_b200.core.dial_core import delay_setting
    D = args.max_delay
    try:
        delay_setting(D)
    except ValueError as e:
        ap.error(f"--max-delay: {e}")
    if D < 1 or args.steps <= D:
        ap.error("--max-delay must be at least 1 and --steps larger than it")
    import numpy as np
    import torch
    from baseline_configs import BASELINE, dial_config, product_env
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import MBDPI, DeviceLoop

    cfg = dial_config(0, world=1)
    env = product_env(BASELINE[0]["env"])
    m = env.sys.model
    plant_map = None
    if args.plant is not None:
        plant_map = yaml.safe_load(args.plant)
    elif args.payload is not None:
        plant_map = {"body_mass": {"base": float(m.arrays["body_mass"][m.body_id("base")]) + args.payload}}
    plants = None
    if plant_map is not None:
        import copy
        plant = copy.copy(env)
        try:
            plant.sys = env.sys.tree_replace(plant_map)
        except (KeyError, ValueError) as e:
            ap.error(f"--plant: {e}")
    cases = [(0, False)] + [(d, p) for d in range(1, D + 1) for p in (False, True)]
    B = len(cases)
    if plant_map is not None:
        plants = [plant] * B
    mb = MBDPI(cfg, env, n_instances=B, n_ensemble=1 if plants else 0)
    _, rng_reset = drandom.split(drandom.PRNGKey(cfg.seed))
    states = [(plants[b] if plants else env).reset(rng_reset) for b in range(B)]
    rngs = np.stack([drandom.split(drandom.PRNGKey(cfg.seed))[1]] * B)
    loop = DeviceLoop(mb, states, rngs, envs=plants, ensemble=[env.sys] if plants else None,
                      delay=[{"steps": d, "predict": p} for d, p in cases])
    rew, pos, plan_pos = [], [], []
    for t in range(args.steps):
        loop.step(cfg.Ndiffuse_init if t == 0 else cfg.Ndiffuse)
        rew.append(loop.buf["reward"].clone())
        pos.append(loop.buf["qpos"][:, :3].clone())
        plan_pos.append(loop.planning_state()["qpos"][:, :3])
    rew, pos, plan_pos = (torch.stack(x).cpu().numpy() for x in (rew, pos, plan_pos))
    rows = []
    for b, (d, p) in enumerate(cases):
        err = plan_pos[:args.steps - d, b] - pos[d:, b]          # planning state after step t vs plant after t + d
        rows.append(dict(delay=d, delay_ms=20 * d, predict=p, mean_reward=float(rew[:, b].mean()),
                         min_height=float(pos[:, b, 2].min()), fell=bool((pos[:, b, 2] < args.fall_height).any()),
                         rms_base_pos_err=float(np.sqrt((err ** 2).sum(-1).mean()))))
    print(f"Go2 trot, configs[0] size (N={cfg.Nsample}, H={cfg.Hsample}, Ndiffuse={cfg.Ndiffuse}), {args.steps} steps, "
          f"plant {plant_map or 'nominal'}")
    print("| delay | ms | predict | mean reward | min height | fell | RMS base position error (m) |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['delay']} | {r['delay_ms']} | {'yes' if r['predict'] else 'no'} | {r['mean_reward']:.4f} | "
              f"{r['min_height']:.3f} | {'yes' if r['fell'] else 'no'} | {r['rms_base_pos_err']:.2e} |")
    print(json.dumps(dict(steps=args.steps, max_delay=D, plant=plant_map, results=rows, gpu=gpu_info())))


if __name__ == "__main__":
    main()
