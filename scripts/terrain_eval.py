"""How the Go2 trot does on rough ground and slopes, with a blind planner and a perceptive one.

    python scripts/terrain_eval.py --steps 200 --delay 2:predict --plant '{substeps: 4}' --push '[{step: 60, body: base, force: [60, 0, 0], steps: 5}]'

Go2 trot at BASELINE configs[0] size.  One control-step graph runs one instance per ground and planner
(DeviceLoop(..., terrain=...)): rough ground (value noise, wavelength 0.3 m) of amplitude 0, 2, 4 and 6 cm and
slopes of 0, 5, 10 and 15 degrees rising along +x, each beyond a flat start patch of radius 0.3 m, each once with a
blind planner (it plans on the flat floor) and once with a perceptive one (it plans on the same ground).  Every
instance starts from the same reset state with the same planner rng, so the instances differ by their ground and
planner only.  --delay, --plant (a plant spec) and --push (a push spec) apply to every instance.  Prints per
instance the mean env-step reward, the mean absolute error of the base's world-frame forward velocity against the
commanded one over the second half of the run, the minimum height of the base above the ground beneath it and
whether it fell below --fall-height, then one JSON line.  Each number is one run on one seed, not a mean over
seeds."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_instances import gpu_info  # noqa: E402

GROUNDS = ([(f"rough {a} cm", {"kind": "rough", "amplitude": a / 100, "wavelength": 0.3, "seed": 1, "flat_radius": 0.3})
            for a in (0, 2, 4, 6)]
           + [(f"slope {d} deg", {"kind": "slope", "angle": float(d), "flat_radius": 0.3}) for d in (0, 5, 10, 15)])


def instances():
    """(ground label, planner label, terrain spec) of every instance, blind and perceptive per ground."""
    return [(g, p, dict(spec, planner=p == "perceptive")) for g, spec in GROUNDS for p in ("blind", "perceptive")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--seed", type=int, default=None, help="the run's seed (default: the config's)")
    ap.add_argument("--delay", default=None, metavar="STEPS[:predict]")
    ap.add_argument("--plant", default=None, metavar="SPEC", help="a plant spec (YAML flow mapping) for every instance")
    ap.add_argument("--push", default=None, metavar="SPEC", help="a push spec (YAML flow list) for every instance")
    ap.add_argument("--fall-height", type=float, default=0.15, help="base height above the ground counted as a fall")
    args = ap.parse_args()
    import numpy as np
    import torch
    import yaml
    from baseline_configs import dial_config, product_env
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200 import terrain as T
    from dial_mpc_b200.core.dial_core import MBDPI, DeviceLoop, delay_spec

    delay = None
    if args.delay is not None:
        try:
            delay = delay_spec(args.delay)
        except ValueError as e:
            ap.error(f"--delay: {e}")
    plant = yaml.safe_load(args.plant) if args.plant is not None else None
    push = yaml.safe_load(args.push) if args.push is not None else None
    runs = instances()
    B = len(runs)
    cfg, env = dial_config(0, world=1), product_env("unitree_go2_walk")
    if args.seed is not None:
        cfg.seed = args.seed
    vx = float(env._config.default_vx)
    mb = MBDPI(cfg, env, n_instances=B)
    _, rng_reset = drandom.split(drandom.PRNGKey(cfg.seed))
    states = [env.reset(rng_reset) for _ in range(B)]
    rngs = np.stack([drandom.split(drandom.PRNGKey(cfg.seed))[1]] * B)
    loop = DeviceLoop(mb, states, rngs, delay=delay, plant=plant, pushes=push, terrain=[s for _, _, s in runs])
    grounds = [T.terrain_setting(s).terrain for _, _, s in runs]
    rew, pos, vel = [], [], []
    for t in range(args.steps):
        loop.step(initial=(t == 0))
        rew.append(loop.buf["reward"].clone())
        pos.append(loop.buf["qpos"][:, :3].clone())
        vel.append(loop.buf["qvel"][:, 0].clone())
    rew, pos, vel = (torch.stack(x).double().cpu().numpy() for x in (rew, pos, vel))
    half = args.steps // 2
    rows = []
    for b, (g, p, spec) in enumerate(runs):
        above = pos[:, b, 2] - T.height(grounds[b], pos[:, b, 0], pos[:, b, 1])
        rows.append(dict(ground=g, planner=p, spec=spec, mean_reward=float(rew[:, b].mean()),
                         vel_err=float(np.abs(vel[half:, b] - vx).mean()), min_height=float(above.min()),
                         fell=bool(above.min() < args.fall_height), final_x=float(pos[-1, b, 0])))
    extra = ", ".join(x for x in (f"delay {args.delay}" if args.delay else "", f"plant {args.plant}" if args.plant else "",
                                  f"push {args.push}" if args.push else "") if x) or "no delay, plant or push"
    print(f"Go2 trot, configs[0] size (N={cfg.Nsample}, H={cfg.Hsample}, Ndiffuse={cfg.Ndiffuse}), {args.steps} steps, "
          f"seed {cfg.seed} (one run), {extra}; commanded forward velocity {vx:g} m/s")
    print("| ground | planner | mean reward | forward-velocity error [m/s] | min base height above ground [m] | fell |")
    print("|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['ground']} | {r['planner']} | {r['mean_reward']:.4f} | {r['vel_err']:.3f} | {r['min_height']:.3f} | "
              f"{'yes' if r['fell'] else 'no'} |")
    print(json.dumps(dict(steps=args.steps, delay=args.delay, plant=args.plant, push=args.push, results=rows,
                          gpu=gpu_info())))


if __name__ == "__main__":
    main()
