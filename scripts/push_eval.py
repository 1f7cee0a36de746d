"""Push recovery of Go2 trot: how hard a shove of the base the closed loop absorbs.

    python scripts/push_eval.py --steps 150 --magnitudes 50 100 150 200 --delay 2 --ensemble payload.yaml

Go2 trot at BASELINE configs[0] size.  One control-step graph runs one instance per (direction, magnitude): the
base is pushed at --push-step by a horizontal force in one of 8 directions (every 45 degrees, at the base's
origin), held for --push-steps env steps, so the impulse is magnitude x push-steps x dt [N s]
(DeviceLoop(..., pushes=...)).  The planner is not told about the push.  Every instance starts from the same reset
state with the same planner rng, so the instances differ by their push only.  --delay adds a control latency
(predicting through it with ':predict'), --ensemble an ensemble file as dial_core's --ensemble reads it (members,
plant, risk, adapt, prior).  Prints per magnitude the number of directions survived (the base stays above
--fall-height for every step after the push), the minimum base height and the mean env-step reward over the
directions, the largest impulse every direction survived, then one JSON line.  Each number is one run per seed,
not a mean over seeds."""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_instances import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=150)
    ap.add_argument("--push-step", type=int, default=40, help="the post-step counter the push fires at first")
    ap.add_argument("--push-steps", type=int, default=5, help="env steps the force is held for")
    ap.add_argument("--magnitudes", type=float, nargs="+", default=[50.0, 100.0, 150.0, 200.0, 250.0], metavar="N")
    ap.add_argument("--fall-height", type=float, default=0.15)
    ap.add_argument("--seed", type=int, default=None, help="the run's seed (default: the config's)")
    ap.add_argument("--delay", default=None, metavar="STEPS[:predict]")
    ap.add_argument("--ensemble", default=None, metavar="FILE.yaml")
    args = ap.parse_args()
    if args.steps <= args.push_step + args.push_steps:
        ap.error("--steps must run past the push")
    import numpy as np
    import torch
    import yaml
    from baseline_configs import BASELINE, dial_config, product_env
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import MBDPI, DeviceLoop, delay_spec, load_ensemble, load_setting

    cfg = dial_config(0, world=1)
    if args.seed is not None:
        cfg.seed = args.seed
    env = product_env(BASELINE[0]["env"])
    delay = None
    if args.delay is not None:
        try:
            delay = delay_spec(args.delay)
        except ValueError as e:
            ap.error(f"--delay: {e}")
    members, plant, kw = None, None, {}
    if args.ensemble is not None:
        spec = yaml.safe_load(open(args.ensemble))
        members, plant = load_ensemble(spec, env)
        for key in ("risk", "adapt", "prior"):
            kw[key] = load_setting(spec, key, len(members), env.sys.nv)
    plant_env = env
    if plant is not None:
        plant_env = product_env(BASELINE[0]["env"])
        plant_env.sys = env.sys.tree_replace(plant)
    dt = float(env.plan_desc().n_frames) * float(np.float32(env.sys.model.timestep))
    cases = [(f, d) for f in args.magnitudes for d in range(8)]
    pushes = [[{"step": args.push_step, "steps": args.push_steps, "body": "base",
                "force": [f * math.cos(d * math.pi / 4), f * math.sin(d * math.pi / 4), 0.0]}] for f, d in cases]
    B = len(cases)
    mb = MBDPI(cfg, env, n_instances=B, n_ensemble=len(members) if members else 0)
    _, rng_reset = drandom.split(drandom.PRNGKey(cfg.seed))
    states = [plant_env.reset(rng_reset) for _ in range(B)]
    rngs = np.stack([drandom.split(drandom.PRNGKey(cfg.seed))[1]] * B)
    loop = DeviceLoop(mb, states, rngs, envs=[plant_env] * B if members else None, ensemble=members,
                      delay=delay, pushes=pushes, **{k: v for k, v in kw.items() if v is not None})
    rew, z, step = [], [], []
    for t in range(args.steps):
        loop.step(initial=(t == 0))
        rew.append(loop.buf["reward"].clone())
        z.append(loop.buf["qpos"][:, 2].clone())
        step.append(loop.buf["counters"][:, 0].clone())
    rew, z = torch.stack(rew).cpu().numpy(), torch.stack(z).cpu().numpy()
    after = torch.stack(step).cpu().numpy()[:, 0] >= args.push_step
    rows = []
    for f in args.magnitudes:
        idx = [b for b, (g, _) in enumerate(cases) if g == f]
        zmin = z[after][:, idx].min(0)
        rows.append(dict(force=f, impulse=f * args.push_steps * dt, survived=int((zmin >= args.fall_height).sum()),
                         directions=len(idx), min_height=float(zmin.min()), mean_reward=float(rew[:, idx].mean())))
    ok = [r["impulse"] for r in rows if r["survived"] == r["directions"]]
    label = (f"delay {args.delay}" if args.delay else "no delay") + (f", ensemble {os.path.basename(args.ensemble)}"
                                                                     if args.ensemble else "")
    print(f"Go2 trot, configs[0] size (N={cfg.Nsample}, H={cfg.Hsample}, Ndiffuse={cfg.Ndiffuse}), {args.steps} steps, "
          f"seed {cfg.seed} (one run), {label}; base pushed at step {args.push_step} for {args.push_steps} env steps "
          f"of {dt * 1e3:.0f} ms in 8 horizontal directions")
    print("| force [N] | impulse [N s] | directions survived | min base height | mean reward |")
    print("|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['force']:g} | {r['impulse']:.2f} | {r['survived']}/{r['directions']} | {r['min_height']:.3f} | "
              f"{r['mean_reward']:.4f} |")
    print(f"largest impulse survived in every direction: {max(ok) if ok else 0.0:.2f} N s")
    print(json.dumps(dict(steps=args.steps, seed=cfg.seed, delay=args.delay, ensemble=args.ensemble,
                          push_step=args.push_step, push_steps=args.push_steps, results=rows,
                          largest_impulse_survived=max(ok) if ok else 0.0, gpu=gpu_info())))


if __name__ == "__main__":
    main()
