"""Closed-loop cost of a noisy, late state estimate, and what predicting through the observation delay recovers.

    python scripts/observe_eval.py --steps 200

Go2 trot at BASELINE configs[0] size.  One control-step graph runs one instance per setting
(DeviceLoop(..., observe=...)): the exact plant state; joint-position noise of standard deviation 0.01, 0.03
and 0.05 rad on every hinge; base linear and angular velocity noise of 0.1 and 0.3 (m/s, rad/s); and an
observation delay of 1..4 control steps (20 ms each), once planning from the late record and once predicting
through it with the actions applied since (a delay setting {steps: 0, predict: true}).  Every instance starts from
the same reset state with the same planner rng and the same noise seed, so the instances differ by their
observation only.  Prints per instance the mean env-step reward, the minimum base height, whether the robot fell
(base height below --fall-height at any step), and the RMS error against the plant at the same step of the
observation and of the planning state (qpos and qvel, every component), then one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_instances import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--fall-height", type=float, default=0.15)
    ap.add_argument("--seed", type=int, default=0, help="the noise seed of every instance")
    args = ap.parse_args()
    if args.steps < 5:
        ap.error("--steps must be at least 5")
    import numpy as np
    import torch
    from baseline_configs import BASELINE, dial_config, product_env
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import MBDPI, DeviceLoop

    cfg = dial_config(0, world=1)
    env = product_env(BASELINE[0]["env"])
    joints = [n for n, t in zip(env.sys.model.names["joint"], env.sys.model.arrays["jnt_type"]) if t == 3]
    # (label, observe spec, predict through the observation delay)
    cases = [("exact", None, False)]
    cases += [(f"joint q sigma {s}", {"qpos": {j: s for j in joints}, "seed": args.seed}, False) for s in (0.01, 0.03, 0.05)]
    cases += [(f"base v sigma {s}", {"qvel": {"": s}, "seed": args.seed}, False) for s in (0.1, 0.3)]
    cases += [(f"delay {k}{' predict' if p else ''}", {"delay": k}, p) for k in range(1, 5) for p in (False, True)]
    B = len(cases)
    mb = MBDPI(cfg, env, n_instances=B)
    _, rng_reset = drandom.split(drandom.PRNGKey(cfg.seed))
    states = [env.reset(rng_reset) for _ in range(B)]
    rngs = np.stack([drandom.split(drandom.PRNGKey(cfg.seed))[1]] * B)
    loop = DeviceLoop(mb, states, rngs, observe=[c[1] for c in cases],
                      delay=[{"steps": 0, "predict": True} if c[2] else 0 for c in cases])
    rew, z, err = [], [], {k: [] for k in ("obs_q", "obs_v", "plan_q", "plan_v")}
    for t in range(args.steps):
        loop.step(cfg.Ndiffuse_init if t == 0 else cfg.Ndiffuse)
        ob, ps = loop.observed_state(), loop.planning_state()
        q, v = loop.buf["qpos"], loop.buf["qvel"]
        rew.append(loop.buf["reward"].clone())
        z.append(q[:, 2].clone())
        err["obs_q"].append(((ob["qpos"] - q) ** 2).mean(-1))
        err["obs_v"].append(((ob["qvel"] - v) ** 2).mean(-1))
        err["plan_q"].append(((ps["qpos"] - q) ** 2).mean(-1))
        err["plan_v"].append(((ps["qvel"] - v) ** 2).mean(-1))
    rew, z = torch.stack(rew).cpu().numpy(), torch.stack(z).cpu().numpy()
    rms = {k: np.sqrt(torch.stack(x).mean(0).cpu().numpy()) for k, x in err.items()}
    rows = []
    for b, (label, spec, p) in enumerate(cases):
        rows.append(dict(setting=label, observe=spec, predict=p, mean_reward=float(rew[:, b].mean()),
                         min_height=float(z[:, b].min()), fell=bool((z[:, b] < args.fall_height).any()),
                         **{f"rms_{k}": float(rms[k][b]) for k in rms}))
    print(f"Go2 trot, configs[0] size (N={cfg.Nsample}, H={cfg.Hsample}, Ndiffuse={cfg.Ndiffuse}), {args.steps} steps, "
          f"noise seed {args.seed}")
    print("| setting | mean reward | min height | fell | RMS obs qpos | RMS obs qvel | RMS plan qpos | RMS plan qvel |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['setting']} | {r['mean_reward']:.4f} | {r['min_height']:.3f} | {'yes' if r['fell'] else 'no'} | "
              f"{r['rms_obs_q']:.2e} | {r['rms_obs_v']:.2e} | {r['rms_plan_q']:.2e} | {r['rms_plan_v']:.2e} |")
    print(json.dumps(dict(steps=args.steps, seed=args.seed, results=rows, gpu=gpu_info())))


if __name__ == "__main__":
    main()
