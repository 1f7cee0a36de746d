"""Closed-loop comparison of a nominal planner and an ensemble planner on robots that differ from the model.

    python scripts/ensemble_eval.py --plants 8 --steps 200 --ensemble 4 [--risk mean worst cvar:0.5]

Go2 trot at BASELINE configs[0] size.  B plants span a payload on the base of +0 ... +6 kg and a foot friction
of 1.0 ... 0.4 (plant b: payload 6 b / (B-1) kg, friction 1 - 0.6 b / (B-1)); every instance starts from the
same reset state and its own planner rng.  Planner A plans on the nominal model (n_ens = 1, the plain mismatch
experiment).  Planner B plans on a K-member ensemble spanning the same range (member k: payload 6 k / (K-1) kg,
friction 1 - 0.6 k / (K-1)) and weights every sample by a risk measure of its member rewards; --risk lists
the measures (mean, worst, cvar:ALPHA; default mean), one ensemble planner each.  Every planner runs the
reference's closed loop (env step, shift, Ndiffuse iterations) for --steps control steps in one control-step
graph per step, B instances at a time.  --adapt SIGMA[:FORGET] adds, for each measure, an ensemble planner
that adapts its belief over the members to its plant at every env step (DeviceLoop(..., adapt=...)), and
reports the final belief on the member nearest the plant.  Prints a table per plant: mean env-step reward,
minimum base height and whether the robot fell (base height below --fall-height at any step), and one JSON
line."""
import argparse
import copy
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scripts.bench_instances import adapt_spec, gpu_info, risk_spec  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--plants", type=int, default=8)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--ensemble", type=int, default=4)
    ap.add_argument("--fall-height", type=float, default=0.15)
    ap.add_argument("--risk", nargs="+", default=["mean"], metavar="MEASURE",
                    help="one ensemble planner per measure: mean, worst or cvar:ALPHA (default: mean)")
    ap.add_argument("--adapt", default=None, metavar="SIGMA[:FORGET]",
                    help="also run, per measure, an ensemble planner adapting its belief to the plant")
    args = ap.parse_args()
    if args.plants < 2 or args.ensemble < 2 or args.steps < 1:
        ap.error("--plants and --ensemble must be at least 2, --steps at least 1")
    from dial_mpc_b200.core.dial_core import risk_setting
    risks = []
    for tok in args.risk:
        try:
            spec = risk_spec(tok)
            risk_setting(spec, args.ensemble)
        except ValueError as e:
            ap.error(f"--risk {tok}: {e}")
        risks.append((tok, spec))
    adapt = None
    if args.adapt is not None:
        try:
            adapt = adapt_spec(args.adapt)
        except ValueError as e:
            ap.error(f"--adapt {args.adapt}: {e}")
    import numpy as np
    import torch
    from baseline_configs import BASELINE, dial_config, product_env
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import MBDPI, DeviceLoop

    cfg = dial_config(0, world=1)
    env = product_env(BASELINE[0]["env"])
    m = env.sys.model
    base = m.body_id("base")

    def model(f):
        """env's model with payload 6 f kg on the base and the feet's sliding friction scaled by 1 - 0.6 f
        (f in [0, 1]; the contact pairs of the Go2 scene are the four feet on the floor)."""
        fr = m.arrays["pair_friction"].copy()
        fr[:, :2] *= 1.0 - 0.6 * f
        e = copy.copy(env)
        e.sys = env.sys.tree_replace({"body_mass": {"base": m.arrays["body_mass"][base] + 6.0 * f},
                                      "pair_friction": fr})
        return e

    B, K = args.plants, args.ensemble
    plants = [model(b / (B - 1)) for b in range(B)]
    members = [model(k / (K - 1)).sys for k in range(K)]
    rng, rng_reset = drandom.split(drandom.PRNGKey(cfg.seed))
    results = {}
    # the member nearest plant b: payload and friction both move with f, so the nearest f
    nearest = [int(round(b / (B - 1) * (K - 1))) for b in range(B)]
    planners = [("nominal", [env.sys], None, None)]
    planners += [(f"ensemble{K}" if tok == "mean" else f"ensemble{K}-{tok}", members, spec, None) for tok, spec in risks]
    if adapt is not None:
        planners += [(f"adapt{K}" if tok == "mean" else f"adapt{K}-{tok}", members, spec, adapt) for tok, spec in risks]
    for name, ens, risk, ad in planners:
        mb = MBDPI(cfg, env, n_instances=B, n_ensemble=len(ens))
        states = [p.reset(rng_reset) for p in plants]
        rngs = np.stack([drandom.split(drandom.PRNGKey(cfg.seed + b))[1] for b in range(B)])
        loop = DeviceLoop(mb, states, rngs, envs=plants, ensemble=ens, risk=risk, adapt=ad)
        rew, height = [], []
        for t in range(args.steps):
            loop.step(cfg.Ndiffuse_init if t == 0 else cfg.Ndiffuse)
            rew.append(loop.buf["reward"].clone())
            height.append(loop.buf["qpos"][:, 2].clone())
        rew, height = torch.stack(rew).cpu().numpy(), torch.stack(height).cpu().numpy()
        results[name] = dict(mean_reward=rew.mean(0).tolist(), min_height=height.min(0).tolist(),
                             fell=(height < args.fall_height).any(0).tolist())
        if ad is not None:
            w = loop.belief().cpu().numpy()
            results[name]["belief_nearest"] = [float(w[b, nearest[b]]) for b in range(B)]
    print(f"Go2 trot, configs[0] size (N={cfg.Nsample}, H={cfg.Hsample}, Ndiffuse={cfg.Ndiffuse}), {args.steps} steps")
    names = list(results)
    print("| payload kg | friction | " + " | ".join(f"{n} reward | {n} min height | {n} fell" for n in names) + " |")
    print("|---|---|" + "---|---|---|" * len(names))
    for b in range(B):
        f = b / (B - 1)
        cells = []
        for n in names:
            r = results[n]
            cells += [f"{r['mean_reward'][b]:.3f}", f"{r['min_height'][b]:.3f}", "yes" if r["fell"][b] else "no"]
        print(f"| {6 * f:.2f} | {1 - 0.6 * f:.2f} | " + " | ".join(cells) + " |")
    adaptive = [n for n in names if "belief_nearest" in results[n]]
    if adaptive:
        print("| payload kg | friction | nearest member | " + " | ".join(f"{n} belief on it" for n in adaptive) + " |")
        print("|---|---|---|" + "---|" * len(adaptive))
        for b in range(B):
            f = b / (B - 1)
            print(f"| {6 * f:.2f} | {1 - 0.6 * f:.2f} | {nearest[b]} | "
                  + " | ".join(f"{results[n]['belief_nearest'][b]:.3f}" for n in adaptive) + " |")
    for n in names:
        r = results[n]
        print(f"{n}: mean reward {np.mean(r['mean_reward']):.4f}, falls {sum(r['fell'])} of {B}")
    print(json.dumps(dict(steps=args.steps, plants=B, ensemble=K, risk=args.risk, adapt=args.adapt, results=results,
                          gpu=gpu_info())))


if __name__ == "__main__":
    main()
