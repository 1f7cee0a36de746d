"""Throughput of B independent planner instances in one control-step graph (dial_plan_desc.n_inst).

    python scripts/bench_instances.py --config 0 --instances 16 --steps 20 --warmup 5

Times the same public call as bench.py's headline, ``DeviceLoop.step(Ndiffuse, env_step=2)``, on a
plan of B instances of a BASELINE config: the synthetic state of bench.py (reset + 10 zero-action
env steps) for every instance, instance b's planner rng PRNGKey(seed + b), a 256 MiB L2 flush between
steps outside the timed CUDA events.  Prints one JSON line: value = B * Ndiffuse * Nsample * Hsample
/ step time, ms per control step, and the card, power limit and SM clocks read in the same run.
``--instances 1`` is the single-instance plan (bench.py's timed step).  ``--distinct-tasks``: instance b
plans its own velocity command (vx spread over [-1, 1], a per-instance task bound through
``DeviceLoop(..., envs=...)``) instead of the config's shared one.  ``--distinct-models``: instance b
runs its own physical model (base mass +3 kg * b / B, foot friction 1 - 0.5 b / B where the model has
feet ``FR FL RR RL``, else every pair's friction scaled so; a per-instance model bound through
``dial_plan_set_instance_model``)."""
import argparse
import copy
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001  (reported in the line, never fatal)
        return f"nvidia-smi unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=0)
    ap.add_argument("--instances", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--distinct-tasks", action="store_true",
                    help="bind one task per instance: B distinct forward-velocity commands")
    ap.add_argument("--distinct-models", action="store_true",
                    help="bind one physical model per instance: B distinct base masses and foot frictions")
    args = ap.parse_args()
    if args.instances < 1 or args.steps < 1:
        ap.error("--instances and --steps must be at least 1")
    import numpy as np
    import torch
    from baseline_configs import BASELINE, dial_config, product_env
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import MBDPI, DeviceLoop

    B, b = args.instances, BASELINE[args.config]
    cfg = dial_config(args.config, world=1)
    env = product_env(b["env"])
    mb = MBDPI(cfg, env, n_instances=B)
    state = env.reset(drandom.PRNGKey(0))
    for _ in range(10):
        state = env.step(state, torch.zeros(mb.nu, device=mb.device))
    envs = None
    if args.distinct_tasks:
        from dataclasses import replace
        import dial_mpc_b200.envs as E
        if not hasattr(env._config, "default_vx"):
            ap.error(f"--distinct-tasks sweeps default_vx, which {type(env).__name__} has not")
        envs = [E.get_environment(b["env"], config=replace(env._config, default_vx=float(v)))
                for v in np.linspace(-1.0, 1.0, B)]
    if args.distinct_models:
        m = env.sys.model
        torso = int(env.plan_desc().torso_body)
        base = [env if envs is None else envs[i] for i in range(B)]
        envs = []
        for i, e in enumerate(base):
            e = copy.copy(e)
            e.sys = e.sys.tree_replace({"body_mass": {m.names["body"][torso]: m.arrays["body_mass"][torso] + 3.0 * i / B},
                                        "pair_friction": m.arrays["pair_friction"] * (1.0 - 0.5 * i / B)})
            envs.append(e)
    if B == 1:
        loop = DeviceLoop(mb, state, drandom.PRNGKey(cfg.seed), envs=envs)
    else:
        loop = DeviceLoop(mb, [state] * B, np.stack([drandom.PRNGKey(cfg.seed + i) for i in range(B)]), envs=envs)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=mb.device)
    for _ in range(max(args.warmup, 3)):
        loop.step(cfg.Ndiffuse, env_step=2)
    torch.cuda.synchronize()
    evs = []
    for _ in range(args.steps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        loop.step(cfg.Ndiffuse, env_step=2)
        e1.record()
        evs.append((e0, e1))
    torch.cuda.synchronize()
    t = sum(a.elapsed_time(e) for a, e in evs) / 1e3 / args.steps
    rows = B * (cfg.Nsample + 1)
    print(json.dumps(dict(config=f"{b['name']} (BASELINE configs[{args.config}])", instances=B, distinct_tasks=args.distinct_tasks,
                          distinct_models=args.distinct_models, rows_per_rollout=rows,
                          Nsample=cfg.Nsample, Hsample=cfg.Hsample, Ndiffuse=cfg.Ndiffuse, steps=args.steps,
                          value=B * cfg.Ndiffuse * cfg.Nsample * cfg.Hsample / t, unit="sample-steps/s",
                          ms_per_step=1e3 * t, gpu=gpu_info())))


if __name__ == "__main__":
    main()
