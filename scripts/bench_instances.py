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
``dial_plan_set_instance_model``).  ``--ensemble K``: every instance plans against K member models
(dial_plan_desc.n_ens) spread as ``--distinct-models`` spreads the instances (member k: base mass
+3 kg * k / K, friction 1 - 0.5 k / K), bound through ``dial_plan_set_ensemble_model``, and scores each
sample by the ``--risk`` measure of its member rewards (mean, worst or cvar:ALPHA; default mean).
``--schedules``, ``--delays``, ``--observe``, ``--pushes`` and ``--plant`` each take one spec for every instance or
a list of one per instance (null: none), as YAML text or a YAML file.
``--delays SPEC_OR_FILE``: delay specs (``DeviceLoop(..., delay=...)``: an int or ``{steps: d, predict: true}``), so that the step also moves the action queues and, for predicting instances,
runs the prediction launches (use ``--env-step 1`` for the queues to move).
``--observe SPEC_OR_FILE``: each instance plans from an observation of its plant (``DeviceLoop(..., observe=...)``):
a YAML flow mapping applied to every instance (``'{delay: 2, qpos: 0.01, qvel: 0.1}'``) or a YAML file holding
one such mapping or a list of one per instance (null: none), so that the step also runs the observe launch and,
for instances predicting through ``--delays``, max(k + d) prediction launches (use ``--env-step 1`` for the
rings to move).
``--pushes FILE.yaml``: each instance's plant is pushed between env steps (``DeviceLoop(..., pushes=...)``): one
push spec for every instance or a list of one per instance (null: none), so that every step with an env step also
runs the push launch (use ``--env-step 1``; an entry firing in every step measures the cost of a push).
``--plant SPEC``: every instance's plant steps at its own fidelity (``DeviceLoop(..., plant=...)``): a YAML flow
mapping such as ``'{substeps: 4, iterations: 100, ls_iterations: 50, tolerance: 1e-8}'`` applied to every instance,
or a YAML file with one spec or a list of one per instance (null: none), so that a step with an env step runs one
plant launch per distinct substep count (use ``--env-step 1``).
``--terrain SPEC``: every instance's ground (``DeviceLoop(..., terrain=...)``): a YAML flow mapping such as
``'{kind: rough, amplitude: 0.03, wavelength: 0.3, seed: 1, planner: true}'`` applied to every instance, or a YAML
file with one spec or a list of one per instance (null: none); the launches that read a terrain run the terrain
build of the rollout kernel.
``--profile-kernels``: instead of the timing, run the steps without graph capture under torch.profiler and
print the mean device time per launch of the rollout, update, ensemble reduction, delay queue, observe and push
kernels."""
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


def risk_spec(tok: str) -> dict:
    """A --risk token (mean, worst or cvar:ALPHA) -> the risk spec of DeviceLoop(..., risk=...)."""
    agg, colon, a = tok.partition(":")
    if not colon:
        return {"aggregate": agg}
    try:
        return {"aggregate": agg, "alpha": float(a)}
    except ValueError:
        raise ValueError(f"alpha must be a number, got {a!r}") from None


def adapt_spec(tok: str) -> dict:
    """An --adapt token (SIGMA or SIGMA:FORGET) -> the adapt spec of DeviceLoop(..., adapt=...)."""
    s, colon, f = tok.partition(":")
    try:
        return dict({"sigma": float(s)}, **({"forget": float(f)} if colon else {}))
    except ValueError:
        raise ValueError(f"SIGMA[:FORGET] must be numbers, got {tok!r}") from None


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
    ap.add_argument("--ensemble", type=int, default=0, metavar="K",
                    help="plan every instance against K member models: K distinct base masses and foot frictions")
    ap.add_argument("--risk", default="mean", metavar="MEASURE",
                    help="with --ensemble: the risk measure of every instance, mean, worst or cvar:ALPHA")
    ap.add_argument("--adapt", default=None, metavar="SIGMA[:FORGET]",
                    help="with --ensemble K >= 2: every instance adapts its belief over the members to its plant")
    ap.add_argument("--env-step", type=int, default=2, choices=(1, 2),
                    help="the timed steps' env_step: 2 (shift + plan, the default) or 1 (env step + shift + plan; "
                         "--adapt runs its predictions and belief update in env steps only)")
    ap.add_argument("--schedules", default=None, metavar="FILE.yaml",
                    help="a schedule spec for every instance or a list of one per instance (null: the config's; "
                         "DeviceLoop(..., schedule=...)); each instance then runs its own Ndiffuse")
    ap.add_argument("--delays", default=None, metavar="FILE.yaml",
                    help="a delay spec for every instance or a list of one per instance (an int or "
                         "{steps: d, predict: true}; DeviceLoop(..., delay=...))")
    ap.add_argument("--observe", default=None, metavar="SPEC_OR_FILE",
                    help="an observe spec for every instance (a YAML flow mapping such as '{delay: 2, qpos: 0.01}') or "
                         "a YAML file with one spec or a list of one per instance (DeviceLoop(..., observe=...))")
    ap.add_argument("--pushes", default=None, metavar="FILE.yaml",
                    help="a YAML file with one push spec for every instance or a list of one per instance (null: none) "
                         "(DeviceLoop(..., pushes=...)); a push launch runs after every env step (--env-step 1), and "
                         "a spec such as [{step: 1, steps: 1000000000, body: base, force: [50, 0, 0]}] fires in every one")
    ap.add_argument("--plant", default=None, metavar="SPEC_OR_FILE",
                    help="a plant spec for every instance (a YAML flow mapping such as '{substeps: 4}') or a YAML file "
                         "with one spec or a list of one per instance (DeviceLoop(..., plant=...))")
    ap.add_argument("--terrain", default=None, metavar="SPEC_OR_FILE",
                    help="a terrain spec for every instance (a YAML flow mapping such as '{kind: slope, angle: 10, "
                         "planner: true}') or a YAML file with one spec or a list of one per instance "
                         "(DeviceLoop(..., terrain=...))")
    ap.add_argument("--profile-kernels", action="store_true",
                    help="print per-kernel device times (eager launches under torch.profiler) instead of the step time")
    args = ap.parse_args()
    if args.instances < 1 or args.steps < 1:
        ap.error("--instances and --steps must be at least 1")
    if args.risk != "mean" and not args.ensemble:
        ap.error("--risk needs --ensemble K")
    if args.adapt is not None and args.ensemble < 2:
        ap.error("--adapt needs --ensemble K with K >= 2")
    if args.profile_kernels:
        os.environ["DIAL_NO_GRAPH"] = "1"     # kernels of a replayed graph are not listed one by one
    import numpy as np
    import torch
    from baseline_configs import BASELINE, dial_config, product_env
    from dial_mpc_b200 import random as drandom
    from dial_mpc_b200.core.dial_core import MBDPI, DeviceLoop, resolve_settings

    B, b = args.instances, BASELINE[args.config]
    cfg = dial_config(args.config, world=1)
    env = product_env(b["env"])
    mb = MBDPI(cfg, env, n_instances=B, n_ensemble=args.ensemble)
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
    m = env.sys.model
    torso = int(env.plan_desc().torso_body)

    def spread(e, f):
        """e with base mass + 3 kg * f and every contact pair's friction scaled by 1 - 0.5 f."""
        e = copy.copy(e)
        e.sys = e.sys.tree_replace({"body_mass": {m.names["body"][torso]: m.arrays["body_mass"][torso] + 3.0 * f},
                                    "pair_friction": m.arrays["pair_friction"] * (1.0 - 0.5 * f)})
        return e
    if args.distinct_models:
        base = [env if envs is None else envs[i] for i in range(B)]
        envs = [spread(e, i / B) for i, e in enumerate(base)]
    members = [spread(env, k / args.ensemble).sys for k in range(args.ensemble)] if args.ensemble else None
    try:
        risk = risk_spec(args.risk) if args.ensemble else None
    except ValueError as e:
        ap.error(f"--risk {args.risk}: {e}")
    try:
        adapt = adapt_spec(args.adapt) if args.adapt is not None else None
    except ValueError as e:
        ap.error(f"--adapt {args.adapt}: {e}")
    import yaml
    # each per-instance setting is one spec for every instance or a list of B (DeviceLoop's rule), given as YAML text
    # or a YAML file
    given, settings = {}, {}
    for key, opt, text in (("schedule", "--schedules", args.schedules), ("delay", "--delays", args.delays),
                           ("observe", "--observe", args.observe), ("pushes", "--pushes", args.pushes),
                           ("plant", "--plant", args.plant), ("terrain", "--terrain", args.terrain)):
        if text is not None:
            try:
                given[key] = yaml.safe_load(open(text) if os.path.isfile(text) else text)
                settings.update(resolve_settings(B, args.ensemble, env, cfg, **{key: given[key]}))
            except (ValueError, yaml.YAMLError) as e:
                ap.error(f"{opt} {text}: {e}")
    setting = lambda key, none: [s for _, s in settings.get(key, [(None, none)] * B)]
    n_diffuse = [cfg.Ndiffuse if s is None else s.Ndiffuse for s in setting("schedule", None)]
    # a predicting instance's prediction runs through its observation delay and its control latency
    n_pred = max([d + (o[0] if o else 0) for (d, p), o in zip(setting("delay", (0, False)), setting("observe", None))
                  if p] or [0])
    # with plant settings the env step is one launch per distinct substep count
    n_plant = len({1 if f is None else f.substeps for f in setting("plant", None)})
    if B == 1:
        loop = DeviceLoop(mb, state, drandom.PRNGKey(cfg.seed), envs=envs, ensemble=members, risk=risk, adapt=adapt,
                          **given)
    else:
        loop = DeviceLoop(mb, [state] * B, np.stack([drandom.PRNGKey(cfg.seed + i) for i in range(B)]), envs=envs,
                          ensemble=members, risk=risk, adapt=adapt, **given)
    es = args.env_step
    # without --schedules every step runs the config's Ndiffuse on every instance, as before
    nd = None if "schedule" in given else cfg.Ndiffuse
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=mb.device)
    for _ in range(max(args.warmup, 3)):
        loop.step(nd, env_step=es)
    torch.cuda.synchronize()
    if args.profile_kernels:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                loop.step(nd, env_step=es)
            torch.cuda.synchronize()
        acc, rollouts = {}, []
        for ev in prof.events():
            if ev.device_type.name != "CUDA":
                continue
            if "rollout_kernel" in ev.name:
                rollouts.append((ev.time_range.start, ev.time_range.elapsed_us()))
            for key in ("update_kernel", "ensemble_reduce_kernel", "trajbar", "ens_gather_kernel", "ens_belief_kernel",
                        "delay_queue_kernel", "observe_kernel", "push_kernel"):
                if key in ev.name:
                    n, tot = acc.get(key, (0, 0.0))
                    acc[key] = (n + 1, tot + ev.time_range.elapsed_us())
        # the rollout launches of one step in order: [member prediction, env step (env_step 1)], [the delay
        # prediction steps], the planner's
        per_step = ["prediction"] * (es == 1 and adapt is not None) + ["env step"] * (es == 1) * n_plant + \
            ["delay prediction"] * n_pred + ["plan"] * max(n_diffuse)
        for i, (_, us) in enumerate(sorted(rollouts)):
            key = f"rollout_kernel ({per_step[i % len(per_step)]})"
            n, tot = acc.get(key, (0, 0.0))
            acc[key] = (n + 1, tot + us)
        print(json.dumps(dict(config=f"{b['name']} (BASELINE configs[{args.config}])", instances=B, ensemble=args.ensemble,
                              risk=args.risk, adapt=args.adapt, delays=args.delays, observe=args.observe, pushes=args.pushes, plant=args.plant, terrain=args.terrain, env_step=es, kernels_us_per_launch={k: tot / n for k, (n, tot) in acc.items()},
                              launches_per_step={k: n / args.steps for k, (n, tot) in acc.items()}, gpu=gpu_info())))
        return
    evs = []
    for _ in range(args.steps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        loop.step(nd, env_step=es)
        e1.record()
        evs.append((e0, e1))
    torch.cuda.synchronize()
    t = sum(a.elapsed_time(e) for a, e in evs) / 1e3 / args.steps
    rows = B * max(args.ensemble, 1) * (cfg.Nsample + 1)
    print(json.dumps(dict(config=f"{b['name']} (BASELINE configs[{args.config}])", instances=B, distinct_tasks=args.distinct_tasks,
                          distinct_models=args.distinct_models, ensemble=args.ensemble, risk=args.risk, adapt=args.adapt, env_step=es, rows_per_rollout=rows,
                          Nsample=cfg.Nsample, Hsample=cfg.Hsample, Ndiffuse=cfg.Ndiffuse, steps=args.steps,
                          schedules=args.schedules, delays=args.delays, observe=args.observe, pushes=args.pushes, plant=args.plant, terrain=args.terrain, Ndiffuse_per_instance=n_diffuse if "schedule" in given else None,
                          value=sum(n_diffuse) * cfg.Nsample * cfg.Hsample / t, unit="sample-steps/s",
                          ms_per_step=1e3 * t, gpu=gpu_info())))


if __name__ == "__main__":
    main()
