"""The per-instance settings on the CPU, pinned against tests/golden/instance_settings.json: the full text of every
error the spec parsers raise for the bad specs of the test_instance_* / test_ensemble* rejection tables, the full
error text and exit code of the command line for each flag and --instance-overrides key, and the keyword arguments
main() hands to DeviceLoop (one instance) or run_instances (batched) for a matrix of command lines, with MBDPI,
DeviceLoop, run_instances and the env's reset replaced by recorders (the specs compared as written, but a delay
spec as the (steps, predict) it sets).  Regenerate the golden file (only when a
change to these outputs is intended) with ``python -m tests.test_instance_settings``."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import yaml

from dial_mpc_b200 import _capi

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "instance_settings.json")


def _go2():
    import dial_mpc_b200.envs as E
    return E.get_environment("unitree_go2_walk", config=E.get_config("unitree_go2_walk")())


def _cases(module, func, argname):
    """The first argument of every case of ``module.func``'s parametrize table."""
    import importlib
    fn = getattr(importlib.import_module(f"tests.{module}"), func)
    (mark,) = [m for m in fn.pytestmark if m.name == "parametrize"]
    assert mark.args[0].split(",")[0].strip() == argname
    return [case[0] for case in mark.args[1]]


def parser_cases():
    """(parser name, bad spec) for every rejection table of the parsers, plus the missing-key cases."""
    out = [("risk", s) for s in _cases("test_ensemble_risk", "test_risk_setting_names_the_bad_value", "risk")]
    out += [("adapt", s) for s in _cases("test_ensemble_adapt", "test_adapt_setting_names_the_bad_value", "adapt")]
    out += [("prior", s) for s in _cases("test_ensemble_adapt", "test_prior_setting_names_the_bad_value", "w")]
    out += [("schedule", s) for s in _cases("test_instance_schedule", "test_schedule_setting_names_the_bad_key_or_value",
                                            "spec")]
    out += [("delay", s) for s in _cases("test_instance_delay", "test_delay_setting_names_the_bad_key_or_value", "spec")]
    out += [("observe", s) for s in _cases("test_instance_observation", "test_observe_setting_names_the_bad_key_or_value",
                                           "spec")]
    out += [("push", s) for s in _cases("test_instance_pushes", "test_push_setting_names_the_bad_entry", "spec")]
    out += [("plant", s) for s in _cases("test_instance_plant", "test_plant_setting_rejections", "spec")]
    # missing keys and the wrong container for each parser
    out += [("risk", {}), ("risk", {"alpha": 0.5}), ("risk", None), ("adapt", {}), ("adapt", None), ("prior", 3),
            ("prior", None), ("prior", [1, "x", 0]), ("prior", [1, True, 0]), ("schedule", None),
            ("delay", {}), ("delay", None), ("delay", {"steps": None}), ("observe", None), ("observe", {"seed": 2 ** 32}),
            ("push", 3), ("push", [{}]), ("push", [{"body": "base", "step": 1, "pos": "abc"}]), ("plant", 3),
            ("plant", {"sim_dt": "x"}), ("plant", {"ls_iterations": 0}), ("plant", {"tolerance": 1e39}),
            ("adapt", {"sigma": True}), ("adapt", {"sigma": 0.1, "forget": "x"}), ("risk", {"aggregate": "cvar",
                                                                                              "alpha": True})]
    return out


def parser_message(name, spec):
    from dial_mpc_b200.core import dial_core as D
    from tests.test_instance_schedule import BASE
    call = dict(risk=lambda: D.risk_setting(spec, 4), adapt=lambda: D.adapt_setting(spec, 4, 18),
                prior=lambda: D.prior_setting(spec, 3), schedule=lambda: D.schedule_setting(spec, BASE),
                delay=lambda: D.delay_setting(spec), observe=lambda: D.observe_setting(spec, _go2().sys),
                push=lambda: D.push_setting(spec, _go2().sys), plant=lambda: D.plant_setting(spec, _go2().sys))[name]
    try:
        call()
    except ValueError as e:
        return str(e)
    return None


# ---- the command line ----------------------------------------------------------------------------------------
ENSEMBLE = {"members": [{}, {"body_mass": {"base": 8.0}}], "plant": {"body_mass": {"base": 7.0}},
            "risk": {"aggregate": "cvar", "alpha": 0.5}, "adapt": {"sigma": 0.2}, "prior": [3, 1]}
ENSEMBLE_NO_PLANT = {"members": [{}, {"dof_damping": {"FR_hip_joint": 1.0}}]}
OV_ALL = [{"delay": 2, "observe": {"delay": 1, "qpos": 0.01}, "push": [{"step": 3, "body": "base", "force": [1, 0, 0]}],
           "plant": {"substeps": 2}, "default_vx": 0.3, "temp_sample": 0.1, "Ndiffuse": 3},
          {},
          {"delay": {"steps": 3, "predict": True}, "sys": {"body_mass": {"base": 6.0}}, "plant": {"iterations": 3}}]
OV_ENS = [{"risk": {"aggregate": "worst"}, "adapt": {"sigma": 0.1, "forget": 0.9}}, None,
          {"adapt": {"sigma": 0.3}, "observe": {"qvel": 0.1}}]
OV_PLAIN = [{"default_vx": 0.2}, {"default_vx": 0.4}, {"sys": {"body_mass": {"base": 6.5}}}]
TOP = ["--delay", "1:predict", "--observe", "{delay: 2, qvel: 0.05, seed: 3}",
       "--push", "[{step: 5, steps: 2, body: base, torque: [0, 0, 1]}]", "--plant", "{sim_dt: 0.01}"]

# (argv, files): "@name" in argv is the path of files[name] written as YAML
KWARGS_MATRIX = [
    ([], {}),
    (["--delay", "2"], {}),
    (["--delay", "3:predict"], {}),
    (["--delay", "0"], {}),
    (["--observe", "{delay: 1, qpos: 0.01}"], {}),
    (["--observe", "{}"], {}),
    (["--push", "[{step: 3, body: base, force: [1, 0, 0]}]"], {}),
    (["--push", "[]"], {}),
    (["--plant", "{substeps: 2}"], {}),
    (["--plant", "{}"], {}),
    (TOP, {}),
    (["--ensemble", "@ens"], {"ens": ENSEMBLE}),
    (["--ensemble", "@ens"], {"ens": ENSEMBLE_NO_PLANT}),
    (["--ensemble", "@ens"] + TOP, {"ens": ENSEMBLE}),
    (["--instances", "3"], {}),
    (["--instances", "3", "--delay", "2"], {}),
    (["--instances", "3", "--observe", "{qpos: 0.02}"], {}),
    (["--instances", "3", "--push", "[{step: 2, body: base}]"], {}),
    (["--instances", "3", "--plant", "{substeps: 3}"], {}),
    (["--instances", "3"] + TOP, {}),
    (["--instances", "3", "--ensemble", "@ens"], {"ens": ENSEMBLE}),
    (["--instances", "3", "--ensemble", "@ens"] + TOP, {"ens": ENSEMBLE}),
    (["--instances", "3", "--ensemble", "@ens"], {"ens": ENSEMBLE_NO_PLANT}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": OV_PLAIN}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": OV_ALL}),
    (["--instances", "3", "--instance-overrides", "@ov"] + TOP, {"ov": OV_ALL}),
    (["--instances", "3", "--instance-overrides", "@ov"] + TOP, {"ov": OV_PLAIN}),
    (["--instances", "3", "--instance-overrides", "@ov", "--ensemble", "@ens"], {"ov": OV_ENS, "ens": ENSEMBLE}),
    (["--instances", "3", "--instance-overrides", "@ov", "--ensemble", "@ens"] + TOP,
     {"ov": OV_ALL, "ens": ENSEMBLE}),
    (["--instances", "3", "--instance-overrides", "@ov", "--ensemble", "@ens", "--delay", "4"],
     {"ov": OV_ENS, "ens": ENSEMBLE_NO_PLANT}),
]

# (argv, files) whose run ends in a parser.error (or a usage error)
CLI_ERRORS = [
    (["--delay", "x"], {}), (["--delay", "17"], {}), (["--delay", "-1"], {}), (["--delay", "3:predicted"], {}),
    (["--delay", "3:"], {}), (["--delay", " 2"], {}), (["--delay", "2", "--eager"], {}),
    (["--observe", "{delay: 20}"], {}), (["--observe", "[1, 2]"], {}), (["--observe", "{delay: 1"], {}),
    (["--observe", "{qvel: {foot: 1}}"], {}), (["--observe", "{delay: 1}", "--eager"], {}),
    (["--push", "{step: 1}"], {}), (["--push", "[{step: 3, body: base, force: [1, 2, x]}]"], {}),
    (["--push", "[{step: 1"], {}), (["--push", "[{step: 3, body: base}]", "--eager"], {}),
    (["--plant", "{substeps: 0}"], {}), (["--plant", "{sim_dt: 0.003}"], {}), (["--plant", "[4]"], {}),
    (["--plant", "{a: ["], {}), (["--plant", "{substeps: 4}", "--eager"], {}),
    (["--ensemble", "@ens", "--eager"], {"ens": ENSEMBLE}),
    (["--ensemble", "@ens"], {"ens": dict(ENSEMBLE, risk={"aggregate": "median"})}),
    (["--ensemble", "@ens"], {"ens": dict(ENSEMBLE, adapt={"sigma": 0})}),
    (["--ensemble", "@ens"], {"ens": dict(ENSEMBLE, prior=[1])}),
    (["--ensemble", "@ens"], {"ens": {"members": [{}], "adapt": {"sigma": 0.1}}}),
    (["--instances", "2", "--eager"], {}), (["--instances", "0"], {}),
    (["--instances", "1", "--instance-overrides", "@ov"], {"ov": [{}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}, {"colour": 1}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}, 3]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}, {"sys": 3}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}, {"sys": {"nq": 3}}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}, {"Nsample": 8}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}, {"Ndiffuse": 0}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{"delay": 1}, {}, {"delay": 20}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}, {"delay": {"step": 2}}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}, {"delay": [2]}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}, {"observe": {"delay": 30}}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}, {"observe": 2}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}, {"push": [{"step": 0, "body": "base"}]}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}, {"push": {"step": 1}}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}, {"plant": {"iterations": 500}}]}),
    (["--instances", "3", "--instance-overrides", "@ov"], {"ov": [{}, {}, {"plant": [2]}]}),
    (["--instances", "2", "--instance-overrides", "@ov"], {"ov": [{}, {"risk": {"aggregate": "worst"}}]}),
    (["--instances", "2", "--instance-overrides", "@ov"], {"ov": [{"adapt": {"sigma": 0.1}}, {}]}),
    (["--instances", "2", "--instance-overrides", "@ov", "--ensemble", "@ens"],
     {"ov": [{}, {"risk": {"aggregate": "cvar"}}], "ens": ENSEMBLE}),
    (["--instances", "2", "--instance-overrides", "@ov", "--ensemble", "@ens"],
     {"ov": [{}, {"adapt": {"sigma": [1, 2]}}], "ens": ENSEMBLE}),
    (["--instances", "2", "--instance-overrides", "@ov", "--ensemble", "@ens"],
     {"ov": [{}, {"adapt": {"sigma": 1}}], "ens": {"members": [{}]}}),
]

# (argv, files) run on the go2 trot example with randomize_tasks on
RAND_ERRORS = [
    (["--observe", "{delay: 2}"], {}),
    (["--instances", "2", "--instance-overrides", "@ov"], {"ov": [{}, {"observe": {"delay": 1}}]}),
]
RAND_OK = [
    (["--observe", "{qpos: 0.01}"], {}),
    (["--instances", "2", "--instance-overrides", "@ov"], {"ov": [{}, {"observe": {"delay": 0, "qvel": 0.1}}]}),
]


class _Stop(Exception):
    pass


def _digest(b):
    return hashlib.sha256(bytes(b)).hexdigest()[:16]


def _env_record(e):
    return [type(e).__name__, _digest(e.plan_desc()), _digest(_capi.fill_model_desc(e.sys.model))]


def _jsonable(v):
    if isinstance(v, dict):
        return {str(k): _jsonable(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return [_jsonable(x) for x in v]
    if isinstance(v, (np.integer, np.floating)):
        return ["np", type(v).__name__, v.item()]
    if v is None or isinstance(v, (bool, int, float, str)):
        return v
    if hasattr(v, "plan_desc"):
        return ["env"] + _env_record(v)
    m = getattr(v, "model", v)
    if hasattr(m, "arrays"):
        return ["model", _digest(_capi.fill_model_desc(m))]
    return ["repr", repr(v)]


def _argv(tmp_path, argv, files, config=None):
    paths = {}
    for name, content in files.items():
        p = tmp_path / f"{name}.yaml"
        p.write_text(yaml.safe_dump(content))
        paths[name] = str(p)
    head = ["dial_core", "--config", config] if config else ["dial_core", "--example", "unitree_go2_trot"]
    return head + [paths[a[1:]] if a.startswith("@") else a for a in argv]


def _rand_config(tmp_path):
    from dial_mpc_b200.utils.io_utils import get_example_path
    cfg = yaml.safe_load(open(get_example_path("unitree_go2_trot.yaml")))
    cfg["randomize_tasks"] = True
    path = tmp_path / "rand.yaml"
    path.write_text(yaml.safe_dump(cfg))
    return str(path)


def run_main(tmp_path, monkeypatch, capsys, argv, files, config=None):
    """main() on the command line with recorders: ("error", exit code, last stderr line) or ("call", what main()
    hands to DeviceLoop / run_instances)."""
    from dial_mpc_b200.core import dial_core as D
    got = {}
    get_env = D.dial_envs.get_environment

    def get_environment(*a, **k):
        env = get_env(*a, **k)
        env.reset = lambda rng: ("state", _env_record(env))
        return env

    class FakeMBDPI:
        def __init__(self, args, env, **kw):
            got["MBDPI"] = _jsonable(kw)
            self.nu, self.device, self.world_size = env.action_size, "cpu", 1

    class RecordingLoop(D.DeviceLoop):
        def __init__(self, mbdpi, state, rng, Y0=None, **kw):
            got["DeviceLoop"] = dict(state=_jsonable(state), kwargs=_jsonable(delay_as_set(kw)))
            raise _Stop

    def delay_as_set(kw):
        """The delay keyword as the (steps, predict) each instance is set to: (0, False) for a missing one."""
        d = kw.get("delay")
        if d is not None:
            one = lambda s: (0, False) if s is None else D.delay_setting(s)
            kw["delay"] = [one(s) for s in d] if isinstance(d, list) else one(d)
        return kw

    def run_instances(dial_config, env, B, Nstep, **kw):
        got["run_instances"] = dict(env=_env_record(env), B=B, Nstep=Nstep, kwargs=_jsonable(delay_as_set(kw)))
        raise _Stop

    monkeypatch.setattr(D.dial_envs, "get_environment", get_environment)
    monkeypatch.setattr(D, "MBDPI", FakeMBDPI)
    monkeypatch.setattr(D, "DeviceLoop", RecordingLoop)
    monkeypatch.setattr(D, "run_instances", run_instances)
    monkeypatch.setattr(sys, "argv", _argv(tmp_path, argv, files, config))
    try:
        D.main()
    except SystemExit as e:
        err = capsys.readouterr().err.replace(str(tmp_path), "<tmp>")
        return ["error", e.code, err[err.find(": error: ") + 2:].rstrip()]
    except _Stop:
        capsys.readouterr()
        return ["call", got]
    raise AssertionError("main() returned without an error or a run")


def _key(argv, files):
    return json.dumps([argv, files], sort_keys=True)


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


# ---- the tests --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("i", range(len(parser_cases())))
def test_parser_message(i):
    name, spec = parser_cases()[i]
    want = _golden()["parsers"][f"{name} {spec!r}"]
    assert parser_message(name, spec) == want


@pytest.mark.parametrize("argv, files", CLI_ERRORS + KWARGS_MATRIX)
def test_command_line(tmp_path, monkeypatch, capsys, argv, files):
    assert run_main(tmp_path, monkeypatch, capsys, argv, files) == _golden()["cli"][_key(argv, files)]


@pytest.mark.parametrize("argv, files", RAND_ERRORS + RAND_OK)
def test_command_line_randomize_tasks(tmp_path, monkeypatch, capsys, argv, files):
    got = run_main(tmp_path, monkeypatch, capsys, argv, files, config=_rand_config(tmp_path))
    assert got == _golden()["rand"][_key(argv, files)]


# ---- resolve_settings: DeviceLoop's checks, without a plan ---------------------------------------------------------
def _resolve(B=3, K=0, world_size=1, rand=False, **kw):
    from dial_mpc_b200.core.dial_core import resolve_settings
    from tests.test_instance_schedule import BASE
    return resolve_settings(B, K, _go2(), BASE, world_size, rand, **kw)


def test_resolve_one_spec_or_b():
    assert _resolve(delay=2) == {"delay": [(2, (2, False))] * 3}
    got = _resolve(delay=[0, None, {"steps": 2, "predict": True}], plant=[{"substeps": 2}, None, {}])
    assert [s for _, s in got["delay"]] == [(0, False), (0, False), (2, True)]
    assert [None if f is None else f.substeps for _, f in got["plant"]] == [2, None, 1]
    one = [{"step": 1, "body": "base"}]
    assert [len(t) for _, t in _resolve(pushes=one)["pushes"]] == [1, 1, 1]
    assert [len(t) for _, t in _resolve(pushes=[one, None, []])["pushes"]] == [1, 0, 0]
    assert [k for k, _, _, _ in (s for _, s in _resolve(observe={"delay": 4})["observe"])] == [4, 4, 4]
    assert _resolve(B=2, K=2, prior=[[1, 0], [0, 1]])["prior"][1][1].tolist() == [0.0, 1.0]
    assert _resolve(B=2, K=2, prior=np.array([1.0, 3.0]))["prior"][0][1].tolist() == [1.0, 3.0]
    env = _go2()
    assert _resolve(B=2, envs=[env, env])["envs"] == [(env, None), (env, None)]


def test_resolve_identity_settings():
    from dial_mpc_b200.core.dial_core import SETTINGS
    identity = {s.key: s.identity for s in SETTINGS}
    got = _resolve(B=1, delay=0, observe={"seed": 3}, pushes=[], plant=None, adapt=None)
    assert set(got) == {"delay", "observe", "pushes"}
    assert all(identity[k](v[0][1]) for k, v in got.items())
    assert not identity["delay"](_resolve(B=1, delay={"steps": 0, "predict": True})["delay"][0][1])
    assert not identity["observe"](_resolve(B=1, observe={"qvel": 0.1})["observe"][0][1])
    assert not identity["plant"](_resolve(B=1, plant={})["plant"][0][1])


@pytest.mark.parametrize("kw, msg", [
    (dict(B=3, delay=[1, 2]), "delay must be one delay spec or a list of 3, got a list of 2"),
    (dict(B=2, observe=[{}, {}, {}]), "observe must be one observe spec or a list of 2, got a list of 3"),
    (dict(B=2, pushes=[[], [], None]), "pushes must be one push spec or a list of 2, got a list of 3"),
    (dict(B=2, plant=[{}, None, {}]), "plant must be one plant spec or a list of 2, got a list of 3"),
    (dict(B=2, schedule=[{}]), "schedule must be one schedule spec or a list of 2, got a list of 1"),
    (dict(B=2, K=1, risk=[{"aggregate": "mean"}] * 3), "risk must be one risk spec or a list of 2, got a list of 3"),
    (dict(B=2, K=2, adapt=[None]), "adapt must be one adapt spec or a list of 2, got a list of 1"),
    (dict(B=2, K=2, prior=[[1, 1]] * 3), "prior must be K weights or a list of 2 such lists, got a list of 3"),
    (dict(B=2, K=2, ensemble=[[1, 2]] * 3), "ensemble must be a list of 2 models or 2 such lists, got a list of 3"),
    (dict(B=2, K=2, ensemble=[[1, 2], [1]]), "ensemble must be a list of 2 models or 2 such lists, got [2, 1]"),
    (dict(B=2, envs=[None]), "a plan of 2 instances needs 2 envs, got 1"),
    (dict(K=0, risk={"aggregate": "mean"}), "risk= needs an MBDPI built with n_ensemble >= 1"),
    (dict(K=0, ensemble=[1]), "ensemble= needs an MBDPI built with n_ensemble >= 1"),
    (dict(K=1, adapt={"sigma": 1}), "adapt= needs an MBDPI built with n_ensemble >= 2"),
    (dict(K=1, prior=[1]), "prior= needs an MBDPI built with n_ensemble >= 2"),
    (dict(world_size=2, delay=1), "delay= needs an unsharded plan (world_size 1)"),
    (dict(world_size=2, observe={}), "observe= needs an unsharded plan (world_size 1)"),
    (dict(world_size=2, pushes=[]), "pushes= needs an unsharded plan (world_size 1)"),
    (dict(world_size=2, plant={}), "plant= needs an unsharded plan (world_size 1)"),
    (dict(rand=True, observe=[None, {"qpos": 0.1}, {"delay": 1}]),
     "an observation delay needs a loop without randomize_tasks: its rollouts would start before the current command "
     "window (noise alone is allowed)"),
    (dict(B=2, delay=[1, 17]), "steps must be an int in 0..16, got 17"),
    (dict(B=2, pushes=[[], [{"step": 1}]]), "push 0: needs body, the name of the body pushed"),
])
def test_resolve_rejections(kw, msg):
    with pytest.raises(ValueError) as e:
        _resolve(**kw)
    assert str(e.value) == msg


def test_numpy_scalars_are_numbers():
    """Every numeric field takes NumPy int and float scalars as it takes Python numbers; bools stay rejected."""
    from dial_mpc_b200.core import dial_core as D
    from tests.test_instance_schedule import BASE
    f32, f64, i64 = np.float32, np.float64, np.int64
    assert D.risk_setting({"aggregate": "cvar", "alpha": f32(0.5)}, 4)[1] == 0.5
    forget, prune, sigma = D.adapt_setting({"sigma": f32(0.25), "forget": f32(0.5), "prune": i64(0)}, 4, 18)
    assert (forget, prune, sigma[0]) == (0.5, 0.0, f32(0.25))
    assert D.adapt_setting({"sigma": [f32(0.5)] * 18}, 4, 18)[2][17] == f32(0.5)
    cfg = D.schedule_setting({"temp_sample": f32(0.25), "sigma_scale": i64(1), "traj_diffuse_factor": f64(0.5),
                              "Ndiffuse": i64(3)}, BASE)
    assert (cfg.temp_sample, cfg.sigma_scale, cfg.Ndiffuse) == (0.25, 1, 3) and type(cfg.Ndiffuse) is int
    assert D.prior_setting([i64(1), f32(2), 0.5], 3).tolist() == [1.0, 2.0, 0.5]
    assert D.observe_setting({"delay": i64(2), "qpos": f32(0.5), "seed": i64(1)}, _go2())[0] == 2
    assert D.plant_setting({"substeps": i64(2), "tolerance": f32(0.5)}, _go2()).substeps == 2
    assert D.delay_setting({"steps": i64(2), "predict": np.bool_(True)}) == (2, True)
    for call in (lambda: D.risk_setting({"aggregate": "cvar", "alpha": np.bool_(True)}, 4),
                 lambda: D.adapt_setting({"sigma": np.bool_(True)}, 4, 18),
                 lambda: D.schedule_setting({"temp_sample": np.bool_(True)}, BASE),
                 lambda: D.schedule_setting({"Ndiffuse": True}, BASE),
                 lambda: D.prior_setting([np.bool_(True), 1, 1], 3),
                 lambda: D.plant_setting({"tolerance": np.bool_(False)}, _go2())):
        with pytest.raises(ValueError):
            call()


def _regenerate():
    import tempfile

    class MP:
        def __init__(self):
            self.undo = []

        def setattr(self, obj, name, value):
            self.undo.append((obj, name, getattr(obj, name)))
            setattr(obj, name, value)

        def restore(self):
            for obj, name, value in reversed(self.undo):
                setattr(obj, name, value)
            self.undo = []

    class Cap:
        def readouterr(self):
            sys.stderr.flush()
            out = _Err.buf.getvalue()
            _Err.buf.seek(0)
            _Err.buf.truncate()
            return type("R", (), {"err": out})()

    import io
    import pathlib

    class _Err:
        buf = io.StringIO()

    out = {"parsers": {f"{n} {s!r}": parser_message(n, s) for n, s in parser_cases()}, "cli": {}, "rand": {}}
    real_err = sys.stderr
    with tempfile.TemporaryDirectory() as d:
        tmp = pathlib.Path(d)
        for table, cases, rand in (("cli", CLI_ERRORS + KWARGS_MATRIX, False), ("rand", RAND_ERRORS + RAND_OK, True)):
            for argv, files in cases:
                mp = MP()
                sys.stderr = _Err.buf
                try:
                    out[table][_key(argv, files)] = run_main(tmp, mp, Cap(), argv, files,
                                                             config=_rand_config(tmp) if rand else None)
                finally:
                    sys.stderr = real_err
                    mp.restore()
    with open(GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    _regenerate()
