"""Per-instance control latency on the CPU: the delay spec (delay_setting) and its errors, the CLI errors of
--delay and of the delay key of --instance-overrides, a NumPy restatement of the action queue against the
queue step the kernels run (delay_queue_step, on the warp emulator), and the prediction launches with
per-instance lengths against chains of single-row env steps."""
import ctypes as C
import re
import sys

import numpy as np
import pytest

from dial_mpc_b200 import _capi
from dial_mpc_b200.utils.spline import interp_matrix
from tests.conftest import make_pair
from tests.emul import emul
from tests.test_emul_batch import _instances

DMAX = _capi.DEFINES["DIAL_MAXDELAY"]


@pytest.mark.parametrize("spec, want", [(0, (0, False)), (3, (3, False)), (np.int64(16), (16, False)),
                                        ({"steps": 2}, (2, False)), ({"steps": 4, "predict": True}, (4, True)),
                                        ({"steps": 0, "predict": True}, (0, True))])
def test_delay_setting(spec, want):
    from dial_mpc_b200.core.dial_core import delay_setting
    assert delay_setting(spec) == want


@pytest.mark.parametrize("spec, match", [
    (-1, r"steps must be an int in 0\.\.16, got -1"),
    (17, r"steps must be an int in 0\.\.16, got 17"),
    (2.0, r"a delay spec is an int .* got 2\.0"),
    (True, r"a delay spec is an int"),
    ("3", r"a delay spec is an int"),
    ({"steps": 1.5}, r"steps must be an int in 0\.\.16, got 1\.5"),
    ({"predict": True}, r"needs steps"),
    ({"steps": 2, "predict": 1}, r"predict must be true or false, got 1"),
    ({"steps": 2, "lag": 1}, r"unknown key 'lag'"),
])
def test_delay_setting_names_the_bad_key_or_value(spec, match):
    from dial_mpc_b200.core.dial_core import delay_setting
    with pytest.raises(ValueError, match=match):
        delay_setting(spec)


def _main(monkeypatch, capsys, argv):
    from dial_mpc_b200.core import dial_core
    monkeypatch.setattr(sys, "argv", ["dial_core", "--example", "unitree_go2_trot"] + argv)
    with pytest.raises(SystemExit) as e:
        dial_core.main()
    return e.value.code, capsys.readouterr().err


@pytest.mark.parametrize("value, match", [
    ("x", r"--delay: STEPS must be an int, got 'x'"),
    ("17", r"--delay: steps must be an int in 0\.\.16, got 17"),
    ("-1", r"--delay: steps must be an int in 0\.\.16, got -1"),
    ("3:predicted", r"--delay: the suffix must be ':predict'"),
    ("3:", r"--delay: the suffix must be ':predict'"),
])
def test_cli_delay_errors(monkeypatch, capsys, value, match):
    code, err = _main(monkeypatch, capsys, ["--delay", value])
    assert code == 2 and re.search(match, err), err


def test_cli_delay_excludes_eager(monkeypatch, capsys):
    code, err = _main(monkeypatch, capsys, ["--delay", "2", "--eager"])
    assert code == 2 and "--delay runs on the CUDA-graph loop; it excludes --eager" in err, err


@pytest.mark.parametrize("entry, match", [
    ({"delay": 20}, r"delay: steps must be an int in 0\.\.16, got 20"),
    ({"delay": {"steps": 2, "predict": "yes"}}, r"delay: predict must be true or false"),
    ({"delay": {"step": 2}}, r"delay: unknown key 'step'"),
    ({"delay": [2]}, r"delay: a delay spec is an int"),
])
def test_cli_instance_override_delay_errors(tmp_path, monkeypatch, capsys, entry, match):
    import yaml
    ov = tmp_path / "ov.yaml"
    ov.write_text(yaml.safe_dump([{"delay": 1}, {}, entry]))
    code, err = _main(monkeypatch, capsys, ["--instances", "3", "--instance-overrides", str(ov)])
    assert code == 2 and re.search(r"--instance-overrides entry 2: " + match, err), err


# ---- warp emulator ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    lib = emul.build()
    assert lib.emul_sizeof(emul.SIZEOF["DelaySetting"]) == 8
    return lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def env_launch(env, desc, nrows, rows_per_inst, us, us_row, iter_lim, iter_, s, rews):
    """One env-step launch (mode 0, H = 1) as dial_mpc_step issues it, in place on the instance-major state s
    (qpos, qvel, warm, cnt): nrows rows, rows_per_inst per instance, action row r at us + r us_row; with
    iter_lim, the rows of an instance with iter_ >= iter_lim[b] do not run."""
    emul.launch(env, desc, mode=0, nrows=nrows, H=1, rows_per_inst=rows_per_inst, us=us, us_row=us_row,
                iter_lim=iter_lim, iter=iter_, qpos0=s["qpos"], qvel0=s["qvel"], warm0=s["warm"], counters_in=s["cnt"],
                qpos_out=s["qpos"], qvel_out=s["qvel"], warm_out=s["warm"], counters_out=s["cnt"], rewss=rews)


class Queue:
    """The queue of include/dial_b200.h restated: a list of d actions, front first."""

    def __init__(self, d, y0):
        self.q = [np.array(y0, np.float32) for _ in range(d)]

    def step(self, y0, pop):
        """Returns the applied action (pop) or None, and the pending rows [DMAX, nu]."""
        a = None
        if pop:
            self.q.append(np.array(y0, np.float32))
            a = self.q.pop(0)
        nu = len(y0)
        pend = np.zeros((DMAX, nu), np.float32)
        for j, x in enumerate(self.q):
            pend[j] = x
        return a, pend


class Ring:
    """The ring the kernels keep, stepped by delay_queue_step (emulator build)."""

    def __init__(self, lib, d, y0, nu):
        self.lib, self.d, self.nu = lib, d, nu
        self.ring = np.zeros((DMAX, nu), np.float32)
        self.ring[:d] = y0     # delay_refill_kernel: d copies of Y[b][0], front at slot 0
        self.head = 0

    def step(self, y0, pop, threads):
        y0 = np.ascontiguousarray(y0, np.float32)
        applied = np.full(self.nu, np.nan, np.float32)
        pend = np.full((DMAX, self.nu), np.nan, np.float32)
        h = self.lib.emul_delay_queue_step(_p(self.ring), self.head, self.d, self.nu, _p(y0), _p(applied), _p(pend),
                                           int(pop), threads)
        assert h >= 0
        self.head = h
        return (applied if pop else None), pend


@pytest.mark.parametrize("d", [0, 1, 2, 5, DMAX])
def test_queue_equals_restatement(lib, d):
    """Applied actions and pending rows over a run of env steps (and steps without one, which do not move the
    queue), bit for bit; the action pushed at step t is applied at step t + d."""
    nu = 12
    rng = np.random.default_rng(d)
    y0 = rng.uniform(-1, 1, nu).astype(np.float32)
    Q, R = Queue(d, y0), Ring(lib, d, y0, nu)
    pushed = []
    for t in range(3 * DMAX + 5):
        pop = t % 7 not in (3, 5)       # env_step 0 / 2 now and then
        y = rng.uniform(-1, 1, nu).astype(np.float32)
        qa, qp = Q.step(y, pop)
        ra, rp = R.step(y, pop, threads=1 + t % 4)
        assert np.array_equal(qp, rp), t
        if pop:
            assert np.array_equal(qa, ra), t
            pushed.append(y)
            if len(pushed) > d:
                assert np.array_equal(ra, pushed[-1 - d]), t
            else:
                assert np.array_equal(ra, y0), t      # the refill
        assert not np.isnan(rp).any()


def test_queue_change_of_delay_refills(lib):
    """A new delay refills the queue with d copies of the current Y[b][0], from which it moves on."""
    nu = 3
    rng = np.random.default_rng(1)
    y = lambda: rng.uniform(-1, 1, nu).astype(np.float32)
    cur = y()
    Q, R = Queue(4, cur), Ring(lib, 4, cur, nu)
    for t in range(6):
        cur = y()
        assert np.array_equal(Q.step(cur, True)[0], R.step(cur, True, 2)[0])
    for d in (2, 0, 7):
        Q, R = Queue(d, cur), Ring(lib, d, cur, nu)
        for t in range(d + 3):
            nxt = y()
            qa, qp = Q.step(nxt, True)
            ra, rp = R.step(nxt, True, 3)
            assert np.array_equal(qa, ra) and np.array_equal(qp, rp), (d, t)
            if t < d:
                assert np.array_equal(ra, cur), (d, t)     # the refill's copies come out first


def test_prediction_launches_equal_single_row_chains():
    """The prediction launches of one graph step: launch j rolls one row per instance with action pending[b][j],
    in place, and instance b runs only while j < its prediction length.  Three Go2 seq-jump instances with
    delays 0, 2 and 5 equal, bit for bit, chains of d single-instance env steps; the chains of the delayed
    instances cross the first stage boundary of the jump sequence (dt 0.02, jump_dt 1: the step from 49)."""
    env, o = make_pair("unitree_go2_seq_jump")
    B, Hn = 3, 3
    nu = env.action_size
    rng = np.random.default_rng(11)
    qpos, qvel, warm, _ = _instances(o, B, nu, Hn, rng)
    qpos, qvel, warm = (np.ascontiguousarray(a, np.float32) for a in (qpos, qvel, warm))
    counters = np.array([[49, 0], [48, 0], [46, 0]], np.int32)
    lens = np.array([0, 2, 5], np.int32)
    pending = np.zeros((B, DMAX, nu), np.float32)
    for b in range(B):
        pending[b, :lens[b]] = rng.uniform(-1, 1, (lens[b], nu))
    desc = env.plan_desc(Nsample=4, Hsample=6, Hnode=Hn, temp_sample=0.05,
                         M_n2u=interp_matrix(np.linspace(0, 1, Hn + 1), np.linspace(0, 1, 7)), n_inst=B)
    bat = dict(qpos=qpos.copy(), qvel=qvel.copy(), warm=warm.copy(), cnt=counters.copy())
    rew = np.zeros(B, np.float32)
    for j in range(int(lens.max())):
        env_launch(env, desc, B, 1, pending.reshape(-1)[j * nu:], DMAX * nu, lens, j, bat, rew)
    for b in range(B):
        one = dict(qpos=qpos[b:b + 1].copy(), qvel=qvel[b:b + 1].copy(), warm=warm[b:b + 1].copy(),
                   cnt=counters[b:b + 1].copy())
        r1 = np.zeros(1, np.float32)
        for j in range(lens[b]):
            act = np.ascontiguousarray(pending[b, j][None])
            env_launch(env, desc, 1, 0, act, 0, None, 0, one, r1)
        for k in ("qpos", "qvel", "warm", "cnt"):
            assert np.array_equal(bat[k][b], one[k][0]), (b, k)
        assert bat["cnt"][b, 0] == counters[b, 0] + lens[b]
    # the instance without a prediction is untouched; the delayed ones crossed into stage 1
    assert np.array_equal(bat["qpos"][0], qpos[0]) and tuple(bat["cnt"][0]) == (49, 0)
    assert bat["cnt"][1, 1] == 1 and bat["cnt"][2, 1] == 1
