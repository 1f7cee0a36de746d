"""CPU tests of the ensemble risk measure (dial_plan_set_ensemble_risk): a NumPy fp32 restatement of the
host derivation and of the reduction's per-sample arithmetic, the shared device code (ens_risk_derive /
ens_risk_reduce of csrc/dial_device.cuh) built with g++ against it bit for bit, and the ``risk`` entries
of the ``--ensemble`` file and of ``--instance-overrides``.

Subnormal rewards are not covered: the library is built with -use_fast_math, which flushes them to zero
on the GPU, while the g++ build keeps them."""
import ctypes as C
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from dial_mpc_b200 import _capi
from tests.test_ensemble import member_mean

EMUL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emul")
MEAN, CVAR = _capi.DEFINES["DIAL_ENS_MEAN"], _capi.DEFINES["DIAL_ENS_CVAR"]
KMAX = _capi.DEFINES["DIAL_MAXENS"]
f32 = np.float32


# ---- the restatement -----------------------------------------------------------------------------------
def derive(K, mode, alpha):
    """(mode, n_tail, frac, denom) as dial_plan_set_ensemble_risk derives them; alpha crosses the C ABI
    as a float."""
    if mode == MEAN:
        return MEAN, K, f32(0), f32(K)
    t = float(f32(alpha)) * K
    if t <= 1 + 1e-6:
        return CVAR, 1, f32(0), f32(1)
    if abs(t - round(t)) <= 1e-6 * K:
        return CVAR, int(round(t)), f32(0), f32(round(t))
    n = math.floor(t)
    return CVAR, n, f32(t - n), f32(t)


def risk_reduce(r, mode, alpha):
    """r [K, n] fp32 member rewards -> [n] fp32 scores, the reduction kernel restated."""
    r = np.asarray(r, f32)
    K = r.shape[0]
    if mode == MEAN:
        return member_mean(r[None])[0]
    _, n_tail, frac, denom = derive(K, mode, alpha)
    s = np.take_along_axis(r, np.argsort(r, axis=0, kind="stable"), axis=0)   # ascending, ties in member order
    with np.errstate(invalid="ignore", over="ignore"):
        acc = s[0].copy()
        for j in range(1, n_tail):
            acc = acc + s[j]
        if frac > 0:
            acc = acc + frac * s[n_tail]           # fp32 multiply, then fp32 add
        out = (acc / denom).astype(f32)
    out[np.isnan(r).any(0)] = np.nan
    return out


def same_bits(a, b):
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


# ---- the g++ build of the device code ------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emul_risk") / "libdial_emul_risk.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I", EMUL, "-shared", "-fPIC", "-o", so,
                           os.path.join(EMUL, "emul_risk.cpp")])
    L = C.CDLL(so)
    L.emul_risk_derive.argtypes = [C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p]
    L.emul_risk_reduce.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]
    return L


def emul_derive(lib, K, mode, alpha):
    i, f = np.zeros(2, np.int32), np.zeros(2, f32)
    lib.emul_risk_derive(K, mode, alpha, i.ctypes.data, f.ctypes.data)
    return int(i[0]), int(i[1]), f[0], f[1]


def emul_reduce(lib, r, mode, alpha):
    r = np.ascontiguousarray(r, f32)
    out = np.empty(r.shape[1], f32)
    lib.emul_risk_reduce(r.ctypes.data, r.shape[0], r.shape[1], mode, alpha, out.ctypes.data)
    return out


def alphas(K):
    """alpha < 1/K, 1/K, alpha K just below and just above every integer (inside and outside the 1e-6 K
    snap), a few in between, and 1."""
    out = [1e-3, 0.5 / K, 1.0 / K, 1.0]
    for m in range(1, K + 1):
        for d in (-1e-7, 1e-7, -1e-3, 1e-3, 0.37):
            a = (m + d) / K
            if 0 < a <= 1:
                out.append(a)
    return out


def samples(K, n=96, seed=0):
    """[K, n]: Gaussian rewards, quantised columns with many ties, and columns with +-0, +-inf and a NaN."""
    g = np.random.default_rng(seed + K)
    r = g.normal(size=(K, n)).astype(f32)
    r[:, 16:40] = np.round(r[:, 16:40] * 2) / 2                        # ties
    r[:, 40:48] = np.where(g.random((K, 8)) < 0.5, f32(0.0), f32(-0.0))  # signed zeros
    r[:, 48:52] = r[:, 48:52] * 0                                     # zeros of either sign with the normals' signs
    r[g.integers(K), 52] = np.inf
    r[g.integers(K), 53] = -np.inf
    r[:2, 54] = [np.inf, -np.inf]
    r[:, 55] = np.inf
    r[g.integers(K), 56] = np.nan
    r[:, 57] = -np.inf
    return r


# ---- the restatement's own properties ------------------------------------------------------------------
@pytest.mark.parametrize("K", [2, 3, 4, 7, 16])
def test_restatement_special_cases(K):
    r = samples(K)
    fin = np.isfinite(r).all(0)
    worst = risk_reduce(r, CVAR, 1.0 / K)
    assert np.array_equal(worst[fin], r[:, fin].min(0))               # == (zeros of either sign compare equal)
    assert same_bits(risk_reduce(r, MEAN, 0.0), member_mean(r[None])[0])
    for m in range(1, K + 1):
        got = risk_reduce(r[:, fin], CVAR, m / K)
        s = np.sort(r[:, fin], axis=0, kind="stable")
        acc = s[0].copy()
        for j in range(1, m):
            acc = acc + s[j]
        assert np.array_equal(got, acc / f32(m)), m
    # CVaR with alpha = 1 is the mean up to rounding only
    np.testing.assert_allclose(risk_reduce(r[:, fin], CVAR, 1.0), r[:, fin].astype(np.float64).mean(0), rtol=1e-5, atol=1e-6)
    assert np.isnan(risk_reduce(r, CVAR, 0.5)[56]) and np.isnan(risk_reduce(r, MEAN, 0)[56])


def test_derivation_branches():
    assert derive(4, CVAR, 0.25) == (CVAR, 1, 0, 1)                   # worst
    assert derive(4, CVAR, 0.1) == (CVAR, 1, 0, 1)                    # alpha < 1/K: still the minimum
    assert derive(4, CVAR, 0.5) == (CVAR, 2, 0, 2)
    assert derive(4, CVAR, 0.5 + 1e-7)[1:3] == (2, 0)                 # snapped to the integer
    t = float(f32(0.6)) * 4                                          # alpha as the float the C ABI receives
    assert derive(4, CVAR, 0.6) == (CVAR, 2, f32(t - 2), f32(t))
    assert derive(16, CVAR, 1.0) == (CVAR, 16, 0, 16)
    assert derive(16, CVAR, 15.5 / 16)[1] == 15                       # the tail reaches the last element


# ---- the device code against the restatement -----------------------------------------------------------
@pytest.mark.parametrize("K", list(range(2, KMAX + 1)))
def test_device_code_equals_restatement(lib, K):
    r = samples(K)
    for mode, a in [(MEAN, 0.0)] + [(CVAR, a) for a in alphas(K)]:
        want = derive(K, mode, a)
        got = emul_derive(lib, K, mode, a)
        assert got[:2] == want[:2] and same_bits(got[2], want[2]) and same_bits(got[3], want[3]), (K, mode, a, got, want)
        assert same_bits(emul_reduce(lib, r, mode, a), risk_reduce(r, mode, a)), (K, mode, a)


def test_tail_at_the_last_element(lib):
    K = 16
    r = samples(K, seed=5)
    a = 15.5 / 16
    assert derive(K, CVAR, a)[1] == 15 and derive(K, CVAR, a)[2] > 0
    # the largest member carries weight frac: moving it changes the score
    got = emul_reduce(lib, r, CVAR, a)
    assert same_bits(got, risk_reduce(r, CVAR, a))
    r2 = r.copy()
    top = np.argmax(np.where(np.isnan(r2), -np.inf, r2), axis=0)
    r2[top[0], 0] += 1
    assert emul_reduce(lib, r2, CVAR, a)[0] != got[0]


def test_ties_keep_member_order(lib):
    # -0 before +0 (and the reverse) with the worst case: the first of the tied members is the score
    r = np.array([[-0.0, 0.0, 1.0], [0.0, -0.0, 1.0]], f32).T.copy()   # [K=3, n=2]
    got = emul_reduce(lib, r, CVAR, 1 / 3)
    assert same_bits(got, risk_reduce(r, CVAR, 1 / 3))
    assert np.signbit(got[0]) and not np.signbit(got[1])


# ---- risk specs and the CLI ----------------------------------------------------------------------------
def test_risk_setting():
    from dial_mpc_b200.core.dial_core import load_ensemble, load_setting, risk_setting
    from tests.test_ensemble import _go2
    assert risk_setting({"aggregate": "mean"}, 4) == (MEAN, 1.0)
    assert risk_setting({"aggregate": "worst"}, 4) == (CVAR, 0.25)
    assert risk_setting({"aggregate": "cvar", "alpha": 0.5}, 4) == (CVAR, 0.5)
    assert risk_setting({"aggregate": "cvar", "alpha": 1}, 4) == (CVAR, 1.0)
    assert derive(7, *risk_setting({"aggregate": "worst"}, 7))[1:] == (1, 0, 1)
    spec = {"members": [{}, {}], "risk": {"aggregate": "cvar", "alpha": 0.5}}
    members, plant = load_ensemble(spec, _go2())
    assert len(members) == 2 and plant is None
    assert load_setting(spec, "risk", 2) == {"aggregate": "cvar", "alpha": 0.5}
    assert load_setting({"members": [{}]}, "risk", 1) is None


BAD_RISK = [
    ({"aggregate": "median"}, r"aggregate must be one of mean, worst, cvar, got 'median'"),
    ({"aggregate": "cvar", "alpha": 0}, r"alpha must be a finite number in \(0, 1\], got 0"),
    ({"aggregate": "cvar", "alpha": -0.5}, r"alpha must be .* got -0.5"),
    ({"aggregate": "cvar", "alpha": 1.5}, r"alpha must be .* got 1.5"),
    ({"aggregate": "cvar", "alpha": float("nan")}, r"alpha must be .* got nan"),
    ({"aggregate": "cvar", "alpha": float("inf")}, r"alpha must be .* got inf"),
    ({"aggregate": "cvar"}, r"cvar needs alpha"),
    ({"aggregate": "worst", "alpha": 0.5}, r"alpha applies to aggregate cvar only"),
    ({"aggregate": "cvar", "alpha": 0.5, "beta": 1}, r"unknown key 'beta'"),
    ("worst", r"a risk spec maps 'aggregate'"),
]


@pytest.mark.parametrize("risk, match", BAD_RISK)
def test_risk_setting_names_the_bad_value(risk, match):
    from dial_mpc_b200.core.dial_core import risk_setting
    with pytest.raises(ValueError, match=match):
        risk_setting(risk, 4)


def _main(monkeypatch, capsys, argv):
    from dial_mpc_b200.core import dial_core
    monkeypatch.setattr(sys, "argv", ["dial_core", "--example", "unitree_go2_trot"] + argv)
    with pytest.raises(SystemExit) as e:
        dial_core.main()
    return e.value.code, capsys.readouterr().err


@pytest.mark.parametrize("risk, match", BAD_RISK[:6] + BAD_RISK[8:9])
def test_cli_ensemble_file_risk_errors(tmp_path, monkeypatch, capsys, risk, match):
    import yaml
    f = tmp_path / "ens.yaml"
    f.write_text(yaml.safe_dump({"members": [{}, {"body_mass": {"base": 9.0}}], "risk": risk}))
    code, err = _main(monkeypatch, capsys, ["--ensemble", str(f)])
    assert code == 2 and re.search(r"--ensemble .*ens\.yaml: risk: " + match, err), err


@pytest.mark.parametrize("risk, match", BAD_RISK[:6] + BAD_RISK[8:9])
def test_cli_instance_override_risk_errors(tmp_path, monkeypatch, capsys, risk, match):
    import yaml
    ens, ov = tmp_path / "ens.yaml", tmp_path / "ov.yaml"
    ens.write_text(yaml.safe_dump({"members": [{}, {"body_mass": {"base": 9.0}}]}))
    ov.write_text(yaml.safe_dump([{"risk": {"aggregate": "worst"}}, {"default_vx": 0.5, "risk": risk}]))
    code, err = _main(monkeypatch, capsys, ["--instances", "2", "--ensemble", str(ens), "--instance-overrides", str(ov)])
    assert code == 2 and re.search(r"--instance-overrides entry 1: risk: " + match, err), err


def test_cli_instance_override_risk_needs_ensemble(tmp_path, monkeypatch, capsys):
    import yaml
    ov = tmp_path / "ov.yaml"
    ov.write_text(yaml.safe_dump([{}, {"risk": {"aggregate": "worst"}}]))
    code, err = _main(monkeypatch, capsys, ["--instances", "2", "--instance-overrides", str(ov)])
    assert code == 2 and "--instance-overrides entry 1: risk needs --ensemble" in err, err
