"""CPU tests of adapting an ensemble plan to its plant (dial_plan_set_ensemble_adapt): a NumPy fp32
restatement of the belief-weighted risk measures and a fp64 restatement of the belief update, against the
shared device code (ens_risk_reduce_weighted / ens_member_loglik / ens_belief_update of
csrc/dial_device.cuh) built with g++ bit for bit; the member-prediction launch's row mapping on the warp
emulator; and the ``adapt`` / ``prior`` entries of the ``--ensemble`` file and of ``--instance-overrides``.

Subnormal weights and rewards are not covered: the library is built with -use_fast_math, which flushes
them to zero on the GPU, while the g++ build keeps them.  The restatement of the update uses Python's
``math.exp`` / ``math.log``, the C library's, as the g++ build does; the GPU's fp64 exp and log may
differ from them in the last bit (tests/test_gpu_ensemble_adapt.py states its tolerance)."""
import math
import re
import sys

import numpy as np
import pytest

from dial_mpc_b200 import _capi
from tests.emul import emul
from tests.test_ensemble import FEET, _go2
from tests.test_ensemble_risk import CVAR, KMAX, MEAN, alphas, derive, same_bits, samples

CAP = 1.0e4
f32 = np.float32


# ---- the restatement -----------------------------------------------------------------------------------
def kept_members(w, prune):
    """Member k counts when w_k > 0 and w_k >= prune, or when w_k is the largest weight."""
    w = np.asarray(w, f32)
    wmax = w.max()
    return [bool(x > 0 and (x >= f32(prune) or x == wmax)) for x in w]


def weighted_reduce(r, mode, alpha, w, prune):
    """r [K, n] fp32 member rewards under the belief w [K] -> [n] fp32 scores, the weighted branches of the
    reduction kernel restated."""
    r, w = np.asarray(r, f32), np.asarray(w, f32)
    K, n = r.shape
    kept = kept_members(w, prune)
    W = f32(-0.0)
    for k in range(K):
        if kept[k]:
            W = f32(W + w[k])
    nan = np.zeros(n, bool)
    for k in range(K):
        if kept[k]:
            nan |= np.isnan(r[k])
    with np.errstate(invalid="ignore", over="ignore"):
        if mode == MEAN:
            acc = np.full(n, -0.0, f32)
            for k in range(K):
                if kept[k]:
                    acc = acc + w[k] * r[k]
            out = (acc / W).astype(f32)
        elif float(f32(alpha)) * K <= 1 + 1e-6:                # the worst case
            out = np.full(n, np.inf, f32)
            for k in range(K):
                if kept[k]:
                    out = np.where(r[k] < out, r[k], out)
        else:
            s = np.where(np.array(kept)[:, None], r, f32(np.inf)).astype(f32)
            v = np.where(kept, w, f32(0)).astype(f32)
            order = np.argsort(s, axis=0, kind="stable")      # ascending, ties in member order
            S, V = np.take_along_axis(s, order, axis=0), v[order]
            tau = f32(f32(alpha) * W)
            acc, m = np.full(n, -0.0, f32), np.zeros(n, f32)
            for j in range(K):
                act = (V[j] > 0) & (m < tau)
                t = np.minimum(V[j], tau - m)
                acc = np.where(act, acc + t * S[j], acc)
                m = np.where(act, m + t, m)
            out = (acc / m).astype(f32)
    out[nan] = np.nan
    return out


def member_loglik(vhat, v, sigma):
    """l of one member: -min(e / 2, C), e summed over the dofs in fp64 from the fp32 values; NaN -> -C."""
    e = 0.0
    for a, b, s in zip(np.asarray(vhat, f32), np.asarray(v, f32), np.asarray(sigma, f32)):
        d = (float(a) - float(b)) / float(s)
        e = e + d * d
    h = e * 0.5
    return -h if h <= CAP else -CAP


def belief_update(L, ell, forget):
    """(L, w) after one update of the log-belief L [K] (fp64) with the log-likelihoods ell [K]."""
    L = [float(f32(forget)) * x + l for x, l in zip(L, ell)]
    M = -math.inf
    for x in L:
        M = x if x > M else M
    s = 0.0
    for x in L:
        s = s + math.exp(x - M)
    lse = M + math.log(s)
    L = [x - lse for x in L]
    return L, np.array([math.exp(x) for x in L], f32)


# ---- the g++ build of the device code ------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    return emul.build()


def emul_reduce(lib, r, mode, alpha, w, prune):
    r, w = np.ascontiguousarray(r, f32), np.ascontiguousarray(w, f32)
    out = np.empty(r.shape[1], f32)
    lib.emul_adapt_reduce(r.ctypes.data, r.shape[0], r.shape[1], mode, alpha, w.ctypes.data, prune, out.ctypes.data)
    return out


def emul_update(lib, vhat, v, sigma, forget, L):
    vhat, v, sigma = (np.ascontiguousarray(a, f32) for a in (vhat, v, sigma))
    K, nv = vhat.shape
    L = np.array(L, np.float64)
    w, ell = np.empty(K, f32), np.empty(K, np.float64)
    lib.emul_adapt_update(vhat.ctypes.data, v.ctypes.data, sigma.ctypes.data, K, nv, forget, L.ctypes.data,
                          w.ctypes.data, ell.ctypes.data)
    return L, w, ell


def beliefs(K, seed=0):
    """(name, w [K], prunes): uniform, one-hot, some zero weights, a member exactly at the prune threshold,
    and a random belief."""
    g = np.random.default_rng(100 + K)
    uni = np.full(K, f32(math.exp(math.log(1.0 / K))), f32)
    hot = np.zeros(K, f32)
    hot[1] = 1
    zero = g.dirichlet(np.ones(K)).astype(f32)
    zero[g.permutation(K)[:K // 2]] = 0
    zero[np.argmax(zero)] += f32(0.5)                # a clear argmax
    rnd = g.dirichlet(np.ones(K) * 0.7).astype(f32)
    at = g.dirichlet(np.ones(K)).astype(f32)
    small = np.sort(at)[K // 3]                      # not the largest, so it is pruned on its own merits
    if small >= 1.0 / K:
        small = f32(0.4 / K)
        at[np.argsort(at)[K // 3]] = small
    prunes = (0.0, f32(0.5 / K), f32(0.999 / K))
    return [("uniform", uni, prunes), ("one-hot", hot, prunes), ("zeros", zero, prunes), ("random", rnd, prunes),
            ("at-threshold", at, (float(small),))]


def rewards(K, w, prune, n=96, seed=0):
    """samples(K) with NaN, +inf and -inf in a kept member and in a left-out one (when there is one)."""
    r = samples(K, n, seed)
    kept = kept_members(w, prune)
    ik = kept.index(True)
    r[ik, 60], r[ik, 61], r[ik, 62] = np.nan, np.inf, -np.inf
    if False in kept:
        io = kept.index(False)
        r[io, 63], r[io, 64], r[io, 65] = np.nan, np.inf, -np.inf
        r[io, 66] = -1e30                           # the lowest reward, left out
    return r


# ---- the restatement's own properties ------------------------------------------------------------------
@pytest.mark.parametrize("K", [2, 3, 4, 7, 16])
def test_weighted_restatement_special_cases(K):
    uni = np.full(K, f32(1.0 / K), f32)
    r = samples(K)
    fin = np.isfinite(r).all(0)
    # uniform weights: the unweighted measures up to rounding; the worst case exactly
    from tests.test_ensemble_risk import risk_reduce
    np.testing.assert_allclose(weighted_reduce(r[:, fin], MEAN, 1, uni, 0), risk_reduce(r[:, fin], MEAN, 0),
                               rtol=1e-5, atol=1e-6)
    assert np.array_equal(weighted_reduce(r[:, fin], CVAR, 1.0 / K, uni, 0), r[:, fin].min(0))
    for m in range(1, K + 1):
        np.testing.assert_allclose(weighted_reduce(r[:, fin], CVAR, m / K, uni, 0), risk_reduce(r[:, fin], CVAR, m / K),
                                   rtol=1e-5, atol=1e-5)
    # a one-hot belief scores by that member alone under every measure
    hot = np.zeros(K, f32)
    hot[K - 1] = 1
    for mode, a in ((MEAN, 1), (CVAR, 0.5), (CVAR, 1.0 / K)):
        assert same_bits(weighted_reduce(r[:, fin], mode, a, hot, 0), r[K - 1, fin])
    # CVaR with alpha = 1 under any belief is its weighted mean up to rounding
    w = np.random.default_rng(K).dirichlet(np.ones(K)).astype(f32)
    np.testing.assert_allclose(weighted_reduce(r[:, fin], CVAR, 1.0, w, 0), weighted_reduce(r[:, fin], MEAN, 1, w, 0),
                               rtol=1e-5, atol=1e-5)


def test_pruned_members_are_ignored():
    K = 4
    w = np.array([0.6, 0.3, 0.05, 0.05], f32)
    r = np.array([[1.0], [2.0], [np.nan], [-np.inf]], f32)
    for mode, a in ((MEAN, 1), (CVAR, 0.5), (CVAR, 0.25)):
        assert np.isnan(weighted_reduce(r, mode, a, w, 0.0))[0]
        assert not np.isnan(weighted_reduce(r, mode, a, w, 0.1))[0]
    assert weighted_reduce(r, CVAR, 0.25, w, 0.1)[0] == 1.0
    # CVaR 0.5 of mass 0.9: tau = 0.45, all of it on the lower reward
    assert weighted_reduce(r, CVAR, 0.5, w, 0.1)[0] == 1.0
    # prune never removes the argmax, even at its weight
    assert weighted_reduce(r[:2], MEAN, 1, np.array([0.5, 0.5], f32), 0.5)[0] == f32(1.5)


# ---- the device code against the restatement -----------------------------------------------------------
@pytest.mark.parametrize("K", list(range(2, KMAX + 1)))
def test_weighted_device_code_equals_restatement(lib, K):
    for name, w, prunes in beliefs(K):
        for prune in prunes:
            assert float(f32(prune)) < 1.0 / K
            r = rewards(K, w, prune)
            for mode, a in [(MEAN, 1.0)] + [(CVAR, a) for a in alphas(K)]:
                want = weighted_reduce(r, mode, a, w, prune)
                got = emul_reduce(lib, r, mode, a, w, prune)
                assert same_bits(got, want), (K, name, prune, mode, a)
            if name == "at-threshold":        # the member at the threshold counts
                assert kept_members(w, prune).count(True) >= 2


def test_left_out_member_at_the_bottom_does_not_move_the_score(lib):
    K = 5
    w = np.array([0.4, 0.3, 0.2, 0.06, 0.04], f32)
    r = samples(K, seed=3)[:, :16].copy()
    base = emul_reduce(lib, r, CVAR, 0.3, w, 0.05)
    r[4] = -1e30
    assert same_bits(emul_reduce(lib, r, CVAR, 0.3, w, 0.05), base)
    assert not same_bits(emul_reduce(lib, r, CVAR, 0.3, w, 0.0), base)


def _update_case(K, nv, seed):
    g = np.random.default_rng(seed)
    v = g.normal(size=nv).astype(f32)
    vhat = (v + g.normal(size=(K, nv)) * g.uniform(0.01, 0.5, size=(K, 1))).astype(f32)
    vhat[0] = v                                      # a member that predicts the plant exactly
    sigma = g.uniform(0.05, 0.5, nv).astype(f32)
    return vhat, v, sigma


@pytest.mark.parametrize("K", [2, 3, 4, 16])
@pytest.mark.parametrize("forget", [1.0, 0.9, 0.5])
def test_belief_update_equals_restatement(lib, K, forget):
    nv = 18
    L = [math.log(1.0 / K)] * K
    for step in range(12):
        vhat, v, sigma = _update_case(K, nv, 1000 * K + step)
        if step == 3:
            vhat[K - 1, 2] = np.nan                  # a blown-up member: capped at -C
        if step == 4:
            vhat[1] = vhat[1] * 1e20                 # a residual that overflows: -C
        ell = [member_loglik(vhat[k], v, sigma) for k in range(K)]
        assert ell[0] == 0 and (step != 3 or ell[K - 1] == -CAP)
        want_L, want_w = belief_update(L, ell, forget)
        got_L, got_w, got_ell = emul_update(lib, vhat, v, sigma, forget, L)
        assert np.array_equal(got_ell.view(np.int64), np.array(ell).view(np.int64)), step
        assert np.array_equal(got_L.view(np.int64), np.array(want_L).view(np.int64)), step
        assert same_bits(got_w, want_w), step
        L = want_L
    assert np.argmax(L) == 0


def test_belief_update_edges(lib):
    K, nv = 4, 6
    vhat, v, sigma = _update_case(K, nv, 7)
    # an excluded member (prior weight 0) stays at -inf, whatever it predicts
    L = [math.log(0.5), -math.inf, math.log(0.25), math.log(0.25)]
    vhat[1] = v
    for forget in (1.0, 0.8):
        got_L, got_w, _ = emul_update(lib, vhat, v, sigma, forget, L)
        want_L, want_w = belief_update(L, [member_loglik(vhat[k], v, sigma) for k in range(K)], forget)
        assert got_L[1] == -math.inf and got_w[1] == 0
        assert np.array_equal(got_L, want_L) and same_bits(got_w, want_w)
    # a NaN plant state: every member gets -C, and the belief moves by rounding only
    vn = v.copy()
    vn[0] = np.nan
    L = [math.log(x) for x in (0.1, 0.2, 0.3, 0.4)]
    got_L, got_w, got_ell = emul_update(lib, vhat, vn, sigma, 1.0, L)
    assert (got_ell == -CAP).all()
    np.testing.assert_allclose(got_w, [0.1, 0.2, 0.3, 0.4], rtol=1e-6)
    assert np.array_equal(got_L, belief_update(L, [-CAP] * K, 1.0)[0])


# ---- emulator: the member-prediction launch ------------------------------------------------------------
def test_prediction_rows_equal_single_instance_env_steps(lib):
    """mpc_enqueue's prediction launch: rows b K + k, rows_per_inst = K, rows_per_model = 1, one member model
    per CTA, per-instance tasks at task_rows = K; each row is bitwise a dial_env_step (one row, the member's
    model as the plan's) from instance b's state with the action Y[b][0]."""
    from tests.conftest import make_pair
    from tests.test_ensemble import _desc_with_task
    env, o = make_pair("unitree_go2_walk")
    m0 = env.sys.model
    fr = [0.4, 0.4, 0.02, 0.01, 0.01]
    members = [env.sys.tree_replace({"body_mass": {"base": m0.arrays["body_mass"][1] + 3.0}}).model,
               env.sys.tree_replace({"pair_friction": {f: fr for f in FEET}}).model,
               env.sys.tree_replace({"dof_damping": m0.arrays["dof_damping"] * 2}).model]
    B, K, nu, nv = 2, 3, env.action_size, m0.nv
    g = np.random.default_rng(5)
    s = o.reset()
    qpos = np.repeat(s.qpos[None] if s.qpos.ndim == 1 else s.qpos, B, 0).astype(f32)
    qpos[:, 2] += g.uniform(-0.02, 0.02, B)
    qpos[:, 7:7 + nu] += g.normal(size=(B, nu)) * 0.05
    qvel = (g.normal(size=(B, nv)) * 0.2).astype(f32)
    warm = (g.normal(size=(B, nv)) * 0.1).astype(f32)
    Y0 = np.clip(g.normal(size=(B, nu)) * 0.4, -1, 1).astype(f32)       # Y[b][0]
    counters = np.array([[3, 0], [41, 0]], np.int32)
    tasks = [env.task(), env.task()]
    tasks[1].vel_cmd[0] = 0.8
    desc = env.plan_desc(n_inst=B, n_ens=K, Nsample=4, Hsample=6, Hnode=3)
    single = env.plan_desc(Nsample=4, Hsample=6, Hnode=3)
    md = _capi.fill_model_desc(m0)
    slots = [members[k] for b in range(B) for k in range(K)]
    tarr = (_capi.dial_task * B)(*tasks)
    us = np.ascontiguousarray(np.repeat(Y0, K, 0))                     # the gather: row b K + k = Y[b][0]
    qd = np.zeros((B * K, nv), f32)
    emul.launch(md, desc, models=slots, mode=0, nrows=B * K, H=1, rows_per_inst=K, rows_per_model=1, tasks=tarr,
                task_rows=K, qpos0=qpos, qvel0=qvel, warm0=warm, counters_in=counters, us=us, qd=qd)
    for b in range(B):
        for k in range(K):
            one = np.zeros((1, nv), f32)
            emul.launch(members[k], _desc_with_task(single, tasks[b]), mode=0, nrows=1, H=1,
                        qpos0=qpos[b:b + 1].copy(), qvel0=qvel[b:b + 1].copy(), warm0=warm[b:b + 1].copy(),
                        counters_in=counters[b:b + 1].copy(), us=Y0[b:b + 1].copy(), qvel_out=one)
            assert np.array_equal(qd[b * K + k], one[0]), (b, k)
        # the members were read: their predictions differ from one another
        assert not np.array_equal(qd[b * K], qd[b * K + 1]) and not np.array_equal(qd[b * K], qd[b * K + 2]), b
    assert not np.array_equal(qd[0], qd[K])


# ---- adapt specs and the CLI ---------------------------------------------------------------------------
def test_adapt_setting():
    from dial_mpc_b200.core.dial_core import adapt_setting, load_ensemble, load_setting, prior_setting
    forget, prune, sigma = adapt_setting({"sigma": 0.1}, 4, 18)
    assert (forget, prune) == (1.0, 0.0) and sigma.dtype == f32 and sigma.shape == (18,) and (sigma == f32(0.1)).all()
    s = [0.1] * 6 + [0.5] * 12
    forget, prune, sigma = adapt_setting({"sigma": s, "forget": 0.9, "prune": 0.2}, 4, 18)
    assert (forget, prune) == (0.9, 0.2) and np.array_equal(sigma, np.array(s, f32))
    assert np.array_equal(prior_setting([1, 0, 3], 3), np.array([1, 0, 3], f32))
    env = _go2()
    spec = {"members": [{}, {}], "adapt": {"sigma": 0.2, "forget": 0.95}, "prior": [3, 1]}
    members, plant = load_ensemble(spec, env)
    assert len(members) == 2
    assert load_setting(spec, "adapt", 2, env.sys.nv) == {"sigma": 0.2, "forget": 0.95}
    assert load_setting(spec, "prior", 2) == [3.0, 1.0]
    assert load_setting({"members": [{}, {}]}, "adapt", 2, 18) is None
    assert load_setting({"members": [{}, {}]}, "prior", 2) is None


BAD_ADAPT = [
    ({"forget": 0.9}, r"adapt needs sigma"),
    ({"sigma": [0.1] * 3}, r"sigma must be one number or a list of 18 \(one per dof\), got a list of 3"),
    ({"sigma": 0}, r"sigma must be a finite number > 0 .* got 0"),
    ({"sigma": [0.1] * 17 + [-1]}, r"sigma must be finite and > 0, got -1"),
    ({"sigma": float("nan")}, r"sigma must be .* got nan"),
    ({"sigma": 0.1, "forget": 0}, r"forget must be a finite number in \(0, 1\], got 0"),
    ({"sigma": 0.1, "forget": 1.5}, r"forget must be .* got 1.5"),
    ({"sigma": 0.1, "prune": 0.25}, r"prune must be a number in \[0, 1/K\) = \[0, 0.25\), got 0.25"),
    ({"sigma": 0.1, "prune": -0.1}, r"prune must be .* got -0.1"),
    ({"sigma": 0.1, "gain": 1}, r"unknown key 'gain'"),
    (0.1, r"an adapt spec maps 'sigma'"),
]


@pytest.mark.parametrize("adapt, match", BAD_ADAPT)
def test_adapt_setting_names_the_bad_value(adapt, match):
    from dial_mpc_b200.core.dial_core import adapt_setting
    with pytest.raises(ValueError, match=match):
        adapt_setting(adapt, 4, 18)


@pytest.mark.parametrize("w, match", [([1, 2], r"list of 3 weights"), ([1, -1, 1], r"finite and >= 0, got -1"),
                                      ([0, 0, 0], r"positive sum"), ([1, float("inf"), 0], r"got inf"),
                                      ("abc", r"list of 3 weights")])
def test_prior_setting_names_the_bad_value(w, match):
    from dial_mpc_b200.core.dial_core import prior_setting
    with pytest.raises(ValueError, match=match):
        prior_setting(w, 3)


def _main(monkeypatch, capsys, argv):
    from dial_mpc_b200.core import dial_core
    monkeypatch.setattr(sys, "argv", ["dial_core", "--example", "unitree_go2_trot"] + argv)
    with pytest.raises(SystemExit) as e:
        dial_core.main()
    return e.value.code, capsys.readouterr().err


FOUR = [{}, {"body_mass": {"base": 9.0}}, {}, {}]


@pytest.mark.parametrize("adapt, match", BAD_ADAPT)
def test_cli_ensemble_file_adapt_errors(tmp_path, monkeypatch, capsys, adapt, match):
    import yaml
    f = tmp_path / "ens.yaml"
    f.write_text(yaml.safe_dump({"members": FOUR, "adapt": adapt}))
    code, err = _main(monkeypatch, capsys, ["--ensemble", str(f)])
    assert code == 2 and re.search(r"--ensemble .*ens\.yaml: adapt: " + match, err), err


@pytest.mark.parametrize("extra, match", [
    ({"members": [{}], "adapt": {"sigma": 0.1}}, r"adapt: needs an ensemble of at least 2 members, got 1"),
    ({"members": FOUR, "prior": [1, 1]}, r"prior: a belief is a list of 4 weights"),
    ({"members": FOUR, "prior": [1, 0, 0, -2]}, r"prior: every weight must be finite and >= 0, got -2"),
    ({"members": FOUR, "prior": [0, 0, 0, 0]}, r"prior: the weights must have a positive sum"),
    ({"members": [{}], "prior": [1]}, r"prior: needs an ensemble of at least 2 members"),
])
def test_cli_ensemble_file_prior_and_size_errors(tmp_path, monkeypatch, capsys, extra, match):
    import yaml
    f = tmp_path / "ens.yaml"
    f.write_text(yaml.safe_dump(extra))
    code, err = _main(monkeypatch, capsys, ["--ensemble", str(f)])
    assert code == 2 and re.search(r"--ensemble .*ens\.yaml: " + match, err), err


@pytest.mark.parametrize("adapt, match", BAD_ADAPT[:3] + BAD_ADAPT[5:10])
def test_cli_instance_override_adapt_errors(tmp_path, monkeypatch, capsys, adapt, match):
    import yaml
    ens, ov = tmp_path / "ens.yaml", tmp_path / "ov.yaml"
    ens.write_text(yaml.safe_dump({"members": FOUR}))
    ov.write_text(yaml.safe_dump([{"adapt": {"sigma": 0.1}}, {"default_vx": 0.5, "adapt": adapt}]))
    code, err = _main(monkeypatch, capsys, ["--instances", "2", "--ensemble", str(ens), "--instance-overrides", str(ov)])
    assert code == 2 and re.search(r"--instance-overrides entry 1: adapt: " + match, err), err


def test_cli_instance_override_adapt_needs_ensemble(tmp_path, monkeypatch, capsys):
    import yaml
    ov = tmp_path / "ov.yaml"
    ov.write_text(yaml.safe_dump([{}, {"adapt": {"sigma": 0.1}}]))
    code, err = _main(monkeypatch, capsys, ["--instances", "2", "--instance-overrides", str(ov)])
    assert code == 2 and "--instance-overrides entry 1: adapt needs --ensemble" in err, err
