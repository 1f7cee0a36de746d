"""CPU tests of the fp64 update reference (oracle/planner_oracle.py: softmax_weights_fp64,
reverse_update_fp64) and of the erfinv tail helper that the GPU update tests
(tests/test_gpu_update.py) use to pick sampler elements."""
import types

import numpy as np
import pytest
import torch
from scipy.special import erf, erfinv

from oracle import planner_oracle as po


def _emul_plan(N, Hn, temp):
    from tests.emul.emul import EmulPlan
    env = types.SimpleNamespace(sys=types.SimpleNamespace(nq=19, nv=18, nu=12, nbody=14))
    desc = types.SimpleNamespace(Nsample=N, Ntotal=N, Hsample=16, Hnode=Hn, temp_sample=temp, shard_offset=0)
    return EmulPlan(env, desc)


@pytest.mark.parametrize("N,Hn,seed", [(1, 1, 0), (2, 4, 1), (255, 4, 2), (2048, 7, 3)])
def test_reference_equals_emulated_update_on_ordinary_rewards(N, Hn, seed):
    """Finite rewards with a finite mean row: the guarded reference is the reference formula
    (dial_core.py:125-132) that EmulPlan restates."""
    rng = np.random.default_rng(seed)
    temp = 0.05
    rews = (rng.normal(size=N + 1) * 0.3 - 1.0).astype(np.float32)
    eps = rng.standard_normal((N, Hn + 1, 12)).astype(np.float32)
    Ybar = (rng.standard_normal((Hn + 1, 12)) * 0.4).astype(np.float32)
    noise = (0.9 ** np.arange(Hn + 1)[::-1]).astype(np.float32)
    w, Y = po.reverse_update_fp64(rews, temp, eps, Ybar, noise)
    plan = _emul_plan(N, Hn, temp)
    Yo, wo = torch.empty(Hn + 1, 12), torch.empty(N + 1)
    plan.reverse_update(torch.from_numpy(eps), None, torch.from_numpy(Ybar), torch.from_numpy(noise),
                        torch.from_numpy(rews), Yo, wo)
    assert np.abs(w - wo.numpy()).max() <= 1e-6 * w.max()      # EmulPlan returns fp32
    assert np.abs(Y - Yo.numpy()).max() < 1e-6
    assert abs(w.sum() - 1) < 1e-12 and (w >= 0).all()


def test_reference_guards():
    rng = np.random.default_rng(4)
    r = rng.normal(size=101) * 0.3 - 1.0
    w = po.softmax_weights_fp64(r, 0.05)
    # diverged samples: weight 0, left out of the statistics
    r2 = r.copy()
    r2[[5, 7, 9]] = [np.nan, np.inf, -np.inf]
    w2 = po.softmax_weights_fp64(r2, 0.05)
    keep = np.ones(101, bool)
    keep[[5, 7, 9]] = False
    assert (w2[~keep] == 0).all()
    assert np.allclose(w2[keep], po.softmax_weights_fp64(r[keep], 0.05), rtol=1e-12, atol=0)
    # a NaN mean-row reward is only a lost reference point of the shift: the mean row gets weight 0,
    # the other samples the softmax of their own rewards
    r3 = r.copy()
    r3[-1] = np.nan
    w3 = po.softmax_weights_fp64(r3, 0.05)
    assert w3[-1] == 0 and np.allclose(w3[:-1], po.softmax_weights_fp64(r[:-1], 0.05), rtol=1e-12, atol=0)
    # finite rewards: the reference formula, logits relative to the mean row
    logp = (r - r[-1]) / r.std() / 0.05
    wr = np.exp(logp - logp.max())
    assert np.allclose(w, wr / wr.sum(), rtol=1e-12, atol=0)
    # flat finite rewards: uniform over the finite samples
    r4 = np.full(11, -2.5)
    r4[3] = np.nan
    w4 = po.softmax_weights_fp64(r4, 0.05)
    assert w4[3] == 0 and np.allclose(np.delete(w4, 3), 0.1, rtol=1e-15)
    # no finite reward: the whole weight on the mean row
    w5 = po.softmax_weights_fp64(np.array([np.nan, -np.inf, np.inf, np.nan]), 0.05)
    assert w5.tolist() == [0, 0, 0, 1]
    # a single finite reward (one-hot weights: how the GPU tests read the sampler)
    r6 = np.full(9, -np.inf)
    r6[4], r6[-1] = 0.0, np.nan
    assert po.softmax_weights_fp64(r6, 0.05).tolist() == [0, 0, 0, 0, 1, 0, 0, 0, 0]
    # a finite outlier far below the bulk: weight exp(-200) here (std = 1e20 / sqrt(101)), not uniform
    r7 = r.copy()
    r7[17] = -1e20
    w7 = po.softmax_weights_fp64(r7, 0.05)
    assert w7[17] < 1e-80 and abs(w7.sum() - 1) < 1e-12 and np.ptp(np.delete(w7, 17)) < 1e-12


def _bits_scalar(key, i, n):
    """Element i of jax.random.bits(key, (n,)), legacy layout, one Threefry call (the kernels'
    jax_bits_legacy): counters split in halves, an odd count padded with one zero counter."""
    half = (n + 1) // 2
    x0, x1 = (i, i + half) if i < half else (i - half, i)
    if x1 >= n:
        x1 = 0
    a, b = po.threefry2x32(key, np.uint32([x0]), np.uint32([x1]))
    return int((b if i >= half else a)[0])


@pytest.mark.parametrize("n", [1, 2, 7, 60, 95 * 31, 96 * 2048])
def test_legacy_bits_layout_odd_and_even_counts(n):
    key = (0x12345678, 0x9ABCDEF0)
    bits = po.jax_random_bits_legacy(key, n)
    half = (n + 1) // 2
    for i in sorted({0, n - 1, max(half - 1, 0), min(half, n - 1), n // 3}):
        assert int(bits[i]) == _bits_scalar(key, i, n), i


@pytest.mark.parametrize("n", [95 * 2047, 60 * 2048])
def test_erfinv_tail_indices(n):
    key = tuple(int(v) for v in po.jax_split_legacy((0, 7))[1])
    idx = po.erfinv_tail_indices(key, n)
    eps = po.jax_normal_legacy(key, (n,))
    # the branch boundary w = 5 is |u| = sqrt(1 - e^-5) = 0.99663, |eps| = 2.9314
    edge = np.sqrt(2.0) * erfinv(np.sqrt(1 - np.exp(-5.0)))
    assert abs(edge - 2.9314) < 1e-4
    rest = np.delete(eps, idx)
    assert np.abs(eps[idx]).min() >= edge - 1e-5 and np.abs(rest).max() <= edge + 1e-5
    assert abs(len(idx) / n - (1 - erf(edge / np.sqrt(2)))) < 1e-3     # P(|eps| > 2.93) = 0.34 %
    assert (eps[idx] > 0).any() and (eps[idx] < 0).any()


def test_xla_erfinv_restatement():
    """erfinv_xla is the exact erfinv to about 3 fp32 ulp of eps, except near |u| = 1, where its one
    fp32 rounding (u * u) moves it by up to d eps / du * 2^-24 |u| = (pi/2)^0.5 exp(eps^2 / 2) 2^-24 |u|."""
    g = np.random.default_rng(5)
    u = np.concatenate([g.uniform(-1, 1, 200000), 1 - 10.0 ** -g.uniform(2, 7, 20000)]).astype(np.float32)
    u = u[np.abs(u) < 1]
    exact = np.sqrt(2.0) * erfinv(u.astype(np.float64))
    xla = np.sqrt(2.0) * po.erfinv_xla(u)
    ulp = np.spacing(np.abs(exact).astype(np.float32)).astype(np.float64)
    bulk = np.abs(u) < 0.99
    assert (np.abs(xla - exact)[bulk] / ulp[bulk]).max() < 3
    cond = np.sqrt(np.pi / 2) * np.exp(exact ** 2 / 2) * 2.0 ** -24 * np.abs(u.astype(np.float64))
    assert (np.abs(xla - exact) <= 3 * ulp + cond).all()
    assert (np.abs(xla - exact)[~bulk] / ulp[~bulk]).max() > 10       # the rounding does show near |u| = 1
    a, b = po.jax_normal_legacy_xla((3, 4), (95, 31)), po.jax_normal_legacy((3, 4), (95, 31))
    assert a.shape == b.shape and np.abs(a - b).max() < 1e-4
