"""GPU parity: K5 prioritized-replay trees vs the float32 NumPy oracle - BIT-EXACT indices, leaves, sums, weights."""
import random

import numpy as np
import pytest
import torch

from oracle.replay import PerReplayOracle, UniformReplayOracle

pytestmark = pytest.mark.gpu


def _step(rng, N, obs_shape, u8):
    if u8:
        o = rng.integers(0, 256, size=(N,) + obs_shape, dtype=np.uint8)
        o2 = rng.integers(0, 256, size=(N,) + obs_shape, dtype=np.uint8)
    else:
        o = rng.normal(size=(N,) + obs_shape).astype(np.float32)
        o2 = rng.normal(size=(N,) + obs_shape).astype(np.float32)
    return o, rng.integers(0, 4, N), rng.normal(size=N).astype(np.float32), rng.random(N) < 0.1, o2


@pytest.mark.parametrize("N,S,B,obs_shape,u8,alpha", [(4, 64, 32, (3,), False, 0.5), (2, 100, 64, (12, 12, 4), True, 0.6),
                                                       (16, 37, 512, (5,), False, 0.5)])
def test_per_buffer_bit_exact(N, S, B, obs_shape, u8, alpha):
    from xuance_b200.common import PerOffPolicyBuffer, Box, Discrete
    rng = np.random.default_rng(N + S)
    space = Box(0, 255, obs_shape, np.uint8) if u8 else Box(-9, 9, obs_shape, np.float32)
    prod = PerOffPolicyBuffer(space, Discrete(4), None, N, N * S, B, alpha=alpha, device="cuda:0")
    orc = PerReplayOracle(obs_shape, (), N, N * S, B, alpha=alpha, obs_dtype=np.uint8 if u8 else np.float32)
    for t in range(int(S * 1.5)):       # wraps the ring
        st = _step(rng, N, obs_shape, u8)
        prod.store(*st), orc.store(*st)
        if t > 3 and t % 4 == 0:
            random.seed(t)
            sp = prod.sample(0.4)
            random.seed(t)
            so = orc.sample(0.4)
            assert np.array_equal(sp["step_choices"].cpu().numpy(), so["step_choices"]), t
            assert np.array_equal(sp["weights"].cpu().numpy(), so["weights"]), t
            for k in ("obs", "actions", "obs_next", "rewards", "terminals"):
                assert np.array_equal(sp[k].cpu().numpy(), so[k]), k
            td = np.abs(rng.normal(size=B)).astype(np.float32)
            td[1] = 0.0
            prod.update_priorities(sp["step_choices"], td)
            orc.update_priorities(so["step_choices"], td)
            assert np.array_equal(prod._max_priority.cpu().numpy(), orc.max_priority)
            ps, pm = prod._it_sum.cpu().numpy(), prod._it_min.cpu().numpy()
            for i in range(N):
                assert np.array_equal(ps[i], orc.sum[i].v), (t, i)
                assert np.array_equal(pm[i], orc.min[i].v), (t, i)
    assert prod.ptr == orc.ptr and prod.size == orc.size


def test_per_full_capacity_properties():
    """BASELINE config 3 scale (2^20 transitions, 16 envs, cap 65536 per env) on small rows: after random priority
    updates every internal node equals op(children) (float32), the root equals the float32 pairwise tree-sum, and
    sampled indices land on positive-priority leaves with in-range masses."""
    from xuance_b200.common import PerOffPolicyBuffer, Box, Discrete
    N, S, B = 16, 65536, 512
    prod = PerOffPolicyBuffer(Box(-1, 1, (2,), np.float32), Discrete(4), None, N, N * S, B, alpha=0.5, device="cuda:0")
    # fill the ring directly (store() is exercised above); leaves = 1^alpha
    prod.ptr, prod.size = 0, S
    leaves = torch.rand((N, S), device="cuda:0") + 0.01
    cap = prod._it_capacity
    prod._it_sum[:, cap:cap + S] = leaves
    prod._it_min[:, cap:cap + S] = leaves
    lvl = cap // 2
    while lvl >= 1:
        prod._it_sum[:, lvl:2 * lvl] = prod._it_sum[:, 2 * lvl:4 * lvl:2] + prod._it_sum[:, 2 * lvl + 1:4 * lvl:2]
        prod._it_min[:, lvl:2 * lvl] = torch.minimum(prod._it_min[:, 2 * lvl:4 * lvl:2], prod._it_min[:, 2 * lvl + 1:4 * lvl:2])
        lvl //= 2
    rng = np.random.default_rng(0)
    for it in range(5):
        s = prod.sample(0.5, uniforms=rng.random((N, B // N)))
        sc = s["step_choices"]
        assert int(sc.min()) >= 0 and int(sc.max()) < S
        prod.update_priorities(sc, torch.rand(B, device="cuda:0") * 3)
    t, m = prod._it_sum, prod._it_min
    lvl = cap // 2
    while lvl >= 1:
        assert torch.equal(t[:, lvl:2 * lvl], t[:, 2 * lvl:4 * lvl:2] + t[:, 2 * lvl + 1:4 * lvl:2])
        assert torch.equal(m[:, lvl:2 * lvl], torch.minimum(m[:, 2 * lvl:4 * lvl:2], m[:, 2 * lvl + 1:4 * lvl:2]))
        lvl //= 2


def test_uniform_replay_matches_oracle():
    from xuance_b200.common import DummyOffPolicyBuffer, DummyOffPolicyBuffer_Atari, Box, Discrete
    rng = np.random.default_rng(2)
    for u8, shape, cls in ((False, (17,), DummyOffPolicyBuffer), (True, (84, 84, 4), DummyOffPolicyBuffer_Atari)):
        N, S, B = 4, 24, 64
        space = Box(0, 255, shape, np.uint8) if u8 else Box(-9, 9, shape, np.float32)
        prod = cls(space, Discrete(4), None, N, N * S, B, device="cuda:0")
        orc = UniformReplayOracle(shape, (), N, N * S, B, obs_dtype=np.uint8 if u8 else np.float32)
        for t in range(30):
            st = _step(rng, N, shape, u8)
            prod.store(*st), orc.store(*st)
        np.random.seed(7)
        sp = prod.sample()
        np.random.seed(7)
        so = orc.sample()
        for k in ("obs", "actions", "obs_next", "rewards", "terminals"):
            assert np.array_equal(sp[k].cpu().numpy(), so[k]), k


def test_continuous_action_replay():
    from xuance_b200.common import DummyOffPolicyBuffer, Box
    rng = np.random.default_rng(4)
    N, S, B = 4, 16, 32
    prod = DummyOffPolicyBuffer(Box(-9, 9, (17,), np.float32), Box(-1, 1, (6,), np.float32), None, N, N * S, B, device="cuda:0")
    orc = UniformReplayOracle((17,), (6,), N, N * S, B)
    for t in range(20):
        o = rng.normal(size=(N, 17)).astype(np.float32)
        a = rng.uniform(-1, 1, size=(N, 6)).astype(np.float32)
        r = rng.normal(size=N).astype(np.float32)
        d = rng.random(N) < 0.1
        o2 = rng.normal(size=(N, 17)).astype(np.float32)
        prod.store(o, a, r, d, o2), orc.store(o, a, r, d, o2)
    np.random.seed(1)
    sp = prod.sample()
    np.random.seed(1)
    so = orc.sample()
    for k in ("obs", "actions", "obs_next", "rewards", "terminals"):
        assert np.array_equal(sp[k].cpu().numpy(), so[k]), k


@pytest.mark.parametrize("alpha", [0.5, 0.6, 0.4, 1.0, 0.25])
def test_powf_restatement_bit_exact(alpha):
    """The device restatement of glibc powf == numpy's float32 ** python-float (what the reference evaluates for
    every PER leaf, memory_tools.py:547,596) on 200k priorities incl. tiny / huge / exact-power-of-two inputs, and one
    value from every binade from 2^-149 (subnormal) to 2^127 plus both ends of each."""
    from xuance_b200 import _lib
    rng = np.random.default_rng(int(alpha * 100))
    p = np.abs(rng.normal(size=200_000)).astype(np.float32) * np.float32(3.0) + np.float32(1e-8)
    p[:8] = np.array([1e-8, 1.0, 2.0, 0.5, 1e-3, 1e3, 7.0, 0.3333333], np.float32)
    e = np.arange(-149, 128)
    binades = np.concatenate([np.ldexp(rng.uniform(1.0, 1.99, e.size), e), np.ldexp(1.0, e),
                              np.ldexp(2.0 - 2.0 ** -23, e)]).astype(np.float32)
    p = np.concatenate([p, binades[binades > 0]])
    want = np.array([x ** alpha for x in p], dtype=np.float32)      # numpy scalar power -> libm powf
    d = torch.from_numpy(p).cuda()
    out = torch.empty_like(d)
    _lib.call("xb_powf_libm", _lib.ptr(d), float(np.float32(alpha)), _lib.ptr(out), p.size)
    assert np.array_equal(out.cpu().numpy(), want)
