"""K5 (the prioritized-replay segment trees, csrc/per_tree.cu) against the float32 oracle bit for bit where the parity test of
tests/test_gpu_per.py does not reach: the production shape (16 envs, 2^16 leaves per env, k = 32), the block-stride loops of
the sample and update kernels (k > 256), padded leaves, the smallest and a just-wrapped ring, duplicated indices, and
priorities at the edges of float32.

The oracle's trees are seeded with the device's leaves through a vectorised float32 builder; internal nodes are a pure
function of the leaves, and test_tree_builder_equals_sequential_sets proves on the CPU that the builder equals the
oracle's own sequential TreeF32.set."""
import numpy as np
import pytest
import torch

from oracle.replay import PerReplayOracle, TreeF32, next_pow2

F32 = np.float32
DEV = "cuda:0"
gpu = pytest.mark.gpu


def build_tree(leaves, kind):
    """[2 cap] float32 heap over cap leaves, rebuilt level by level: a parent is fl32(left + right) or Python's min(left,
    right) (right only if strictly smaller), as TreeF32 computes it."""
    leaves = np.asarray(leaves, F32)
    cap = leaves.shape[-1]
    v = np.full(leaves.shape[:-1] + (2 * cap,), 0.0 if kind == "sum" else np.inf, F32)
    v[..., cap:] = leaves
    lvl = cap // 2
    while lvl >= 1:
        l, r = v[..., 2 * lvl:4 * lvl:2], v[..., 2 * lvl + 1:4 * lvl:2]
        v[..., lvl:2 * lvl] = (l + r) if kind == "sum" else np.where(r < l, r, l)
        lvl //= 2
    return v


@pytest.mark.parametrize("cap", [1, 2, 8, 64, 1024])
def test_tree_builder_equals_sequential_sets(cap):
    """CPU: random leaves (with zeros, repeated values and infinities among the min leaves) set one at a time in random
    order, some twice, through TreeF32.set give the builder's trees bit for bit."""
    rng = np.random.default_rng(cap)
    leaves = (rng.random(cap) * 3).astype(F32)
    leaves[rng.random(cap) < 0.2] = 0.0
    leaves[rng.random(cap) < 0.2] = F32(0.7)
    for kind in ("sum", "min"):
        t = TreeF32(cap, kind)
        order = np.concatenate([rng.permutation(cap), rng.integers(0, cap, cap // 2)])
        for i in order:
            t.set(int(i), leaves[i] + F32(1.0))                  # a first value, overwritten below
        want = leaves.copy()
        if kind == "min":
            want[rng.random(cap) < 0.3] = np.inf
        for i in rng.permutation(cap):
            t.set(int(i), want[i])
        assert np.array_equal(build_tree(want, kind), t.v), kind


# ------------------------------------------------------------------------------------------------------------ GPU
def _pair(N, n_size, B, alpha, size, ptr, rng, max_priority=1.0):
    """(device buffer, oracle) with identical trees: leaves [0, size) random in (0.01, 3.01), the rest unset."""
    from xuance_b200.common import PerOffPolicyBuffer, Box, Discrete
    prod = PerOffPolicyBuffer(Box(-1, 1, (1,), np.float32), Discrete(4), None, N, N * n_size, B, alpha=alpha, device=DEV)
    orc = PerReplayOracle((1,), (), N, N * n_size, B, alpha=alpha)
    cap = next_pow2(n_size)
    assert prod._it_capacity == cap
    s = np.zeros((N, cap), F32)
    s[:, :size] = (rng.random((N, size)) * 3 + 0.01).astype(F32)
    m = s.copy()
    m[:, size:] = np.inf
    st, mt = build_tree(s, "sum"), build_tree(m, "min")
    prod._it_sum.copy_(torch.from_numpy(st))
    prod._it_min.copy_(torch.from_numpy(mt))
    prod._max_priority.fill_(max_priority)
    for i in range(N):
        orc.sum[i].v, orc.min[i].v = st[i].copy(), mt[i].copy()
    orc.max_priority[:] = F32(max_priority)
    prod.ptr = orc.ptr = ptr
    prod.size = orc.size = size
    return prod, orc


def _same_trees(prod, orc, what):
    assert np.array_equal(prod._max_priority.cpu().numpy(), orc.max_priority), what
    ps, pm = prod._it_sum.cpu().numpy(), prod._it_min.cpu().numpy()
    for i in range(prod.n_envs):
        assert np.array_equal(ps[i], orc.sum[i].v), (what, "sum", i, np.flatnonzero(ps[i] != orc.sum[i].v)[:8])
        assert np.array_equal(pm[i], orc.min[i].v), (what, "min", i, np.flatnonzero(pm[i] != orc.min[i].v)[:8])


def _sample(prod, orc, rng, beta, what):
    """Sample both with the same uniforms; indices, flat indices and weights must be identical.  Returns the indices."""
    from xuance_b200 import _lib
    N, k = prod.n_envs, prod._k
    u = rng.random((N, k)).astype(F32)
    sp, so = prod.sample(beta, uniforms=u), orc.sample(beta, uniforms=u)
    steps = sp["step_choices"].cpu().numpy()
    assert np.array_equal(steps, so["step_choices"]), what
    assert np.array_equal(sp["weights"].cpu().numpy(), so["weights"]), what
    # the flat (env, step) rows the gather reads: the same launch through the ABI, which exposes them
    step_d = torch.empty((N, k), dtype=torch.int64, device=DEV)
    flat = torch.empty((N * k,), dtype=torch.int64, device=DEV)
    w = torch.empty((N, k), dtype=torch.float64, device=DEV)
    _lib.call("xb_per_sample", _lib.ptr(prod._it_sum), _lib.ptr(prod._it_min), _lib.ptr(torch.from_numpy(u).to(DEV)), N,
              prod._it_capacity, prod.size, k, prod.n_size, float(F32(prod.size ** (-beta))), _lib.ptr(step_d),
              _lib.ptr(flat), _lib.ptr(w))
    assert np.array_equal(step_d.cpu().numpy(), steps), what
    assert np.array_equal(flat.cpu().numpy(), (np.arange(N)[:, None] * prod.n_size + steps).reshape(-1)), what
    assert np.array_equal(w.cpu().numpy(), so["weights"]), what
    return steps


def _update(prod, orc, idx, prios, what):
    prod.update_priorities(torch.as_tensor(np.asarray(idx, np.int64), device=DEV), torch.as_tensor(np.asarray(prios, F32), device=DEV))
    orc.update_priorities(np.asarray(idx, np.int64), np.asarray(prios, F32))
    _same_trees(prod, orc, what)


def _store(prod, orc, ptr, rng, what):
    N = prod.n_envs
    prod.ptr = orc.ptr = ptr
    step = (rng.normal(size=(N, 1)).astype(F32), rng.integers(0, 4, N), rng.normal(size=N).astype(F32),
            rng.random(N) < 0.1, rng.normal(size=(N, 1)).astype(F32))
    prod.store(*step), orc.store(*step)
    assert prod.ptr == orc.ptr and prod.size == orc.size
    _same_trees(prod, orc, what)


@gpu
def test_production_scale_rounds_bit_exact():
    """configs/perdqn/atari.yaml's shape: 16 envs, buffer_size 2^20 (n_size = cap = 65536), B = 512, alpha 0.5.  Rounds of
    sample -> update_priorities -> store with the insert pointer at 0, cap - 1 and in between; after each step the
    indices, flat indices, weights, max priorities and both whole trees equal the oracle's."""
    rng = np.random.default_rng(0)
    N, n_size, B = 16, 2 ** 16, 512
    prod, orc = _pair(N, n_size, B, 0.5, n_size, 0, rng, max_priority=2.5)
    _same_trees(prod, orc, "seeded")
    for r, ptr in enumerate((0, n_size - 1, 12345, 0)):
        steps = _sample(prod, orc, rng, 0.4 + 0.1 * r, "round %d sample" % r)
        td = np.abs(rng.normal(size=B) * 2).astype(F32)
        td[::37] = 0.0
        if r == 1:
            td[5] = 7.5                                       # raises max_priority: the next insert uses it
        _update(prod, orc, steps, td, "round %d update" % r)
        _store(prod, orc, ptr, rng, "round %d store at %d" % (r, ptr))


@gpu
@pytest.mark.parametrize("N,n_size,B", [(1, 3000, 1024), (2, 3000, 600), (2, 4096, 600)])
def test_block_stride_loops_and_padded_leaves(N, n_size, B):
    """k = B / N > 256 (1024, and 300 = not a multiple of 32): both kernels' block-stride loops and the 8-warp max
    reduction with partly filled warps; n_size 3000 pads the tree to 4096 leaves."""
    rng = np.random.default_rng(B + n_size)
    prod, orc = _pair(N, n_size, B, 0.6, n_size - 17, n_size - 17, rng)
    for r in range(3):
        steps = _sample(prod, orc, rng, 0.4, "round %d" % r)
        td = np.abs(rng.normal(size=B)).astype(F32)
        td[rng.integers(0, B)] = 9.0 + r                      # the batch max sits in a random warp
        _update(prod, orc, steps, td, "round %d update" % r)
        _store(prod, orc, prod.ptr, rng, "round %d store" % r)


@gpu
def test_smallest_and_just_wrapped_ring():
    """size = 2 (the least the sampler accepts), then a ring filled to n_size and wrapped by one store."""
    rng = np.random.default_rng(5)
    prod, orc = _pair(2, 100, 64, 0.5, 2, 2, rng)
    for r in range(2):
        steps = _sample(prod, orc, rng, 0.4, "size 2")
        _update(prod, orc, steps, np.abs(rng.normal(size=64)).astype(F32), "size 2 update")
    prod, orc = _pair(2, 100, 64, 0.5, 100, 99, rng)
    _store(prod, orc, 99, rng, "fill the last slot")
    assert prod.ptr == 0
    _store(prod, orc, 0, rng, "wrap")
    steps = _sample(prod, orc, rng, 0.4, "wrapped")
    _update(prod, orc, steps, np.abs(rng.normal(size=64)).astype(F32), "wrapped update")


@gpu
def test_duplicate_indices():
    """Duplicated leaves in one update: the last writer's priority wins the leaf, the batch maximum wins max_priority -
    all k indices equal; pairs whose later item has the smaller priority; and pairs j, j + 256 that straddle the
    kernel's 256-thread stride."""
    rng = np.random.default_rng(9)
    N, n_size, B = 2, 1000, 600
    k = B // N
    prod, orc = _pair(N, n_size, B, 0.5, n_size, 0, rng)
    prios = (rng.random(B) * 2 + 0.1).astype(F32)
    _update(prod, orc, np.full((N, k), 17), prios, "all equal")
    idx = rng.integers(0, n_size, (N, k))
    idx[:, 1::2] = idx[:, 0::2]                               # pairs (2j, 2j + 1)
    p = prios.reshape(N, k).copy()
    p[:, 1::2] = p[:, 0::2] * F32(0.5)                         # the later duplicate is smaller
    _update(prod, orc, idx, p.reshape(-1), "pairs, later smaller")
    idx = rng.permutation(n_size)[:N * k].reshape(N, k)
    for j in (0, 3, 31, 40):
        idx[:, j + 256] = idx[:, j]                           # same thread, next stride iteration
    p = (rng.random((N, k)) + 0.1).astype(F32)
    p[:, 3] = 50.0                                            # the first of a pair holds the batch max
    _update(prod, orc, idx, p.reshape(-1), "pairs across the stride")


EDGE_PRIOS = [0.0, -0.0, 1e-8, 2.0 ** -149, 3 * 2.0 ** -149, 2.0 ** -140, 1e-40, 2.0 ** -127, 2.0 ** -126 * 0.999,
              2.0 ** -126, 2.0 ** 126, 2.0 ** 127, 3.0e38, float(np.finfo(F32).max)]


@gpu
@pytest.mark.parametrize("alpha", [0.5, 0.6, 1.0])
def test_priority_edges(alpha):
    """Priorities 0.0 and -0.0 (both become 1e-8), exactly 1e-8, subnormals and values >= 2^126: leaves (float32 ** alpha
    through the device's libm restatement), trees and max_priority equal the oracle's.  At alpha = 1 the sums overflow to
    inf, in both."""
    rng = np.random.default_rng(int(alpha * 10))
    N, n_size, B = 2, 512, 64
    prod, orc = _pair(N, n_size, B, alpha, n_size, 0, rng)
    idx = rng.permutation(n_size)[:B].reshape(N, B // N)
    p = np.array((EDGE_PRIOS * 5)[:B], F32)
    with np.errstate(over="ignore"):
        _update(prod, orc, idx, p, "edge priorities")
