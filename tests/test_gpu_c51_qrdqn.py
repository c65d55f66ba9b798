"""GPU tests of C51 and QR-DQN: the K6Z kernels against their float64 references at edge row counts and (A, N) shapes up to
the limits, Tz / projection weights / QR backup bit-exact against the torch expressions, first-index ties, NaN
propagation, sharded minibatches and launch-to-launch determinism; C51_Learner / QRDQN_Learner against the torch-CPU
oracle (across a target sync, clip on / off, eager / graphed) and against the reference fixture; checkpoints; acting;
CartPole-v1 learning through get_runner; and a SyntheticAtari agent on the K12 encoder."""
import os
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from dist_refs import (greedy_ref, c51_ref, qrdqn_ref, torch_tz, torch_projection, torch_qr_backup,  # noqa: E402
                       supports_of, loss_batch, fixture_batch, fixture_state_dict, OBS, HIDDEN, N_ACT, ATOMS, QUANTILES,
                       V_MIN, V_MAX, GAMMA, LR, SYNC, N_UPDATES, CLIP_NORM)
from oracle_dist import DistModelOracle, DistLearnerOracle  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "c51_qrdqn_update.npz")
BIG = 2048 * 8 + 3            # past one full grid (2048 blocks of 8 rows): the grid-stride loop runs
N_OF = {"c51": ATOMS, "qrdqn": QUANTILES}


def _lib():
    from xuance_b200 import _lib
    return _lib


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _greedy(z, sup=None, probs=True):
    L = _lib()
    z = _t(z)
    B, A, N = z.shape
    act = torch.full((B,), -1, dtype=torch.int64, device=DEV)
    q = torch.full((B, A), float("nan"), device=DEV)
    p = torch.full_like(z, float("nan")) if (sup is not None and probs) else None
    L.call("xb_dist_greedy", L.ptr(z), L.ptr(None if sup is None else _t(sup)), B, A, N, L.ptr(act), L.ptr(q), L.ptr(p))
    return act.cpu().numpy(), q.cpu().numpy(), None if p is None else p.cpu().numpy()


def _loss(algo, d, gamma=GAMMA, v_min=-10.0, v_max=10.0, B_total=None, rows=None):
    L = _lib()
    x = {k: _t(d[k]) for k in ("z_eval", "z_next", "actions", "rew", "ter")}
    if rows is not None:
        x = {k: v[rows].contiguous() for k, v in x.items()}
    B, A, N = x["z_eval"].shape
    grad = torch.full_like(x["z_eval"], float("nan"))
    ta = torch.full((B,), -1, dtype=torch.int64, device=DEV)
    stats = torch.full((4,), float("nan"), device=DEV)
    if algo == "c51":
        sup = supports_of(v_min, v_max, N).to(DEV)
        L.call("xb_c51_loss_fwd_bwd", L.ptr(x["z_eval"]), L.ptr(x["z_next"]), L.ptr(sup), L.ptr(x["actions"]),
               L.ptr(x["rew"]), L.ptr(x["ter"]), B, A, N, B_total or B, gamma, v_min, v_max, (v_max - v_min) / (N - 1),
               L.ptr(grad), L.ptr(ta), None, L.ptr(stats), L.ptr(L.scratch(DEV)))
    else:
        L.call("xb_qrdqn_loss_fwd_bwd", L.ptr(x["z_eval"]), L.ptr(x["z_next"]), L.ptr(x["actions"]), L.ptr(x["rew"]),
               L.ptr(x["ter"]), B, A, N, B_total or B, gamma, L.ptr(grad), L.ptr(ta), L.ptr(stats),
               L.ptr(L.scratch(DEV)))
    return grad.cpu().numpy(), ta.cpu().numpy(), stats.cpu().numpy()


# ====================================================================================================== K6Z kernels
SHAPES = [(4, 51), (18, 51), (4, 20), (18, 20), (1, 2), (256, 64), (7, 33)]
CASES = [(B, A, N) for B in (1, 255, 256, 257) for A, N in SHAPES] + [(BIG, 4, 51), (BIG, 18, 20)]


@pytest.mark.parametrize("B,A,N", CASES)
def test_greedy_matches_float64(B, A, N):
    d = loss_batch(np.random.default_rng(B % 997 + A * N), B, A, N)
    z = d["z_next"]
    sup = supports_of(-10.0, 10.0, N).numpy()
    for s in (sup, None):
        a, q, p = _greedy(z, s)
        ra, rq, rp = greedy_ref(z, s)
        np.testing.assert_allclose(q, rq, rtol=2e-5, atol=2e-5)
        if s is not None:
            np.testing.assert_allclose(p, rp, rtol=2e-5, atol=1e-7)
        # the argmax agrees wherever the float64 top-two gap is wider than float32 rounding
        srt = np.sort(rq, -1)
        clear = (srt[:, -1] - srt[:, -2] > 1e-4) if A > 1 else np.ones(B, bool)
        np.testing.assert_array_equal(a[clear], ra[clear])


@pytest.mark.parametrize("B,A,N", CASES)
def test_c51_loss_matches_float64(B, A, N):
    d = loss_batch(np.random.default_rng(B % 991 + A * N + 1), B, A, N)
    sup = supports_of(-10.0, 10.0, N).numpy()
    g, ta, st = _loss("c51", d)
    rg, rta, rl, _, _ = c51_ref(d["z_eval"], d["z_next"], sup, d["actions"], d["rew"], d["ter"], GAMMA, -10.0, 10.0, B)
    np.testing.assert_array_equal(ta, _greedy(d["z_next"], sup)[0])        # the shared routine: the same target action
    np.testing.assert_array_equal(ta, rta)
    np.testing.assert_allclose(st[0], rl, rtol=2e-5, atol=1e-6)
    assert (st[1:] == 0).all()
    np.testing.assert_allclose(g, rg, rtol=1e-4, atol=1e-4 * np.abs(rg).max())
    taken = np.zeros((B, A), bool)
    taken[np.arange(B), d["actions"].astype(int)] = True
    assert (g[~taken] == 0).all()                                          # the other actions' rows are exactly 0


@pytest.mark.parametrize("B,A,N", CASES)
def test_qrdqn_loss_matches_float64(B, A, N):
    d = loss_batch(np.random.default_rng(B % 983 + A * N + 2), B, A, N)
    g, ta, st = _loss("qrdqn", d)
    rg, rta, rl, _ = qrdqn_ref(d["z_eval"], d["z_next"], d["actions"], d["rew"], d["ter"], GAMMA, B)
    np.testing.assert_array_equal(ta, _greedy(d["z_next"])[0])
    np.testing.assert_array_equal(ta, rta)
    np.testing.assert_allclose(st[0], rl, rtol=2e-5, atol=1e-6)
    np.testing.assert_allclose(g, rg, rtol=1e-5, atol=1e-5 * np.abs(rg).max())


@pytest.mark.parametrize("N", [2, 20, 51, 64])
def test_tz_projection_and_backup_are_the_torch_expressions_bit_for_bit(N):
    """A one-hot target distribution at atom j (logits 0 there, -1e4 elsewhere: p'_j = 1 and every other p' = 0 exactly)
    makes the kernel's target_dist row j of the projection, so target_dist = torch's clamp(1 - |Tz_j - z_i| / dz, 0, 1)
    bit for bit for every i: Tz_j and the weights both.  QR: with theta_eval = 0, dq = (0 - y) * float32(2 / (B*N)), so the
    backup y is read back exactly."""
    L = _lib()
    B = 300
    rng = np.random.default_rng(N)
    v_min, v_max = -10.0, 10.0
    sup = supports_of(v_min, v_max, N)
    rew = rng.normal(0.0, 8.0, B).astype(np.float32)
    ter = (rng.random(B) < 0.3).astype(np.float32)
    rew[0], ter[0] = sup[1].item(), 1.0
    T = torch.from_numpy
    tz = torch_tz(T(rew), T(ter), sup, GAMMA, v_min, v_max)
    assert torch.equal(tz, torch_tz(_t(rew), _t(ter), sup.to(DEV), GAMMA, v_min, v_max).cpu())
    assert (tz == v_min).any() and (tz == v_max).any()
    proj = torch_projection(tz, sup, (v_max - v_min) / (N - 1)).numpy()
    assert proj[0, 0, 1] == 1.0                                             # Tz exactly on an atom
    sup_dev = sup.to(DEV)
    for j in sorted({0, 1, N // 2, N - 1}):
        zn = np.full((B, 1, N), -1e4, np.float32)
        zn[:, 0, j] = 0.0
        x = dict(z_eval=_t(np.zeros((B, 1, N), np.float32)), z_next=_t(zn), act=_t(np.zeros(B, np.float32)),
                 rew=_t(rew), ter=_t(ter))
        grad, td = torch.empty_like(x["z_eval"]), torch.full((B, N), float("nan"), device=DEV)
        ta = torch.empty(B, dtype=torch.int64, device=DEV)
        stats = torch.empty(4, device=DEV)
        L.call("xb_c51_loss_fwd_bwd", L.ptr(x["z_eval"]), L.ptr(x["z_next"]), L.ptr(sup_dev), L.ptr(x["act"]),
               L.ptr(x["rew"]), L.ptr(x["ter"]), B, 1, N, B, GAMMA, v_min, v_max, (v_max - v_min) / (N - 1),
               L.ptr(grad), L.ptr(ta), L.ptr(td), L.ptr(stats), L.ptr(L.scratch(DEV)))
        np.testing.assert_array_equal(td.cpu().numpy(), proj[:, j, :], err_msg=f"j={j}")
    th = rng.normal(0.0, 3.0, (B, 3, N)).astype(np.float32)
    d = dict(z_eval=np.zeros_like(th), z_next=th, actions=np.zeros(B, np.float32), rew=rew, ter=ter)
    g, ta, _ = _loss("qrdqn", d)
    y = torch_qr_backup(T(rew), T(ter), T(th)[np.arange(B), ta], GAMMA).numpy()
    assert torch.equal(torch_qr_backup(_t(rew), _t(ter), _t(th)[torch.arange(B), _t(ta)], GAMMA).cpu(), T(y))
    np.testing.assert_array_equal(g[:, 0], (np.float32(0) - y) * np.float32(2.0 / (B * N)))


def test_ties_pick_the_first_index():
    rng = np.random.default_rng(7)
    B, A, N = 257, 6, 51
    z = rng.normal(size=(B, A, N)).astype(np.float32)
    z[:, 1, N - 1] += 100.0              # action 1: all mass on the top atom (C51), the largest mean (QR) ...
    z[:, 3] = z[:, 1]                    # ... and the same row again at 3, 4 and (every other row) 5
    z[:, 4] = z[:, 1]
    z[::2, 5] = z[::2, 1]
    sup = supports_of(-10.0, 10.0, N).numpy()
    for s in (sup, None):
        a, q, _ = _greedy(z, s)
        assert (a == 1).all() and (q[:, 1] == q[:, 3]).all()
    d = dict(z_eval=z, z_next=z, actions=np.zeros(B, np.float32), rew=np.zeros(B, np.float32), ter=np.zeros(B, np.float32))
    assert (_loss("c51", d)[1] == 1).all() and (_loss("qrdqn", d)[1] == 1).all()


def test_nan_reaches_the_loss():
    B, A, N = 64, 4, 51
    for algo in ("c51", "qrdqn"):
        n = N if algo == "c51" else 20
        d = loss_batch(np.random.default_rng(2), B, A, n)
        d["rew"][5] = np.nan
        g, _, st = _loss(algo, d)
        assert np.isnan(st[0]) and np.isnan(g[5]).any() and np.isfinite(g[6:]).all()
        d = loss_batch(np.random.default_rng(2), B, A, n)
        d["z_eval"][9, int(d["actions"][9]), 3] = np.nan
        assert np.isnan(_loss(algo, d)[2][0])
        d = loss_batch(np.random.default_rng(2), B, A, n)
        d["z_next"][11, :, 0] = np.nan                       # a NaN Q is torch.argmax's maximum
        _, ta, st = _loss(algo, d)
        assert ta[11] == 0 and np.isnan(st[0])
        d = loss_batch(np.random.default_rng(2), B, A, n)
        d["actions"][4] = A                                  # out of range: no row selected, no read, NaN loss
        g, _, st = _loss(algo, d)
        assert np.isnan(st[0]) and (g[4] == 0).all()


@pytest.mark.parametrize("G", [2, 3, 8])
def test_sharded_minibatch_sums_to_the_unsharded_launch(G):
    B = 257
    for algo, N in (("c51", 51), ("qrdqn", 20)):
        d = loss_batch(np.random.default_rng(G), B, 4, N)
        full = _loss(algo, d)
        outs = [_loss(algo, d, B_total=B, rows=torch.from_numpy(r).to(DEV)) for r in np.array_split(np.arange(B), G)]
        np.testing.assert_array_equal(np.concatenate([o[0] for o in outs]), full[0])
        np.testing.assert_array_equal(np.concatenate([o[1] for o in outs]), full[1])
        np.testing.assert_allclose(sum(o[2] for o in outs), full[2], rtol=1e-6, atol=1e-7)


def test_launches_on_a_side_stream_equal_the_default_stream():
    """The stream handle reaches the launch whole: the three entry points on a non-default stream (as in CUDA-graph
    capture or a caller's torch.cuda.stream) give what they give on the default stream."""
    d = loss_batch(np.random.default_rng(13), 257, 4, 51)
    sup = supports_of(-10.0, 10.0, 51).numpy()
    want = (_greedy(d["z_next"], sup), _loss("c51", d), _loss("qrdqn", dict(d, z_eval=d["z_eval"][..., :20],
                                                                            z_next=d["z_next"][..., :20])))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        assert torch.cuda.current_stream().cuda_stream != 0
        got = (_greedy(d["z_next"], sup), _loss("c51", d), _loss("qrdqn", dict(d, z_eval=d["z_eval"][..., :20],
                                                                               z_next=d["z_next"][..., :20])))
    torch.cuda.synchronize()
    for w, g in zip(want, got):
        for x, y in zip(w, g):
            np.testing.assert_array_equal(x, y)


def test_statistics_are_bit_identical_from_launch_to_launch():
    for algo, N in (("c51", 51), ("qrdqn", 20)):
        d = loss_batch(np.random.default_rng(11), BIG, 4, N)
        g0, _, s0 = _loss(algo, d)
        for _ in range(2):
            g1, _, s1 = _loss(algo, d)
            assert s1.tobytes() == s0.tobytes()
            np.testing.assert_array_equal(g1, g0)


# ====================================================================================================== learners
def _product_model(algo, obs_dim, n_actions, hidden, n_atoms, v_min=V_MIN, v_max=V_MAX):
    from xuance_b200.common import Discrete
    from xuance_b200.torch.rl_models import Basic_MLP, C51DeepQNetwork, QRDeepQNetwork
    init, act = torch.nn.init.orthogonal_, torch.nn.ReLU
    rep = Basic_MLP((obs_dim,), [hidden], None, init, act, DEV)
    if algo == "c51":
        return C51DeepQNetwork(rep, [hidden], Discrete(n_actions), n_atoms, v_min, v_max, None, init, act, DEV).to(DEV)
    return QRDeepQNetwork(rep, [hidden], Discrete(n_actions), n_atoms, None, init, act, DEV).to(DEV)


def _learner_cfg(graph, **kw):
    cfg = dict(distributed_training=False, episode_length=1000, use_grad_clip=False, grad_clip_norm=0.5, device=DEV,
               model_dir="/tmp/xb_dist", running_steps=64, parallels=4, start_training=0, training_frequency=1,
               learning_rate=LR, gamma=GAMMA, sync_frequency=SYNC, end_factor_lr_decay=0.5, use_cuda_graph=graph)
    cfg.update(kw)
    return Namespace(**cfg)


def _learner(algo, model, cfg):
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import REGISTRY_Learners
    return REGISTRY_Learners["C51_Learner" if algo == "c51" else "QRDQN_Learner"](cfg, model, BaseCallback())


@pytest.mark.parametrize("algo,clip,graph", [(a, c, g) for a in ("c51", "qrdqn") for c in (False, True)
                                             for g in (False, True)])
def test_learner_matches_oracle(algo, clip, graph):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    obs_dim, A, B, H = 5, 4, 256, 64
    N = N_OF[algo]
    om = DistModelOracle(algo, obs_dim, A, N, (H,), (H,), V_MIN, V_MAX)
    model = _product_model(algo, obs_dim, A, H, N)
    model.load_state_dict(om.state_dict(), strict=True)
    lrn = _learner(algo, model, _learner_cfg(graph, use_grad_clip=clip, grad_clip_norm=0.2, sync_frequency=3))
    orc = DistLearnerOracle(om, lr=LR, gamma=GAMMA, sync_frequency=3, use_grad_clip=clip, grad_clip_norm=0.2,
                            end_factor_lr_decay=0.5, total_iters=lrn.total_iters)
    rng = np.random.default_rng(1)
    for it in range(7):
        s = {"obs": rng.normal(size=(B, obs_dim)).astype(np.float32),
             "actions": rng.integers(0, A, B).astype(np.float32),
             "obs_next": rng.normal(size=(B, obs_dim)).astype(np.float32),
             "rewards": rng.normal(0, 6, B).astype(np.float32), "terminals": (rng.random(B) < 0.2).astype(np.float32)}
        io = orc.update(**s)
        ip = lrn.update(**{k: _t(v) for k, v in s.items()})
        assert set(ip) == {"Qloss", "learning_rate"}
        assert ip["learning_rate"] == io["learning_rate"]
        np.testing.assert_allclose(ip["Qloss"], io["Qloss"], rtol=2e-4, atol=2e-5, err_msg=f"it{it}")
        if (it + 1) % 3 == 0:     # the hard copy
            for p, q in zip(model.eval_parameters(), model.target_parameters()):
                assert torch.equal(p, q)
    so, sp = om.state_dict(), model.state_dict()
    assert set(so) == set(sp)
    for k in so:
        np.testing.assert_allclose(sp[k].cpu().numpy(), so[k].numpy(), rtol=2e-3, atol=2e-4, err_msg=k)


@pytest.mark.parametrize("algo,clip", [("c51", False), ("c51", True), ("qrdqn", False), ("qrdqn", True)])
def test_learner_matches_reference_fixture(algo, clip):
    torch.backends.cuda.matmul.allow_tf32 = False
    g = np.load(GOLDEN)
    pre = f"{algo}/clip{int(clip)}/"
    model = _product_model(algo, OBS, N_ACT, HIDDEN, N_OF[algo])
    model.load_state_dict({k[len(pre + "init/"):]: torch.from_numpy(g[k]) for k in g if k.startswith(pre + "init/")},
                          strict=True)
    lrn = _learner(algo, model, _learner_cfg(False, use_grad_clip=clip, grad_clip_norm=CLIP_NORM))
    assert lrn.total_iters == int(g[pre + "total_iters"])
    rng = np.random.default_rng(80 + 2 * (algo == "qrdqn") + clip)
    for it in range(N_UPDATES):
        info = lrn.update(**{k: _t(v) for k, v in fixture_batch(rng).items()})
        np.testing.assert_allclose([info["Qloss"], info["learning_rate"]], g[pre + "infos"][it], rtol=2e-4, atol=2e-5,
                                   err_msg=f"it{it}")
        for k, v in model.state_dict().items():
            np.testing.assert_allclose(v.cpu().numpy(), g[f"{pre}it{it}/{k}"], rtol=2e-3, atol=2e-4,
                                       err_msg=f"it{it} {k}")


def test_reference_state_dict_loads_strictly_and_checkpoints_round_trip(tmp_path):
    g = np.load(GOLDEN)
    for algo in ("c51", "qrdqn"):
        pre = f"{algo}/clip0/it3/"
        ref = {k[len(pre):]: torch.from_numpy(g[k]) for k in g if k.startswith(pre)}
        assert ("supports" in ref) == (algo == "c51")
        model = _product_model(algo, OBS, N_ACT, HIDDEN, N_OF[algo])
        model.load_state_dict(ref, strict=True)
        lrn = _learner(algo, model, _learner_cfg(False))
        rng = np.random.default_rng(0)
        for _ in range(3):
            lrn.update(**{k: _t(v) for k, v in fixture_batch(rng).items()})
        path = str(tmp_path / f"{algo}.pth")
        lrn.save_model(path)
        model2 = _product_model(algo, OBS, N_ACT, HIDDEN, N_OF[algo])
        lrn2 = _learner(algo, model2, _learner_cfg(False))
        lrn2.load_model(path)
        for k, v in model.state_dict().items():
            assert torch.equal(v, model2.state_dict()[k]), k
        assert lrn.optimizer.step_count == lrn2.optimizer.step_count
        assert torch.equal(lrn.optimizer.exp_avg, lrn2.optimizer.exp_avg)


# ====================================================================================================== acting
def _agent(algo, **over):
    from xuance_b200.common import Box, Discrete
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import REGISTRY_Agents
    cfg = get_arguments(algo, "classic_control", "CartPole-v1")
    for k, v in dict(device=DEV, model_dir="/tmp/xb_models/" + algo, logger=None, buffer_size=10000, **over).items():
        setattr(cfg, k, v)
    return REGISTRY_Agents[cfg.agent](cfg, None, Box(-4, 4, (4,), np.float32), Discrete(2))


@pytest.mark.parametrize("algo", ["c51", "qrdqn"])
def test_get_actions_greedy_test_mode_and_epsilon_greedy(algo):
    agent = _agent(algo)
    assert type(agent.learner).__name__ == algo.upper() + "_Learner"
    obs = np.random.default_rng(0).normal(size=(10, 4)).astype(np.float32) * 2
    m = agent.model
    with torch.no_grad():
        z = m.forward_raw(_t(obs)).cpu().numpy()
        out = m(_t(obs))
    sup = m.supports.cpu().numpy() if algo == "c51" else None
    a, _, p = _greedy(z, sup)
    np.testing.assert_array_equal(out.actions.cpu().numpy(), a)
    want_vals = p if algo == "c51" else z
    np.testing.assert_array_equal(out.values.cpu().numpy(), want_vals)
    # under autograd the values are the reference's (torch softmax for C51) and the actions the same kernel's
    out_g = m(_t(obs))
    assert out_g.values.requires_grad and torch.equal(out_g.actions, out.actions)
    ra = greedy_ref(z, sup)[0]
    np.testing.assert_array_equal(a, ra)
    np.testing.assert_array_equal(agent.get_actions(obs, test_mode=True).env_actions, a)
    np.testing.assert_array_equal(m.greedy_actions(_t(obs)).cpu().numpy(), a)     # acting: no probabilities written
    np.testing.assert_array_equal(m.act(_t(obs)).cpu().numpy(), a)
    # epsilon-greedy: OffPolicyAgent.exploration, i.e. torch's stream
    agent.e_greedy = 0.5
    torch.manual_seed(5)
    got = agent.get_actions(obs).env_actions
    torch.manual_seed(5)
    mask = torch.rand(agent.n_envs, device=DEV) < 0.5
    rnd = torch.randint(0, 2, size=(agent.n_envs,), device=DEV)
    np.testing.assert_array_equal(got, torch.where(mask, rnd, _t(a)).cpu().numpy())
    # the target network's greedy action is the same routine on the target head
    with torch.no_grad():
        t = m.target(_t(obs))
        zt = m.target_raw(_t(obs)).cpu().numpy()
    np.testing.assert_array_equal(t.actions.cpu().numpy(), _greedy(zt, sup)[0])


# ====================================================================================================== learning
# CartPole-v1 with the shipped nested configs (10 envs, B = 256, start_training 1000, one update per vector step) for
# CARTPOLE[algo][0] training steps.  Mean score of 10 greedy test episodes before -> after, on an H100 80GB HBM3 with a
# 400 W power limit (a constant-action policy scores about 9-11):
#   C51,   40000 steps:  seed 1 66.8 -> 120.9 (the seed the test runs; 24 s),  seed 2 10.2 -> 124.3,
#                        seed 3 52.5 -> 500.0,  seed 4 39.5 -> 112.2,  seed 5 11.9 -> 129.6
#   QR-DQN, 40000 steps: seed 1 9.2 -> 231.8 (the seed the test runs; 9 s),  seed 2 8.9 -> 195.5,
#                        seed 3 9.2 -> 176.9,  seed 4 9.1 -> 201.0,  seed 5 9.7 -> 232.1
# The required scores, 80 (C51) and 100 (QR-DQN), are below the worst run of each.
CARTPOLE = {"c51": (40000, 80.0), "qrdqn": (40000, 100.0)}   # (training steps, required mean test score)


@pytest.mark.parametrize("algo", ["c51", "qrdqn"])
def test_cartpole_learns(algo):
    from xuance_b200 import get_runner
    steps, score = CARTPOLE[algo]
    runner = get_runner(algo, "classic_control", "CartPole-v1",
                        parser_args=Namespace(device=DEV, running_steps=steps, model_dir="/tmp/xb_models/%s_cp" % algo))
    agent = runner.agent
    assert agent.n_envs == 10 and type(agent.learner).__name__ == algo.upper() + "_Learner"
    before = float(np.mean(agent.test(test_episodes=10)))
    runner.run("train", running_steps=steps)
    assert {"Qloss", "learning_rate"} <= set(agent.logged)
    after = float(np.mean(agent.test(test_episodes=10)))
    runner.finish()
    print("%s cartpole before %.1f after %.1f" % (algo, before, after))
    assert after > score and after > before, (before, after)


@pytest.mark.parametrize("algo", ["c51", "qrdqn"])
def test_synthetic_atari_trains_on_the_k12_encoder(algo):
    """A SyntheticAtari agent with compute: tc trains past start_training; one update on the K12 encoder agrees with the
    same update on the fp32 encoder within the smoke test's K12 tolerance."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from xuance_b200 import get_runner
    over = dict(device=DEV, compute="tc", parallels=4, buffer_size=2000, start_training=64, running_steps=200,
                model_dir="/tmp/xb_models/%s_atari" % algo)
    runner = get_runner(algo, "atari", "SyntheticAtari", parser_args=Namespace(**over))
    agent = runner.agent
    assert agent.model.representation.compute == "tc" and agent.action_space.n == 4
    runner.run("train", running_steps=over["running_steps"])
    assert agent.learner.iterations > 0 and np.isfinite(agent.logged["Qloss"])
    # one update: K12 encoder vs the fp32 encoder, from the same weights and batch
    samples = agent.memory.sample()
    over32 = dict(over, compute="fp32", model_dir="/tmp/xb_models/%s_atari32" % algo)
    agent32 = get_runner(algo, "atari", "SyntheticAtari", parser_args=Namespace(**over32)).agent
    agent32.model.load_state_dict(agent.model.state_dict())
    lt = _learner(algo, agent.model, agent.learner.config)
    l32 = _learner(algo, agent32.model, agent32.learner.config)
    it, i32 = lt.update(**samples), l32.update(**samples)
    np.testing.assert_allclose(it["Qloss"], i32["Qloss"], rtol=1e-3, atol=1e-4)
    for (k, p), (_, q) in zip(agent32.model.state_dict().items(), agent.model.state_dict().items()):
        np.testing.assert_allclose(q.cpu().numpy(), p.cpu().numpy(), rtol=5e-3, atol=5e-4, err_msg=k)
