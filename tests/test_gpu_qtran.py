"""GPU tests of QTRAN_base / QTRAN_alt: the K9Q kernels against the float64 restatements (tests/qtran_refs.py) - select
bit for bit, the encoder and the loss within stated tolerances; shards and launch-to-launch identity; QTRAN_Learner
against the torch-CPU float64 oracle (tests/oracle_qtran.py), eager and graphed; graphed equals eager; checkpoints; and
both variants learning through REGISTRY_Agents."""
from argparse import Namespace

import numpy as np
import pytest
import torch

import qtran_refs as R
import test_qtran as T
from oracle_qtran import QTRANOracle, build_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _lib():
    from xuance_b200 import _lib as L
    return L


# ---------------------------------------------------------------- select
def _run_select(q_all, q_tgt, avail, filled, double_q):
    L = _lib()
    B, n, T1, A = q_all.shape
    T = T1 - 1
    g = torch.empty((B, n, T1), dtype=torch.int32, device=DEV)
    nx = torch.empty((B, n, T), dtype=torch.int32, device=DEV)
    fs = torch.zeros(1, device=DEV)
    L.call("xb_qtran_select", L.ptr(q_all), L.ptr(q_tgt), L.ptr(avail), A if avail is not None else 0, L.ptr(filled),
           B, n, T, A, int(double_q), L.ptr(g), L.ptr(nx), L.ptr(fs), L.ptr(L.scratch(DEV)))
    return g.cpu(), nx.cpu(), fs.cpu()


@pytest.mark.parametrize("n,A", [(n, A) for n in (1, 3, 5, 8, 32) for A in (1, 2, 9, 12, 33, 64)])
def test_select_matches_float64_bit_for_bit(n, A):
    rng = np.random.default_rng(n * 100 + A)
    for B in (1, 2, 31, 32, 33, 1024):
        for T in (1, 60):
            if B * n * (T + 1) * A > 8_000_000:
                continue
            for masked in (False, True):
                q_all = R.quantised(rng, (B, n, T + 1, A), 4.0)      # coarse grid: many ties
                q_tgt = R.quantised(rng, (B, n, T + 1, A), 4.0)
                avail = None
                if masked:
                    avail = torch.from_numpy((rng.random((B, n, T + 1, A)) < 0.6).astype(np.uint8))
                    avail[..., -1] = 1
                filled = torch.from_numpy((rng.random((B, T)) < 0.8).astype(np.float32))
                for double_q in (True, False):
                    d = lambda x: None if x is None else x.to(DEV).contiguous()
                    g, nx, fs = _run_select(d(q_all), d(q_tgt), d(avail), d(filled), double_q)
                    wg, wn = R.select_ref(q_all, q_tgt, avail, double_q)
                    assert torch.equal(g.long(), wg) and torch.equal(nx.long(), wn), (B, T, masked, double_q)
                    assert fs.item() == filled.double().sum().item()


# ---------------------------------------------------------------- encoder
def _enc_inputs(rng, B, n, T, S, H, A, int_actions):
    D = H + A
    st = R.quantised(rng, (B, T + 1, S))
    h = R.quantised(rng, (B, n, T + 1, H)) * 0.5
    mask = torch.from_numpy((rng.random((B, n, T)) < 0.8).astype(np.float32))
    acts = torch.from_numpy(rng.integers(0, A, (B, n, T)).astype(np.int32 if int_actions else np.float32))
    w1, w2 = R.quantised(rng, (D, D)) * 0.1, R.quantised(rng, (D, D)) * 0.1
    b1, b2 = R.quantised(rng, (D,)) * 0.1, R.quantised(rng, (D,)) * 0.1
    return st, h, mask, acts, w1, b1, w2, b2


ENC_SHAPES = [(1, 1, 1, 8, 4, 1, 5), (2, 3, 5, 10, 8, 6, 7), (4, 5, 12, 98, 64, 12, 9), (3, 32, 4, 20, 64, 64, 11),
              (33, 8, 3, 30, 64, 33, 13),
              (1024, 3, 60, 10, 16, 4, 17)]   # (B, n, T, S, H, A, seed); the last has 180-row weight-gradient chunks


@pytest.mark.parametrize("mode", [R.BASE, R.ALT])
@pytest.mark.parametrize("B,n,T,S,H,A,seed", ENC_SHAPES)
def test_encoder_forward_and_backward_match_float64(mode, B, n, T, S, H, A, seed):
    """Forward within 2e-5 of the largest |x|, every gradient within 2e-5 of its largest entry (float32 sums of <= 128
    products against float64).  ReLU's derivative jumps at 0: where a live agent's pre-activation lies within 1e-5 of 0,
    float32 and float64 may take different sides, so such agents (under 0.3 % of the live agent-rows) are made dead in
    the inputs; a dead agent's pre-activation W1[:, H+a] + b1 has the same sign in float32 and float64."""
    from xuance_b200.torch.rl_models.qtran import qtran_encode
    rng = np.random.default_rng(seed)
    for t0 in (0, 1):
        st, h, mask, acts, w1, b1, w2, b2 = _enc_inputs(rng, B, n, T, S, H, A, t0 == 1)
        hs = torch.cat([h[:, :, :T].double() * mask.double().unsqueeze(-1),
                        torch.nn.functional.one_hot(acts.long(), A).double()], dim=-1)
        z = torch.nn.functional.linear(hs, w1.double(), b1.double())
        near = ((z.abs() < 1e-5) & mask.bool().unsqueeze(-1)).any(-1)      # [B, n, T]
        assert near.double().mean().item() < 5e-3
        mask[near] = 0.0                  # a dead agent's pre-activation is W1[:, H+a] + b1: the same sign in both
        leaves = [x.to(DEV).requires_grad_(True) for x in (h, w1, b1, w2, b2)]
        x = qtran_encode(mode, st.to(DEV), t0, leaves[0], mask.to(DEV), acts.to(DEV), *leaves[1:])
        ref_leaves = [x_.double().requires_grad_(True) for x_ in (h, w1, b1, w2, b2)]
        xr = R.encode_ref(mode, st.double(), t0, ref_leaves[0], mask.double(), acts, *ref_leaves[1:])
        scale = xr.abs().max().item()
        np.testing.assert_allclose(x.detach().cpu().double().numpy(), xr.detach().numpy(), rtol=0, atol=2e-5 * scale)
        dx = R.quantised(rng, tuple(x.shape))
        x.backward(dx.to(DEV))
        xr.backward(dx.double())
        for got, want in zip(leaves, ref_leaves):
            w = want.grad.numpy()
            np.testing.assert_allclose(got.grad.cpu().double().numpy(), w, rtol=0, atol=2e-5 * max(np.abs(w).max(), 1e-3))
        assert not leaves[0].grad[:, :, T].any()                               # step T feeds no encoding


def test_encoder_backward_is_bit_identical_across_launches():
    from xuance_b200.torch.rl_models.qtran import qtran_encode
    rng = np.random.default_rng(3)
    st, h, mask, acts, w1, b1, w2, b2 = _enc_inputs(rng, 32, 5, 60, 98, 64, 12, False)
    dx = None
    outs = []
    for _ in range(3):
        leaves = [x.to(DEV).requires_grad_(True) for x in (h, w1, b1, w2, b2)]
        x = qtran_encode(R.ALT, st.to(DEV), 0, leaves[0], mask.to(DEV), acts.to(DEV), *leaves[1:])
        if dx is None:
            dx = torch.randn_like(x)
        x.backward(dx)
        outs.append([x.detach().clone()] + [l.grad.clone() for l in leaves])
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert torch.equal(a, b)


# ---------------------------------------------------------------- loss
def _loss_inputs(rng, mode, B, n, T, A):
    q_all = R.quantised(rng, (B, n, T + 1, A), 8.0)
    actions = torch.from_numpy(rng.integers(0, A, (B, n, T)).astype(np.float32))
    greedy = torch.from_numpy(rng.integers(0, A, (B, n, T + 1)).astype(np.int32))
    same = torch.from_numpy(rng.random((B, n, T)) < 0.3)
    greedy[:, :, :T][same] = actions.int()[same]                              # g = a: both contributions add
    nxt = torch.from_numpy(rng.integers(0, A, (B, n, T)).astype(np.int32))
    mask = torch.from_numpy((rng.random((B, n, T)) < 0.8).astype(np.float32))
    filled = torch.from_numpy((rng.random((B, T)) < 0.85).astype(np.float32))
    filled[0, 0] = 1.0
    rewards = R.quantised(rng, (B, n, T), 4.0)
    terminals = torch.from_numpy((rng.random((B, n, T)) < 0.2).astype(np.float32))
    rows = B * T * n if mode == R.ALT else B * T
    shape = (rows, A) if mode == R.ALT else (rows,)
    qjt, qjt_g, qjt_n = (R.quantised(rng, shape, 8.0) for _ in range(3))
    v = R.quantised(rng, (B * T,), 8.0)
    return q_all, actions, greedy, nxt, mask, filled, rewards, terminals, qjt, qjt_g, qjt_n, v


def _run_loss(mode, ins, gamma, lo, ln, filled_sum=None, rows_total=None):
    L = _lib()
    q_all, actions, greedy, nxt, mask, filled, rewards, terminals, qjt, qjt_g, qjt_n, v = [x.to(DEV).contiguous() for x in ins]
    B, n, T1, A = q_all.shape
    T = T1 - 1
    fs = torch.tensor([filled.sum().item() if filled_sum is None else filled_sum], device=DEV)
    dqjt, dv, dq = torch.empty_like(qjt), torch.empty_like(v), torch.zeros_like(q_all)
    stats = torch.zeros(5, device=DEV)
    L.call("xb_qtran_loss_fwd_bwd", mode, L.ptr(q_all), L.ptr(actions), L.ptr(greedy), L.ptr(nxt), L.ptr(mask),
           L.ptr(filled), L.ptr(rewards), L.ptr(terminals), L.ptr(qjt), L.ptr(qjt_g), L.ptr(qjt_n), L.ptr(v), L.ptr(fs),
           B, n, T, A, gamma, lo, ln, B * T if rows_total is None else rows_total, L.ptr(dqjt), L.ptr(dv), L.ptr(dq),
           L.ptr(stats), L.ptr(L.scratch(DEV)))
    return stats.cpu().double(), dq.cpu().double(), dqjt.cpu().double(), dv.cpu().double()


@pytest.mark.parametrize("mode", [R.BASE, R.ALT])
@pytest.mark.parametrize("B,n,T,A", [(1, 1, 1, 1), (2, 1, 5, 4), (3, 3, 7, 1), (4, 5, 12, 12), (2, 32, 3, 64),
                                     (33, 8, 4, 9)])
def test_loss_matches_float64_autograd(mode, B, n, T, A):
    """Statistics within 1e-6 relative, gradients within 1e-6 of their largest entry (float64 inside, float32 out)."""
    rng = np.random.default_rng(B * 1000 + n * 10 + A)
    ins = _loss_inputs(rng, mode, B, n, T, A)
    got = _run_loss(mode, ins, 0.99, 1.0, 0.5)
    q_all, actions, greedy, nxt, mask, filled, rewards, terminals, qjt, qjt_g, qjt_n, v = ins
    want = R.loss_grads(mode, q_all, actions, greedy, nxt, mask, filled, rewards, terminals, qjt, qjt_g, qjt_n, v,
                        np.float32(0.99).item(), 1.0, 0.5)
    np.testing.assert_allclose(got[0].numpy(), want[0].numpy(), rtol=1e-6, atol=1e-7)
    for g, w in zip(got[1:], want[1:]):
        w = w.reshape(g.shape).numpy()
        np.testing.assert_allclose(g.numpy(), w, rtol=0, atol=1e-6 * max(np.abs(w).max(), 1e-6))


@pytest.mark.parametrize("G", [2, 3, 8])
@pytest.mark.parametrize("mode", [R.BASE, R.ALT])
def test_loss_shards_sum_to_the_full_batch(G, mode):
    rng = np.random.default_rng(G + 10 * mode)
    B, n, T, A = 24, 5, 6, 12
    ins = _loss_inputs(rng, mode, B, n, T, A)
    full = _run_loss(mode, ins, 0.99, 1.0, 1.0)
    fs = ins[5].sum().item()
    per = B // G
    rows = lambda b0, b1: T * (n if mode == R.ALT else 1) * np.array([b0, b1])
    tot = torch.zeros(5, dtype=torch.float64)
    for s in range(G):
        b0, b1 = s * per, (s + 1) * per
        sl = []
        for k, x in enumerate(ins):
            if k >= 8:                                  # qjt, qjt_g, qjt_n, v: rows b*T(+i)
                r0, r1 = rows(b0, b1) if k < 11 else (b0 * T, b1 * T)
                sl.append(x[r0:r1])
            else:
                sl.append(x[b0:b1])
        out = _run_loss(mode, sl, 0.99, 1.0, 1.0, filled_sum=fs, rows_total=B * T)
        tot += out[0]
        np.testing.assert_allclose(out[1].numpy(), full[1][b0:b1].numpy(), rtol=0, atol=0)
    np.testing.assert_allclose(tot.numpy(), full[0].numpy(), rtol=1e-6, atol=1e-7)


def test_select_and_loss_are_bit_identical_across_launches():
    rng = np.random.default_rng(11)
    B, n, T, A = 32, 5, 60, 12
    q_all, q_tgt = (R.quantised(rng, (B, n, T + 1, A), 4.0).to(DEV) for _ in range(2))
    avail = torch.from_numpy((rng.random((B, n, T + 1, A)) < 0.6).astype(np.uint8))
    avail[..., -1] = 1
    filled = torch.from_numpy((rng.random((B, T)) < 0.8).astype(np.float32)).to(DEV)
    sel = [_run_select(q_all, q_tgt, avail.to(DEV), filled, False) for _ in range(3)]
    for mode in (R.BASE, R.ALT):
        ins = _loss_inputs(rng, mode, B, n, T, A)
        outs = [_run_loss(mode, ins, 0.99, 1.0, 1.0) for _ in range(3)]
        for o in outs[1:]:
            for a, b in zip(outs[0], o):
                assert torch.equal(a, b)
    for o in sel[1:]:
        for a, b in zip(sel[0], o):
            assert torch.equal(a, b)


# ---------------------------------------------------------------- learner
def _product_model(agent, n, obs_dim, A, S, hid=32, qhid=32):
    return build_model(agent, n, obs_dim, A, S, hid, qhid, DEV)


def _learner(grouping, model, **over):
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import QTRAN_Learner
    cfg = dict(device=DEV, model_dir="/tmp/xb200_qtran_models", use_cuda_graph=False, use_grad_clip=True,
               grad_clip_norm=0.5, parallels=4, running_steps=100000, start_training=0, use_rnn=True,
               use_actions_mask=True, learning_rate=7e-4, sync_frequency=2, gamma=0.99, end_factor_lr_decay=0.5,
               use_linear_lr_decay=True, agent="QTRAN_base", double_q=True, lambda_opt=1.0, lambda_nopt=1.0)
    cfg.update(over)
    return QTRAN_Learner(Namespace(**cfg), grouping, model, BaseCallback())


def _sample(rng, keys, B, T, obs_dim, A, S):
    from wqmix_refs import fix_sample
    return fix_sample(rng, keys, B=B, T=T, obs_dim=obs_dim, A=A, S=S)


INFO_KEYS = ("loss_td", "loss_opt", "loss_nopt", "loss", "Q_joint")


def _run(agent, double_q, use_graph, updates=3, seed=0):
    _no_tf32()
    torch.manual_seed(seed)
    n, obs_dim, A, S, T, B = 4, 20, 7, 10, 12, 6
    keys, grouping, model = _product_model(agent, n, obs_dim, A, S)
    lrn = _learner(grouping, model, agent=agent, double_q=double_q, use_cuda_graph=use_graph, episode_length=T)
    rng = np.random.default_rng(seed + 1)
    out = []
    for _ in range(updates):
        s = _sample(rng, keys, B, T, obs_dim, A, S)
        orc = QTRANOracle(model, double_q=double_q, gamma=0.99)
        want, grads = orc.losses(s), orc.grads(s)
        out.append((lrn.update(s), want, grads))
    return model, lrn, out


@pytest.mark.parametrize("agent", ["QTRAN_base", "QTRAN_alt"])
@pytest.mark.parametrize("double_q", [True, False])
@pytest.mark.parametrize("use_graph", [False, True])
def test_learner_matches_the_oracle(agent, double_q, use_graph):
    """Every update's five statistics against the float64 oracle on the same parameters (within 1e-4 relative)."""
    _, _, out = _run(agent, double_q, use_graph)
    for it, (info, want, _) in enumerate(out):
        np.testing.assert_allclose([info[k] for k in INFO_KEYS], want, rtol=1e-4, atol=1e-6, err_msg=f"it{it}")


@pytest.mark.parametrize("agent", ["QTRAN_base", "QTRAN_alt"])
def test_learner_gradient_matches_the_oracle(agent):
    """The gradient of one update, read from the optimiser's flat bucket before the step, against the oracle's."""
    _no_tf32()
    torch.manual_seed(2)
    n, obs_dim, A, S, T, B = 3, 12, 6, 8, 9, 5
    keys, grouping, model = _product_model(agent, n, obs_dim, A, S)
    lrn = _learner(grouping, model, agent=agent, episode_length=T)
    s = _sample(np.random.default_rng(5), keys, B, T, obs_dim, A, S)
    want = QTRANOracle(model).grads(s)
    d = lrn._stacked(s)
    lrn.optimizer.prepare()
    lrn.optimizer.zero_grad()
    args = [d[k] for k in ("obs", "actions", "rewards", "terminals", "agent_mask", "filled", "state")] + [d["avail"]]
    orig = lrn.optimizer.launch
    lrn.optimizer.launch = lambda **kw: None                     # keep the gradient, skip the step
    try:
        lrn._device_update(*args)
    finally:
        lrn.optimizer.launch = orig
    names = {id(p): k for k, p in model.named_parameters()}
    for p in model.parameters_model:
        w = want[names[id(p)]].numpy()
        g = p.grad.detach().cpu().double().numpy()
        np.testing.assert_allclose(g, w, rtol=0, atol=1e-4 * max(np.abs(w).max(), 1e-3), err_msg=names[id(p)])


def test_graphed_update_is_bit_equal_to_eager():
    m_e, _, o_e = _run("QTRAN_alt", False, False, updates=3, seed=4)
    m_g, _, o_g = _run("QTRAN_alt", False, True, updates=3, seed=4)
    for (a, _, _), (b, _, _) in zip(o_e, o_g):
        assert a == b
    for (k, v), (_, w) in zip(m_e.state_dict().items(), m_g.state_dict().items()):
        assert torch.equal(v, w), k


def test_checkpoint_round_trip(tmp_path):
    _no_tf32()
    torch.manual_seed(1)
    rng = np.random.default_rng(1)
    keys, grouping, model = _product_model("QTRAN_base", 3, 12, 7, 10)
    lrn = _learner(grouping, model, end_factor_lr_decay=1.0, episode_length=8)
    samples = [_sample(rng, keys, 6, 8, 12, 7, 10) for _ in range(3)]
    for s in samples[:2]:
        lrn.update(s)
    path = str(tmp_path / "qtran.pth")
    lrn.save_model(path)
    _, grouping2, model2 = _product_model("QTRAN_base", 3, 12, 7, 10)
    lrn2 = _learner(grouping2, model2, end_factor_lr_decay=1.0, episode_length=8)
    lrn2.load_model(path)
    lrn2.iterations = lrn.iterations
    for (k, v), (_, w) in zip(model.state_dict().items(), model2.state_dict().items()):
        assert torch.equal(v, w), k
    assert lrn.update(samples[2]) == lrn2.update(samples[2])


def _agent_config(**over):
    from xuance_b200.common.common_tools import get_arguments
    cfg = get_arguments("qtran", "sc2", "3m")
    base = dict(vectorize="Dummy_StarCraft2", parallels=8, buffer_size=64, batch_size=16, learning_rate=2e-3, gamma=0.5,
                start_greedy=1.0, end_greedy=0.05, decay_step_greedy=12000, start_training=200, running_steps=40000,
                n_epochs=4, sync_frequency=20, device=DEV, model_dir="/tmp/xb200_qtran_models",
                log_dir="/tmp/xb200_qtran_logs", episode_limit=20, p_death=0.02, distributed_training=False,
                use_cuda_graph=False)
    base.update(over)
    for k, v in base.items():
        setattr(cfg, k, v)
    return cfg


@pytest.mark.parametrize("agent", ["QTRAN_base", "QTRAN_alt"])
def test_qtran_learns_through_the_agent_registry(agent):
    """REGISTRY_Agents["QTRAN_base"] / ["QTRAN_alt"] on the cue-following SMAC-shaped env (3m): the greedy team score
    rises."""
    from xuance_b200.environment import make_envs
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.rl_models import QTranMixingNetwork
    cfg = _agent_config(agent=agent)
    envs = make_envs(cfg)
    ag = REGISTRY_Agents[agent](cfg, envs)
    assert isinstance(ag.model, QTranMixingNetwork) and ag.use_actions_mask
    before = float(np.mean(ag.test(16, make_envs(cfg))))
    info = ag.train(cfg.running_steps // cfg.parallels)
    assert set(INFO_KEYS) <= set(info) and np.isfinite(info["loss"])
    after = float(np.mean(ag.test(32, make_envs(cfg))))
    assert after > before + 2.0, (before, after)
    ag.finish()


# ---------------------------------------------------------------- against the reference fixture (tests/golden/qtran_update.npz)
@pytest.mark.parametrize("agent,double_q", T.FIX_CASES)
@pytest.mark.parametrize("use_graph", [False, True])
def test_learner_reproduces_the_reference_fixture(agent, double_q, use_graph):
    """A reference state_dict loads strictly; every update's logged values within 1e-4 relative of the reference and
    the whole state_dict after the target sync and after the last update within 2e-5 + 1e-4 relative."""
    _no_tf32()
    d = np.load(T.GOLDEN)
    pre = f"{agent}/dq{int(double_q)}/"
    keys, grouping, model = _product_model(agent, T.FIX_N, T.FIX_OBS, T.FIX_A, T.FIX_S, T.FIX_HID, T.FIX_QH)
    model.load_state_dict(T.fixture_init(d, pre), strict=True)
    lrn = _learner(grouping, model, agent=agent, double_q=double_q, use_cuda_graph=use_graph, episode_length=8,
                   use_grad_clip=False)
    assert lrn.total_iters == int(d[pre + "total_iters"])
    for it in range(T.FIX_UPDATES):
        info = lrn.update(T.fixture_sample(d, pre, it, keys))
        np.testing.assert_allclose([info[k] for k in T.FIX_INFO_KEYS], d[pre + "infos"][it], rtol=1e-4, atol=1e-6,
                                   err_msg=f"{pre}it{it}")
        if it in T.FIX_SNAPSHOTS:
            flat = np.concatenate([v.cpu().numpy().reshape(-1) for v in model.state_dict().values()])
            np.testing.assert_allclose(flat, d[f"{pre}after{it}"], rtol=1e-4, atol=2e-5, err_msg=f"{pre}after{it}")
