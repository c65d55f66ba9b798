"""CPU: the float64 kernel references of tests/kernel_refs.py agree with the oracle's torch formulas (oracle/), so that the
GPU edge tests (tests/test_gpu_kernel_edges.py) compare the kernels with pinned references.  The oracle learners run on
stub models whose outputs are the kernels' inputs: their autograd gradients at those outputs are what the kernels write."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import kernel_refs as kr
from oracle.learners import ppo_clip_terms, DQNLearnerOracle
from oracle.qmix import MixerOracle, QMIXLearnerOracle
from oracle.sac import SACLearnerOracle, SACModelOracle

D = torch.float64
close = lambda got, want, tol=1e-12: np.testing.assert_allclose(got, want, rtol=tol, atol=tol)


def _param(x, dtype=D):
    return nn.Parameter(torch.tensor(np.asarray(x), dtype=dtype))


@pytest.mark.parametrize("loss_kind", [0, 1])
def test_ppo_reference_matches_oracle_autograd(loss_kind):
    rng = np.random.default_rng(loss_kind)
    B, A, clip, vf, ent = 64, 5, 0.25, 0.25, 0.01            # clip exact in float32: the kernel's bounds are float32
    logits = (rng.normal(size=(B, A)) * 3).astype(np.float32)
    act = rng.integers(0, A, B).astype(np.float32)
    lp = kr._log_softmax(logits)[np.arange(B), act.astype(int)]
    ratio = np.concatenate([rng.uniform(0.5, 0.74, B // 4), rng.uniform(0.76, 1.24, B // 4),
                            rng.uniform(1.26, 2.0, B // 4), np.ones(B - 3 * (B // 4))])
    old = (lp - np.log(ratio)).astype(np.float32)
    adv = rng.normal(size=B).astype(np.float32)
    adv[::7] = 0.0
    v, ret = rng.normal(size=B).astype(np.float32), rng.normal(size=B).astype(np.float32)
    tz, tv = _param(logits), _param(v)
    a_t, adv_t, ret_t = torch.tensor(act, dtype=D), torch.tensor(adv, dtype=D), torch.tensor(ret, dtype=D)
    if loss_kind == 0:
        a_loss, c_loss, e_loss, r = ppo_clip_terms(tz, tv, a_t, ret_t, adv_t, torch.tensor(old, dtype=D), clip)
        r = r.detach().numpy()
        cf = ((r < 1 - clip).sum() + (r > 1 + clip).sum()) / B           # PPOLearnerOracle's clip_ratio
    else:                                                                 # the A2C branch of PPOLearnerOracle.update
        dist = torch.distributions.Categorical(logits=tz)
        a_loss = -(adv_t * dist.log_prob(a_t)).mean()
        c_loss, e_loss, cf = nn.functional.mse_loss(tv, ret_t), dist.entropy().mean(), 0.0
    loss = a_loss - ent * e_loss + vf * c_loss
    loss.backward()
    dz, dv, st = kr.ppo_loss(logits, v, act, old, adv, ret, B, np.float32(clip), vf, ent, loss_kind)
    close(dz, tz.grad.numpy())
    close(dv, tv.grad.numpy())
    # ppo_clip_terms rounds the ratio to float32 (ppo_learner.py's .float()), so the surrogate agrees to float32 precision
    close(st, [a_loss.item(), c_loss.item(), e_loss.item(), v.astype(np.float64).mean(), cf, loss.item()], tol=4 * kr.EPS32)


class _Stub(nn.Module):
    """A 'network' whose output is a given tensor: forward(key) returns self.out[key]."""

    def __init__(self, **outs):
        super().__init__()
        self.out = nn.ParameterDict({k: _param(v, torch.float32) for k, v in outs.items()})

    def forward(self, key):
        return self.out[str(int(np.asarray(key).reshape(-1)[0]))]


@pytest.mark.parametrize("double_q", [False, True])
def test_dqn_reference_matches_oracle_learner(double_q):
    rng = np.random.default_rng(3)
    B, A = 40, 4
    qe, qn = rng.normal(size=(B, A)).astype(np.float32), rng.normal(size=(B, A)).astype(np.float32)
    qs = rng.integers(0, 3, size=(B, A)).astype(np.float32)              # duplicated maxima in most rows
    act, rew = rng.integers(0, A, B).astype(np.float32), rng.normal(size=B).astype(np.float32)
    ter = (rng.random(B) < 0.3).astype(np.float32)
    model = _Stub(**{"0": qe, "1": qs})
    model.target = _Stub(**{"1": qn})
    orc = DQNLearnerOracle(model, gamma=0.99, double_q=double_q)
    info = orc.update(obs=np.zeros(1), actions=act, obs_next=np.ones(1), rewards=rew, terminals=ter)
    dq, td32, td, st = kr.dqn_td(qe, qn, qs if double_q else None, act, rew, ter, B, 0.99)
    grad = model.out["0"].grad.numpy()
    np.testing.assert_allclose(dq, grad, rtol=4 * kr.EPS32, atol=1e-9)   # torch's gradient is float32
    np.testing.assert_allclose(st, [info["Qloss"], info["predictQ"]], rtol=1e-6)
    # the float32 restatement is torch's float32 expression of dqn_learner.py, bit for bit
    tq = torch.from_numpy(qn)
    mx = tq.max(-1).values if not double_q else tq.gather(-1, torch.from_numpy(qs).argmax(-1, keepdim=True))[:, 0]
    y = torch.from_numpy(rew) + 0.99 * (1 - torch.from_numpy(ter)) * mx
    assert np.array_equal(td32, (y - torch.from_numpy(qe).gather(-1, torch.from_numpy(act).long()[:, None])[:, 0]).numpy())
    np.testing.assert_allclose(td, td32, rtol=0, atol=8 * kr.EPS32 * 4)


def test_sac_reference_matches_oracle_learner():
    rng = np.random.default_rng(4)
    B, alpha, gamma = 48, 0.37, 0.99
    lp, q1, q2 = (rng.normal(size=(3, B)) * 2).astype(np.float32)
    q2[::3] = q1[::3]                                                      # torch.min ties
    aq1, aq2, tq, lpn, rew = rng.normal(size=(5, B)).astype(np.float32)
    ter = (rng.random(B) < 0.3).astype(np.float32)

    class M(nn.Module):
        def __init__(self):
            super().__init__()
            self.actor, self.critic = _Stub(**{"0": lp}), _Stub(**{"0": aq1, "1": aq2})
            self.q_pol = _Stub(**{"0": q1, "1": q2})
            self.target_critic = _Stub(**{"0": aq1, "1": aq2})

        def Qpolicy(self, obs, noise):
            return self.actor(0), self.q_pol(0), self.q_pol(1)

        def Qaction(self, obs, act):
            return self.critic(0), self.critic(1)

        def Qtarget(self, obs, noise):
            return torch.from_numpy(lpn), torch.from_numpy(tq)

        def soft_update(self, tau):
            pass

    m = M()
    info = SACLearnerOracle(m, alpha=alpha, gamma=gamma, auto_alpha=False).update(
        None, None, obs=np.zeros(1), actions=np.zeros(1), obs_next=np.zeros(1), rewards=rew, terminals=ter)
    dlp, dq1, dq2, st = kr.sac_actor(lp, q1, q2, alpha, B)
    g = lambda mod, k: mod.out[k].grad.numpy()
    np.testing.assert_allclose(dlp, g(m.actor, "0"), rtol=4 * kr.EPS32)
    assert np.array_equal(dq1 != 0, g(m.q_pol, "0") != 0) and np.array_equal(dq2 != 0, g(m.q_pol, "1") != 0)
    np.testing.assert_allclose(dq1, g(m.q_pol, "0"), rtol=4 * kr.EPS32)      # 1/2 - 1/2 on the tied rows
    np.testing.assert_allclose(dq2, g(m.q_pol, "1"), rtol=4 * kr.EPS32)
    np.testing.assert_allclose(st[:2], [info["Ploss"], info["Qvalue"]], rtol=1e-6)
    cq1, cq2, y, cst = kr.sac_critic(aq1, aq2, tq, lpn, rew, ter, alpha, gamma, B)
    np.testing.assert_allclose(cst, [info["Qloss"]], rtol=1e-6)
    np.testing.assert_allclose(cq1, g(m.critic, "0"), rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(cq2, g(m.critic, "1"), rtol=1e-5, atol=1e-7)
    # float32 backup = oracle/sac.py's expression in float32, bit for bit
    tv = torch.from_numpy(tq) - alpha * torch.from_numpy(lpn)
    want = torch.from_numpy(rew) + (1 - torch.from_numpy(ter)) * gamma * tv
    assert np.array_equal(kr.sac_backup_f32(tq, lpn, rew, ter, alpha, gamma), want.numpy())


def test_soft_update_restatement_is_the_oracle_soft_update():
    rng = np.random.default_rng(5)
    t, s = rng.normal(size=(2, 1001)).astype(np.float32)
    stub = nn.Module()
    stub.critic, stub.target_critic = _Stub(**{"0": s}), _Stub(**{"0": t})
    SACModelOracle.soft_update(stub, 0.005)
    assert np.array_equal(kr.soft_update_f32(t, s, 0.005), stub.target_critic.out["0"].detach().numpy())


@pytest.mark.parametrize("double_q,mask", [(True, False), (False, False), (True, True)])
def test_qmix_references_match_oracle_learner(double_q, mask):
    rng = np.random.default_rng(6)
    B, n, T, A = 3, 4, 5, 6
    keys = [f"agent_{i}" for i in range(n)]
    q_all = rng.integers(-2, 3, size=(B, n, T + 1, A)).astype(np.float32)   # ties in the double-Q arg-max
    q_tgt = rng.normal(size=(B, n, T + 1, A)).astype(np.float32)
    actions = rng.integers(0, A, size=(B, n, T)).astype(np.float32)
    rewards = rng.normal(size=(B, n, T)).astype(np.float32)
    terminals = rng.random((B, n, T)) < 0.5
    terminals[0, :, 1] = True                                              # one team-terminal step
    agent_mask = (rng.random((B, n, T)) < 0.8).astype(np.float32)
    filled = (rng.random((B, T)) < 0.8).astype(np.float32)
    avail = (rng.random((B, n, T + 1, A)) < 0.6).astype(np.uint8)
    avail[0, 0, 2] = 0                                                     # nothing available
    wmix = rng.normal(size=n).astype(np.float32)
    seen = {}

    class Mixer(nn.Module):
        def __init__(self, name):
            super().__init__()
            self.name, self.b = name, nn.Parameter(torch.zeros(B * T))

        def forward(self, values, state):
            if values.requires_grad:
                values.retain_grad()
            seen[self.name] = values
            return (values * torch.from_numpy(wmix)).sum(1) + self.b

    class Q(nn.Module):
        def __init__(self, x):
            super().__init__()
            self.x = nn.Parameter(torch.tensor(x).reshape(B * n, T + 1, A))     # a copy: the Adam step moves it

        def forward(self, packed):
            return self.x

    class Model(nn.Module):
        def __init__(self):
            super().__init__()
            self.individual_q_networks = nn.ModuleDict({"shared": Q(q_all)})
            self.target_individual_q_networks = nn.ModuleDict({"shared": Q(q_tgt)})
            self.eval_Qtot, self.target_Qtot = Mixer("eval"), Mixer("target")

        def parameters_model(self):
            return list(self.individual_q_networks.parameters()) + list(self.eval_Qtot.parameters())

    model = Model()
    per = lambda x: {k: x[:, i] for i, k in enumerate(keys)}
    sample = dict(batch_size=B, sequence_length=T, obs=per(np.zeros((B, n, T + 1, 1), np.float32)), actions=per(actions),
                  rewards=per(rewards), terminals=per(terminals), agent_mask=per(agent_mask), filled=filled,
                  state=np.zeros((B, T + 1, 1), np.float32), avail_actions=per(avail))
    info = QMIXLearnerOracle(model, keys, double_q=double_q, detach_q_eval=False, use_actions_mask=mask,
                             sync_frequency=100).update(sample)
    qe_t, qn_t, fs = kr.qmix_select(q_all, q_tgt, actions, agent_mask, filled, avail if mask else None, double_q)
    assert np.array_equal(qe_t, seen["eval"].detach().numpy())
    assert np.array_equal(qn_t, seen["target"].detach().numpy())
    assert fs == filled.sum()
    q_tot = seen["eval"].detach().numpy() @ wmix.astype(np.float64)
    q_tot_next = seen["target"].detach().numpy() @ wmix.astype(np.float64)
    dq_tot, st = kr.qmix_td(q_tot, q_tot_next, rewards, terminals, filled, fs, 0.99, B * T)
    np.testing.assert_allclose(st, [info["loss_Q"], info["predictQ"]], rtol=1e-5)
    np.testing.assert_allclose(dq_tot, model.eval_Qtot.b.grad.numpy(), rtol=1e-5, atol=1e-7)
    dq_all = kr.qmix_select_bwd(seen["eval"].grad.numpy(), actions, agent_mask, filled, A)
    assert np.array_equal(dq_all, model.individual_q_networks["shared"].x.grad.numpy().reshape(B, n, T + 1, A))


@pytest.mark.parametrize("n,H", [(3, 8), (9, 5)])
def test_mixer_reference_matches_oracle_mixer(n, H):
    """MixerOracle runs in float32 (it casts the states), so the float64 reference of its epilogue agrees to float32
    rounding of sums of n and H terms."""
    torch.manual_seed(n)
    R, S = 17, 7
    om = MixerOracle(S, H, 6, n)
    q = torch.randn(R, n, requires_grad=True)
    st = torch.randn(R, S)
    g = torch.randn(R)
    y = om(q, st).view(-1)
    y.backward(g)
    with torch.no_grad():
        w1, b1, w2, b2 = om.hyper_w_1(st), om.hyper_b_1(st), om.hyper_w_2(st), om.hyper_b_2(st)
    q_tot, dq, _, _, _ = kr.qmix_mix(q.detach().numpy(), w1.numpy(), b1.numpy(), w2.numpy(), b2.numpy(), g.numpy(), n, H)
    close(q_tot, y.detach().numpy(), tol=1e-5)
    close(dq, q.grad.numpy(), tol=1e-5)


@pytest.mark.parametrize("max_norm", [0.0625, 128.0, 0.0])      # exact in float32, as the kernel takes it
def test_adam_and_norm_references_match_torch(max_norm):
    rng = np.random.default_rng(7)
    b1, b2, eps, lr = 0.875, 0.998046875, 2.0 ** -17, 1e-3                  # exact in float32
    p0 = rng.normal(size=37)
    p = torch.tensor(p0, requires_grad=True)
    opt = torch.optim.Adam([p], lr=lr, betas=(b1, b2), eps=eps)
    rp, rm, rv = p0.copy(), np.zeros(37), np.zeros(37)
    for t in range(1, 4):
        g = (rng.normal(size=37) * 0.01).astype(np.float32)
        p.grad = torch.tensor(g, dtype=D)
        norm = kr.grad_norm(g, 1.0)
        close(norm, torch.linalg.vector_norm(p.grad).item())
        if max_norm > 0:
            torch.nn.utils.clip_grad_norm_([p], max_norm)
        opt.step()
        rp, _, rm, rv = kr.adam_step(rp, g, rm, rv, lr / (1 - b1 ** t), np.sqrt(1 - b2 ** t), b1, b2, eps,
                                     kr.adam_coef(norm, max_norm, 1.0))
        close(rp, p.detach().numpy())
        close(rm, opt.state[p]["exp_avg"].numpy())
        close(rv, opt.state[p]["exp_avg_sq"].numpy())


def test_advantage_statistics_match_the_oracle_buffer():
    from oracle.onpolicy import OnPolicyBufferOracle
    rng = np.random.default_rng(8)
    buf = OnPolicyBufferOracle((1,), (), {}, 4, 50)
    buf.size = buf.n_size
    buf.advantages[:] = (rng.normal(size=(4, 50)) * 3 + 0.5).astype(np.float32)
    idx = rng.permutation(200)[:128]
    want = buf.sample(idx)["advantages"]
    x = buf.advantages.reshape(-1)[idx]
    mean, std = kr.adv_stats(x)
    close(mean, np.mean(x.astype(np.float64)))
    close(std, np.std(x.astype(np.float64)))
    # the float32 restatement with float32-rounded statistics stays within a few ulp of the oracle's float32 arithmetic
    got = kr.adv_normalize_f32(x, [mean, std])
    np.testing.assert_allclose(got, want, rtol=0, atol=8 * kr.EPS32 * (np.abs(x).max() + abs(mean)) / std)
