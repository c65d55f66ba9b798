"""GPU parity: QMIX episode replay (bit-exact), K9 mixer / selection / TD kernels and QMIX_Learner.update vs the oracle."""
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn as nn

from helpers import qmix_episode_stream
from oracle.qmix import QMIXModelOracle, QMIXLearnerOracle, EpisodeReplayOracle, MixerOracle

pytestmark = pytest.mark.gpu


def _product_model(n, obs_dim, A, S, device="cuda:0"):
    from xuance_b200.common import AgentGrouping, Discrete
    from xuance_b200.torch.rl_models import (Basic_RNN, AgentFeatureEncoder, DiscreteActionValueCritic, QMIX_Mixer,
                                             MixingQNetwork)
    keys = [f"agent_{i}" for i in range(n)]
    rep = Basic_RNN(input_shape=(obs_dim,), hidden_sizes=None, initialize=nn.init.orthogonal_, activation=nn.ReLU,
                    device=device, fc_hidden_sizes=[64], recurrent_hidden_size=64, N_recurrent_layers=1, dropout=0, rnn='GRU')
    q = nn.ModuleDict({'shared': DiscreteActionValueCritic(AgentFeatureEncoder(rep), Discrete(A), [64], None,
                                                           nn.init.orthogonal_, nn.ReLU, device)})
    grouping = AgentGrouping.shared(keys)
    return keys, grouping, MixingQNetwork(grouping, q, QMIX_Mixer(S, 32, 32, n, device), use_rnn=True, device=device).to(device)


def _buffers(keys, obs_dim, A, S, n_envs, C, Be, T, device="cuda:0"):
    from xuance_b200.common import MARL_OffPolicyBuffer_RNN, Box, Discrete
    prod = MARL_OffPolicyBuffer_RNN(agent_keys=keys, state_space=Box(-1, 1, (S,)),
                                    obs_space={k: Box(-1, 1, (obs_dim,)) for k in keys},
                                    act_space={k: Discrete(A) for k in keys}, n_envs=n_envs, buffer_size=C,
                                    batch_size=Be, max_episode_steps=T, device=device)
    return prod, EpisodeReplayOracle(keys, obs_dim, S, n_envs, C, Be, T)


@pytest.mark.parametrize("T", [12, 61])
def test_episode_replay_bit_exact(T):
    n, obs_dim, A, S = 5, 72, 12, 98
    keys = [f"agent_{i}" for i in range(n)]
    n_envs, C, Be = 3, 12, 6
    prod, orc = _buffers(keys, obs_dim, A, S, n_envs, C, Be, T)
    for ev in qmix_episode_stream(np.random.default_rng(T), keys, n_envs, T, obs_dim, A, S, 6):   # wraps the ring
        if ev[0] == 'store':
            prod.store(**ev[1]), orc.store(**ev[1])
        else:
            prod.finish_path(ev[1], **ev[2]), orc.finish_path(ev[1], **ev[2])
    assert prod.ptr == orc.ptr and prod.size == orc.size
    for it in range(3):
        np.random.seed(it)
        sp = prod.sample()
        np.random.seed(it)
        so = orc.sample()
        for k in ('obs', 'actions', 'rewards', 'terminals', 'agent_mask'):
            for a in keys:
                assert np.array_equal(sp[k][a].cpu().numpy(), so[k][a]), (k, a)
                assert sp[k][a].cpu().numpy().dtype == so[k][a].dtype, k
        assert np.array_equal(sp['filled'].cpu().numpy(), so['filled'])
        assert np.array_equal(sp['state'].cpu().numpy(), so['state'])
        assert sp['batch_size'] == so['batch_size'] and sp['sequence_length'] == so['sequence_length']


@pytest.mark.parametrize("R,n,S,H", [(1920, 5, 98, 32), (777, 3, 40, 32), (64, 8, 120, 64)])
def test_mixer_forward_backward_matches_torch(R, n, S, H):
    from xuance_b200.torch.rl_models import QMIX_Mixer
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(R)
    om = MixerOracle(S, H, 32, n)
    pm = QMIX_Mixer(S, H, 32, n, "cuda:0")
    pm.load_state_dict(om.state_dict())
    q = torch.randn(R, n)
    q[:5] = 0.0
    st = torch.randn(R, S)
    qo = q.clone().requires_grad_(True)
    qp = q.clone().cuda().requires_grad_(True)
    yo = om(qo, st)
    yp = pm(qp, st.cuda())
    np.testing.assert_allclose(yp.detach().cpu().numpy(), yo.detach().numpy(), rtol=1e-5, atol=1e-5)
    g = torch.randn(R, 1)
    yo.backward(g)
    yp.backward(g.cuda())
    np.testing.assert_allclose(qp.grad.cpu().numpy(), qo.grad.numpy(), rtol=1e-4, atol=1e-6)
    for (k, po), (_, pp) in zip(om.named_parameters(), pm.named_parameters()):
        np.testing.assert_allclose(pp.grad.cpu().numpy(), po.grad.numpy(), rtol=2e-4, atol=2e-5, err_msg=k)


@pytest.mark.parametrize("detach,double_q,graph", [(True, True, False), (False, True, False), (False, False, False),
                                                   (False, True, True)])
def test_qmix_learner_matches_oracle(detach, double_q, graph):
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners.qmix_learner import QMIX_Learner
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(0)
    n, obs_dim, A, S, T = 5, 72, 12, 98, 20
    keys, grouping, model = _product_model(n, obs_dim, A, S)
    om = QMIXModelOracle(n, obs_dim, A, S)
    model.load_state_dict(om.state_dict(), strict=True)
    cfg = Namespace(distributed_training=False, episode_length=T, use_grad_clip=True, grad_clip_norm=10.0,
                    device="cuda:0", model_dir="/tmp/x", running_steps=100000, parallels=4, use_parameter_sharing=True,
                    use_rnn=True, use_actions_mask=False, learning_rate=7e-4, sync_frequency=2, double_q=double_q,
                    n_epochs=1, start_training=0, gamma=0.99, end_factor_lr_decay=0.5, qmix_rnn_detach_q_eval=detach,
                    use_cuda_graph=graph)
    lrn = QMIX_Learner(cfg, grouping, model, BaseCallback())
    orc = QMIXLearnerOracle(om, keys, learning_rate=7e-4, sync_frequency=2, double_q=double_q, use_grad_clip=True,
                            grad_clip_norm=10.0, end_factor_lr_decay=0.5, total_iters=lrn.total_iters,
                            detach_q_eval=detach)
    n_envs, C, Be = 4, 16, 8
    prod, ob = _buffers(keys, obs_dim, A, S, n_envs, C, Be, T)
    for ev in qmix_episode_stream(np.random.default_rng(1), keys, n_envs, T, obs_dim, A, S, 4):
        if ev[0] == 'store':
            prod.store(**ev[1]), ob.store(**ev[1])
        else:
            prod.finish_path(ev[1], **ev[2]), ob.finish_path(ev[1], **ev[2])
    for it in range(4):
        np.random.seed(it)
        sp = prod.sample()
        np.random.seed(it)
        so = ob.sample()
        ip, io = lrn.update(sp), orc.update(so)
        np.testing.assert_allclose(ip["loss_Q"], io["loss_Q"], rtol=5e-4, atol=1e-6, err_msg=f"it{it}")
        np.testing.assert_allclose(ip["predictQ"], io["predictQ"], rtol=5e-4, atol=1e-5)
        assert ip["learning_rate"] == io["learning_rate"]
    so_, sp_ = om.state_dict(), model.state_dict()
    for k in so_:
        np.testing.assert_allclose(sp_[k].cpu().numpy(), so_[k].numpy(), rtol=2e-3, atol=3e-4, err_msg=k)
    agents_moved = any(not torch.equal(sp_[k].cpu(), QMIXModelOracle.__init__ and v) for k, v in []) if False else None


@pytest.mark.parametrize("R,n,S,fusable", [(1920, 5, 98, True), (128, 5, 98, True), (1000, 8, 112, True), (77, 3, 17, False), (245760, 5, 98, True), (300, 2, 160, False), (999, 5, 98, True), (129, 4, 104, True)])
def test_tensor_core_mixer_forward(R, n, S, fusable):
    """K9-TC (wgmma, register accumulators, bf16 hi/lo split x 4 products) vs the fp32 torch-CPU mixer."""
    from xuance_b200.torch.rl_models import QMIX_Mixer
    torch.manual_seed(R + n)
    om = MixerOracle(S, 32, 32, n)
    pm = QMIX_Mixer(S, 32, 32, n, "cuda:0")
    pm.load_state_dict(om.state_dict())
    q = torch.randn(R, n) * 2
    st = torch.randn(R, S)
    with torch.no_grad():
        want = om(q, st).reshape(-1).numpy()
        assert pm._fusable() == fusable
        got = pm(q.cuda(), st.cuda()).reshape(-1).cpu().numpy()         # no-grad forward -> fused tensor-core path
        pm.use_tensor_core_forward = False
        plain = pm(q.cuda(), st.cuda()).reshape(-1).cpu().numpy()       # cuBLAS + K9 mix epilogue
    np.testing.assert_allclose(plain, want, rtol=1e-5, atol=1e-5)
    scale = np.abs(want).mean()
    err = np.abs(got - want).max()
    assert err <= 2e-4 * max(scale, 1.0), (err, scale)
    np.testing.assert_allclose(got, want, rtol=2e-3, atol=2e-4 * max(scale, 1.0))
