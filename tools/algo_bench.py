#!/usr/bin/env python
"""Secondary measurements for BASELINE configs 3-5 (parity-test cases, not the headline): sample + update throughput of
DQN+PER (2^20-transition HBM replay, B=512), SAC (1M replay, B=1024) and QMIX (5 agents x 72-d, T=60, 32 episodes)
on one GPU, next to the oracle port of the reference's torch-CPU path on the host; and ``ppo_gauss``, continuous-control
PPO in the shape of the reference's ppo/mujoco.yaml (train_epochs env-steps/s); ``mappo``, MAPPO in the shape of
configs/mappo/sc2/5m_vs_6m.yaml (train_epochs env-steps/s); ``mappo_rnn``, recurrent MAPPO in the shape of
configs/mappo/sc2/3m.yaml (update, eager and graphed); ``wqmix``, CW-QMIX in the shape of configs/wqmix/sc2/5m_vs_6m.yaml
(update, eager and graphed); ``dcg``, DCG in the shape of configs/dcg/sc2/5m_vs_6m.yaml (update, eager and graphed);
``qtran``, QTRAN_alt in the shape of configs/qtran/sc2/5m_vs_6m.yaml (update, eager and graphed);
``iql``, IQL in the shape of configs/iql/sc2/5m_vs_6m.yaml (update, eager and graphed);
``vdac``, VDAC (QMIX mixer) in the shape of configs/vdac/sc2/5m_vs_6m.yaml (update, eager and graphed);
``sacdis``, SAC-Discrete in the shape of
configs/sac/CartPole-v1.yaml and at 18 actions with automatic entropy tuning (train_epochs, eager and graphed); ``ddpg`` and
``td3``, DDPG / TD3 in the shape of the reference's ddpg/mujoco.yaml and td3/mujoco.yaml (sample + update, eager and
graphed); ``c51`` and ``qrdqn`` on CartPole (Basic_MLP 128, B=256) and SyntheticAtari (Basic_CNN, B=32) shapes (update,
eager and graphed); ``drqn``, DRQN in the shape of configs/drqn/classic_control/CartPole-v1.yaml (update, eager and
graphed); ``coma``, COMA in the shape of configs/coma/sc2/5m_vs_6m.yaml (update, eager and graphed); ``npg``, NPG in
the shapes of configs/npg/classic_control/{CartPole,Pendulum}-v1.yaml (update, eager and graphed, next to the reference's
dense float32 inverse restated on the GPU).  Prints one JSON object.

    python tools/algo_bench.py [--iters 200] [--cpu-iters 5] [--no-cpu] [--graph]
    torchrun --nnodes=1 --nproc-per-node G --master-addr 127.0.0.1 tools/algo_bench.py --no-cpu --graph    (G GPUs)

Multi-GPU (BASELINE configs 3 and 5 are multi-GPU configurations): one process per GPU; the replay is sharded (envs / episodes
per rank), every update takes batch/G rows from every rank, the gradient bucket (+ logged statistics) is all-reduced once per
update inside the captured graph; the time of an update is the max over ranks (barrier + synchronize on both sides) and the
global batch is fixed (strong scaling).
"""
import argparse
import json
import os
import sys
import time
from argparse import Namespace

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
RANK, WORLD, LOCAL = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))
DEV = "cuda:%d" % LOCAL


def timed(fn, iters, warm=10):
    import torch.distributed as dist
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    if WORLD > 1:
        dist.barrier()
        torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / 1e3 / iters], dtype=torch.float64, device=DEV)
    if WORLD > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def cpu_timed(fn, iters):
    fn()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    return (time.perf_counter() - t0) / iters


def bench_perdqn(args):
    from xuance_b200.common import PerOffPolicyBuffer, Box, Discrete, BaseCallback
    from xuance_b200.torch.rl_models import Basic_CNN, DeepQNetwork
    from xuance_b200.torch.learners import PerDQN_Learner
    N, S, B, A = 16 // WORLD, 65536, 512 // WORLD, 4          # this rank's envs and its share of the 512-row batch
    buf = PerOffPolicyBuffer(Box(0, 255, (84, 84, 4), np.uint8), Discrete(A), None, N, N * S, B, alpha=0.5, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(RANK)
    for t in range(64):   # real stores through K1 + K5 insert, then the rest of the ring is declared filled
        o = torch.randint(0, 256, (N, 84, 84, 4), dtype=torch.uint8, device=DEV, generator=g)
        buf.store(o, torch.randint(0, A, (N,), device=DEV), torch.randn(N, device=DEV), torch.zeros(N, device=DEV), o)
    buf.size = S
    leaves = torch.rand((N, S), device=DEV) + 0.01
    cap = buf._it_capacity
    buf._it_sum[:, cap:cap + S], buf._it_min[:, cap:cap + S] = leaves, leaves
    lvl = cap // 2
    while lvl >= 1:
        buf._it_sum[:, lvl:2 * lvl] = buf._it_sum[:, 2 * lvl:4 * lvl:2] + buf._it_sum[:, 2 * lvl + 1:4 * lvl:2]
        buf._it_min[:, lvl:2 * lvl] = torch.minimum(buf._it_min[:, 2 * lvl:4 * lvl:2], buf._it_min[:, 2 * lvl + 1:4 * lvl:2])
        lvl //= 2
    rep = Basic_CNN(input_shape=(84, 84, 4), kernels=[8, 4, 3], strides=[4, 2, 1], filters=[32, 64, 64], activation=nn.ReLU, device=DEV)
    model = DeepQNetwork(rep, [512], Discrete(A), None, None, nn.ReLU, DEV).to(DEV)
    cfg = Namespace(distributed_training=WORLD > 1, episode_length=1000, use_grad_clip=False, grad_clip_norm=0.5, device=DEV,
                    model_dir="/tmp/x", running_steps=10**7, parallels=N * WORLD, learning_rate=1e-4, gamma=0.99,
                    sync_frequency=500, start_training=0, training_frequency=1, compute=args.compute, tc_planes=3)
    if args.compute != "fp32":
        rep.tc_planes = 3
        rep.set_compute(args.compute)
    cfg.use_cuda_graph = args.graph
    lrn = PerDQN_Learner(cfg, model, BaseCallback())

    def step():
        s = buf.sample(0.4)
        td, _ = lrn.update(sync=False, **s)
        buf.update_priorities(s["step_choices"], td)

    dt = timed(step, args.iters)
    out = {"config": "DQN+PER, 2^20-transition uint8 HBM replay (59 GB), 16 envs, B=512 (global), encoder compute=%s" % args.compute,
           "gpu_updates_per_s": 1 / dt, "gpu_transitions_per_s": B * WORLD / dt, "gpu_ms_per_update": dt * 1e3}
    if not args.no_cpu:
        from oracle.replay import PerReplayOracle
        from oracle.nets import DeepQNetworkOracle
        from oracle.learners import DQNLearnerOracle
        Sc = 1024   # the reference stores float32 image replay: 2^20 would need 226 GB of host RAM (SURVEY row P2)
        ob = PerReplayOracle((84, 84, 4), (), N, N * Sc, B, alpha=0.5, obs_dtype=np.uint8)
        rng = np.random.default_rng(0)
        for t in range(Sc):
            o = rng.integers(0, 256, size=(N, 84, 84, 4), dtype=np.uint8)
            ob.store(o, rng.integers(0, A, N), rng.normal(size=N).astype(np.float32), np.zeros(N, bool), o)
        ol = DQNLearnerOracle(DeepQNetworkOracle(A), per=True)

        def cstep():
            s = ob.sample(0.4)
            td, _ = ol.update(**s)
            ob.update_priorities(s["step_choices"], td)

        cdt = cpu_timed(cstep, args.cpu_iters)
        out.update(cpu_updates_per_s=1 / cdt, cpu_ms_per_update=cdt * 1e3, cpu_replay_capacity=N * Sc,
                   cpu_threads=torch.get_num_threads(), speedup=cdt / dt)
    return out


def bench_sac(args):
    from copy import deepcopy
    from xuance_b200.common import DummyOffPolicyBuffer, Box, BaseCallback
    from xuance_b200.torch.rl_models import Basic_Identical, SAC_GaussianActor, TwinActionValueCritic, SoftActorCritic
    from xuance_b200.torch.learners import REGISTRY_Learners
    N, S, B, od, ad = 4, 250000 // WORLD, 1024 // WORLD, 17, 6
    aspace = Box(-1, 1, (ad,), np.float32)
    buf = DummyOffPolicyBuffer(Box(-10, 10, (od,), np.float32), aspace, None, N, N * S, B, device=DEV)
    buf._obs.normal_(), buf._next_obs.normal_(), buf._act_rows.uniform_(-1, 1), buf._fields.normal_()
    buf.size = S
    rep = Basic_Identical((od,), device=DEV)
    model = SoftActorCritic(SAC_GaussianActor(rep, [256, 256], aspace, None, None, nn.LeakyReLU, nn.Tanh, DEV),
                            TwinActionValueCritic(deepcopy(rep), aspace, [256, 256], None, None, nn.LeakyReLU, DEV)).to(DEV)
    cfg = Namespace(distributed_training=WORLD > 1, episode_length=1000, use_grad_clip=False, grad_clip_norm=0.5, device=DEV,
                    model_dir="/tmp/x", running_steps=10**6, parallels=N, start_training=0, training_frequency=1,
                    learning_rate_actor=1e-3, learning_rate_critic=1e-3, tau=0.005, gamma=0.99, alpha=0.2,
                    use_automatic_entropy_tuning=True)
    cfg.use_cuda_graph = args.graph
    lrn = REGISTRY_Learners["SAC_Learner"](cfg, model, BaseCallback())
    dt = timed(lambda: lrn.update(sync=False, **buf.sample()), args.iters)
    out = {"config": "SAC, 17-d obs / 6-d act, 1M replay, B=1024 (global), MLP 256-256", "gpu_updates_per_s": 1 / dt,
           "gpu_transitions_per_s": B * WORLD / dt, "gpu_ms_per_update": dt * 1e3}
    if not args.no_cpu:
        from oracle.replay import UniformReplayOracle
        from oracle.sac import SACModelOracle, SACLearnerOracle
        ob = UniformReplayOracle((od,), (ad,), N, N * S, B)
        ob.observations[...] = np.random.default_rng(0).normal(size=ob.observations.shape)
        ob.size = S
        ol = SACLearnerOracle(SACModelOracle(od, ad))
        cdt = cpu_timed(lambda: ol.update(torch.randn(B, ad), torch.randn(B, ad), **ob.sample()), max(args.cpu_iters, 20))
        out.update(cpu_updates_per_s=1 / cdt, cpu_ms_per_update=cdt * 1e3, cpu_threads=torch.get_num_threads(), speedup=cdt / dt)
    return out


def bench_qmix(args, Be=32):
    from helpers import qmix_episode_stream
    from test_gpu_qmix import _product_model, _buffers
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import REGISTRY_Learners
    n, od, A, S, T = 5, 72, 12, 98, 60
    Be_global, Be = Be, Be // WORLD                              # this rank's share of the episodes of an update
    keys, grouping, model = _product_model(n, od, A, S, device=DEV)
    n_envs, C = 8, max(256, 2 * Be)
    prod, ob = _buffers(keys, od, A, S, n_envs, C, Be, T, device=DEV)
    for ev in qmix_episode_stream(np.random.default_rng(RANK), keys, n_envs, T, od, A, S, C // n_envs):
        if ev[0] == 'store':
            prod.store(**ev[1]), ob.store(**ev[1])
        else:
            prod.finish_path(ev[1], **ev[2]), ob.finish_path(ev[1], **ev[2])
    cfg = Namespace(distributed_training=WORLD > 1, episode_length=T, use_grad_clip=False, grad_clip_norm=10.0, device=DEV,
                    model_dir="/tmp/x", running_steps=10**7, parallels=n_envs, use_parameter_sharing=True, use_rnn=True,
                    use_actions_mask=False, learning_rate=7e-4, sync_frequency=200, double_q=True, n_epochs=1,
                    start_training=0, gamma=0.99)
    cfg.use_cuda_graph = args.graph
    lrn = REGISTRY_Learners["QMIX_Learner"](cfg, grouping, model, BaseCallback())
    dt = timed(lambda: lrn.update(prod.sample(), sync=False), args.iters)
    out = {"config": f"QMIX, 5 agents x 72-d, S=98, A=12, T=60, {Be_global} episodes/update (global), GRU 64 + mixer 32/32",
           "gpu_updates_per_s": 1 / dt, "gpu_agent_steps_per_s": Be_global * T * n / dt, "gpu_ms_per_update": dt * 1e3}
    if not args.no_cpu:
        from oracle.qmix import QMIXModelOracle, QMIXLearnerOracle
        ol = QMIXLearnerOracle(QMIXModelOracle(n, od, A, S), keys, detach_q_eval=False)
        cdt = cpu_timed(lambda: ol.update(ob.sample()), max(args.cpu_iters, 10))
        out.update(cpu_updates_per_s=1 / cdt, cpu_ms_per_update=cdt * 1e3, cpu_threads=torch.get_num_threads(), speedup=cdt / dt)
    return out


def bench_wqmix(args, B=32):
    """One WQMIX_Learner update in the shape of configs/wqmix/sc2/5m_vs_6m.yaml (5 agents x 72-d, S=98, A=12, T=60, 32
    episodes, GRU 64, QMIX mixer 32/64, feed-forward mixer 256, action masks, CW-QMIX), eager and graphed, on a device-resident
    sample; next to the torch-CPU oracle of the same update."""
    import wqmix_refs as R
    from oracle_wqmix import WQMIXModelOracle, WQMIXLearnerOracle
    from test_gpu_wqmix import _product_model
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import REGISTRY_Learners
    n, od, A, S, T = 5, 72, 12, 98, 60
    keys = [f"agent_{i}" for i in range(n)]
    sample = R.fix_sample(np.random.default_rng(0), keys, B=B, T=T, obs_dim=od, A=A, S=S)
    dev = lambda x: {k: dev(v) for k, v in x.items()} if isinstance(x, dict) else (
        torch.as_tensor(x, device=DEV) if isinstance(x, np.ndarray) else x)
    dsample = dev(sample)
    out = {"config": f"CW-QMIX, 5 agents x 72-d, S=98, A=12, T=60, {B} episodes/update, GRU 64, mixer 32/64, "
                     f"feed-forward mixer 256, action masks"}
    for graph in (False, True):
        torch.manual_seed(0)
        _, grouping, model = _product_model(n, od, A, S, 64, 32, 64, 256)
        cfg = Namespace(agent="CWQMIX", alpha=0.1, distributed_training=False, episode_length=T, use_grad_clip=False,
                        grad_clip_norm=0.5, device=DEV, model_dir="/tmp/x", running_steps=10**7, parallels=8,
                        use_parameter_sharing=True, use_rnn=True, use_actions_mask=True, learning_rate=7e-4,
                        sync_frequency=200, double_q=True, n_epochs=1, start_training=0, gamma=0.99,
                        use_cuda_graph=graph)
        lrn = REGISTRY_Learners["WQMIX_Learner"](cfg, grouping, model, BaseCallback())
        dt = timed(lambda: lrn.update(dsample, sync=False), args.iters)
        out["gpu_ms_per_update_graphed" if graph else "gpu_ms_per_update_eager"] = dt * 1e3
    out["gpu_agent_steps_per_s_graphed"] = B * T * n / (out["gpu_ms_per_update_graphed"] / 1e3)
    if not args.no_cpu:
        ol = WQMIXLearnerOracle(WQMIXModelOracle(n, od, A, S), keys, agent="CWQMIX", detach_q_eval=False)
        cdt = cpu_timed(lambda: ol.update(sample), max(args.cpu_iters, 5))
        out.update(cpu_ms_per_update=cdt * 1e3, cpu_threads=torch.get_num_threads(),
                   speedup_graphed=cdt * 1e3 / out["gpu_ms_per_update_graphed"])
    return out


def bench_dcg(args, B=32):
    """One DCG_Learner update in the shape of configs/dcg/sc2/5m_vs_6m.yaml (5 agents x 72-d, A=12, T=60, 32 episodes, K13
    GRU 64, utility / payoff heads 64, FULL graph: E = 10, 8 normalised message iterations, action masks), eager and
    graphed, on a device-resident sample; next to the torch-CPU oracle of the same update."""
    import dcg_refs
    import wqmix_refs as R
    from oracle_dcg import DCGModelOracle, DCGLearnerOracle
    import torch.nn as nn
    from xuance_b200.common import AgentGrouping, BaseCallback, Discrete
    from xuance_b200.torch.learners import REGISTRY_Learners
    from xuance_b200.torch.rl_models import (AgentFeatureEncoder, Basic_RNN_K13, DCG_Utility, DCG_Payoff,
                                             Coordination_Graph, DeepCoordinationGraph)
    n, od, A, T = 5, 72, 12, 60

    def product_model(H=64):
        rep = Basic_RNN_K13(input_shape=(od,), initialize=nn.init.orthogonal_, activation=nn.ReLU, device=DEV,
                            fc_hidden_sizes=[H], recurrent_hidden_size=H)
        g = Coordination_Graph(n, "FULL", DEV)
        g.set_coordination_graph()
        grouping = AgentGrouping.shared(keys)
        model = DeepCoordinationGraph(grouping, {k: Discrete(A) for k in keys},
                                      nn.ModuleDict({'shared': AgentFeatureEncoder(rep)}), DCG_Utility(H, H, A, DEV),
                                      DCG_Payoff(2 * H, H, A, False, 1, DEV), g, use_rnn=True, device=DEV).to(DEV)
        return grouping, model

    keys = [f"agent_{i}" for i in range(n)]
    sample = R.fix_sample(np.random.default_rng(0), keys, B=B, T=T, obs_dim=od, A=A, S=4)
    dev = lambda x: {k: dev(v) for k, v in x.items()} if isinstance(x, dict) else (
        torch.as_tensor(x, device=DEV) if isinstance(x, np.ndarray) else x)
    dsample = dev(sample)
    out = {"config": f"DCG, 5 agents x 72-d, A=12, T=60, {B} episodes/update, GRU 64, heads 64, FULL graph (E=10), "
                     f"8 normalised iterations, action masks"}
    for graph in (False, True):
        torch.manual_seed(0)
        grouping, model = product_model()
        cfg = Namespace(agent="DCG", distributed_training=False, episode_length=T, use_grad_clip=False,
                        grad_clip_norm=0.5, device=DEV, model_dir="/tmp/x", running_steps=10**7, parallels=8,
                        use_parameter_sharing=True, use_rnn=True, use_actions_mask=True, learning_rate=7e-4,
                        sync_frequency=200, n_epochs=1, start_training=0, gamma=0.99, use_cuda_graph=graph)
        lrn = REGISTRY_Learners["DCG_Learner"](cfg, grouping, model, BaseCallback())
        dt = timed(lambda: lrn.update(dsample, sync=False), args.iters)
        out["gpu_ms_per_update_graphed" if graph else "gpu_ms_per_update_eager"] = dt * 1e3
    if not args.no_cpu:
        ol = DCGLearnerOracle(DCGModelOracle(n, od, A), keys, dcg_refs.graph_edges(n, "FULL"))
        cdt = cpu_timed(lambda: ol.update(sample), max(args.cpu_iters, 5))
        out.update(cpu_ms_per_update=cdt * 1e3, cpu_threads=torch.get_num_threads(),
                   speedup_graphed=cdt * 1e3 / out["gpu_ms_per_update_graphed"])
    return out


def bench_qtran(args, B=32):
    """One QTRAN_Learner update (QTRAN_alt) in the shape of configs/qtran/sc2/5m_vs_6m.yaml (5 agents x 72-d, S=98, A=12,
    T=60, 32 episodes, K13 GRU 64, Q_jt / V_jt 64, action masks), eager and graphed, on a device-resident sample; next to
    the torch-CPU float64 oracle of the same update."""
    import wqmix_refs as R
    from oracle_qtran import QTRANOracle, build_model
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import REGISTRY_Learners
    n, od, A, S, T = 5, 72, 12, 98, 60
    keys = [f"agent_{i}" for i in range(n)]
    sample = R.fix_sample(np.random.default_rng(0), keys, B=B, T=T, obs_dim=od, A=A, S=S)
    dev = lambda x: {k: dev(v) for k, v in x.items()} if isinstance(x, dict) else (
        torch.as_tensor(x, device=DEV) if isinstance(x, np.ndarray) else x)
    dsample = dev(sample)
    out = {"config": f"QTRAN_alt, 5 agents x 72-d, S=98, A=12, T=60, {B} episodes/update, GRU 64, Q_jt / V_jt 64, "
                     f"action masks"}
    for graph in (False, True):
        torch.manual_seed(0)
        _, grouping, model = build_model("QTRAN_alt", n, od, A, S, 64, 64, DEV)
        cfg = Namespace(agent="QTRAN_alt", distributed_training=False, episode_length=T, use_grad_clip=False,
                        grad_clip_norm=0.5, device=DEV, model_dir="/tmp/x", running_steps=10**7, parallels=8,
                        use_parameter_sharing=True, use_rnn=True, use_actions_mask=True, learning_rate=7e-4,
                        sync_frequency=200, n_epochs=1, start_training=0, gamma=0.99, double_q=True, lambda_opt=1.0,
                        lambda_nopt=1.0, use_cuda_graph=graph)
        lrn = REGISTRY_Learners["QTRAN_Learner"](cfg, grouping, model, BaseCallback())
        dt = timed(lambda: lrn.update(dsample, sync=False), args.iters)
        out["gpu_ms_per_update_graphed" if graph else "gpu_ms_per_update_eager"] = dt * 1e3
    if not args.no_cpu:
        orc = QTRANOracle(model, total_iters=10**6)
        cdt = cpu_timed(lambda: orc.update(sample), max(args.cpu_iters, 5))
        out.update(cpu_ms_per_update=cdt * 1e3, cpu_threads=torch.get_num_threads(),
                   speedup_graphed=cdt * 1e3 / out["gpu_ms_per_update_graphed"])
    return out


def bench_iql(args, B=32):
    """One IQL_Learner update in the shape of configs/iql/sc2/5m_vs_6m.yaml (5 agents x 72-d, A=12, T=60, 32 episodes,
    K13 GRU 64, Q head 64, double-Q, action masks), eager and graphed, on a device-resident sample; next to the torch-CPU
    float64 oracle of the same update."""
    import wqmix_refs as R
    from oracle_iql import IQLOracle, build_model
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import REGISTRY_Learners
    n, od, A, T = 5, 72, 12, 60
    keys = [f"agent_{i}" for i in range(n)]
    sample = R.fix_sample(np.random.default_rng(0), keys, B=B, T=T, obs_dim=od, A=A, S=4)
    dev = lambda x: {k: dev(v) for k, v in x.items()} if isinstance(x, dict) else (
        torch.as_tensor(x, device=DEV) if isinstance(x, np.ndarray) else x)
    dsample = dev(sample)
    out = {"config": f"IQL, 5 agents x 72-d, A=12, T=60, {B} episodes/update, GRU 64, Q head 64, double-Q, "
                     f"action masks"}
    for graph in (False, True):
        torch.manual_seed(0)
        _, grouping, model = build_model(n, od, A, 64, DEV)
        cfg = Namespace(agent="IQL", distributed_training=False, episode_length=T, use_grad_clip=False,
                        grad_clip_norm=0.5, device=DEV, model_dir="/tmp/x", running_steps=10**7, parallels=8,
                        use_parameter_sharing=True, use_rnn=True, use_actions_mask=True, learning_rate=7e-4,
                        sync_frequency=200, n_epochs=1, start_training=0, gamma=0.99, double_q=True,
                        use_cuda_graph=graph)
        lrn = REGISTRY_Learners["IQL_Learner"](cfg, grouping, model, BaseCallback())
        dt = timed(lambda: lrn.update(dsample, sync=False), args.iters)
        out["gpu_ms_per_update_graphed" if graph else "gpu_ms_per_update_eager"] = dt * 1e3
    if not args.no_cpu:
        orc = IQLOracle(model, total_iters=10**6)
        cdt = cpu_timed(lambda: orc.update(sample), max(args.cpu_iters, 5))
        out.update(cpu_ms_per_update=cdt * 1e3, cpu_threads=torch.get_num_threads(),
                   speedup_graphed=cdt * 1e3 / out["gpu_ms_per_update_graphed"])
    return out


def bench_ppo_gauss(args):
    """PPO with a Gaussian policy in the shape of the reference's ppo/mujoco.yaml (Ant-v4: 27-d obs, 8-d action): 16 envs x
    256 steps, 16 epochs x 8 minibatches of 512, Basic_Identical + actor / critic [256, 256].  The measured unit is
    ``train_epochs`` over one stored rollout (128 minibatch updates); env-steps/s = 4096 / its time."""
    from xuance_b200.common import Box
    from xuance_b200.torch.agents import PPO_Agent
    N, T, od, ad, epochs, mb = 16, 256, 27, 8, 16, 8
    cfg = Namespace(agent="PPO", learner="PPO_Learner", representation="Basic_Identical", env_name="MuJoCo",
                    distributed_training=False, device=DEV, seed=1, parallels=N, running_steps=10**6, horizon_size=T,
                    n_epochs=epochs, n_minibatch=mb, learning_rate=4e-4, vf_coef=0.25, ent_coef=0.0, clip_range=0.2,
                    gamma=0.99, use_gae=True, gae_lambda=0.95, use_advnorm=True, use_grad_clip=True, grad_clip_norm=0.5,
                    use_obsnorm=False, use_rewnorm=False, activation="leaky_relu", activation_action="tanh",
                    actor_hidden_size=[256, 256], critic_hidden_size=[256, 256], model_dir="/tmp/x", logger=None,
                    episode_length=None, use_cuda_graph=args.graph)
    agent = PPO_Agent(cfg, None, Box(-np.inf, np.inf, (od,), np.float32), Box(-1, 1, (ad,), np.float32))
    rng = np.random.default_rng(0)
    ro = dict(obs=rng.normal(size=(T, N, od)).astype(np.float32), acts=np.clip(rng.normal(size=(T, N, ad)), -1, 1).astype(np.float32),
              rews=rng.normal(size=(T, N)).astype(np.float32), vals=rng.normal(size=(T, N)).astype(np.float32),
              terms=rng.random((T, N)) < 0.005, logp=(rng.normal(size=(T, N)) * 0.3 - 7.0).astype(np.float32))
    for t in range(T):
        agent.memory.store(ro["obs"][t], ro["acts"][t], ro["rews"][t], ro["vals"][t], ro["terms"][t], {"old_logp": ro["logp"][t]})
    for i in range(N):
        agent.memory.finish_path(0.0, i)
    iters = max(2, args.iters // 40)
    dt = timed(lambda: agent.train_epochs(epochs), iters, warm=1)
    out = {"config": "PPO Gaussian policy, Ant-v4 shape (27-d obs, 8-d action), 16 envs x 256, 16 epochs x 8 minibatches "
                     "of 512, Basic_Identical + actor/critic MLP 256-256", "gpu_env_steps_per_s": N * T / dt,
           "gpu_ms_per_train_epochs": dt * 1e3, "gpu_ms_per_update": dt * 1e3 / (epochs * mb)}
    if not args.no_cpu:
        from oracle.onpolicy import OnPolicyBufferOracle
        from oracle_gauss import GaussianActorCriticOracle, PPOGaussLearnerOracle
        ob = OnPolicyBufferOracle((od,), (ad,), {"old_logp": ()}, N, T)
        for t in range(T):
            ob.store(ro["obs"][t], ro["acts"][t], ro["rews"][t], ro["vals"][t], ro["terms"][t], {"old_logp": ro["logp"][t]})
        for i in range(N):
            ob.finish_path(0.0, i)
        ol = PPOGaussLearnerOracle(GaussianActorCriticOracle(od, ad, rep_hidden=(), actor_hidden=(256, 256),
                                                             critic_hidden=(256, 256)), learning_rate=4e-4, ent_coef=0.0)
        idx = np.arange(N * T)
        cdt = cpu_timed(lambda: ol.update(**ob.sample(np.random.permutation(idx)[:N * T // mb])), max(args.cpu_iters, 20))
        out.update(cpu_ms_per_update=cdt * 1e3, cpu_env_steps_per_s=N * T / (cdt * epochs * mb),
                   cpu_threads=torch.get_num_threads(), speedup=cdt * epochs * mb / dt)
    return out


def bench_mappo(args):
    """MAPPO in the shape of configs/mappo/sc2/5m_vs_6m.yaml (feed-forward; SMAC 5m_vs_6m shape: 5 agents, 72-d obs, 12
    actions with masks): 8 envs x 128 steps x 5 agents = 5120 rows per update, 10 epochs x 1 minibatch.  The measured
    unit is ``train_epochs`` over one stored rollout (the buffer is kept between repetitions); env-steps/s = 1024 / its
    time.  The LayerNorm of the config is left out on both sides (the CPU oracle's MLPs have none)."""
    from xuance_b200.common import Box, Discrete
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import MAPPO_Agents
    N, T, n, od, A, epochs = 8, 128, 5, 72, 12, 10
    cfg = get_arguments("mappo", "sc2", config_path=os.path.join(ROOT, "xuance_b200", "configs", "mappo", "sc2",
                                                                  "5m_vs_6m.yaml"))
    for k, v in dict(device=DEV, parallels=N, buffer_size=N * T, n_epochs=epochs, n_minibatch=1, logger=None,
                     model_dir="/tmp/x", use_cuda_graph=args.graph, distributed_training=False).items():
        setattr(cfg, k, v)
    del cfg.normalize
    keys = ["agent_%d" % i for i in range(n)]
    agent = MAPPO_Agents(cfg, None, n, keys, None, {k: Box(-1, 1, (od,), np.float32) for k in keys},
                         {k: Discrete(A) for k in keys})
    rng = np.random.default_rng(0)
    for t in range(T):
        avail = {k: (rng.random((N, A)) > 0.3).astype(np.int64) for k in keys}
        for k in keys:
            avail[k][:, 0] = 1
        agent.memory.store(obs={k: rng.uniform(-1, 1, (N, od)).astype(np.float32) for k in keys},
                           actions={k: np.zeros(N, np.float32) for k in keys},
                           log_pi_old={k: np.full(N, -2.3, np.float32) for k in keys},
                           rewards={k: rng.random(N).astype(np.float32) for k in keys},
                           values={k: rng.normal(size=N).astype(np.float32) for k in keys},
                           terminals={k: rng.random(N) < 0.01 for k in keys},
                           agent_mask={k: rng.random(N) > 0.05 for k in keys}, avail_actions=avail)
    for i in range(N):
        agent.memory.finish_path(i, agent.agent_grouping, {k: np.float32(0.1) for k in keys},
                                 agent.learner.value_normalizer)
    agent.memory.clear = lambda: None          # keep the stored rollout for every repetition
    iters = max(2, args.iters // 40)
    dt = timed(lambda: agent.train_epochs(epochs), iters, warm=1)
    R = N * T * n
    out = {"config": "MAPPO 5m_vs_6m shape (5 agents, 72-d obs, 12 masked actions), 8 envs x 128 steps, 10 epochs x 1 "
                     "minibatch of 5120 rows, Basic_MLP 64 + actor / critic MLP 64-64, value clip + ValueNorm + Huber",
           "gpu_env_steps_per_s": N * T / dt, "gpu_ms_per_train_epochs": dt * 1e3, "gpu_ms_per_update": dt * 1e3 / epochs}
    if not args.no_cpu:
        from oracle_mappo import MAPPOModelOracle, MAPPOLearnerOracle
        ol = MAPPOLearnerOracle(MAPPOModelOracle(od, A, (64,), (64, 64), (64, 64)), cfg)
        av = torch.from_numpy(rng.random((R, A)) > 0.3)
        av[:, 0] = True
        b = [torch.from_numpy(x) for x in (rng.uniform(-1, 1, (R, od)).astype(np.float32), np.zeros(R, np.float32),
                                           np.full(R, -2.3, np.float32), rng.normal(size=R).astype(np.float32),
                                           rng.normal(size=R).astype(np.float32), rng.normal(size=R).astype(np.float32),
                                           (rng.random(R) > 0.05).astype(np.float32))]
        cdt = cpu_timed(lambda: ol.update(*b, av), max(args.cpu_iters, 10))
        out.update(cpu_ms_per_update=cdt * 1e3, cpu_env_steps_per_s=N * T / (cdt * epochs),
                   cpu_threads=torch.get_num_threads(), speedup=cdt * epochs / dt)
    return out


def bench_mappo_rnn(args):
    """Recurrent MAPPO in the shape of configs/mappo/sc2/3m.yaml: one MAPPO_Learner.update over its minibatch of 128
    episodes x 3 agents x T = 60 (384 GRU sequences, 23040 rows; fc [64, 64, 64], GRU 64, LayerNorm, 9 masked actions),
    eager and as a CUDA graph, next to the torch-CPU oracle's update (nn.GRU on the host) on the same model."""
    import copy
    from xuance_b200.common import Box, Discrete
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import MAPPO_Agents
    from oracle_mappo import MAPPOLearnerOracle
    from oracle_mappo_rnn import RecurrentModelOracle
    B, n, T, od, A = 128, 3, 60, 30, 9
    keys = ["agent_%d" % i for i in range(n)]
    rng = np.random.default_rng(0)
    S = B * n
    avail = np.zeros((S, T, 12), np.uint8)
    avail[..., :A] = rng.random((S, T, A)) > 0.3
    avail[..., 0] = 1
    lengths = np.tile(rng.integers(20, T + 1, B), n)
    st = dict(obs=rng.uniform(-1, 1, (S, T, od)).astype(np.float32), actions=np.zeros((S, T), np.float32),
              log_pi_old=np.full((S, T), -2.2, np.float32), advantages=rng.normal(size=(S, T)).astype(np.float32),
              values=rng.normal(size=(S, T)).astype(np.float32), returns=rng.normal(size=(S, T)).astype(np.float32),
              agent_mask=(rng.random((S, T)) > 0.05).astype(np.float32),
              filled=(np.arange(T)[None] < lengths[:, None]).astype(np.float32), avail_actions=avail)
    sample = {'_stacked': {k: torch.from_numpy(v).to(DEV) for k, v in st.items()}, 'batch_size': B,
              'sequence_length': T}
    out = {"config": "recurrent MAPPO 3m shape: 128 episodes x 3 agents x T = 60 per update, Basic_RNN (fc 64-64-64, "
                     "GRU 64, LayerNorm) actor and critic, 9 masked actions, value clip + ValueNorm + Huber"}
    model = None
    for graph in (False, True):
        cfg = get_arguments("mappo", "sc2", "3m")
        for k, v in dict(device=DEV, parallels=8, logger=None, model_dir="/tmp/x", use_cuda_graph=graph,
                         distributed_training=False, episode_length=T).items():
            setattr(cfg, k, v)
        torch.manual_seed(0)
        agent = MAPPO_Agents(cfg, None, n, keys, None, {k: Box(-1, 1, (od,), np.float32) for k in keys},
                             {k: Discrete(A) for k in keys})
        if model is None:
            model = copy.deepcopy(agent.model)
        dt = timed(lambda: agent.learner.update(sample, sync=False), max(5, args.iters // 10), warm=3)
        out["gpu_ms_per_update_" + ("graph" if graph else "eager")] = dt * 1e3
    if not args.no_cpu:
        ol = MAPPOLearnerOracle(RecurrentModelOracle(model), cfg)
        t = {k: torch.from_numpy(v) for k, v in st.items()}
        fl = lambda k: t[k].reshape(-1)
        b = (t['obs'], fl('actions'), fl('log_pi_old'), fl('advantages'), fl('values'), fl('returns'),
             fl('agent_mask') * fl('filled'), t['avail_actions'][..., :A].reshape(-1, A) != 0)
        cdt = cpu_timed(lambda: ol.update(*b), max(args.cpu_iters, 3))
        out.update(cpu_ms_per_update=cdt * 1e3, cpu_threads=torch.get_num_threads(),
                   speedup_eager=cdt * 1e3 / out["gpu_ms_per_update_eager"],
                   speedup_graph=cdt * 1e3 / out["gpu_ms_per_update_graph"])
    return out


def bench_vdac(args):
    """VDAC with the QMIX mixer in the shape of configs/vdac/sc2/5m_vs_6m.yaml: one VDAC_Learner.update over its minibatch
    of 8 episodes x 5 agents x T = 60 (GRU 64, LayerNorm, 12 masked actions, global state 98), eager and as a CUDA graph."""
    from xuance_b200.common import Box, Discrete
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import VDAC_Agents
    B, n, T, od, A, sd = 8, 5, 60, 72, 12, 98
    keys = ["agent_%d" % i for i in range(n)]
    rng = np.random.default_rng(0)
    S = B * n
    avail = np.zeros((S, T, 12), np.uint8)
    avail[..., :A] = rng.random((S, T, A)) > 0.3
    avail[..., 0] = 1
    lengths = np.tile(rng.integers(20, T + 1, B), n)
    st = dict(obs=rng.uniform(-1, 1, (S, T, od)).astype(np.float32), actions=np.zeros((S, T), np.float32),
              advantages=rng.normal(size=(S, T)).astype(np.float32), values=rng.normal(size=(S, T)).astype(np.float32),
              returns=rng.normal(size=(S, T)).astype(np.float32),
              agent_mask=(rng.random((S, T)) > 0.05).astype(np.float32),
              filled=(np.arange(T)[None] < lengths[:, None]).astype(np.float32), avail_actions=avail,
              state=np.tile(rng.normal(size=(B, T, sd)).astype(np.float32), (n, 1, 1)))
    sample = {'_stacked': {k: torch.from_numpy(v).to(DEV) for k, v in st.items()}, 'batch_size': B,
              'sequence_length': T}
    out = {"config": "VDAC (QMIX mixer) 5m_vs_6m shape: 8 episodes x 5 agents x T = 60 per update, Basic_RNN (fc 64, "
                     "GRU 64, LayerNorm) actor and critic, 12 masked actions, value clip + ValueNorm + Huber"}
    for graph in (False, True):
        cfg = get_arguments("vdac", "sc2", "5m_vs_6m")
        for k, v in dict(device=DEV, parallels=8, logger=None, model_dir="/tmp/x", use_cuda_graph=graph,
                         distributed_training=False, episode_length=T).items():
            setattr(cfg, k, v)
        torch.manual_seed(0)
        agent = VDAC_Agents(cfg, None, n, keys, Box(-1, 1, (sd,), np.float32),
                            {k: Box(-1, 1, (od,), np.float32) for k in keys}, {k: Discrete(A) for k in keys})
        dt = timed(lambda: agent.learner.update(sample, sync=False), max(5, args.iters // 10), warm=3)
        out["gpu_ms_per_update_" + ("graph" if graph else "eager")] = dt * 1e3
    return out


def bench_sacdis(args):
    """SAC-Discrete: ``train_epochs(1)`` (one replay sample of 256 rows + one SACDIS_Learner.update) of a SAC_Agent built
    from configs/sac/CartPole-v1.yaml (4-d obs, A = 2, Basic_MLP 128, heads [128], alpha fixed), and the same at A = 18 with
    use_automatic_entropy_tuning on.  Eager and CUDA-graphed, next to the torch-CPU oracle's update on the host."""
    from xuance_b200 import _lib
    from xuance_b200.common import Box, Discrete
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import SAC_Agent
    out = {}
    for name, A, auto in (("cartpole_A2", 2, False), ("A18_auto_alpha", 18, True)):
        od, N, S = 4, 10, 20000
        res = {"config": "SAC-Discrete, %d-d obs, A = %d, B = 256, Basic_MLP 128 + heads [128], auto alpha %s"
                         % (od, A, auto)}
        for graph in (False, True):
            cfg = get_arguments("sac", "classic_control", "CartPole-v1")
            for k, v in dict(device=DEV, use_cuda_graph=graph, use_automatic_entropy_tuning=auto, model_dir="/tmp/x",
                             logger=None, distributed_training=False).items():
                setattr(cfg, k, v)
            agent = SAC_Agent(cfg, None, Box(-10, 10, (od,), np.float32), Discrete(A))
            buf = agent.memory
            buf._obs.normal_(), buf._next_obs.normal_(), buf._fields.uniform_(0, 1)
            buf._fields[buf._fid["actions"]].mul_(A).floor_()
            buf._fields[buf._fid["terminals"]].copy_((buf._fields[buf._fid["terminals"]] < 0.05).float())
            buf.size = S
            if not graph:
                agent.train_epochs(1)
                before = _lib.launch_count
                agent.train_epochs(1)
                res["xb_launches_per_update"] = _lib.launch_count - before
            dt = timed(lambda: agent.train_epochs(1), args.iters)
            res["gpu_%s_ms_per_update" % ("graphed" if graph else "eager")] = dt * 1e3
            res["gpu_%s_updates_per_s" % ("graphed" if graph else "eager")] = 1 / dt
        if not args.no_cpu:
            from oracle_sacdis import SACDISModelOracle, SACDISLearnerOracle
            ol = SACDISLearnerOracle(SACDISModelOracle(od, A, (128,), (128,), (128,)), auto_alpha=auto)
            rng = np.random.default_rng(0)
            s = {"obs": rng.normal(size=(256, od)).astype(np.float32), "obs_next": rng.normal(size=(256, od)).astype(np.float32),
                 "actions": rng.integers(0, A, 256).astype(np.float32), "rewards": rng.random(256).astype(np.float32),
                 "terminals": (rng.random(256) < 0.05).astype(np.float32)}
            cdt = cpu_timed(lambda: ol.update(**s), max(args.cpu_iters, 20))
            res.update(cpu_ms_per_update=cdt * 1e3, cpu_threads=torch.get_num_threads(),
                       speedup_eager=cdt / (res["gpu_eager_ms_per_update"] / 1e3),
                       speedup_graphed=cdt / (res["gpu_graphed_ms_per_update"] / 1e3))
        out[name] = res
    return out


def bench_ddpg_td3(args, algo):
    """DDPG / TD3 in the shape of the reference's ddpg/mujoco.yaml and td3/mujoco.yaml: 17-d observations, 6 action
    components, Basic_Identical representation, actor and critic MLPs [400, 300] with leaky_relu, B = 100 (DDPG) or 256
    (TD3, actor_update_delay 2: the time is the mean over critic-only and actor iterations).  One replay sample + one
    update, eager and CUDA-graphed, next to the torch-CPU oracle's update on the host."""
    from copy import deepcopy
    from xuance_b200 import _lib
    from xuance_b200.common import DummyOffPolicyBuffer, Box, BaseCallback
    from xuance_b200.torch.rl_models import (Basic_Identical, DeterministicActor, ActionValueCritic, TwinActionValueCritic,
                                             DeterministicActorCritic, TwinDelayedActorCritic)
    from xuance_b200.torch.learners import REGISTRY_Learners
    twin = algo == "td3"
    N, S, B, od, ad = 4, 250000, 256 if twin else 100, 17, 6
    aspace = Box(-1, 1, (ad,), np.float32)
    res = {"config": "%s, 17-d obs / 6-d act, 1M replay, B=%d, Basic_Identical + MLP 400-300 leaky_relu%s"
                     % (algo.upper(), B, ", actor_update_delay 2" if twin else "")}
    for graph in (False, True):
        buf = DummyOffPolicyBuffer(Box(-10, 10, (od,), np.float32), aspace, None, N, N * S, B, device=DEV)
        buf._obs.normal_(), buf._next_obs.normal_(), buf._act_rows.uniform_(-1, 1), buf._fields.normal_()
        buf.size = S
        rep = Basic_Identical((od,), device=DEV)
        actor = DeterministicActor(rep, [400, 300], aspace, None, None, nn.LeakyReLU, nn.Tanh, DEV)
        if twin:
            model = TwinDelayedActorCritic(actor, TwinActionValueCritic(deepcopy(rep), aspace, [400, 300], None, None,
                                                                        nn.LeakyReLU, DEV))
        else:
            model = DeterministicActorCritic(actor, ActionValueCritic(deepcopy(rep), aspace, [400, 300], None, None,
                                                                      nn.LeakyReLU, DEV))
        cfg = Namespace(distributed_training=False, episode_length=1000, use_grad_clip=False, grad_clip_norm=0.5,
                        device=DEV, model_dir="/tmp/x", running_steps=10**6, parallels=N, start_training=0,
                        training_frequency=1, learning_rate_actor=1e-3, learning_rate_critic=1e-3, tau=0.005,
                        gamma=0.99, actor_update_delay=2, use_cuda_graph=graph)
        lrn = REGISTRY_Learners["TD3_Learner" if twin else "DDPG_Learner"](cfg, model.to(DEV), BaseCallback())
        if not graph:
            lrn.update(sync=False, **buf.sample())
            before = _lib.launch_count
            lrn.update(sync=False, **buf.sample())
            lrn.update(sync=False, **buf.sample())
            res["xb_launches_per_2_updates"] = _lib.launch_count - before
        dt = timed(lambda: lrn.update(sync=False, **buf.sample()), args.iters)
        res["gpu_%s_ms_per_update" % ("graphed" if graph else "eager")] = dt * 1e3
        res["gpu_%s_updates_per_s" % ("graphed" if graph else "eager")] = 1 / dt
    if not args.no_cpu:
        from oracle_ddpg import DDPGModelOracle, DDPGLearnerOracle
        ol = DDPGLearnerOracle(DDPGModelOracle(od, ad, -np.ones(ad, np.float32), np.ones(ad, np.float32), twin, (),
                                               (400, 300), (400, 300), act=nn.LeakyReLU),
                               actor_update_delay=2 if twin else 1)
        rng = np.random.default_rng(0)
        s = {"obs": rng.normal(size=(B, od)).astype(np.float32), "obs_next": rng.normal(size=(B, od)).astype(np.float32),
             "actions": rng.uniform(-1, 1, (B, ad)).astype(np.float32), "rewards": rng.random(B).astype(np.float32),
             "terminals": (rng.random(B) < 0.05).astype(np.float32)}
        noise = rng.normal(size=(B, ad)).astype(np.float32) if twin else None
        cdt = cpu_timed(lambda: ol.update(noise_next=noise, **s), max(args.cpu_iters, 20))
        res.update(cpu_ms_per_update=cdt * 1e3, cpu_threads=torch.get_num_threads(),
                   speedup_eager=cdt / (res["gpu_eager_ms_per_update"] / 1e3),
                   speedup_graphed=cdt / (res["gpu_graphed_ms_per_update"] / 1e3))
    return res


def bench_dist_dqn(args, algo):
    """C51 / QR-DQN updates at the shapes of the shipped configs: CartPole-v1 (4-d observations, 2 actions, Basic_MLP [128]
    + head [128], B = 256) and SyntheticAtari (84x84x4 uint8, 4 actions, Basic_CNN 32-64-64 + head [512], B = 32; fp32
    cuDNN encoder).  One update on a fixed batch, eager and CUDA-graphed, with the xb200 launches per update, next to the
    torch-CPU oracle's update on the host at the same shape."""
    from xuance_b200 import _lib
    from xuance_b200.common import Discrete, BaseCallback
    from xuance_b200.torch.rl_models import Basic_MLP, Basic_CNN, C51DeepQNetwork, QRDeepQNetwork
    from xuance_b200.torch.learners import REGISTRY_Learners
    N = 51 if algo == "c51" else 20
    res = {}
    rng = np.random.default_rng(0)
    for shape, B, A in (("cartpole", 256, 2), ("atari", 32, 4)):
        r = {"config": "%s %s: B=%d, A=%d, N=%d" % (algo.upper(), shape, B, A, N)}
        if shape == "cartpole":
            obs = lambda: rng.normal(size=(B, 4)).astype(np.float32)
        else:
            obs = lambda: rng.integers(0, 256, (B, 84, 84, 4), dtype=np.uint8)
        s = {"obs": obs(), "obs_next": obs(), "actions": rng.integers(0, A, B).astype(np.float32),
             "rewards": rng.normal(size=B).astype(np.float32), "terminals": (rng.random(B) < 0.05).astype(np.float32)}
        s_dev = {k: torch.as_tensor(v, device=DEV) for k, v in s.items()}
        for graph in (False, True):
            if shape == "cartpole":
                rep = Basic_MLP((4,), [128], None, nn.init.orthogonal_, nn.ReLU, DEV)
                hidden = [128]
            else:
                rep = Basic_CNN((84, 84, 4), kernels=[8, 4, 3], strides=[4, 2, 1], filters=[32, 64, 64], normalize=None,
                                initialize=nn.init.orthogonal_, activation=nn.ReLU, device=DEV)
                hidden = [512]
            if algo == "c51":
                model = C51DeepQNetwork(rep, hidden, Discrete(A), N, 0, 200, None, nn.init.orthogonal_, nn.ReLU, DEV)
            else:
                model = QRDeepQNetwork(rep, hidden, Discrete(A), N, None, nn.init.orthogonal_, nn.ReLU, DEV)
            cfg = Namespace(distributed_training=False, episode_length=1000, use_grad_clip=False, grad_clip_norm=0.5,
                            device=DEV, model_dir="/tmp/x", running_steps=10**6, parallels=10, start_training=0,
                            training_frequency=1, learning_rate=1e-3, gamma=0.99, sync_frequency=100,
                            use_cuda_graph=graph)
            lrn = REGISTRY_Learners["C51_Learner" if algo == "c51" else "QRDQN_Learner"](cfg, model.to(DEV),
                                                                                         BaseCallback())
            if not graph:
                lrn.update(sync=False, **s_dev)
                before = _lib.launch_count
                lrn.update(sync=False, **s_dev)
                r["xb_launches_per_update"] = _lib.launch_count - before
            dt = timed(lambda: lrn.update(sync=False, **s_dev), args.iters)
            r["gpu_%s_ms_per_update" % ("graphed" if graph else "eager")] = dt * 1e3
        if not args.no_cpu:
            from oracle_dist import DistModelOracle, DistLearnerOracle
            if shape == "cartpole":
                om = DistModelOracle(algo, 4, A, N, (128,), (128,), 0, 200)
            else:
                om = DistModelOracle(algo, None, A, N, q_hidden=(512,), v_min=0, v_max=200, pixels=True)
            ol = DistLearnerOracle(om, sync_frequency=100)
            cdt = cpu_timed(lambda: ol.update(**s), max(args.cpu_iters, 20))
            r.update(cpu_ms_per_update=cdt * 1e3, cpu_threads=torch.get_num_threads(),
                     speedup_eager=cdt / (r["gpu_eager_ms_per_update"] / 1e3),
                     speedup_graphed=cdt / (r["gpu_graphed_ms_per_update"] / 1e3))
        res[shape] = r
    return res


def bench_drqn(args, repeats=3):
    """DRQN in the shape of configs/drqn/classic_control/CartPole-v1.yaml: one DRQN_Learner.update over B = 8 windows of
    L = 50 steps (Basic_MLP 128, LSTM 128, 2 actions), eager and as a CUDA graph, each repeated ``repeats`` times, next to
    the torch-CPU oracle's update (nn.LSTM on the host) on the same shape."""
    import subprocess
    from xuance_b200.common import Box, Discrete
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import DRQN_Agent
    from oracle_drqn import DRQNOracle, DRQNLearnerOracle
    B, L, od, A = 8, 50, 4, 2
    rng = np.random.default_rng(0)
    sample = {"obs": torch.from_numpy(rng.standard_normal((B, L + 1, od)).astype(np.float32)).to(DEV),
              "actions": torch.from_numpy(rng.integers(0, A, (B, L)).astype(np.float32)).to(DEV),
              "rewards": torch.ones(B, L, device=DEV), "terminals": torch.zeros(B, L, device=DEV), "batch_size": B}
    out = {"config": "DRQN CartPole-v1 shape: B = 8 windows x L = 50, Basic_MLP 128, LSTM 128, 2 actions",
           "gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                 capture_output=True, text=True).stdout.strip()}
    for graph in (False, True):
        cfg = get_arguments("drqn", "classic_control", "CartPole-v1")
        for k, v in dict(device=DEV, logger=None, model_dir="/tmp/x", use_cuda_graph=graph, episode_length=500).items():
            setattr(cfg, k, v)
        agent = DRQN_Agent(cfg, observation_space=Box(-np.inf, np.inf, (od,), np.float32), action_space=Discrete(A))
        out["gpu_ms_per_update_" + ("graph" if graph else "eager")] = [
            round(timed(lambda: agent.learner.update(sync=False, **sample), args.iters, warm=5) * 1e3, 4)
            for _ in range(repeats)]
    if not args.no_cpu:
        ol = DRQNLearnerOracle(DRQNOracle("LSTM", 128, od, 128, A))
        cs = {k: v.cpu() for k, v in sample.items() if k != "batch_size"}
        out["cpu_ms_per_update"] = round(cpu_timed(lambda: ol.update(**cs), max(args.cpu_iters, 3)) * 1e3, 3)
        out["cpu_threads"] = torch.get_num_threads()
    return out


def bench_coma(args):
    """COMA in the shape of configs/coma/sc2/5m_vs_6m.yaml: one COMA_Learner.update over its minibatch of 8 episodes x 5
    agents x T = 60 (fc 64, GRU 64, LayerNorm actor and critic encoders, critic MLP 128-128 over the 98 + 64 + 5 * 12
    counterfactual input, 12 actions), eager and as a CUDA graph, next to the torch-CPU oracle's update (nn.GRU on the
    host) on the same model and sample."""
    import copy
    import subprocess
    from xuance_b200.common import Box, Discrete
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import COMA_Agents
    from oracle_coma import COMALearnerOracle
    B, n, T, od, A, sd = 8, 5, 60, 72, 12, 98
    keys = ["agent_%d" % i for i in range(n)]
    rng = np.random.default_rng(0)
    S = B * n
    lengths = np.tile(rng.integers(20, T + 1, B), n)
    st = dict(obs=rng.uniform(-1, 1, (S, T, od)).astype(np.float32),
              actions=rng.integers(0, A, (S, T)).astype(np.float32),
              advantages=rng.normal(size=(S, T)).astype(np.float32), values=rng.normal(size=(S, T)).astype(np.float32),
              returns=rng.normal(size=(S, T)).astype(np.float32),
              agent_mask=(rng.random((S, T)) > 0.05).astype(np.float32),
              filled=(np.arange(T)[None] < lengths[:, None]).astype(np.float32),
              state=np.tile(rng.normal(size=(B, T, sd)).astype(np.float32), (n, 1, 1)))
    sample = {'_stacked': {k: torch.from_numpy(v).to(DEV) for k, v in st.items()}, 'batch_size': B,
              'sequence_length': T}
    out = {"config": "COMA 5m_vs_6m shape: 8 episodes x 5 agents x T = 60 per update, Basic_RNN (fc 64, GRU 64, "
                     "LayerNorm) actor and critic encoders, critic MLP 128-128, 12 actions, epsilon 0.5",
           "gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                 capture_output=True, text=True).stdout.strip()}
    model = None
    for graph in (False, True):
        cfg = get_arguments("coma", "sc2", "5m_vs_6m")
        for k, v in dict(device=DEV, parallels=8, logger=None, model_dir="/tmp/x", use_cuda_graph=graph,
                         distributed_training=False, episode_length=T).items():
            setattr(cfg, k, v)
        torch.manual_seed(0)
        agent = COMA_Agents(cfg, None, n, keys, Box(-1, 1, (sd,), np.float32),
                            {k: Box(-1, 1, (od,), np.float32) for k in keys}, {k: Discrete(A) for k in keys})
        if model is None:
            model = copy.deepcopy(agent.model)
        dt = timed(lambda: agent.learner.update(sample, 0.5, sync=False), max(5, args.iters // 10), warm=3)
        out["gpu_ms_per_update_" + ("graph" if graph else "eager")] = dt * 1e3
    if not args.no_cpu:
        ol = COMALearnerOracle(model, (n, False, 0.5), cfg=vars(cfg))
        t = {k: torch.from_numpy(v) for k, v in st.items()}
        b = dict(obs=t['obs'].reshape(n, B, T, od).transpose(0, 1).reshape(S, T, od),
                 **{k: t[f].reshape(n, B, T).transpose(0, 1).reshape(-1) for k, f in
                    (("actions", "actions"), ("returns", "returns"))},
                 mask=(t['agent_mask'] * t['filled']).reshape(n, B, T).transpose(0, 1).reshape(-1),
                 avail=None, state=t['state'][:B], B=B, n=n, T=T)
        cdt = cpu_timed(lambda: ol.update(b, 0.5), max(args.cpu_iters, 3))
        out.update(cpu_ms_per_update=cdt * 1e3, cpu_threads=torch.get_num_threads(),
                   speedup_eager=cdt * 1e3 / out["gpu_ms_per_update_eager"],
                   speedup_graph=cdt * 1e3 / out["gpu_ms_per_update_graph"])
    return out


def _gpu_identity():
    """The card's name and power limit, read next to the measurement."""
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(LOCAL)],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "nvidia-smi unavailable"
    return {"device": torch.cuda.get_device_name(LOCAL), "nvidia_smi": q}


def bench_npg(args, repeats=3):
    """One NPG_Learner update in the shapes of the shipped configs: CartPole-v1 (Basic_MLP 128, actor / critic 128, 2
    actions, 10 envs x 256 steps in 8 minibatches: B = 320) and Pendulum-v1 (Basic_MLP 256, actor 256, critic 256, 1 action
    component, 10 x 128 in one minibatch: B = 1280), eager and graphed, on device-resident samples, repeated ``repeats``
    times.  Next to it, the reference's natural gradient of ONE CartPole-shape minibatch restated on the GPU: per actor
    tensor a dense float32 P x P F = kappa s s^T + 1e-3 I, torch.linalg.inv(F) and F^-1 g (the largest P is 16384)."""
    from xuance_b200.common import Box, Discrete
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import REGISTRY_Agents
    out = {"gpu": _gpu_identity()}
    shapes = {"cartpole": ("CartPole-v1", Box(-5, 5, (4,), np.float32), Discrete(2)),
              "pendulum": ("Pendulum-v1", Box(-8, 8, (3,), np.float32), Box(-2, 2, (1,), np.float32))}
    for name, (env_id, obs_space, act_space) in shapes.items():
        res = {}
        for graph in (False, True):
            cfg = get_arguments("npg", "classic_control", env_id,
                                parser_args=Namespace(device=DEV, use_cuda_graph=graph, model_dir="/tmp/xb_npg_bench"))
            torch.manual_seed(0)
            agent = REGISTRY_Agents["NPG"](cfg, None, obs_space, act_space)
            B = agent.batch_size
            rng = np.random.default_rng(0)
            acts = (rng.normal(size=(B, 1)) * 0.4) if isinstance(act_space, Box) else rng.integers(0, 2, B)
            s = {"obs": torch.as_tensor(rng.normal(size=(B,) + obs_space.shape), dtype=torch.float32, device=DEV),
                 "actions": torch.as_tensor(acts, dtype=torch.float32, device=DEV),
                 "returns": torch.as_tensor(rng.normal(size=B), dtype=torch.float32, device=DEV),
                 "advantages": torch.as_tensor(rng.normal(size=B), dtype=torch.float32, device=DEV)}
            lrn = agent.learner
            key = "gpu_ms_per_update_graphed" if graph else "gpu_ms_per_update_eager"
            res[key] = [timed(lambda: lrn.update(sync=False, **s), args.iters) * 1e3 for _ in range(repeats)]
            res["B"], res["actor_params"] = B, [p.numel() for p in agent.model.actor.parameters()]
        out[name] = res
        if name == "cartpole":
            out["cartpole_dense_inverse_restatement"] = _npg_dense_restatement(agent, s, repeats)
    return out


def _npg_dense_restatement(agent, s, repeats):
    """The reference's F^-1 g (npg_learner.py:100-113) for one minibatch, restated on the GPU in float32 (the reference
    itself runs this on whatever device the learner uses): one dense inverse per actor tensor."""
    model, H = agent.model, agent.config.horizon_size
    params = list(model.actor.parameters())
    logits = model.logits(s["obs"])
    logp = torch.distributions.Categorical(logits=logits).log_prob(s["actions"].long())
    scores = [x.reshape(-1) for x in torch.autograd.grad(logp.sum(), params, retain_graph=True)]
    grads = [x.reshape(-1) for x in torch.autograd.grad(-(s["advantages"] * logp).mean(), params)]
    kappa = logp.sum().item() / H

    def step():
        for sc, g in zip(scores, grads):
            F = torch.outer(sc, sc) * kappa + 1e-3 * torch.eye(sc.numel(), device=DEV)
            torch.linalg.inv(F) @ g
    step()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    return {"what": "restatement of the reference's dense float32 inverse, one CartPole-shape minibatch (B = %d)"
            % s["actions"].shape[0], "largest_P": max(x.numel() for x in scores), "gpu_ms_per_minibatch": times}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--cpu-iters", type=int, default=5)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--only", default="")
    ap.add_argument("--graph", action="store_true", help="capture the learners' device update in a CUDA graph")
    ap.add_argument("--compute", default="fp32", choices=["fp32", "tc"], help="pixel encoder of the PER-DQN network")
    args = ap.parse_args()
    torch.cuda.set_device(LOCAL)
    torch.manual_seed(0)          # identical initial weights on every rank
    if WORLD > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device(DEV))
        args.no_cpu = True
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    only = set(x for x in args.only.split(",") if x)
    res = {}
    if not only or "perdqn" in only:
        res["perdqn"] = bench_perdqn(args)
    if not only or "sac" in only:
        res["sac"] = bench_sac(args)
    if not only or "qmix" in only:
        res["qmix"] = bench_qmix(args)
        res["qmix_4096"] = bench_qmix(Namespace(**{**vars(args), "iters": 20, "no_cpu": True}), Be=1024)
    if (not only and WORLD == 1) or "wqmix" in only:
        res["wqmix"] = bench_wqmix(args)
    if (not only and WORLD == 1) or "dcg" in only:
        res["dcg"] = bench_dcg(args)
    if (not only and WORLD == 1) or "qtran" in only:
        res["qtran"] = bench_qtran(args)
    if (not only and WORLD == 1) or "iql" in only:
        res["iql"] = bench_iql(args)
    if (not only and WORLD == 1) or "ppo_gauss" in only:
        res["ppo_gauss"] = bench_ppo_gauss(args)
    if (not only and WORLD == 1) or "mappo" in only:
        res["mappo"] = bench_mappo(args)
    if (not only and WORLD == 1) or "mappo_rnn" in only:
        res["mappo_rnn"] = bench_mappo_rnn(args)
    if (not only and WORLD == 1) or "vdac" in only:
        res["vdac"] = bench_vdac(args)
    if (not only and WORLD == 1) or "sacdis" in only:
        res["sacdis"] = bench_sacdis(args)
    for algo in ("ddpg", "td3"):
        if (not only and WORLD == 1) or algo in only:
            res[algo] = bench_ddpg_td3(args, algo)
    for algo in ("c51", "qrdqn"):
        if (not only and WORLD == 1) or algo in only:
            res[algo] = bench_dist_dqn(args, algo)
    if (not only and WORLD == 1) or "drqn" in only:
        res["drqn"] = bench_drqn(args)
    if (not only and WORLD == 1) or "coma" in only:
        res["coma"] = bench_coma(args)
    if (not only and WORLD == 1) or "npg" in only:
        res["npg"] = bench_npg(args)
    res["cuda_graph"] = bool(args.graph)
    res["n_gpus"] = WORLD
    if RANK == 0:
        print(json.dumps(res))
    if WORLD > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
