"""Generate tests/golden/dcg_update.npz by running the UNMODIFIED reference DCG_Learner (agi-brain/xuance v1.4.4).

Run in the build container only (needs the reference checkout):   python tests/golden/make_golden_dcg.py
Reuses make_golden.py's reference import (read-only, with the oracle/ref_stubs import stubs) and adds the
torch_scatter stub of tests/golden/ref_stubs (scatter_add on index_add_).

Per case (FIX_CASES below: DCG and DCG_S; FULL, CYCLE and VDN; msg_normalized on and off; one low-rank payoff;
n_msg_iterations = 0 for DCG and DCG_S - without payoffs q_dcg leaves V(s) out too, so DCG_S on VDN or with 0
iterations never trains its bias head): the reference's DeepCoordinationGraph (GRU agents, DCG_Utility, DCG_Payoff,
ValueHead for DCG_S, as dcg_agents.py:52-107 builds it) and FIX_UPDATES DCG_Learner.update calls with sync_frequency = 2 on padded episode
batches with dead agents and action masks (tests/wqmix_refs.py fix_sample).  Recorded: the initial state_dict, every
sample, every info dict and the whole state_dict after updates FIX_SNAPSHOTS.

Also recorded, for every graph type: act() on recorded hidden states with masks, the actions and the final utility U.
act() returns only the actions, so its source runs here with ``return actions_greedy`` replaced by
``return actions_greedy, utility``; nothing else of it changes."""
import inspect
import os
import sys
import textwrap

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_stubs"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from make_golden import ENV, HERE, _learner_cfg  # noqa: E402  (imports the reference and sets up sys.path)
from gymnasium.spaces import Discrete, Box  # noqa: E402
from xuance.common import AgentGrouping, BaseCallback  # noqa: E402
from xuance.torch.rl_models.representations.rnn import Basic_RNN  # noqa: E402
from xuance.torch.rl_models.representations.agent_feature import AgentFeatureEncoder  # noqa: E402
from xuance.torch.rl_models.modules.identity_encoder import build_identity_encoder, IdentityFeatureFusion  # noqa: E402
from xuance.torch.rl_models.heads import ValueHead, DCG_Utility, DCG_Payoff, Coordination_Graph  # noqa: E402
from xuance.torch.rl_models.architectures import DeepCoordinationGraph  # noqa: E402
import xuance.torch.learners.multi_agent_rl.dcg_learner as reference_dcg  # noqa: E402
from xuance.torch.learners.multi_agent_rl.dcg_learner import DCG_Learner  # noqa: E402
from wqmix_refs import fix_sample  # noqa: E402

FIX_N, FIX_OBS, FIX_A, FIX_S, FIX_T, FIX_B, FIX_HID = 4, 12, 6, 10, 8, 6, 16
FIX_UPDATES, FIX_SNAPSHOTS = 4, (1, 3)
FIX_INFO_KEYS = ("loss_Q", "predictQ", "learning_rate")
# (name, agent, graph_type, msg_normalized, low_rank_payoff, n_msg_iterations)
FIX_CASES = [("dcg_full", "DCG", "FULL", True, False, 8), ("dcg_s_full", "DCG_S", "FULL", True, False, 8),
             ("dcg_cycle_raw", "DCG", "CYCLE", False, False, 8), ("dcg_s_cycle_lowrank", "DCG_S", "CYCLE", True, True, 4),
             ("dcg_iter0", "DCG", "FULL", True, False, 0), ("dcg_s_iter0", "DCG_S", "FULL", True, False, 0),
             ("dcg_s_vdn", "DCG_S", "VDN", True, False, 8)]
FIX_RANK = 3
SAMPLE_FIELDS = ("obs", "actions", "rewards", "terminals", "agent_mask", "avail_actions")


def case_config(agent, graph, normalized, low_rank, n_iter):
    return dict(agent=agent, episode_length=FIX_T, use_grad_clip=False, grad_clip_norm=0.5, parallels=4,
                running_steps=100000, start_training=0, n_epochs=1, use_parameter_sharing=True, use_rnn=True,
                use_actions_mask=True, learning_rate=7e-4, sync_frequency=2, gamma=0.99, end_factor_lr_decay=0.5,
                use_linear_lr_decay=True, distributed_training=False, graph_type=graph, msg_normalized=normalized,
                low_rank_payoff=low_rank, payoff_rank=FIX_RANK, n_msg_iterations=n_iter, double_q=True)


def acting_learner():
    """DCG_Learner whose act() also returns the final utility (the one expression changed, see the module doc)."""
    ns = dict(vars(reference_dcg))
    src = textwrap.dedent(inspect.getsource(DCG_Learner.act))
    assert src.count("return actions_greedy") == 1
    exec(src.replace("return actions_greedy", "return actions_greedy, utility"), ns)
    return type("DCG_Learner", (DCG_Learner,), {"act": ns["act"]})


def build_reference_model(seed, agent, graph, low_rank):
    torch.manual_seed(seed)
    keys = [f"agent_{i}" for i in range(FIX_N)]
    init, act = torch.nn.init.orthogonal_, torch.nn.ReLU
    rep = Basic_RNN(input_shape=(FIX_OBS,), hidden_sizes=None, initialize=init, activation=act, device='cpu',
                    fc_hidden_sizes=[FIX_HID], recurrent_hidden_size=FIX_HID, N_recurrent_layers=1, dropout=0, rnn='GRU')
    enc = AgentFeatureEncoder(rep, build_identity_encoder(FIX_N, 'none', None, 'cpu'),
                              IdentityFeatureFusion(FIX_HID, 0, 'concat'))
    utility = DCG_Utility(FIX_HID, FIX_HID, FIX_A, 'cpu')
    payoffs = DCG_Payoff(2 * FIX_HID, FIX_HID, FIX_A, low_rank, FIX_RANK, 'cpu')
    g = Coordination_Graph(FIX_N, graph, 'cpu')
    g.set_coordination_graph()
    bias = ValueHead(FIX_S, [FIX_HID], None, init, act, 'cpu') if agent == "DCG_S" else None
    grouping = AgentGrouping.shared(keys)
    model = DeepCoordinationGraph(grouping, {k: Discrete(FIX_A) for k in keys}, torch.nn.ModuleDict({'shared': enc}),
                                  utility, payoffs, g, dcg_s=agent == "DCG_S", bias=bias, use_rnn=True, device='cpu')
    return keys, grouping, model


def golden(out, ci, name, agent, graph, normalized, low_rank, n_iter):
    pre = name + "/"
    keys, grouping, model = build_reference_model(200 + ci, agent, graph, low_rank)
    for k, v in model.state_dict().items():
        out[f"{pre}init/{k}"] = v.numpy().copy()
    lrn = DCG_Learner(_learner_cfg(**case_config(agent, graph, normalized, low_rank, n_iter)), grouping, model,
                      BaseCallback())
    out[pre + "total_iters"] = np.array(lrn.total_iters)
    rng = np.random.default_rng(200 + ci)
    infos = []
    for it in range(FIX_UPDATES):
        s = fix_sample(rng, keys, B=FIX_B, T=FIX_T, obs_dim=FIX_OBS, A=FIX_A, S=FIX_S)
        for f in SAMPLE_FIELDS:
            x = np.stack([np.asarray(s[f][k]) for k in keys], axis=1)
            out[f"{pre}in{it}/{f}"] = x.astype(np.uint8) if f == "avail_actions" else x
        out[f"{pre}in{it}/filled"], out[f"{pre}in{it}/state"] = s["filled"], s["state"]
        info = lrn.update(s)
        infos.append([float(info[k]) for k in FIX_INFO_KEYS])
        if it in FIX_SNAPSHOTS:
            out[f"{pre}after{it}"] = np.concatenate([v.numpy().reshape(-1) for v in model.state_dict().values()])
    out[pre + "infos"] = np.array(infos, np.float64)


def golden_act(out):
    """act() of the reference for every graph type on recorded hidden states [R, n, H] with masks."""
    rng = np.random.default_rng(7)
    R = 64
    for gi, graph in enumerate(("FULL", "CYCLE", "LINE", "STAR", "VDN")):
        keys, grouping, model = build_reference_model(300 + gi, "DCG", graph, False)
        cfg = _learner_cfg(**case_config("DCG", graph, True, False, 8))
        lrn = acting_learner()(cfg, grouping, model, BaseCallback())
        h = torch.from_numpy(rng.normal(size=(R, FIX_N, FIX_HID)).astype(np.float32))
        avail = (rng.random((R, FIX_N, FIX_A)) < 0.6)
        avail[..., 1] = True
        actions, utility = lrn.act(h, avail_actions=torch.from_numpy(avail.astype(np.float32)))
        pre = f"act/{graph}/"
        for k, v in model.state_dict().items():
            if k.startswith(("utility.", "payoffs.")):
                out[pre + k] = v.numpy().copy()
        out[pre + "hidden"], out[pre + "avail"] = h.numpy(), avail.astype(np.uint8)
        out[pre + "actions"], out[pre + "U"] = actions.numpy(), utility.numpy()


if __name__ == "__main__":
    out = {"env": ENV}
    for ci, case in enumerate(FIX_CASES):
        golden(out, ci, *case)
    golden_act(out)
    path = os.path.join(HERE, "dcg_update.npz")
    np.savez_compressed(path, **out)
    print("dcg_update.npz", os.path.getsize(path))
