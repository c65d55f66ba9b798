"""Generate tests/golden/qtran_update.npz by running the reference QTRAN_Learner (agi-brain/xuance v1.4.4).

Run in the build container only (needs the reference checkout):   python tests/golden/make_golden_qtran.py
Reuses make_golden.py's reference import (read-only, with the oracle/ref_stubs import stubs).

Per case (FIX_CASES: QTRAN_base and QTRAN_alt, double_q on and off): the reference's QTranMixingNetwork (GRU agents,
VDN_Mixer, QTRAN_Base / QTRAN_Alt, as qtran_agents.py:45-101 builds it) and FIX_UPDATES QTRAN_Learner.update calls with
sync_frequency = 2 on padded episode batches with dead agents and action masks (tests/wqmix_refs.py fix_sample;
use_actions_mask=True, use_rnn=True), under a MultiAgentBaseCallback.  Recorded: the initial state_dict, every sample,
every info dict and the whole state_dict after updates FIX_SNAPSHOTS.

With one parameter-sharing group (every shipped sc2 config) update_rnn raises as written, so the learner runs with
exactly these expressions corrected in memory, each occurring once in update_rnn (DESIGN.md section 4):
  * ``hidden_state[key] = hidden_state[key][:, :-1]`` and the ``hidden_state_next`` line (:242-243) index the
    group-keyed embeddings by agent key (KeyError 'agent_0'): every group's embeddings are sliced once before the loop;
  * ``AgentGroupedTensor(actions_next_greedy | actions_greedy_eval, ...)`` (:275, :285) wrap agent-keyed dicts as
    group-keyed ones: ``AgentGroupedTensor.from_agent_wise``;
  * QTRAN_alt: ``actions[k]`` (:302) and ``q_eval[k]`` (:326) subscript AgentGroupedTensors: ``.agent_wise[k]``; the plain
    dicts handed to Q_tran_target / Q_tran (:305, :317) are wrapped with ``from_agent_wise``.
Evidence that the corrections only re-key: on independent groups (where the uncorrected QTRAN_base runs) the corrected
and the uncorrected learner give exactly the same info dicts; ``rekey_check`` records that comparison."""
import inspect
import os
import textwrap
from copy import deepcopy

import numpy as np
import torch

from make_golden import ENV, HERE, _learner_cfg  # noqa: E402  (imports the reference and sets up sys.path)
from gymnasium.spaces import Discrete  # noqa: E402
from xuance.common import AgentGrouping, MultiAgentBaseCallback  # noqa: E402
from xuance.torch.rl_models.representations.rnn import Basic_RNN  # noqa: E402
from xuance.torch.rl_models.representations.agent_feature import AgentFeatureEncoder  # noqa: E402
from xuance.torch.rl_models.modules.identity_encoder import build_identity_encoder, IdentityFeatureFusion  # noqa: E402
from xuance.torch.rl_models.critics.base_critics import DiscreteActionValueCritic  # noqa: E402
from xuance.torch.rl_models.heads.q_mix_head import VDN_Mixer, QTRAN_Base, QTRAN_Alt  # noqa: E402
from xuance.torch.rl_models.architectures.multi_agent.value_factorization import QTranMixingNetwork  # noqa: E402
import xuance.torch.learners.multi_agent_rl.qtran_learner as reference_qtran  # noqa: E402
from xuance.torch.learners.multi_agent_rl.qtran_learner import QTRAN_Learner  # noqa: E402
from wqmix_refs import fix_sample  # noqa: E402

FIX_N, FIX_OBS, FIX_A, FIX_S, FIX_T, FIX_B, FIX_HID, FIX_QH = 3, 12, 7, 10, 8, 6, 16, 16
FIX_UPDATES, FIX_SNAPSHOTS = 4, (1, 3)
FIX_CASES = [(agent, dq) for agent in ("QTRAN_base", "QTRAN_alt") for dq in (True, False)]
FIX_INFO_KEYS = ("loss_td", "loss_opt", "loss_nopt", "loss", "Q_joint", "learning_rate")
SAMPLE_FIELDS = ("obs", "actions", "rewards", "terminals", "agent_mask", "avail_actions")

CORRECTIONS = [
    ("            hidden_state[key] = hidden_state[key][:, :-1]\n", ""),
    ("            hidden_state_next[key] = hidden_state_next[key][:, :-1]\n", ""),
    ("        q_eval_a, q_eval_greedy_a, q_next, q_next_a = {}, {}, {}, {}\n",
     "        hidden_state = {k: v[:, :-1] for k, v in hidden_state.items()}\n"
     "        hidden_state_next = {k: v[:, :-1] for k, v in hidden_state_next.items()}\n"
     "        q_eval_a, q_eval_greedy_a, q_next, q_next_a = {}, {}, {}, {}\n"),
    ("AgentGroupedTensor(actions_next_greedy, self.agent_grouping)",
     "AgentGroupedTensor.from_agent_wise(actions_next_greedy, self.agent_grouping)"),
    ("AgentGroupedTensor(actions_greedy_eval, self.agent_grouping)",
     "AgentGroupedTensor.from_agent_wise(actions_greedy_eval, self.agent_grouping)"),
    ("torch.stack([actions[k] for k in self.agent_keys], dim=2)",
     "torch.stack([actions.agent_wise[k] for k in self.agent_keys], dim=2)"),
    ("torch.stack([q_eval[k][:, :-1] for k in self.agent_keys]",
     "torch.stack([q_eval.agent_wise[k][:, :-1] for k in self.agent_keys]"),
    ("hidden_state_next, actions_next_greedy, agent_mask)",
     "hidden_state_next,\n                AgentGroupedTensor.from_agent_wise(actions_next_greedy, self.agent_grouping), agent_mask)"),
    ("hidden_state, actions_greedy_eval, agent_mask)",
     "hidden_state,\n                AgentGroupedTensor.from_agent_wise(actions_greedy_eval, self.agent_grouping), agent_mask)"),
]


def corrected_learner():
    """QTRAN_Learner with the raising expressions of update_rnn corrected (each must occur exactly once)."""
    ns = dict(vars(reference_qtran))
    src = inspect.getsource(QTRAN_Learner.update_rnn)           # class indentation: the patterns above match it
    for old, new in CORRECTIONS:
        assert src.count(old) == 1, old
        src = src.replace(old, new)
    exec(textwrap.dedent(src), ns)
    return type("QTRAN_Learner", (QTRAN_Learner,), {"update_rnn": ns["update_rnn"]})


def case_config(agent, double_q, shared=True):
    return dict(agent=agent, episode_length=FIX_T, use_grad_clip=False, grad_clip_norm=0.5, parallels=4,
                running_steps=100000, start_training=0, n_epochs=1, use_parameter_sharing=shared, use_rnn=True,
                use_actions_mask=True, learning_rate=7e-4, sync_frequency=2, double_q=double_q, gamma=0.99,
                lambda_opt=1.0, lambda_nopt=1.0, end_factor_lr_decay=0.5, use_linear_lr_decay=True,
                distributed_training=False, n_agents=FIX_N)


def case_seed(agent, double_q):
    return 400 + 10 * (agent == "QTRAN_alt") + int(double_q)


def build_reference_model(seed, agent, shared=True):
    torch.manual_seed(seed)
    keys = [f"agent_{i}" for i in range(FIX_N)]
    init, act = torch.nn.init.orthogonal_, torch.nn.ReLU
    grouping = AgentGrouping.shared(keys) if shared else AgentGrouping.independent(keys)
    q = torch.nn.ModuleDict()
    for g in grouping.group_keys:
        rep = Basic_RNN(input_shape=(FIX_OBS,), hidden_sizes=None, initialize=init, activation=act, device='cpu',
                        fc_hidden_sizes=[FIX_HID], recurrent_hidden_size=FIX_HID, N_recurrent_layers=1, dropout=0,
                        rnn='GRU')
        enc = AgentFeatureEncoder(rep, build_identity_encoder(FIX_N, 'none', None, 'cpu'),
                                  IdentityFeatureFusion(FIX_HID, 0, 'concat'))
        q[g] = DiscreteActionValueCritic(enc, Discrete(FIX_A), [FIX_HID], None, init, act, 'cpu')
    head = (QTRAN_Base if agent == "QTRAN_base" else QTRAN_Alt)(
        dim_state=FIX_S, action_space={k: Discrete(FIX_A) for k in keys}, dim_hidden=FIX_QH, n_agents=FIX_N,
        dim_utility_hidden=FIX_HID, use_parameter_sharing=shared, device='cpu')
    model = QTranMixingNetwork(grouping, q, VDN_Mixer(), head, use_rnn=True, device='cpu')
    return keys, grouping, model


def golden(out, agent, double_q):
    pre = f"{agent}/dq{int(double_q)}/"
    seed = case_seed(agent, double_q)
    keys, grouping, model = build_reference_model(seed, agent)
    for k, v in model.state_dict().items():
        out[f"{pre}init/{k}"] = v.numpy().copy()
    lrn = corrected_learner()(_learner_cfg(**case_config(agent, double_q)), grouping, model, MultiAgentBaseCallback())
    out[pre + "total_iters"] = np.array(lrn.total_iters)
    rng = np.random.default_rng(seed)
    infos = []
    for it in range(FIX_UPDATES):
        s = fix_sample(rng, keys, B=FIX_B, T=FIX_T, obs_dim=FIX_OBS, A=FIX_A, S=FIX_S)
        for f in SAMPLE_FIELDS:
            x = np.stack([np.asarray(s[f][k]) for k in keys], axis=1)
            out[f"{pre}in{it}/{f}"] = x.astype(np.uint8) if f == "avail_actions" else x
        out[f"{pre}in{it}/filled"], out[f"{pre}in{it}/state"] = s["filled"], s["state"]
        info = lrn.update(s)
        infos.append([float(info[k]) for k in FIX_INFO_KEYS])
        if it in FIX_SNAPSHOTS:            # the whole state_dict, flattened in its key order (the init/ keys give shapes)
            out[f"{pre}after{it}"] = np.concatenate([v.numpy().reshape(-1) for v in model.state_dict().values()])
    out[pre + "infos"] = np.array(infos, np.float64)


def rekey_check(out):
    """QTRAN_base on independent groups: the uncorrected and the corrected learner, same weights and samples."""
    runs = []
    _, grouping, model = build_reference_model(499, "QTRAN_base", shared=False)
    keys = grouping.agent_keys
    for cls in (QTRAN_Learner, corrected_learner()):
        m = deepcopy(model)
        lrn = cls(_learner_cfg(**case_config("QTRAN_base", True, shared=False)), grouping, m, MultiAgentBaseCallback())
        rng = np.random.default_rng(499)
        runs.append([[float(v) for v in lrn.update(fix_sample(rng, keys, B=FIX_B, T=FIX_T, obs_dim=FIX_OBS, A=FIX_A,
                                                                  S=FIX_S)).values()] for _ in range(3)])
    assert runs[0] == runs[1], runs
    out["rekey_check/infos"] = np.array(runs, np.float64)


if __name__ == "__main__":
    out = {"env": ENV}
    rekey_check(out)
    for agent, double_q in FIX_CASES:
        golden(out, agent, double_q)
    path = os.path.join(HERE, "qtran_update.npz")
    np.savez_compressed(path, **out)
    print("qtran_update.npz", os.path.getsize(path))
