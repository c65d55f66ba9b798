"""Generate tests/golden/iql_update.npz by running the reference IQL_Learner (agi-brain/xuance v1.4.4).

Run in the build container only (needs the reference checkout):   python tests/golden/make_golden_iql.py
Reuses make_golden.py's reference import (read-only, with the oracle/ref_stubs import stubs).

Per case (FIX_CASES: n in {1, 3} x double_q on and off x action masks on and off): the reference's MixingQNetwork (GRU
agents, IndependentMixer, as iql_agents.py:44-84 builds it) and FIX_UPDATES IQL_Learner.update calls with
sync_frequency = 2 on padded episode batches with dead agents and per-agent rewards and terminals (tests/wqmix_refs.py
fix_sample; use_rnn=True), under a MultiAgentBaseCallback.  Recorded: the initial state_dict, every sample, every info
dict, the reference's greedy next actions of every update and the whole state_dict after every update.

The unmodified learner cannot train with use_rnn=True, so each case first runs one update of it on a copy of the model
and records what it does (``<case>unmodified``: the exception's class and message, or whether the parameters moved).
The fixture then runs the learner with ``_forward_transitions`` corrected in memory (each pattern below occurs once;
DESIGN.md section 4):
  * ``q_eval.grouped_tensor = {k: v[:, :, :-1] ...}`` (:58) runs inside torch.no_grad(): the view keeps requires_grad
    but has no grad_fn, so ``loss.backward()`` returns without error and no parameter receives a gradient (the update
    changes nothing): the slice moves in front of the no_grad block;
  * with action masks, ``batch.avail_actions.group(group)[:, 1:]`` (:78) slices the agent axis: ``[:, :, 1:]``."""
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
from xuance.torch.rl_models.heads.q_mix_head import IndependentMixer  # noqa: E402
from xuance.torch.rl_models.architectures.multi_agent.value_factorization import MixingQNetwork  # noqa: E402
import xuance.torch.learners.multi_agent_rl.iql_learner as reference_iql  # noqa: E402
from xuance.torch.learners.multi_agent_rl.iql_learner import IQL_Learner  # noqa: E402
from wqmix_refs import fix_sample  # noqa: E402

FIX_OBS, FIX_A, FIX_S, FIX_T, FIX_B, FIX_HID = 12, 7, 10, 8, 6, 16
FIX_UPDATES = 4
FIX_CASES = [(n, dq, mask) for n in (1, 3) for dq in (True, False) for mask in (True, False)]
FIX_INFO_KEYS = ("loss_Q", "predictQ", "learning_rate")
SAMPLE_FIELDS = ("obs", "actions", "rewards", "terminals", "agent_mask", "avail_actions")

SLICE_IN_NO_GRAD = "            q_eval.grouped_tensor = {k: v[:, :, :-1] for k, v in q_eval.grouped_tensor.items()}\n"
CORRECTIONS = [
    (SLICE_IN_NO_GRAD, ""),
    ("    with torch.no_grad():\n",
     "    if self.use_rnn:\n"
     "        q_eval.grouped_tensor = {k: v[:, :, :-1] for k, v in q_eval.grouped_tensor.items()}\n"
     "    with torch.no_grad():\n"),
    ("batch.avail_actions.group(group)[:, 1:]", "batch.avail_actions.group(group)[:, :, 1:]"),
]


def corrected_learner():
    """IQL_Learner with _forward_transitions corrected (each pattern must occur exactly once) and its greedy next actions
    kept for the fixture."""
    src = textwrap.dedent(inspect.getsource(IQL_Learner._forward_transitions))
    for old, new in CORRECTIONS:
        assert src.count(old) == 1, old
        src = src.replace(old, new)
    scope = {}
    exec(compile(src, "iql_learner.py (corrected)", "exec"), vars(reference_iql), scope)
    fwd = scope["_forward_transitions"]

    def _forward_transitions(self, batch):
        q_eval, q_next, actions_next = fwd(self, batch)
        self.last_actions_next = {k: v.detach().clone() for k, v in actions_next.grouped_tensor.items()}
        return q_eval, q_next, actions_next
    return type("IQL_Learner", (IQL_Learner,), {"_forward_transitions": _forward_transitions})


def case_name(n, double_q, mask):
    return f"n{n}/dq{int(double_q)}/m{int(mask)}/"


def case_config(n, double_q, mask):
    return dict(agent="IQL", episode_length=FIX_T, use_grad_clip=False, grad_clip_norm=0.5, parallels=4,
                running_steps=100000, start_training=0, n_epochs=1, use_parameter_sharing=True, use_rnn=True,
                use_actions_mask=mask, learning_rate=7e-4, sync_frequency=2, double_q=double_q, gamma=0.99,
                end_factor_lr_decay=0.5, use_linear_lr_decay=True, distributed_training=False, n_agents=n)


def case_seed(n, double_q, mask):
    return 700 + 10 * n + 2 * int(double_q) + int(mask)


def build_reference_model(seed, n):
    torch.manual_seed(seed)
    keys = [f"agent_{i}" for i in range(n)]
    init, act = torch.nn.init.orthogonal_, torch.nn.ReLU
    grouping = AgentGrouping.shared(keys)
    rep = Basic_RNN(input_shape=(FIX_OBS,), hidden_sizes=None, initialize=init, activation=act, device='cpu',
                    fc_hidden_sizes=[FIX_HID], recurrent_hidden_size=FIX_HID, N_recurrent_layers=1, dropout=0,
                    rnn='GRU')
    enc = AgentFeatureEncoder(rep, build_identity_encoder(n, 'none', None, 'cpu'),
                              IdentityFeatureFusion(FIX_HID, 0, 'concat'))
    q = torch.nn.ModuleDict({"shared": DiscreteActionValueCritic(enc, Discrete(FIX_A), [FIX_HID], None, init, act,
                                                                 'cpu')})
    model = MixingQNetwork(grouping, q, IndependentMixer(), use_rnn=True, device='cpu')
    return keys, grouping, model


def unmodified(out, pre, n, double_q, mask, model, keys, grouping):
    """One update of the UNMODIFIED learner on a copy of the model: what it raises, or whether it moved a parameter."""
    lrn = IQL_Learner(_learner_cfg(**case_config(n, double_q, mask)), grouping, deepcopy(model),
                      MultiAgentBaseCallback())
    s = fix_sample(np.random.default_rng(case_seed(n, double_q, mask)), keys, B=FIX_B, T=FIX_T, obs_dim=FIX_OBS,
                   A=FIX_A, S=FIX_S)
    before = [v.clone() for v in lrn.model.state_dict().values()]
    try:
        lrn.update(s)
        moved = any(not torch.equal(a, b) for a, b in zip(before, lrn.model.state_dict().values()))
        what = "ran: parameters " + ("changed" if moved else "unchanged")
    except Exception as e:                                   # noqa: BLE001  (recorded, not handled)
        what = f"{type(e).__name__}: {str(e).splitlines()[0]}"
    out[pre + "unmodified"] = np.array(what)
    return what


def golden(out, n, double_q, mask):
    pre = case_name(n, double_q, mask)
    seed = case_seed(n, double_q, mask)
    keys, grouping, model = build_reference_model(seed, n)
    for k, v in model.state_dict().items():
        out[f"{pre}init/{k}"] = v.numpy().copy()
    print(pre, "unmodified:", unmodified(out, pre, n, double_q, mask, model, keys, grouping))
    lrn = corrected_learner()(_learner_cfg(**case_config(n, double_q, mask)), grouping, model, MultiAgentBaseCallback())
    out[pre + "total_iters"] = np.array(lrn.total_iters)
    rng = np.random.default_rng(seed)
    infos = []
    for it in range(FIX_UPDATES):
        s = fix_sample(rng, keys, B=FIX_B, T=FIX_T, obs_dim=FIX_OBS, A=FIX_A, S=FIX_S)
        for f in SAMPLE_FIELDS:
            x = np.stack([np.asarray(s[f][k]) for k in keys], axis=1)
            out[f"{pre}in{it}/{f}"] = x.astype(np.uint8) if f == "avail_actions" else x
        out[f"{pre}in{it}/filled"] = s["filled"]
        info = lrn.update(s)
        infos.append([float(info[f"shared/{k}"]) for k in FIX_INFO_KEYS])
        out[f"{pre}greedy{it}"] = lrn.last_actions_next["shared"].numpy().astype(np.int32)      # [B, n, T]
        # the whole state_dict, flattened in its key order (the init/ keys give the shapes)
        out[f"{pre}after{it}"] = np.concatenate([v.numpy().reshape(-1) for v in model.state_dict().values()])
    out[pre + "infos"] = np.array(infos, np.float64)


if __name__ == "__main__":
    out = {"env": ENV}
    for n, double_q, mask in FIX_CASES:
        golden(out, n, double_q, mask)
    path = os.path.join(HERE, "iql_update.npz")
    np.savez_compressed(path, **out)
    print("iql_update.npz", os.path.getsize(path))
