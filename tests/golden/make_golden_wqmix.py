"""Generate tests/golden/wqmix_update.npz by running the UNMODIFIED reference WQMIX_Learner (agi-brain/xuance v1.4.4).

Run in the build container only (needs the reference checkout):   python tests/golden/make_golden_wqmix.py
Reuses make_golden.py's reference import (read-only, with the oracle/ref_stubs import stubs).

Per case (tests/wqmix_refs.py FIX_CASES: OW-QMIX and CW-QMIX, double_q on and off): the reference's
WeightedMixingQNetwork (GRU agents, QMIX_Mixer, QMIX_FF_Mixer, as wqmix_agents.py:36-88 builds it) and FIX_UPDATES
WQMIX_Learner.update calls with sync_frequency = 2 on padded episode batches with dead agents and action masks
(use_actions_mask=True, use_rnn=True).  Recorded: the initial state_dict, every sample, every info dict and the full
state_dict after updates FIX_SNAPSHOTS (the one that syncs the targets and the last).

Only OW-QMIX with double_q runs in the reference as it is.  Two expressions raise for use_rnn (DESIGN.md section 4):
  * double_q=False: ``q_next.argmax(dim=-1, keepdim=True).long().unsqueeze(-1)`` (wqmix_learner.py:114) adds one axis
    too many for the gather ("Index tensor must have the same number of dimensions");
  * CW-QMIX: ``batch.actions[group]`` (:178) subscripts an AgentGroupedTensor, which has no __getitem__.
For those cases the reference learner runs with exactly those expressions corrected in memory (``keepdim`` dropped,
``.group(group)``); nothing else of it changes.  ``<case>/corrected`` records which cases needed it."""
import inspect
import os
import textwrap

import numpy as np
import torch

from make_golden import ENV, HERE, _learner_cfg  # noqa: E402  (imports the reference and sets up sys.path)
from gymnasium.spaces import Discrete  # noqa: E402
from xuance.common import AgentGrouping, BaseCallback  # noqa: E402
from xuance.torch.rl_models.representations.rnn import Basic_RNN  # noqa: E402
from xuance.torch.rl_models.representations.agent_feature import AgentFeatureEncoder  # noqa: E402
from xuance.torch.rl_models.modules.identity_encoder import build_identity_encoder, IdentityFeatureFusion  # noqa: E402
from xuance.torch.rl_models.critics.base_critics import DiscreteActionValueCritic  # noqa: E402
from xuance.torch.rl_models.heads.q_mix_head import QMIX_Mixer, QMIX_FF_Mixer  # noqa: E402
from xuance.torch.rl_models.architectures.multi_agent.value_factorization import WeightedMixingQNetwork  # noqa: E402
import xuance.torch.learners.multi_agent_rl.wqmix_learner as reference_wqmix  # noqa: E402
from xuance.torch.learners.multi_agent_rl.wqmix_learner import WQMIX_Learner  # noqa: E402
from wqmix_refs import (FIX_N, FIX_OBS, FIX_A, FIX_S, FIX_HID, FIX_MIX, FIX_HYPER, FIX_FF, FIX_UPDATES, FIX_SNAPSHOTS,  # noqa
                        FIX_CASES, FIX_INFO_KEYS, fix_case_seed, fix_learner_config, fix_sample)

SAMPLE_FIELDS = ("obs", "actions", "rewards", "terminals", "agent_mask", "avail_actions")
CORRECTIONS = {"_forward_transitions": [(".argmax(dim=-1, keepdim=True).long().unsqueeze(-1)",
                                         ".argmax(dim=-1).long().unsqueeze(-1)")],
               "update": [("batch.actions[group]", "batch.actions.group(group)")]}


def corrected_learner():
    """WQMIX_Learner with the two raising expressions corrected (each must occur exactly once in the method)."""
    ns, attrs = dict(vars(reference_wqmix)), {}
    for name, subs in CORRECTIONS.items():
        src = textwrap.dedent(inspect.getsource(getattr(WQMIX_Learner, name)))
        for old, new in subs:
            assert src.count(old) == 1, (name, old)
            src = src.replace(old, new)
        exec(src, ns)
        attrs[name] = ns[name]
    return type("WQMIX_Learner", (WQMIX_Learner,), attrs)


def build_reference_model(seed):
    torch.manual_seed(seed)
    keys = [f"agent_{i}" for i in range(FIX_N)]
    init, act = torch.nn.init.orthogonal_, torch.nn.ReLU
    rep = Basic_RNN(input_shape=(FIX_OBS,), hidden_sizes=None, initialize=init, activation=act, device='cpu',
                    fc_hidden_sizes=[FIX_HID], recurrent_hidden_size=FIX_HID, N_recurrent_layers=1, dropout=0, rnn='GRU')
    enc = AgentFeatureEncoder(rep, build_identity_encoder(FIX_N, 'none', None, 'cpu'),
                              IdentityFeatureFusion(FIX_HID, 0, 'concat'))
    q = torch.nn.ModuleDict({'shared': DiscreteActionValueCritic(enc, Discrete(FIX_A), [FIX_HID], None, init, act, 'cpu')})
    grouping = AgentGrouping.shared(keys)
    model = WeightedMixingQNetwork(grouping, q, QMIX_Mixer(FIX_S, FIX_MIX, FIX_HYPER, FIX_N, 'cpu'),
                                   QMIX_FF_Mixer(FIX_S, FIX_FF, FIX_N, 'cpu'), use_rnn=True, device='cpu')
    return keys, grouping, model


def golden(out, agent, double_q):
    pre = f"{agent}/dq{int(double_q)}/"
    seed = fix_case_seed(agent, double_q)
    keys, grouping, model = build_reference_model(seed)
    for k, v in model.state_dict().items():
        out[f"{pre}init/{k}"] = v.numpy().copy()
    corrected = agent == "CWQMIX" or not double_q
    out[pre + "corrected"] = np.array(corrected)
    cls = corrected_learner() if corrected else WQMIX_Learner
    lrn = cls(_learner_cfg(**fix_learner_config(agent, double_q)), grouping, model, BaseCallback())
    out[pre + "total_iters"] = np.array(lrn.total_iters)
    rng = np.random.default_rng(seed)
    infos = []
    for it in range(FIX_UPDATES):
        s = fix_sample(rng, keys)
        for f in SAMPLE_FIELDS:
            x = np.stack([np.asarray(s[f][k]) for k in keys], axis=1)
            out[f"{pre}in{it}/{f}"] = x.astype(np.uint8) if f == "avail_actions" else x
        out[f"{pre}in{it}/filled"], out[f"{pre}in{it}/state"] = s["filled"], s["state"]
        info = lrn.update(s)
        infos.append([float(info[k]) for k in FIX_INFO_KEYS])
        if it in FIX_SNAPSHOTS:            # the whole state_dict, flattened in its key order (the init/ keys give shapes)
            out[f"{pre}after{it}"] = np.concatenate([v.numpy().reshape(-1) for v in model.state_dict().values()])
    out[pre + "infos"] = np.array(infos, np.float64)


if __name__ == "__main__":
    out = {"env": ENV}
    for agent, double_q in FIX_CASES:
        golden(out, agent, double_q)
    path = os.path.join(HERE, "wqmix_update.npz")
    np.savez_compressed(path, **out)
    print("wqmix_update.npz", os.path.getsize(path))
