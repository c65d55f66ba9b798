"""Generate tests/golden/ppg_update.npz by running the UNMODIFIED reference (agi-brain/xuance v1.4.4 @ 4f0b05b).

Run in the build container only (needs the reference checkout):   python tests/golden/make_golden_ppg.py
Reuses make_golden.py's reference import (read-only, with the oracle/ref_stubs import stubs).

Per case (tests/ppg_refs.py FIX_CASES: Categorical / Gaussian policy, n_minibatch 1 and 2, grad clipping off and on):
the reference's PhasicActorCritic (CategoricalActor or GaussianActor and two StateValueCritics on deep copies of one
Basic_MLP, as ppg_agent.py:47-93 builds it) and one full PPG_Learner cycle as ppg_agent.py:163-201 runs it: one index
array shuffled in place before every epoch of every phase, update_actor / update_critic, the relabel through the actor
and split_distributions, update_auxiliary_critic.  Recorded: the initial state_dict, the rows, the acting-time old_logp
(merge_distributions(old).log_prob(a)), every minibatch's indices and info dict, the state_dict and every parameter's
Adam state (step, exp_avg, exp_avg_sq; absent = never stepped) after each phase, and the relabelled parameters."""
import os
from copy import deepcopy

import numpy as np
import torch

from make_golden import ENV, HERE, _learner_cfg  # noqa: E402  (imports the reference and sets up sys.path)
from gymnasium.spaces import Box, Discrete  # noqa: E402
from xuance.common import BaseCallback  # noqa: E402
from xuance.torch.rl_models.representations.mlp import Basic_MLP  # noqa: E402
from xuance.torch.rl_models import CategoricalActor, GaussianActor, StateValueCritic  # noqa: E402
from xuance.torch.rl_models.architectures import PhasicActorCritic  # noqa: E402
from xuance.torch.rl_models.modules import split_distributions  # noqa: E402
from xuance.torch.learners.policy_gradient.ppg_learner import PPG_Learner  # noqa: E402
from ppg_refs import (FIX_OBS, FIX_HIDDEN, FIX_ROWS, FIX_A, FIX_D, FIX_NEPOCH, FIX_CASES, FIX_INFO_KEYS,  # noqa: E402
                      fix_learner_config, fix_rows, fix_case_seed)


def build_reference_model(kind, seed):
    torch.manual_seed(seed)
    init, act = torch.nn.init.orthogonal_, torch.nn.ReLU
    rep = Basic_MLP((FIX_OBS,), [FIX_HIDDEN], None, init, act, 'cpu')
    if kind == "gauss":
        actor = GaussianActor(rep, [FIX_HIDDEN], Box(-1, 1, (FIX_D,), np.float32), None, init, act, torch.nn.Tanh, 'cpu')
    else:
        actor = CategoricalActor(rep, [FIX_HIDDEN], Discrete(FIX_A), None, init, act, 'cpu')
    critic = StateValueCritic(deepcopy(rep), [FIX_HIDDEN], None, init, act, 'cpu')
    aux_critic = StateValueCritic(deepcopy(rep), [FIX_HIDDEN], None, init, act, 'cpu')
    return PhasicActorCritic(actor, critic, aux_critic)


def record_state(out, pre, model, opt):
    names = dict((id(p), n) for n, p in model.named_parameters())
    for k, v in model.state_dict().items():
        out[f"{pre}{k}"] = v.detach().numpy().copy()
    for p, st in opt.state.items():
        n = names[id(p)]
        out[f"{pre}adam/{n}/step"] = np.array(float(st["step"]))
        out[f"{pre}adam/{n}/exp_avg"] = st["exp_avg"].numpy().copy()
        out[f"{pre}adam/{n}/exp_avg_sq"] = st["exp_avg_sq"].numpy().copy()


def golden(out, kind, mb, clip):
    pre = f"{kind}/mb{mb}/clip{clip}/"
    seed = fix_case_seed(kind, mb, clip)
    model = build_reference_model(kind, seed)
    lrn = PPG_Learner(_learner_cfg(**fix_learner_config(mb, clip)), model, BaseCallback())
    out[pre + "total_iters"] = np.array(lrn.total_iters)
    for k, v in model.state_dict().items():
        out[f"{pre}init/{k}"] = v.detach().numpy().copy()
    obs, act, adv, ret = fix_rows(kind, seed)
    out[pre + "in/obs"], out[pre + "in/actions"], out[pre + "in/advantages"], out[pre + "in/returns"] = obs, act, adv, ret
    obs_t, act_t = torch.from_numpy(obs), torch.from_numpy(act if kind == "gauss" else act.astype(np.int64))
    with torch.no_grad():                  # acting: the distributions the rollout stored, and their log-probabilities
        old = split_distributions(model.actor(obs_t).distributions)
        out[pre + "in/old_logp"] = model.actor(obs_t).distributions.log_prob(act_t).numpy()
    np.random.seed(seed)
    indexes = np.arange(FIX_ROWS)
    batch = FIX_ROWS // mb
    for phase, update in (("actor", lrn.update_actor), ("critic", lrn.update_critic),
                          ("aux", lrn.update_auxiliary_critic)):
        if phase == "aux":                 # the relabel: get_actions over the buffer's observations
            with torch.no_grad():
                d = model.actor(obs_t).distributions
                if kind == "gauss":
                    out[pre + "relabel/mu"], out[pre + "relabel/std"] = d.mu.numpy(), d.std.numpy()
                else:
                    out[pre + "relabel/logits"] = d.logits.numpy()
                old = split_distributions(d)
        idxs, infos = [], []
        for _ in range(FIX_NEPOCH[phase]):
            np.random.shuffle(indexes)
            for start in range(0, FIX_ROWS, batch):
                idx = indexes[start:start + batch].copy()
                samples = {"obs": obs[idx], "actions": act_t[idx].numpy(), "advantages": adv[idx], "returns": ret[idx],
                           "aux_batch": {"old_dist": old[idx]}}
                info = update(**samples)
                idxs.append(idx)
                infos.append([float(info[k]) for k in FIX_INFO_KEYS[phase]])
        out[f"{pre}idx/{phase}"] = np.stack(idxs)
        out[f"{pre}info/{phase}"] = np.array(infos, np.float64)
        record_state(out, f"{pre}after/{phase}/", model, lrn.optimizer)


if __name__ == "__main__":
    out = {"env": ENV}
    for kind, mb, clip in FIX_CASES:
        golden(out, kind, mb, clip)
    path = os.path.join(HERE, "ppg_update.npz")
    np.savez_compressed(path, **out)
    print("ppg_update.npz", os.path.getsize(path))
