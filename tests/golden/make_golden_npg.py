"""Generate tests/golden/npg_update.npz by running the reference NPG_Learner (agi-brain/xuance v1.4.4 @ 4f0b05b).

Run in the build container only (needs the reference checkout):   python tests/golden/make_golden_npg.py
Reuses make_golden.py's reference import (read-only, with the oracle/ref_stubs import stubs).

The unmodified learner raises on its first update: npg_learner.py:38 reads ``model_output.distribution``, which
ModelOutput does not have (it has ``distributions``).  That AttributeError is recorded (``unpatched_error``), and then
exactly one correction is applied in memory: ``ModelOutput.distribution`` becomes an alias of ``distributions``.  Nothing
else of the reference changes.

Per case (tests/npg_refs.py FIX_CASES: Categorical / Gaussian policy, n_minibatch 1 and 2, grad clipping off and on):
the reference's ActorCritic (CategoricalActor or GaussianActor on a Basic_MLP, a StateValueCritic on a deep copy of it,
as npg_agent.py:37-67 builds it) and FIX_UPDATES learner updates on fixed minibatches.  Recorded: the initial
state_dict, the rows and minibatch indices, every update's info dict, state_dict and both optimisers' Adam state, each
actor tensor's natural gradient as the actor optimiser's step sees it (after the clip), and per actor tensor the kappa
and the conditioning ratio (lam + kappa s.s) / lam of the F the reference inverted."""
import os
from copy import deepcopy

import numpy as np
import torch

from make_golden import ENV, HERE, _learner_cfg  # noqa: E402  (imports the reference and sets up sys.path)
from gymnasium.spaces import Box, Discrete  # noqa: E402
from xuance.common import BaseCallback  # noqa: E402
from xuance.torch.rl_models.representations.mlp import Basic_MLP  # noqa: E402
from xuance.torch.rl_models import CategoricalActor, GaussianActor, StateValueCritic, ActorCritic  # noqa: E402
from xuance.torch.rl_models.modules import outputs  # noqa: E402
from xuance.torch.learners.policy_gradient.npg_learner import NPG_Learner  # noqa: E402
from npg_refs import (FIX_OBS, FIX_HIDDEN, FIX_A, FIX_D, FIX_CASES, FIX_INFO_KEYS, LAM,  # noqa: E402
                      fix_learner_config, fix_rows, fix_indices, fix_case_seed)


def build_reference_model(kind, seed):
    torch.manual_seed(seed)
    init, act = torch.nn.init.orthogonal_, torch.nn.ReLU
    rep = Basic_MLP((FIX_OBS,), [FIX_HIDDEN], None, init, act, 'cpu')
    if kind == "gauss":
        actor = GaussianActor(rep, [FIX_HIDDEN], Box(-1, 1, (FIX_D,), np.float32), None, init, act, torch.nn.Tanh, 'cpu')
    else:
        actor = CategoricalActor(rep, [FIX_HIDDEN], Discrete(FIX_A), None, init, act, 'cpu')
    critic = StateValueCritic(deepcopy(rep), [FIX_HIDDEN], None, init, act, 'cpu')
    return ActorCritic(actor, critic)


def record_adam(out, pre, model, opt):
    names = dict((id(p), n) for n, p in model.named_parameters())
    for p, st in opt.state.items():
        n = names[id(p)]
        out[f"{pre}adam/{n}/step"] = np.array(float(st["step"]))
        out[f"{pre}adam/{n}/exp_avg"] = st["exp_avg"].numpy().copy()
        out[f"{pre}adam/{n}/exp_avg_sq"] = st["exp_avg_sq"].numpy().copy()


def samples_of(obs, act, adv, ret, idx, kind):
    a = torch.from_numpy(act[idx]) if kind == "gauss" else torch.from_numpy(act[idx].astype(np.int64))
    return {"obs": torch.from_numpy(obs[idx]), "actions": a, "advantages": torch.from_numpy(adv[idx]),
            "returns": torch.from_numpy(ret[idx])}


def unpatched_error():
    """The unmodified learner's first update (npg_learner.py:38)."""
    assert not hasattr(outputs.ModelOutput, "distribution")
    kind, mb, clip = FIX_CASES[0]
    seed = fix_case_seed(kind, mb, clip)
    lrn = NPG_Learner(_learner_cfg(**fix_learner_config(mb, clip)), build_reference_model(kind, seed), BaseCallback())
    obs, act, adv, ret = fix_rows(kind, seed)
    try:
        lrn.update(**samples_of(obs, act, adv, ret, np.arange(len(ret)), kind))
    except AttributeError as e:
        return repr(e)
    raise AssertionError("the unmodified reference NPG_Learner no longer raises")


def golden(out, kind, mb, clip):
    pre = f"{kind}/mb{mb}/clip{clip}/"
    seed = fix_case_seed(kind, mb, clip)
    model = build_reference_model(kind, seed)
    lrn = NPG_Learner(_learner_cfg(**fix_learner_config(mb, clip)), model, BaseCallback())
    for k, v in model.state_dict().items():
        out[f"{pre}init/{k}"] = v.detach().numpy().copy()
    obs, act, adv, ret = fix_rows(kind, seed)
    out[pre + "in/obs"], out[pre + "in/actions"], out[pre + "in/advantages"], out[pre + "in/returns"] = obs, act, adv, ret
    idxs = fix_indices(mb, seed)
    out[pre + "idx"] = idxs
    names = dict((id(p), n) for n, p in model.named_parameters())
    actor_names = [names[id(p)] for p in model.actor.parameters()]
    out[pre + "actor_names"] = np.array(actor_names)
    fisher = []                 # per update: [kappa, ratio] per actor tensor, in parameter order
    orig_fisher = lrn.compute_fisher_information

    def fisher_wrap(param, obs_b, act_b):
        f_inv = orig_fisher(param, obs_b, act_b)
        lp = model(obs_b).distribution.log_prob(act_b)
        s = torch.autograd.grad(lp.sum(), param)[0].reshape(-1).double()
        kappa = lp.sum().item() / lrn.config.horizon_size
        fisher[-1].append([kappa, (LAM + kappa * float(s @ s)) / LAM])
        return f_inv
    lrn.compute_fisher_information = fisher_wrap
    nat = []
    orig_step = lrn.actor_optimizer.step

    def step_wrap(*a, **kw):
        nat.append({names[id(p)]: p.grad.detach().numpy().copy() for p in model.actor.parameters()})
        return orig_step(*a, **kw)
    lrn.actor_optimizer.step = step_wrap
    infos = []
    for u, idx in enumerate(idxs):
        fisher.append([])
        info = lrn.update(**samples_of(obs, act, adv, ret, idx, kind))
        infos.append([float(info[k]) for k in FIX_INFO_KEYS])
        after = f"{pre}after{u}/"
        for k, v in model.state_dict().items():
            out[after + k] = v.detach().numpy().copy()
        record_adam(out, after, model, lrn.actor_optimizer)
        record_adam(out, after, model, lrn.critic_optimizer)
        for n, g in nat[-1].items():
            out[f"{after}natgrad/{n}"] = g
    out[pre + "info"] = np.array(infos, np.float64)
    out[pre + "fisher"] = np.array(fisher, np.float64)


if __name__ == "__main__":
    out = {"env": ENV, "unpatched_error": np.array(unpatched_error())}
    outputs.ModelOutput.distribution = property(lambda self: self.distributions)
    for kind, mb, clip in FIX_CASES:
        golden(out, kind, mb, clip)
    path = os.path.join(HERE, "npg_update.npz")
    np.savez_compressed(path, **out)
    print("npg_update.npz", os.path.getsize(path))
