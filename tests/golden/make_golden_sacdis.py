"""Generate tests/golden/sacdis_update.npz by running the UNMODIFIED reference (agi-brain/xuance v1.4.4 @ 4f0b05b).

Run in the build container only (needs the reference checkout):   python tests/golden/make_golden_sacdis.py
Reuses make_golden.py's reference import (read-only, with the oracle/ref_stubs import stubs) and environment-of-record
string; writes only this one fixture.

Three SACDIS_Learner.update calls (sacdis_learner.py:41-129) on the reference's own CategoricalActor /
TwinDiscreteActionValueCritic / SoftActorCriticDiscrete over Basic_MLP encoders (8-d observations, 32 units, heads [32],
A = 5), batch 48 (tests/sacdis_refs.py: rows scaled so that some probabilities underflow to exactly 0 and some to
subnormals; q1 == q2 in every other column at the first update; terminal rows):
* ``auto0/``: use_automatic_entropy_tuning False, as the reference runs it;
* ``auto1/``: use_automatic_entropy_tuning True.  The reference learner reads ``model.action_space.n`` for its target
  entropy, an attribute SoftActorCriticDiscrete does not have, so its constructor raises AttributeError (recorded in
  ``note/auto_alpha_error``).  The updates are recorded with ``model.action_space = Discrete(A)`` set on the reference
  INSTANCE before construction - a state change in the harness, not a source change (DESIGN.md section 4)."""
import os
from copy import deepcopy

import numpy as np
import torch

from make_golden import ENV, HERE, _learner_cfg  # noqa: E402  (imports the reference and sets up sys.path)
from gymnasium.spaces import Discrete  # noqa: E402
from xuance.common import BaseCallback  # noqa: E402
from xuance.torch.rl_models.representations.mlp import Basic_MLP  # noqa: E402
from xuance.torch.rl_models import CategoricalActor, TwinDiscreteActionValueCritic  # noqa: E402
from xuance.torch.rl_models.architectures import SoftActorCriticDiscrete  # noqa: E402
from xuance.torch.learners import SACDIS_Learner  # noqa: E402
from sacdis_refs import OBS, A_FIX, HIDDEN, fixture_batch, fixture_state_dict  # noqa: E402


def build_reference_model():
    init, act = torch.nn.init.orthogonal_, torch.nn.ReLU
    rep = Basic_MLP((OBS,), [HIDDEN], None, init, act, 'cpu')
    actor = CategoricalActor(rep, [HIDDEN], Discrete(A_FIX), None, init, act, 'cpu')
    critic = TwinDiscreteActionValueCritic(deepcopy(rep), Discrete(A_FIX), [HIDDEN], None, init, act, 'cpu')
    model = SoftActorCriticDiscrete(actor=actor, critic=critic)
    model.load_state_dict(fixture_state_dict(model.state_dict()))
    return model


def learner_cfg(auto):
    return _learner_cfg(learning_rate_actor=1e-3, learning_rate_critic=1e-3, tau=0.005, alpha=0.2, gamma=0.99,
                        use_automatic_entropy_tuning=auto, use_grad_clip=False, end_factor_lr_decay=0.7, parallels=4,
                        running_steps=100000, start_training=0, training_frequency=1)


def golden(out, auto):
    model = build_reference_model()
    if auto:
        try:
            SACDIS_Learner(learner_cfg(True), model, BaseCallback())
            raise RuntimeError("the reference learner constructed with auto-tuning on: the recorded defect is gone")
        except AttributeError as e:
            out["note/auto_alpha_error"] = np.array(str(e))
        model.action_space = Discrete(A_FIX)
    lrn = SACDIS_Learner(learner_cfg(auto), model, BaseCallback())
    out[f"auto{int(auto)}/total_iters"] = lrn.total_iters
    rng = np.random.default_rng(90 + auto)
    keys = ["Qloss", "Ploss", "Qvalue", "actor_lr", "critic_lr"] + (["alpha_loss", "alpha"] if auto else [])
    infos = []
    for it in range(3):
        s = fixture_batch(rng)
        if it == 0:
            with torch.no_grad():
                p = model.actor(torch.from_numpy(s["obs"])).distributions.probs
            out[f"auto{int(auto)}/probs0"] = p.numpy()
        info = lrn.update(**s)
        infos.append([float(info[k]) for k in keys])
    out[f"auto{int(auto)}/infos"] = np.array(infos, np.float64)
    for k, v in model.state_dict().items():
        out[f"auto{int(auto)}/final/{k}"] = v.detach().numpy().copy()


if __name__ == "__main__":
    out = {"env": ENV}
    golden(out, False)
    golden(out, True)
    path = os.path.join(HERE, "sacdis_update.npz")
    np.savez_compressed(path, **out)
    print("sacdis_update.npz", os.path.getsize(path))
