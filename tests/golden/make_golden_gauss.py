"""Generate tests/golden/ppo_gauss_update.npz by running the UNMODIFIED reference (agi-brain/xuance v1.4.4 @ 4f0b05b).

Run in the build container only (needs /root/reference):   python tests/golden/make_golden_gauss.py
Reuses make_golden.py's reference import (read-only, with the oracle/ref_stubs import stubs), learner configuration and
environment-of-record string; writes only this one fixture, so the other fixtures are never rewritten."""
import os

import numpy as np
import torch

from make_golden import ENV, HERE, _learner_cfg  # noqa: E402  (imports the reference and sets up sys.path)
from xuance.common import BaseCallback  # noqa: E402
from xuance.torch.learners import PPO_Learner  # noqa: E402
from xuance.torch.rl_models.representations.mlp import Basic_MLP  # noqa: E402
from xuance.torch.rl_models.heads import GaussianActorHead, ValueHead  # noqa: E402
from xuance.torch.rl_models.architectures.single_agent.actor_critic import SharedActorCritic  # noqa: E402
from helpers import seeded_state_dict  # noqa: E402
from gauss_refs import ppo_gauss_samples  # noqa: E402


def golden_ppo_gauss(path=os.path.join(HERE, "ppo_gauss_update.npz")):
    """Three PPO updates of the reference learner on SharedActorCritic(Basic_MLP, GaussianActorHead(Tanh), ValueHead) for
    a 17-d observation and a 6-d Box action, B = 64.  Initial weights: helpers.seeded_state_dict (no construction-order
    contract).  Update 1 drives most ratios outside the clip range.  Keeps the info dicts, per-tensor digests of the final
    parameters and actor.log_std in full."""
    out = {"env": ENV}
    obs_dim, D, B = 17, 6, 64
    act = torch.nn.LeakyReLU
    rep = Basic_MLP((obs_dim,), [64], None, None, act, "cpu")
    actor = GaussianActorHead(64, [64], D, None, None, act, torch.nn.Tanh, "cpu")
    critic = ValueHead(64, [64], None, None, act, "cpu")
    model = SharedActorCritic(rep, actor, critic)
    model.load_state_dict(seeded_state_dict(model.state_dict(), 17))
    learner = PPO_Learner(_learner_cfg(), model, BaseCallback())
    out["total_iters"] = learner.total_iters
    rng = np.random.default_rng(23)
    infos = []
    for it in range(3):
        s = ppo_gauss_samples(rng, it, B, obs_dim, D)
        info = learner.update(**s)
        infos.append([info["actor_loss"], info["critic_loss"], info["entropy"], info["learning_rate"],
                      info["predict_value"], float(info["clip_ratio"])])
    out["infos"] = np.array(infos, dtype=np.float64)
    for k, v in model.state_dict().items():
        flat = v.detach().reshape(-1)
        out[f"final_head/{k}"] = flat[:64].numpy().copy()
        out[f"final_digest/{k}"] = np.array([flat.double().sum().item(), flat.double().abs().sum().item()])
    out["final/actor.log_std"] = model.actor.log_std.detach().numpy().copy()
    np.savez_compressed(path, **out)


if __name__ == "__main__":
    golden_ppo_gauss()
    print("ppo_gauss_update.npz", os.path.getsize(os.path.join(HERE, "ppo_gauss_update.npz")))
