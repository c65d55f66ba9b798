"""Generate tests/golden/ddpg_td3_update.npz by running the UNMODIFIED reference (agi-brain/xuance v1.4.4 @ 4f0b05b).

Run in the build container only (needs the reference checkout):   python tests/golden/make_golden_ddpg_td3.py
Reuses make_golden.py's reference import (read-only, with the oracle/ref_stubs import stubs) and environment-of-record
string; writes only this one fixture.

Four updates each of DDPG_Learner (ddpg_learner.py:34-94) and TD3_Learner (td3_learner.py:35-100, actor_update_delay 2)
on the reference's own DeterministicActor / ActionValueCritic / TwinActionValueCritic / DeterministicActorCritic /
TwinDelayedActorCritic over Basic_MLP encoders (8-d observations, 32 units, heads [32], 3 action components with the
asymmetric bounds of tests/ddpg_refs.py, so that the clamp binds on tanh outputs by themselves), batch 48 with terminal
rows; once with use_grad_clip off (``<algo>/clip0/``) and once on with a binding norm (``<algo>/clip1/``).  Per update:
the info dict (NaN where a key is absent: TD3 logs Ploss on actor iterations only) and the full state_dict.  TD3's only
random draw is randn_like in Qtarget: the generator is reseeded before every update and the draw is recorded
(``noise``).  ``explore/`` holds the reference's OffPolicyAgent.exploration on given actions with a recorded draw."""
import os
from copy import deepcopy
from types import SimpleNamespace

import numpy as np
import torch

from make_golden import ENV, HERE, _learner_cfg  # noqa: E402  (imports the reference and sets up sys.path)
from gymnasium.spaces import Box  # noqa: E402
from xuance.common import BaseCallback  # noqa: E402
from xuance.torch.rl_models.representations.mlp import Basic_MLP  # noqa: E402
from xuance.torch.rl_models import DeterministicActor, ActionValueCritic, TwinActionValueCritic  # noqa: E402
from xuance.torch.rl_models.architectures import DeterministicActorCritic, TwinDelayedActorCritic  # noqa: E402
from xuance.torch.learners import DDPG_Learner, TD3_Learner  # noqa: E402
from xuance.torch.agents.core.off_policy import OffPolicyAgent  # noqa: E402
from ddpg_refs import (OBS, ACT, HIDDEN, LOW, HIGH, SIGMA, NOISE_CLIP, DELAY, N_UPDATES, CLIP_NORM,  # noqa: E402
                       fixture_batch, fixture_state_dict)

KEYS = {"ddpg": ["Qloss", "Ploss", "Qvalue", "actor_lr", "critic_lr"],
        "td3": ["Qloss", "Ploss", "QvalueA", "QvalueB", "actor_lr", "critic_lr"]}


def build_reference_model(twin):
    init, act = torch.nn.init.orthogonal_, torch.nn.ReLU
    space = Box(LOW, HIGH)
    rep = Basic_MLP((OBS,), [HIDDEN], None, init, act, 'cpu')
    actor = DeterministicActor(rep, [HIDDEN], space, None, init, act, torch.nn.Tanh, 'cpu')
    if twin:
        critic = TwinActionValueCritic(deepcopy(rep), space, [HIDDEN], None, init, act, 'cpu')
        model = TwinDelayedActorCritic(actor, critic, target_policy_noise=SIGMA, target_noise_clip=NOISE_CLIP)
    else:
        critic = ActionValueCritic(deepcopy(rep), space, [HIDDEN], None, init, act, 'cpu')
        model = DeterministicActorCritic(actor, critic)
    model.load_state_dict(fixture_state_dict(model.state_dict()))
    return model


def learner_cfg(clip):
    return _learner_cfg(learning_rate_actor=1e-3, learning_rate_critic=2e-3, tau=0.05, gamma=0.98,
                        use_grad_clip=clip, grad_clip_norm=CLIP_NORM, end_factor_lr_decay=0.5, parallels=4,
                        running_steps=64, start_training=0, training_frequency=1, actor_update_delay=DELAY)


def golden(out, algo, clip):
    twin = algo == "td3"
    pre = f"{algo}/clip{int(clip)}/"
    model = build_reference_model(twin)
    lrn = (TD3_Learner if twin else DDPG_Learner)(learner_cfg(clip), model, BaseCallback())
    out[pre + "total_iters"] = lrn.total_iters
    rng = np.random.default_rng(70 + 2 * twin + clip)
    infos, noises = [], []
    for it in range(N_UPDATES):
        s = fixture_batch(rng)
        seed = 1000 * (1 + twin) + 10 * clip + it
        torch.manual_seed(seed)
        noises.append(torch.randn(len(s["obs"]), ACT).numpy())
        torch.manual_seed(seed)
        info = lrn.update(**s)
        infos.append([float(info.get(k, np.nan)) for k in KEYS[algo]])
        for k, v in model.state_dict().items():
            out[f"{pre}it{it}/{k}"] = v.detach().numpy().copy()
    out[pre + "infos"] = np.array(infos, np.float64)
    if twin:
        out[pre + "noise"] = np.stack(noises)


def golden_exploration(out):
    rng = np.random.default_rng(5)
    a = torch.from_numpy(rng.uniform(-1.0, 1.0, (64, ACT)).astype(np.float32))
    agent = SimpleNamespace(e_greedy=None, noise_scale=0.7, n_envs=64, device='cpu', action_space=Box(LOW, HIGH),
                            actions_low_tensor=torch.as_tensor(LOW), actions_high_tensor=torch.as_tensor(HIGH))
    torch.manual_seed(11)
    noise = torch.randn_like(a)
    torch.manual_seed(11)
    x = OffPolicyAgent.exploration(agent, a)
    out.update({"explore/actions": a.numpy(), "explore/noise": noise.numpy(), "explore/noise_scale": 0.7,
                "explore/out": x.numpy()})


if __name__ == "__main__":
    out = {"env": ENV}
    for algo in ("ddpg", "td3"):
        for clip in (False, True):
            golden(out, algo, clip)
    golden_exploration(out)
    path = os.path.join(HERE, "ddpg_td3_update.npz")
    np.savez_compressed(path, **out)
    print("ddpg_td3_update.npz", os.path.getsize(path))
