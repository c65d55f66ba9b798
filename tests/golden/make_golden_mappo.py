"""Generate tests/golden/mappo_update.npz by running the UNMODIFIED reference (agi-brain/xuance v1.4.4 @ 4f0b05b).

Run in the build container only (needs /root/reference):   python tests/golden/make_golden_mappo.py
Reuses make_golden.py's reference import (read-only, with the oracle/ref_stubs import stubs) and environment-of-record
string; writes only this one fixture.

* buffer/<case>: MARL_OnPolicyBuffer (memory_tools_marl.py:63-270), 3 agents x 2 envs x 12 steps, for use_gae in
  {True, False} x ValueNorm {off, on} (except non-GAE with ValueNorm, which raises in the reference): store, finish_path of env 0 on a terminal step at t = 4 (value_next the Python
  float 0.0, as the reference agent passes it), a ValueNorm update, finish_path of both envs on the full buffer
  (np.float32 bootstraps), then sample() with per-agent advantage normalisation.
* learner: three MAPPO_Learner.update calls (mappo_learner.py:24-149) on CategoricalActor / CentralizedStateValueCritic /
  MultiAgentActorCritic (Basic_MLP 32, heads [32]), 3 agents, obs 12, A = 7, action masks, agent-mask zeros, value
  clipping, ValueNorm and Huber(delta = 1) on; update 1 puts every ratio outside the clip range."""
import os

import numpy as np
import torch

from make_golden import ENV, HERE, _learner_cfg  # noqa: E402  (imports the reference and sets up sys.path)
from gymnasium.spaces import Box, Discrete  # noqa: E402
from xuance.common import AgentGrouping, MultiAgentBaseCallback  # noqa: E402
from xuance.common.memory_tools_marl import MARL_OnPolicyBuffer  # noqa: E402
from xuance.torch.utils import ValueNorm  # noqa: E402
from xuance.torch.rl_models.representations.mlp import Basic_MLP  # noqa: E402
from xuance.torch.rl_models.representations.agent_feature import AgentFeatureEncoder  # noqa: E402
from xuance.torch.rl_models.modules.identity_encoder import build_identity_encoder, IdentityFeatureFusion  # noqa
from xuance.torch.rl_models import CategoricalActor, CentralizedStateValueCritic  # noqa: E402
from xuance.torch.rl_models.architectures import MultiAgentActorCritic  # noqa: E402
from xuance.torch.learners.multi_agent_rl.mappo_learner import MAPPO_Learner  # noqa: E402
from helpers import seeded_state_dict  # noqa: E402
from mappo_refs import mappo_buffer_steps, mappo_learner_batch  # noqa: E402

N_AGENTS, OBS, A = 3, 12, 7
KEYS = [f"agent_{i}" for i in range(N_AGENTS)]


def golden_buffer(out):
    grouping = AgentGrouping.shared(KEYS)
    n_envs, T = 2, 12
    for use_gae in (True, False):
        for use_vn in (False, True):
            if use_vn and not use_gae:
                # the reference cannot run this case: denormalize() returns [1, T+1] and `advantages[:-1]` then slices
                # the wrong axis (memory_tools_marl.py:234-235 raises a shape mismatch); DESIGN.md section 4
                continue
            case = f"buffer/gae{int(use_gae)}_vn{int(use_vn)}"
            rng = np.random.default_rng(5 + 2 * use_gae + use_vn)
            buf = MARL_OnPolicyBuffer(KEYS, None, {k: Box(-1, 1, (OBS,)) for k in KEYS}, {k: Discrete(A) for k in KEYS},
                                      n_envs, n_envs * T, use_gae=use_gae, use_advnorm=True, gamma=0.99, gae_lam=0.95,
                                      use_actions_mask=True, avail_actions_shape={k: (A,) for k in KEYS})
            vn = {"shared": ValueNorm(1)} if use_vn else None
            if use_vn:
                vn["shared"].update(torch.from_numpy(rng.normal(1.0, 4.0, (40, 1)).astype(np.float32)))
            steps, nexts, vn_upd = mappo_buffer_steps(rng, KEYS, n_envs, T, OBS, A)
            for t, st in enumerate(steps):
                buf.store(**st)
                if t == 4:
                    buf.finish_path(0, grouping, {k: 0.0 for k in KEYS}, vn)
                    if use_vn:
                        vn["shared"].update(torch.from_numpy(vn_upd.reshape(-1, 1)))
            for e in range(n_envs):
                buf.finish_path(e, grouping, nexts[e], vn)
            idx = rng.permutation(n_envs * T)[:14]
            s = buf.sample(idx)
            out[f"{case}/idx"] = idx
            for k in ("returns", "advantages"):
                out[f"{case}/{k}"] = np.stack([buf.data[k][a] for a in KEYS])            # [agent, env, T]
            out[f"{case}/sample_advantages"] = np.stack([s["advantages"][a] for a in KEYS])
            if use_vn:
                out[f"{case}/vn_state"] = np.array([vn["shared"].running_mean.item(),
                                                    vn["shared"].running_mean_sq.item(),
                                                    vn["shared"].debiasing_term.item()], np.float32)


def build_reference_model():
    g = AgentGrouping.shared(KEYS)
    init, act = torch.nn.init.orthogonal_, torch.nn.ReLU
    enc = lambda: AgentFeatureEncoder(Basic_MLP((OBS,), [32], None, init, act, 'cpu'),
                                      build_identity_encoder(N_AGENTS, 'none', None, 'cpu'),
                                      IdentityFeatureFusion(32, 0, 'concat'))
    actors = torch.nn.ModuleDict({'shared': CategoricalActor(enc(), [32], Discrete(A), None, init, act, 'cpu')})
    critics = torch.nn.ModuleDict({'shared': CentralizedStateValueCritic(g, torch.nn.ModuleDict({'shared': enc()}),
                                                                         None, [32], None, init, act, False, 'cpu')})
    return g, MultiAgentActorCritic(g, actors, critics, use_rnn=False, device='cpu')


def learner_cfg():
    return _learner_cfg(use_parameter_sharing=True, use_rnn=False, use_actions_mask=True, use_global_state=False,
                        clip_range=0.05, use_value_clip=True, value_clip_range=0.05, use_value_norm=True,
                        use_huber_loss=True, huber_delta=1.0, vf_coef=1.0, ent_coef=0.01, learning_rate=7e-4,
                        use_linear_lr_decay=False, end_factor_lr_decay=0.5, use_grad_clip=True, grad_clip_norm=10.0,
                        buffer_size=32, running_steps=3200, n_epochs=10, n_minibatch=1, parallels=8,
                        weight_decay=0.0)


def golden_learner(out):
    g, model = build_reference_model()
    model.load_state_dict(seeded_state_dict(model.state_dict(), 31))
    lrn = MAPPO_Learner(learner_cfg(), g, model, MultiAgentBaseCallback())
    rng = np.random.default_rng(77)
    infos = []
    for it in range(3):
        b = mappo_learner_batch(rng, it, 32, KEYS, OBS, A)
        sample = {k: ({a: b[k][i] for i, a in enumerate(KEYS)} if isinstance(b[k], np.ndarray) else b[k])
                  for k in b}
        info = lrn.update(sample)
        infos.append([info[f"shared/{k}"] for k in ("actor_loss", "critic_loss", "entropy", "predict_value")]
                     + [info["loss"], info["gradient_norm"], info["learning_rate"]])
        vn = lrn.value_normalizer["shared"]
        out[f"learner/vn_state/{it}"] = np.array([vn.running_mean.item(), vn.running_mean_sq.item(),
                                                  vn.debiasing_term.item()], np.float32)
    out["learner/infos"] = np.array(infos, np.float64)
    for k, v in model.state_dict().items():
        out[f"learner/final/{k}"] = v.detach().numpy().copy()


if __name__ == "__main__":
    out = {"env": ENV}
    golden_buffer(out)
    golden_learner(out)
    path = os.path.join(HERE, "mappo_update.npz")
    np.savez_compressed(path, **out)
    print("mappo_update.npz", os.path.getsize(path))
