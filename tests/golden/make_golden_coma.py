"""Generate tests/golden/coma_update.npz by running the UNMODIFIED reference COMA_Learner (agi-brain/xuance v1.4.4).

Run where the reference checkout exists (CPU only):   python tests/golden/make_golden_coma.py
Reuses make_golden.py's reference import (read-only, with the oracle/ref_stubs import stubs).

Per case (tests/coma_refs.py FIX_CASES: n in {1, 3} agents, action masks off and on, epsilon in {0, 0.3}): the reference's
model as coma_agents.py builds it (LayerNorm Basic_RNN GRU encoders for the actor and the critic, CategoricalActor,
CounterfactualCentralizedCritic, CounterfactualMultiAgentActorCritic with its target critics), and FIX_UPDATES updates
with gradient clipping across a target sync (sync_frequency = FIX_SYNC) on padded episode batches with dead agents
(tests/vdac_refs.py fix_sample).  Recorded: the initial state_dict, every sample, every info dict, the whole state_dict
after updates FIX_SNAPSHOTS and, on the last sample and the final weights, the acting outputs: the epsilon-mixed
probabilities, the deterministic (arg-max) actions and the target critics' Q of those actions, over whole sequences from
zero recurrent states."""
import os

import numpy as np
import torch

from make_golden import ENV, HERE, _learner_cfg  # noqa: E402  (imports the reference and sets up sys.path)
from gymnasium.spaces import Box, Discrete  # noqa: E402
from torch.nn.functional import one_hot  # noqa: E402
from xuance.common import AgentGrouping, MultiAgentBaseCallback  # noqa: E402
from xuance.torch.rl_models.representations.rnn import Basic_RNN  # noqa: E402
from xuance.torch.rl_models.representations.agent_feature import AgentFeatureEncoder  # noqa: E402
from xuance.torch.rl_models.modules.identity_encoder import build_identity_encoder, IdentityFeatureFusion  # noqa: E402
from xuance.torch.rl_models import CategoricalActor, CounterfactualCentralizedCritic  # noqa: E402
from xuance.torch.rl_models.architectures import CounterfactualMultiAgentActorCritic  # noqa: E402
from xuance.torch.learners.multi_agent_rl.coma_learner import COMA_Learner  # noqa: E402
from coma_refs import (FIX_OBS, FIX_A, FIX_S, FIX_HID, FIX_UPDATES, FIX_SNAPSHOTS, FIX_CASES, SAMPLE_FIELDS,  # noqa
                       INFO_KEYS, case_name, case_config, case_seed, fix_sample)


def build_reference_model(seed, n):
    torch.manual_seed(seed)
    keys = [f"agent_{i}" for i in range(n)]
    grouping = AgentGrouping.shared(keys)
    norm, init, act = torch.nn.LayerNorm, torch.nn.init.orthogonal_, torch.nn.ReLU

    def enc():
        rep = Basic_RNN(input_shape=(FIX_OBS,), hidden_sizes=None, normalize=norm, initialize=init, activation=act,
                        device="cpu", fc_hidden_sizes=[FIX_HID], recurrent_hidden_size=FIX_HID, N_recurrent_layers=1,
                        dropout=0, rnn="GRU")
        ide = build_identity_encoder(num_identities=n, mode="none", embedding_dim=None, device="cpu")
        fus = IdentityFeatureFusion(observation_feature_dim=rep.output_shapes['state'][0],
                                    identity_feature_dim=ide.output_dim, mode="concat")
        return AgentFeatureEncoder(representation=rep, identity_encoder=ide, fusion=fus)

    actors = torch.nn.ModuleDict({"shared": CategoricalActor(representation=enc(), actor_hidden_size=[FIX_HID],
                                                             action_space=Discrete(FIX_A), normalizer=norm,
                                                             initializer=init, activation=act, device="cpu")})
    critic = CounterfactualCentralizedCritic(grouping=grouping, representations=torch.nn.ModuleDict({"shared": enc()}),
                                             state_space=Box(-1, 1, (FIX_S,)),
                                             action_space={k: Discrete(FIX_A) for k in keys},
                                             critic_hidden_size=[FIX_HID, FIX_HID], normalizer=norm, initializer=init,
                                             activation=act, use_rnn=True, device="cpu")
    model = CounterfactualMultiAgentActorCritic(grouping=grouping, actors=actors, critics=critic, use_rnn=True,
                                                device="cpu")
    return keys, grouping, model


@torch.no_grad()
def acting(out, pre, lrn, model, s, eps, keys):
    """The reference's acting path (actor_critic.py:249-304 with deterministic=True, then get_values(target=True) on the
    joint one-hot of the chosen actions) over the sample's whole sequences from zero states."""
    batch = lrn.build_training_data(sample=s, use_actions_mask=lrn.use_actions_mask, use_global_state=True)
    B = batch.batch_size
    po = model(observations=batch.observations, agent_indices=batch.agent_indices, avail_actions=batch.avail_actions,
               rnn_states=model.init_actor_rnn_states(B), epsilon=eps, deterministic=True)
    acts = po.actions.group("shared").reshape(B, len(keys), -1)               # [B, n, T]
    joint = torch.cat([one_hot(acts[:, j], FIX_A) for j in range(len(keys))], dim=-1)   # [B, T, n*A]
    vo = model.get_values(states=batch.global_states, observations=batch.observations, joint_actions=joint,
                          agent_indices=batch.agent_indices, rnn_states=model.init_critic_rnn_states(B), target=True)
    q = vo.values.group("shared").reshape(B * len(keys) * acts.shape[-1], FIX_A)
    out[pre + "act/probs"] = po.distributions["shared"].probs.reshape(-1, FIX_A).numpy().copy()
    out[pre + "act/actions"] = acts.reshape(-1).numpy().astype(np.float32)
    out[pre + "act/q_taken"] = q.gather(-1, acts.reshape(-1, 1)).reshape(-1).numpy().copy()


def golden(out, case):
    n, masks, eps = case
    pre = case_name(case) + "/"
    seed = case_seed(case)
    keys, grouping, model = build_reference_model(seed, n)
    for k, v in model.state_dict().items():
        out[f"{pre}init/{k}"] = v.numpy().copy()
    lrn = COMA_Learner(_learner_cfg(**case_config(case)), grouping, model, MultiAgentBaseCallback())
    out[pre + "total_iters"] = np.array(lrn.total_iters)
    rng = np.random.default_rng(seed)
    infos = []
    for it in range(FIX_UPDATES):
        s = fix_sample(rng, keys, True)
        for f in SAMPLE_FIELDS:
            if f in ("state", "filled"):
                out[f"{pre}in{it}/{f}"] = np.asarray(s[f])
                continue
            x = np.stack([np.asarray(s[f][k]) for k in keys], axis=1)
            out[f"{pre}in{it}/{f}"] = x.astype(np.uint8) if f == "avail_actions" else x
        info = lrn.update(s, eps)
        infos.append([float(info[k]) for k in INFO_KEYS])
        if it in FIX_SNAPSHOTS:
            out[f"{pre}after{it}"] = np.concatenate([v.numpy().reshape(-1) for v in model.state_dict().values()])
    out[pre + "infos"] = np.array(infos, np.float64)
    acting(out, pre, lrn, model, s, eps, keys)


if __name__ == "__main__":
    out = {"env": ENV}
    for case in FIX_CASES:
        golden(out, case)
    path = os.path.join(HERE, "coma_update.npz")
    np.savez_compressed(path, **out)
    print("coma_update.npz", os.path.getsize(path))
