"""Generate tests/golden/vdac_update.npz by running the UNMODIFIED reference VDAC_Learner and IAC_Learner
(agi-brain/xuance v1.4.4).

Run in the build container only (needs the reference checkout):   python tests/golden/make_golden_vdac.py
Reuses make_golden.py's reference import (read-only, with the oracle/ref_stubs import stubs).

Per case (tests/vdac_refs.py FIX_CASES: VDAC with the VDN and the QMIX mixer, and IAC; use_rnn on and off; value clipping
and the Huber loss on and off): the reference's model as vdac_agents.py / iac_agents.py build it (LayerNorm Basic_RNN GRU
encoders with use_rnn, LayerNorm Basic_MLP ones without, CategoricalActor and StateValueCritic, VDN_Mixer or QMIX_Mixer),
and FIX_UPDATES updates on padded episode batches with dead agents and action masks (tests/vdac_refs.py fix_sample),
under a MultiAgentBaseCallback.  Recorded: the initial state_dict, every sample, every info dict and the whole
state_dict after updates FIX_SNAPSHOTS."""
import os

import numpy as np
import torch

from make_golden import ENV, HERE, _learner_cfg  # noqa: E402  (imports the reference and sets up sys.path)
from gymnasium.spaces import Discrete  # noqa: E402
from xuance.common import AgentGrouping, MultiAgentBaseCallback  # noqa: E402
from xuance.torch.rl_models.representations.rnn import Basic_RNN  # noqa: E402
from xuance.torch.rl_models.representations.mlp import Basic_MLP  # noqa: E402
from xuance.torch.rl_models.representations.agent_feature import AgentFeatureEncoder  # noqa: E402
from xuance.torch.rl_models.modules.identity_encoder import build_identity_encoder, IdentityFeatureFusion  # noqa: E402
from xuance.torch.rl_models import CategoricalActor, StateValueCritic  # noqa: E402
from xuance.torch.rl_models.heads import VDN_Mixer, QMIX_Mixer  # noqa: E402
from xuance.torch.rl_models.architectures import ValueDecompositionActorCritic, IndependentActorCritic  # noqa: E402
from xuance.torch.learners.multi_agent_rl.vdac_learner import VDAC_Learner  # noqa: E402
from xuance.torch.learners.multi_agent_rl.iac_learner import IAC_Learner  # noqa: E402
from vdac_refs import (FIX_N, FIX_OBS, FIX_A, FIX_S, FIX_T, FIX_HID, FIX_MIX_HID, FIX_HYPER_HID, FIX_UPDATES,  # noqa
                       FIX_SNAPSHOTS, FIX_CASES, SAMPLE_FIELDS, case_name, case_config, case_seed, fix_sample, info_keys)


def build_reference_model(seed, mixer, use_rnn):
    torch.manual_seed(seed)
    keys = [f"agent_{i}" for i in range(FIX_N)]
    grouping = AgentGrouping.shared(keys)
    norm, init, act = torch.nn.LayerNorm, torch.nn.init.orthogonal_, torch.nn.ReLU

    def enc():
        if use_rnn:
            rep = Basic_RNN(input_shape=(FIX_OBS,), hidden_sizes=None, normalize=norm, initialize=init, activation=act,
                            device="cpu", fc_hidden_sizes=[FIX_HID], recurrent_hidden_size=FIX_HID,
                            N_recurrent_layers=1, dropout=0, rnn="GRU")
        else:
            rep = Basic_MLP(input_shape=(FIX_OBS,), hidden_sizes=[FIX_HID], normalize=norm, initialize=init,
                            activation=act, device="cpu")
        ide = build_identity_encoder(num_identities=FIX_N, mode="none", embedding_dim=None, device="cpu")
        fus = IdentityFeatureFusion(observation_feature_dim=rep.output_shapes['state'][0],
                                    identity_feature_dim=ide.output_dim, mode="concat")
        return AgentFeatureEncoder(representation=rep, identity_encoder=ide, fusion=fus)

    actors = torch.nn.ModuleDict({"shared": CategoricalActor(representation=enc(), actor_hidden_size=[],
                                                             action_space=Discrete(FIX_A), normalizer=norm,
                                                             initializer=init, activation=act, device="cpu")})
    critics = torch.nn.ModuleDict({"shared": StateValueCritic(representation=enc(), critic_hidden_size=[],
                                                              normalizer=norm, initializer=init, activation=act,
                                                              device="cpu")})
    if mixer == "IAC":
        model = IndependentActorCritic(grouping=grouping, actors=actors, critics=critics, use_rnn=use_rnn,
                                       device="cpu")
    else:
        mix = VDN_Mixer() if mixer == "VDN" else QMIX_Mixer(FIX_S, FIX_MIX_HID, FIX_HYPER_HID, FIX_N, "cpu")
        model = ValueDecompositionActorCritic(grouping=grouping, actors=actors, critics=critics, mixer=mix,
                                              use_rnn=use_rnn, device="cpu")
    return keys, grouping, model


def golden(out, case):
    mixer, use_rnn, clip, huber = case
    pre = case_name(case) + "/"
    seed = case_seed(case)
    keys, grouping, model = build_reference_model(seed, mixer, use_rnn)
    for k, v in model.state_dict().items():
        out[f"{pre}init/{k}"] = v.numpy().copy()
    cls = IAC_Learner if mixer == "IAC" else VDAC_Learner
    lrn = cls(_learner_cfg(**case_config(case)), grouping, model, MultiAgentBaseCallback())
    out[pre + "total_iters"] = np.array(lrn.total_iters)
    rng = np.random.default_rng(seed)
    infos = []
    for it in range(FIX_UPDATES):
        s = fix_sample(rng, keys, use_rnn)
        for f in SAMPLE_FIELDS:
            if f in ("state", "filled"):
                if f in s:
                    out[f"{pre}in{it}/{f}"] = np.asarray(s[f])
                continue
            x = np.stack([np.asarray(s[f][k]) for k in keys], axis=1)
            out[f"{pre}in{it}/{f}"] = x.astype(np.uint8) if f == "avail_actions" else x
        info = lrn.update(s)
        infos.append([float(info[k]) for k in info_keys(mixer)])
        if it in FIX_SNAPSHOTS:
            out[f"{pre}after{it}"] = np.concatenate([v.numpy().reshape(-1) for v in model.state_dict().values()])
    out[pre + "infos"] = np.array(infos, np.float64)


if __name__ == "__main__":
    out = {"env": ENV}
    for case in FIX_CASES:
        golden(out, case)
    path = os.path.join(HERE, "vdac_update.npz")
    np.savez_compressed(path, **out)
    print("vdac_update.npz", os.path.getsize(path))
