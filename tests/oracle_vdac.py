"""Torch-CPU oracle of the VDAC / IAC learners, pinned to tests/golden/vdac_update.npz (generated from the unmodified
reference).  ``VDACLearnerOracle`` restates VDAC_Learner.update / IAC_Learner.update (vdac_learner.py:24-147,
iac_learner.py:179-289) with torch autograd of the reference's expressions (tests/vdac_refs.py reference_loss),
torch.optim.Adam(eps=1e-5), clip_grad_norm_ and LinearLR, on a CPU copy of the product model in which each GRU runs
through nn.GRU (tests/oracle_mappo_rnn.py CPUBasicRNN) and the QMIX mixer is restated in torch (q_mix_head.py:28-95)."""
import copy

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle_mappo_rnn import CPUBasicRNN
from vdac_refs import (FIX_N, FIX_OBS, FIX_A, FIX_S, FIX_HID, FIX_MIX_HID, FIX_HYPER_HID, case_config, reference_loss)


def build_product_model(case, device):
    """The product's model for a fixture case (the layout VDAC_Agents / IAC_Agents build), on ``device``."""
    from xuance_b200.common import AgentGrouping
    from xuance_b200.common.spaces import Discrete
    from xuance_b200.torch.rl_models import (CategoricalActor, StateValueCritic, Basic_RNN_K13, Basic_MLP, QMIX_Mixer,
                                             VDN_mixer, IndependentActorCritic, ValueDecompositionActorCritic)
    from xuance_b200.torch.rl_models.qmix import AgentFeatureEncoder
    mixer, use_rnn = case[0], case[1]
    keys = [f"agent_{i}" for i in range(FIX_N)]
    grouping = AgentGrouping.shared(keys)
    norm, init, act = nn.LayerNorm, nn.init.orthogonal_, nn.ReLU

    def enc():
        if use_rnn:
            return AgentFeatureEncoder(Basic_RNN_K13(input_shape=(FIX_OBS,), normalize=norm, initialize=init,
                                                     activation=act, device=device, fc_hidden_sizes=[FIX_HID],
                                                     recurrent_hidden_size=FIX_HID, N_recurrent_layers=1, rnn="GRU"))
        return AgentFeatureEncoder(Basic_MLP(input_shape=(FIX_OBS,), hidden_sizes=[FIX_HID], normalize=norm,
                                             initialize=init, activation=act, device=device))

    actors = nn.ModuleDict({"shared": CategoricalActor(enc(), [], Discrete(FIX_A), norm, init, act, device)})
    critics = nn.ModuleDict({"shared": StateValueCritic(enc(), [], norm, init, act, device)})
    if mixer == "IAC":
        model = IndependentActorCritic(grouping, actors, critics, use_rnn=use_rnn, device=device)
    else:
        mix = VDN_mixer() if mixer == "VDN" else QMIX_Mixer(FIX_S, FIX_MIX_HID, FIX_HYPER_HID, FIX_N, device)
        model = ValueDecompositionActorCritic(grouping, actors, critics, mix, use_rnn=use_rnn, device=device)
    return grouping, model.to(device)


def qmix_cpu(mixer, q, s):
    """q_mix_head.py:28-95 in torch: q [rows, n], s [rows, S] -> [rows]."""
    n, H = mixer.n_agents, mixer.dim_hidden
    w1 = torch.abs(mixer.hyper_w_1(s)).view(-1, n, H)
    b1 = mixer.hyper_b_1(s).view(-1, 1, H)
    hidden = F.elu(torch.bmm(q.view(-1, 1, n), w1) + b1)
    w2 = torch.abs(mixer.hyper_w_2(s)).view(-1, H, 1)
    b2 = mixer.hyper_b_2(s).view(-1, 1, 1)
    return (torch.bmm(hidden, w2) + b2).reshape(-1)


def fixture_batch(g, pre, it, use_rnn):
    """A fixture sample as (b, i, t)-ordered CPU tensors: obs [B*n, T, obs] (use_rnn) or [B*n, obs], rows [R], avail
    [R, A], state [B*T, S] and the loss mask."""
    x = lambda f: torch.from_numpy(np.asarray(g[f"{pre}in{it}/{f}"]))
    obs = x("obs")
    B, n = obs.shape[0], obs.shape[1]
    obs = obs.reshape(B * n, *obs.shape[2:])
    rows = lambda f: x(f).reshape(-1).to(torch.float32)
    mask = x("agent_mask").to(torch.float32)
    if use_rnn:
        mask = mask * x("filled").to(torch.float32)[:, None, :]
    st = x("state")
    return dict(obs=obs, actions=rows("actions"), adv=rows("advantages"), values=rows("values"),
                returns=rows("returns"), mask=mask.reshape(-1), avail=x("avail_actions").reshape(-1, FIX_A),
                state=st.reshape(-1, st.shape[-1]).to(torch.float32), B=B, n=n, T=obs.shape[1] if use_rnn else 1)


class VDACLearnerOracle:
    def __init__(self, model, case, row_order=False):
        self.case, self.cfg = case, case_config(case)
        self.m = copy.deepcopy(model).cpu()
        if case[1]:
            for part in (self.m.actors["shared"], self.m.critics["shared"]):
                part.representation.obs_representation = CPUBasicRNN(part.representation.obs_representation)
        self.mode = {"IAC": 0, "VDN": 1, "QMIX": 2}[case[0]]
        self.row_order = int(row_order and case[1] and self.mode != 0)
        c = self.cfg
        self.optimizer = torch.optim.Adam(self.m.parameters(), lr=c["learning_rate"], eps=1e-5)
        total = (c["running_steps"] // c["episode_length"]) // c["buffer_size"] if case[1] else \
            c["running_steps"] // c["buffer_size"]
        self.scheduler = torch.optim.lr_scheduler.LinearLR(self.optimizer, 1.0, c["end_factor_lr_decay"], total)

    def state_dict(self):
        return self.m.state_dict()

    def update(self, b):
        c, m = self.cfg, self.m
        a, cr = m.actors["shared"], m.critics["shared"]
        logits = a.actor_head.logits(a.representation(b["obs"]).embeddings).reshape(-1, FIX_A)
        v = cr.critic_head(cr.representation(b["obs"]).embeddings).reshape(-1)
        if self.mode == 2:
            v = qmix_cpu(m.v_tot, v.reshape(b["B"], b["n"], b["T"]).transpose(1, 2).reshape(-1, b["n"]), b["state"])
        al, cl, el, pred, loss = reference_loss(
            logits, b["avail"], b["actions"], b["adv"], v, b["values"], b["returns"], b["mask"], b["n"], b["T"],
            self.mode, self.row_order, c["value_clip_range"] if c["use_value_clip"] else 0.0,
            c["huber_delta"] if c["use_huber_loss"] else 0.0, c["vf_coef"], c["ent_coef"])
        self.optimizer.zero_grad()
        loss.backward()
        gn = float(nn.utils.clip_grad_norm_(m.parameters(), c["grad_clip_norm"]))
        self.optimizer.step()
        if self.mode == 0 or c["use_linear_lr_decay"]:
            self.scheduler.step()
        return {"actor_loss": al.item(), "critic_loss": cl.item(), "entropy": el.item(),
                "predict_value": pred.mean().item(), "loss": loss.item(), "gradient_norm": gn,
                "learning_rate": self.optimizer.param_groups[0]["lr"]}

    def info_row(self, info):
        """The info in the fixture's column order (vdac_refs.info_keys)."""
        if self.mode == 0:
            return [info[k] for k in ("gradient_norm", "actor_loss", "critic_loss", "entropy", "loss", "predict_value",
                                      "learning_rate")]
        return [info[k] for k in ("actor_loss", "critic_loss", "entropy", "predict_value", "gradient_norm",
                                  "learning_rate", "loss")]
