"""Torch-CPU oracle of the COMA learner, pinned to tests/golden/coma_update.npz (generated from the unmodified reference).
``COMALearnerOracle`` restates COMA_Learner.update (coma_learner.py:45-153) with torch autograd of the reference's
expressions (tests/coma_refs.py reference_loss and critic_input_reference), two torch.optim.Adam(eps=1e-5) with
clip_grad_norm_ and LinearLR each, and the target sync, on a CPU copy of the product model in which each GRU runs through
nn.GRU (tests/oracle_mappo_rnn.py CPUBasicRNN)."""
import copy

import numpy as np
import torch
import torch.nn as nn

from oracle_mappo_rnn import CPUBasicRNN
from coma_refs import FIX_OBS, FIX_A, FIX_S, FIX_HID, case_config, reference_loss, critic_input_reference


def build_product_model(case, device):
    """The product's model for a fixture case (the layout COMA_Agents builds), on ``device``."""
    from xuance_b200.common import AgentGrouping
    from xuance_b200.common.spaces import Box, Discrete
    from xuance_b200.torch.rl_models import (CategoricalActor, Basic_RNN_K13, CounterfactualCentralizedCritic,
                                             CounterfactualMultiAgentActorCritic)
    from xuance_b200.torch.rl_models.qmix import AgentFeatureEncoder
    n = case[0]
    keys = [f"agent_{i}" for i in range(n)]
    grouping = AgentGrouping.shared(keys)
    norm, init, act = nn.LayerNorm, nn.init.orthogonal_, nn.ReLU

    def enc():
        return AgentFeatureEncoder(Basic_RNN_K13(input_shape=(FIX_OBS,), normalize=norm, initialize=init,
                                                 activation=act, device=device, fc_hidden_sizes=[FIX_HID],
                                                 recurrent_hidden_size=FIX_HID, N_recurrent_layers=1, rnn="GRU"))

    actors = nn.ModuleDict({"shared": CategoricalActor(enc(), [FIX_HID], Discrete(FIX_A), norm, init, act, device)})
    critic = CounterfactualCentralizedCritic(grouping, nn.ModuleDict({"shared": enc()}), Box(-1, 1, (FIX_S,)),
                                             {k: Discrete(FIX_A) for k in keys}, [FIX_HID, FIX_HID], norm, init, act,
                                             use_rnn=True, device=device)
    model = CounterfactualMultiAgentActorCritic(grouping, actors, critic, use_rnn=True, device=device)
    return grouping, model.to(device)


def fixture_batch(g, pre, it):
    """A fixture sample as (b, i, t)-ordered CPU tensors: obs [B*n, T, obs], actions / returns / mask [R], avail
    [R, A], state [B, T, S]."""
    x = lambda f: torch.from_numpy(np.asarray(g[f"{pre}in{it}/{f}"]))
    obs = x("obs")
    B, n, T = obs.shape[:3]
    rows = lambda f: x(f).reshape(-1).to(torch.float32)
    mask = x("agent_mask").to(torch.float32) * x("filled").to(torch.float32)[:, None, :]
    return dict(obs=obs.reshape(B * n, T, -1), actions=rows("actions"), returns=rows("returns"), mask=mask.reshape(-1),
                avail=x("avail_actions").reshape(-1, FIX_A), state=x("state").to(torch.float32), B=B, n=n, T=T)


class COMALearnerOracle:
    def __init__(self, model, case, cfg=None):
        self.case, self.cfg = case, case_config(case) if cfg is None else cfg
        self.m = copy.deepcopy(model).cpu()
        g = "shared"
        for enc in (self.m.actors[g].representation, self.m.critics.representations[g],
                    self.m.target_critics.representations[g]):
            enc.obs_representation = CPUBasicRNN(enc.obs_representation)
        c = self.cfg
        total = (c["running_steps"] // c["episode_length"]) // c["buffer_size"]
        self.opt = {"actor": torch.optim.Adam(self.m.actors.parameters(), lr=c["learning_rate_actor"], eps=1e-5),
                    "critic": torch.optim.Adam(self.m.critics.parameters(), lr=c["learning_rate_critic"], eps=1e-5)}
        self.sch = {k: torch.optim.lr_scheduler.LinearLR(v, 1.0, c["end_factor_lr_decay"], total)
                    for k, v in self.opt.items()}
        self.iterations = 0

    def state_dict(self):
        return self.m.state_dict()

    def q_values(self, b, critics):
        feat = critics.representations["shared"](b["obs"]).embeddings
        x = critic_input_reference(b["state"], feat.reshape(b["B"], b["n"], b["T"], -1),
                                   b["actions"].reshape(b["B"], b["n"], b["T"]), critics.critic_head.n_actions)
        return critics.critic_head(x.reshape(-1, x.shape[-1]))

    def update(self, b, eps):
        c, m = self.cfg, self.m
        self.iterations += 1
        a = m.actors["shared"]
        logits = a.actor_head.logits(a.representation(b["obs"]).embeddings).reshape(-1, a.action_dim)
        q = self.q_values(b, m.critics)
        avail = b["avail"] if c["use_actions_mask"] else None
        la, lc, adv = reference_loss(logits, avail, q, b["actions"], b["returns"], b["mask"], eps)
        self.opt["critic"].zero_grad()
        lc.backward()
        nn.utils.clip_grad_norm_(m.critics.parameters(), c["grad_clip_norm"])
        self.opt["critic"].step()
        self.sch["critic"].step()
        if self.iterations % c["sync_frequency"] == 0:
            with torch.no_grad():
                for ep, tp in zip(m.critics.parameters(), m.target_critics.parameters()):
                    tp.copy_(ep)
        self.opt["actor"].zero_grad()
        la.backward()
        gn = float(nn.utils.clip_grad_norm_(m.actors.parameters(), c["grad_clip_norm"]))
        self.opt["actor"].step()
        self.sch["actor"].step()
        return {"gradient_norm_actor": gn, "learning_rate_actor": self.opt["actor"].param_groups[0]["lr"],
                "learning_rate_critic": self.opt["critic"].param_groups[0]["lr"], "actor_loss": la.item(),
                "critic_loss": lc.item(), "advantage": adv.mean().item()}
