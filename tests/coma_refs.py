"""Float64 restatement of K4C and the fixture settings shared by tests/golden/make_golden_coma.py, tests/oracle_coma.py
and the tests.

* ``k4c_ref``               the loss kernel's forward and its closed-form gradients in float64 (NumPy): the rules of
                            include/xb200.h K4C;
* ``reference_loss``        the reference's expressions (coma_learner.py:88-106, the epsilon mix of actor_critic.py:285
                            and torch's Categorical(probs) normalisation) on torch tensors;
* ``k4c_autograd``          ``reference_loss`` in float64 autograd;
* ``critic_input_reference`` the reference's critic-input assembly (centralized_critics.py:259-286: repeat, one_hot,
                            agent mask multiply, cat) on torch tensors.

Rows are in the buffer's (b, i, t) order, r = (b*n + i)*T + t."""
import numpy as np
import torch

from vdac_refs import fix_sample  # noqa: F401  (the same padded-episode samples with dead agents and action masks)

FIX_OBS, FIX_A, FIX_S, FIX_T, FIX_B, FIX_HID = 8, 5, 6, 6, 4, 16
FIX_UPDATES, FIX_SNAPSHOTS, FIX_SYNC = 4, (1, 3), 2
# (n agents, use_actions_mask, epsilon)
FIX_CASES = [(3, True, 0.3), (3, False, 0.0), (1, True, 0.0), (1, False, 0.3)]
SAMPLE_FIELDS = ("obs", "actions", "returns", "agent_mask", "avail_actions", "state", "filled")
INFO_KEYS = ("gradient_norm_actor", "learning_rate_actor", "learning_rate_critic", "actor_loss", "critic_loss",
             "advantage")


def case_name(case):
    n, masks, eps = case
    return f"n{n}_mask{int(masks)}_eps{eps}"


def case_seed(case):
    return 900 + 10 * FIX_CASES.index(case)


def case_config(case):
    n, masks, eps = case
    return dict(agent="COMA", use_rnn=True, use_actions_mask=masks, use_global_state=True, gamma=0.99,
                use_grad_clip=True, grad_clip_norm=0.5, learning_rate=7e-4, learning_rate_actor=7e-4,
                learning_rate_critic=1e-3, weight_decay=0, use_linear_lr_decay=False, end_factor_lr_decay=0.5,
                running_steps=96, episode_length=FIX_T, buffer_size=FIX_B, n_epochs=1, n_minibatch=1,
                use_parameter_sharing=True, n_agents=n, distributed_training=False, use_gae=True, gae_lambda=0.8,
                use_advnorm=False, clip_type=1, parallels=2, sync_frequency=FIX_SYNC, use_value_clip=False,
                value_clip_range=None, use_huber_loss=False, huber_delta=None, use_value_norm=False, vf_coef=None,
                ent_coef=None)


# ---------------------------------------------------------------- the loss
def k4c_ref(logits, avail, q, actions, ret, mask, eps, M=None, R_total=None):
    """Float64 K4C loss.  Returns (stats[3] = loss_a, loss_c, advantage mean; dlogits [R, A]; dq [R, A])."""
    f = lambda x: np.asarray(x, np.float64)
    logits, q, ret, mask = f(logits), f(q), f(ret), f(mask)
    R, A = logits.shape
    M = mask.sum() if M is None else M
    R_total = R if R_total is None else R_total
    av = np.ones((R, A), bool) if avail is None else np.asarray(avail)[:, :A] != 0
    z = np.where(av, logits, -1e10)
    p = np.exp(z - z.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    qm = (1.0 - eps) * p + eps / A
    wv = np.where(av, qm, 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        pi = wv / wv.sum(1, keepdims=True)
        rows, a = np.arange(R), np.asarray(actions).astype(np.int64)
        base = (pi * q).sum(1)
        adv = q[rows, a] - base
        logpi = np.log(pi[rows, a])
        w = mask / M
        coef = np.where(pi[rows, a] > 0, -adv * w * (1.0 - eps) * p[rows, a] / qm[rows, a], np.nan)
        dz = np.where(av, coef[:, None] * (np.eye(A)[a] - p), 0.0)
        td = (q[rows, a] - ret) * mask
        dq = np.zeros((R, A))
        dq[rows, a] = 2.0 * td * w
        stats = np.array([(-adv * logpi * mask).sum() / M, (td * td).sum() / M, adv.sum() / R_total])
    return stats, dz, dq


def reference_loss(lg, avail, q, actions, ret, mask, eps):
    """coma_learner.py:88-106 with the model's epsilon mix on torch tensors.  Returns (loss_a, loss_c, advantages)."""
    A = lg.shape[-1]
    z = lg if avail is None else torch.where(avail[:, :A] != 0, lg, torch.full_like(lg, -1e10))
    probs = torch.distributions.Categorical(logits=z).probs
    probs = (1 - eps) * probs + eps * 1 / A                              # actor_critic.py:285
    pi_probs = torch.distributions.Categorical(probs=probs).probs
    if avail is not None:
        pi_probs = pi_probs.clone()
        pi_probs[avail[:, :A] == 0] = 0.0
        pi_probs = pi_probs / pi_probs.sum(dim=-1, keepdim=True)
    a = actions.long().unsqueeze(-1)
    baseline = (pi_probs * q).sum(-1).reshape(-1)
    pi_taken = pi_probs.gather(-1, a)
    q_taken = q.gather(-1, a).reshape(-1)
    log_pi_taken = torch.log(pi_taken).reshape(-1)
    advantages = (q_taken - baseline).detach()
    loss_a = -(advantages * log_pi_taken * mask).sum() / mask.sum()
    td_error = (q_taken - ret) * mask
    loss_c = (td_error ** 2).sum() / mask.sum()
    return loss_a, loss_c, advantages


def k4c_autograd(logits, avail, q, actions, ret, mask, eps):
    """reference_loss in float64 autograd.  Returns (stats[3], dlogits, dq)."""
    t = lambda x: None if x is None else torch.as_tensor(np.asarray(x, np.float64))
    lg, qq = t(logits).requires_grad_(True), t(q).requires_grad_(True)
    la, lc, adv = reference_loss(lg, t(avail), qq, t(actions), t(ret), t(mask), eps)
    (la + lc).backward()
    return np.array([la.item(), lc.item(), adv.mean().item()]), lg.grad.numpy(), qq.grad.numpy()


# ---------------------------------------------------------------- the critic input
def critic_input_reference(state, feat, actions, A):
    """centralized_critics.py:259-286 (use_rnn): state [B, T, S], feat [B, n, T, F], actions [B, n, T] ->
    [B, n, T, S + F + n*A]."""
    B, n, T = actions.shape
    joint = torch.cat([torch.nn.functional.one_hot(actions[:, j].long(), A) for j in range(n)], dim=-1).float()
    agent_mask = (1 - torch.eye(n, dtype=torch.float32)).unsqueeze(-1)
    agent_mask = agent_mask.repeat(1, 1, A).reshape(n, -1).unsqueeze(0).unsqueeze(2)
    expanded_states = state.unsqueeze(1).repeat(1, n, 1, 1)
    expanded_joint_actions = joint.unsqueeze(1).repeat(1, n, 1, 1)
    return torch.cat([expanded_states, feat, expanded_joint_actions * agent_mask], dim=-1)
