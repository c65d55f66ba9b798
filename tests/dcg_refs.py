"""Float64 restatements of the K9C Deep Coordination Graph kernels (xb_dcg_greedy, xb_dcg_q_fwd, xb_dcg_td_fwd_bwd,
xb_dcg_q_bwd) in the order include/xb200.h documents, so the GPU results must equal them bit for bit.  Pure torch on
the CPU, vectorised over instances: every step is one IEEE operation per element, so the order is the kernel's.

Instances are given flat: f [R, n, A] float32 utility outputs, pay [2, R, E, A*A] float32 raw payoff outputs (the two
orientations), edges as lists of (from, to)."""
import numpy as np
import torch

NEG = -1e10


def graph_edges(n, graph_type):
    """coordination_graph.py:122-134 restated: the edge lists of the five graph types."""
    if graph_type == "CYCLE":
        return [(i, i + 1) for i in range(n - 1)] + [(n - 1, 0)]
    if graph_type == "LINE":
        return [(i, i + 1) for i in range(n - 1)]
    if graph_type == "STAR":
        return [(0, i + 1) for i in range(n - 1)]
    if graph_type == "VDN":
        return []
    if graph_type == "FULL":
        return [(j, i + j + 1) for j in range(n - 1) for i in range(n - j - 1)]
    raise AttributeError(graph_type)


def payoff_matrix(pay, E):
    """F_e[i][j] = float32((P0[i*A+j] + P1[j*A+i]) / 2) / E in float64: [R, E, A, A]."""
    R, A = pay.shape[1], int(round(pay.shape[-1] ** 0.5))
    p0 = pay[0].reshape(R, E, A, A)
    p1 = pay[1].reshape(R, E, A, A).transpose(-1, -2)
    return ((p0 + p1) * 0.5).double() / E


def greedy_ref(f, pay, edges, n_iter, normalize, avail=None):
    """The max-plus greedy: (actions int64 [R, n], U float64 [R, n, A])."""
    R, n, A = f.shape
    E = len(edges)
    u = f.double() / n
    U = (u + 0.0) + 0.0
    if E > 0 and n_iter > 0:
        F = payoff_matrix(pay, E)                                        # [R, E, i, j]
        fr = torch.tensor([e[0] for e in edges])
        to = torch.tensor([e[1] for e in edges])
        mf = torch.zeros(R, E, A, dtype=torch.float64)                   # from -> to, over a_to
        mb = torch.zeros(R, E, A, dtype=torch.float64)                   # to -> from, over a_from
        for _ in range(n_iter):
            nf = ((U[:, fr] - mb).unsqueeze(-1) + F).amax(dim=-2)        # max over i
            nb = ((U[:, to] - mf).unsqueeze(-2) + F).amax(dim=-1)        # max over j
            if normalize:
                sf = torch.zeros(R, E, 1, dtype=torch.float64)
                sb = torch.zeros(R, E, 1, dtype=torch.float64)
                for a in range(A):                                       # the means, summed in action order
                    sf = sf + nf[..., a:a + 1]
                    sb = sb + nb[..., a:a + 1]
                nf, nb = nf - sf / A, nb - sb / A
            mf, mb = nf, nb
            sum_f = torch.zeros(R, n, A, dtype=torch.float64)
            sum_b = torch.zeros(R, n, A, dtype=torch.float64)
            for e, (i, j) in enumerate(edges):                           # edge-index order
                sum_f[:, j] = sum_f[:, j] + mf[:, e]
                sum_b[:, i] = sum_b[:, i] + mb[:, e]
            U = (u + sum_f) + sum_b
    Um = U if avail is None else torch.where(torch.as_tensor(avail) != 0, U, torch.tensor(NEG, dtype=torch.float64))
    return Um.argmax(dim=-1), U


def q_ref(f, pay, edges, acts, use_payoff):
    """q_dcg: (sum_v u_v[a_v]) + (sum_e F_e[a_from][a_to]) per instance, sums in order from 0 (float64 [R])."""
    R, n, A = f.shape
    E = len(edges)
    acts = torch.as_tensor(acts).long()
    u = f.double() / n
    su = torch.zeros(R, dtype=torch.float64)
    for v in range(n):
        su = su + u[:, v].gather(-1, acts[:, v:v + 1]).squeeze(-1)
    if not use_payoff or E == 0:
        return su
    F = payoff_matrix(pay, E)
    sp = torch.zeros(R, dtype=torch.float64)
    rows = torch.arange(R)
    for e, (i, j) in enumerate(edges):
        sp = sp + F[rows, e, acts[:, i], acts[:, j]]
    return su + sp


def td_ref(q_eval, q_next, v, v_next, rewards, terminals, filled, filled_sum, gamma, rows_total):
    """The TD kernel in its order: (dq float64 [B*T], dv float32 or None, stats float64 [2])."""
    B, n, T = rewards.shape
    rs = torch.zeros(B, T, dtype=torch.float32)
    for i in range(n):
        rs = rs + rewards[:, i]
    r = (rs / n).reshape(-1)
    d = (terminals != 0).all(dim=1).reshape(-1)
    disc = torch.where(d, torch.tensor(0.0), torch.tensor(1.0)) * torch.tensor(gamma, dtype=torch.float32)
    q = q_eval if v is None else q_eval + v.double()
    qn = q_next if v_next is None else q_next + v_next.double()
    y = r.double() + disc.double() * qn
    f = filled.double().reshape(-1)
    td = (q - y) * f
    dq = 2.0 * td * f / float(filled_sum)
    stats = torch.stack([(td * td).sum() / float(filled_sum), q.sum() / rows_total])
    return dq, (None if v is None else dq.float()), stats


def q_bwd_ref(dq, acts, edges, n, A, use_payoff):
    """The scatter: df [R, n, A] and dp [2, R, E, A*A] float32 from dq [R] and the taken actions [R, n]."""
    R, E = dq.shape[0], len(edges)
    acts = torch.as_tensor(acts).long()
    rows = torch.arange(R)
    df = torch.zeros(R, n, A)
    gu = (dq / n).float()
    for v in range(n):
        df[rows, v, acts[:, v]] = gu
    dp = torch.zeros(2, R, E, A * A)
    if use_payoff and E > 0:
        gp = (dq / E).float() * 0.5
        for e, (i, j) in enumerate(edges):
            dp[0, rows, e, acts[:, i] * A + acts[:, j]] = gp
            dp[1, rows, e, acts[:, j] * A + acts[:, i]] = gp
    return df, dp


# ---------------------------------------------------------------- the reference formulas under float64 autograd
def q_autograd(f, pay, edges, acts, use_payoff):
    """dcg_learner.py:90-104 and coordination_graph.py:87-103 as the reference writes them (float64 through autograd
    from float32 leaves): returns (Q [R], d f, d pay) for the seed dQ = 1."""
    f = f.clone().requires_grad_(True)
    pay = pay.clone().requires_grad_(True)
    R, n, A = f.shape
    E = len(edges)
    acts = torch.as_tensor(acts).long()
    f_mean = f.double() / n
    Q = f_mean.gather(-1, acts.unsqueeze(-1)).sum(dim=1).squeeze(-1)
    if use_payoff and E > 0:
        P = pay.view(2, R, E, A, A).clone()
        P1t = P[1].transpose(-1, -2)
        fij = torch.stack([P[0], P1t]).mean(dim=0)
        fr = torch.tensor([e[0] for e in edges])
        to = torch.tensor([e[1] for e in edges])
        idx = (acts[:, fr] * A + acts[:, to]).unsqueeze(-1)
        Q = Q + (fij.double() / E).reshape(R, E, A * A).gather(-1, idx).sum(dim=1).squeeze(-1)
    Q.sum().backward()
    return Q.detach(), f.grad, pay.grad


def quantised(rng, shape, step=0.25):
    """Coarse float32 values (multiples of ``step``): exact ties occur often."""
    return torch.from_numpy((np.round(rng.normal(size=shape) / step) * step).astype(np.float32))
