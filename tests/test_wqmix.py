"""CPU tests of Weighted QMIX: the float64 kernel restatements (tests/wqmix_refs.py) against torch autograd and by hand,
the torch-CPU oracle (reference as it runs: detach switch on) against the reference fixture, the K9W argument checks,
the shipped configs, the registries and the out-of-scope errors, and ptxas on the new kernels."""
import os
import re
import shutil
import subprocess
from argparse import Namespace

import numpy as np
import pytest
import torch

import wqmix_refs as R
from oracle_wqmix import WQMIXModelOracle, WQMIXLearnerOracle
from xuance_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "wqmix_update.npz")
NVCC = build._nvcc()


def _loss_inputs(rng, B, n, T, ties=False, dead=False, padded=False):
    q_tot = torch.from_numpy(rng.normal(size=B * T).astype(np.float32))
    q_ff = torch.from_numpy(rng.normal(size=B * T).astype(np.float32))
    q_ff_next = torch.from_numpy(rng.normal(size=B * T).astype(np.float32))
    rewards = torch.from_numpy(rng.normal(size=(B, n, T)).astype(np.float32))
    terminals = torch.from_numpy((rng.random((B, n, T)) < 0.3).astype(np.float32))
    filled = torch.ones(B, T)
    if padded:
        filled[:, T // 2:] = 0.0
    agree = torch.from_numpy(rng.random(B * T) < 0.3)
    if ties:     # td == 0 and y == q_ff exactly on some rows: gamma = 0 and one reward per agent => y = r exactly
        rewards[:] = 0.5
        q_tot[::3] = 0.5
        q_ff[::2] = 0.5
    if dead:
        agree[:] = False
    return q_tot, q_ff, q_ff_next, rewards, terminals, filled, agree


@pytest.mark.parametrize("mode", [R.OW, R.CW])
@pytest.mark.parametrize("B,n,T,case", [(4, 3, 5, "plain"), (3, 1, 7, "n1"), (5, 4, 6, "ties"), (2, 3, 8, "padded"),
                                        (3, 5, 4, "dead")])
def test_loss_ref_matches_autograd(mode, B, n, T, case):
    rng = np.random.default_rng(B * 7 + n + T)
    q_tot, q_ff, q_ff_next, rewards, terminals, filled, agree = _loss_inputs(
        rng, B, n, T, ties=case == "ties", dead=case == "dead", padded=case == "padded")
    gamma = 0.0 if case == "ties" else 0.99
    dq_tot, dq_ff, stats = R.loss_ref(q_tot, q_ff, q_ff_next, rewards, terminals, filled, agree, filled.sum(), mode,
                                      0.1, gamma, B * T)
    g_tot, g_ff, s_auto = R.loss_autograd(q_tot, q_ff, q_ff_next, rewards, terminals, filled, agree, mode, 0.1, gamma)
    np.testing.assert_allclose(dq_tot.numpy(), g_tot.numpy(), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(dq_ff.numpy(), g_ff.numpy(), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(stats.numpy(), s_auto.numpy(), rtol=1e-12, atol=1e-15)
    if case == "ties":
        y = R.team_targets(rewards, terminals, q_ff_next, gamma)
        td = q_tot.double() - y
        assert (td == 0).any() and (y == q_ff.double()).any()
        w = R.weights(mode, 0.1, td, y, q_ff.double(), agree)
        # td == 0 is not "td < 0" (OW) and y == q_ff is not "y > q_ff" (CW): the tie keeps alpha (CW: unless agree)
        tie = (td == 0) if mode == R.OW else (y == q_ff.double()) & ~agree
        assert tie.any() and (w[tie] == 0.1).all()
    if case == "padded":
        assert (dq_tot.reshape(B, T)[:, T // 2:] == 0).all() and (dq_ff.reshape(B, T)[:, T // 2:] == 0).all()


def test_select_ref_first_index_ties_masks_dead_agents_and_agreement():
    B, n, T, A = 2, 2, 3, 4
    q = torch.zeros(B, n, T + 1, A)
    q[..., 2] = 1.0
    q[..., 3] = 1.0                                # tie between 2 and 3: the first wins
    avail = torch.ones(B, n, T + 1, A, dtype=torch.uint8)
    avail[0, 0, 1, 2] = 0                          # unavailable: next best is 3
    actions = torch.full((B, n, T), 2.0)
    agent_mask = torch.ones(B, n, T)
    agent_mask[1, 1, 2] = 0.0                      # a dead agent clears the agreement of its row
    filled = torch.ones(B, T)
    filled[0, 2] = 0.0                             # a padded step too
    qc = torch.arange(B * n * (T + 1) * A, dtype=torch.float32).reshape(B, n, T + 1, A)
    qe, qct, qn, g, agree, fs = R.select_ref(q, qc, qc + 0.5, qc - 0.5, actions, agent_mask, filled, avail, True)
    assert g[0, 0, 1] == 3 and (g[0, 0, 0] == 2) and (g[1] == 2).all()
    assert agree.tolist() == [True, False, False, True, True, False]
    assert fs == 5.0
    assert qct[1, 0] == qc[0, 0, 1, 3] and qn[0, 0] == qc[0, 0, 1, 3] + 0.5   # g_{t+1} of step 0 is the masked 3
    # double_q = 0: the next action is the unmasked argmax of the target agent values
    _, _, qn0, _, _, _ = R.select_ref(q, qc, qc + 0.5, qc - 0.5, actions, agent_mask, filled, avail, False)
    assert qn0[0, 0] == qc[0, 0, 1, 3] + 0.5        # qc - 0.5 grows with the index: argmax = A - 1
    # A = 1: everything selects index 0
    _, _, _, g1, _, _ = R.select_ref(q[..., :1], qc[..., :1], qc[..., :1], qc[..., :1], actions * 0, agent_mask,
                                     filled, None, True)
    assert (g1 == 0).all()


def test_select_bwd_ref_is_the_gather_adjoint():
    rng = np.random.default_rng(3)
    B, n, T, A = 3, 4, 5, 6
    q_all = torch.from_numpy(rng.normal(size=(B, n, T + 1, A))).requires_grad_(True)
    q_cent = torch.from_numpy(rng.normal(size=(B, n, T + 1, A))).requires_grad_(True)
    actions = torch.from_numpy(rng.integers(0, A, (B, n, T)).astype(np.float32))
    agent_mask = torch.from_numpy((rng.random((B, n, T)) < 0.8).astype(np.float32))
    filled = torch.from_numpy((rng.random((B, T)) < 0.8).astype(np.float32))
    g = R.masked_argmax(q_all.detach(), None)[:, :, :-1]
    m = agent_mask.double() * filled.double().unsqueeze(1)
    qe = q_all[:, :, :-1].gather(-1, actions.long().unsqueeze(-1)).squeeze(-1) * m
    qc = q_cent[:, :, :-1].gather(-1, g.unsqueeze(-1)).squeeze(-1) * m
    de, dc = torch.from_numpy(rng.normal(size=(B * T, n))), torch.from_numpy(rng.normal(size=(B * T, n)))
    rows = lambda x: x.permute(0, 2, 1).reshape(B * T, n)
    ((rows(qe) * de).sum() + (rows(qc) * dc).sum()).backward()
    ge, gc = R.select_bwd_ref(de, dc, actions, g, agent_mask, filled, A)
    assert torch.equal(ge, q_all.grad) and torch.equal(gc, q_cent.grad)


def _fixture_learner_pair(d, agent, double_q):
    pre = f"{agent}/dq{int(double_q)}/"
    init = {k[len(pre) + 5:]: torch.from_numpy(d[k]) for k in d.files if k.startswith(pre + "init/")}
    return pre, init


@pytest.mark.parametrize("agent,double_q", R.FIX_CASES)
def test_oracle_with_the_detach_switch_reproduces_the_reference(agent, double_q):
    d = np.load(GOLDEN)
    pre, init = _fixture_learner_pair(d, agent, double_q)
    keys = [f"agent_{i}" for i in range(R.FIX_N)]
    om = WQMIXModelOracle(R.FIX_N, R.FIX_OBS, R.FIX_A, R.FIX_S, R.FIX_HID, R.FIX_MIX, R.FIX_HYPER, R.FIX_FF)
    om.load_state_dict(init, strict=True)
    cfg = R.fix_learner_config(agent, double_q)
    orc = WQMIXLearnerOracle(om, keys, agent=agent, alpha=cfg["alpha"], learning_rate=cfg["learning_rate"],
                             gamma=cfg["gamma"], sync_frequency=cfg["sync_frequency"], double_q=double_q,
                             end_factor_lr_decay=cfg["end_factor_lr_decay"], total_iters=int(d[pre + "total_iters"]),
                             detach_q_eval=True, use_actions_mask=True)
    for it in range(R.FIX_UPDATES):
        info = orc.update(fixture_sample(d, pre, it, keys))
        np.testing.assert_allclose([info[k] for k in R.FIX_INFO_KEYS], d[pre + "infos"][it], rtol=2e-6, atol=1e-7)
        if it in R.FIX_SNAPSHOTS:
            got = np.concatenate([v.numpy().reshape(-1) for v in om.state_dict().values()])
            np.testing.assert_allclose(got, d[f"{pre}after{it}"], rtol=1e-5, atol=1e-6)
    # the reference trains only the two mixers: both sets of agent networks keep their initial weights
    for k, v in om.state_dict().items():
        if k.startswith(("individual_q_networks", "individual_q_centralized")):
            assert torch.equal(v, init[k]), k


def fixture_sample(d, pre, it, keys):
    """The sample dict of update ``it`` of a fixture case (the replay's sample() layout)."""
    p = f"{pre}in{it}/"
    s = {f: {k: d[p + f][:, i] for i, k in enumerate(keys)}
         for f in ("obs", "actions", "rewards", "terminals", "agent_mask", "avail_actions")}
    B, T = d[p + "filled"].shape
    s.update(filled=d[p + "filled"], state=d[p + "state"], batch_size=B, sequence_length=T)
    return s


def test_argument_checks_without_gpu():
    from xuance_b200 import _lib
    lib = _lib.load()
    EINVAL, ERANGE = -1, -3
    j = 256  # any non-NULL pointer: validation returns before the device is touched
    sel = lambda **k: lib.xb_wqmix_select_fwd(j, j, j, k.get("q_tgt", j), j, j, j, k.get("avail"), k.get("ld", 0),
                                              k.get("B", 4), k.get("n", 5), 6, k.get("A", 12), k.get("dq", 1), j, j, j,
                                              k.get("greedy", j), j, j, j, None)
    assert sel(B=0) == EINVAL and sel(A=0) == EINVAL and sel(n=0) == EINVAL
    assert sel(greedy=None) == EINVAL
    assert sel(avail=j, ld=11) == EINVAL                              # avail rows shorter than A
    assert sel(dq=0, q_tgt=None) == EINVAL                            # double_q = 0 needs the target agent values
    assert sel(n=17) == ERANGE
    bwd = lambda de, dqa, dc, dqc, n=5: lib.xb_wqmix_select_bwd(de, dc, j, j, j, j, 4, n, 6, 12, dqa, dqc, None)
    assert bwd(j, None, j, j) == EINVAL and bwd(None, None, None, None) == EINVAL and bwd(j, j, j, j, n=17) == ERANGE
    loss = lambda mode=0, agree=None, rows=24, n=5: lib.xb_wqmix_loss_fwd_bwd(j, j, j, j, j, j, agree, j, 4, n, 6, mode,
                                                                              0.1, 0.99, rows, j, j, j, j, None)
    assert loss(rows=23) == EINVAL                    # rows_total is the global B*T: never below the local one
    assert loss(mode=2) == EINVAL
    assert loss(mode=1) == EINVAL                     # CW needs the agreement flags
    assert loss(n=17) == ERANGE


def _cfg(**over):
    from xuance_b200.common.common_tools import get_arguments
    cfg = get_arguments("wqmix", "sc2", "5m_vs_6m")
    cfg.device = "cpu"
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


def test_shipped_configs_and_registries():
    import yaml
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.learners import REGISTRY_Learners
    for env_id in ("5m_vs_6m", "3m"):
        cfg = get_arguments("wqmix", "sc2", env_id)
        assert cfg.env_id == env_id and cfg.agent == "OWQMIX" and cfg.learner == "WQMIX_Learner"
        assert cfg.alpha == 0.1 and cfg.hidden_dim_ff_mix_net == 256 and cfg.use_rnn and cfg.use_actions_mask
        assert cfg.qmix_rnn_detach_q_eval is False
    assert REGISTRY_Agents["OWQMIX"] is REGISTRY_Agents["CWQMIX"]
    assert REGISTRY_Agents["OWQMIX"].__name__ == "WQMIX_Agents"
    assert REGISTRY_Learners["WQMIX_Learner"].__name__ == "WQMIX_Learner"
    # every config.X the agent / learner classes read without a default is defined by basic.yaml + the yaml
    root = os.path.join(ROOT, "xuance_b200")
    src = "".join(open(os.path.join(root, *f.split("/"))).read() for f in
                  ("torch/agents/marl.py", "torch/agents/wqmix_agents.py", "torch/learners/qmix_learner.py", "torch/learners/wqmix_learner.py",
                   "torch/agents/agent.py", "torch/learners/learner.py"))
    hard = set(re.findall(r"(?<![a-zA-Z_])(?:self\.)?config\.([a-zA-Z_][a-zA-Z0-9_]*)\b(?!\s*=[^=])", src))
    soft = set(re.findall(r"(?:getattr|hasattr)\((?:self\.)?config,\s*.([a-zA-Z_0-9]+).", src))
    base = set(yaml.safe_load(open(os.path.join(root, "configs", "basic.yaml"))))
    for env_id in ("5m_vs_6m", "3m"):
        y = yaml.safe_load(open(os.path.join(root, "configs", "wqmix", "sc2", f"{env_id}.yaml")))
        assert not sorted(hard - soft - base - set(y)), env_id


def test_out_of_scope_configurations_fail_at_construction():
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.agents import REGISTRY_Agents
    keys = ["agent_0", "agent_1", "agent_2"]
    kw = dict(num_agents=3, agent_keys=keys, state_space=Box(-1, 1, (10,), np.float32),
              observation_space={k: Box(-1, 1, (12,), np.float32) for k in keys},
              action_space={k: Discrete(7) for k in keys})
    with pytest.raises(NotImplementedError, match="use_rnn"):
        REGISTRY_Agents["OWQMIX"](_cfg(use_rnn=False), **kw)
    with pytest.raises(NotImplementedError, match="use_parameter_sharing"):
        REGISTRY_Agents["CWQMIX"](_cfg(agent="CWQMIX", use_parameter_sharing=False), **kw)


def test_learner_refuses_unknown_agents_and_feed_forward_agents():
    from xuance_b200.torch.learners import WQMIX_Learner
    with pytest.raises(AttributeError, match="QTRAN"):
        WQMIX_Learner(Namespace(agent="QTRAN", use_rnn=True), None, None, None)
    with pytest.raises(NotImplementedError, match="use_rnn"):
        WQMIX_Learner(Namespace(agent="OWQMIX", use_rnn=False), None, None, None)


@pytest.mark.skipif(shutil.which(NVCC) is None and not os.path.exists(NVCC), reason="nvcc not available")
def test_wqmix_kernels_compile_without_spills(tmp_path):
    flags = [f for f in build.NVCC_FLAGS if f not in ("--use_fast_math=false", "-shared")]
    cmd = [NVCC] + flags + ["-c", os.path.join(build.CSRC, "wqmix.cu"), "-o", str(tmp_path / "wqmix.o")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    kernels, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S*wqmix\S*)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = sum(int(x) for x in m.groups())
            cur = None
    assert len(kernels) == 3, log
    assert {k: v for k, v in kernels.items() if v} == {}
