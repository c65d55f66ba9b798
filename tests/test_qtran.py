"""CPU tests of QTRAN_base / QTRAN_alt: the float64 restatements (tests/qtran_refs.py) against hand-computed cases (ties,
en = 0, dead and padded agents, n = 1, A = 1, masked next actions), the K9Q argument checks, the shipped configs, the
registries and the out-of-scope errors, and ptxas on the new kernels."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import qtran_refs as R
from xuance_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_select_ref_ties_masks_and_next_actions():
    q = torch.tensor([[[[1.0, 3.0, 3.0], [2.0, 2.0, 0.0]]]])                # [B=1, n=1, T+1=2, A=3]
    qt = torch.tensor([[[[0.0, 0.0, 0.0], [1.0, 5.0, 5.0]]]])
    g, nx = R.select_ref(q, qt, None, True)
    assert g.tolist() == [[[1, 0]]] and nx.tolist() == [[[0]]]              # first maximal index
    g, nx = R.select_ref(q, qt, None, False)
    assert nx.tolist() == [[[1]]]
    av = torch.tensor([[[[1, 0, 1], [1, 0, 0]]]], dtype=torch.uint8)
    g, nx = R.select_ref(q, qt, av, False)
    assert g.tolist() == [[[2, 0]]] and nx.tolist() == [[[0]]]              # the target's arg-max is masked too


def _by_hand_inputs(n, A, T=1):
    q_all = torch.arange(n * (T + 1) * A, dtype=torch.float32).reshape(1, n, T + 1, A) / 8.0
    actions = torch.zeros(1, n, T)
    greedy = torch.full((1, n, T + 1), A - 1, dtype=torch.int32)
    nxt = torch.zeros(1, n, T, dtype=torch.int32)
    mask = torch.ones(1, n, T)
    filled = torch.ones(1, T)
    return q_all, actions, greedy, nxt, mask, filled


def test_base_loss_ref_by_hand():
    q_all, actions, greedy, nxt, mask, filled = _by_hand_inputs(2, 3)
    mask[0, 1] = 0.0                                                        # a dead agent leaves both VDN sums
    rewards, terminals = torch.tensor([[[1.0], [3.0]]]), torch.zeros(1, 2, 1)
    qjt, qjt_g, qjt_n, v = torch.tensor([2.0]), torch.tensor([1.0]), torch.tensor([4.0]), torch.tensor([0.5])
    stats, dq, dqjt, dv = R.loss_grads(R.BASE, q_all, actions, greedy, nxt, mask, filled, rewards, terminals, qjt, qjt_g,
                                       qjt_n, v, 0.5, 1.0, 1.0)
    y = 2.0 + 0.5 * 4.0
    q_tot, q_tot_g = 0.0, 2.0 / 8.0                                         # agent 0: q[0,0,0] = 0, q[0,0,2] = 2/8
    td, eo, en = 2.0 - y, q_tot_g - 1.0 + 0.5, min(q_tot - 2.0 + 0.5, 0.0)
    assert stats.tolist() == pytest.approx([td ** 2, eo ** 2, en ** 2, td ** 2 + eo ** 2 + en ** 2, 2.0])
    assert dqjt.item() == pytest.approx(2 * td) and dv.item() == pytest.approx(2 * eo + 2 * en)
    assert dq[0, 0, 0, 0].item() == pytest.approx(2 * en) and dq[0, 0, 0, 2].item() == pytest.approx(2 * eo)
    assert not dq[0, 1].any()                                               # dead agent: no gradient


def test_base_nopt_is_zero_above_the_hinge_and_padding_drops_rows():
    q_all, actions, greedy, nxt, mask, filled = _by_hand_inputs(1, 2, T=2)
    filled[0, 1] = 0.0
    z = torch.zeros(2)
    stats, dq, _, dv = R.loss_grads(R.BASE, q_all, actions, greedy, nxt, mask, filled, torch.zeros(1, 1, 2),
                                    torch.zeros(1, 1, 2), torch.tensor([-5.0, 9.0]), z, z, z, 0.9, 1.0, 1.0)
    assert stats[2].item() == 0.0                                           # Q_tot - Q_jt + V > 0: en = 0
    assert stats[4].item() == pytest.approx(2.0)                            # Q_joint: padded rows included
    assert not dq[0, 0, 1].any()                                            # the padded step gets nothing


def test_alt_loss_ref_n1_a1_and_the_argmin():
    # n = 1: the leave-one-out sum is empty; A = 1: the min has one candidate
    q_all, actions, greedy, nxt, mask, filled = _by_hand_inputs(1, 1)
    qjt, qjt_g, qjt_n, v = torch.tensor([[3.0]]), torch.tensor([[1.0]]), torch.tensor([[2.0]]), torch.tensor([0.25])
    stats, dq, dqjt, dv = R.loss_grads(R.ALT, q_all, actions, greedy, nxt, mask, filled, torch.ones(1, 1, 1),
                                       torch.zeros(1, 1, 1), qjt, qjt_g, qjt_n, v, 0.5, 1.0, 1.0)
    td, eo, en = 3.0 - 2.0, 0.0 - 1.0 + 0.25, 0.0 - 3.0 + 0.25
    assert stats.tolist() == pytest.approx([td ** 2, eo ** 2, en ** 2, td ** 2 + eo ** 2 + en ** 2, 3.0])
    assert dq[0, 0, 0, 0].item() == pytest.approx(2 * eo + 2 * en)       # g = a = argmin: all three add
    # n = 2 with a tie in the nopt minimum: the first index wins, unavailable or not
    q_all, actions, greedy, nxt, mask, filled = _by_hand_inputs(2, 3)
    q_all.zero_()
    qjt = torch.zeros(2, 3)
    qjt[0] = torch.tensor([0.0, 1.0, 1.0])
    stats, dq, dqjt, _ = R.loss_grads(R.ALT, q_all, actions, greedy, nxt, mask, filled, torch.zeros(1, 2, 1),
                                      torch.ones(1, 2, 1), qjt, torch.zeros(2, 3), torch.zeros(2, 3),
                                      torch.tensor([0.0]), 0.5, 1.0, 1.0)
    assert dq[0, 0, 0, 1].item() != 0.0 and dq[0, 0, 0, 2].item() == 0.0   # agent 0's arg-min is action 1
    assert dqjt[:, 1:].abs().sum().item() == 0.0                            # Q_jt gets TD at the taken action only


def test_encode_ref_is_the_reference_assembly():
    rng = np.random.default_rng(0)
    B, n, T, S, H, A = 2, 3, 4, 5, 6, 4
    D = H + A
    st, h = torch.randn(B, T + 1, S, dtype=torch.float64), torch.randn(B, n, T + 1, H, dtype=torch.float64)
    mask = torch.from_numpy((rng.random((B, n, T)) < 0.7).astype(np.float64))
    acts = torch.from_numpy(rng.integers(0, A, (B, n, T)))
    w1, b1, w2, b2 = (torch.randn(*s, dtype=torch.float64) for s in ((D, D), (D,), (D, D), (D,)))
    xb = R.encode_ref(R.BASE, st, 1, h, mask, acts, w1, b1, w2, b2)
    xa = R.encode_ref(R.ALT, st, 1, h, mask, acts, w1, b1, w2, b2)
    b, t = 1, 2
    e = []
    for i in range(n):
        u = torch.cat([h[b, i, t] * mask[b, i, t], torch.nn.functional.one_hot(acts[b, i, t], A).double()])
        e.append(w2 @ torch.relu(w1 @ u + b1) + b2)
    r = b * T + t
    torch.testing.assert_close(xb[r], torch.cat([st[b, t + 1], sum(e)]))
    for i in range(n):
        loo = sum(e[i] for j in range(n) if j != i)                     # (n-1) e_i, as q_mix_head.py:283-285 runs
        torch.testing.assert_close(xa[r * n + i], torch.cat([st[b, t + 1], loo, torch.eye(n, dtype=torch.float64)[i]]))


def test_abi_symbols_and_argument_checks_without_gpu():
    from xuance_b200 import _lib
    for s in ("xb_qtran_select", "xb_qtran_encode_fwd", "xb_qtran_encode_bwd_work", "xb_qtran_encode_bwd",
              "xb_qtran_loss_fwd_bwd"):
        assert s in _lib.exported_symbols()
    lib = _lib.load()
    EINVAL, ERANGE = -1, -3
    j = 256  # any non-NULL pointer: validation returns before the device is touched
    sel = lambda **k: lib.xb_qtran_select(j, k.get("qt", j), None, 0, j, k.get("B", 4), k.get("n", 5), 6,
                                          k.get("A", 12), k.get("dq", 0), j, j, j, j, None)
    assert sel(B=0) == EINVAL and sel(qt=None) == EINVAL
    assert sel(n=33) == ERANGE and sel(A=65) == ERANGE and sel(n=0) == EINVAL
    enc = lambda **k: lib.xb_qtran_encode_fwd(k.get("mode", 0), j, k.get("t0", 0), j, j, k.get("af", j), k.get("ai"),
                                              k.get("aT", 6), j, j, j, j, 4, 5, 6, 10, k.get("H", 64), 12, j, None, None)
    assert enc(mode=2) == EINVAL and enc(t0=2) == EINVAL and enc(af=None) == EINVAL and enc(ai=j) == EINVAL
    assert enc(aT=5) == EINVAL and enc(H=65) == ERANGE and enc(H=0) == EINVAL
    need = lib.xb_qtran_encode_bwd_work(4, 5, 6, 64, 12)
    assert need == 2 * 120 * 76 + 1 * (2 * 76 * 76 + 2 * 76)
    bwd = lambda **k: lib.xb_qtran_encode_bwd(0, j, j, j, j, None, 6, j, j, k.get("pre", j), 4, 5, 6, 10, 64, 12,
                                              j, j, j, j, j, j, k.get("wf", need), None)
    assert bwd(wf=need - 1) == EINVAL and bwd(pre=None) == EINVAL
    loss = lambda **k: lib.xb_qtran_loss_fwd_bwd(k.get("mode", 1), *([j] * 13), 4, 5, 6, 12, 0.99, 1.0, 1.0,
                                                 k.get("rows", 24), j, j, j, j, j, None)
    assert loss(mode=3) == EINVAL and loss(rows=23) == EINVAL


def test_shipped_configs_and_registries():
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.learners import REGISTRY_Learners
    for env_id in ("5m_vs_6m", "3m"):
        cfg = get_arguments("qtran", "sc2", env_id)
        assert cfg.env_id == env_id and cfg.agent == "QTRAN_base" and cfg.learner == "QTRAN_Learner"
        assert cfg.qtran_net_hidden_dim == 64 and cfg.lambda_opt == 1.0 and cfg.lambda_nopt == 1.0
        assert cfg.q_hidden_size[0] == cfg.recurrent_hidden_size == 64 and cfg.use_rnn and cfg.use_actions_mask
    assert REGISTRY_Agents["QTRAN_base"] is REGISTRY_Agents["QTRAN_alt"]
    assert REGISTRY_Agents["QTRAN_base"].__name__ == "QTRAN_Agents"
    assert REGISTRY_Learners["QTRAN_Learner"].__name__ == "QTRAN_Learner"


def test_reference_parameter_names():
    """A reference QTranMixingNetwork state_dict has these keys (value_factorization.py:321-346, q_mix_head.py:176-189)."""
    from xuance_b200.common import Discrete
    from xuance_b200.torch.rl_models import QTRAN_Base, QTRAN_Alt
    sp = {k: Discrete(5) for k in ("a", "b", "c")}
    for cls, q_out, extra in ((QTRAN_Base, 1, 0), (QTRAN_Alt, 5, 3)):
        m = cls(10, sp, 64, 3, 64, True, "cpu")
        shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        assert shapes == {"Q_jt.0.weight": (64, 10 + 69 + extra), "Q_jt.0.bias": (64,), "Q_jt.2.weight": (64, 64),
                          "Q_jt.2.bias": (64,), "Q_jt.4.weight": (q_out, 64), "Q_jt.4.bias": (q_out,),
                          "V_jt.0.weight": (64, 10), "V_jt.0.bias": (64,), "V_jt.2.weight": (64, 64),
                          "V_jt.2.bias": (64,), "V_jt.4.weight": (1, 64), "V_jt.4.bias": (1,),
                          "action_encoding.0.weight": (69, 69), "action_encoding.0.bias": (69,),
                          "action_encoding.2.weight": (69, 69), "action_encoding.2.bias": (69,)}


def _cfg(**over):
    from xuance_b200.common.common_tools import get_arguments
    cfg = get_arguments("qtran", "sc2", "3m")
    cfg.device = "cpu"
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


def test_out_of_scope_configurations_fail_at_construction():
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.agents import REGISTRY_Agents
    keys = ["a0", "a1", "a2"]
    spaces = dict(num_agents=3, agent_keys=keys, state_space=Box(-1, 1, (10,)),
                  observation_space={k: Box(-1, 1, (8,)) for k in keys}, action_space={k: Discrete(6) for k in keys})
    with pytest.raises(NotImplementedError, match="use_rnn"):
        REGISTRY_Agents["QTRAN_base"](_cfg(use_rnn=False), **spaces)
    with pytest.raises(NotImplementedError, match="LSTM"):
        REGISTRY_Agents["QTRAN_alt"](_cfg(rnn="LSTM"), **spaces)
    with pytest.raises(ValueError, match="q_hidden_size"):
        REGISTRY_Agents["QTRAN_base"](_cfg(q_hidden_size=[32]), **spaces)
    with pytest.raises(NotImplementedError, match="parameter-sharing"):
        REGISTRY_Agents["QTRAN_base"](_cfg(use_parameter_sharing=False), **spaces)
    big = dict(spaces, action_space={k: Discrete(65) for k in keys})
    with pytest.raises(NotImplementedError, match="A <= 64"):
        REGISTRY_Agents["QTRAN_base"](_cfg(), **big)
    from xuance_b200.torch.learners import QTRAN_Learner
    with pytest.raises(ValueError, match="QMIX"):
        QTRAN_Learner(_cfg(agent="QMIX"), None, None, None)


def test_qtran_kernels_compile_without_spills(tmp_path):
    flags = [f for f in build.NVCC_FLAGS if f not in ("--use_fast_math=false", "-shared")]
    cmd = [build._nvcc()] + flags + ["-c", os.path.join(build.CSRC, "qtran.cu"), "-o", str(tmp_path / "qtran.o")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    kernels, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S*qtran\S*)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = sum(int(x) for x in m.groups())
            cur = None
    assert len(kernels) == 9, log
    assert {k: v for k, v in kernels.items() if v} == {}


# ---------------------------------------------------------------- the reference fixture (tests/golden/qtran_update.npz)
GOLDEN = os.path.join(ROOT, "tests", "golden", "qtran_update.npz")
# as make_golden_qtran.py records them
FIX_N, FIX_OBS, FIX_A, FIX_S, FIX_HID, FIX_QH = 3, 12, 7, 10, 16, 16
FIX_UPDATES, FIX_SNAPSHOTS = 4, (1, 3)
FIX_CASES = [(agent, dq) for agent in ("QTRAN_base", "QTRAN_alt") for dq in (True, False)]
FIX_INFO_KEYS = ("loss_td", "loss_opt", "loss_nopt", "loss", "Q_joint", "learning_rate")


def fixture_init(d, pre):
    return {k[len(pre) + 5:]: torch.from_numpy(d[k]) for k in d.files if k.startswith(pre + "init/")}


def fixture_sample(d, pre, it, keys):
    p = f"{pre}in{it}/"
    s = {f: {k: d[p + f][:, i] for i, k in enumerate(keys)}
         for f in ("obs", "actions", "rewards", "terminals", "agent_mask", "avail_actions")}
    B, T = d[p + "filled"].shape
    s.update(filled=d[p + "filled"], state=d[p + "state"], batch_size=B, sequence_length=T)
    return s


def test_reference_state_dict_loads_strictly_and_the_corrections_only_rekey():
    from oracle_qtran import build_model
    d = np.load(GOLDEN)
    for agent, dq in FIX_CASES:
        _, _, model = build_model(agent, FIX_N, FIX_OBS, FIX_A, FIX_S, FIX_HID, FIX_QH, "cpu")
        model.load_state_dict(fixture_init(d, f"{agent}/dq{int(dq)}/"), strict=True)
    runs = d["rekey_check/infos"]                       # uncorrected vs corrected reference, independent groups
    assert runs.shape[0] == 2 and np.array_equal(runs[0], runs[1])


@pytest.mark.parametrize("agent,double_q", FIX_CASES)
def test_oracle_reproduces_the_reference_fixture(agent, double_q):
    """The float64 oracle against every update of the reference (float32): the logged values within 1e-5 relative,
    the whole state_dict after the target sync and after the last update within 1e-5 + 1e-5 relative."""
    from oracle_qtran import QTRANOracle, build_model
    d = np.load(GOLDEN)
    pre = f"{agent}/dq{int(double_q)}/"
    keys, _, model = build_model(agent, FIX_N, FIX_OBS, FIX_A, FIX_S, FIX_HID, FIX_QH, "cpu")
    model.load_state_dict(fixture_init(d, pre), strict=True)
    orc = QTRANOracle(model, double_q=double_q, total_iters=int(d[pre + "total_iters"]))
    for it in range(FIX_UPDATES):
        info = orc.update(fixture_sample(d, pre, it, keys))
        np.testing.assert_allclose([info[k] for k in FIX_INFO_KEYS], d[pre + "infos"][it], rtol=1e-5, atol=1e-7,
                                   err_msg=f"{pre}it{it}")
        if it in FIX_SNAPSHOTS:
            got = np.concatenate([v.numpy().reshape(-1) for v in orc.m.state_dict().values()])
            np.testing.assert_allclose(got, d[f"{pre}after{it}"], rtol=1e-5, atol=1e-5, err_msg=f"{pre}after{it}")
