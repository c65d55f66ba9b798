"""CPU tests of VDAC and IAC: the float64 restatement of K4V against float64 autograd of the reference's expressions (ties,
n = 1, A = 1, T = 1, all-masked rows, Huber at delta), the two V_tot row orders, the torch-CPU oracle against every case of
the reference fixture (tests/golden/vdac_update.npz), a strict load of the reference state_dict, ABI argument checks,
configs, registries, the out-of-scope errors and ptxas on K4V."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from vdac_refs import (FIX_CASES, FIX_UPDATES, FIX_SNAPSHOTS, case_name, k4v_ref, k4v_autograd, pred_index)
from oracle_vdac import build_product_model, VDACLearnerOracle, fixture_batch
from xuance_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "vdac_update.npz")


def _inputs(rng, B, T, n, A, mode, masks=True):
    R = B * n * T
    av = None
    acts = rng.integers(0, A, R)
    if masks:
        av = (rng.random((R, A)) < 0.6).astype(np.uint8)
        av[np.arange(R), acts] = 1
    return dict(logits=rng.normal(0, 2, (R, A)), avail=av, actions=acts.astype(np.float32), adv=rng.normal(0, 1, R),
                value=rng.normal(0, 1, B * T if mode == 2 else R), old_value=rng.normal(0, 1, R),
                ret=rng.normal(0, 2, R), mask=(rng.random(R) > 0.3).astype(np.float64) if masks else np.ones(R))


@pytest.mark.parametrize("mode,row_order", [(0, 0), (1, 0), (1, 1), (2, 0), (2, 1)])
@pytest.mark.parametrize("B,T,n,A", [(3, 5, 3, 6), (2, 1, 4, 3), (4, 7, 1, 5), (2, 4, 3, 1), (1, 1, 1, 1)])
@pytest.mark.parametrize("vclip,hdelta", [(0.0, 0.0), (0.3, 0.0), (0.0, 1.0), (0.3, 1.0)])
def test_restatement_matches_reference_autograd(mode, row_order, B, T, n, A, vclip, hdelta):
    rng = np.random.default_rng(B * 100 + T * 10 + n + A + 7 * mode + row_order)
    d = _inputs(rng, B, T, n, A, mode)
    args = (d["logits"], d["avail"], d["actions"], d["adv"], d["value"], d["old_value"], d["ret"], d["mask"])
    st, dl, dv = k4v_ref(*args, None, n, T, mode, row_order, vclip, hdelta, 0.5, 0.01)
    ast, adl, adv = k4v_autograd(*args, n, T, mode, row_order, vclip, hdelta, 0.5, 0.01)
    np.testing.assert_allclose(st, ast, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dl, adl, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(dv, adv, rtol=1e-10, atol=1e-12)


def test_restatement_ties_huber_at_delta_and_masked_rows():
    """The clip boundary, the max tie (each side 1/2), Huber at |d| = delta, and rows with mask 0 (no gradient)."""
    n, T, A = 2, 2, 3
    R = n * T
    logits, acts = np.zeros((R, A)), np.zeros(R, np.float32)
    # row 0: v - ret = delta exactly; rows 1-3: clipped and unclipped losses equal (v == old value)
    value, old, ret = np.array([1.0, 0.5, 0.5, 0.5]), np.array([1.0, 0.5, 0.5, 0.5]), np.array([0.0, 0.0, 0.0, 0.0])
    mask = np.array([1.0, 1.0, 0.0, 1.0])
    for vclip in (0.0, 0.5):
        args = (logits, None, acts, np.ones(R), value, old, ret, mask)
        st, dl, dv = k4v_ref(*args, None, n, T, 0, 0, vclip, 1.0, 1.0, 0.0)
        ast, adl, adv = k4v_autograd(*args, n, T, 0, 0, vclip, 1.0, 1.0, 0.0)
        np.testing.assert_allclose(st, ast, rtol=1e-12)
        np.testing.assert_allclose(dv, adv, rtol=1e-12, atol=1e-15)
        assert dv[2] == 0 and np.all(dl[2] == 0)
        np.testing.assert_allclose(dv[0], 1.0 / 3.0)            # Huber gradient delta at |d| = delta, weight 1/M


def test_all_masked_batch_gives_nan_as_the_reference():
    rng = np.random.default_rng(1)
    d = _inputs(rng, 2, 3, 2, 4, 1)
    d["mask"][:] = 0
    st, dl, dv = k4v_ref(d["logits"], d["avail"], d["actions"], d["adv"], d["value"], d["old_value"], d["ret"],
                         d["mask"], None, 2, 3, 1, 0, 0.0, 0.0, 0.5, 0.01)
    assert np.isnan(st[:3]).all() and np.isnan(dv).all()


def test_row_orders_differ_at_T_gt_1_and_coincide_at_T_1():
    for B, n, T in ((2, 3, 4), (3, 5, 1)):
        a, b = pred_index(B, n, T, 0), pred_index(B, n, T, 1)
        assert np.array_equal(a, b) == (T == 1)
    # the reference's pairing, as its probe shows it: V_tot of row floor(r / n) against the target of row r = (b, i, t)
    assert pred_index(2, 3, 4, 1)[:6].tolist() == [0, 0, 0, 1, 1, 1]
    assert pred_index(2, 3, 4, 0)[:6].tolist() == [0, 1, 2, 3, 0, 1]


def test_row_orders_differ_on_the_fixture_sample():
    """Evidence on the fixture's first recurrent VDN sample: the reference pairing and the aligned pairing give different
    critic losses; on the feed-forward case (T = 1) they are identical."""
    g = np.load(GOLDEN)
    losses = {}
    for case in (FIX_CASES[0], FIX_CASES[3]):
        pre = case_name(case) + "/"
        for ro in (True, False):
            _, model = build_product_model(case, "cpu")
            model.load_state_dict({k[len(pre) + 5:]: torch.from_numpy(g[k]) for k in g.files
                                   if k.startswith(pre + "init/")}, strict=True)
            losses[case, ro] = VDACLearnerOracle(model, case, row_order=ro).update(fixture_batch(g, pre, 0, case[1]))
    rnn, ff = FIX_CASES[0], FIX_CASES[3]
    assert abs(losses[rnn, True]["critic_loss"] - losses[rnn, False]["critic_loss"]) > 1e-3
    assert losses[ff, True] == losses[ff, False]


@pytest.mark.parametrize("case", FIX_CASES, ids=case_name)
def test_oracle_reproduces_the_reference_fixture(case):
    """The oracle (reference row order for the recurrent VDAC cases) against every update of the unmodified reference;
    the fixture's initial state_dict loads into the product model with strict=True."""
    g = np.load(GOLDEN)
    pre = case_name(case) + "/"
    _, model = build_product_model(case, "cpu")
    keys = [k[len(pre) + 5:] for k in g.files if k.startswith(pre + "init/")]
    model.load_state_dict({k: torch.from_numpy(g[pre + "init/" + k]) for k in keys}, strict=True)
    orc = VDACLearnerOracle(model, case, row_order=True)
    for it in range(FIX_UPDATES):
        info = orc.info_row(orc.update(fixture_batch(g, pre, it, case[1])))
        np.testing.assert_allclose(info, g[pre + "infos"][it], rtol=1e-5, atol=1e-7, err_msg=f"update {it}")
        if it in FIX_SNAPSHOTS:
            sd = orc.state_dict()
            flat = np.concatenate([sd[k].detach().numpy().reshape(-1) for k in keys])
            np.testing.assert_allclose(flat, g[pre + f"after{it}"], rtol=1e-5, atol=1e-6)


def test_abi_symbol_and_argument_checks_without_gpu():
    from xuance_b200 import _lib
    assert "xb_vdac_loss_fwd_bwd" in _lib.exported_symbols()
    lib = _lib.load()
    EINVAL, ERANGE = -1, -3
    j = 256  # any non-NULL pointer: validation returns before the device is touched

    def call(**k):
        R, A, n, T = k.get("R", 24), k.get("A", 5), k.get("n", 3), k.get("T", 4)
        return lib.xb_vdac_loss_fwd_bwd(k.get("logits", j), k.get("avail"), k.get("ld", 0), j, j, j, k.get("old", j),
                                        j, j, None, j, R, A, n, T, k.get("mode", 1), k.get("ro", 0),
                                        k.get("Rt", R), k.get("vclip", 0.2), 1.0, 0.5, 0.01, j, j, j, j, None)
    assert call(logits=None) == EINVAL and call(old=None) == EINVAL and call(R=0) == EINVAL
    assert call(Rt=12) == EINVAL and call(mode=3) == EINVAL and call(ro=2) == EINVAL and call(R=23) == EINVAL
    assert call(n=0) == EINVAL and call(T=0) == EINVAL and call(avail=j, ld=4) == EINVAL
    assert call(A=65) == ERANGE and call(n=33, R=33 * 4) == ERANGE


def test_shipped_configs_and_registries():
    import yaml
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.learners import REGISTRY_Learners
    for algo, agent, learner in (("vdac", "VDAC", "VDAC_Learner"), ("iac", "IAC", "IAC_Learner")):
        for env_id in ("3m", "5m_vs_6m"):
            cfg = vars(get_arguments(algo, "sc2", env_id))
            path = os.path.join(ROOT, "xuance_b200", "configs", algo, "sc2", env_id + ".yaml")
            for k, v in yaml.safe_load(open(path)).items():
                assert cfg[k] == v, k
            assert (cfg["agent"], cfg["learner"], cfg["use_rnn"], cfg["rnn"], cfg["recurrent_hidden_size"]) == \
                (agent, learner, True, "GRU", 64)
        assert REGISTRY_Agents[agent].__name__ == agent + "_Agents"
        assert REGISTRY_Learners[learner].__name__ == learner
        for env in ("mpe", "atari"):
            with pytest.raises(AttributeError, match="no config"):
                get_arguments(algo, env, "simple_spread_v3")
    assert get_arguments("vdac", "sc2", "3m").mixer == "QMIX"


def _cfg(algo="vdac", **over):
    from xuance_b200.common.common_tools import get_arguments
    cfg = get_arguments(algo, "sc2", "3m")
    cfg.device = "cpu"
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


def test_out_of_scope_configurations_fail_at_construction():
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.agents import REGISTRY_Agents

    def spaces(n=3, act=None):
        keys = [f"a{i}" for i in range(n)]
        return dict(num_agents=n, agent_keys=keys, state_space=Box(-1, 1, (10,)),
                    observation_space={k: Box(-1, 1, (8,)) for k in keys},
                    action_space={k: act or Discrete(6) for k in keys})
    for algo, name in (("vdac", "VDAC"), ("iac", "IAC")):
        with pytest.raises(NotImplementedError, match="parameter-sharing"):
            REGISTRY_Agents[name](_cfg(algo, use_parameter_sharing=False), **spaces())
        with pytest.raises(NotImplementedError, match="LSTM"):
            REGISTRY_Agents[name](_cfg(algo, rnn="LSTM"), **spaces())
        with pytest.raises(NotImplementedError, match="N_recurrent_layers"):
            REGISTRY_Agents[name](_cfg(algo, N_recurrent_layers=2), **spaces())
        with pytest.raises(NotImplementedError, match="recurrent_hidden_size"):
            REGISTRY_Agents[name](_cfg(algo, recurrent_hidden_size=65), **spaces())
        with pytest.raises(NotImplementedError, match="Box"):
            REGISTRY_Agents[name](_cfg(algo), **spaces(act=Box(-1, 1, (2,))))
    with pytest.raises(NotImplementedError, match="mixer"):
        REGISTRY_Agents["VDAC"](_cfg(mixer="Independent"), **spaces())
    with pytest.raises(NotImplementedError, match="16 agents"):
        REGISTRY_Agents["VDAC"](_cfg(mixer="QMIX"), **spaces(n=17))
    from xuance_b200.torch.learners import VDAC_Learner
    with pytest.raises(NotImplementedError, match="mixer"):
        VDAC_Learner._mix_mode(_cfg(mixer="Independent"))


def test_k4v_compiles_without_spills(tmp_path):
    flags = [f for f in build.NVCC_FLAGS if f not in ("--use_fast_math=false", "-shared")]
    cmd = [build._nvcc()] + flags + ["-c", os.path.join(build.CSRC, "vdac.cu"), "-o", str(tmp_path / "vdac.o")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    kernels, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S*vdac\S*)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = sum(int(x) for x in m.groups())
            cur = None
    assert len(kernels) == 5, log
    assert {k: v for k, v in kernels.items() if v} == {}
