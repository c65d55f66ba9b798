"""CPU tests of COMA: the float64 restatement of K4C against float64 autograd of the reference's expressions (epsilon 0,
0.3 and 1, masked renormalisation, all-but-one masked, A = 1, n = 1, M = 0 and a zero-probability taken action), the
torch-CPU oracle against every case and update of the reference fixture (tests/golden/coma_update.npz), a strict load of
the reference state_dict, ABI argument checks, configs, registries, the out-of-scope errors and ptxas on K4C."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from coma_refs import (FIX_CASES, FIX_UPDATES, FIX_SNAPSHOTS, INFO_KEYS, case_name, k4c_ref, k4c_autograd)
from oracle_coma import build_product_model, COMALearnerOracle, fixture_batch
from xuance_b200 import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "coma_update.npz")


def _inputs(rng, R, A, masks=True):
    acts = rng.integers(0, A, R)
    av = None
    if masks:
        av = (rng.random((R, A)) < 0.6).astype(np.uint8)
        av[np.arange(R), acts] = 1
    return dict(logits=rng.normal(0, 2, (R, A)), avail=av, q=rng.normal(0, 1, (R, A)), actions=acts.astype(np.float32),
                ret=rng.normal(0, 2, R), mask=(rng.random(R) > 0.3).astype(np.float64))


def _both(d, eps):
    args = (d["logits"], d["avail"], d["q"], d["actions"], d["ret"], d["mask"], eps)
    return k4c_ref(*args), k4c_autograd(*args)


@pytest.mark.parametrize("eps", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("R,A", [(1, 1), (7, 1), (12, 5), (40, 9), (3, 64)])
@pytest.mark.parametrize("masks", [False, True])
def test_restatement_matches_reference_autograd(eps, R, A, masks):
    d = _inputs(np.random.default_rng(R * 100 + A + int(10 * eps) + masks), R, A, masks)
    (st, dl, dq), (ast, adl, adq) = _both(d, eps)
    np.testing.assert_allclose(st, ast, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(dl, adl, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(dq, adq, rtol=1e-12, atol=1e-15)
    assert np.count_nonzero(dq, axis=1).max() <= 1
    if masks:
        assert np.all(dl[d["avail"] == 0] == 0)


def test_all_but_one_masked_and_n1_rows():
    """Rows where only the taken action is available (pi = 1 after the renormalisation: zero advantage and gradient)."""
    rng = np.random.default_rng(2)
    d = _inputs(rng, 6, 4)
    d["avail"][:] = 0
    d["avail"][np.arange(6), d["actions"].astype(int)] = 1
    for eps in (0.0, 0.3):
        (st, dl, dq), (ast, adl, adq) = _both(d, eps)
        np.testing.assert_allclose(st, ast, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(dl, adl, atol=1e-12)
        assert np.all(np.abs(dl) < 1e-12) and abs(st[0]) < 1e-12


def test_zero_mask_sum_gives_nan_as_the_reference():
    d = _inputs(np.random.default_rng(1), 8, 5)
    d["mask"][:] = 0
    (st, dl, dq), (ast, _, _) = _both(d, 0.3)
    assert np.isnan(st[:2]).all() and np.isnan(ast[:2]).all()
    assert np.isnan(dq[np.arange(8), d["actions"].astype(int)]).all()


def test_zero_probability_taken_action_gives_nan_as_the_reference():
    """An unavailable taken action (which the epsilon mix lets the reference's acting draw) has pi = 0 after the
    renormalisation: log pi = -inf, and autograd gives NaN at the row's available logits; other rows stay finite."""
    d = _inputs(np.random.default_rng(4), 6, 5)
    a0 = int(d["actions"][0])
    d["avail"][0] = 1
    d["avail"][0, a0] = 0
    d["mask"][:] = 1
    (st, dl, dq), (ast, adl, adq) = _both(d, 0.3)
    assert not np.isfinite(st[0]) and not np.isfinite(ast[0])
    assert np.isnan(dl[0][d["avail"][0] != 0]).all() and np.isnan(adl[0][d["avail"][0] != 0]).all()
    assert np.all(dl[0][d["avail"][0] == 0] == 0)
    np.testing.assert_allclose(dl[1:], adl[1:], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(st[1:], ast[1:], rtol=1e-12)


@pytest.mark.parametrize("case", FIX_CASES, ids=case_name)
def test_oracle_reproduces_the_reference_fixture(case):
    """The oracle against every update of the unmodified reference; the fixture's initial state_dict (actors, critics
    and target critics) loads into the product model with strict=True."""
    g = np.load(GOLDEN)
    pre = case_name(case) + "/"
    _, model = build_product_model(case, "cpu")
    keys = [k[len(pre) + 5:] for k in g.files if k.startswith(pre + "init/")]
    assert any(k.startswith("target_critics.") for k in keys)
    model.load_state_dict({k: torch.from_numpy(g[pre + "init/" + k]) for k in keys}, strict=True)
    orc = COMALearnerOracle(model, case)
    for it in range(FIX_UPDATES):
        info = orc.update(fixture_batch(g, pre, it), case[2])
        np.testing.assert_allclose([info[k] for k in INFO_KEYS], g[pre + "infos"][it], rtol=1e-5, atol=1e-7,
                                   err_msg=f"update {it}")
        if it in FIX_SNAPSHOTS:
            sd = orc.state_dict()
            flat = np.concatenate([sd[k].detach().numpy().reshape(-1) for k in keys])
            np.testing.assert_allclose(flat, g[pre + f"after{it}"], rtol=1e-5, atol=1e-6)


def test_abi_symbols_and_argument_checks_without_gpu():
    from xuance_b200 import _lib
    for s in ("xb_coma_critic_input", "xb_coma_loss_fwd_bwd", "xb_coma_act"):
        assert s in _lib.exported_symbols()
    lib = _lib.load()
    EINVAL, ERANGE = -1, -3
    j = 256  # any non-NULL pointer: validation returns before the device is touched

    def ci(**k):
        return lib.xb_coma_critic_input(k.get("state", j), j, j, k.get("B", 2), k.get("n", 3), k.get("T", 4), 6, 8,
                                        k.get("A", 5), j, None)
    assert ci(state=None) == EINVAL and ci(B=0) == EINVAL and ci(T=0) == EINVAL and ci(A=0) == EINVAL
    assert ci(A=65) == ERANGE and ci(n=33) == ERANGE

    def loss(**k):
        R = k.get("R", 24)
        return lib.xb_coma_loss_fwd_bwd(k.get("logits", j), k.get("avail"), k.get("ld", 0), j, j, j, j,
                                        k.get("eps", j), j, R, k.get("A", 5), k.get("Rt", R), j, j, j, j, None)
    assert loss(logits=None) == EINVAL and loss(eps=None) == EINVAL and loss(R=0) == EINVAL
    assert loss(Rt=12) == EINVAL and loss(avail=j, ld=4) == EINVAL and loss(A=0) == EINVAL
    assert loss(A=65) == ERANGE

    def act(**k):
        return lib.xb_coma_act(k.get("logits", j), k.get("avail"), k.get("ld", 0), j, None, k.get("N", 6),
                               k.get("A", 5), k.get("out", j), None, None, None)
    assert act(logits=None) == EINVAL and act(N=0) == EINVAL and act(out=None) == EINVAL
    assert act(avail=j, ld=3) == EINVAL and act(A=65) == ERANGE


def test_shipped_configs_and_registries():
    import yaml
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.learners import REGISTRY_Learners
    for env_id in ("3m", "5m_vs_6m"):
        cfg = vars(get_arguments("coma", "sc2", env_id))
        path = os.path.join(ROOT, "xuance_b200", "configs", "coma", "sc2", env_id + ".yaml")
        for k, v in yaml.safe_load(open(path)).items():
            assert cfg[k] == v, k
        assert (cfg["agent"], cfg["learner"], cfg["use_rnn"], cfg["rnn"], cfg["recurrent_hidden_size"],
                cfg["sync_frequency"], cfg["gae_lambda"]) == ("COMA", "COMA_Learner", True, "GRU", 64, 200, 0.8)
    assert REGISTRY_Agents["COMA"].__name__ == "COMA_Agents"
    assert REGISTRY_Learners["COMA_Learner"].__name__ == "COMA_Learner"
    with pytest.raises(AttributeError, match="no config"):
        get_arguments("coma", "mpe", "simple_spread_v3")


def _cfg(**over):
    from xuance_b200.common.common_tools import get_arguments
    cfg = get_arguments("coma", "sc2", "3m")
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
    COMA = REGISTRY_Agents["COMA"]
    for over, match in ((dict(use_rnn=False), "use_rnn"), (dict(rnn="LSTM"), "LSTM"),
                        (dict(N_recurrent_layers=2), "N_recurrent_layers"), (dict(dropout=0.1), "dropout"),
                        (dict(recurrent_hidden_size=65), "recurrent_hidden_size"),
                        (dict(use_parameter_sharing=False), "parameter-sharing")):
        with pytest.raises(NotImplementedError, match=match):
            COMA(_cfg(**over), **spaces())
    with pytest.raises(NotImplementedError, match="64 actions"):
        COMA(_cfg(), **spaces(act=Discrete(65)))
    with pytest.raises(NotImplementedError, match="32 agents"):
        COMA(_cfg(), **spaces(n=33))
    with pytest.raises(ValueError, match="Discrete"):
        COMA(_cfg(), **spaces(act=Box(-1, 1, (2,))))


def test_k4c_compiles_without_spills(tmp_path):
    flags = [f for f in build.NVCC_FLAGS if f not in ("--use_fast_math=false", "-shared")]
    cmd = [build._nvcc()] + flags + ["-c", os.path.join(build.CSRC, "coma.cu"), "-o", str(tmp_path / "coma.o")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    kernels, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S*coma\S*)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            kernels[cur] = sum(int(x) for x in m.groups())
            cur = None
    assert len(kernels) == 11, log
    assert {k: v for k, v in kernels.items() if v} == {}
