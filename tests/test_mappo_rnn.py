"""CPU tests of recurrent MAPPO: the 3m config and shape, the reference behaviour the buffer fixture pins (stale staging
tail, no advantage normalisation, the non-GAE ValueNorm failure), and the scope errors that need no GPU."""
import os

import numpy as np
import pytest
import yaml

from mappo_rnn_refs import KEYS, N_AGENTS, T_MAX, SAMPLE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "mappo_rnn_buffer.npz")
CONFIG = os.path.join(ROOT, "xuance_b200", "configs", "mappo", "sc2", "3m.yaml")


def test_3m_config_resolves_with_the_reference_keys():
    from xuance_b200.common.common_tools import get_arguments
    cfg = vars(get_arguments("mappo", "sc2", "3m"))
    for k, v in yaml.safe_load(open(CONFIG)).items():
        assert cfg[k] == v, k
    assert (cfg["use_rnn"], cfg["representation"], cfg["rnn"], cfg["N_recurrent_layers"], cfg["normalize"]) == \
        (True, "Basic_RNN", "GRU", 1, "LayerNorm")
    assert cfg["fc_hidden_sizes"] == [64, 64, 64] and cfg["recurrent_hidden_size"] == 64 and cfg["buffer_size"] == 128
    ff = yaml.safe_load(open(os.path.join(ROOT, "xuance_b200", "configs", "mappo", "sc2", "5m_vs_6m.yaml")))
    assert ff["use_rnn"] is False and ff["representation"] == "Basic_MLP"


def test_3m_shape():
    from xuance_b200.environment.ma_envs import SMAC_SHAPES, SyntheticSMACEnv
    assert SMAC_SHAPES["3m"] == dict(n_agents=3, obs_dim=30, state_dim=48, n_actions=9, episode_limit=60)
    env = SyntheticSMACEnv(seed=1, map_name="3m")
    assert (env.num_agents, env.obs_dim, env.state_dim, env.n_actions, env.max_episode_steps) == (3, 30, 48, 9, 60)


def test_fixture_pins_the_reference_behaviour():
    g = np.load(GOLDEN)
    case = "gae1_vn1/"
    # env 0 finished an episode of 3 steps, then one of 2: the staging keeps the first episode's step 2 behind the
    # second's tail (store_episodes clears only `filled`), and the ring slot of the second episode carries it along
    for f in ("rewards", "values", "returns", "advantages"):
        for k in KEYS:
            ring = g[case + f"data/{f}/{k}"]
            assert ring[1, 2] == ring[0, 2] and ring[1, 2] != 0, f     # slot 0: env 0 ep 1, slot 1: env 0 ep 2
    assert g[case + "data/filled"][1].sum() == 2 and g[case + "data/filled"][0].sum() == 3
    # no advantage normalisation in the recurrent sample, although use_advnorm=True
    for k in KEYS:
        np.testing.assert_array_equal(g[case + f"sample/advantages/{k}"], g[case + f"data/advantages/{k}"][SAMPLE])
        assert abs(g[case + f"sample/advantages/{k}"][g[case + "sample/filled"]].mean()) > 1e-3
    # non-GAE with a ValueNorm: the reference fails with a shape error
    assert "gae0_vn1/raises" in g.files and "gae0_vn1/data/returns/agent_0" not in g.files
    assert g["gae1_vn0/sample_meta"].tolist() == [len(SAMPLE), T_MAX]
    assert N_AGENTS == len(KEYS)


def test_ippo_keeps_raising():
    from xuance_b200.torch.agents.mappo_agents import IPPO_Agents
    with pytest.raises(NotImplementedError, match="IPPO"):
        IPPO_Agents(None)
