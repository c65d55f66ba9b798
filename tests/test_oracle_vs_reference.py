"""CPU: the oracle next to the unmodified reference on fresh seeded inputs - the second way the oracle is pinned (the first
is tests/golden/*.npz).  The reference's side was recorded by tests/golden/make_reference_live.py into
tests/golden/reference_live.pkl.gz; models start from helpers.seeded_state_dict on both sides, final parameters are
compared on helpers.param_sample."""
import gzip
import os
import pickle
import random

import numpy as np
import pytest
import torch

from helpers import synth_rollout, fill_buffers, qmix_episode_stream, same_structure as _same, seeded_state_dict, \
    param_sample, digest

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_live.pkl.gz")


@pytest.fixture(scope="module")
def ref():
    with gzip.open(FIXTURE, "rb") as fh:
        return pickle.load(fh)


def _close_params(sd, want, rtol=1e-5, atol=1e-6):
    got = param_sample(sd)
    assert set(got) == set(want)
    for k in want:
        np.testing.assert_allclose(got[k], want[k], rtol=rtol, atol=atol, err_msg=k)


@pytest.mark.parametrize("seed,use_gae", [(0, True), (1, True), (2, False)])
def test_onpolicy_buffer_live(ref, seed, use_gae):
    from oracle.onpolicy import OnPolicyBufferOracle
    r = ref["onpolicy"][seed]
    rng = np.random.default_rng(seed)
    N, T = 5, 33
    ro = synth_rollout(rng, N, T, (3,), obs_dtype=np.float32, p_term=0.1)
    o = OnPolicyBufferOracle((3,), (), {'old_logp': ()}, N, T, use_gae=use_gae)
    fill_buffers([o], ro, [(4, 1, np.float32(0.2)), (9, 3, 0.0), (20, 1, np.float32(-0.7))])
    assert np.array_equal(r["returns"], o.returns) and np.array_equal(r["advantages"], o.advantages)
    idx = rng.permutation(N * T)[:50]
    s2 = o.sample(idx)
    for k in ('obs', 'actions', 'returns', 'values', 'advantages'):
        assert np.array_equal(r["sample"][k], s2[k]) and r["sample"][k].dtype == s2[k].dtype, k


@pytest.mark.parametrize("alpha", [0.5, 0.6])
def test_per_buffer_live(ref, alpha):
    from oracle.replay import PerReplayOracle
    events = iter(ref["per"][alpha])
    rng = np.random.default_rng(int(alpha * 10))
    N, S, B = 4, 64, 32
    o = PerReplayOracle((3,), (), N, N * S, B, alpha=alpha)
    for t in range(100):
        st = (rng.normal(size=(N, 3)).astype(np.float32), rng.integers(0, 4, N), rng.normal(size=N).astype(np.float32),
              rng.random(N) < 0.1, rng.normal(size=(N, 3)).astype(np.float32))
        o.store(*st)
        if t > 10 and t % 3 == 0:
            r = next(events)
            assert r["t"] == t
            random.seed(t)
            s2 = o.sample(0.4)
            assert np.array_equal(r['step_choices'], s2['step_choices']) and np.array_equal(r['weights'], s2['weights'])
            td = np.abs(rng.normal(size=B)).astype(np.float32)
            td[3] = 0
            o.update_priorities(s2['step_choices'], td)
            for i in range(N):
                assert r["sum"][i] == digest(o.sum[i].v.astype(np.float64))
                assert r["min"][i] == digest(o.min[i].v.astype(np.float64))
            assert np.array_equal(r["max_priority"], o.max_priority)


def _qmix_oracle(n, obs_dim, A, S, total_iters, lr_decay=0.5, seed=0):
    from oracle.qmix import QMIXModelOracle, QMIXLearnerOracle
    keys = [f"agent_{i}" for i in range(n)]
    om = QMIXModelOracle(n, obs_dim, A, S)
    om.load_state_dict(seeded_state_dict(om.state_dict(), seed), strict=True)
    orc = QMIXLearnerOracle(om, keys, learning_rate=7e-4, sync_frequency=2, double_q=True, end_factor_lr_decay=lr_decay,
                            total_iters=total_iters, detach_q_eval=True)   # the reference as it is (see oracle/qmix.py)
    return keys, om, orc


def test_qmix_buffer_and_learner_live(ref):
    from oracle.qmix import EpisodeReplayOracle
    r = ref["qmix"]
    n, obs_dim, A, S, T = 5, 72, 12, 98, 12
    keys, om, orc = _qmix_oracle(n, obs_dim, A, S, r["total_iters"])
    init = {k: v.clone() for k, v in om.state_dict().items()}
    n_envs, C, Be = 3, 12, 6
    ob = EpisodeReplayOracle(keys, obs_dim, S, n_envs, C, Be, T)
    for ev in qmix_episode_stream(np.random.default_rng(0), keys, n_envs, T, obs_dim, A, S, 5):
        if ev[0] == 'store':
            ob.store(**ev[1])
        else:
            ob.finish_path(ev[1], **ev[2])
    for k in ('obs', 'actions', 'rewards', 'terminals', 'agent_mask'):
        for a in keys:
            assert r["data"][k][a] == digest(ob.data[k][a]), k
    assert r["data"]['filled'] == digest(ob.data['filled']) and r["data"]['state'] == digest(ob.data['state'])
    assert r["ptr"] == ob.ptr and r["size"] == ob.size
    for it in range(3):
        np.random.seed(it)
        i2 = orc.update(ob.sample())
        i1 = r["updates"][it]
        np.testing.assert_allclose(i1['loss_Q'], i2['loss_Q'], rtol=1e-5)
        np.testing.assert_allclose(i1['predictQ'], i2['predictQ'], rtol=1e-5, atol=1e-7)
        assert i1['learning_rate'] == i2['learning_rate']
    sd = om.state_dict()
    _close_params(sd, r["final"])
    # reference quirk (asserted on the reference when the fixture was recorded): with use_rnn=True its agent networks
    # never receive a gradient - only the mixer moves; the oracle in detach_q_eval mode does the same
    moved = {k for k in sd if k.startswith("individual_q_networks") and not torch.equal(sd[k], init[k])}
    assert not moved, moved


def test_sac_learner_live(ref):
    from oracle.sac import SACModelOracle, SACLearnerOracle
    r = ref["sac"]
    obs_dim, act_dim, B = 17, 6, 64
    om = SACModelOracle(obs_dim, act_dim)
    om.load_state_dict(seeded_state_dict(om.state_dict(), 1), strict=True)
    orc = SACLearnerOracle(om, end_factor_lr_decay=0.7, total_iters=r["total_iters"])
    rng = np.random.default_rng(1)
    for it in range(3):
        s = {"obs": rng.normal(size=(B, obs_dim)).astype(np.float32),
             "actions": rng.uniform(-1, 1, size=(B, act_dim)).astype(np.float32),
             "obs_next": rng.normal(size=(B, obs_dim)).astype(np.float32),
             "rewards": rng.normal(size=B).astype(np.float32), "terminals": (rng.random(B) < 0.1).astype(np.float32)}
        # the reference drew its noise from torch's global RNG seeded with 100 + it: replay the same stream
        torch.manual_seed(100 + it)
        n1 = torch.randn(B, act_dim)
        n2 = torch.randn(B, act_dim)
        i2 = orc.update(n1, n2, **s)
        for k in ("Qloss", "Ploss", "Qvalue", "alpha", "alpha_loss"):
            np.testing.assert_allclose(i2[k], r["updates"][it][k], rtol=1e-5, atol=1e-6, err_msg=k)
    _close_params(om.state_dict(), r["final"])


@pytest.mark.parametrize("kind", ["a2c", "pg", "ddqn"])
def test_sibling_learners_live(ref, kind):
    """A2C / PG / DDQN (SURVEY.md section 8f-3): oracle variants next to the reference learners."""
    from oracle.nets import SharedActorCriticOracle, DeepQNetworkOracle
    from oracle.learners import PPOLearnerOracle, DQNLearnerOracle
    r = ref["siblings"][kind]
    A, B = 5, 12
    rng = np.random.default_rng(3)
    if kind == "ddqn":
        om = DeepQNetworkOracle(A)
        om.load_state_dict(seeded_state_dict(om.state_dict(), 2), strict=True)
        orc = DQNLearnerOracle(om, learning_rate=2.5e-4, sync_frequency=2, use_grad_clip=True, end_factor_lr_decay=0.5,
                               total_iters=r["total_iters"], double_q=True)
    else:
        om = SharedActorCriticOracle(A)
        om.load_state_dict(seeded_state_dict(om.state_dict(), 2), strict=True)
        # a2c_learner.py:21: LinearLR(total_iters=config.running_steps); pg_learner.py:22: total_iters=self.total_iters
        orc = PPOLearnerOracle(om, end_factor_lr_decay=0.5, kind=kind,
                               total_iters=4096 * 10 if kind == "a2c" else r["total_iters"])
    for it in range(3):
        s = {"obs": rng.integers(0, 256, size=(B, 84, 84, 4), dtype=np.uint8).astype(np.float32),
             "actions": rng.integers(0, A, size=B).astype(np.float32),
             "returns": rng.normal(size=B).astype(np.float32), "advantages": rng.normal(size=B).astype(np.float32),
             "aux_batch": {"old_logp": np.zeros(B, np.float32)},
             "obs_next": rng.integers(0, 256, size=(B, 84, 84, 4), dtype=np.uint8).astype(np.float32),
             "rewards": rng.normal(size=B).astype(np.float32), "terminals": (rng.random(B) < 0.2).astype(np.float32)}
        i2, i1 = orc.update(**s), r["updates"][it]
        if kind == "ddqn":
            np.testing.assert_allclose(i2["Qloss"], i1["Qloss"], rtol=1e-5)
        else:
            np.testing.assert_allclose(i2["actor_loss"], i1["actor_loss"], rtol=1e-5, atol=1e-7)
            np.testing.assert_allclose(i2["entropy"], i1["entropy"], rtol=1e-5)
    _close_params(om.state_dict(), r["final"])


def test_multi_agent_vector_env_live(ref):
    """DummyVecMultiAgentEnv + XuanCeMultiAgentEnvWrapper (the QMIX caller side, vector_envs/dummy/dummy_vec_maenv.py:17-84,
    environment/utils/wrapper.py:141-226) next to the reference classes' recorded run over the SAME raw synthetic
    environments: identical observations, reward / terminated dicts, truncation flags and infos (episode_step,
    episode_score, agent_mask, avail_actions, state, reset_obs / reset_avail_actions / reset_state at episode ends) step
    for step."""
    from xuance_b200.environment.ma_envs import SyntheticSMACEnv, XuanCeMultiAgentEnvWrapper
    from xuance_b200.environment.vector_envs.dummy_vec_maenv import DummyVecMultiAgentEnv
    r = ref["ma_vec_env"]
    kw = dict(n_agents=3, obs_dim=16, state_dim=20, n_actions=5, episode_limit=7, p_death=0.1)
    n_envs = 3
    ov = DummyVecMultiAgentEnv([lambda env_seed=0: XuanCeMultiAgentEnvWrapper(SyntheticSMACEnv(seed=env_seed, **kw))
                                for _ in range(n_envs)], 11)
    assert r["num_envs"] == ov.num_envs and r["agents"] == list(ov.agents) and r["num_agents"] == ov.num_agents
    assert r["max_episode_steps"] == ov.max_episode_steps and r["state_shape"] == tuple(ov.state_space.shape)
    (ro, ri), (oo, oi) = r["reset"], ov.reset()
    _same(ro, oo, "reset obs"), _same(ri, oi, "reset info")
    ends = 0
    for t, st in enumerate(r["steps"]):
        o = ov.step(st["actions"])
        for name, x, y in zip(("obs", "rewards", "terminated", "truncated", "infos"), st["out"], o):
            _same(x, y, "t=%d %s" % (t, name))
        _same(st["state"], ov.buf_state, "state"), _same(st["avail"], ov.buf_avail_actions, "avail")
        ends += sum("reset_obs" in i for i in st["out"][4])
    assert ends >= 5                                    # episode ends (death of all agents / truncation) were exercised
    ov.close()


def test_qmix_action_mask_variant_against_the_reference_with_its_slice_corrected(ref):
    """use_rnn=True with use_actions_mask=True: the reference slices the AGENT axis of the availability mask
    (iql_learner.py:78, ``[:, 1:]``) and raises; the evidently intended statement slices the time axis (``[:, :, 1:]``).
    The oracle's masked variant (and through it xb_qmix_select_fwd's masked arg-max / target, tests/test_gpu_qmix.py) is pinned
    here against the reference learner with that ONE expression corrected in memory when the fixture was recorded
    (tests/golden/make_reference_live.py; nothing of the reference source is stored here), on the samples its replay
    buffer drew."""
    r = ref["qmix_action_mask"]
    assert r["unpatched_raised"]                        # the reference as it is cannot run this configuration
    n, obs_dim, A, S = 4, 24, 7, 30
    _, om, orc = _qmix_oracle(n, obs_dim, A, S, r["total_iters"], seed=3)
    snap = {k: v.clone() for k, v in om.state_dict().items()}
    orc.use_actions_mask = True
    for it in range(3):
        s = r["samples"][it]
        assert s['avail_actions'][f"agent_0"].shape[-1] == A
        i2, i1 = orc.update(s), r["updates"][it]
        np.testing.assert_allclose(i1['loss_Q'], i2['loss_Q'], rtol=1e-5)
        np.testing.assert_allclose(i1['predictQ'], i2['predictQ'], rtol=1e-5, atol=1e-7)
    _close_params(om.state_dict(), r["final"])
    # the masks mattered: the same first update without them has a different loss
    _, om_m, orc_m = _qmix_oracle(n, obs_dim, A, S, r["total_iters"], seed=3)
    _, om_u, orc_u = _qmix_oracle(n, obs_dim, A, S, r["total_iters"], seed=3)
    om_m.load_state_dict(snap, strict=True), om_u.load_state_dict(snap, strict=True)
    om_m.copy_target(), om_u.copy_target()
    orc_m.use_actions_mask = True
    s = r["samples"][0]
    assert abs(orc_m.update(s)['loss_Q'] - orc_u.update(s)['loss_Q']) > 1e-6
