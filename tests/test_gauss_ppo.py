"""CPU side of continuous-control PPO: the Gaussian oracle against the reference's fixture, the float64 references of K4G /
K10G against torch autograd, the C-ABI argument checks of the new entry points, and the Pendulum environment."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import gauss_refs as gr
from gauss_refs import ppo_gauss_samples
from helpers import seeded_state_dict
from oracle_gauss import GaussianActorCriticOracle, PPOGaussLearnerOracle, ppo_gauss_terms, pg_gauss_terms

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
D64 = torch.float64


def test_ppo_gauss_update_matches_reference():
    """Three updates of the Gaussian restatement reproduce the unmodified reference's PPO_Learner on
    SharedActorCritic(Basic_MLP, GaussianActorHead(Tanh), ValueHead) (tests/golden/ppo_gauss_update.npz)."""
    g = np.load(os.path.join(G, "ppo_gauss_update.npz"))
    obs_dim, D, B = 17, 6, 64
    model = GaussianActorCriticOracle(obs_dim, D)
    model.load_state_dict(seeded_state_dict(model.state_dict(), 17))
    lrn = PPOGaussLearnerOracle(model, end_factor_lr_decay=0.5, total_iters=int(g["total_iters"]))
    rng = np.random.default_rng(23)
    for it in range(3):
        info = lrn.update(**ppo_gauss_samples(rng, it, B, obs_dim, D))
        got = [info["actor_loss"], info["critic_loss"], info["entropy"], info["learning_rate"], info["predict_value"],
               float(info["clip_ratio"])]
        np.testing.assert_allclose(got, g["infos"][it], rtol=1e-5, atol=1e-7)
    assert g["infos"][1][5] > 0.9            # the off-policy batch: nearly every ratio is outside the clip range
    for k, v in model.state_dict().items():
        flat = v.detach().reshape(-1)
        np.testing.assert_allclose(flat[:64].numpy(), g[f"final_head/{k}"], rtol=1e-4, atol=1e-7, err_msg=k)
        np.testing.assert_allclose(flat.double().abs().sum().item(), g[f"final_digest/{k}"][1], rtol=1e-6)
    np.testing.assert_allclose(model.actor.log_std.detach().numpy(), g["final/actor.log_std"], rtol=1e-5, atol=1e-7)


def _gauss_inputs(rng, B, D, spread=1.0):
    mu = (rng.normal(size=(B, D)) * 0.7).astype(np.float32)
    ls = (rng.normal(size=D) * 0.4).astype(np.float32)
    x = (mu + np.exp(ls) * rng.normal(size=(B, D)) * spread).astype(np.float32)
    return mu, ls, x


@pytest.mark.parametrize("loss_kind", [0, 1])
def test_ppo_gauss_reference_matches_oracle_autograd(loss_kind):
    rng = np.random.default_rng(10 + loss_kind)
    B, D, clip, vf, ent = 64, 5, 0.25, 0.25, 0.01
    mu, ls, x = _gauss_inputs(rng, B, D)
    terms, _ = gr.gauss_logp_terms(mu, ls, x)
    ratio = np.concatenate([rng.uniform(0.5, 0.74, B // 4), rng.uniform(0.76, 1.24, B // 4),
                            rng.uniform(1.26, 2.0, B // 4), np.ones(B - 3 * (B // 4))])
    old = (terms.sum(1) - np.log(ratio)).astype(np.float32)
    adv = rng.normal(size=B).astype(np.float32)
    adv[::7] = 0.0
    v, ret = rng.normal(size=B).astype(np.float32), rng.normal(size=B).astype(np.float32)
    p = lambda a: nn.Parameter(torch.tensor(a, dtype=D64))
    tmu, tls, tv = p(mu), p(ls), p(v)
    a_t, adv_t, ret_t = torch.tensor(x, dtype=D64), torch.tensor(adv, dtype=D64), torch.tensor(ret, dtype=D64)
    if loss_kind == 0:
        a_loss, c_loss, e_loss, r = ppo_gauss_terms(tmu, tls, tv, a_t, ret_t, adv_t, torch.tensor(old, dtype=D64), clip)
        r = r.detach().numpy()
        cf = ((r < 1 - clip).sum() + (r > 1 + clip).sum()) / B
    else:
        a_loss, e_loss, _ = pg_gauss_terms(tmu, tls, a_t, adv_t)
        c_loss, cf = nn.functional.mse_loss(tv, ret_t), 0.0
    loss = a_loss - ent * e_loss + vf * c_loss
    loss.backward()
    dmu, dls, dv, st = gr.ppo_gauss_loss(mu, ls, v, x, old, adv, ret, B, np.float32(clip), vf, ent, loss_kind)
    close = lambda got, want, tol=1e-12: np.testing.assert_allclose(got, want, rtol=tol, atol=tol)
    close(dmu, tmu.grad.numpy())
    close(dls, tls.grad.numpy())
    close(dv, tv.grad.numpy())
    # ppo_gauss_terms rounds the ratio to float32 (ppo_learner.py's .float()): the surrogate agrees to float32 precision
    close(st, [a_loss.item(), c_loss.item(), e_loss.item(), v.astype(np.float64).mean(), cf, loss.item()], tol=4 * gr.EPS32)


@pytest.mark.parametrize("mode", ["forced", "stochastic", "deterministic"])
def test_gaussian_act_reference_matches_torch_normal(mode):
    from xuance_b200.torch.rl_models import DiagGaussianDistribution
    rng = np.random.default_rng(3)
    N, D = 40, 6
    mu, ls, x = _gauss_inputs(rng, N, D)
    noise = rng.normal(size=(N, D)).astype(np.float32)
    act, logp, ent = gr.gaussian_act(mu, ls, noise=noise if mode == "stochastic" else None,
                                     forced=x if mode == "forced" else None)
    d = DiagGaussianDistribution(D)
    d.set_param(torch.tensor(mu, dtype=D64), torch.tensor(ls, dtype=D64).exp())
    want = {"forced": x, "stochastic": mu.astype(np.float64) + np.exp(ls.astype(np.float64)) * noise,
            "deterministic": d.deterministic_sample().numpy()}[mode]
    if mode == "forced":
        assert act is None
    else:
        np.testing.assert_allclose(act, want, rtol=1e-15, atol=1e-15)
    np.testing.assert_allclose(logp, d.log_prob(torch.tensor(want, dtype=D64)).numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(ent, d.entropy().numpy(), rtol=1e-12, atol=1e-12)


def test_gauss_entry_points_validate_without_gpu():
    from xuance_b200 import _lib
    lib = _lib.load()
    j = ctypes.c_void_p(0x1000)   # never dereferenced: validation fails first
    EINVAL, ERANGE = -1, -3
    for name in ("xb_ppo_gauss_loss_fwd_bwd", "xb_ppo_gauss_ws_doubles", "xb_gaussian_act"):
        assert name in _lib.exported_symbols() and hasattr(lib, name)
    assert lib.xb_ppo_gauss_ws_doubles(8, 6) == 6 and lib.xb_ppo_gauss_ws_doubles(257, 6) == 12
    assert lib.xb_ppo_gauss_ws_doubles(1 << 40, 64) == 64 * 2048

    def k4g(B=8, D=6, B_total=8, old=j, kind=0, dmu=j, ws_n=1 << 20):
        return lib.xb_ppo_gauss_loss_fwd_bwd(j, j, j, j, old, j, j, B, D, B_total, 0.2, 0.25, 0.01, kind, dmu, j, j, j,
                                             j, j, ws_n, None)
    assert k4g(D=65) == ERANGE
    assert k4g(B_total=4) == EINVAL                 # B_total < B
    assert k4g(old=None) == EINVAL                  # the clip surrogate needs old_logp
    assert k4g(kind=2) == EINVAL
    assert k4g(dmu=None) == EINVAL
    assert k4g(D=0) == EINVAL and k4g(B=0) == EINVAL
    assert k4g(ws_n=5) == EINVAL                    # workspace smaller than D * blocks
    assert lib.xb_gaussian_act(j, j, j, None, 8, 6, None, None, None, None) == EINVAL     # no output
    assert lib.xb_gaussian_act(j, None, j, None, 8, 6, j, None, None, None) == EINVAL     # no log_std
    assert lib.xb_gaussian_act(j, j, j, None, 0, 6, j, None, None, None) == EINVAL


def test_pendulum_env_contract_and_torque_clip():
    from xuance_b200.environment import REGISTRY_ENV, XuanCeEnvWrapper, DummyVecEnv
    from xuance_b200.environment.envs import PendulumEnv
    assert REGISTRY_ENV["Pendulum-v1"] is PendulumEnv
    env = PendulumEnv(seed=0)
    assert env.action_space.shape == (1,) and env.observation_space.shape == (3,)
    obs, info = env.reset(seed=4)
    assert obs.dtype == np.float32 and obs.shape == (3,) and abs(obs[0] ** 2 + obs[1] ** 2 - 1) < 1e-6
    # a torque beyond the limit acts as the limit: same next state and the cost of u = 2
    a, b = PendulumEnv(seed=1), PendulumEnv(seed=1)
    a.reset(seed=9), b.reset(seed=9)
    th, thdot = a.state
    o1, r1, t1, tr1, _ = a.step(np.array([7.5], np.float32))
    o2, r2, _, _, _ = b.step(np.array([2.0], np.float32))
    assert np.array_equal(o1, o2) and r1 == r2 and not t1 and not tr1
    norm = ((th + np.pi) % (2 * np.pi)) - np.pi
    assert r1 == pytest.approx(-(norm ** 2 + 0.1 * thdot ** 2 + 0.001 * 4.0))
    o3, _, _, _, _ = b.step(np.array([-30.0], np.float32))
    c = PendulumEnv(seed=1)
    c.reset(seed=9)
    c.step(np.array([2.0]))
    assert np.array_equal(o3, c.step(np.array([-2.0]))[0])
    # truncation after 200 steps, never terminated; the vector env reports reset observations and scores
    vec = DummyVecEnv([lambda i=i: XuanCeEnvWrapper(PendulumEnv(seed=i)) for i in range(3)], 0)
    obs, _ = vec.reset()
    assert obs.shape == (3, 3)
    for t in range(200):
        obs, rew, term, trunc, infos = vec.step(np.zeros((3, 1), np.float32))
        assert not term.any() and rew.shape == (3,) and (rew <= 0).all()
        assert trunc.all() == (t == 199)
    assert all("reset_obs" in i and i["episode_step"] == 200 for i in infos)


def test_pendulum_config_resolves():
    from xuance_b200.common.common_tools import get_arguments
    cfg = get_arguments("ppo", "classic_control", "Pendulum-v1")
    assert cfg.env_id == "Pendulum-v1" and cfg.policy == "Gaussian_AC" and cfg.activation_action == "tanh"
    assert (cfg.parallels, cfg.horizon_size, cfg.n_epochs, cfg.n_minibatch) == (10, 256, 8, 8)
