"""GPU: continuous-control PPO.  K4G (xb_ppo_gauss_loss_fwd_bwd) and K10G (xb_gaussian_act) through the C-ABI against the
float64 references of tests/gauss_refs.py at every D tier, the row counts where grid reductions go wrong, clip-heavy and
far-outside-the-clip ratios, the sharded-minibatch contract and run-to-run determinism; then PPO_Learner / A2C / PG on a
Box-space model against the Gaussian oracle and the reference's fixture, CUDA-graph capture, device staging of Box actions,
and learning on Pendulum-v1 with host and device rollouts.

Tolerances follow tests/test_gpu_kernel_edges.py: EPS = 2^-24, and each bound is built from the magnitude of what the
kernel adds (not of the result, which may cancel), with the number of roundings stated."""
import os
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn as nn

import gauss_refs as gr
from gauss_refs import ppo_gauss_samples
from helpers import seeded_state_dict, ppo_config

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EPS = gr.EPS32
f32 = np.float32
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
HP = dict(clip=0.2, vf_coef=0.25, ent_coef=0.01)


def _lib():
    from xuance_b200 import _lib
    return _lib


def _big_rows():
    """First row count in the grid-stride regime (XB_MAX_PARTIALS blocks of 256 threads)."""
    max_partials = (_lib().load().xb_scratch_doubles() - 8) // 8
    return max_partials * 256 + 257


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _within(got, want, tol, what):
    got = np.asarray(got.cpu().numpy() if torch.is_tensor(got) else got, np.float64)
    want, tol = np.broadcast_to(np.asarray(want, np.float64), got.shape), np.broadcast_to(tol, got.shape)
    err = np.abs(got - want)
    bad = ~(err <= tol)                       # NaN (an unwritten output) fails too
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, np.nan_to_num(err / np.maximum(tol, 1e-300), nan=np.inf), 0)), got.shape)
        raise AssertionError(f"{what}: {bad.sum()} of {bad.size} outside tolerance; at {i}: got {got[i]!r} want {want[i]!r} "
                             f"tol {tol[i]!r}")


# ====================================================================================================== K4G
def _gauss_inputs(B, D, seed):
    """mu in +-1.5, log_std in [-1.5, 1], actions mu + sigma * N(0, 1.5^2); ratios in six classes: both sides of 1 -+ clip
    (never within 1e-2 of a bound), exactly 1, and far outside (e^-12..e^-5, e^5..e^12); adv = 0 on 10 % of the rows."""
    rng = np.random.default_rng(seed)
    mu = rng.uniform(-1.5, 1.5, (B, D)).astype(f32)
    ls = rng.uniform(-1.5, 1.0, D).astype(f32)
    x = (mu + np.exp(ls) * rng.normal(size=(B, D)) * 1.5).astype(f32)
    logp = gr.gauss_logp_terms(mu, ls, x)[0].sum(1)
    kind = rng.integers(0, 6, B)
    ratio = np.select([kind == 0, kind == 1, kind == 2, kind == 3, kind == 4],
                      [rng.uniform(0.3, 0.79, B), rng.uniform(0.81, 1.19, B), rng.uniform(1.21, 3.0, B),
                       np.ones(B), np.exp(rng.uniform(-12, -5, B))], np.exp(rng.uniform(5, 12, B)))
    adv = rng.normal(size=B).astype(f32)
    adv[rng.random(B) < 0.1] = 0.0
    return dict(mu=mu, log_std=ls, value=rng.normal(size=B).astype(f32), actions=x,
                old_logp=(logp - np.log(ratio)).astype(f32), adv=adv, ret=rng.normal(size=B).astype(f32))


def _ws(D):
    return torch.full((int(_lib().load().xb_ppo_gauss_ws_doubles(1 << 40, D)),), float("nan"), dtype=torch.float64,
                      device=DEV)


def _run_gauss(x, lo, hi, B_total, kind, scratch, ws=None):
    B, D = hi - lo, x["mu"].shape[1]
    t = {k: _t(v if k == "log_std" else v[lo:hi]) for k, v in x.items()}
    ws = _ws(D) if ws is None else ws
    dmu, dls, dv, st = _nan(B, D), _nan(D), _nan(B), _nan(8)
    L = _lib()
    L.call("xb_ppo_gauss_loss_fwd_bwd", *[L.ptr(t[k]) for k in ("mu", "log_std", "value", "actions", "old_logp", "adv",
                                                                  "ret")],
           B, D, B_total, HP["clip"], HP["vf_coef"], HP["ent_coef"], kind, *[L.ptr(v) for v in (dmu, dls, dv, st, scratch, ws)],
           ws.numel())
    return dmu, dls, dv, st


def _gauss_ref_and_tol(x, B_total, kind):
    """z_j = (x - mu) * (1 / sigma): x - mu, 1/exp and the product are 4 roundings relative to c_j = (|x| + |mu|) / sigma +
    |z_j|; logp adds D + 2 roundings of the magnitudes z^2/2 + |log_std| + log sqrt(2 pi) of its terms, so |logp error| <=
    e = 4 EPS sum_j |z_j| c_j + (D + 2) EPS sum_j (z_j^2/2 + |log_std_j| + log sqrt(2 pi)).
    ratio, d_logp (6 more roundings) then carry a relative error e + 8 EPS:
      dmu_j      : |d_logp| ((e + 10 EPS) |z_j| + 4 EPS c_j) / sigma_j
      dlog_std_j : sum_b |d_logp| ((e + 10 EPS)(z^2 + 1) + 8 EPS c_j |z_j|), + 2 EPS of the result (double sums, 1 rounding)."""
    mu, ls, xa = (np.asarray(x[k], np.float64) for k in ("mu", "log_std", "actions"))
    dmu, dls, dv, st = gr.ppo_gauss_loss(x["mu"], x["log_std"], x["value"], x["actions"], x["old_logp"], x["adv"],
                                         x["ret"], B_total, f32(HP["clip"]), f32(HP["vf_coef"]), f32(HP["ent_coef"]), kind)
    terms, z = gr.gauss_logp_terms(x["mu"], x["log_std"], x["actions"])
    B, D = z.shape
    sig = np.exp(ls)[None, :]
    c = (np.abs(xa) + np.abs(mu)) / sig + np.abs(z)
    mag = 0.5 * z * z + np.abs(ls)[None, :] + gr.LOG_SQRT_2PI          # what each log-prob term adds up
    e = 4 * EPS * (np.abs(z) * c).sum(1) + (D + 2) * EPS * mag.sum(1)
    logp = terms.sum(1)
    ratio = np.exp(logp - x["old_logp"]) if kind == 0 else np.ones(B)
    dl = np.abs(x["adv"]) * np.maximum(ratio, 1.0) / B_total
    r = (e + 10 * EPS)[:, None]
    tol_dmu = dl[:, None] * (r * np.abs(z) + 4 * EPS * c) / sig
    tol_dls = (dl[:, None] * (r * (z * z + 1) + 8 * EPS * c * np.abs(z))).sum(0) + 2 * EPS * np.abs(dls) \
        + 2 * EPS * HP["ent_coef"] * B / B_total
    v, rr = x["value"].astype(np.float64), x["ret"].astype(np.float64)
    tol_dv = 4 * EPS * HP["vf_coef"] * 2 * (np.abs(v) + np.abs(rr)) / B_total
    smin_mag = np.abs(x["adv"]) * (np.maximum(ratio, 1.0 + HP["clip"]) * (e + 8 * EPS) if kind == 0 else e + np.abs(logp) * 2 * EPS)
    ent_terms = (0.5 + gr.LOG_SQRT_2PI + np.abs(ls)).sum()             # summands, not their (cancelling) sum
    t_a = smin_mag.sum() / B_total
    t_c = 4 * EPS * ((v - rr) ** 2).sum() / B_total
    t_e = (D + 2) * EPS * ent_terms * B / B_total
    t_v = 2 * EPS * np.abs(v).sum() / B_total
    tol_st = np.array([t_a, t_c, t_e, t_v, 0.0, t_a + HP["ent_coef"] * t_e + HP["vf_coef"] * t_c])
    tol_st += 4 * EPS * (np.abs(st) + np.abs(st[0]) + np.abs(st[2]) * HP["ent_coef"] + np.abs(st[1]))
    return (dmu, dls, dv, st), (tol_dmu, tol_dls, tol_dv, tol_st)


def _check_gauss(out, x, B_total, kind, what=""):
    (dmu, dls, dv, st), (tmu, tls, tv, ts) = _gauss_ref_and_tol(x, B_total, kind)
    _within(out[0], dmu, tmu, what + "dmu")
    _within(out[1], dls, tls, what + "dlog_std")
    _within(out[2], dv, tv, what + "dvalue")
    got = out[3].cpu().numpy().astype(np.float64)
    _within(got[:6], st, ts, what + "stats")
    assert round(got[4] * B_total) == round(st[4] * B_total), what + "clip fraction counts a different number of rows"
    assert got[6] == 0 and got[7] == 0


@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("D", [1, 2, 3, 4, 5, 6, 8, 9, 17, 32, 33, 64])
def test_ppo_gauss_loss_tiers_and_row_counts(D, kind):
    scratch = _lib().scratch(DEV)
    sizes = [1, 255, 256, 257] + ([_big_rows()] if D in (1, 6) else [])
    for B in sizes:
        x = _gauss_inputs(B, D, seed=B * 100 + D)
        _check_gauss(_run_gauss(x, 0, B, B, kind, scratch), x, B, kind, f"D={D} B={B} kind={kind}: ")


def _shards(B, G):
    edges = np.linspace(0, B, G + 1).astype(int)
    return list(zip(edges[:-1], edges[1:]))


@pytest.mark.parametrize("G", [2, 3, 8])
def test_ppo_gauss_sharded_minibatch_contract(G):
    """A rank's shard launched with the global B_total writes the global minibatch's dmu / dvalue rows bit for bit; its
    dlog_std and statistics sum over the shards to the unsharded ones (one float32 rounding per shard and per sum)."""
    scratch = _lib().scratch(DEV)
    for D in (6, 33):
        B = 2400
        x = _gauss_inputs(B, D, seed=G + D)
        whole = _run_gauss(x, 0, B, B, 0, scratch)
        parts = [_run_gauss(x, lo, hi, B, 0, scratch) for lo, hi in _shards(B, G)]
        for i, name in ((0, "dmu"), (2, "dvalue")):
            np.testing.assert_array_equal(torch.cat([p[i] for p in parts]).cpu().numpy(), whole[i].cpu().numpy(), name)
        for i, name in ((1, "dlog_std"), (3, "stats")):
            ps = np.stack([p[i].cpu().numpy().astype(np.float64) for p in parts])
            w = whole[i].cpu().numpy().astype(np.float64)
            _within(ps.sum(0), w, (G + 1) * EPS * (np.abs(ps).sum(0) + np.abs(w)), f"G={G} D={D} summed {name}")
        summed = (whole[0], torch.from_numpy(sum(p[1].cpu().numpy() for p in parts)), whole[2],
                  torch.from_numpy(sum(p[3].cpu().numpy() for p in parts)))
        _check_gauss(summed, x, B, 0, f"G={G} D={D} summed: ")


def test_ppo_gauss_dlog_std_is_deterministic():
    """dlog_std (and every other output) is bit-identical over three launches at the full 2048-block grid, and over
    launches interleaved with K4 on one shared scratch and one workspace."""
    B = _big_rows()
    x = _gauss_inputs(B, 6, seed=5)
    runs = [_run_gauss(x, 0, B, B, 0, _lib().scratch(DEV)) for _ in range(3)]
    for r in runs[1:]:
        for a, b in zip(r, runs[0]):
            assert torch.equal(a, b)
    _check_gauss(runs[0], x, B, 0, "full grid: ")
    small = _gauss_inputs(300, 17, seed=6)
    solo_small = _run_gauss(small, 0, 300, 300, 1, _lib().scratch(DEV))
    L = _lib()
    scratch, ws = L.scratch(DEV), _ws(64)
    rng = np.random.default_rng(7)
    logits = _t(rng.normal(size=(1000, 6)).astype(f32))
    k4 = [_t(a) for a in (rng.normal(size=1000).astype(f32), rng.integers(0, 6, 1000).astype(f32),
                          rng.normal(size=1000).astype(f32) - 1.8, rng.normal(size=1000).astype(f32),
                          rng.normal(size=1000).astype(f32))]
    for rnd in range(2):
        assert all(torch.equal(a, b) for a, b in zip(_run_gauss(x, 0, B, B, 0, scratch, ws), runs[0])), rnd
        dz, dv, st = _nan(1000, 6), _nan(1000), _nan(8)
        L.call("xb_ppo_loss_fwd_bwd", L.ptr(logits), *[L.ptr(t) for t in k4], 1000, 6, 1000, 0.2, 0.25, 0.01, 0,
               *[L.ptr(t) for t in (dz, dv, st, scratch)])
        assert all(torch.equal(a, b) for a, b in zip(_run_gauss(small, 0, 300, 300, 1, scratch, ws), solo_small)), rnd
    _check_gauss(solo_small, small, 300, 1, "interleaved: ")


# ====================================================================================================== K10G
@pytest.mark.parametrize("D", [1, 6, 17, 64, 100])
@pytest.mark.parametrize("N", [1, 16, 129])
def test_gaussian_act_modes_against_float64(N, D):
    from xuance_b200.torch.utils.rollout_glue import gaussian_act
    from xuance_b200.torch.rl_models import DiagGaussianDistribution
    rng = np.random.default_rng(N * 1000 + D)
    mu = rng.uniform(-1.5, 1.5, (N, D)).astype(f32)
    ls = rng.uniform(-1.5, 1.0, D).astype(f32)
    noise = rng.normal(size=(N, D)).astype(f32)
    forced = (mu + np.exp(ls) * rng.normal(size=(N, D)) * 2).astype(f32)
    sig = np.exp(ls.astype(np.float64))[None, :]
    ent_tol = (D + 2) * EPS * (0.5 + gr.LOG_SQRT_2PI + np.abs(ls.astype(np.float64))).sum()   # summands: H may cancel

    def lp_tol(x):
        terms, z = gr.gauss_logp_terms(mu, ls, x)
        c = (np.abs(x) + np.abs(mu)) / sig + np.abs(z)
        mag = 0.5 * z * z + np.abs(ls.astype(np.float64))[None, :] + gr.LOG_SQRT_2PI
        return 4 * EPS * (np.abs(z) * c).sum(1) + (D + 2) * EPS * mag.sum(1)

    mu_d, ls_d = _t(mu), _t(ls)
    ent = torch.full((N,), float("nan"), device=DEV)
    # stochastic: a = mu + sigma * noise (one rounding each for exp, product and sum)
    out = gaussian_act(mu_d, ls_d, noise=_t(noise), entropy=ent)
    a = out["actions"].cpu().numpy()
    ref_a, ref_lp, ref_ent = gr.gaussian_act(mu, ls, noise=noise)
    _within(a, ref_a, 4 * EPS * (np.abs(mu) + sig * np.abs(noise)), f"N={N} D={D} stochastic actions")
    # the log-prob is of the float32 action the kernel wrote
    _within(out["logp"], gr.gaussian_act(mu, ls, forced=a)[1], lp_tol(a.astype(np.float64)), "stochastic logp")
    _within(ent, ref_ent, ent_tol, "entropy")
    # deterministic: a = mu exactly
    out = gaussian_act(mu_d, ls_d)
    assert np.array_equal(out["actions"].cpu().numpy(), mu)
    _, ref_lp, _ = gr.gaussian_act(mu, ls)
    _within(out["logp"], ref_lp, lp_tol(mu.astype(np.float64)), "deterministic logp")
    # forced: the log-prob of given actions; no action is written
    sentinel = _nan(N, D)
    lp = _nan(N)
    out = gaussian_act(mu_d, ls_d, noise=_t(noise), forced_actions=_t(forced), actions_f32=sentinel, logp=lp)
    assert torch.isnan(sentinel).all()
    _, ref_lp, _ = gr.gaussian_act(mu, ls, forced=forced)
    _within(lp, ref_lp, lp_tol(forced.astype(np.float64)), "forced logp")
    d = DiagGaussianDistribution(D)                                  # the host distribution, float32 torch on the CPU
    d.set_param(torch.from_numpy(mu), torch.from_numpy(ls).exp())
    host = d.log_prob(torch.from_numpy(forced)).numpy()
    _within(lp, host, 2 * lp_tol(forced.astype(np.float64)) + 2 * EPS * np.abs(host), "forced logp vs host")


# ====================================================================================================== learners
OBS, ACT_D, BATCH = 17, 6, 64


def _product_gauss_model(device=DEV):
    from xuance_b200.torch.rl_models import Basic_MLP, GaussianActorHead, ValueHead, SharedActorCritic
    act = nn.LeakyReLU
    rep = Basic_MLP((OBS,), [64], None, None, act, device)
    actor = GaussianActorHead(64, [64], ACT_D, None, None, act, nn.Tanh, device)
    critic = ValueHead(64, [64], None, None, act, device)
    return SharedActorCritic(rep, actor, critic)


def _pair(seed=17):
    from oracle_gauss import GaussianActorCriticOracle
    torch.backends.cuda.matmul.allow_tf32 = False
    oracle_model = GaussianActorCriticOracle(OBS, ACT_D)
    oracle_model.load_state_dict(seeded_state_dict(oracle_model.state_dict(), seed))
    model = _product_gauss_model()
    model.load_state_dict(oracle_model.state_dict())          # the reference's parameter names on both sides
    return oracle_model, model


@pytest.mark.parametrize("kind", ["ppo", "a2c", "pg"])
def test_gauss_learners_match_oracle(kind):
    """Three updates on identical inputs / initial weights, with the tolerances of test_ppo_learner_update_matches_oracle."""
    from xuance_b200.torch.learners import PPO_Learner, A2C_Learner, PG_Learner
    from xuance_b200.common import BaseCallback
    from oracle_gauss import PPOGaussLearnerOracle
    oracle_model, model = _pair()
    cfg = ppo_config(DEV, running_steps=256 * 128 * 10)
    learner = {"ppo": PPO_Learner, "a2c": A2C_Learner, "pg": PG_Learner}[kind](cfg, model, BaseCallback())
    orc = PPOGaussLearnerOracle(oracle_model, end_factor_lr_decay=0.5, kind=kind,
                                total_iters=cfg.running_steps if kind == "a2c" else learner.total_iters)
    rng = np.random.default_rng(5)
    for it in range(3):
        s = ppo_gauss_samples(rng, it, BATCH, OBS, ACT_D)
        io = orc.update(**s)
        ip = learner.update(**dict(s, obs=torch.from_numpy(s["obs"]).to(DEV)))
        if kind == "ppo":
            for k in ("actor_loss", "critic_loss", "entropy", "predict_value"):
                np.testing.assert_allclose(ip[k], io[k], rtol=2e-4, atol=1e-5, err_msg=k)
            np.testing.assert_allclose(ip["clip_ratio"], float(io["clip_ratio"]), atol=1.0 / BATCH + 1e-7)
        else:
            np.testing.assert_allclose(ip["actor-loss"], io["actor_loss"], rtol=2e-4, atol=1e-5)
            np.testing.assert_allclose(ip["entropy"], io["entropy"], rtol=2e-4)
        assert ip["learning_rate"] == io["learning_rate"]
    so, sp = oracle_model.state_dict(), model.state_dict()
    for k in so:
        np.testing.assert_allclose(sp[k].cpu().numpy(), so[k].numpy(), rtol=1e-3, atol=1e-4, err_msg=k)


def test_gauss_ppo_learner_matches_reference_fixture():
    """The product's PPO_Learner reproduces the unmodified reference's three updates (tests/golden/ppo_gauss_update.npz)."""
    from xuance_b200.torch.learners import PPO_Learner
    from xuance_b200.common import BaseCallback
    g = np.load(os.path.join(G, "ppo_gauss_update.npz"))
    _, model = _pair()
    learner = PPO_Learner(ppo_config(DEV, running_steps=4096 * 10, parallels=32), model, BaseCallback())
    assert learner.total_iters == int(g["total_iters"])
    rng = np.random.default_rng(23)
    for it in range(3):
        s = ppo_gauss_samples(rng, it, BATCH, OBS, ACT_D)
        info = learner.update(**s)
        got = [info["actor_loss"], info["critic_loss"], info["entropy"], info["learning_rate"], info["predict_value"]]
        np.testing.assert_allclose(got, g["infos"][it][:5], rtol=2e-4, atol=1e-5)
        np.testing.assert_allclose(info["clip_ratio"], g["infos"][it][5], atol=1.0 / BATCH + 1e-7)
    for k, v in model.state_dict().items():
        flat = v.detach().reshape(-1).cpu()
        np.testing.assert_allclose(flat[:64].numpy(), g[f"final_head/{k}"], rtol=1e-3, atol=1e-4, err_msg=k)
    np.testing.assert_allclose(model.actor.log_std.detach().cpu().numpy(), g["final/actor.log_std"], rtol=1e-3,
                               atol=1e-4)


def _box_agent_config(**kw):
    base = dict(agent="PPO", learner="PPO_Learner", representation="Basic_MLP", env_name="Classic Control",
                distributed_training=False, device=DEV, seed=3, parallels=8, running_steps=100000, horizon_size=32,
                n_epochs=2, n_minibatch=4, learning_rate=4e-4, vf_coef=0.25, ent_coef=0.01, clip_range=0.2, gamma=0.99,
                use_gae=True, gae_lambda=0.95, use_advnorm=True, use_grad_clip=True, grad_clip_norm=0.5,
                use_obsnorm=False, use_rewnorm=False, activation="leaky_relu", activation_action="tanh",
                representation_hidden_size=[64], actor_hidden_size=[64], critic_hidden_size=[64],
                model_dir="/tmp/xb_models/gauss", logger=None, episode_length=None)
    base.update(kw)
    return Namespace(**base)


def _fill_box(memory, rng, N, T, obs_dim, D):
    for t in range(T):
        memory.store(rng.normal(size=(N, obs_dim)).astype(np.float32), rng.normal(size=(N, D)).astype(np.float32),
                     rng.normal(size=N).astype(np.float32), rng.normal(size=N).astype(np.float32), rng.random(N) < 0.05,
                     {"old_logp": (rng.normal(size=N) * 0.3 - 5.0).astype(np.float32)})
    for i in range(N):
        memory.finish_path(0.3, i)


def test_gauss_train_epochs_cuda_graph_matches_eager():
    from xuance_b200.common import Box
    from xuance_b200.torch.agents import PPO_Agent
    torch.backends.cuda.matmul.allow_tf32 = False
    results = []
    for graph in (False, True):
        cfg = _box_agent_config(use_cuda_graph=graph)
        torch.manual_seed(0)
        agent = PPO_Agent(cfg, None, Box(-10, 10, (OBS,), np.float32), Box(-1, 1, (ACT_D,), np.float32))
        assert agent.learner._gaussian
        agent.model.load_state_dict(seeded_state_dict(agent.model.state_dict(), 4))
        _fill_box(agent.memory, np.random.default_rng(0), 8, 32, OBS, ACT_D)
        np.random.seed(11)
        agent.train_epochs(2)
        info = agent.train_epochs(2)          # second call replays the captured graphs
        results.append((info, {k: v.clone() for k, v in agent.model.state_dict().items()}))
    (i0, p0), (i1, p1) = results
    for k in ("actor_loss", "critic_loss", "entropy", "predict_value", "clip_ratio"):
        np.testing.assert_allclose(i1[k], i0[k], rtol=1e-5, atol=1e-6, err_msg=k)
    for k in p0:
        np.testing.assert_allclose(p1[k].cpu().numpy(), p0[k].cpu().numpy(), rtol=1e-5, atol=1e-6, err_msg=k)


def test_store_staged_equals_store_for_box_actions():
    from xuance_b200.common import DummyOnPolicyBuffer, Box
    rng = np.random.default_rng(0)
    N, T, D = 6, 9, 3
    space, aspace = Box(-10, 10, (5,), np.float32), Box(-2, 2, (D,), np.float32)
    a = DummyOnPolicyBuffer(space, aspace, {"old_logp": ()}, N, T, device=DEV)
    b = DummyOnPolicyBuffer(space, aspace, {"old_logp": ()}, N, T, device=DEV)
    slots = b.policy_slots()
    assert set(slots) == {"actions", "values", "aux:old_logp"} and tuple(slots["actions"].shape) == (N, D)
    for t in range(T + 3):      # wraps the ring
        obs = rng.normal(size=(N, 5)).astype(np.float32)
        acts, vals = rng.normal(size=(N, D)).astype(np.float32), rng.normal(size=N).astype(np.float32)
        logp, rews, terms = rng.normal(size=N).astype(np.float32), rng.normal(size=N).astype(np.float32), rng.random(N) < 0.3
        a.store(obs, acts, rews, vals, terms, {"old_logp": logp})
        slots["actions"].copy_(torch.from_numpy(acts))
        slots["values"].copy_(torch.from_numpy(vals))
        slots["aux:old_logp"].copy_(torch.from_numpy(logp))
        b.store_staged(torch.from_numpy(obs).to(DEV), rews, terms)
        assert a.ptr == b.ptr and a.size == b.size
    assert torch.equal(a.observations, b.observations)
    assert torch.equal(a._fields[:a._n_store], b._fields[:b._n_store])
    assert torch.equal(a.actions, b.actions)


def test_box_agent_model_and_limits():
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.agents import PPO_Agent
    from xuance_b200.torch.rl_models import GaussianActorHead, CategoricalActorHead
    agent = PPO_Agent(_box_agent_config(), None, Box(-10, 10, (OBS,), np.float32), Box(-1, 1, (ACT_D,), np.float32))
    assert isinstance(agent.model.actor, GaussianActorHead) and isinstance(agent.model.actor.mu[-1], nn.Tanh)
    assert "actor.log_std" in agent.model.state_dict() and "actor.mu.2.weight" in agent.model.state_dict()
    agent = PPO_Agent(_box_agent_config(), None, Box(-10, 10, (OBS,), np.float32), Discrete(3))
    assert isinstance(agent.model.actor, CategoricalActorHead) and not agent.learner._gaussian
    with pytest.raises(NotImplementedError, match="64"):
        PPO_Agent(_box_agent_config(), None, Box(-10, 10, (OBS,), np.float32), Box(-1, 1, (65,), np.float32))
    with pytest.raises(NotImplementedError):
        PPO_Agent(_box_agent_config(), None, Box(-10, 10, (OBS,), np.float32), Box(-1, 1, (2, 3), np.float32))


# ====================================================================================================== learning
# Pendulum-v1 with the reference's hyper-parameters (10 envs x 256 steps per rollout, 8 epochs x 8 minibatches), 122880
# training steps (48 rollouts).  Mean score of 10 stochastic test episodes before -> after training, on an H100 80GB HBM3
# at its 700 W limit (a random policy scores about -1200 to -1500):
#   seed 1: host -1469.6 -> -291.7 (+1178), device -1469.6 -> -485.8 (+984)     (the seed the test runs; 21 s / 14 s)
#   seed 2: host -1342.9 -> -305.4 (+1038), device -1342.9 -> -269.5 (+1073)
#   seed 3: host -1166.2 -> -577.1 (+589),  device -1166.2 -> -219.5 (+947)
# At 61440 steps the gains were only +240 to +484, hence the longer run.  The required gain, 300, is half the smallest.
PENDULUM_STEPS = 122880
PENDULUM_GAIN = 300.0


@pytest.mark.parametrize("device_rollout", [False, True])
def test_ppo_pendulum_learns(device_rollout):
    from xuance_b200 import get_runner
    runner = get_runner("ppo", "classic_control", "Pendulum-v1",
                        parser_args=Namespace(device=DEV, running_steps=PENDULUM_STEPS, device_rollout=device_rollout,
                                              model_dir="/tmp/xb_models/ppo_pendulum_%d" % device_rollout))
    agent = runner.agent
    assert agent.n_envs == 10 and agent.learner._gaussian
    before = float(np.mean(agent.test(test_episodes=10)))
    runner.run("train", running_steps=PENDULUM_STEPS)
    assert {"actor_loss", "critic_loss", "entropy", "clip_ratio"} <= set(agent.logged)
    after = float(np.mean(agent.test(test_episodes=10)))
    runner.finish()
    print("pendulum device_rollout=%s before %.1f after %.1f" % (device_rollout, before, after))
    assert after > before + PENDULUM_GAIN, (before, after)
