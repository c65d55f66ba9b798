"""GPU tests of COMA: K4C's critic input bit for bit against the reference's assembly over the B / T / n / A grid, the loss
kernel against the float64 restatement from one row to more than 2048 * 256 rows, shard sums and launch identity, acting
against the reference fixture (tests/golden/coma_update.npz); the learner against the fixture and the torch-CPU oracle,
eager and as a CUDA graph with epsilon changing between replays; and REGISTRY_Agents["COMA"] learning on the 3m-shaped
SyntheticSMACEnv with a checkpoint round-trip."""
import os
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from coma_refs import (FIX_CASES, FIX_UPDATES, FIX_SNAPSHOTS, FIX_A, INFO_KEYS, case_name, case_config,  # noqa: E402
                       k4c_ref, critic_input_reference)
from oracle_coma import build_product_model, COMALearnerOracle, fixture_batch  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "coma_update.npz")


def _t(x):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


# ---------------------------------------------------------------- critic input
# (B, T, n, A): every listed B, T, n and A occurs, sized so the output stays below ~1 GB
CI_SHAPES = [(1, 1, 1, 1), (2, 60, 3, 2), (31, 1, 5, 9), (33, 60, 8, 12), (1024, 1, 32, 64), (2, 60, 32, 33),
             (1024, 60, 3, 9), (31, 60, 1, 64), (33, 1, 32, 2), (1, 60, 5, 33), (1024, 1, 8, 1), (2, 1, 1, 12)]


@pytest.mark.parametrize("B,T,n,A", CI_SHAPES)
def test_critic_input_is_bit_exact_against_the_reference_assembly(B, T, n, A):
    from xuance_b200.torch.rl_models.coma import critic_input
    rng = np.random.default_rng(B + 7 * T + 11 * n + 13 * A)
    S, F = 7, 16
    state = torch.from_numpy(rng.normal(size=(B, T, S)).astype(np.float32))
    feat = torch.from_numpy(rng.normal(size=(B, n, T, F)).astype(np.float32))
    acts = torch.from_numpy(rng.integers(0, A, (B, n, T)).astype(np.float32))
    ref = critic_input_reference(state, feat, acts, A).reshape(B * n * T, -1)
    got = critic_input(state.to(DEV), feat.reshape(-1, F).to(DEV), acts.to(DEV), n, A).cpu()
    assert got.shape == ref.shape and torch.equal(got, ref)


def test_critic_input_backward_is_the_feature_slice():
    from xuance_b200.torch.rl_models.coma import critic_input
    B, T, n, A, S, F = 3, 4, 3, 5, 6, 8
    feat = torch.randn(B * n * T, F, device=DEV, requires_grad=True)
    out = critic_input(torch.randn(B, T, S, device=DEV), feat, torch.zeros(B, n, T, device=DEV), n, A)
    g = torch.randn_like(out)
    out.backward(g)
    assert torch.equal(feat.grad, g[:, S:S + F])


# ---------------------------------------------------------------- the loss kernel
def _inputs(rng, R, A, masks):
    acts = rng.integers(0, A, R)
    d = dict(logits=rng.normal(0, 2, (R, A)).astype(np.float32), q=rng.normal(0, 1, (R, A)).astype(np.float32),
             actions=acts.astype(np.float32), ret=rng.normal(0, 2, R).astype(np.float32),
             mask=(rng.random(R) > 0.3).astype(np.float32), avail=None)
    if masks:
        av = (rng.random((R, A)) < 0.6).astype(np.uint8)
        av[np.arange(R), acts] = 1
        d["avail"] = av
    return d


def _k4c(d, eps, M=None, R_total=None):
    """One K4C loss launch; returns (stats[8], dlogits, dq) on the host."""
    from xuance_b200 import _lib
    lg, av, q, act, ret, mk = (_t(d[k]) for k in ("logits", "avail", "q", "actions", "ret", "mask"))
    R, A = lg.shape
    prep = torch.tensor([float(mk.sum().item()) if M is None else M, 0, 0, 0], dtype=torch.float64, device=DEV)
    e = torch.tensor([eps], dtype=torch.float32, device=DEV)
    dl, dq = torch.empty_like(lg), torch.empty_like(q)
    stats = torch.full((8,), 7.0, dtype=torch.float32, device=DEV)
    _lib.call("xb_coma_loss_fwd_bwd", _lib.ptr(lg), _lib.ptr(av), 0 if av is None else A, _lib.ptr(q), _lib.ptr(act),
              _lib.ptr(ret), _lib.ptr(mk), _lib.ptr(e), _lib.ptr(prep), R, A, R if R_total is None else R_total,
              _lib.ptr(dl), _lib.ptr(dq), _lib.ptr(stats), _lib.ptr(_lib.scratch(DEV)))
    return stats.cpu().numpy(), dl.cpu().numpy(), dq.cpu().numpy()


# Tolerances: the kernel works in float32 (softmax, the mix, the renormalisation, an A-term baseline) and sums the
# statistics in float64.  Each gradient entry is a product of O(1) float32 factors with the weight mask / M, so its error
# is a few ulp of the largest entry of its array: atol = 2e-5 * max |ref|.  The advantage subtracts an A-term float32
# baseline from Q[a] (cancellation), so the statistics get rtol 1e-4 and atol 1e-4 * their scale.
def _close(a, b, what, rtol=2e-5):
    scale = max(1e-30, float(np.max(np.abs(b)))) if np.size(b) else 1.0
    np.testing.assert_allclose(a, b, rtol=rtol, atol=rtol * scale, err_msg=what)


@pytest.mark.parametrize("R,A", [(1, 1), (255, 12), (256, 9), (257, 64), (2048 * 256 + 1000, 12)])
@pytest.mark.parametrize("eps", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("masks", [False, True])
def test_loss_kernel_matches_float64(R, A, eps, masks):
    rng = np.random.default_rng(R + A + int(10 * eps) + 3 * masks)
    d = _inputs(rng, R, A, masks)
    st, dl, dq = _k4c(d, eps)
    rs, rdl, rdq = k4c_ref(d["logits"], d["avail"], d["q"], d["actions"], d["ret"], d["mask"], eps)
    tag = f"R={R} A={A} eps={eps} masks={masks}"
    np.testing.assert_allclose(st[:3], rs, rtol=1e-4, atol=1e-4 * max(1.0, float(np.abs(rs).max())),
                               err_msg="stats " + tag)
    assert np.all(st[3:] == 0)
    _close(dl, rdl, "dlogits " + tag)
    _close(dq, rdq, "dq " + tag)
    assert np.count_nonzero(dq, axis=1).max() <= 1
    if masks:
        assert np.all(dl[d["avail"] == 0] == 0)


def test_loss_kernel_edge_rows():
    """M = 0 gives NaN; a zero-probability taken action gives -inf / NaN in its row only, 0 at unavailable entries."""
    d = _inputs(np.random.default_rng(1), 6, 5, True)
    d["mask"][:] = 0
    st, dl, dq = _k4c(d, 0.3)
    assert np.isnan(st[0]) and np.isnan(st[1])
    d = _inputs(np.random.default_rng(2), 6, 5, True)
    a0 = int(d["actions"][0])
    d["avail"][0] = 1
    d["avail"][0, a0] = 0
    st, dl, dq = _k4c(d, 0.3)
    rs, rdl, rdq = k4c_ref(d["logits"], d["avail"], d["q"], d["actions"], d["ret"], d["mask"], 0.3)
    assert np.isnan(dl[0][d["avail"][0] != 0]).all() and np.all(dl[0][d["avail"][0] == 0] == 0)
    assert not np.isfinite(st[0]) and not np.isfinite(rs[0])
    _close(dl[1:], rdl[1:], "finite rows")


@pytest.mark.parametrize("G", [2, 3, 8])
def test_loss_kernel_shards_sum_to_the_unsharded_result(G):
    rng = np.random.default_rng(7 + G)
    R, A = 24 * 300, 12
    d = _inputs(rng, R, A, True)
    M = float(d["mask"].sum())
    full = _k4c(d, 0.3)
    stats, dls, dqs = np.zeros(8), [], []
    w = R // G
    for s in range(G):
        part = {k: (None if v is None else v[s * w:(s + 1) * w]) for k, v in d.items()}
        st, dl, dq = _k4c(part, 0.3, M=M, R_total=R)
        stats += st
        dls.append(dl)
        dqs.append(dq)
    np.testing.assert_allclose(stats[:3], full[0][:3], rtol=1e-5, atol=1e-6)
    assert np.array_equal(np.concatenate(dls), full[1]) and np.array_equal(np.concatenate(dqs), full[2])


def test_loss_kernel_is_bit_identical_across_launches():
    d = _inputs(np.random.default_rng(3), 2048 * 256 + 1000, 12, True)
    a, b = _k4c(d, 0.3), _k4c(d, 0.3)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


# ---------------------------------------------------------------- fixture helpers
def _load(g, pre, model, which):
    """The fixture's initial ("init") or final (the last snapshot) reference weights into the product model."""
    keys = [k[len(pre) + 5:] for k in g.files if k.startswith(pre + "init/")]
    if which == "init":
        sd = {k: torch.from_numpy(g[pre + "init/" + k]) for k in keys}
    else:
        flat, sd, o = g[pre + f"after{FIX_SNAPSHOTS[-1]}"], {}, 0
        for k in keys:
            shp = g[pre + "init/" + k].shape
            sd[k] = torch.from_numpy(flat[o:o + int(np.prod(shp))].reshape(shp).copy())
            o += int(np.prod(shp))
    model.load_state_dict(sd, strict=True)
    return keys


def _fixture_model(g, case, which="init"):
    grouping, model = build_product_model(case, DEV)
    _load(g, case_name(case) + "/", model, which)
    return grouping, model


def _stacked(g, pre, it):
    """A fixture sample in the device buffers' agent-major '_stacked' layout (row k*B + b)."""
    x = lambda f: torch.from_numpy(np.asarray(g[f"{pre}in{it}/{f}"])).to(DEV)
    obs = x("obs")
    B, n = obs.shape[:2]
    am = lambda t: t.transpose(0, 1).reshape(n * B, *t.shape[2:]).contiguous().float()
    st = {k: am(x(k)) for k in ("obs", "actions", "returns", "agent_mask")}
    T = obs.shape[2]
    st["advantages"] = torch.zeros(n * B, T, device=DEV)
    st["values"] = torch.zeros(n * B, T, device=DEV)
    st["avail_actions"] = x("avail_actions").transpose(0, 1).reshape(n * B, T, FIX_A).contiguous()
    state = x("state").float()
    st["state"] = state.unsqueeze(0).expand(n, *state.shape).reshape(n * B, *state.shape[1:]).contiguous()
    st["filled"] = x("filled").float().unsqueeze(0).expand(n, B, -1).reshape(n * B, -1).contiguous()
    return {"_stacked": st, "batch_size": B}


def _learner(case, model, grouping, **over):
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import REGISTRY_Learners
    cfg = Namespace(**dict(case_config(case), device=DEV, **over))
    return REGISTRY_Learners["COMA_Learner"](cfg, grouping, model, BaseCallback())


@pytest.fixture
def strict_fp32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


# ---------------------------------------------------------------- acting
@pytest.mark.parametrize("case", FIX_CASES, ids=case_name)
def test_act_matches_the_reference_fixture(case, strict_fp32):
    """xb_coma_act on the product actor (final fixture weights) against the reference's acting on the fixture's last
    sample: the arg-max actions, log pi of the mixed distribution and the target critics' Q of those actions; and the
    inverse-CDF draw on seeded uniforms against the same draw on the reference's probabilities."""
    from xuance_b200 import _lib
    g = np.load(GOLDEN)
    pre = case_name(case) + "/"
    n, masks, eps = case
    _, model = _fixture_model(g, case, "final")
    b = fixture_batch(g, pre, FIX_UPDATES - 1)
    probs = g[pre + "act/probs"].astype(np.float64)
    with torch.no_grad():
        logits = model.logits(b["obs"].to(DEV)).reshape(-1, FIX_A).contiguous()
        R = logits.shape[0]
        av = b["avail"].to(DEV).to(torch.uint8).contiguous() if masks else None
        e = torch.tensor([eps], dtype=torch.float32, device=DEV)
        u = torch.from_numpy(np.random.default_rng(5).random(R).astype(np.float32)).to(DEV)
        outs = []
        for uu in (None, u):
            af, ai, lp = (torch.empty(R, device=DEV), torch.empty(R, dtype=torch.int32, device=DEV),
                          torch.empty(R, device=DEV))
            _lib.call("xb_coma_act", _lib.ptr(logits), _lib.ptr(av), 0 if av is None else FIX_A, _lib.ptr(e),
                      _lib.ptr(uu), R, FIX_A, _lib.ptr(af), _lib.ptr(ai), _lib.ptr(lp))
            outs.append((af, ai.cpu().numpy(), lp.cpu().numpy()))
        af, ai, lp = outs[0]
        assert np.array_equal(ai, g[pre + "act/actions"].astype(np.int64))
        assert np.array_equal(af.cpu().numpy(), g[pre + "act/actions"])
        np.testing.assert_allclose(lp, np.log(probs[np.arange(R), ai]), rtol=1e-5, atol=1e-5)
        q = model.q_values(b["state"].to(DEV), b["obs"].to(DEV), af.reshape(b["B"], n, b["T"]), target=True)
        qa = q.gather(1, torch.from_numpy(ai).long().to(DEV).unsqueeze(1)).squeeze(1).cpu().numpy()
        np.testing.assert_allclose(qa, g[pre + "act/q_taken"], rtol=1e-4, atol=1e-5)
        # the draw: inverse CDF over the reference's probabilities; a disagreement may only sit on a CDF boundary
        cdf = np.cumsum(probs, 1)
        un = u.cpu().numpy().astype(np.float64)
        want = np.minimum((un[:, None] >= cdf).sum(1), FIX_A - 1)
        got = outs[1][1]
        near = np.abs(cdf - un[:, None]).min(1) < 1e-5
        assert np.all((got == want) | near)
        if eps > 0 and masks:
            assert (probs[b["avail"].numpy() == 0] > 0).all()      # the mix gives unavailable actions eps / A


# ---------------------------------------------------------------- learner
@pytest.mark.parametrize("case", FIX_CASES, ids=case_name)
@pytest.mark.parametrize("graph", [False, True])
def test_learner_matches_the_reference_fixture(case, graph, strict_fp32):
    g = np.load(GOLDEN)
    pre = case_name(case) + "/"
    grouping, model = _fixture_model(g, case)
    learner = _learner(case, model, grouping, use_cuda_graph=graph)
    keys = [k[len(pre) + 5:] for k in g.files if k.startswith(pre + "init/")]
    for it in range(FIX_UPDATES):
        info = learner.update(_stacked(g, pre, it), case[2])
        got = np.array([info[k] for k in INFO_KEYS])
        np.testing.assert_allclose(got, g[pre + "infos"][it], rtol=2e-4, atol=2e-5, err_msg=f"{pre} update {it}")
        if it in FIX_SNAPSHOTS:
            sd = model.state_dict()
            flat = np.concatenate([sd[k].detach().cpu().numpy().reshape(-1) for k in keys])
            np.testing.assert_allclose(flat, g[pre + f"after{it}"], rtol=1e-4, atol=3e-5, err_msg=f"{pre} params {it}")


EPS_SCHEDULE = (0.5, 0.3, 0.1, 0.0)


@pytest.mark.parametrize("case", [FIX_CASES[0], FIX_CASES[1]], ids=case_name)
def test_learner_graph_follows_a_changing_epsilon_and_equals_eager(case, strict_fp32):
    """Graphed replays read epsilon from the device: with epsilon changing on every update the graphed learner equals
    the eager one bit for bit, and both follow the oracle."""
    g = np.load(GOLDEN)
    pre = case_name(case) + "/"
    outs = []
    for graph in (False, True):
        grouping, model = _fixture_model(g, case)
        learner = _learner(case, model, grouping, use_cuda_graph=graph)
        infos = [learner.update(_stacked(g, pre, it), EPS_SCHEDULE[it]) for it in range(FIX_UPDATES)]
        outs.append(([p.detach().cpu().numpy() for p in model.parameters()], infos, model.state_dict()))
    for a, b in zip(outs[0][0], outs[1][0]):
        assert np.array_equal(a, b)
    assert outs[0][1] == outs[1][1]
    _, model = _fixture_model(g, case)
    oracle = COMALearnerOracle(model, case)
    for it in range(FIX_UPDATES):
        oinfo = oracle.update(fixture_batch(g, pre, it), EPS_SCHEDULE[it])
        for k in INFO_KEYS:
            np.testing.assert_allclose(outs[1][1][it][k], oinfo[k], rtol=2e-4, atol=2e-5, err_msg=f"{k} {it}")
    osd = oracle.state_dict()
    for k, p in outs[1][2].items():
        np.testing.assert_allclose(p.cpu().numpy(), osd[k].numpy(), rtol=1e-4, atol=3e-5, err_msg=k)


# ---------------------------------------------------------------- agent
def test_learns_through_the_agent_registry():
    """REGISTRY_Agents["COMA"] from the shipped 3m config on the cue-following SMAC-shaped env: the greedy team score
    rises above its untrained value by a fixed margin; checkpoints round-trip."""
    from xuance_b200.common.common_tools import get_arguments
    from xuance_b200.environment import make_envs
    from xuance_b200.torch.agents import REGISTRY_Agents
    cfg = get_arguments("coma", "sc2", "3m")
    for k, v in dict(device=DEV, vectorize="Dummy_StarCraft2", model_dir="/tmp/xb200_coma_models",
                     log_dir="/tmp/xb200_coma_logs", parallels=8, buffer_size=16, n_epochs=5, running_steps=24000,
                     episode_limit=20, p_death=0.02, learning_rate_actor=2e-3, learning_rate_critic=2e-3,
                     sync_frequency=10, decay_step_greedy=12000).items():
        setattr(cfg, k, v)
    envs = make_envs(cfg)
    agent = REGISTRY_Agents[cfg.agent](cfg, envs)
    assert agent.use_rnn and type(agent.memory).__name__ == "MARL_OnPolicyBuffer_RNN"
    obs, _ = envs.reset()
    ha, hc = agent.init_rnn_states(cfg.parallels)
    out = agent.get_actions(obs, state=envs.buf_state, avail_actions_list=envs.buf_avail_actions, rnn_states_actor=ha,
                            rnn_states_critic=hc)
    assert len(out.env_actions) == cfg.parallels and all(np.isfinite(v).all() for v in out.values.values())
    before = float(np.mean(agent.test(16, test_envs=make_envs(cfg))))
    agent.train(cfg.running_steps // cfg.parallels)
    info = agent.logged
    after = float(np.mean(agent.test(32, test_envs=make_envs(cfg))))
    print("coma learning: before %.3f after %.3f epsilon %.3f" % (before, after, agent.egreedy))
    assert np.isfinite(info["actor_loss"]) and np.isfinite(info["critic_loss"])
    assert after > before + 1.0, (before, after)
    path = "/tmp/xb200_coma_ckpt.pth"
    agent.save_model(os.path.basename(path), model_path=os.path.dirname(path))
    fresh = REGISTRY_Agents[cfg.agent](cfg, make_envs(cfg))
    fresh.load_model(path)
    for (n, p), (_, q) in zip(agent.model.state_dict().items(), fresh.model.state_dict().items()):
        assert torch.equal(p, q), n
    agent.finish()
    fresh.finish()
