"""GPU tests of VDAC and IAC: K4V (xb_vdac_loss_fwd_bwd) against the float64 restatement over the B / T / n / A grid in
every mix mode and row order, shard sums and launch identity; the learners against the reference fixture
(tests/golden/vdac_update.npz) and the torch-CPU oracle, eager and as a CUDA graph; checkpoints; acting through K10; and
REGISTRY_Agents["VDAC"] (VDN and QMIX) and ["IAC"] learning on the 3m-shaped SyntheticSMACEnv."""
import os
import sys
from argparse import Namespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from vdac_refs import FIX_CASES, FIX_UPDATES, FIX_SNAPSHOTS, FIX_A, case_name, case_config, k4v_ref  # noqa: E402
from oracle_vdac import build_product_model, VDACLearnerOracle, fixture_batch  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vdac_update.npz")

# (B, T, n, A): every listed B, T, n and A occurs; sizes kept so the float64 restatement stays quick
SHAPES = [(1, 1, 1, 1), (2, 60, 3, 2), (31, 1, 5, 9), (32, 60, 8, 12), (33, 60, 5, 33), (1024, 1, 32, 64),
          (2, 1, 32, 9), (33, 1, 8, 64), (1024, 60, 3, 9), (31, 60, 1, 12), (1, 60, 32, 2), (32, 1, 3, 33)]


def _inputs(rng, B, T, n, A, masks, mode):
    R = B * n * T
    d = dict(logits=rng.normal(0, 2, (R, A)).astype(np.float32),
             actions=rng.integers(0, A, R).astype(np.float32),
             adv=rng.normal(0, 1, R).astype(np.float32),
             value=rng.normal(0, 1, B * T if mode == 2 else R).astype(np.float32),
             old_value=rng.normal(0, 1, R).astype(np.float32),
             ret=rng.normal(0, 2, R).astype(np.float32),
             mask=(rng.random(R) > 0.3).astype(np.float32) if masks else np.ones(R, np.float32),
             avail=None)
    if masks:
        av = (rng.random((R, A)) < 0.6).astype(np.uint8)
        av[np.arange(R), d["actions"].astype(int)] = 1
        d["avail"] = av
    return d


def _k4v(d, n, T, mode, row_order, vclip, hdelta, vf=0.5, ent=0.01, M=None, R_total=None, vn=None):
    """One K4V launch; returns (stats[8], dlogits, dvalue) on the host."""
    from xuance_b200 import _lib
    t = lambda x: None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(DEV)
    lg, av, act, adv, v, vo, ret, mk = (t(d[k]) for k in ("logits", "avail", "actions", "adv", "value", "old_value",
                                                          "ret", "mask"))
    R, A = lg.shape
    prep = torch.tensor([float(mk.sum().item()) if M is None else M, 0, 0, 0], dtype=torch.float64, device=DEV)
    vn_t = None if vn is None else torch.tensor(vn, dtype=torch.float32, device=DEV)
    dl, dv = torch.empty_like(lg), torch.empty_like(v)
    stats = torch.zeros(8, dtype=torch.float32, device=DEV)
    _lib.call("xb_vdac_loss_fwd_bwd", _lib.ptr(lg), _lib.ptr(av), 0 if av is None else A, _lib.ptr(act), _lib.ptr(adv),
              _lib.ptr(v), _lib.ptr(vo), _lib.ptr(ret), _lib.ptr(mk), _lib.ptr(vn_t), _lib.ptr(prep), R, A, n, T, mode,
              row_order, R if R_total is None else R_total, vclip, hdelta, vf, ent, _lib.ptr(dl), _lib.ptr(dv),
              _lib.ptr(stats), _lib.ptr(_lib.scratch(DEV)))
    return stats.cpu().numpy(), dl.cpu().numpy(), dv.cpu().numpy()


def _close(a, b, what, rtol=2e-5):
    scale = max(1.0, float(np.max(np.abs(b)))) if np.size(b) else 1.0
    np.testing.assert_allclose(a, b, rtol=rtol, atol=rtol * scale, err_msg=what)


@pytest.mark.parametrize("mode,row_order", [(0, 0), (1, 0), (1, 1), (2, 0), (2, 1)])
@pytest.mark.parametrize("masks", [False, True])
def test_k4v_matches_float64(mode, row_order, masks):
    rng = np.random.default_rng(100 + 10 * mode + row_order + 5 * masks)
    for j, (B, T, n, A) in enumerate(SHAPES):
        d = _inputs(rng, B, T, n, A, masks, mode)
        vclip, hdelta = (0.2, 1.0) if j % 2 else (0.0, 0.0)
        vn = (0.3, 1.7) if j % 3 == 0 else None
        st, dl, dv = _k4v(d, n, T, mode, row_order, vclip, hdelta, vn=vn)
        rs, rdl, rdv = k4v_ref(d["logits"], d["avail"], d["actions"], d["adv"], d["value"], d["old_value"], d["ret"],
                               d["mask"], vn, n, T, mode, row_order, vclip, hdelta, 0.5, 0.01)
        tag = f"B={B} T={T} n={n} A={A}"
        _close(st[:5], rs, "stats " + tag, rtol=1e-4)
        assert np.all(st[5:] == 0)
        _close(dl, rdl, "dlogits " + tag)
        _close(dv, rdv, "dvalue " + tag, rtol=1e-4)
        if masks:
            assert np.all(dl[d["avail"] == 0] == 0)


def test_k4v_ties_and_all_masked():
    """Huber at delta and the clip boundary ties, and a zero mask sum (NaN as in the reference)."""
    B, T, n, A = 2, 3, 2, 4
    R = B * n * T
    d = dict(logits=np.zeros((R, A), np.float32), actions=np.zeros(R, np.float32), adv=np.ones(R, np.float32),
             value=np.full(R, 1.0, np.float32), old_value=np.full(R, 1.0, np.float32),
             ret=np.full(R, 0.0, np.float32), mask=np.ones(R, np.float32), avail=None)
    st, dl, dv = _k4v(d, n, T, 0, 0, 0.2, 1.0)
    rs, rdl, rdv = k4v_ref(d["logits"], None, d["actions"], d["adv"], d["value"], d["old_value"], d["ret"], d["mask"],
                           None, n, T, 0, 0, 0.2, 1.0, 0.5, 0.01)
    _close(st[:5], rs, "tie stats")
    _close(dv, rdv, "tie dvalue")
    d["mask"][:] = 0
    st, dl, dv = _k4v(d, n, T, 1, 0, 0.0, 0.0)
    assert np.isnan(st[0]) and np.isnan(dl).all()


@pytest.mark.parametrize("G", [2, 3, 8])
@pytest.mark.parametrize("mode,row_order", [(0, 0), (1, 1), (2, 0)])
def test_k4v_shards_sum_to_the_unsharded_result(G, mode, row_order):
    rng = np.random.default_rng(7 + G)
    B, T, n, A = 24, 60, 3, 9
    d = _inputs(rng, B, T, n, A, True, mode)
    M = float(d["mask"].sum())
    full = _k4v(d, n, T, mode, row_order, 0.2, 1.0)
    stats = np.zeros(8)
    dls, dvs = [], []
    rows, vrows = n * T * (B // G), (T if mode == 2 else n * T) * (B // G)
    for s in range(G):
        sl = lambda x, w: x[s * w:(s + 1) * w]
        part = {k: (None if v is None else sl(v, vrows if k == "value" else rows)) for k, v in d.items()}
        st, dl, dv = _k4v(part, n, T, mode, row_order, 0.2, 1.0, M=M, R_total=B * n * T)
        stats += st
        dls.append(dl)
        dvs.append(dv)
    np.testing.assert_allclose(stats[:5], full[0][:5], rtol=1e-5, atol=1e-6)
    assert np.array_equal(np.concatenate(dls), full[1]) and np.array_equal(np.concatenate(dvs), full[2])


def test_k4v_is_bit_identical_across_launches():
    rng = np.random.default_rng(3)
    for mode, ro in ((0, 0), (1, 1), (2, 0)):
        d = _inputs(rng, 1024, 60, 3, 9, True, mode)
        a, b = _k4v(d, 3, 60, mode, ro, 0.2, 1.0), _k4v(d, 3, 60, mode, ro, 0.2, 1.0)
        for x, y in zip(a, b):
            assert np.array_equal(x, y)


def test_k4v_row_orders_differ_at_T_gt_1_and_agree_at_T_1():
    rng = np.random.default_rng(5)
    for T in (6, 1):
        d = _inputs(rng, 4, T, 3, 5, True, 1)
        a, b = _k4v(d, 3, T, 1, 0, 0.0, 0.0), _k4v(d, 3, T, 1, 1, 0.0, 0.0)
        same = np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2])
        assert same == (T == 1)


# ---------------------------------------------------------------- learners
def _stacked(g, pre, it, use_rnn):
    """A fixture sample in the device buffers' agent-major '_stacked' layout (row k*B + b)."""
    x = lambda f: torch.from_numpy(np.asarray(g[f"{pre}in{it}/{f}"])).to(DEV)
    obs = x("obs")
    B, n = obs.shape[:2]
    am = lambda t: t.transpose(0, 1).reshape(n * B, *t.shape[2:]).contiguous().float()
    st = {k: am(x(k)) for k in ("obs", "actions", "advantages", "values", "returns", "agent_mask")}
    st["avail_actions"] = x("avail_actions").transpose(0, 1).reshape(n * B, *obs.shape[2:-1], FIX_A).contiguous()
    state = x("state").float()
    st["state"] = state.unsqueeze(0).expand(n, *state.shape).reshape(n * B, *state.shape[1:]).contiguous()
    if use_rnn:
        st["filled"] = x("filled").float().unsqueeze(0).expand(n, B, -1).reshape(n * B, -1).contiguous()
    return {"_stacked": st, "batch_size": B}


def _learner(case, model, grouping, **over):
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import REGISTRY_Learners
    cfg = Namespace(**dict(case_config(case), device=DEV, **over))
    name = "IAC_Learner" if case[0] == "IAC" else "VDAC_Learner"
    return REGISTRY_Learners[name](cfg, grouping, model, BaseCallback())


def _fixture_model(g, case):
    pre = case_name(case) + "/"
    grouping, model = build_product_model(case, DEV)
    sd = {k[len(pre) + 5:]: torch.from_numpy(g[k]) for k in g.files if k.startswith(pre + "init/")}
    model.load_state_dict(sd, strict=True)
    return grouping, model


@pytest.fixture
def strict_fp32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


@pytest.mark.parametrize("case", FIX_CASES, ids=case_name)
@pytest.mark.parametrize("graph", [False, True])
def test_learner_matches_the_reference_fixture(case, graph, strict_fp32):
    from vdac_refs import info_keys
    g = np.load(GOLDEN)
    pre = case_name(case) + "/"
    grouping, model = _fixture_model(g, case)
    learner = _learner(case, model, grouping, use_cuda_graph=graph, vdac_rnn_reference_row_order=True)
    keys = [k[len(pre) + 5:] for k in g.files if k.startswith(pre + "init/")]
    for it in range(FIX_UPDATES):
        info = learner.update(_stacked(g, pre, it, case[1]))
        got = np.array([info[k] for k in info_keys(case[0])])
        np.testing.assert_allclose(got, g[pre + "infos"][it], rtol=2e-4, atol=2e-5, err_msg=f"{pre} update {it}")
        if it in FIX_SNAPSHOTS:
            sd = model.state_dict()
            flat = np.concatenate([sd[k].detach().cpu().numpy().reshape(-1) for k in keys])
            np.testing.assert_allclose(flat, g[pre + f"after{it}"], rtol=1e-4, atol=3e-5, err_msg=f"{pre} params {it}")


@pytest.mark.parametrize("case", [c for c in FIX_CASES if c[1]], ids=case_name)
def test_learner_aligned_row_order_matches_the_oracle(case, strict_fp32):
    """The default (aligned) pairing against the oracle's aligned variant on the fixture's samples."""
    g = np.load(GOLDEN)
    pre = case_name(case) + "/"
    grouping, model = _fixture_model(g, case)
    oracle = VDACLearnerOracle(model, case, row_order=False)
    learner = _learner(case, model, grouping)
    for it in range(FIX_UPDATES):
        info = learner.update(_stacked(g, pre, it, case[1]))
        oinfo = oracle.update(fixture_batch(g, pre, it, case[1]))
        for k in ("actor_loss", "critic_loss", "entropy", "predict_value"):
            np.testing.assert_allclose(info["shared/" + k], oinfo[k], rtol=2e-4, atol=2e-5, err_msg=k)
        np.testing.assert_allclose(info["gradient_norm"], oinfo["gradient_norm"], rtol=2e-4)
    osd = oracle.state_dict()
    for k, p in model.state_dict().items():
        np.testing.assert_allclose(p.cpu().numpy(), osd[k].numpy(), rtol=1e-4, atol=3e-5, err_msg=k)


@pytest.mark.parametrize("case", [FIX_CASES[0], FIX_CASES[1], FIX_CASES[2], FIX_CASES[4]], ids=case_name)
def test_learner_cuda_graph_matches_eager(case):
    g = np.load(GOLDEN)
    pre = case_name(case) + "/"
    outs = []
    for graph in (False, True):
        grouping, model = _fixture_model(g, case)
        learner = _learner(case, model, grouping, use_cuda_graph=graph, use_value_norm=True)
        infos = [learner.update(_stacked(g, pre, it, case[1])) for it in range(FIX_UPDATES)]
        outs.append(([p.detach().cpu().numpy() for p in model.parameters()], infos,
                     learner.value_normalizer["shared"].running_mean.item()))
    for a, b in zip(outs[0][0], outs[1][0]):
        assert np.array_equal(a, b)
    assert outs[0][1] == outs[1][1] and outs[0][2] == outs[1][2]


# ---------------------------------------------------------------- agents
def _cfg3m(algo, **over):
    from xuance_b200.common.common_tools import get_arguments
    cfg = get_arguments(algo, "sc2", "3m")
    for k, v in dict(device=DEV, vectorize="Dummy_StarCraft2", model_dir=f"/tmp/xb200_{algo}_models",
                     log_dir=f"/tmp/xb200_{algo}_logs").items():
        setattr(cfg, k, v)
    for k, v in over.items():
        setattr(cfg, k, v)
    return cfg


@pytest.mark.parametrize("algo,mixer", [("vdac", "VDN"), ("vdac", "QMIX"), ("iac", None)])
def test_learns_through_the_agent_registry(algo, mixer):
    """REGISTRY_Agents["VDAC"] / ["IAC"] from the shipped 3m configs on the cue-following SMAC-shaped env: the greedy
    team score rises above its untrained value; checkpoints round-trip."""
    from xuance_b200.environment import make_envs
    from xuance_b200.torch.agents import REGISTRY_Agents
    over = dict(parallels=8, buffer_size=32, n_epochs=5, running_steps=16000, episode_limit=20, p_death=0.02,
                learning_rate=2e-3, ent_coef=0.01)
    if mixer:
        over["mixer"] = mixer
    cfg = _cfg3m(algo, **over)
    envs = make_envs(cfg)
    agent = REGISTRY_Agents[cfg.agent](cfg, envs)
    assert agent.use_rnn and type(agent.memory).__name__ == "MARL_OnPolicyBuffer_RNN"
    # acting: K10 actions, values broadcast per env (V_tot for VDAC), one host read
    obs, _ = envs.reset()
    out = agent.get_actions(obs, state=envs.buf_state, avail_actions_list=envs.buf_avail_actions,
                            rnn_states_actor=agent.init_rnn_states(cfg.parallels)[0],
                            rnn_states_critic=agent.init_rnn_states(cfg.parallels)[1])
    for e, acts in enumerate(out.env_actions):
        for k, a in acts.items():
            assert envs.buf_avail_actions[e][k][a]
    if algo == "vdac":
        v = np.stack([out.values[k] for k in agent.agent_keys])
        assert np.all(v == v[:1])
    before = float(np.mean(agent.test(16, test_envs=make_envs(cfg))))
    agent.train(cfg.running_steps // cfg.parallels)
    info = agent.logged
    after = float(np.mean(agent.test(32, test_envs=make_envs(cfg))))
    print("%s %s learning: before %.3f after %.3f" % (algo, mixer, before, after))
    assert np.isfinite(info.get("loss", info.get("shared/total_loss", np.nan)))
    assert after > before + 1.0, (before, after)
    path = f"/tmp/xb200_{algo}_ckpt.pth"
    agent.save_model(os.path.basename(path), model_path=os.path.dirname(path))
    fresh = REGISTRY_Agents[cfg.agent](cfg, make_envs(cfg))
    fresh.load_model(path)
    for (n, p), (_, q) in zip(agent.model.state_dict().items(), fresh.model.state_dict().items()):
        assert torch.equal(p, q), n
    agent.finish()
    fresh.finish()
