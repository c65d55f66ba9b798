"""GPU tests of IQL: K9I against the restatement (tests/iql_refs.py) - the greedy next actions, next values and targets
bit for bit against the float32 reference expression, dq and the statistics within stated tolerances of float64 - over the
B / T / n / A / mask grid; shards and launch-to-launch identity; IQL_Learner against the reference fixture and the
torch-CPU float64 oracle (tests/oracle_iql.py), eager and graphed; graphed equals eager; checkpoints of the learner and
of the replay; and learning through REGISTRY_Agents."""
from argparse import Namespace

import numpy as np
import pytest
import torch

import iql_refs as R
import test_iql as TI
from oracle_iql import IQLOracle, build_model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _lib():
    from xuance_b200 import _lib as L
    return L


def _run_k9i(x, double_q, gamma=0.99, msum=None, rows_total=None, extras=True):
    """One xb_iql_prepare (unless msum is given) + xb_iql_td_fwd_bwd on CPU inputs x; returns CPU outputs."""
    L = _lib()
    d = {k: (None if v is None else v.to(DEV).contiguous()) for k, v in x.items()}
    B, n, T1, A = d["q_all"].shape
    T = T1 - 1
    scratch = L.scratch(DEV)
    if msum is None:
        msum = torch.zeros(1, dtype=torch.float64, device=DEV)
        L.call("xb_iql_prepare", L.ptr(d["agent_mask"]), L.ptr(d["filled"]), B, n, T, L.ptr(msum), L.ptr(scratch))
    else:
        msum = torch.tensor([float(msum)], dtype=torch.float64, device=DEV)
    dq = torch.full_like(d["q_all"], 7.0)                   # every element must be written
    stats = torch.zeros(2, device=DEV)
    nxt = torch.empty((B, n, T), dtype=torch.int32, device=DEV) if extras else None
    qn = torch.empty((B, n, T), device=DEV) if extras else None
    y = torch.empty((B, n, T), device=DEV) if extras else None
    av = d["avail"]
    L.call("xb_iql_td_fwd_bwd", L.ptr(d["q_all"]), L.ptr(d["q_tgt"]), L.ptr(d["actions"]), L.ptr(d["rewards"]),
           L.ptr(d["terminals"]), L.ptr(d["agent_mask"]), L.ptr(d["filled"]), L.ptr(av),
           av.shape[3] if av is not None else 0, L.ptr(msum), B, n, T, A, int(double_q), gamma,
           rows_total if rows_total is not None else B * n * T, L.ptr(dq), L.ptr(stats), L.ptr(scratch), L.ptr(nxt),
           L.ptr(qn), L.ptr(y))
    out = dict(msum=msum.item(), dq=dq.cpu(), stats=stats.cpu())
    if extras:
        out.update(next=nxt.cpu(), q_next=qn.cpu(), y=y.cpu())
    return out


def _check_against_reference(x, double_q, got, gamma=0.99):
    args = (x["q_all"], x["q_tgt"], x["actions"], x["rewards"], x["terminals"], x["agent_mask"], x["filled"],
            x["avail"], double_q, gamma)
    # float32: the reference expression itself -> bit for bit
    _, _, nxt32, qn32, y32, m32 = R.forward(*args)
    assert torch.equal(got["next"].long(), nxt32)
    assert torch.equal(got["q_next"].reshape(-1), qn32)
    assert torch.equal(got["y"].reshape(-1), y32)
    # float64 from the (bit-exact) float32 targets: dq and the statistics
    A = x["q_all"].shape[-1]
    m = m32.double()
    M = m.sum().item()
    assert got["msum"] == M
    q = x["q_all"][:, :, :-1].double().reshape(-1, A)
    a = x["actions"].long().reshape(-1)
    qe = q.gather(-1, a.unsqueeze(-1)).reshape(-1)
    td = (qe - y32.double()) * m
    want = torch.zeros_like(x["q_all"], dtype=torch.float64)
    g = torch.zeros_like(q)
    g.scatter_(-1, a.unsqueeze(-1), (2 * td * m / M).unsqueeze(-1))
    want[:, :, :-1] = g.reshape(want[:, :, :-1].shape)
    scale = max(torch.nan_to_num(want).abs().max().item(), 1e-30)
    np.testing.assert_allclose(got["dq"].double().numpy(), want.numpy(), rtol=2e-6, atol=1e-6 * scale)
    assert not got["dq"][:, :, -1].any()
    loss = (td ** 2).sum().item() / M if M else float("nan")              # M = 0: 0/0, as the reference
    np.testing.assert_allclose(got["stats"].double().numpy(), [loss, qe.mean().item()], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("n,A", [(n, A) for n in (1, 3, 5, 8, 32) for A in (1, 2, 9, 12, 33, 64)])
def test_k9i_matches_the_reference(n, A):
    rng = np.random.default_rng(n * 100 + A)
    done = 0
    for B in (1, 2, 31, 32, 33, 1024):
        for T in (1, 60):
            if B * n * (T + 1) * A > 4_000_000:
                continue
            for masked in (False, True):
                x = R.inputs(rng, B, n, T, A, masked=masked, quantum=4.0)        # coarse grid: many ties
                if masked and (B + T) % 2:                                        # a wider mask row: avail_ld > A
                    x["avail"] = torch.cat([x["avail"], torch.ones(B, n, T + 1, 3, dtype=torch.uint8)], -1)
                for double_q in (True, False):
                    _check_against_reference(x, double_q, _run_k9i(x, double_q), gamma=0.99)
                    done += 1
    assert done >= 8


def test_k9i_edge_rows():
    """An all-unavailable next row (target -1e10), d = 1, an empty mask (M = 0: NaN loss and gradient), A = 1."""
    rng = np.random.default_rng(3)
    x = R.inputs(rng, 2, 3, 5, 4, masked=True)
    x["avail"][0, 1, 3] = 0
    x["terminals"][1] = 1.0
    for double_q in (True, False):
        got = _run_k9i(x, double_q)
        _check_against_reference(x, double_q, got)
        assert got["q_next"][0, 1, 2].item() == -1e10
    x["agent_mask"].zero_()
    got = _run_k9i(x, True)
    assert np.isnan(got["stats"][0].item()) and np.isfinite(got["stats"][1].item())
    assert got["msum"] == 0.0
    x = R.inputs(rng, 3, 1, 4, 1, masked=False)
    _check_against_reference(x, False, _run_k9i(x, False))


@pytest.mark.parametrize("G", [2, 3, 8])
def test_k9i_shards_match_the_whole_batch(G):
    """With the global M and rows_total, each shard's dq is bit-equal to its slice of the whole-batch launch and the
    shards' statistics sum to the whole."""
    rng = np.random.default_rng(G)
    B, n, T, A = 24, 5, 12, 12
    x = R.inputs(rng, B, n, T, A, masked=True)
    whole = _run_k9i(x, True, extras=False)
    stats = torch.zeros(2, dtype=torch.float64)
    for s in range(G):
        lo, hi = s * B // G, (s + 1) * B // G
        part = {k: (None if v is None else v[lo:hi]) for k, v in x.items()}
        got = _run_k9i(part, True, msum=whole["msum"], rows_total=B * n * T, extras=False)
        assert torch.equal(got["dq"], whole["dq"][lo:hi])
        stats += got["stats"].double()
    np.testing.assert_allclose(stats.numpy(), whole["stats"].double().numpy(), rtol=1e-6, atol=1e-7)


def test_k9i_is_bit_identical_across_launches():
    x = R.inputs(np.random.default_rng(11), 64, 8, 60, 33, masked=True)
    a, b = _run_k9i(x, True), _run_k9i(x, True)
    for k in ("dq", "stats", "next", "q_next", "y"):
        assert torch.equal(a[k], b[k]), k
    assert a["msum"] == b["msum"]


# ---------------------------------------------------------------- learner
def _learner(grouping, model, **over):
    from xuance_b200.common import BaseCallback
    from xuance_b200.torch.learners import IQL_Learner
    cfg = dict(device=DEV, model_dir="/tmp/xb200_iql_models", use_cuda_graph=False, use_grad_clip=False,
               grad_clip_norm=0.5, parallels=4, running_steps=100000, start_training=0, use_rnn=True,
               use_actions_mask=True, learning_rate=7e-4, sync_frequency=2, gamma=0.99, end_factor_lr_decay=0.5,
               use_linear_lr_decay=True, agent="IQL", double_q=True, episode_length=8)
    cfg.update(over)
    return IQL_Learner(Namespace(**cfg), grouping, model, BaseCallback())


def _sample(rng, keys, B, T, obs_dim, A):
    from wqmix_refs import fix_sample
    return fix_sample(rng, keys, B=B, T=T, obs_dim=obs_dim, A=A, S=4)


INFO = ("loss_Q", "predictQ")


def _run(double_q, use_graph, updates=3, seed=0, clip=False):
    _no_tf32()
    torch.manual_seed(seed)
    n, obs_dim, A, T, B, hid = 4, 20, 7, 12, 6, 32
    keys, grouping, model = build_model(n, obs_dim, A, hid, DEV)
    lrn = _learner(grouping, model, double_q=double_q, use_cuda_graph=use_graph, episode_length=T,
                   use_grad_clip=clip)
    rng = np.random.default_rng(seed + 1)
    out = []
    for _ in range(updates):
        s = _sample(rng, keys, B, T, obs_dim, A)
        want = IQLOracle(model, double_q=double_q).losses(s)
        out.append((lrn.update(s), want))
    return model, lrn, out


@pytest.mark.parametrize("double_q", [True, False])
@pytest.mark.parametrize("use_graph", [False, True])
def test_learner_matches_the_oracle(double_q, use_graph):
    """Every update's statistics against the float64 oracle on the same parameters (within 1e-4 relative)."""
    _, _, out = _run(double_q, use_graph)
    for it, (info, want) in enumerate(out):
        assert set(info) >= {"shared/learning_rate", "shared/loss_Q", "shared/predictQ"}
        np.testing.assert_allclose([info[f"shared/{k}"] for k in INFO], want, rtol=1e-4, atol=1e-6, err_msg=f"it{it}")


def test_learner_gradient_matches_the_oracle():
    """The gradient of one update, read from the optimiser's flat bucket before the step, against the oracle's."""
    _no_tf32()
    torch.manual_seed(2)
    n, obs_dim, A, T, B = 3, 12, 6, 9, 5
    keys, grouping, model = build_model(n, obs_dim, A, 32, DEV)
    lrn = _learner(grouping, model, episode_length=T)
    s = _sample(np.random.default_rng(5), keys, B, T, obs_dim, A)
    want = IQLOracle(model).grads(s)
    d = lrn._stacked(s)
    lrn.optimizer.prepare()
    lrn.optimizer.zero_grad()
    args = [d[k] for k in ("obs", "actions", "rewards", "terminals", "agent_mask", "filled", "state")] + [d["avail"]]
    orig = lrn.optimizer.launch
    lrn.optimizer.launch = lambda **kw: None                     # keep the gradient, skip the step
    try:
        lrn._device_update(*args)
    finally:
        lrn.optimizer.launch = orig
    names = {id(p): k for k, p in model.named_parameters()}
    for p in model.parameters_model:
        w = want[names[id(p)]].numpy()
        g = p.grad.detach().cpu().double().numpy()
        np.testing.assert_allclose(g, w, rtol=0, atol=1e-4 * max(np.abs(w).max(), 1e-3), err_msg=names[id(p)])


def test_graphed_update_is_bit_equal_to_eager():
    m_e, _, o_e = _run(False, False, updates=3, seed=4, clip=True)
    m_g, _, o_g = _run(False, True, updates=3, seed=4, clip=True)
    for (a, _), (b, _) in zip(o_e, o_g):
        assert a == b
    for (k, v), (_, w) in zip(m_e.state_dict().items(), m_g.state_dict().items()):
        assert torch.equal(v, w), k


@pytest.mark.parametrize("n,double_q,mask", TI.FIX_CASES)
@pytest.mark.parametrize("use_graph", [False, True])
def test_learner_reproduces_the_reference_fixture(n, double_q, mask, use_graph):
    """A reference state_dict loads strictly; every update's logged values within 1e-4 relative of the reference and
    the whole state_dict after every update within 2e-5 + 1e-4 relative."""
    _no_tf32()
    d = np.load(TI.GOLDEN)
    pre = TI.case_name(n, double_q, mask)
    keys, grouping, model = build_model(n, TI.FIX_OBS, TI.FIX_A, TI.FIX_HID, DEV)
    model.load_state_dict(TI.fixture_init(d, pre), strict=True)
    lrn = _learner(grouping, model, double_q=double_q, use_actions_mask=mask, use_cuda_graph=use_graph,
                   episode_length=TI.FIX_T)
    assert lrn.total_iters == int(d[pre + "total_iters"])
    for it in range(TI.FIX_UPDATES):
        info = lrn.update(TI.fixture_sample(d, pre, it, keys))
        np.testing.assert_allclose([info[f"shared/{k}"] for k in TI.FIX_INFO_KEYS], d[pre + "infos"][it], rtol=1e-4,
                                   atol=1e-6, err_msg=f"{pre}it{it}")
        flat = np.concatenate([v.cpu().numpy().reshape(-1) for v in model.state_dict().values()])
        np.testing.assert_allclose(flat, d[f"{pre}after{it}"], rtol=1e-4, atol=2e-5, err_msg=f"{pre}after{it}")


def test_learner_checkpoint_round_trip(tmp_path):
    _no_tf32()
    torch.manual_seed(1)
    rng = np.random.default_rng(1)
    keys, grouping, model = build_model(3, 12, 7, 32, DEV)
    lrn = _learner(grouping, model, end_factor_lr_decay=1.0)
    samples = [_sample(rng, keys, 6, 8, 12, 7) for _ in range(3)]
    for s in samples[:2]:
        lrn.update(s)
    path = str(tmp_path / "iql.pth")
    lrn.save_model(path)
    _, grouping2, model2 = build_model(3, 12, 7, 32, DEV)
    lrn2 = _learner(grouping2, model2, end_factor_lr_decay=1.0)
    lrn2.load_model(path)
    lrn2.iterations = lrn.iterations
    for (k, v), (_, w) in zip(model.state_dict().items(), model2.state_dict().items()):
        assert torch.equal(v, w), k
    assert lrn.update(samples[2]) == lrn2.update(samples[2])


# ---------------------------------------------------------------- the agent
def _agent_config(**over):
    from xuance_b200.common.common_tools import get_arguments
    cfg = get_arguments("iql", "sc2", "3m")
    base = dict(vectorize="Dummy_StarCraft2", parallels=8, buffer_size=64, batch_size=16, learning_rate=2e-3, gamma=0.5,
                start_greedy=1.0, end_greedy=0.05, decay_step_greedy=12000, start_training=200, running_steps=40000,
                n_epochs=4, sync_frequency=20, device=DEV, model_dir="/tmp/xb200_iql_models",
                log_dir="/tmp/xb200_iql_logs", episode_limit=20, p_death=0.02, distributed_training=False,
                use_cuda_graph=False)
    base.update(over)
    for k, v in base.items():
        setattr(cfg, k, v)
    return cfg


def test_iql_learns_through_the_agent_registry():
    """REGISTRY_Agents["IQL"] with the shipped 3m config on the cue-following SMAC-shaped env: the greedy team score
    rises."""
    from xuance_b200.environment import make_envs
    from xuance_b200.torch.agents import REGISTRY_Agents
    from xuance_b200.torch.rl_models import IndependentMixer, MixingQNetwork
    cfg = _agent_config()
    envs = make_envs(cfg)
    ag = REGISTRY_Agents["IQL"](cfg, envs)
    assert isinstance(ag.model, MixingQNetwork) and isinstance(ag.model.eval_Qtot, IndependentMixer)
    assert ag.use_actions_mask and not ag.use_global_state
    before = float(np.mean(ag.test(16, make_envs(cfg))))
    info = ag.train(cfg.running_steps // cfg.parallels)
    assert {"shared/loss_Q", "shared/predictQ", "shared/learning_rate"} <= set(info)
    assert np.isfinite(info["shared/loss_Q"])
    after = float(np.mean(ag.test(32, make_envs(cfg))))
    assert after > before + 2.0, (before, after)
    ag.finish()


def test_acting_greedy_equals_the_learners_greedy_and_the_replay_round_trips():
    """Step-by-step acting (model.forward with its GRU state and the masks) picks, at steps 1..T, the actions K9I takes
    as its greedy next actions from the learner's sequence forward (rows whose top two values are 1e-4 apart or more);
    the replay's state_dict restores a buffer that samples the same batch."""
    from xuance_b200.environment import make_envs
    from xuance_b200.torch.agents import REGISTRY_Agents
    _no_tf32()
    cfg = _agent_config(running_steps=3000, start_training=100)
    envs = make_envs(cfg)
    ag = REGISTRY_Agents["IQL"](cfg, envs)
    ag.train(cfg.running_steps // cfg.parallels)
    np.random.seed(3)
    s = ag.memory.sample()
    d = ag.learner._stacked(s)
    obs, avail = d["obs"], d["avail"]
    B, n, T1 = obs.shape[:3]
    T = T1 - 1
    with torch.no_grad():
        q_all = ag.model.q_values(obs.flatten(0, 1)).reshape(B, n, T1, -1).contiguous()
        A = q_all.shape[-1]
        rnn = ag.model.init_rnn_states(B)
        acts = []
        for t in range(T1):
            a, _, rnn = ag.model(observations=obs[:, :, t].reshape(B * n, -1),
                                 avail_actions=avail[:, :, t, :A].reshape(B * n, A), rnn_states=rnn)
            acts.append(a.reshape(B, n))
    acting = torch.stack(acts, 2)[:, :, 1:].cpu()
    x = {k: d[k].cpu() for k in ("actions", "rewards", "terminals", "agent_mask", "filled")}
    x.update(q_all=q_all.cpu(), q_tgt=q_all.cpu(), avail=avail.cpu())
    got = _run_k9i(x, True)
    qm = q_all[:, :, 1:].masked_fill(avail[:, :, 1:, :A] == 0, -1e10).cpu()
    top2 = qm.topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1]) >= 1e-4
    assert clear.float().mean().item() > 0.5
    assert torch.equal(acting[clear], got["next"].long()[clear])
    # the replay round trip
    sd = ag.memory.state_dict()
    ag2 = REGISTRY_Agents["IQL"](cfg, envs)
    ag2.memory.load_state_dict(sd)
    np.random.seed(4)
    sa = ag.memory.sample()
    np.random.seed(4)
    sb = ag2.memory.sample()
    for k, v in sa["_stacked"].items():
        assert torch.equal(v, sb["_stacked"][k]), k
    ag.finish()
    ag2.finish()
