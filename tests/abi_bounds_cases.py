"""The case table of the banded-operand harness (tests/abi_bounds.py): one record per kernel-launching entry point of
include/xb200.h, with its operands and their documented roles, a builder of legal inputs, the launch, and the float64 check
of the family's own test at the family's stated tolerance.  Shapes sit where the kernel's control flow turns: 1 row and 257
rows for row reductions plus one grid-stride launch above XB_MAX_PARTIALS * 256 rows per reduction kernel, each template
tier's maximum and maximum + 1, n = 1, 2, 3 (mod 4) for the float4 streams, and the documented NULL options.

Family helpers are imported where they are used, so this table imports on a machine without a GPU (the CPU test checks it
against the header)."""
import numpy as np
import torch

from abi_bounds import Case, Op

f32 = np.float32
XB_MAX_PARTIALS = 2048
BIG = XB_MAX_PARTIALS * 256 + 1           # first row count in the grid-stride regime of the two-level reductions


def _lib():
    from xuance_b200 import _lib
    return _lib


def _call(name, *args):
    L = _lib()
    L.call(name, *[L.ptr(a) if (a is None or torch.is_tensor(a)) else a for a in args])


def _np(t):
    return t.detach().cpu().numpy()


def _err(got, want):
    """Largest |got - want| (float64)."""
    return float(np.max(np.abs(np.asarray(_np(got) if torch.is_tensor(got) else got, np.float64) - np.asarray(want, np.float64)),
                        initial=0.0))


def _exact(got, want, what):
    g = _np(got) if torch.is_tensor(got) else np.asarray(got)
    assert np.array_equal(g, np.asarray(want, g.dtype)), f"{what}: not bit-equal to the restatement"
    return 0.0


def IN(x, mis=False, dtype=None, legal=0, ld=None, shape=None):
    x = np.asarray(x)
    dt = dtype or {np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64,
                   np.dtype(np.int32): torch.int32, np.dtype(np.int64): torch.int64, np.dtype(np.uint8): torch.uint8}[x.dtype]
    return Op("in", shape or x.shape, dt, data=x, mis=mis, legal=legal, ld=ld)


def OUT(*shape, dtype=torch.float32, mis=False, role="out", unwritten=None):
    return Op(role, shape, dtype, mis=mis, unwritten=unwritten)


def INOUT(x, mis=False):
    return Op("inout", np.asarray(x).shape, torch.float32 if np.asarray(x).dtype == np.float32 else torch.float64,
              data=np.asarray(x), mis=mis)


def SCRATCH():
    return Op("scratch", (XB_MAX_PARTIALS * 8 + 8,), torch.float64)


CASES = []


def case(name, shapes, values=None):
    def deco(fn):
        build, launch = fn()
        CASES.append(Case(name, shapes, build, launch, values))
        return fn
    return deco


# ================================================================================================ K7 optimiser
def _g(rng, n):
    return (rng.normal(size=n) * 1e-2).astype(f32)


def _sumsq_values(got, x, s):
    import test_gpu_kernel_edges as ke
    import kernel_refs as kr
    want = kr.grad_norm(x["g"], 0.75)
    ke._within(got["norm"], [want], 2 * kr.EPS32 * want, "norm")          # test_grad_sumsq_tails' bound
    return {"norm": _err(got["norm"], [want])}


@case("xb_grad_sumsq", [dict(n=1), dict(n=2), dict(n=3), dict(n=257), dict(n=4 * BIG + 3)], _sumsq_values)
def _():
    return (lambda s, rng: dict(g=IN(_g(rng, s["n"])), norm=OUT(1), scratch=SCRATCH()),
            lambda t, s: _call("xb_grad_sumsq", t["g"], s["n"], 0.75, t["norm"], t["scratch"]))


ADAM = dict(b1=0.9, b2=0.999, eps=1e-5, lr=1e-3, scale=0.5)


def _adam_build(s, rng):
    n = s["n"]
    g = _g(rng, n)
    g[::5] *= 1e-5
    norm = np.array([np.sqrt((g.astype(np.float64) ** 2).sum()) * ADAM["scale"]], f32)
    hyper = np.array([ADAM["lr"] / (1 - ADAM["b1"]), np.sqrt(1 - ADAM["b2"]), ADAM["lr"], 0.0], f32)
    return dict(p=INOUT(rng.normal(size=n).astype(f32)), g=INOUT(g), m=INOUT(np.zeros(n, f32)), v=INOUT(np.zeros(n, f32)),
                hyper=IN(hyper), norm=IN(norm))


def _adam_values(got, x, s):
    """Step 1 of test_adam_step_against_float64_and_torch: its float64 rule and bounds, clipping active, write-back on."""
    import test_gpu_kernel_edges as ke
    import kernel_refs as kr
    EPS = kr.EPS32
    max_norm = 0.5 * float(x["norm"][0])                        # clipping active
    coef = kr.adam_coef(float(x["norm"][0]), max_norm, ADAM["scale"])
    hp = x["hyper"]
    p, g, m, v = kr.adam_step(x["p"], x["g"], x["m"], x["v"], hp[0], hp[1], ADAM["b1"], ADAM["b2"], ADAM["eps"], coef)
    mm = ADAM["b1"] * np.abs(x["m"].astype(np.float64)) + (1 - ADAM["b1"]) * np.abs(g)
    vv = ADAM["b2"] * np.abs(x["v"].astype(np.float64)) + (1 - ADAM["b2"]) * g * g
    ke._within(got["p"], p, 2 * EPS * np.abs(x["p"]) + 32 * EPS * np.abs(p - x["p"]), "p")
    ke._within(got["m"], m, 16 * EPS * mm, "m")
    ke._within(got["v"], v, 16 * EPS * vv, "v")
    ke._within(got["g"], g, 8 * EPS * np.abs(g), "g (write-back)")
    return {k: _err(got[k], w) for k, w in (("p", p), ("m", m), ("v", v), ("g", g))}


@case("xb_adam_step", [dict(n=1), dict(n=4 * 64 + 1), dict(n=4 * 300 + 2), dict(n=4 * 1000 + 3)], _adam_values)
def _():
    return (_adam_build,
            lambda t, s: _call("xb_adam_step", t["p"], t["g"], t["m"], t["v"], s["n"], t["hyper"], ADAM["b1"], ADAM["b2"],
                               ADAM["eps"], 0.5 * float(t["norm"].item()), t["norm"], ADAM["scale"], 1))


def _soft_values(got, x, s):
    import kernel_refs as kr
    return {"target": _exact(got["target"], kr.soft_update_f32(x["target"], x["source"], 0.005), "target")}


@case("xb_soft_update", [dict(n=n, align=a) for n in (1, 4 * 257 + 2, 4 * 1000 + 3) for a in (16, 4)], _soft_values)
def _():
    return (lambda s, rng: dict(target=INOUT((rng.normal(size=s["n"]) * 3).astype(f32), mis=True),
                                source=IN((rng.normal(size=s["n"]) * 3).astype(f32), mis=True)),
            lambda t, s: _call("xb_soft_update", t["target"], t["source"], s["n"], 0.005))


# ================================================================================================ K8 SAC
ALPHA, SAC_GAMMA = f32(0.37), 0.99


def _sac_actor_values(got, x, s):
    """test_gpu_kernel_edges._check_sac's actor bounds."""
    import test_gpu_kernel_edges as ke
    import kernel_refs as kr
    EPS, B = kr.EPS32, s["B"]
    dlp, dq1, dq2, st = kr.sac_actor(x["log_pi"], x["q1"], x["q2"], ALPHA, B)
    ke._within(got["dlog_pi"], dlp, 2 * EPS * np.abs(dlp), "dlog_pi")
    ke._within(got["dq1"], dq1, EPS * np.abs(dq1), "dq1")
    ke._within(got["dq2"], dq2, EPS * np.abs(dq2), "dq2")
    lp, mq = x["log_pi"].astype(np.float64), np.minimum(x["q1"], x["q2"]).astype(np.float64)
    g = _np(got["stats"])
    ke._within(g[:3], st, [2 * EPS * (np.abs(ALPHA * lp) + np.abs(mq)).sum() / B + 2 * EPS * abs(st[0]),
                           2 * EPS * np.abs(mq).sum() / B, 2 * EPS * np.abs(lp).sum() / B], "stats")
    assert g[3] == 0
    return {"dlog_pi": _err(got["dlog_pi"], dlp), "dq1": _err(got["dq1"], dq1), "stats": _err(g[:3], st)}


@case("xb_sac_actor_loss", [dict(B=1), dict(B=257), dict(B=BIG)], _sac_actor_values)
def _():
    def build(s, rng):
        import test_gpu_kernel_edges as ke
        x = ke._sac_inputs(s["B"], seed=s["B"])
        B = s["B"]
        return dict(log_pi=IN(x["log_pi"]), q1=IN(x["q1"]), q2=IN(x["q2"]), alpha=IN(np.array([ALPHA], f32)),
                    dlog_pi=OUT(B), dq1=OUT(B), dq2=OUT(B), stats=OUT(4), scratch=SCRATCH())
    return build, lambda t, s: _call("xb_sac_actor_loss", t["log_pi"], t["q1"], t["q2"], t["alpha"], s["B"], s["B"],
                                     t["dlog_pi"], t["dq1"], t["dq2"], t["stats"], t["scratch"])


def _sac_critic_values(got, x, s):
    """test_gpu_kernel_edges._check_sac's critic bounds: backup bit-exact, dq and Qloss from the backup's error."""
    import test_gpu_kernel_edges as ke
    import kernel_refs as kr
    EPS, B = kr.EPS32, s["B"]
    cq1, cq2, y, cst = kr.sac_critic(x["q1"], x["q2"], x["target_q"], x["log_pi_next"], x["rew"], x["term"], ALPHA,
                                     SAC_GAMMA, B)
    _exact(got["backup"], kr.sac_backup_f32(x["target_q"], x["log_pi_next"], x["rew"], x["term"], ALPHA, SAC_GAMMA),
           "backup")
    d0 = 3 * EPS * (np.abs(x["rew"]) + np.abs(x["target_q"]) + np.abs(ALPHA * x["log_pi_next"]))
    qtol = 4 * EPS * cst[0]
    for q, name, ref in ((x["q1"], "dq1", cq1), (x["q2"], "dq2", cq2)):
        e = q - y
        d = EPS * np.abs(e) + d0
        ke._within(got[name], ref, 2 * d / B + 2 * EPS * np.abs(ref), name)
        qtol += (2 * np.abs(e) * d).sum() / B
    ke._within(_np(got["stats"])[:1], cst, qtol, "Qloss")
    assert _np(got["stats"])[1] == 0
    return {"dq1": _err(got["dq1"], cq1), "dq2": _err(got["dq2"], cq2), "Qloss": _err(_np(got["stats"])[:1], cst)}


@case("xb_sac_critic_loss", [dict(B=1), dict(B=257), dict(B=BIG)], _sac_critic_values)
def _():
    def build(s, rng):
        import test_gpu_kernel_edges as ke
        x = ke._sac_inputs(s["B"], seed=s["B"])
        B = s["B"]
        return dict(q1=IN(x["aq1"]), q2=IN(x["aq2"]), target_q=IN(x["target_q"]), log_pi_next=IN(x["log_pi_next"]),
                    rew=IN(x["rew"]), term=IN(x["term"]), alpha=IN(np.array([ALPHA], f32)),
                    dq1=OUT(B), dq2=OUT(B), backup=OUT(B), stats=OUT(2), scratch=SCRATCH())
    return build, lambda t, s: _call("xb_sac_critic_loss", t["q1"], t["q2"], t["target_q"], t["log_pi_next"], t["rew"],
                                     t["term"], t["alpha"], SAC_GAMMA, s["B"], s["B"], t["dq1"], t["dq2"], t["backup"],
                                     t["stats"], t["scratch"])


# ================================================================================================ K4 PPO / K6 DQN
def _ppo_values(got, x, s):
    import test_gpu_kernel_edges as ke
    Bt = s.get("Bt", s["B"])
    ke._check_ppo((got["dlogits"], got["dvalue"], got["stats"]), x, Bt, s["kind"])
    import kernel_refs as kr
    dz, dv, _ = kr.ppo_loss(x["logits"], x["value"], x["actions"], x["old_logp"], x["adv"], x["ret"], Bt, f32(0.2),
                            f32(0.25), f32(0.01), s["kind"])
    return {"dlogits": _err(got["dlogits"], dz), "dvalue": _err(got["dvalue"], dv)}


# template tiers A <= 4 / 8 / 18 / 32 / 64 (losses.cu): each maximum and maximum + 1; Bt > B: a shard of a larger minibatch
@case("xb_ppo_loss_fwd_bwd", [dict(B=1, A=1, kind=0), dict(B=257, A=4, kind=0), dict(B=257, A=5, kind=1),
                              dict(B=257, A=8, kind=0), dict(B=257, A=9, kind=1), dict(B=257, A=18, kind=0),
                              dict(B=257, A=19, kind=0), dict(B=257, A=32, kind=1), dict(B=257, A=33, kind=0),
                              dict(B=257, A=64, kind=0), dict(B=257, A=6, kind=0, Bt=1000), dict(B=BIG, A=4, kind=0)],
      _ppo_values)
def _():
    def build(s, rng):
        import test_gpu_kernel_edges as ke
        x = ke._ppo_inputs(s["B"], s["A"], seed=s["B"] + s["A"])
        B, A = s["B"], s["A"]
        return dict(**{k: IN(v) for k, v in x.items()}, dlogits=OUT(B, A), dvalue=OUT(B), stats=OUT(8), scratch=SCRATCH())
    return build, lambda t, s: _call("xb_ppo_loss_fwd_bwd", t["logits"], t["value"], t["actions"], t["old_logp"], t["adv"],
                                     t["ret"], s["B"], s["A"], s.get("Bt", s["B"]), 0.2, 0.25, 0.01, s["kind"], t["dlogits"],
                                     t["dvalue"], t["stats"], t["scratch"])


def _dqn_values(got, x, s):
    import test_gpu_kernel_edges as ke
    import kernel_refs as kr
    ke._check_dqn((got["dq"], got["td"], got["stats"]), x, s["B"], s["dq"])
    dq, _, td, _ = kr.dqn_td(x["q_eval"], x["q_next"], x.get("q_sel") if s["dq"] else None, x["actions"], x["rew"],
                             x["term"], s["B"], 0.99)
    return {"dq": _err(got["dq"], dq), "td": _err(got["td"], td)}


@case("xb_dqn_td_fwd_bwd", [dict(B=1, A=1, dq=0), dict(B=257, A=6, dq=1), dict(B=257, A=18, dq=0),
                            dict(B=BIG, A=6, dq=1)], _dqn_values)
def _():
    def build(s, rng):
        import test_gpu_kernel_edges as ke
        x = ke._dqn_inputs(s["B"], s["A"], seed=s["B"] + s["A"])
        if not s["dq"]:
            x.pop("q_sel")
        B, A = s["B"], s["A"]
        return dict(**{k: IN(v) for k, v in x.items()}, dq=OUT(B, A), td=OUT(B), stats=OUT(4), scratch=SCRATCH())
    return build, lambda t, s: _call("xb_dqn_td_fwd_bwd", t["q_eval"], t["q_next"], t.get("q_sel"), t["actions"],
                                     t["rew"], t["term"], s["B"], s["A"], s["B"], 0.99, t["dq"], t["td"], t["stats"],
                                     t["scratch"])


# ================================================================================================ K3 scalars
def _gs_values(got, x, s):
    import test_gpu_kernel_edges as ke
    import kernel_refs as kr
    idx = x["idx"] if "idx" in x else np.arange(s["B"])
    g = _np(got["out"])
    sel = x["fields"][:, idx]
    _exact(g[0], sel[0], "field 0")
    _exact(g[2], sel[2], "field 2")
    mean, std = kr.adv_stats(sel[1])
    st = _np(got["stats"])
    ke._within(st, [mean, std], [2 * kr.EPS32 * abs(mean), 4 * kr.EPS32 * std], "statistics")
    _exact(g[1], kr.adv_normalize_f32(sel[1], st), "normalised field")
    return {"stats": _err(st, [mean, std])}


@case("xb_gather_scalars", [dict(B=1, idx=1), dict(B=257, idx=0), dict(B=BIG, idx=1)], _gs_values)
def _():
    def build(s, rng):
        B, F = s["B"], 3
        slots = B + 37
        fields = (rng.normal(size=(F, slots)) + 0.3).astype(f32)
        idx = IN(rng.permutation(slots)[:B].astype(np.int64)) if s["idx"] else None
        return dict(fields=IN(fields), idx=idx, out=OUT(F, B), stats=OUT(2), scratch=SCRATCH())
    return build, lambda t, s: _call("xb_gather_scalars", t["fields"], t["fields"].shape[1], t["idx"], s["B"], 3, t["out"],
                                     1, t["stats"], t["scratch"])


@case("xb_adv_normalize", [dict(B=1), dict(B=4 * 257 + 1), dict(B=BIG)],
      lambda got, x, s: {"adv": _exact(got["adv"], __import__("kernel_refs").adv_normalize_f32(x["adv"], x["stats"]), "adv")})
def _():
    return (lambda s, rng: dict(adv=INOUT(rng.normal(size=s["B"]).astype(f32)), stats=IN(np.array([0.25, 1.75], f32))),
            lambda t, s: _call("xb_adv_normalize", t["adv"], s["B"], t["stats"]))


# ================================================================================================ K13 / K13L
def _rnn_problem(s, gates):
    """test_gpu_gru_k13 / test_gpu_drqn's scale: U(+-1/sqrt(H)) weights, unit-scale projected inputs."""
    S, T, H = s["S"], s["T"], s["H"]
    rng = np.random.default_rng(S * 7 + T * 3 + H)
    k = 1.0 / np.sqrt(H)
    u = lambda *shape: ((rng.random(shape) * 2 - 1) * k).astype(f32)
    return dict(xg=rng.normal(size=(S, T, gates * H)).astype(f32), w_hh=u(gates * H, H), b_hh=u(gates * H),
                h0=(rng.normal(size=(S, H)) * 0.5).astype(f32) if s["state"] else None,
                c0=rng.normal(size=(S, H)).astype(f32) if s["state"] else None,
                dy=rng.normal(size=(S, T, H)).astype(f32),
                dhT=rng.normal(size=(S, H)).astype(f32) if s["state"] else None,
                dcT=rng.normal(size=(S, H)).astype(f32) if s["state"] else None)


def _rel(got, ref):
    """K13's error measure: relative to max(1, max |ref|) (test_gpu_gru_k13._rel_err)."""
    ref = np.asarray(ref, np.float64)
    return float(np.abs(_np(got).astype(np.float64) - ref).max() / max(1.0, np.abs(ref).max()))


K13_TOL = 1e-6                            # TOL_FWD = TOL_BWD of test_gpu_gru_k13.py and test_gpu_drqn.py


def _rel_check(got, refs):
    errs = {k: _rel(got[k], v) for k, v in refs.items() if got.get(k) is not None}
    assert all(e <= K13_TOL for e in errs.values()), errs          # a NaN error fails too
    return errs


RNN_SHAPES = [dict(S=1, T=1, H=1, state=0), dict(S=5, T=3, H=33, state=1), dict(S=9, T=2, H=64, state=1)]
LSTM_SHAPES = RNN_SHAPES[:2] + [dict(S=5, T=2, H=128, state=1)]


@case("xb_gru_seq_fwd", RNN_SHAPES,
      lambda got, x, s: _rel_check(got, dict(zip(("y", "hT", "gates"), __import__("gru_refs").gru_fwd(
          x["xg"], x["w_hh"], x["b_hh"], x.get("h0"))))))
def _():
    def build(s, rng):
        p = _rnn_problem(s, 3)
        S, T, H = s["S"], s["T"], s["H"]
        return dict(xg=IN(p["xg"]), w_hh=IN(p["w_hh"]), b_hh=IN(p["b_hh"]), h0=IN(p["h0"]) if s["state"] else None,
                    y=OUT(S, T, H), hT=OUT(S, H), gates=OUT(S, T, 4 * H))
    return build, lambda t, s: _call("xb_gru_seq_fwd", t["xg"], t["w_hh"], t["b_hh"], t["h0"], s["S"], s["T"], s["H"],
                                     t["y"], t["hT"], t["gates"])


def _gru_bwd_build(s, rng):
    from gru_refs import gru_fwd
    p = _rnn_problem(s, 3)
    S, T, H = s["S"], s["T"], s["H"]
    y, _, gates = gru_fwd(p["xg"], p["w_hh"], p["b_hh"], p["h0"])
    return dict(dy=IN(p["dy"]), dhT=IN(p["dhT"]) if s["state"] else None, w_hh=IN(p["w_hh"]), gates=IN(gates.astype(f32)),
                y=IN(y.astype(f32)), h0=IN(p["h0"]) if s["state"] else None,
                dxg=OUT(S, T, 3 * H), dgh=OUT(S, T, 3 * H), dh0=OUT(S, H))


@case("xb_gru_seq_bwd", RNN_SHAPES,
      lambda got, x, s: _rel_check(got, dict(zip(("dxg", "dgh", "dh0"), __import__("gru_refs").gru_bwd(
          x["dy"], x.get("dhT"), x["w_hh"], x["gates"], x["y"], x.get("h0"))))))
def _():
    return _gru_bwd_build, lambda t, s: _call("xb_gru_seq_bwd", t["dy"], t["dhT"], t["w_hh"], t["gates"], t["y"], t["h0"],
                                              s["S"], s["T"], s["H"], t["dxg"], t["dgh"], t["dh0"])


@case("xb_lstm_seq_fwd", LSTM_SHAPES,
      lambda got, x, s: _rel_check(got, dict(zip(("y", "hT", "cT", "gates"), __import__("lstm_refs").lstm_fwd(
          x["xg"], x["w_hh"], x["b_hh"], x.get("h0"), x.get("c0"))))))
def _():
    def build(s, rng):
        p = _rnn_problem(s, 4)
        S, T, H = s["S"], s["T"], s["H"]
        st = s["state"]
        return dict(xg=IN(p["xg"]), w_hh=IN(p["w_hh"]), b_hh=IN(p["b_hh"]), h0=IN(p["h0"]) if st else None,
                    c0=IN(p["c0"]) if st else None, y=OUT(S, T, H), hT=OUT(S, H), cT=OUT(S, H), gates=OUT(S, T, 5 * H))
    return build, lambda t, s: _call("xb_lstm_seq_fwd", t["xg"], t["w_hh"], t["b_hh"], t["h0"], t["c0"], s["S"], s["T"],
                                     s["H"], t["y"], t["hT"], t["cT"], t["gates"])


def _lstm_bwd_build(s, rng):
    from lstm_refs import lstm_fwd
    p = _rnn_problem(s, 4)
    S, T, H = s["S"], s["T"], s["H"]
    st = s["state"]
    _, _, _, gates = lstm_fwd(p["xg"], p["w_hh"], p["b_hh"], p["h0"], p["c0"])
    return dict(dy=IN(p["dy"]), dhT=IN(p["dhT"]) if st else None, dcT=IN(p["dcT"]) if st else None, w_hh=IN(p["w_hh"]),
                gates=IN(gates.astype(f32)), c0=IN(p["c0"]) if st else None,
                dxg=OUT(S, T, 4 * H), dh0=OUT(S, H), dc0=OUT(S, H))


@case("xb_lstm_seq_bwd", LSTM_SHAPES,
      lambda got, x, s: _rel_check(got, dict(zip(("dxg", "dh0", "dc0"), __import__("lstm_refs").lstm_bwd(
          x["dy"], x.get("dhT"), x.get("dcT"), x["w_hh"], x["gates"], x.get("c0"))))))
def _():
    return _lstm_bwd_build, lambda t, s: _call("xb_lstm_seq_bwd", t["dy"], t["dhT"], t["dcT"], t["w_hh"], t["gates"],
                                               t["c0"], s["S"], s["T"], s["H"], t["dxg"], t["dh0"], t["dc0"])


# ================================================================================================ K1 / K3 byte movers
def _rows(rng, n_rows, row_bytes):
    """Row data as int32 words (finite float32 bit patterns, never an output payload)."""
    return rng.normal(size=(n_rows, row_bytes // 4)).astype(f32).view(np.int32)


STORE_SHAPES = [dict(row_bytes=4, F=1, N=1, T=3, align=4), dict(row_bytes=12, F=0, N=5, T=2, align=4),
                dict(row_bytes=2048, F=2, N=3, T=4), dict(row_bytes=2064, F=3, N=257, T=2)]


def _store_values(got, x, s):
    N, T, W, F = s["N"], s["T"], s["row_bytes"] // 4, s["F"]
    step = x["step"] if "step" in x else np.full(N, s["T"] - 1)
    want = x["dst"].copy()
    ok = (step >= 0) & (step < T)
    want[np.arange(N)[ok], step[ok]] = x["src"][ok]
    _exact(got["dst"], want, "rows")
    if F:
        sw = x["sdst"].copy()
        sw[:, np.arange(N)[ok], step[ok]] = x["ssrc"][:, ok]
        _exact(got["sdst"], sw, "scalars")
    return {"rows": 0.0}


def _store_build(s, rng, at):
    N, T, W, F = s["N"], s["T"], s["row_bytes"] // 4, s["F"]
    ops = dict(dst=INOUT_I(_rows(rng, N * T, s["row_bytes"]).reshape(N, T, W), mis=True),
               src=IN(_rows(rng, N, s["row_bytes"]), mis=True),
               sdst=INOUT(rng.normal(size=(F, N, T)).astype(f32)) if F else None,
               ssrc=IN(rng.normal(size=(F, N)).astype(f32)) if F else None)
    if at:
        step = rng.integers(-1, T + 1, N).astype(np.int32)                  # some rows outside [0, T): not written
        step[0] = T                                                           # ... at least one
        ops["step"] = IN(step)
    return ops


def INOUT_I(x, mis=False):
    return Op("inout", x.shape, torch.int32, data=x, mis=mis)


@case("xb_rollout_store", STORE_SHAPES, _store_values)
def _():
    return (lambda s, rng: _store_build(s, rng, False),
            lambda t, s: _call("xb_rollout_store", t["dst"], t["src"], s["row_bytes"], t["sdst"], t["ssrc"], s["F"], s["N"],
                               s["T"], s["T"] - 1))


@case("xb_rollout_store_at", STORE_SHAPES, _store_values)
def _():
    return (lambda s, rng: _store_build(s, rng, True),
            lambda t, s: _call("xb_rollout_store_at", t["dst"], t["src"], s["row_bytes"], t["sdst"], t["ssrc"], s["F"],
                               s["N"], s["T"], t["step"]))


def _gather_values(got, x, s):
    idx = x["idx"] if "idx" in x else np.arange(s["B"])
    return {"dst": _exact(got["dst"], x["src"][idx], "rows")}


@case("xb_gather_rows", [dict(row_bytes=4, B=1, idx=1, align=4), dict(row_bytes=12, B=257, idx=1, align=4),
                         dict(row_bytes=2048, B=7, idx=0), dict(row_bytes=2064, B=257, idx=1)], _gather_values)
def _():
    def build(s, rng):
        slots = s["B"] + 11
        return dict(src=IN(_rows(rng, slots, s["row_bytes"]), mis=True),
                    idx=IN(rng.integers(0, slots, s["B"]).astype(np.int64)) if s["idx"] else None,
                    dst=OUT(s["B"], s["row_bytes"] // 4, dtype=torch.int32, mis=True))
    return build, lambda t, s: _call("xb_gather_rows", t["src"], t["idx"], s["B"], s["row_bytes"], t["dst"])


# ================================================================================================ K8T DDPG / TD3
def _perturb_values(got, x, s):
    """test_gpu_ddpg_td3's float64 comparison (rtol = atol = 1e-6; torch's float32 expression is pinned bit for bit
    there)."""
    from ddpg_refs import perturb_ref
    want = perturb_ref(x["a"], x["noise"], f32(0.1), f32(s["clip"]) if s["clip"] >= 0 else -1, x["low"], x["high"])
    np.testing.assert_allclose(_np(got["a"]), want, rtol=1e-6, atol=1e-6, err_msg="out (in place)")
    return {"out": _err(got["a"], want)}


@case("xb_perturb_actions", [dict(B=1, D=1, clip=-1.0), dict(B=257, D=3, clip=0.5), dict(B=33, D=6, clip=0.2)],
      _perturb_values)
def _():
    def build(s, rng):
        B, D = s["B"], s["D"]
        return dict(a=INOUT(rng.uniform(-1, 1, (B, D)).astype(f32)), noise=IN(rng.normal(size=(B, D)).astype(f32)),
                    low=IN(np.full(D, -1, f32)), high=IN(np.full(D, 1, f32)))
    return build, lambda t, s: _call("xb_perturb_actions", t["a"], t["noise"], s["B"], s["D"], 0.1, s["clip"], t["low"],
                                     t["high"], t["a"])


def _ddpg_critic_values(got, x, s):
    """test_gpu_ddpg_td3's bounds: backup 1e-6, dq 1e-5 relative, statistics 2e-5."""
    from ddpg_refs import critic_ref
    r1, r2, rb, rst = critic_ref(x["q1"], x.get("q2"), x["tq1"], x.get("tq2"), x["rew"], x["term"], f32(0.99), s["B"])
    np.testing.assert_allclose(_np(got["backup"]), rb, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(_np(got["dq1"]), r1, rtol=1e-5, atol=1e-5 * np.abs(r1).max())
    if s["twin"]:
        np.testing.assert_allclose(_np(got["dq2"]), r2, rtol=1e-5, atol=1e-5 * np.abs(r2).max())
    st = _np(got["stats"])
    np.testing.assert_allclose(st[:3], rst, rtol=2e-5, atol=1e-6)
    assert st[3] == 0.0
    return {"backup": _err(got["backup"], rb), "dq1": _err(got["dq1"], r1), "stats": _err(st[:3], rst)}


def _ddpg_actor_values(got, x, s):
    from ddpg_refs import actor_ref
    B = s["B"]
    s1, _, pl = actor_ref(x["q1"], x.get("q2"), B)
    seed = f32(-1.0) / f32(B)
    _exact(got["dq1"], np.full(B, seed * f32(0.5) if s["twin"] else seed, f32), "dq1")
    if s["twin"]:
        _exact(got["dq2"], _np(got["dq1"]), "dq2")
    np.testing.assert_allclose(_np(got["stats"])[0], pl, rtol=2e-5, atol=1e-7)
    return {"dq1": _err(got["dq1"], s1), "Ploss": _err(_np(got["stats"])[:1], [pl])}


@case("xb_ddpg_critic_loss", [dict(B=1, twin=0), dict(B=257, twin=1), dict(B=BIG, twin=1)], _ddpg_critic_values)
def _():
    def build(s, rng):
        B, tw = s["B"], s["twin"]
        r = lambda: rng.normal(size=B).astype(f32)
        return dict(q1=IN(r()), q2=IN(r()) if tw else None, tq1=IN(r()), tq2=IN(r()) if tw else None, rew=IN(r()),
                    term=IN((rng.random(B) < 0.3).astype(f32)), dq1=OUT(B), dq2=OUT(B) if tw else None, backup=OUT(B),
                    stats=OUT(4), scratch=SCRATCH())
    return build, lambda t, s: _call("xb_ddpg_critic_loss", t["q1"], t["q2"], t["tq1"], t["tq2"], t["rew"], t["term"], 0.99,
                                     s["B"], s["B"], t["dq1"], t["dq2"], t["backup"], t["stats"], t["scratch"])


@case("xb_ddpg_actor_loss", [dict(B=1, twin=0), dict(B=257, twin=1), dict(B=BIG, twin=0)], _ddpg_actor_values)
def _():
    def build(s, rng):
        B, tw = s["B"], s["twin"]
        return dict(q1=IN(rng.normal(size=B).astype(f32)), q2=IN(rng.normal(size=B).astype(f32)) if tw else None,
                    dq1=OUT(B), dq2=OUT(B) if tw else None, stats=OUT(4), scratch=SCRATCH())
    return build, lambda t, s: _call("xb_ddpg_actor_loss", t["q1"], t["q2"], s["B"], s["B"], t["dq1"], t["dq2"], t["stats"],
                                     t["scratch"])


# ================================================================================================ K10 acting
def _gauss_act_values(got, x, s):
    """test_gpu_gauss_ppo's bounds: actions 4 EPS of their summands, logp lp_tol of the float32 action, entropy (D+2) EPS."""
    import gauss_refs as gr
    import test_gpu_kernel_edges as ke
    EPS, D = 2.0 ** -24, s["D"]
    mu, ls = x["mu"], x["log_std"]
    sig = np.exp(ls.astype(np.float64))[None, :]
    errs = {}
    if s["mode"] == "forced":
        a = x["forced"]
    else:
        a = _np(got["actions"])
        ref_a = gr.gaussian_act(mu, ls, noise=x.get("noise"))[0]
        noise = x.get("noise", np.zeros_like(mu))
        ke._within(a, ref_a, 4 * EPS * (np.abs(mu) + sig * np.abs(noise)), "actions")
        errs["actions"] = _err(a, ref_a)
    terms, z = gr.gauss_logp_terms(mu, ls, a.astype(np.float64))
    c = (np.abs(a) + np.abs(mu)) / sig + np.abs(z)
    mag = 0.5 * z * z + np.abs(ls.astype(np.float64))[None, :] + gr.LOG_SQRT_2PI
    _, lp, ent = gr.gaussian_act(mu, ls, forced=a)
    ke._within(got["logp"], lp, 4 * EPS * (np.abs(z) * c).sum(1) + (D + 2) * EPS * mag.sum(1), "logp")
    ke._within(got["entropy"], ent, (D + 2) * EPS * (0.5 + gr.LOG_SQRT_2PI + np.abs(ls.astype(np.float64))).sum(), "entropy")
    errs.update(logp=_err(got["logp"], lp), entropy=_err(got["entropy"], ent))
    return errs


@case("xb_gaussian_act", [dict(N=1, D=1, mode="forced"), dict(N=257, D=3, mode="noise"), dict(N=33, D=64, mode="det")],
      _gauss_act_values)
def _():
    def build(s, rng):
        N, D = s["N"], s["D"]
        forced = s["mode"] == "forced"
        return dict(mu=IN(rng.normal(size=(N, D)).astype(f32)), log_std=IN((rng.normal(size=D) * 0.3).astype(f32)),
                    noise=IN(rng.normal(size=(N, D)).astype(f32)) if s["mode"] == "noise" else None,
                    forced=IN(rng.normal(size=(N, D)).astype(f32)) if forced else None,
                    # with forced actions actions_f32 is documented as not written: every element keeps its sentinel
                    actions=OUT(N, D, role="out_partial", unwritten=np.ones((N, D), bool)) if forced else OUT(N, D),
                    logp=OUT(N), entropy=OUT(N))
    return build, lambda t, s: _call("xb_gaussian_act", t["mu"], t["log_std"], t["noise"], t["forced"], s["N"], s["D"],
                                     t["actions"], t["logp"], t["entropy"])


def _cat_act_values(got, x, s):
    """rollout_refs.categorical_bounds (test_gpu_rollout_edges): logp within E of the action's float64 log-probability,
    entropy within ent_bound; the action is the forced one, the first arg-max, or a draw with an unambiguous cdf."""
    import rollout_refs as rr
    import test_gpu_kernel_edges as ke
    lp, p, _, _ = rr.categorical(x["logits"])
    E, ent_b, delta = rr.categorical_bounds(x["logits"])
    a = _np(got["actions_i32"]).astype(np.int64)
    _exact(got["actions_f32"], a.astype(f32), "actions_f32")
    if s["mode"] == "forced":
        _exact(a, x["forced"].astype(np.int64), "forced actions")
    elif s["mode"] == "det":
        _exact(a, rr.argmax_first(x["logits"]), "arg-max actions")
    else:
        assert rr.draw_allowed(p, x["uniforms"], delta, a).all(), "drawn actions"
    N = len(a)
    ke._within(got["logp"], lp[np.arange(N), a], E[np.arange(N), a], "logp")
    ent = -(np.where(p > 0, p * lp, 0.0)).sum(1)
    ke._within(got["entropy"], ent, ent_b, "entropy")
    return {"logp": _err(got["logp"], lp[np.arange(N), a]), "entropy": _err(got["entropy"], ent)}


@case("xb_categorical_act", [dict(N=1, A=1, mode="uniform"), dict(N=257, A=33, mode="forced"),
                             dict(N=65, A=64, mode="det"), dict(N=300, A=5, mode="uniform")], _cat_act_values)
def _():
    def build(s, rng):
        N, A = s["N"], s["A"]
        return dict(logits=IN((rng.normal(size=(N, A)) * 3).astype(f32)),
                    uniforms=IN(rng.random(N).astype(f32)) if s["mode"] == "uniform" else None,
                    forced=IN(rng.integers(0, A, N).astype(f32)) if s["mode"] == "forced" else None,
                    actions_f32=OUT(N), actions_i32=OUT(N, dtype=torch.int32), logp=OUT(N), entropy=OUT(N))
    return build, lambda t, s: _call("xb_categorical_act", t["logits"], t["uniforms"], t["forced"], s["N"], s["A"],
                                     t["actions_f32"], t["actions_i32"], t["logp"], t["entropy"])


# ================================================================================================ K9 QMIX
def _qmix_sel_build(s, rng):
    B, n, T, A, ld = s["B"], s["n"], s["T"], s["A"], s["ld"]
    q_all = rng.integers(-2, 3, size=(B, n, T + 1, A)).astype(f32)
    return dict(q_all=IN(q_all), q_tgt=IN(rng.normal(size=(B, n, T + 1, A)).astype(f32)),
                actions=IN(rng.integers(0, A, size=(B, n, T)).astype(f32)),
                agent_mask=IN((rng.random((B, n, T)) < 0.8).astype(f32)), filled=IN((rng.random((B, T)) < 0.8).astype(f32)),
                avail=IN((rng.random((B, n, T + 1, A)) < 0.6).astype(np.uint8), ld=ld) if ld else None,
                qe=OUT(B * T, n), qn=OUT(B * T, n), fs=OUT(1), scratch=SCRATCH())


def _qmix_sel_values(got, x, s):
    import kernel_refs as kr
    ref = kr.qmix_select(x["q_all"], x["q_tgt"], x["actions"], x["agent_mask"], x["filled"], x.get("avail"), s["dq"])
    _exact(got["qe"], ref[0], "q_eval_taken")
    _exact(got["qn"], ref[1], "q_next_taken")
    assert float(got["fs"][0]) == ref[2]
    return {"q": 0.0}


@case("xb_qmix_select_fwd", [dict(B=1, n=1, T=1, A=1, ld=0, dq=0), dict(B=3, n=5, T=7, A=6, ld=9, dq=1),
                             dict(B=64, n=9, T=40, A=12, ld=13, dq=0)], _qmix_sel_values)
def _():
    return _qmix_sel_build, lambda t, s: _call("xb_qmix_select_fwd", t["q_all"], t["q_tgt"], t["actions"], t["agent_mask"],
                                               t["filled"], t["avail"], s["ld"], s["B"], s["n"], s["T"], s["A"], s["dq"],
                                               t["qe"], t["qn"], t["fs"], t["scratch"])


@case("xb_qmix_select_bwd", [dict(B=1, n=1, T=1, A=1), dict(B=3, n=5, T=7, A=6), dict(B=64, n=9, T=40, A=12)],
      lambda got, x, s: {"dq_all": _exact(got["dq_all"], __import__("kernel_refs").qmix_select_bwd(
          x["d"], x["actions"], x["agent_mask"], x["filled"], s["A"]), "dq_all")})
def _():
    def build(s, rng):
        B, n, T, A = s["B"], s["n"], s["T"], s["A"]
        return dict(d=IN(rng.normal(size=(B * T, n)).astype(f32)), actions=IN(rng.integers(0, A, (B, n, T)).astype(f32)),
                    agent_mask=IN((rng.random((B, n, T)) < 0.8).astype(f32)), filled=IN((rng.random((B, T)) < 0.8).astype(f32)),
                    dq_all=OUT(B, n, T + 1, A, role="out_scatter"))
    return build, lambda t, s: _call("xb_qmix_select_bwd", t["d"], t["actions"], t["agent_mask"], t["filled"], s["B"], s["n"],
                                     s["T"], s["A"], t["dq_all"])


@case("xb_powf_libm", [dict(n=1, align=4), dict(n=4 * 257 + 2), dict(n=4 * 257 + 3, align=4)],
      lambda got, x, s: {"out": _exact(got["out"], np.array([v ** 0.6 for v in x["x"]], f32), "out")})   # libm powf
def _():
    return (lambda s, rng: dict(x=IN((rng.random(s["n"]) * 3 + 1e-3).astype(f32), mis=True), out=OUT(s["n"], mis=True)),
            lambda t, s: _call("xb_powf_libm", t["x"], float(f32(0.6)), t["out"], s["n"]))


# ================================================================================================ K2 GAE scans
def _gae_build(s, rng, vn):
    N, T = s["N"], s["T"]
    seg = (rng.random((N, T)) < 0.2).astype(np.uint8)
    seg[:, -1] = 1
    cov = rng.integers(0, T + 1, N).astype(np.int32)
    ops = dict(rew=IN(rng.normal(size=(N, T)).astype(f32), mis=True), val=IN(rng.normal(size=(N, T)).astype(f32), mis=True),
               term=IN((rng.random((N, T)) < 0.1).astype(f32), mis=True), seg_end=IN(seg),
               boot=IN(rng.normal(size=(N, T)).astype(f32), mis=True), cov=IN(cov, legal=T))
    if vn:
        ops["start"] = IN(np.minimum(rng.integers(0, 3, N), cov).astype(np.int32))
        ops.update(rm=IN(np.array([0.3], f32)), rmsq=IN(np.array([1.4], f32)), dt=IN(np.array([0.9], f32)))
    # steps outside [start, covered) are documented as not written
    st = ops["start"].data if vn else np.zeros(N, np.int32)
    unw = (np.arange(T)[None, :] < st[:, None]) | (np.arange(T)[None, :] >= cov[:, None]) if vn else None
    role = "out_partial" if vn else "out"
    ops.update(adv=OUT(N, T, mis=True, role=role, unwritten=unw), ret=OUT(N, T, mis=True, role=role, unwritten=unw))
    return ops


GAE_SHAPES = [dict(N=1, T=1, gae=1), dict(N=3, T=4 * 33, gae=1), dict(N=5, T=4 * 33 + 1, gae=0),
              dict(N=2, T=4 * 40, gae=1, align=4), dict(N=4, T=67, gae=1, align=4)]


@case("xb_gae_scan", GAE_SHAPES)
def _():
    return (lambda s, rng: _gae_build(s, rng, False),
            lambda t, s: _call("xb_gae_scan", t["rew"], t["val"], t["term"], t["seg_end"], t["boot"], t["cov"], t["adv"],
                               t["ret"], s["N"], s["T"], 0.99, 0.95, s["gae"]))


@case("xb_gae_scan_vn", GAE_SHAPES)
def _():
    return (lambda s, rng: _gae_build(s, rng, True),
            lambda t, s: _call("xb_gae_scan_vn", t["rew"], t["val"], t["term"], t["seg_end"], t["boot"], t["start"], t["cov"],
                               t["adv"], t["ret"], s["N"], s["T"], 0.99, 0.95, s["gae"], t["rm"], t["rmsq"], t["dt"]))


# ================================================================================================ K3 observations
def _obs_values(got, x, s):
    idx = x["idx"] if "idx" in x else np.arange(s["B"])
    rows = x["src"].reshape(-1, s["H"] * s["W"] * s["C"])[idx]
    fmt = s["fmt"]
    dst = _np(got["dst"]).view(np.uint8).reshape(s["B"], -1)
    if fmt == 0:
        return {"dst": _exact(dst, rows, "u8")}
    val = torch.from_numpy(rows.astype(f32)) / 255.0
    if fmt == 1:
        return {"dst": _exact(dst.view(f32), val.numpy(), "f32")}
    if fmt == 2:
        want = val.view(s["B"], s["H"] * s["W"], s["C"]).transpose(1, 2).reshape(s["B"], -1).numpy()
        return {"dst": _exact(dst.view(f32), want, "f32 nchw")}
    want = val.to(torch.bfloat16 if fmt == 3 else torch.float16).view(torch.int16).numpy()
    return {"dst": _exact(dst.view(np.int16), want, "half")}


@case("xb_gather_obs", [dict(B=1, H=2, W=4, C=2, fmt=0, idx=1), dict(B=257, H=3, W=4, C=4, fmt=2, idx=1),
                        dict(B=33, H=2, W=8, C=4, fmt=1, idx=0), dict(B=17, H=2, W=2, C=4, fmt=3, idx=1),
                        dict(B=9, H=1, W=4, C=4, fmt=4, idx=1)], _obs_values)
def _():
    def build(s, rng):
        row = s["H"] * s["W"] * s["C"]
        slots = s["B"] + 5
        out_bytes = row * {0: 1, 1: 4, 2: 4, 3: 2, 4: 2}[s["fmt"]]
        return dict(src=IN(rng.integers(0, 256, (slots, row)).astype(np.uint8)),
                    idx=IN(rng.integers(0, slots, s["B"]).astype(np.int64)) if s["idx"] else None,
                    dst=OUT(s["B"], out_bytes // 4, dtype=torch.int32))
    return build, lambda t, s: _call("xb_gather_obs", t["src"], t["idx"], s["B"], s["H"], s["W"], s["C"], t["dst"], s["fmt"])


@case("xb_gather_obs_planes", [dict(B=1, row=16, planes=1, idx=1), dict(B=257, row=48, planes=2, idx=1),
                               dict(B=5, row=2048 + 16, planes=3, idx=0)])
def _():
    def build(s, rng):
        slots = s["B"] + 3
        return dict(src=IN(rng.integers(0, 256, (slots, s["row"])).astype(np.uint8)),
                    idx=IN(rng.integers(0, slots, s["B"]).astype(np.int64)) if s["idx"] else None,
                    dst=OUT(s["planes"], s["B"], s["row"] // 2, dtype=torch.int32))
    return build, lambda t, s: _call("xb_gather_obs_planes", t["src"], t["idx"], s["B"], s["row"], s["planes"], t["dst"])


@case("xb_rms_update_normalize", [dict(N=1, D=1, update=1), dict(N=257, D=3, update=1), dict(N=9, D=65, update=0)])
def _():
    def build(s, rng):
        N, D = s["N"], s["D"]
        return dict(x=IN(rng.normal(size=(N, D)).astype(f32)), mean=INOUT(rng.normal(size=D).astype(f32)),
                    var=INOUT((rng.random(D) + 0.5).astype(f32)), out=OUT(N, D))
    return build, lambda t, s: _call("xb_rms_update_normalize", t["x"], s["N"], s["D"], t["mean"], t["var"], 100.0,
                                     s["update"], t["out"], 5.0, 1e-8)


# ================================================================================================ K4G / K4P / K4N
def _gauss_batch(rng, B, D):
    x = dict(mu=rng.normal(size=(B, D)).astype(f32), log_std=(rng.normal(size=D) * 0.3).astype(f32),
             value=rng.normal(size=B).astype(f32), actions=rng.normal(size=(B, D)).astype(f32),
             adv=rng.normal(size=B).astype(f32), ret=rng.normal(size=B).astype(f32))
    return x


GAUSS_SHAPES = [dict(B=1, D=1), dict(B=257, D=5, Bt=600), dict(B=BIG, D=3), dict(B=40, D=64)]


@case("xb_ppo_gauss_loss_fwd_bwd", GAUSS_SHAPES)
def _():
    def build(s, rng):
        B, D = s["B"], s["D"]
        x = _gauss_batch(rng, B, D)
        x["old_logp"] = (rng.normal(size=B) - 3).astype(f32)
        ws = D * min((B + 255) // 256, 2048)
        return dict(**{k: IN(v) for k, v in x.items()}, dmu=OUT(B, D), dlog_std=OUT(D), dvalue=OUT(B), stats=OUT(8),
                    scratch=SCRATCH(), ws=Op("scratch", (ws,), torch.float64))
    return build, lambda t, s: _call("xb_ppo_gauss_loss_fwd_bwd", t["mu"], t["log_std"], t["value"], t["actions"],
                                     t["old_logp"], t["adv"], t["ret"], s["B"], s["D"], s.get("Bt", s["B"]), 0.2, 0.5, 0.01,
                                     0, t["dmu"], t["dlog_std"], t["dvalue"], t["stats"], t["scratch"], t["ws"],
                                     t["ws"].numel())


@case("xb_ppg_aux_loss_fwd_bwd", [dict(B=1, A=1, aux=1), dict(B=257, A=19, aux=1, Bt=700), dict(B=BIG, A=4, aux=0),
                                  dict(B=65, A=64, aux=1, critic_only=1)])
def _():
    def build(s, rng):
        B, A = s["B"], s["A"]
        co = s.get("critic_only", 0)
        return dict(logits=None if co else IN(rng.normal(size=(B, A)).astype(f32)),
                    old=None if co else IN(rng.normal(size=(B, A)).astype(f32)), value=IN(rng.normal(size=B).astype(f32)),
                    aux=IN(rng.normal(size=B).astype(f32)) if s["aux"] else None, ret=IN(rng.normal(size=B).astype(f32)),
                    dlogits=None if co else OUT(B, A), dvalue=OUT(B), daux=OUT(B) if s["aux"] else None, stats=OUT(8),
                    scratch=SCRATCH())
    return build, lambda t, s: _call("xb_ppg_aux_loss_fwd_bwd", t["logits"], t["old"], t["value"], t["aux"], t["ret"], s["B"],
                                     s["A"], s.get("Bt", s["B"]), 1.0, t["dlogits"], t["dvalue"], t["daux"], t["stats"],
                                     t["scratch"])


@case("xb_ppg_aux_gauss_loss_fwd_bwd", [dict(B=1, D=1), dict(B=257, D=7, Bt=300), dict(B=33, D=64)])
def _():
    def build(s, rng):
        B, D = s["B"], s["D"]
        r = lambda *sh: rng.normal(size=sh).astype(f32)
        return dict(mu=IN(r(B, D)), log_std=IN(r(D) * 0.3), old_mu=IN(r(B, D)), old_log_std=IN(r(D) * 0.3), value=IN(r(B)),
                    aux=IN(r(B)), ret=IN(r(B)), dmu=OUT(B, D), dlog_std=OUT(D), dvalue=OUT(B), daux=OUT(B), stats=OUT(8),
                    scratch=SCRATCH())
    return build, lambda t, s: _call("xb_ppg_aux_gauss_loss_fwd_bwd", t["mu"], t["log_std"], t["old_mu"], t["old_log_std"],
                                     t["value"], t["aux"], t["ret"], s["B"], s["D"], s.get("Bt", s["B"]), 1.0, t["dmu"],
                                     t["dlog_std"], t["dvalue"], t["daux"], t["stats"], t["scratch"])


@case("xb_npg_loss_fwd_bwd", [dict(B=1, A=1), dict(B=257, A=33), dict(B=BIG, A=4), dict(B=20, A=64)])
def _():
    def build(s, rng):
        B, A = s["B"], s["A"]
        return dict(logits=IN(rng.normal(size=(B, A)).astype(f32)), value=IN(rng.normal(size=B).astype(f32)),
                    actions=IN(rng.integers(0, A, B).astype(f32)), adv=IN(rng.normal(size=B).astype(f32)),
                    ret=IN(rng.normal(size=B).astype(f32)), dlogits=OUT(B, A), dscore=OUT(B, A), dvalue=OUT(B),
                    stats=OUT(8), logp_sum=OUT(1, dtype=torch.float64), scratch=SCRATCH())
    return build, lambda t, s: _call("xb_npg_loss_fwd_bwd", t["logits"], t["value"], t["actions"], t["adv"], t["ret"], s["B"],
                                     s["A"], t["dlogits"], t["dscore"], t["dvalue"], t["stats"], t["logp_sum"], t["scratch"])


@case("xb_npg_gauss_loss_fwd_bwd", [dict(B=1, D=1), dict(B=257, D=5), dict(B=BIG, D=2), dict(B=17, D=64)])
def _():
    def build(s, rng):
        B, D = s["B"], s["D"]
        x = _gauss_batch(rng, B, D)
        ws = 2 * D * min((B + 7) // 8, 2048)
        return dict(**{k: IN(v) for k, v in x.items()}, dmu=OUT(B, D), dlog_std=OUT(D), smu=OUT(B, D), slog_std=OUT(D),
                    dvalue=OUT(B), stats=OUT(8), logp_sum=OUT(1, dtype=torch.float64), scratch=SCRATCH(),
                    ws=Op("scratch", (ws,), torch.float64))
    return build, lambda t, s: _call("xb_npg_gauss_loss_fwd_bwd", t["mu"], t["log_std"], t["value"], t["actions"], t["adv"],
                                     t["ret"], s["B"], s["D"], t["dmu"], t["dlog_std"], t["smu"], t["slog_std"], t["dvalue"],
                                     t["stats"], t["logp_sum"], t["scratch"], t["ws"], t["ws"].numel())


def _npg_table(lengths):
    from xuance_b200 import _lib
    import ctypes
    offs = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int64)
    ln = np.asarray(lengths, np.int64)
    table = np.zeros(3 * len(ln), np.int64)
    nch = _lib.load().xb_npg_segment_table(offs.ctypes.data_as(ctypes.c_void_p), ln.ctypes.data_as(ctypes.c_void_p),
                                           len(ln), table.ctypes.data_as(ctypes.c_void_p))
    return table, int(nch)


NPG_SEGMENTS = {1: [1], 2: [4097, 3, 8191], 3: [4096, 4096 * 3 + 1]}


@case("xb_npg_natural_grad", [dict(seg=1), dict(seg=2), dict(seg=3)])
def _():
    def build(s, rng):
        ln = NPG_SEGMENTS[s["seg"]]
        table, nch = _npg_table(ln)
        n = sum(ln)
        return dict(g=INOUT(rng.normal(size=n).astype(f32)), s=IN(rng.normal(size=n).astype(f32)),
                    table=IN(table, legal=0), logp_sum=IN(np.array([-3.0])), ws=Op("scratch", (2 * nch,), torch.float64))
    return build, lambda t, s: _call("xb_npg_natural_grad", t["g"], t["s"], t["table"], len(NPG_SEGMENTS[s["seg"]]),
                                     t["ws"].numel() // 2, t["logp_sum"], 10.0, 0.1, t["ws"], t["ws"].numel())


# ================================================================================================ K4M / K4V / K4C
def _masked_rows(rng, R, A, ld):
    av = (rng.random((R, A)) < 0.7).astype(np.uint8)
    act = np.array([rng.choice(np.flatnonzero(r)) if r.any() else 0 for r in av], f32) if ld else \
        rng.integers(0, A, R).astype(f32)
    if ld:
        av[np.arange(R), act.astype(np.int64)] = 1
    return av, act


@case("xb_mappo_prepare", [dict(R=1), dict(R=257), dict(R=BIG)])
def _():
    return (lambda s, rng: dict(mask=IN((rng.random(s["R"]) < 0.8).astype(f32)), ret=IN(rng.normal(size=s["R"]).astype(f32)),
                                block=OUT(4, dtype=torch.float64), scratch=SCRATCH()),
            lambda t, s: _call("xb_mappo_prepare", t["mask"], t["ret"], s["R"], t["block"], t["scratch"]))


@case("xb_value_norm_update", [dict(R=1), dict(R=1000)])
def _():
    return (lambda s, rng: dict(rm=INOUT(np.array([0.2], f32)), rmsq=INOUT(np.array([1.3], f32)), dt=INOUT(np.array([0.7], f32)),
                                block=IN(np.array([s["R"] * 0.8, 3.0, 900.0, 0.0])), mean_std=OUT(2)),
            lambda t, s: _call("xb_value_norm_update", t["rm"], t["rmsq"], t["dt"], t["block"], s["R"], 0.99999,
                               t["mean_std"]))


def _mappo_like_build(s, rng, R, with_old=True):
    A, ld = s["A"], s.get("ld", 0)
    av, act = _masked_rows(rng, R, A, ld)
    mask = (rng.random(R) < 0.8).astype(f32)
    return dict(logits=IN(rng.normal(size=(R, A)).astype(f32)), avail=IN(av, ld=ld) if ld else None, actions=IN(act),
                mask=IN(mask), prep=IN(np.array([max(mask.sum(), 1.0), 0, 0, 0])))


@case("xb_mappo_loss_fwd_bwd", [dict(R=1, A=1, ld=0), dict(R=257, A=19, ld=23, Rt=500), dict(R=BIG, A=5, ld=0),
                                dict(R=65, A=64, ld=67)])
def _():
    def build(s, rng):
        R, A = s["R"], s["A"]
        ops = _mappo_like_build(s, rng, R)
        r = lambda: rng.normal(size=R).astype(f32)
        ops.update(old_logp=IN(r() - 2), adv=IN(r()), value=IN(r()), old_value=IN(r()), ret=IN(r()),
                   vn=IN(np.array([0.1, 1.2], f32)), dlogits=OUT(R, A), dvalue=OUT(R), stats=OUT(8), scratch=SCRATCH())
        return ops
    return build, lambda t, s: _call("xb_mappo_loss_fwd_bwd", t["logits"], t["avail"], s["ld"], t["actions"], t["old_logp"],
                                     t["adv"], t["value"], t["old_value"], t["ret"], t["mask"], t["vn"], t["prep"], s["R"],
                                     s["A"], s.get("Rt", s["R"]), 0.2, 0.2, 10.0, 0.5, 0.01, t["dlogits"], t["dvalue"],
                                     t["stats"], t["scratch"])


@case("xb_vdac_loss_fwd_bwd", [dict(B=1, n=1, T=1, A=1, mode=0, order=0, ld=0), dict(B=3, n=5, T=7, A=9, mode=1, order=1, ld=11),
                               dict(B=4, n=32, T=3, A=64, mode=2, order=0, ld=0), dict(B=2, n=3, T=5, A=33, mode=2, order=1, ld=35)])
def _():
    def build(s, rng):
        B, n, T, A = s["B"], s["n"], s["T"], s["A"]
        R = B * n * T
        ops = _mappo_like_build(s, rng, R)
        nv = B * T if s["mode"] == 2 else R
        r = lambda k: rng.normal(size=k).astype(f32)
        # old_value is per row in every mix mode (the clipped term pairs it with the row's prediction)
        ops.update(adv=IN(r(R)), value=IN(r(nv)), old_value=IN(r(R)), ret=IN(r(R)), vn=None, dlogits=OUT(R, A),
                   dvalue=OUT(nv), stats=OUT(8), scratch=SCRATCH())
        return ops
    return build, lambda t, s: _call("xb_vdac_loss_fwd_bwd", t["logits"], t["avail"], s["ld"], t["actions"], t["adv"],
                                     t["value"], t["old_value"], t["ret"], t["mask"], t["vn"], t["prep"],
                                     s["B"] * s["n"] * s["T"], s["A"], s["n"], s["T"], s["mode"], s["order"],
                                     s["B"] * s["n"] * s["T"], 0.2, 0.0, 0.5, 0.01, t["dlogits"], t["dvalue"], t["stats"],
                                     t["scratch"])


@case("xb_coma_critic_input", [dict(B=1, n=1, T=1, S=1, F=1, A=1), dict(B=3, n=5, T=7, S=13, F=6, A=9),
                               dict(B=2, n=32, T=2, S=5, F=3, A=64)])
def _():
    def build(s, rng):
        B, n, T, S, F, A = (s[k] for k in "BnTSFA")
        R = B * n * T
        return dict(state=IN(rng.normal(size=(B, T, S)).astype(f32)), feat=IN(rng.normal(size=(R, F)).astype(f32)),
                    actions=IN(rng.integers(0, A, (B, n, T)).astype(f32)), out=OUT(R, S + F + n * A))
    return build, lambda t, s: _call("xb_coma_critic_input", t["state"], t["feat"], t["actions"], s["B"], s["n"], s["T"],
                                     s["S"], s["F"], s["A"], t["out"])


@case("xb_coma_loss_fwd_bwd", [dict(R=1, A=1, ld=0), dict(R=257, A=33, ld=37, Rt=300), dict(R=BIG, A=5, ld=0),
                               dict(R=40, A=64, ld=64)])
def _():
    def build(s, rng):
        R, A = s["R"], s["A"]
        ops = _mappo_like_build(s, rng, R)
        ops.update(q=IN(rng.normal(size=(R, A)).astype(f32)), ret=IN(rng.normal(size=R).astype(f32)),
                   eps=IN(np.array([0.05], f32)), dlogits=OUT(R, A), dq=OUT(R, A), stats=OUT(8), scratch=SCRATCH())
        return ops
    return build, lambda t, s: _call("xb_coma_loss_fwd_bwd", t["logits"], t["avail"], s["ld"], t["q"], t["actions"], t["ret"],
                                     t["mask"], t["eps"], t["prep"], s["R"], s["A"], s.get("Rt", s["R"]), t["dlogits"],
                                     t["dq"], t["stats"], t["scratch"])


@case("xb_coma_act", [dict(N=1, A=1, ld=0, eps=0, u=0), dict(N=257, A=33, ld=35, eps=1, u=1), dict(N=9, A=64, ld=0, eps=1, u=0)])
def _():
    def build(s, rng):
        N, A, ld = s["N"], s["A"], s["ld"]
        av, _ = _masked_rows(rng, N, A, ld)
        return dict(logits=IN(rng.normal(size=(N, A)).astype(f32)), avail=IN(av, ld=ld) if ld else None,
                    eps=IN(np.array([0.1], f32)) if s["eps"] else None, u=IN(rng.random(N).astype(f32)) if s["u"] else None,
                    a_f=OUT(N), a_i=OUT(N, dtype=torch.int32), logp=OUT(N))
    return build, lambda t, s: _call("xb_coma_act", t["logits"], t["avail"], s["ld"], t["eps"], t["u"], s["N"], s["A"],
                                     t["a_f"], t["a_i"], t["logp"])


# ================================================================================================ K5 PER trees
def _trees(rng, N, cap, size):
    leaves = np.zeros((N, cap), f32)
    leaves[:, :size] = (rng.random((N, size)) + 0.05).astype(f32)
    st, mt = np.zeros((N, 2 * cap), f32), np.full((N, 2 * cap), np.inf, f32)
    st[:, cap:], mt[:, cap:size + cap] = leaves, leaves[:, :size]
    for i in range(cap - 1, 0, -1):
        st[:, i] = st[:, 2 * i] + st[:, 2 * i + 1]
        mt[:, i] = np.minimum(mt[:, 2 * i], mt[:, 2 * i + 1])
    return st, mt


PER_SHAPES = [dict(N=1, cap=1, size=1, k=1), dict(N=3, cap=64, size=40, k=33), dict(N=2, cap=1024, size=1024, k=257)]


@case("xb_per_insert", PER_SHAPES)
def _():
    def build(s, rng):
        st, mt = _trees(rng, s["N"], s["cap"], s["size"])
        return dict(st=INOUT(st), mt=INOUT(mt), mp=INOUT((rng.random(s["N"]) + 0.5).astype(f32)))
    return build, lambda t, s: _call("xb_per_insert", t["st"], t["mt"], t["mp"], s["N"], s["cap"], s["size"] - 1, 0.6)


@case("xb_per_sample", PER_SHAPES)
def _():
    def build(s, rng):
        N, k = s["N"], s["k"]
        st, mt = _trees(rng, N, s["cap"], s["size"])
        return dict(st=IN(st), mt=IN(mt), u=IN(rng.random((N, k)).astype(f32)), step=OUT(N, k, dtype=torch.int64),
                    flat=OUT(N * k, dtype=torch.int64), w=OUT(N, k, dtype=torch.float64))
    return build, lambda t, s: _call("xb_per_sample", t["st"], t["mt"], t["u"], s["N"], s["cap"], s["size"], s["k"],
                                     s["cap"], float(f32(s["size"]) ** f32(-0.4)), t["step"], t["flat"], t["w"])


@case("xb_per_update", PER_SHAPES)
def _():
    def build(s, rng):
        N, k = s["N"], s["k"]
        st, mt = _trees(rng, N, s["cap"], s["size"])
        prio = (rng.random((N, k)) * 2).astype(f32)
        prio[:, 0] = 0.0
        return dict(st=INOUT(st), mt=INOUT(mt), mp=INOUT((rng.random(N) + 0.5).astype(f32)),
                    idx=IN(rng.integers(0, s["size"], (N, k)).astype(np.int64)), prio=IN(prio))
    return build, lambda t, s: _call("xb_per_update", t["st"], t["mt"], t["mp"], t["idx"], t["prio"], s["N"], s["cap"], s["k"],
                                     0.6)


# ================================================================================================ K6Z C51 / QR-DQN
DIST_SHAPES = [dict(B=1, A=1, N=2), dict(B=257, A=7, N=51, Bt=400), dict(B=33, A=256, N=64), dict(B=65, A=3, N=33)]


def _dist_in(s, rng, c51):
    B, A, N = s["B"], s["A"], s["N"]
    ops = dict(z=IN(rng.normal(size=(B, A, N)).astype(f32)), zn=IN(rng.normal(size=(B, A, N)).astype(f32)),
               actions=IN(rng.integers(0, A, B).astype(f32)), rew=IN(rng.normal(size=B).astype(f32)),
               ter=IN((rng.random(B) < 0.3).astype(f32)), tact=OUT(B, dtype=torch.int64), stats=OUT(4), scratch=SCRATCH())
    if c51:
        ops["sup"] = IN(np.linspace(-10, 10, N).astype(f32))
    return ops


@case("xb_dist_greedy", [dict(B=1, A=1, N=2, c51=1), dict(B=257, A=7, N=51, c51=1), dict(B=33, A=256, N=64, c51=0),
                         dict(B=65, A=3, N=33, c51=0)])
def _():
    def build(s, rng):
        B, A, N, c = s["B"], s["A"], s["N"], s["c51"]
        return dict(z=IN(rng.normal(size=(B, A, N)).astype(f32)), sup=IN(np.linspace(-10, 10, N).astype(f32)) if c else None,
                    act=OUT(B, dtype=torch.int64), q=OUT(B, A), probs=OUT(B, A, N) if c else None)
    return build, lambda t, s: _call("xb_dist_greedy", t["z"], t["sup"], s["B"], s["A"], s["N"], t["act"], t["q"], t["probs"])


@case("xb_c51_loss_fwd_bwd", DIST_SHAPES)
def _():
    def build(s, rng):
        ops = _dist_in(s, rng, True)
        ops.update(dz=OUT(s["B"], s["A"], s["N"]), tdist=OUT(s["B"], s["N"]) if s["A"] != 3 else None)
        return ops
    return build, lambda t, s: _call("xb_c51_loss_fwd_bwd", t["z"], t["zn"], t["sup"], t["actions"], t["rew"], t["ter"], s["B"],
                                     s["A"], s["N"], s.get("Bt", s["B"]), 0.99, -10.0, 10.0, 20.0 / (s["N"] - 1), t["dz"],
                                     t["tact"], t["tdist"], t["stats"], t["scratch"])


@case("xb_qrdqn_loss_fwd_bwd", DIST_SHAPES)
def _():
    def build(s, rng):
        ops = _dist_in(s, rng, False)
        ops["dq"] = OUT(s["B"], s["A"], s["N"])
        return ops
    return build, lambda t, s: _call("xb_qrdqn_loss_fwd_bwd", t["z"], t["zn"], t["actions"], t["rew"], t["ter"], s["B"], s["A"],
                                     s["N"], s.get("Bt", s["B"]), 0.99, t["dq"], t["tact"], t["stats"], t["scratch"])


# ================================================================================================ K8D SAC-Discrete
SACDIS_SHAPES = [dict(B=1, A=1), dict(B=257, A=4), dict(B=257, A=5), dict(B=65, A=8), dict(B=65, A=9), dict(B=65, A=18),
                 dict(B=65, A=19), dict(B=65, A=32), dict(B=65, A=33, Bt=100), dict(B=BIG, A=64)]


@case("xb_sacdis_actor_loss", SACDIS_SHAPES)
def _():
    def build(s, rng):
        B, A = s["B"], s["A"]
        r = lambda: rng.normal(size=(B, A)).astype(f32)
        return dict(logits=IN(r()), q1=IN(r()), q2=IN(r()), alpha=IN(np.array([0.2], f32)), dz=OUT(B, A), stats=OUT(4),
                    scratch=SCRATCH())
    return build, lambda t, s: _call("xb_sacdis_actor_loss", t["logits"], t["q1"], t["q2"], t["alpha"], s["B"], s["A"],
                                     s.get("Bt", s["B"]), t["dz"], t["stats"], t["scratch"])


@case("xb_sacdis_critic_loss", SACDIS_SHAPES)
def _():
    def build(s, rng):
        B, A = s["B"], s["A"]
        r = lambda: rng.normal(size=(B, A)).astype(f32)
        return dict(q1=IN(r()), q2=IN(r()), actions=IN(rng.integers(0, A, B).astype(f32)), ln=IN(r()), tq1=IN(r()), tq2=IN(r()),
                    rew=IN(rng.normal(size=B).astype(f32)), term=IN((rng.random(B) < 0.3).astype(f32)),
                    alpha=IN(np.array([0.2], f32)), dq1=OUT(B, A), dq2=OUT(B, A), backup=OUT(B), stats=OUT(2),
                    scratch=SCRATCH())
    return build, lambda t, s: _call("xb_sacdis_critic_loss", t["q1"], t["q2"], t["actions"], t["ln"], t["tq1"], t["tq2"],
                                     t["rew"], t["term"], t["alpha"], 0.99, s["B"], s["A"], s.get("Bt", s["B"]), t["dq1"],
                                     t["dq2"], t["backup"], t["stats"], t["scratch"])


# ================================================================================================ K9 mixer / TD / K9-TC
MIX_SHAPES = [dict(R=1, n=1, H=32), dict(R=257, n=5, H=48), dict(R=33, n=16, H=64), dict(R=65, n=9, H=32, align=4)]


def _mix_in(s, rng):
    R, n, H = s["R"], s["n"], s["H"]
    return dict(q=IN((rng.normal(size=(R, n)) * 2).astype(f32)),
                w1=IN((rng.normal(size=(R, n * H)) / np.sqrt(n)).astype(f32), mis=True),
                b1=IN(rng.normal(size=(R, H)).astype(f32)), w2=IN((rng.normal(size=(R, H)) / np.sqrt(H)).astype(f32)))


@case("xb_qmix_mix_fwd", MIX_SHAPES)
def _():
    def build(s, rng):
        return dict(**_mix_in(s, rng), b2=IN(rng.normal(size=s["R"]).astype(f32)), q_tot=OUT(s["R"]))
    return build, lambda t, s: _call("xb_qmix_mix_fwd", t["q"], t["w1"], t["b1"], t["w2"], t["b2"], s["R"], s["n"], s["H"],
                                     t["q_tot"])


@case("xb_qmix_mix_bwd", MIX_SHAPES)
def _():
    def build(s, rng):
        R, n, H = s["R"], s["n"], s["H"]
        return dict(g=IN(rng.normal(size=R).astype(f32)), **_mix_in(s, rng), dq=OUT(R, n), dw1=OUT(R, n * H), db1=OUT(R, H),
                    dw2=OUT(R, H))
    return build, lambda t, s: _call("xb_qmix_mix_bwd", t["g"], t["q"], t["w1"], t["b1"], t["w2"], s["R"], s["n"], s["H"],
                                     t["dq"], t["dw1"], t["db1"], t["dw2"])


def _qmix_td_values(got, x, s):
    import test_gpu_kernel_edges as ke
    xx = dict(q_tot=x["q_tot"], q_tot_next=x["q_next"], rewards=x["rew"], terminals=x["term"], filled=x["filled"])
    ke._check_qmix_td((got["dq"], got["stats"]), xx)
    return {"checked": 0.0}


@case("xb_qmix_td", [dict(B=1, n=1, T=1), dict(B=24, n=5, T=13), dict(B=3, n=16, T=100)], _qmix_td_values)
def _():
    def build(s, rng):
        import test_gpu_kernel_edges as ke
        B, n, T = s["B"], s["n"], s["T"]
        x = ke._qmix_td_inputs(B, n, T, seed=B + n + T)
        fs = np.array([x["filled"].sum()], f32)
        return dict(q_tot=IN(x["q_tot"]), q_next=IN(x["q_tot_next"]), rew=IN(x["rewards"]), term=IN(x["terminals"]),
                    filled=IN(x["filled"]), fs=IN(fs), dq=OUT(B * T), stats=OUT(2), scratch=SCRATCH())
    return build, lambda t, s: _call("xb_qmix_td", t["q_tot"], t["q_next"], t["rew"], t["term"], t["filled"], t["fs"], s["B"],
                                     s["n"], s["T"], 0.99, s["B"] * s["T"], t["dq"], t["stats"], t["scratch"])


# S = 97 (the shipped configs' 97-float state rows; smaller S is XB_ERANGE): R = 1, 65 and 129 rows are the staged tails
@case("xb_qmix_mix_fused_fwd", [dict(R=1, S=97, n=1), dict(R=65, S=97, n=8), dict(R=129, S=97, n=5), dict(R=2240, S=97, n=8)])
def _():
    def build(s, rng):
        R, S, n = s["R"], s["S"], s["n"]
        w = lambda *sh: (rng.normal(size=sh) / np.sqrt(sh[-1])).astype(f32)
        ops = dict(states=IN(rng.normal(size=(R, S)).astype(f32)), q=IN(rng.normal(size=(R, n)).astype(f32)))
        for i in range(4):
            ops[f"w{i}"], ops[f"b{i}"] = IN(w(32, S)), IN(w(32))
        ops.update(wb1=IN(w(n * 32, 32)), bwb1=IN(w(n * 32)), wb2=IN(w(32, 32)), bwb2=IN(w(32)), wb2c=IN(w(1, 32)),
                   bwb2c=IN(w(1)), q_tot=OUT(R))
        return ops

    def launch(t, s):
        import ctypes
        L = _lib()
        wp = (ctypes.c_void_p * 4)(*[L.ptr(t[f"w{i}"]) for i in range(4)])
        bp = (ctypes.c_void_p * 4)(*[L.ptr(t[f"b{i}"]) for i in range(4)])
        _call("xb_qmix_mix_fused_fwd", t["states"], t["q"], wp, bp, t["wb1"], t["bwb1"], t["wb2"], t["bwb2"], t["wb2c"],
              t["bwb2c"], s["R"], s["S"], s["n"], 32, 32, t["q_tot"])
    return build, launch


# ================================================================================================ K9W / K9I / K9Q episode heads
def _episode(s, rng, heads=("q_all",)):
    """Heads [B,n,T+1,A], actions / agent_mask [B,n,T], filled [B,T] and, with ld > 0, avail [B,n,T+1,ld] whose taken
    actions are available."""
    B, n, T, A, ld = s["B"], s["n"], s["T"], s["A"], s.get("ld", 0)
    ops = {h: IN(rng.integers(-2, 3, (B, n, T + 1, A)).astype(f32) + (rng.normal(size=(B, n, T + 1, A)) * 0.1).astype(f32))
           for h in heads}
    act = rng.integers(0, A, (B, n, T))
    av = (rng.random((B, n, T + 1, A)) < 0.6).astype(np.uint8)
    av[..., 0] = 1
    av[:, :, :T][np.arange(B)[:, None, None], np.arange(n)[None, :, None], np.arange(T)[None, None, :], act] = 1
    ops.update(actions=IN(act.astype(f32)), agent_mask=IN((rng.random((B, n, T)) < 0.8).astype(f32)),
               filled=IN((rng.random((B, T)) < 0.8).astype(f32)), avail=IN(av, ld=ld) if ld else None)
    return ops


EP_SHAPES = [dict(B=1, n=1, T=1, A=1, ld=0, dq=0), dict(B=3, n=5, T=7, A=6, ld=9, dq=1), dict(B=4, n=16, T=20, A=19, ld=0, dq=0),
             dict(B=2, n=9, T=40, A=33, ld=35, dq=1)]


@case("xb_wqmix_select_fwd", EP_SHAPES)
def _():
    def build(s, rng):
        B, n, T = s["B"], s["n"], s["T"]
        ops = _episode(s, rng, ("q_all", "q_cent", "q_cent_tgt", "q_tgt"))
        if s["dq"]:
            ops["q_tgt"] = None
        ops.update(qe=OUT(B * T, n), qc=OUT(B * T, n), qnc=OUT(B * T, n), greedy=OUT(B, n, T, dtype=torch.int32),
                   agree=OUT(B * T, dtype=torch.uint8), fs=OUT(1), scratch=SCRATCH())
        return ops
    return build, lambda t, s: _call("xb_wqmix_select_fwd", t["q_all"], t["q_cent"], t["q_cent_tgt"], t["q_tgt"], t["actions"],
                                     t["agent_mask"], t["filled"], t["avail"], s["ld"], s["B"], s["n"], s["T"], s["A"], s["dq"],
                                     t["qe"], t["qc"], t["qnc"], t["greedy"], t["agree"], t["fs"], t["scratch"])


@case("xb_wqmix_select_bwd", [dict(B=1, n=1, T=1, A=1, both=1), dict(B=3, n=5, T=7, A=6, both=1), dict(B=4, n=16, T=20, A=19, both=0)])
def _():
    def build(s, rng):
        B, n, T, A = s["B"], s["n"], s["T"], s["A"]
        ops = _episode(s, rng, ())
        ops.update(d_eval=IN(rng.normal(size=(B * T, n)).astype(f32)),
                   d_cent=IN(rng.normal(size=(B * T, n)).astype(f32)) if s["both"] else None,
                   greedy=IN(rng.integers(0, A, (B, n, T)).astype(np.int32)), dq_all=OUT(B, n, T + 1, A, role="out_scatter"),
                   dq_cent=OUT(B, n, T + 1, A, role="out_scatter") if s["both"] else None)
        return ops
    return build, lambda t, s: _call("xb_wqmix_select_bwd", t["d_eval"], t["d_cent"], t["actions"], t["greedy"], t["agent_mask"],
                                     t["filled"], s["B"], s["n"], s["T"], s["A"], t["dq_all"], t["dq_cent"])


@case("xb_wqmix_loss_fwd_bwd", [dict(B=1, n=1, T=1, mode=0), dict(B=24, n=5, T=13, mode=1), dict(B=3, n=16, T=100, mode=0)])
def _():
    def build(s, rng):
        B, n, T = s["B"], s["n"], s["T"]
        r = lambda *sh: rng.normal(size=sh).astype(f32)
        filled = (rng.random((B, T)) < 0.8).astype(f32)
        return dict(q_tot=IN(r(B * T)), q_ff=IN(r(B * T)), q_ff_next=IN(r(B * T)), rew=IN(r(B, n, T)),
                    term=IN((rng.random((B, n, T)) < 0.3).astype(f32)), filled=IN(filled),
                    agree=IN((rng.random(B * T) < 0.5).astype(np.uint8)), fs=IN(np.array([max(filled.sum(), 1)], f32)),
                    dq_tot=OUT(B * T), dq_ff=OUT(B * T), stats=OUT(4), scratch=SCRATCH())
    return build, lambda t, s: _call("xb_wqmix_loss_fwd_bwd", t["q_tot"], t["q_ff"], t["q_ff_next"], t["rew"], t["term"],
                                     t["filled"], t["agree"], t["fs"], s["B"], s["n"], s["T"], s["mode"], 0.1, 0.99,
                                     s["B"] * s["T"], t["dq_tot"], t["dq_ff"], t["stats"], t["scratch"])


@case("xb_iql_prepare", [dict(B=1, n=1, T=1), dict(B=3, n=5, T=7), dict(B=64, n=32, T=129)])
def _():
    def build(s, rng):
        B, n, T = s["B"], s["n"], s["T"]
        return dict(agent_mask=IN((rng.random((B, n, T)) < 0.8).astype(f32)), filled=IN((rng.random((B, T)) < 0.8).astype(f32)),
                    msum=OUT(1, dtype=torch.float64), scratch=SCRATCH())
    return build, lambda t, s: _call("xb_iql_prepare", t["agent_mask"], t["filled"], s["B"], s["n"], s["T"], t["msum"],
                                     t["scratch"])


@case("xb_iql_td_fwd_bwd", EP_SHAPES + [dict(B=2, n=32, T=70, A=64, ld=64, dq=1, Rt=10000)])
def _():
    def build(s, rng):
        B, n, T, A = s["B"], s["n"], s["T"], s["A"]
        ops = _episode(s, rng, ("q_all", "q_tgt"))
        opt = s["dq"]
        ops.update(rew=IN(rng.normal(size=(B, n, T)).astype(f32)), term=IN((rng.random((B, n, T)) < 0.3).astype(f32)),
                   msum=IN(np.array([max(float(ops["agent_mask"].data.sum()), 1.0)])),
                   dq_all=OUT(B, n, T + 1, A), stats=OUT(2), scratch=SCRATCH(),
                   nxt=OUT(B, n, T, dtype=torch.int32) if opt else None, qn=OUT(B, n, T) if opt else None,
                   tgt=OUT(B, n, T) if opt else None)
        return ops
    return build, lambda t, s: _call("xb_iql_td_fwd_bwd", t["q_all"], t["q_tgt"], t["actions"], t["rew"], t["term"],
                                     t["agent_mask"], t["filled"], t["avail"], s["ld"] or s["A"], t["msum"], s["B"], s["n"],
                                     s["T"], s["A"], s["dq"], 0.99, s.get("Rt", s["B"] * s["n"] * s["T"]), t["dq_all"],
                                     t["stats"], t["scratch"], t["nxt"], t["qn"], t["tgt"])


@case("xb_qtran_select", EP_SHAPES)
def _():
    def build(s, rng):
        B, n, T = s["B"], s["n"], s["T"]
        ops = _episode(s, rng, ("q_all", "q_tgt"))
        if s["dq"]:
            ops["q_tgt"] = None
        ops.update(greedy=OUT(B, n, T + 1, dtype=torch.int32), nxt=OUT(B, n, T, dtype=torch.int32), fs=OUT(1),
                   scratch=SCRATCH())
        return ops
    return build, lambda t, s: _call("xb_qtran_select", t["q_all"], t["q_tgt"], t["avail"], s["ld"], t["filled"], s["B"],
                                     s["n"], s["T"], s["A"], s["dq"], t["greedy"], t["nxt"], t["fs"], t["scratch"])


QTRAN_ENC = [dict(mode=0, B=1, n=1, T=1, S=1, H=1, A=1, t0=0, ai=0), dict(mode=1, B=3, n=5, T=7, S=13, H=33, A=6, t0=1, ai=1),
             dict(mode=0, B=2, n=8, T=5, S=9, H=64, A=19, t0=1, ai=0), dict(mode=1, B=2, n=3, T=4, S=5, H=17, A=64, t0=0, ai=0)]


def _qtran_enc_in(s, rng):
    B, n, T, S, H, A = (s[k] for k in "BnTSHA")
    D = H + A
    act = rng.integers(0, A, (B, n, T + 1))
    w = lambda *sh: (rng.normal(size=sh) / np.sqrt(D)).astype(f32)
    return dict(h=IN(rng.normal(size=(B, n, T + 1, H)).astype(f32)), agent_mask=IN((rng.random((B, n, T)) < 0.8).astype(f32)),
                act_f=None if s["ai"] else IN(act.astype(f32)), act_i=IN(act.astype(np.int32)) if s["ai"] else None,
                w1=IN(w(D, D)), b1=IN(w(D)), w2=IN(w(D, D)), b2=IN(w(D)))


def _qtran_width(s):
    D = s["H"] + s["A"]
    R = s["B"] * s["T"]
    return (R, s["S"] + D) if s["mode"] == 0 else (R * s["n"], s["S"] + D + s["n"])


@case("xb_qtran_encode_fwd", QTRAN_ENC)
def _():
    def build(s, rng):
        ops = _qtran_enc_in(s, rng)
        R, D = s["B"] * s["T"], s["H"] + s["A"]
        ops.update(state=IN(rng.normal(size=(s["B"], s["T"] + 1, s["S"])).astype(f32)), x=OUT(*_qtran_width(s)),
                   pre=OUT(R, s["n"], D) if s["mode"] == 0 else None)
        return ops
    return build, lambda t, s: _call("xb_qtran_encode_fwd", s["mode"], t["state"], s["t0"], t["h"], t["agent_mask"], t["act_f"],
                                     t["act_i"], s["T"] + 1, t["w1"], t["b1"], t["w2"], t["b2"], s["B"], s["n"], s["T"], s["S"],
                                     s["H"], s["A"], t["x"], t["pre"])


@case("xb_qtran_encode_bwd", QTRAN_ENC)
def _():
    def build(s, rng):
        ops = _qtran_enc_in(s, rng)
        B, n, T, H, A = (s[k] for k in "BnTHA")
        D = H + A
        work = int(_lib().load().xb_qtran_encode_bwd_work(B, n, T, H, A))
        ops.update(dx=IN(rng.normal(size=_qtran_width(s)).astype(f32)),
                   pre=IN(rng.normal(size=(B * T, n, D)).astype(f32)), dh=OUT(B, n, T + 1, H), dw1=OUT(D, D), db1=OUT(D),
                   dw2=OUT(D, D), db2=OUT(D), work=Op("scratch", (work,), torch.float32))
        return ops
    return build, lambda t, s: _call("xb_qtran_encode_bwd", s["mode"], t["dx"], t["h"], t["agent_mask"], t["act_f"], t["act_i"],
                                     s["T"] + 1, t["w1"], t["w2"], t["pre"], s["B"], s["n"], s["T"], s["S"], s["H"], s["A"],
                                     t["dh"], t["dw1"], t["db1"], t["dw2"], t["db2"], t["work"], t["work"].numel())


@case("xb_qtran_loss_fwd_bwd", [dict(mode=0, B=1, n=1, T=1, A=1), dict(mode=1, B=3, n=5, T=7, A=6),
                                dict(mode=0, B=4, n=16, T=20, A=33), dict(mode=1, B=2, n=9, T=4, A=64)])
def _():
    def build(s, rng):
        B, n, T, A = s["B"], s["n"], s["T"], s["A"]
        R = B * T
        ops = _episode(dict(s, ld=0), rng, ("q_all",))
        jt = (R,) if s["mode"] == 0 else (R * n, A)
        r = lambda *sh: rng.normal(size=sh).astype(f32)
        filled = ops["filled"].data
        ops.update(greedy=IN(rng.integers(0, A, (B, n, T + 1)).astype(np.int32)),
                   nxt=IN(rng.integers(0, A, (B, n, T)).astype(np.int32)), rew=IN(r(B, n, T)),
                   term=IN((rng.random((B, n, T)) < 0.3).astype(f32)), qjt=IN(r(*jt)), qjt_g=IN(r(*jt)), qjt_n=IN(r(*jt)),
                   v=IN(r(R)), fs=IN(np.array([max(filled.sum(), 1)], f32)), dqjt=OUT(*jt), dv=OUT(R),
                   dq_all=OUT(B, n, T + 1, A, role="out_scatter"), stats=OUT(5), scratch=SCRATCH())
        return ops
    return build, lambda t, s: _call("xb_qtran_loss_fwd_bwd", s["mode"], t["q_all"], t["actions"], t["greedy"], t["nxt"],
                                     t["agent_mask"], t["filled"], t["rew"], t["term"], t["qjt"], t["qjt_g"], t["qjt_n"], t["v"],
                                     t["fs"], s["B"], s["n"], s["T"], s["A"], 0.99, 1.0, 1.0, s["B"] * s["T"], t["dqjt"],
                                     t["dv"], t["dq_all"], t["stats"], t["scratch"])


# ================================================================================================ K9C DCG
def _edges(n, E):
    pairs = [(i, j) for i in range(n) for j in range(i + 1, n)][:E]
    return np.array([p[0] for p in pairs], np.int32), np.array([p[1] for p in pairs], np.int32)


# payoff orientations `gap` elements further apart than one orientation's extent: the gap is band
DCG_SHAPES = [dict(B=1, n=2, T=1, A=1, E=1, gap=0, ld=0), dict(B=3, n=5, T=4, A=6, E=10, gap=7, ld=9),
              dict(B=2, n=4, T=3, A=33, E=3, gap=5, ld=0), dict(B=2, n=3, T=2, A=5, E=0, gap=0, ld=7)]


def _pay(s, rng, T1):
    B, E, A = s["B"], s["E"], s["A"]
    ext = B * E * T1 * A * A
    return IN(rng.normal(size=(2, ext)).astype(f32), ld=ext + s["gap"]) if ext else IN(np.zeros((2, 1), f32)), ext + s["gap"]


@case("xb_dcg_greedy", DCG_SHAPES)
def _():
    def build(s, rng):
        B, n, T, A, E, ld = (s[k] for k in ("B", "n", "T", "A", "E", "ld"))
        fr, to = _edges(n, E)
        av = (rng.random((B, n, T + 1, A)) < 0.6).astype(np.uint8)
        av[..., 0] = 1
        return dict(f=IN(rng.normal(size=(B, n, T + 1, A)).astype(f32)), pay=_pay(s, rng, T + 1)[0],
                    fr=IN(fr if E else np.zeros(1, np.int32)), to=IN(to if E else np.zeros(1, np.int32)),
                    avail=IN(av, ld=ld) if ld else None, actions=OUT(B * T, n, dtype=torch.int32),
                    U=OUT(B * T, n, A, dtype=torch.float64))
    return build, lambda t, s: _call("xb_dcg_greedy", t["f"], t["pay"], t["pay"].stride(0), t["fr"], t["to"], t["avail"],
                                     s["ld"], s["B"], s["T"], s["T"] + 1, 1, s["n"], s["A"], s["E"], 4, 1, t["actions"], t["U"])


def _dcg_q_in(s, rng):
    B, n, T, A, E = (s[k] for k in "BnTAE")
    fr, to = _edges(n, E)
    return dict(actions=IN(rng.integers(0, A, (B, n, T)).astype(f32)), fr=IN(fr if E else np.zeros(1, np.int32)),
                to=IN(to if E else np.zeros(1, np.int32)))


@case("xb_dcg_q_fwd", DCG_SHAPES)
def _():
    def build(s, rng):
        B, n, T, A = (s[k] for k in "BnTA")
        ops = _dcg_q_in(s, rng)
        ops.update(fe=IN(rng.normal(size=(B, n, T + 1, A)).astype(f32)), pe=_pay(s, rng, T + 1)[0],
                   ft=IN(rng.normal(size=(B, n, T + 1, A)).astype(f32)), pt=_pay(s, rng, T + 1)[0],
                   greedy=IN(rng.integers(0, A, (B * T, n)).astype(np.int32)), filled=IN((rng.random((B, T)) < 0.8).astype(f32)),
                   qe=OUT(B * T, dtype=torch.float64), qn=OUT(B * T, dtype=torch.float64), fs=OUT(1), scratch=SCRATCH())
        return ops
    return build, lambda t, s: _call("xb_dcg_q_fwd", t["fe"], t["pe"], t["pe"].stride(0), t["ft"], t["pt"], t["pt"].stride(0),
                                     t["actions"], t["greedy"], t["filled"], t["fr"], t["to"], s["B"], s["n"], s["T"], s["A"],
                                     s["E"], int(s["E"] > 0), t["qe"], t["qn"], t["fs"], t["scratch"])


@case("xb_dcg_td_fwd_bwd", [dict(B=1, n=1, T=1, v=0), dict(B=24, n=5, T=13, v=1), dict(B=3, n=16, T=100, v=1)])
def _():
    def build(s, rng):
        B, n, T, v = s["B"], s["n"], s["T"], s["v"]
        filled = (rng.random((B, T)) < 0.8).astype(f32)
        r = lambda *sh: rng.normal(size=sh)
        return dict(qe=IN(r(B * T)), qn=IN(r(B * T)), v=IN(r(B * T).astype(f32)) if v else None,
                    vn=IN(r(B * T).astype(f32)) if v else None, rew=IN(r(B, n, T).astype(f32)),
                    term=IN((rng.random((B, n, T)) < 0.3).astype(f32)), filled=IN(filled),
                    fs=IN(np.array([max(filled.sum(), 1)], f32)), dq=OUT(B * T, dtype=torch.float64),
                    dv=OUT(B * T) if v else None, stats=OUT(2), scratch=SCRATCH())
    return build, lambda t, s: _call("xb_dcg_td_fwd_bwd", t["qe"], t["qn"], t["v"], t["vn"], t["rew"], t["term"], t["filled"],
                                     t["fs"], s["B"], s["n"], s["T"], 0.99, s["B"] * s["T"], t["dq"], t["dv"], t["stats"],
                                     t["scratch"])


@case("xb_dcg_q_bwd", DCG_SHAPES)
def _():
    def build(s, rng):
        B, n, T, A, E = (s[k] for k in "BnTAE")
        ops = _dcg_q_in(s, rng)
        ext = B * E * (T + 1) * A * A
        ops.update(dq=IN(rng.normal(size=B * T)), df=OUT(B, n, T + 1, A, role="out_scatter"),
                   dp=Op("out_scatter", (2, ext), torch.float32, ld=ext + s["gap"]) if E else None)
        return ops
    return build, lambda t, s: _call("xb_dcg_q_bwd", t["dq"], t["actions"], t["fr"], t["to"], s["B"], s["n"], s["T"], s["A"],
                                     s["E"], int(s["E"] > 0), t["df"], t["dp"], t["dp"].stride(0) if s["E"] else 0)
