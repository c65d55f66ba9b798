"""GPU: the ASSEMBLED K12 encoder (``BoxNatureCNN`` / ``TensorCoreNatureCNN`` behind ``compute="tc"``) against float64,
layer by layer and gradient by gradient, with the teacher-forced checker of tests/k12_encoder_refs.py (its docstring
derives the bounds): at the agents' batch sizes (1 .. 8192: PPO minibatch 8192, rollout 256, PER-DQN 512, C51 / QR-DQN 32),
on every documented path switch (XB_K12_HALO, XB_K12_BOX_WGRAD, XB_K12_BOX=0, XB_K12_TMA=0), with the padding of the
persistent padded buffers bitwise zero, gradients added into existing ``.grad`` tensors, inference calls in between,
bit-identical repeats, and inside CUDA graphs (the encoder alone, and PPO train_epochs with compute="tc")."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

import k12_encoder_refs as K
from xuance_b200.torch.utils import tc_conv as tc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _representation(planes=3, basic=False, seed=0):
    """AC_CNN_Atari's encoder as helpers.build_product_ppo_model builds it (orthogonal init), or Basic_CNN, on K12, with
    seeded non-zero biases (the product initialises them to zero, which would hide a bias applied in the wrong place)."""
    from helpers import build_product_ppo_model
    from xuance_b200.torch.rl_models import Basic_CNN
    torch.manual_seed(seed)
    if basic:
        rep = Basic_CNN(input_shape=(84, 84, 4), kernels=[8, 4, 3], strides=[4, 2, 1], filters=[32, 64, 64],
                        activation=nn.ReLU, device=DEV)
    else:
        rep = build_product_ppo_model(4, DEV).representation
    g = torch.Generator(device=DEV).manual_seed(seed + 100)
    with torch.no_grad():
        for m in rep.model:
            if isinstance(m, (nn.Conv2d, nn.Linear)):
                m.bias.copy_((torch.rand(m.bias.shape, device=DEV, generator=g) - 0.5) * 0.2)
    rep.tc_planes = planes
    rep.set_compute("tc")
    return rep


class _Spy:
    """Keeps the planes tc_encode received, its output and the gradient that reaches it (Basic_CNN pools after it)."""

    def __init__(self, monkeypatch):
        self.orig = tc.tc_encode
        monkeypatch.setattr(tc, "tc_encode", self)

    def __call__(self, enc, x_pl, B):
        z = self.orig(enc, x_pl, B)
        self.x_pl, self.B, self.z = x_pl, B, z.detach()
        z.register_hook(lambda g: setattr(self, "dz", g.detach().clone()))
        return z


def _obs(B, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(0, 256, (B, 84, 84, 4), dtype=torch.uint8, device=DEV, generator=g)


def _step(rep, spy, obs, seed):
    """One forward + backward through the representation with fresh gradients; returns them in enc.parameters() order."""
    enc = rep._tc
    for p in enc.parameters():
        p.grad = None
    z = rep(obs).embeddings
    R = torch.randn(z.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))
    (z * R).sum().backward()
    return [p.grad.clone() for p in enc.parameters()]


def _check(rep, spy, obs, seed=1, padding=True):
    grads = _step(rep, spy, obs, seed)
    enc = rep._tc
    ratios = K.check(enc, K.capture(enc, spy.B, spy.x_pl, spy.z, grads), spy.dz)
    if padding and isinstance(enc, tc.BoxNatureCNN):
        K.check_padding(enc, spy.B)
    return ratios


BATCHES = [1, 2, 37, 255, 256, 257, 1024, 2731, 8192]


@pytest.mark.parametrize("B", BATCHES)
def test_every_layer_and_gradient_against_float64(monkeypatch, B):
    """Three planes, the raw uint8 pixels as one plane (the production input, xb_gather_obs_planes); twice on different
    data so that stale values in the persistent buffers would show.  Prints the largest |error| / bound per tensor."""
    spy = _Spy(monkeypatch)
    rep = _representation(3)
    for i in range(2):
        ratios = _check(rep, spy, _obs(B, 10 * B + i), seed=B + i)
    assert isinstance(rep._tc, tc.BoxNatureCNN) and spy.x_pl.shape[0] == 1
    print("K12 encoder B=%d largest |error|/bound: %s" % (B, json.dumps({k: float("%.3g" % v) for k, v in ratios.items()})))


@pytest.mark.parametrize("B", [37, 257])
@pytest.mark.parametrize("planes,form", [(3, "split"), (2, "raw")])
def test_other_operand_forms(monkeypatch, B, planes, form):
    """Three planes of the split x/255 (float observations) and two planes (raw plane, the 2-plane bounds)."""
    spy = _Spy(monkeypatch)
    rep = _representation(planes)
    obs = _obs(B, 7 * B)
    _check(rep, spy, obs.float() if form == "split" else obs)
    assert spy.x_pl.shape[0] == (planes if form == "split" else 1)


@pytest.mark.parametrize("B", [32, 512])
def test_basic_cnn_pooled_encoder(monkeypatch, B):
    """Basic_CNN (the DQN family): conv3 writes the float32 output, amax pooling in _run_tc, the pooled gradient copied
    into conv3's padded output-gradient buffer."""
    spy = _Spy(monkeypatch)
    rep = _representation(3, basic=True)
    _check(rep, spy, _obs(B, 3 * B))
    assert rep._tc.fc is None and spy.z.shape == (B * 100, 64)


@pytest.mark.parametrize("B", [37, 257])
@pytest.mark.parametrize("box_wgrad", ["", "2", "3", "23"])
@pytest.mark.parametrize("halo", ["0", "2", "3"])
def test_path_switches(monkeypatch, halo, box_wgrad, B):
    """XB_K12_HALO x XB_K12_BOX_WGRAD (module globals read at call time)."""
    monkeypatch.setattr(tc, "HALO", halo != "0")
    monkeypatch.setattr(tc, "HALO3", halo == "3")
    monkeypatch.setattr(tc, "BOX_WGRAD2", "2" in box_wgrad)
    monkeypatch.setattr(tc, "BOX_WGRAD3", "3" in box_wgrad)
    spy = _Spy(monkeypatch)
    _check(_representation(3), spy, _obs(B, B + 5))


@pytest.mark.parametrize("basic", [False, True])
@pytest.mark.parametrize("B", [37, 257])
def test_gathered_encoder(monkeypatch, B, basic):
    """TensorCoreNatureCNN (the XB_K12_BOX=0 path), its data gradients recorded by the checker's backend."""
    spy = _Spy(monkeypatch)
    rep = _representation(3, basic=basic)
    rep._tc = tc.TensorCoreNatureCNN(rep._tc.convs, rep._tc.fc, rep._tc.in_hwc, backend=K.RecordingBackend(3))
    _check(rep, spy, _obs(B, B + 9))


_NO_TMA = r"""
import sys, torch
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
import k12_encoder_refs as K
from xuance_b200.torch.utils import tc_conv as tc
from test_gpu_k12_encoder import _representation
d = torch.load(sys.argv[2], weights_only=False)
rep = _representation(3)
rep.load_state_dict(d["state"])
assert type(rep._tc) is tc.TensorCoreNatureCNN          # XB_K12_TMA=0 selects the gathered encoder
enc = tc.TensorCoreNatureCNN(rep._tc.convs, rep._tc.fc, rep._tc.in_hwc, backend=K.RecordingBackend(3))
for B, (x_pl, dz) in d["cases"].items():
    x_pl, dz = x_pl.cuda(), dz.cuda()
    for p in enc.parameters():
        p.grad = None
    z = tc.tc_encode(enc, x_pl, B)
    z.backward(dz)
    K.check(enc, K.capture(enc, B, x_pl, z.detach(), [p.grad.clone() for p in enc.parameters()]), dz)
print("ok")
"""


def test_tma_disabled_in_a_subprocess(tmp_path):
    """XB_K12_TMA=0 is read once by the library (tma_enabled), so it runs in a fresh process: the same checker there."""
    from xuance_b200 import _lib
    rep = _representation(3)
    cases = {}
    for B in (37, 257):
        obs = _obs(B, B + 11)
        raw = torch.empty((1, B, 84, 84, 4), dtype=torch.bfloat16, device=DEV)
        _lib.call("xb_gather_obs_planes", _lib.ptr(obs), None, B, 84 * 84 * 4, 1, _lib.ptr(raw))
        cases[B] = (raw.cpu(), torch.randn(B, 512, generator=torch.Generator().manual_seed(B)))
    src = tmp_path / "in.pt"
    torch.save(dict(state={k: v.cpu() for k, v in rep.state_dict().items()}, cases=cases), src)
    env = dict(os.environ, XB_K12_TMA="0")
    res = subprocess.run([sys.executable, "-c", _NO_TMA, ROOT, str(src)], env=env, capture_output=True, text=True, cwd=ROOT)
    assert res.returncode == 0 and "ok" in res.stdout, res.stdout + res.stderr


def test_gradients_add_into_existing_grad(monkeypatch):
    """``_into``: with every ``.grad`` pre-filled (the flat gradient bucket of the fused optimizer), the result is
    prev + fresh bit for bit (xb_wgrad_reduce adds the finished value once; the Linear bias uses add_)."""
    spy = _Spy(monkeypatch)
    rep = _representation(3)
    enc = rep._tc
    obs = _obs(257, 21)
    fresh = _step(rep, spy, obs, 5)
    g = torch.Generator(device=DEV).manual_seed(6)
    prev = [torch.randn(p.shape, device=DEV, generator=g) for p in enc.parameters()]
    for p, v in zip(enc.parameters(), prev):
        p.grad = v.clone()
    z = rep(obs).embeddings
    (z * torch.randn(z.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))).sum().backward()
    for i, (p, v, f) in enumerate(zip(enc.parameters(), prev, fresh)):
        assert torch.equal(p.grad, v + f), "parameter %d" % i


def _state(enc, B):
    buf = enc._plans[("buf", B)]
    _, sv = enc._saved
    return {k: v.clone() for k, v in buf.items() if k != "act1_pairs"} | {"act3": sv["act3"].clone(), "y": sv["y"].clone()}


def test_inference_calls_leave_a_pending_backward_alone(monkeypatch):
    """forward (keep) at B, then no_grad forwards at B and at 256 (rollout / target calls), then backward: the gradients
    are bit-equal to a run without the inference calls, and the saved activations and buffers are unchanged."""
    spy = _Spy(monkeypatch)
    rep = _representation(3)
    enc = rep._tc
    B = 300
    obs = _obs(B, 31)
    R = torch.randn(B, 512, device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    runs = []
    for inference in (False, True):
        for p in enc.parameters():
            p.grad = None
        z = rep(obs).embeddings
        before = _state(enc, B)
        if inference:
            with torch.no_grad():
                rep(_obs(B, 32))
                rep(_obs(256, 33))
            after = _state(enc, B)
            for k in before:
                assert torch.equal(before[k], after[k]), k
            K.check_padding(enc, B, "buf_inference")
            K.check_padding(enc, 256, "buf_inference")
        (z * R).sum().backward()
        runs.append([p.grad.clone() for p in enc.parameters()])
    for i, (a, b) in enumerate(zip(*runs)):
        assert torch.equal(a, b), "parameter %d" % i


def test_repeated_runs_are_bit_identical(monkeypatch):
    spy = _Spy(monkeypatch)
    rep = _representation(3)
    obs = _obs(1024, 41)
    out = []
    for _ in range(2):
        grads = _step(rep, spy, obs, 3)
        out.append([spy.z.clone()] + grads + list(_state(rep._tc, 1024).values()))
    for i, (a, b) in enumerate(zip(*out)):
        assert torch.equal(a, b), i


def test_cuda_graph_encoder_matches_eager(monkeypatch):
    """Encoder forward + backward captured with torch.cuda.graph, replayed on new observations copied into the static
    input: bit-equal to the eager run on the same data."""
    rep = _representation(3)
    enc = rep._tc
    B = 256
    static_obs = _obs(B, 50).clone()
    R = torch.randn(B, 512, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))

    def step():
        for p in enc.parameters():
            p.grad = None
        z = rep(static_obs).embeddings
        (z * R).sum().backward()
        return z

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    for p in enc.parameters():
        p.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        z_static = step()
    static_grads = [p.grad for p in enc.parameters()]                # written by every replay
    for seed in (51, 52):
        obs = _obs(B, seed)
        static_obs.copy_(obs)
        graph.replay()
        torch.cuda.synchronize()
        got = [z_static.detach().clone()] + [g.clone() for g in static_grads]
        for p in enc.parameters():
            p.grad = None
        z = rep(obs).embeddings
        (z * R).sum().backward()
        want = [z.detach()] + [p.grad.clone() for p in enc.parameters()]
        for i, (a, b) in enumerate(zip(got, want)):
            assert torch.equal(a, b), "seed %d tensor %d" % (seed, i)


def test_ppo_train_epochs_tc_cuda_graph_matches_eager():
    """PPO with compute='tc' (the bench's default mode): OnPolicyAgent.train_epochs with every minibatch update captured
    in a CUDA graph (use_cuda_graph) against the eager path - three updates at B = 256 (256 rows, one minibatch), the
    graph captured once and replayed; losses and every parameter bit-equal."""
    from argparse import Namespace
    from helpers import synth_rollout, fill_buffers
    from xuance_b200.common import Box, Discrete
    from xuance_b200.torch.agents import PPO_Agent
    base = dict(agent="PPO", learner="PPO_Learner", representation="AC_CNN_Atari", env_name="Atari",
                distributed_training=False, device=DEV, seed=3, parallels=8, running_steps=100000, horizon_size=32,
                n_epochs=3, n_minibatch=1, learning_rate=2.5e-4, vf_coef=0.25, ent_coef=0.01, clip_range=0.2, gamma=0.99,
                use_gae=True, gae_lambda=0.95, use_advnorm=True, use_grad_clip=True, grad_clip_norm=0.5, use_obsnorm=False,
                use_rewnorm=False, activation="relu", filters=[32, 64, 64], kernels=[8, 4, 3], strides=[4, 2, 1],
                fc_hidden_sizes=[512], actor_hidden_size=[], critic_hidden_size=[], model_dir="/tmp/xb_models/g_tc",
                logger=None, compute="tc", tc_planes=3, episode_length=None)
    ro = synth_rollout(np.random.default_rng(0), 8, 32, (84, 84, 4))
    results = []
    for graph in (False, True):
        agent = PPO_Agent(Namespace(**dict(base, use_cuda_graph=graph)), None, Box(0, 255, (84, 84, 4), np.uint8), Discrete(4))
        assert agent.model.representation.compute == "tc" and agent.batch_size == 256
        fill_buffers([agent.memory], ro)
        np.random.seed(11)
        info = agent.train_epochs(3)
        assert bool(getattr(agent, "_graphs", None)) == graph          # a graph was captured exactly when asked for
        results.append((info, {k: v.clone() for k, v in agent.model.state_dict().items()}))
    (i0, p0), (i1, p1) = results
    for k in ("actor_loss", "critic_loss", "entropy", "predict_value", "clip_ratio"):
        assert np.array_equal(np.asarray(i1[k]), np.asarray(i0[k])), (k, i1[k], i0[k])
    for k in p0:
        assert torch.equal(p1[k], p0[k]), k
