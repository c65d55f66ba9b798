"""CPU: pins tests/qmix_tc_refs.py - the float64 mixer against the oracle's layers, the bound against the float32 oracle and
against operand perturbations of 2^-16, and shows that a model of K9-TC's split-bf16 arithmetic stays far inside the bound
while the same model with one product dropped does not, so that a wrong reference or a slack bound cannot make
tests/test_gpu_qmix_tc_edges.py pass.  Also holds K9-TC's register spills to their compiled size."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import qmix_tc_refs as qr
from oracle.qmix import MixerOracle
from xuance_b200 import build

f32 = np.float32
# max |err| / (KAPPA M_row) that tests/test_gpu_qmix_tc_edges.py allows the kernel (MAX_RATIO there); the split model of
# the kernel must stay below it and every defect model above it
MAX_RATIO = 0.02
DEFECTS = {"GEMM1 without lo.hi": dict(products1=((0, 0), (0, 1))),
           "GEMM1 without hi.lo": dict(products1=((0, 0), (1, 0))),
           "GEMM2 hi.hi only": dict(products2=((0, 0),))}


def _case(S, n, big, R=3000, seed=0):
    torch.manual_seed(S * 10 + n)
    om = MixerOracle(S, 32, 32, n)
    rng = np.random.default_rng(seed)
    if big:      # hypernetwork weights x 8, states in [-1, 1], q in [-5, 25]
        with torch.no_grad():
            for k, v in om.named_parameters():
                if k.endswith("weight"):
                    v.mul_(8.0)
        st = rng.uniform(-1, 1, (R, S)).astype(f32)
        q = rng.uniform(-5, 25, (R, n)).astype(f32)
    else:
        st = rng.normal(size=(R, S)).astype(f32)
        q = (rng.normal(size=(R, n)) * 2).astype(f32)
    return om, q, st


CASES = [(98, 5, False), (81, 1, False), (132, 1, True), (112, 8, True), (97, 2, False)]


@pytest.mark.parametrize("S,n,big", CASES)
def test_reference_equals_oracle_layers_in_float64(S, n, big):
    """mixer_ref == the oracle's own modules and formula (q_mix_head.py:81-94) run in float64."""
    om, q, st = _case(S, n, big, R=500)
    ref, _ = qr.mixer_ref(qr.mixer_params(om), q, st)
    od = om.double()
    with torch.no_grad():
        s, qq = torch.tensor(st, dtype=torch.float64), torch.tensor(q, dtype=torch.float64).view(-1, 1, n)
        w_1 = torch.abs(od.hyper_w_1(s)).view(-1, n, 32)
        hidden = F.elu(torch.bmm(qq, w_1) + od.hyper_b_1(s).view(-1, 1, 32))
        want = (torch.bmm(hidden, torch.abs(od.hyper_w_2(s)).view(-1, 32, 1)) + od.hyper_b_2(s).view(-1, 1, 1)).view(-1)
    np.testing.assert_allclose(ref, want.numpy(), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("S,n,big", CASES)
def test_float32_oracle_within_bound(S, n, big):
    """The float32 CPU mixer (another float32-grade evaluation of the same network) lies inside KAPPA M_row."""
    om, q, st = _case(S, n, big)
    ref, M = qr.mixer_ref(qr.mixer_params(om), q, st)
    with torch.no_grad():
        got = om(torch.from_numpy(q), torch.from_numpy(st)).view(-1).numpy().astype(np.float64)
    assert (np.abs(got - ref) <= qr.KAPPA * M).all()


@pytest.mark.parametrize("S,n,big", CASES)
def test_bound_holds_under_operand_perturbation(S, n, big):
    """Every operand (states, q, every weight and bias) moved by up to 2^-16 relative, at random: the float64 mixer of
    the perturbed operands stays inside KAPPA M_row of the unperturbed one."""
    om, q, st = _case(S, n, big)
    P = qr.mixer_params(om)
    ref, M = qr.mixer_ref(P, q, st)
    rng = np.random.default_rng(S + n)
    jig = lambda x: np.asarray(x, np.float64) * (1.0 + rng.uniform(-2.0 ** -16, 2.0 ** -16, np.shape(x)))
    Pp = {k: (jig(W), jig(b)) for k, (W, b) in P.items()}
    got, _ = qr.mixer_ref(Pp, jig(q), jig(st))
    r = np.abs(got - ref) / (qr.KAPPA * M)
    assert r.max() <= 1.0, r.max()


@pytest.mark.parametrize("S,n,big", CASES)
def test_split_model_inside_and_defects_outside(S, n, big):
    """The kernel's three-product split (exact sums) stays below MAX_RATIO of the bound; dropping one product of either
    GEMM, as a defective kernel would, exceeds it on the same rows."""
    om, q, st = _case(S, n, big)
    P = qr.mixer_params(om)
    ref, M = qr.mixer_ref(P, q, st)
    ratio = lambda got: np.abs(got - ref) / (qr.KAPPA * M)
    r = ratio(qr.mixer_split(P, q, st))
    assert r.max() <= MAX_RATIO / 4, r.max()
    for name, kw in DEFECTS.items():
        assert ratio(qr.mixer_split(P, q, st, **kw)).max() > MAX_RATIO, name


def test_bound_fails_for_a_dropped_product_on_coherent_operands():
    """Operands whose split residuals all have one sign (positive states just above a bf16 value, positive weights):
    the error of a dropped product then adds up instead of cancelling, and exceeds KAPPA M_row itself."""
    S, n, R = 98, 5, 64
    om, _, _ = _case(S, n, False)
    rng = np.random.default_rng(1)
    hi = np.asarray(qr._bf16(rng.uniform(0.5, 1.0, (R, S)).astype(f32)), f32)
    st = (hi * f32(1 + 2.0 ** -9 * 0.9)).astype(f32)                   # lo = +0.9 half-ulp of hi, every element
    with torch.no_grad():
        for k, v in om.named_parameters():
            v.abs_()
    q = np.abs(rng.normal(size=(R, n))).astype(f32)
    P = qr.mixer_params(om)
    ref, M = qr.mixer_ref(P, q, st)
    assert (np.abs(qr.mixer_split(P, q, st) - ref) <= qr.KAPPA * M).all()
    bad = qr.mixer_split(P, q, st, products1=((0, 0), (0, 1)))
    assert (np.abs(bad - ref) / (qr.KAPPA * M)).max() > 1.0


K9TC_SPILL_STORES = 196      # bytes, ptxas for sm_90a at 255 registers (DESIGN.md, deferred work: K9-TC)


@pytest.mark.skipif(shutil.which(build._nvcc()) is None and not os.path.exists(build._nvcc()), reason="nvcc not available")
def test_k9tc_ptxas_spills_do_not_grow(tmp_path):
    """Compile-time check (no GPU): K9-TC keeps its n <= 8 agent blocks of W1 in registers at 255 registers with at most
    K9TC_SPILL_STORES bytes of spill stores, so a change to its product order cannot silently move them to local memory."""
    flags = [f for f in build.NVCC_FLAGS if f not in ("--use_fast_math=false", "-shared")]
    cmd = [build._nvcc()] + flags + ["-c", os.path.join(build.CSRC, "qmix_tc.cu"), "-o", str(tmp_path / "qmix_tc.o")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    assert res.returncode == 0, log
    found, cur = [], False
    for line in log.splitlines():
        if re.search(r"Compiling entry function '\S*qmix_mix_tc_kernel\S*'", line):
            cur = True
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if cur and m:
            found.append(int(m.group(1)))
            cur = False
    assert len(found) == 1, log
    assert found[0] <= K9TC_SPILL_STORES, found
