"""Float64 restatement of the QMIX mixer (q_mix_head.py:52-95) on float32 inputs, and a first-order error bound for K9-TC
(xb_qmix_mix_fused_fwd, the split-bf16 tensor-core forward).  tests/test_qmix_tc_refs.py pins both on the CPU and
tests/test_gpu_qmix_tc_edges.py compares the kernel with them.

Bound.  As in kernel_refs, an error is measured against the magnitude of what was added, not against the result.  For
every GEMM layer y = x.W^T + b the same layer is run in float64 on |x|.|W|^T + |b| ("mag"); each error is then carried
through the mixer with the Lipschitz constants of relu, abs and ELU (all <= 1) and the per-row products with q:

    err(Z)     <= k mag(Z)                                  Z = X.W1cat^T + c, the four first layers
    err(W1raw) <= k (|Wb1| err(relu Z_w1)/k + mag(W1raw))  the second layers (hyper_w_1, likewise hyper_w_2, hyper_b_2)
    err(pre_h) <= sum_i |q_i| err(w1_ih) + err(b1_h) + k (sum_i |q_i w1_ih| + |b1_h|)
    err(hid_h) <= err(pre_h) + k 2^-7                       the 2^-7 only where pre_h may be <= 0
    err(q_tot) <= sum_h (|w2_h| err(hid_h) + |hid_h| err(w2_h)) + err(b2) + k (sum_h |hid_h w2_h| + |b2|)

and M_row = err(q_tot) / k.  Second-order products of errors are dropped.

Why k = 2^-14.  A float32 x is split x = hi + lo + e with hi = bf16(x), lo = bf16(x - hi): |lo| <= 2^-8 |x| and
|e| <= 2^-16 |x|.  The kernel sums hi.hi + hi.lo + lo.hi, so one product x w differs from it by lo_x lo_w + e_x w + x e_w,
at most (2^-16 (1 + 2^-7) + 2 2^-16) |x||w| < 3.03 2^-16 |x||w|.  The products of two bf16 values are exact in fp32.  The
fp32 accumulation adds 3 ceil(K/16) blocks of 16 products, each add truncating by at most 2^-23 of the running sum
(<= mag); counting one more such error for the sum inside each block, K <= 160 gives at most 60 2^-23 = 0.47 2^-16 of
mag.  Adding the bias in fp32 costs 2^-24 mag.  Together < 3.6 2^-16 mag < 2^-14 mag per layer.  The mixing epilogue
runs in fp32 with at most n + 2 <= 10 (K9-TC) or 34 (the sum over the 32 hidden units) roundings of 2^-24 each,
2^-19 of their magnitude at most, inside the k term given to each.  ELU's expf(x) - 1 has an absolute error of at most
2 ulp(1) + 2^-24 < 2^-21 = k 2^-7 for x <= 0, which no relative term covers (cancellation near 0).

The same bound covers the plain fp32 path (cuBLAS without TF32 + K9, S <= 160 roundings of 2^-24 per layer)."""
import numpy as np
import torch

f32, f64 = np.float32, np.float64
KAPPA = 2.0 ** -14
EXP_ABS = 2.0 ** -7          # ELU's absolute expf error, in units of KAPPA

# first layers in K9-TC's order (hyper_w_1 | hyper_b_1 | hyper_w_2 | hyper_b_2), then the three second layers
FIRST = ("hyper_w_1.0", "hyper_b_1", "hyper_w_2.0", "hyper_b_2.0")
SECOND = ("hyper_w_1.2", "hyper_w_2.2", "hyper_b_2.2")


def mixer_params(module):
    """{layer name: (W float32 [out, in], b float32 [out])} of a QMIX_Mixer or MixerOracle."""
    sd = {k: v.detach().cpu().numpy().astype(f32) for k, v in module.state_dict().items()}
    return {name: (sd[name + ".weight"], sd[name + ".bias"]) for name in FIRST + SECOND}


def _d(x):
    return np.asarray(x, dtype=f64)


def _layer(x, mag_x, W, b):
    """(y, mag, prop) of y = x.W^T + b: mag = |x|.|W|^T + |b| (this layer's own error, / KAPPA) and prop = mag_x.|W|^T
    (the input's error carried through, / KAPPA)."""
    W, b = _d(W), _d(b)
    aW = np.abs(W)
    y = x @ W.T + b
    mag = np.abs(x) @ aW.T + np.abs(b)
    return y, mag, (0.0 if mag_x is None else mag_x @ aW.T)


def mixer_ref(P, q, states):
    """(q_tot float64 [R], M_row float64 [R]) for the mixer with parameters P (mixer_params) on float32 q [R, n] and
    states [R, S]; |K9-TC - q_tot| <= KAPPA M_row per row."""
    X, q = _d(states), _d(q)
    R, n = q.shape
    Z, Mz = {}, {}
    for name in FIRST:
        Z[name], Mz[name], _ = _layer(X, None, *P[name])
    relu = lambda z: np.maximum(z, 0.0)
    sec = {}
    for first, second in zip(("hyper_w_1.0", "hyper_w_2.0", "hyper_b_2.0"), SECOND):
        y, mag, prop = _layer(relu(Z[first]), Mz[first], *P[second])
        sec[second] = (y, mag + prop)
    W1raw, M_W1 = sec["hyper_w_1.2"]
    w1, M_w1 = np.abs(W1raw).reshape(R, n, -1), M_W1.reshape(R, n, -1)
    b1, M_b1 = Z["hyper_b_1"], Mz["hyper_b_1"]
    aq = np.abs(q)
    pre = np.einsum("ri,rih->rh", q, w1) + b1
    M_pre = np.einsum("ri,rih->rh", aq, M_w1) + M_b1 + np.einsum("ri,rih->rh", aq, w1) + np.abs(b1)
    hid = np.where(pre > 0, pre, np.expm1(np.minimum(pre, 0.0)))
    M_hid = M_pre + EXP_ABS * (pre <= KAPPA * M_pre)
    W2raw, M_w2 = sec["hyper_w_2.2"]
    w2 = np.abs(W2raw)
    b2, M_b2 = sec["hyper_b_2.2"][0][:, 0], sec["hyper_b_2.2"][1][:, 0]
    q_tot = (hid * w2).sum(axis=1) + b2
    M = (w2 * M_hid + np.abs(hid) * M_w2).sum(axis=1) + M_b2 + (np.abs(hid) * w2).sum(axis=1) + np.abs(b2)
    return q_tot, M


def mixer_ref_chunked(P, q, states, rows=16384):
    """mixer_ref in row chunks (the float64 intermediates of 2^17 rows would take a few GB)."""
    outs = [mixer_ref(P, q[i:i + rows], states[i:i + rows]) for i in range(0, len(q), rows)]
    return np.concatenate([o[0] for o in outs]), np.concatenate([o[1] for o in outs])


# ---------------------------------------------------------------------------------------------- split-bf16 model
def _bf16(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=f32)).to(torch.bfloat16).to(torch.float32).numpy()


def split(x):
    """(hi, lo) bf16 planes of a float32 array, as K9-TC's store_unit makes them, held in float64."""
    x = np.asarray(x, f32)
    hi = _bf16(x)
    return _d(hi), _d(_bf16(x - hi))


def split_mm(x, W, products):
    """x.W^T from the bf16 planes with the products {(a, b)} (0 = hi, 1 = lo) summed exactly: the kernel's GEMM without
    its fp32 accumulation."""
    xs, ws = split(x), split(W)
    return sum(xs[a] @ ws[b].T for a, b in products)


def mixer_split(P, q, states, products1=((0, 0), (0, 1), (1, 0)), products2=((0, 0), (0, 1), (1, 0))):
    """The mixer with both GEMMs taken from the bf16 planes with the given product sets, everything else in float64 on
    float32-rounded intermediates (what the kernel stages): a model of K9-TC's numerics and of its defects."""
    X, qd = np.asarray(states, f32), _d(q)
    R, n = qd.shape
    Z = {name: split_mm(X, P[name][0], products1) + _d(P[name][1]) for name in FIRST}
    h = {name: np.maximum(Z[name], 0.0).astype(f32) for name in ("hyper_w_1.0", "hyper_w_2.0", "hyper_b_2.0")}
    sec = {s: split_mm(h[f], P[s][0], products2) + _d(P[s][1])
           for f, s in zip(("hyper_w_1.0", "hyper_w_2.0", "hyper_b_2.0"), SECOND)}
    w1 = np.abs(sec["hyper_w_1.2"]).reshape(R, n, -1)
    pre = np.einsum("ri,rih->rh", qd, w1) + Z["hyper_b_1"]
    hid = np.where(pre > 0, pre, np.expm1(np.minimum(pre, 0.0)))
    return (hid * np.abs(sec["hyper_w_2.2"])).sum(axis=1) + sec["hyper_b_2.2"][:, 0]
