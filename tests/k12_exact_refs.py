"""Exact-arithmetic references for K12's weight- and bias-gradient reductions: the split partials of ``xb_wgrad_gather_tc``
(cp.async gather, input windows, pixel-pair windows) and ``xb_wgrad_box_tc``, the column sums (``colsum``) the data-gradient
launches write, and ``xb_wgrad_reduce``, which adds either into a weight or a bias gradient.

Why exact.  A rounding bound over a chain of millions of terms cannot tell one missing 64-site chunk, one repeated split or
one lost column-sum row from accumulated rounding.  Exact arithmetic can:
  * every operand plane holds small dyadic values (``fill``), so every product is a multiple of a common resolution res;
  * if for every compared element sum_k |term_k| <= 2^22 * res (``check_premise``: two bits below float32's 24-bit
    significand), every partial sum of those terms, in any order and at any split, is a multiple of res below 2^24 * res,
    i.e. a float32;
  * the tensor core's truncating add (DESIGN.md section 4) of representable values is then exact, and so is every
    round-to-nearest add after it (plane groups, split partials, fold groups, lanes, column sums).
So the kernels must return the float64 value bit for bit, whatever order they sum in, and any dropped, repeated or misplaced
site, chunk, split, tile, plane group or column-sum row changes an integer-valued result.

A launch multiplies A plane i with the B planes j < PB - i (plane-index sum < PB); the references use exactly those
products.  Fillings:
  * "dense": plane 0 only, x in {0, 1} (the raw uint8 pixel form), g in {0, +-1}: indexing at full size;
  * "sparse": every plane q in {0, +-2^-2q} (2^-2q rather than the 2^-8q of a real split, so that every plane group stays
    exact), g thinned so that the premise holds: the wiring of the plane groups (a product kept or dropped wrongly, a group
    lost).

``reduce_ref`` restates ``xb_wgrad_reduce`` in float32 in its exact order (fold of ceil(splits / 128) consecutive splits
above 256 splits, ``lanes_for`` from the device's SM count, the tiled kernel's sequential sum, the lane kernel's strided
partial sums added by lane 0 in order, ``__fmul_rn(s, scale)``, ``dw + v`` under ``accumulate``), so the reduce is pinned
bit for bit on arbitrary float32 partials too.
"""
import torch

from xuance_b200.torch.utils import tc_conv as tc

LIMIT = 2.0 ** 22              # sum |terms| <= LIMIT * res for every compared element
PACK_TILE_MAX = 8192           # conv_tc.cu: floats of shared memory per block of the tiled pack / reduce


# ------------------------------------------------------------------------------------------------ operands
def fill(shape, planes, mode, gen, density=1.0, signed=True, device="cuda"):
    """bfloat16 plane tensor [planes, *shape] of exact small dyadic values (module docstring).  ``density``: probability that
    an element of a plane is non-zero (dense: plane 0; sparse: each plane on its own); ``signed=False``: values >= 0."""
    out = torch.zeros((planes,) + tuple(shape), dtype=torch.bfloat16, device=device)
    for q in range(1 if mode == "dense" else planes):
        on = torch.rand(shape, generator=gen, device=device) < density
        v = torch.ones(shape, device=device)
        if signed:
            v = torch.where(torch.rand(shape, generator=gen, device=device) < 0.5, -v, v)
        out[q] = torch.where(on, v * 2.0 ** (-2 * q), torch.zeros_like(v)).to(torch.bfloat16)
    return out


def check_premise(mag, res, what):
    """``mag``: sum |terms| of every compared element (float64).  Raises if the exactness premise does not hold, so that a
    fault of the construction is reported as such and not as a kernel error; returns the largest sum / res."""
    worst = float(mag.max()) / res if mag.numel() else 0.0
    assert worst <= LIMIT, ("%s: exactness premise broken: sum |terms| = %.0f res > 2^22 res; the operands are too dense "
                            "for an exact comparison (a construction fault, not a kernel result)" % (what, worst))
    return worst


def kept_pairs(x_pl, g_pl):
    """[(A plane i, sum of the B planes it meets)] in float64: the products a launch keeps (plane-index sum < PB)."""
    pb = g_pl.shape[0]
    return [(x_pl[i].double(), g_pl[:pb - i].double().sum(0)) for i in range(x_pl.shape[0])]


# ------------------------------------------------------------------------------------------------ split rules
def sites_per_split(M, splits):
    """xb_wgrad_sites_per_split: runs of a multiple of 64 sites, 0 when a split would be empty."""
    per = -(-(-(-M // splits)) // tc.KC) * tc.KC
    return 0 if (splits - 1) * per >= M else per


def box_rows_per_split(g_rows, splits, box_h):
    """xb_wgrad_box_tc: runs of whole ``box_h`` grid rows, 0 when a split would be empty."""
    per = -(-(-(-g_rows // splits)) // box_h) * box_h
    return 0 if (splits - 1) * per >= g_rows else per


def max_splits(units, unit):
    """The largest split count whose runs (multiples of ``unit``) leave no split empty."""
    s = -(-units // unit)
    while s > 1 and (s - 1) * (-(-(-(-units // s)) // unit) * unit) >= units:
        s -= 1
    return s


def single_chunk_tail(M, unit=tc.KC):
    """The smallest split count whose last split holds at most one ``unit`` (a one-chunk tail)."""
    for s in range(2, M // unit + 2):
        per = -(-(-(-M // s)) // unit) * unit
        if (s - 1) * per < M and M - (s - 1) * per <= unit:
            return s
    raise AssertionError(M)


def _split_bmm(A, G, per, splits):
    """A [S, k], G [S, n] float64, split s = sites [s * per, min((s + 1) * per, S)) -> [splits, k, n]."""
    S = A.shape[0]
    pad = splits * per - S
    A = torch.cat([A, A.new_zeros(pad, A.shape[1])]) if pad > 0 else A[:splits * per]
    G = torch.cat([G, G.new_zeros(pad, G.shape[1])]) if pad > 0 else G[:splits * per]
    return torch.bmm(A.view(splits, per, -1).transpose(1, 2), G.view(splits, per, -1))


# ------------------------------------------------------------------------------------------------ float64 references
def gather_tap(x, geom, t):
    """Tap t of the gathered GEMM ``geom`` over x [B, IH, IW, C]: [M, C], x[b, y*sy + dy, x*sx + dx], zero outside."""
    B, IH, IW, C = x.shape
    iy = torch.arange(geom.OY, device=x.device) * geom.sy + geom.dy[t]
    ix = torch.arange(geom.OX, device=x.device) * geom.sx + geom.dx[t]
    ok = ((iy >= 0) & (iy < IH))[:, None] & ((ix >= 0) & (ix < IW))[None, :]
    v = x[:, iy.clamp(0, IH - 1)][:, :, ix.clamp(0, IW - 1)] * ok[None, :, :, None]
    return v.reshape(-1, C)


def wgrad_gather_ref(x_pl, g_pl, geom, splits):
    """float64 [splits, K, N] of ``xb_wgrad_gather_tc``: split s sums the sites of its run (``sites_per_split``), column
    k = (tap, c) in the geometry's tap order, over the tensors exactly as given (padding included)."""
    per = sites_per_split(geom.M, splits)
    assert per > 0, (geom.M, splits)
    N = g_pl.shape[-1]
    out = torch.zeros((splits, geom.K, N), dtype=torch.float64, device=g_pl.device)
    for xi, gi in kept_pairs(x_pl, g_pl):
        x = xi.reshape(geom.B, geom.IH, geom.IW, geom.C)
        G = gi.reshape(geom.M, N)
        for t in range(geom.T):
            out[:, t * geom.C:(t + 1) * geom.C] += _split_bmm(gather_tap(x, geom, t), G, per, splits)
    return out


def box_chunk(x, bg, i, rows):
    """Chunk i = (c0, w0, r0) of the box geometry ``bg`` for the merged grid rows ``rows``: [len(rows) * box_px, 64],
    x[R * row_step + r0, w0 + px, c0 .. c0 + 63] over x [rows_in, W, C], zero outside."""
    c0, w0, r0 = bg.chunks[i]
    n_rows, W, _ = x.shape
    row = rows * bg.row_step + r0
    px = torch.arange(bg.box_px, device=x.device) + w0
    ok = ((row >= 0) & (row < n_rows))[:, None] & ((px >= 0) & (px < W))[None, :]
    v = x[row.clamp(0, n_rows - 1)][:, px.clamp(0, W - 1), c0:c0 + 64] * ok[..., None]
    return v.reshape(-1, 64)


def wgrad_box_ref(x_pl, g_pl, bg, box_h, splits):
    """float64 [splits, K, N] of ``xb_wgrad_box_tc``: g_pl [PB, g_rows, box_px, N]; split s sums whole ``box_h`` grid rows."""
    _, g_rows, spr, N = g_pl.shape
    per = box_rows_per_split(g_rows, splits, box_h)
    assert per > 0, (g_rows, splits, box_h)
    rows = torch.arange(g_rows, device=g_pl.device)
    out = torch.zeros((splits, bg.K, N), dtype=torch.float64, device=g_pl.device)
    for xi, gi in kept_pairs(x_pl, g_pl):
        x = xi.reshape(-1, bg.W, bg.C)
        G = gi.reshape(g_rows * spr, N)
        for i in range(len(bg.chunks)):
            out[:, 64 * i:64 * i + 64] += _split_bmm(box_chunk(x, bg, i, rows), G, per * spr, splits)
    return out


def torch_layout(s, N, C, KH, KW):
    """[(kh, kw, c), N] -> torch's [N, C, KH, KW]."""
    return s.t().reshape(N, KH, KW, C).permute(0, 3, 1, 2).contiguous()


def reduced_ref(ref64, N, C, KH, KW, scale=1.0):
    """The exact reduced gradient [N, C, KH, KW] of float64 partials: float32(exact), times float32(scale) rounded once."""
    s = ref64.sum(0)
    if scale != 1.0:
        s = (s.float().double() * float(torch.tensor(scale, dtype=torch.float32))).float()     # one rounding, as __fmul_rn
    return torch_layout(s.float(), N, C, KH, KW)


# ------------------------------------------------------------------------------------------------ xb_wgrad_reduce in float32
def lanes_for(n_splits, groups, total, sm_count):
    lanes = 1
    while lanes < 8 and lanes * 2 <= n_splits and total // (256 // lanes) * groups < sm_count * 16:
        lanes *= 2
    return lanes


def reduce_kind(splits, N, C, KH, KW):
    """Which kernels xb_wgrad_reduce launches: "fold+lane", "tiled" or "lane"."""
    HW = KH * KW
    step = -(-splits // 128) if splits > 256 else 1
    tiled_ok = HW >= 32 and N % 32 == 0 and C % 2 == 0 and 2 * HW * 33 <= PACK_TILE_MAX          # xb_pack_tiled(3, ...)
    if tiled_ok and HW <= 128 and (N // 32) * (C // 2) >= 128 and -(-splits // step) <= 16:
        return "tiled" if step == 1 else "fold+tiled"
    return "lane" if step == 1 else "fold+lane"


def _lane_sums(rows, lanes):
    """rows [groups, n, total] float32: lane l of a group adds rows l, l + lanes, ... in order from 0.0, then lane 0 adds
    lanes 1 .. lanes - 1 in order (reduce_splits); zero rows appended at the end leave every sum unchanged."""
    g, n, total = rows.shape
    pad = (-n) % lanes
    if pad:
        rows = torch.cat([rows, rows.new_zeros(g, pad, total)], 1)
    r = rows.view(g, -1, lanes, total)
    s = torch.zeros((g, lanes, total), dtype=torch.float32, device=rows.device)
    for k in range(r.shape[1]):
        s = s + r[:, k]
    out = s[:, 0]
    for q in range(1, lanes):
        out = out + s[:, q]
    return out


def reduce_ref(partials, N, C, KH, KW, scale=1.0, out=None, accumulate=False, sm_count=None):
    """xb_wgrad_reduce restated in float32, in its order.  ``partials`` [splits, (kh, kw, c), N] (not modified); returns the
    torch-layout [N, C, KH, KW] gradient (``out`` + it under ``accumulate``)."""
    if sm_count is None:
        sm_count = torch.cuda.get_device_properties(partials.device).multi_processor_count
    splits = partials.shape[0]
    total = N * C * KH * KW
    ws = partials.reshape(splits, total).float()
    rows, step = ws, 1
    if splits > 256:
        group = -(-splits // 128)
        groups = -(-splits // group)
        lanes = lanes_for(group, groups, total, sm_count)
        pad = groups * group - splits
        g = torch.cat([ws, ws.new_zeros(pad, total)]) if pad else ws
        rows = _lane_sums(g.view(groups, group, total), lanes)            # the folded first row of every group
        step = group
    kind = reduce_kind(splits, N, C, KH, KW)
    if kind.endswith("tiled"):
        s = torch.zeros(total, dtype=torch.float32, device=ws.device)
        for k in range(rows.shape[0]):
            s = s + rows[k]
    else:
        lanes = lanes_for(rows.shape[0], 1, total, sm_count)
        s = _lane_sums(rows[None], lanes)[0]
    s = s * torch.tensor(scale, dtype=torch.float32, device=s.device)
    dw = torch_layout(s.view(-1, N), N, C, KH, KW)
    if accumulate:
        return out.view(N, C, KH, KW) + dw
    return dw


# ------------------------------------------------------------------------------------------------ recorder
class Recorder:
    """Records the reduction launches of one backward and passes every call through: ``wgrad_gather`` / ``wgrad_box`` (split
    partials), ``wgrad_reduce`` (a weight or, through ``bias_grad``, a bias gradient) and the ``gemm_gather`` /
    ``gemm_box`` / ``gemm_halo`` calls that pass ``colsum``.  ``chains()`` pairs each reduce with the launches that wrote its
    partials (by address), so a replay can rebuild every launch with exact operands of the same shapes and strides.

    For an output-gradient operand (the B operand of a weight gradient, the A operand of a data gradient) it keeps the
    pixels that are non-zero in any plane and channel (``support``): production keeps the padding of those tensors zero,
    and the replay keeps it zero too."""

    NAMES = ("wgrad_gather", "wgrad_box", "wgrad_reduce", "gemm_gather", "gemm_box", "gemm_halo")

    def __init__(self, monkeypatch, module=tc):
        self.calls = []
        self.orig = {}
        for name in self.NAMES:
            self.orig[name] = getattr(module, name)
            monkeypatch.setattr(module, name, self._wrap(name, self.orig[name]))

    @staticmethod
    def _desc(t):
        return None if t is None else dict(shape=tuple(t.shape), stride=tuple(t.stride()), dtype=t.dtype)

    @staticmethod
    def _support(t):
        return (t != 0).any(0).any(-1)

    def _wrap(self, name, fn):
        def call(*args, **kw):
            if name == "wgrad_gather":
                x_pl, g_pl, geom, splits = args[:4]
                n_tile = kw.get("n_tile", args[4] if len(args) > 4 else None)
                res = fn(*args, **kw)
                self.calls.append(dict(kind=name, geom=geom, splits=splits, n_tile=n_tile, x=self._desc(x_pl), g=self._desc(g_pl),
                                       support=self._support(g_pl), ptr=res.data_ptr(), bytes=res.numel() * 4))
                return res
            if name == "wgrad_box":
                x_pl, g_pl, bg, box_h, splits = args[:5]
                res = fn(*args, **kw)
                self.calls.append(dict(kind=name, geom=bg, box_h=box_h, splits=splits, x=self._desc(x_pl), g=self._desc(g_pl),
                                       support=self._support(g_pl), ptr=res.data_ptr(), bytes=res.numel() * 4))
                return res
            if name == "wgrad_reduce":
                partials, N, C, KH, KW = args[:5]
                rec = dict(kind=name, N=N, C=C, KH=KH, KW=KW, splits=partials.shape[0], ptr=partials.data_ptr(),
                           bytes=partials.numel() * 4, scale=float(kw.get("scale", 1.0)), accumulate=bool(kw.get("accumulate", False)),
                           out=self._desc(kw.get("out")))
                self.calls.append(rec)
                return fn(*args, **kw)
            colsum = kw.get("colsum")
            if colsum is None:
                return fn(*args, **kw)
            x_pl, w_pl, geom = args[:3]
            assert kw.get("bias") is None and not kw.get("relu", False), "a column-sum launch is a data gradient"
            extra = {k: kw[k] for k in ("out_ld", "out_c0", "mask_ld", "mask_c0", "n_tile") if kw.get(k) is not None}
            self.calls.append(dict(kind=name, geom=geom, x=self._desc(x_pl), w=self._desc(w_pl), out=self._desc(kw.get("out_pl")),
                                   mask=self._desc(kw.get("relu_mask")), colsum=self._desc(colsum), kw=extra,
                                   support=self._support(x_pl), ptr=colsum.data_ptr(), bytes=colsum.numel() * 4))
            return fn(*args, **kw)
        return call

    def chains(self):
        """[(producers, reduce)]: the launches whose output lies in the memory a reduce read, in call order."""
        out, pending = [], []
        for c in self.calls:
            if c["kind"] != "wgrad_reduce":
                pending.append(c)
                continue
            lo, hi = c["ptr"], c["ptr"] + c["bytes"]
            mine = [p for p in pending if lo <= p["ptr"] < hi]
            assert mine, "a reduce with no recorded producer"
            pending = [p for p in pending if p not in mine]
            out.append((mine, c))
        assert not pending, "launches whose partials no reduce read: %s" % [p["kind"] for p in pending]
        return out


# ------------------------------------------------------------------------------------------------ replay
def density_for(terms, mode):
    """On-probability of the output-gradient operand such that the expected sum |terms| of a compared element with
    ``terms`` products at full density (the other operand at on-probability 1/2) is half the limit: one bit below it,
    with the spread of the sum far below that bit."""
    per_term = 0.5 * (16.0 / 9.0 if mode == "sparse" else 1.0)
    return min(1.0, LIMIT / 2 * (1.0 if mode == "dense" else 2.0 ** -4) / (per_term * terms))


def _build(desc, values):
    t = torch.empty_strided(desc["shape"], desc["stride"], dtype=desc["dtype"], device=values.device)
    t.copy_(values)
    return t


def _expect_equal(got, want, what):
    if torch.equal(got, want):
        return
    bad = (got != want) & ~(torch.isnan(got) & torch.isnan(want))
    i = int(bad.reshape(-1).nonzero()[0])
    where = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), got.shape))
    raise AssertionError("%s: %d of %d elements differ, the first at %s: got %r, exact %r"
                         % (what, int(bad.sum()), got.numel(), where, float(got.reshape(-1)[i]), float(want.reshape(-1)[i])))


def _first_bad_split(got, ref):
    bad = (got != ref).reshape(got.shape[0], -1).any(1)
    return [int(s) for s in bad.nonzero()[:8, 0]]


def replay_wgrad(prod, red, launches, mode, gen, sm_count=None, tag=""):
    """One recorded weight gradient with exact operands: every split partial, the reduced gradient (fresh and added into an
    existing gradient) and the reduce's order.  Returns the largest sum |terms| / res seen."""
    pa, pb = prod["x"]["shape"][0], prod["g"]["shape"][0]
    dev = prod["support"].device
    res = 1.0 if mode == "dense" else 2.0 ** (-2 * (pb - 1))
    sites = prod["geom"].M if prod["kind"] == "wgrad_gather" else prod["g"]["shape"][1] * prod["g"]["shape"][2]
    x = _build(prod["x"], fill(prod["x"]["shape"][1:], pa, mode, gen, 0.5, signed=False, device=dev))
    gv = fill(prod["g"]["shape"][1:], pb, mode, gen, density_for(sites, mode), device=dev)
    g = _build(prod["g"], gv * prod["support"][None, ..., None])
    if prod["kind"] == "wgrad_gather":
        part = launches["wgrad_gather"](x, g, prod["geom"], prod["splits"], n_tile=prod["n_tile"])
        ref, mag = (wgrad_gather_ref(a, b, prod["geom"], prod["splits"]) for a, b in ((x, g), (x.abs(), g.abs())))
    else:
        part = launches["wgrad_box"](x, g, prod["geom"], prod["box_h"], prod["splits"])
        ref, mag = (wgrad_box_ref(a, b, prod["geom"], prod["box_h"], prod["splits"]) for a, b in ((x, g), (x.abs(), g.abs())))
    what = "%s%s %s splits=%d (%s)" % (tag, prod["kind"], mode, prod["splits"], "x".join(map(str, prod["g"]["shape"])))
    worst = check_premise(mag.sum(0), res, what)
    if not torch.equal(part, ref.float()):
        _expect_equal(part, ref.float(), what + " partials, splits %s" % _first_bad_split(part, ref.float()))
    N, C, KH, KW, scale = red["N"], red["C"], red["KH"], red["KW"], red["scale"]
    want = reduced_ref(ref, N, C, KH, KW, scale)
    order = reduce_ref(part, N, C, KH, KW, scale, sm_count=sm_count)
    got = launches["wgrad_reduce"](part.clone(), N, C, KH, KW, scale=scale)
    _expect_equal(got, want, what + " reduced")
    _expect_equal(got, order, what + " reduced vs the reduce's order")
    prev = torch.randn((N, C, KH, KW), generator=gen, device=dev)
    got = launches["wgrad_reduce"](part.clone(), N, C, KH, KW, scale=scale, out=prev.clone(), accumulate=True)
    _expect_equal(got, prev + want, what + " added into an existing gradient")
    return worst


def replay_colsum(prods, red, launches, mode, gen, sm_count=None, tag=""):
    """One recorded bias gradient with exact operands: every data-gradient launch that wrote its column sums (output planes
    the split of the exact values, everything else in the output tensor untouched, every column-sum row exact), then the
    reduced bias (fresh and added into an existing gradient) and the reduce's order.  Returns the largest sum / res."""
    import test_k12_geometry as G
    restated = dict(gemm_gather=G.r_gemm_gather, gemm_box=G.r_gemm_box, gemm_halo=G.r_gemm_halo)
    dev = prods[0]["support"].device
    N, rows = red["N"], red["splits"]
    cs, cs_ref, cs_mag = (torch.full((rows * N,), v, dtype=torch.float32, device=dev) for v in (float("nan"), float("nan"), 0.0))
    terms = sum(p["geom"].M * p["w"]["shape"][1] * p["w"]["shape"][2] for p in prods) / N
    pa = prods[0]["x"]["shape"][0]
    res = 1.0 if mode == "dense" else 2.0 ** (-2 * (pa - 1))
    outs = []
    for p in prods:
        sl = lambda t: t[(p["ptr"] - red["ptr"]) // 4:][:p["bytes"] // 4].view(p["colsum"]["shape"])
        A = _build(p["x"], fill(p["x"]["shape"][1:], pa, mode, gen, density_for(terms, mode), device=dev)
                   * p["support"][None, ..., None])
        W = _build(p["w"], fill(p["w"]["shape"][1:], p["w"]["shape"][0], "dense", gen, 0.5, device=dev))     # plane 0 only
        mask = _build(p["mask"], torch.randn(p["mask"]["shape"], generator=gen, device=dev)) if p["mask"] else None
        out = _build(p["out"], torch.randn(p["out"]["shape"], generator=gen, device=dev))                  # sentinel
        ref_out = out.clone()
        launches[p["kind"]](A, W, p["geom"], out_pl=out, relu_mask=mask, colsum=sl(cs), **p["kw"])
        restated[p["kind"]](A, W, p["geom"], out_pl=ref_out, relu_mask=mask, colsum=sl(cs_ref), **p["kw"])
        restated[p["kind"]](A.abs(), W.abs(), p["geom"], out_pl=ref_out.clone(), relu_mask=mask, colsum=sl(cs_mag), **p["kw"])
        outs.append((p["kind"], out, ref_out))
    what = "%s%s %s rows=%d N=%d" % (tag, "+".join(p["kind"] for p in prods), mode, rows, N)
    worst = check_premise(cs_mag.double().view(-1, N).sum(0), res, what)
    for kind, out, ref_out in outs:
        _expect_equal(out, ref_out, what + " %s output planes" % kind)
    _expect_equal(cs.view(-1, N), cs_ref.view(-1, N), what + " column sums (row, column)")
    want = cs_ref.double().view(-1, N).sum(0).float()
    order = reduce_ref(cs.view(-1, 1, N), N, 1, 1, 1, sm_count=sm_count).view(N)
    got = launches["wgrad_reduce"](cs.clone().view(-1, 1, N), N, 1, 1, 1).view(N)
    _expect_equal(got, want, what + " bias")
    _expect_equal(got, order, what + " bias vs the reduce's order")
    prev = torch.randn(N, generator=gen, device=dev)
    got = launches["wgrad_reduce"](cs.clone().view(-1, 1, N), N, 1, 1, 1, out=prev.clone(), accumulate=True).view(N)
    _expect_equal(got, prev + want, what + " bias added into an existing gradient")
    return worst


def replay(rec, launches, modes=("dense", "sparse"), seed=0, sm_count=None, tag=""):
    """Every chain ``rec`` recorded, in both fillings.  Returns {(kind, mode): largest sum |terms| / res}."""
    worst = {}
    for i, (prods, red) in enumerate(rec.chains()):
        kind = "+".join(sorted({p["kind"] for p in prods}))
        for j, mode in enumerate(modes):
            dev = prods[0]["support"].device
            gen = torch.Generator(device=dev).manual_seed(seed * 1000 + 10 * i + j)
            fn = replay_colsum if prods[0]["kind"].startswith("gemm") else replay_wgrad
            w = fn(prods, red, launches, mode, gen, sm_count, tag) if fn is replay_colsum else fn(prods[0], red, launches, mode, gen, sm_count, tag)
            key = (kind + (" N=%d" % red["N"] if fn is replay_colsum else " K=%d" % (red["C"] * red["KH"] * red["KW"])), mode)
            worst[key] = max(worst.get(key, 0.0), w)
    return worst
