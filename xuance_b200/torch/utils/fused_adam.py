"""Flat-bucket Adam with fused global-norm clipping (K7, include/xb200.h).

Replaces ``torch.nn.utils.clip_grad_norm_`` + ``torch.optim.Adam.step`` as the reference learners call them
(e.g. xuance/torch/learners/policy_gradient/ppo_learner.py:18-22, 61-65): same update rule (Adam, betas
(0.9, 0.999), ``eps`` as given, no weight decay / amsgrad), same clip rule
(coef = min(1, max_norm / (total_norm + 1e-6))).  It IS a ``torch.optim.Optimizer`` so the reference's
``LinearLR`` scheduler, ``optimizer.state_dict()['param_groups'][0]['lr']`` logging and checkpoint format keep
working.  Two kernel launches per step, no host synchronisation."""
import math

import torch

from ... import _lib
from .flat_bucket import FlatBucket


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, front=()):
        params = list(params)
        if weight_decay != 0.0:
            raise NotImplementedError("weight_decay is not on the hot path (reference configs use 0)")
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False,
                        foreach=None, capturable=False, differentiable=False, fused=None)
        super().__init__(params, defaults)
        if len(self.param_groups) != 1:
            raise NotImplementedError("FusedAdam drives exactly one parameter group")
        self.bucket = FlatBucket(self.param_groups[0]["params"], front=front)
        dev = self.bucket.flat.device
        self.exp_avg = torch.zeros_like(self.bucket.flat)
        self.exp_avg_sq = torch.zeros_like(self.bucket.flat)
        self.step_count = 0
        self._hyper = torch.zeros(4, dtype=torch.float32, device=dev)
        self._hyper_host = torch.zeros(4, dtype=torch.float32)
        self._norm = torch.zeros(1, dtype=torch.float32, device=dev)
        self._scratch = _lib.scratch(dev)
        self._step_t = torch.zeros((), dtype=torch.float32)
        for p, m, v in zip(self.bucket.params, self.bucket.views(self.exp_avg), self.bucket.views(self.exp_avg_sq)):
            self.state[p] = {"step": self._step_t, "exp_avg": m, "exp_avg_sq": v}

    @property
    def grad_norm(self):
        """Device scalar: the (pre-clip, post-averaging) global gradient L2 norm of the last clipped step."""
        return self._norm

    def zero_grad(self, set_to_none=False):
        self.bucket.zero_grad()

    def prepare(self):
        """Host half of a step: advance the step count and upload (step_size, bc2_sqrt, lr) for the kernels.  Kept apart
        from ``launch`` so that a CUDA graph can capture the device half only."""
        group = self.param_groups[0]
        self._opt_called = True     # what LRScheduler.step() looks at to tell "optimizer stepped first"
        self.step_count += 1
        self._step_t.fill_(float(self.step_count))
        b1, b2 = group["betas"]
        t = self.step_count
        self._hyper_host[0] = group["lr"] / (1.0 - b1 ** t)
        self._hyper_host[1] = math.sqrt(1.0 - b2 ** t)
        self._hyper_host[2] = group["lr"]
        self._hyper.copy_(self._hyper_host)     # 16-byte pageable H2D: the driver stages it before returning

    @torch.no_grad()
    def launch(self, max_norm=None, grad_scale=1.0, write_back_grad=False):
        """Device half: [global-norm reduction] + clip + Adam over the flat bucket (graph-capturable)."""
        group = self.param_groups[0]
        b1, b2 = group["betas"]
        n = self.bucket.numel
        clip = float(max_norm) if max_norm is not None else -1.0
        if clip > 0:
            _lib.call("xb_grad_sumsq", _lib.ptr(self.bucket.grad), n, float(grad_scale), _lib.ptr(self._norm),
                      _lib.ptr(self._scratch))
        _lib.call("xb_adam_step", _lib.ptr(self.bucket.flat), _lib.ptr(self.bucket.grad), _lib.ptr(self.exp_avg),
                  _lib.ptr(self.exp_avg_sq), n, _lib.ptr(self._hyper), float(b1), float(b2), float(group["eps"]),
                  clip, _lib.ptr(self._norm), float(grad_scale), 1 if write_back_grad else 0)

    @torch.no_grad()
    def step(self, closure=None, max_norm=None, grad_scale=1.0, write_back_grad=False):
        """One Adam step over the bucket.  ``max_norm`` (float or None) applies clip_grad_norm_ semantics first;
        ``grad_scale`` multiplies the gradient (1/world_size after a sum all-reduce)."""
        self.prepare()
        self.launch(max_norm, grad_scale, write_back_grad)
        return None

    def snapshot(self):
        return (self.bucket.flat.clone(), self.exp_avg.clone(), self.exp_avg_sq.clone(), self.step_count)

    def restore(self, snap):
        self.bucket.flat.copy_(snap[0])
        self.exp_avg.copy_(snap[1])
        self.exp_avg_sq.copy_(snap[2])
        self.step_count = snap[3]
        self._step_t.fill_(float(self.step_count))

    def load_state_dict(self, state_dict):
        """Accepts a torch.optim.Adam state_dict (reference checkpoints) and copies it into the flat buffers."""
        groups = state_dict["param_groups"]
        for k in ("lr", "betas", "eps"):
            if k in groups[0]:
                self.param_groups[0][k] = groups[0][k]
        if "initial_lr" in groups[0]:
            self.param_groups[0]["initial_lr"] = groups[0]["initial_lr"]
        st = state_dict.get("state", {})
        # the saved ids enumerate the param group position by position (torch.optim.Optimizer.state_dict); the bucket holds
        # only the trainable, de-duplicated parameters, so map position -> parameter object -> bucket slot
        group_params = self.param_groups[0]["params"]
        saved_ids = groups[0]["params"]
        if len(saved_ids) != len(group_params):
            raise ValueError("optimizer checkpoint has %d parameters, this optimizer %d" % (len(saved_ids), len(group_params)))
        slot = {id(p): i for i, p in enumerate(self.bucket.params)}
        ms, vs = self.bucket.views(self.exp_avg), self.bucket.views(self.exp_avg_sq)
        for pos, pid in enumerate(saved_ids):
            if pid not in st:
                continue
            i = slot.get(id(group_params[pos]))
            if i is None:                     # frozen / duplicate parameter: no moments on this side
                continue
            m, v = st[pid]["exp_avg"], st[pid]["exp_avg_sq"]
            if tuple(m.shape) != tuple(ms[i].shape):
                raise ValueError("optimizer checkpoint: moment of parameter %d has shape %s, expected %s"
                                 % (pos, tuple(m.shape), tuple(ms[i].shape)))
            ms[i].copy_(m)
            vs[i].copy_(v)
            self.step_count = int(float(st[pid]["step"]))
        self._step_t.fill_(float(self.step_count))


class SegmentedAdam(FusedAdam):
    """One ``torch.optim.Adam`` over several parameter groups of which an update steps only some, as the reference's
    PPG learner uses it (ppg_learner.py:19): ``zero_grad()`` sets the gradients to None there, so a phase whose loss
    does not reach a group leaves that group's values, moments and per-parameter ``step`` alone, and
    ``clip_grad_norm_`` covers only the parameters that have a gradient.

    ``segments`` is a list of parameter lists; the flat bucket lays them out back to back, so segment k is the
    contiguous range ``bounds[k]`` and any run of consecutive segments is one range too.  A step over segments ``ks``
    is one K7 ``xb_grad_sumsq`` over their union (when clipping) and one ``xb_adam_step`` per segment with that
    segment's own (step_size, bc2_sqrt, lr) block, i.e. its own bias correction.  ``state_dict()`` shows each
    parameter's own ``step`` and no state for a parameter whose segment has never stepped, as torch's Adam does."""

    def __init__(self, segments, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
        segments = [[p for p in seg if p.requires_grad] for seg in segments]
        flat = [p for seg in segments for p in seg]
        if len({id(p) for p in flat}) != len(flat) or any(not seg for seg in segments):
            raise ValueError("SegmentedAdam: segments must be non-empty and disjoint")
        super().__init__(flat, lr, betas, eps)
        slot = {id(p): i for i, p in enumerate(self.bucket.params)}
        self.seg_params = segments
        self.bounds, end = [], 0
        for seg in segments:
            idx = [slot[id(p)] for p in seg]
            start = self.bucket.offsets[idx[0]]
            stop = max(self.bucket.offsets[i] + self.bucket.params[i].numel() for i in idx)
            assert start == end, "FlatBucket keeps the caller's order: segments are back to back"
            end = -(-stop // 32) * 32
            self.bounds.append((start, end))
        S = len(segments)
        self.seg_steps = [0] * S
        self._seg_step_t = [torch.zeros((), dtype=torch.float32) for _ in range(S)]
        self._seg_hyper = torch.zeros((S, 4), dtype=torch.float32, device=self.bucket.flat.device)
        self._seg_hyper_host = torch.zeros((S, 4), dtype=torch.float32)
        self.state.clear()
        self._views = list(zip(self.bucket.views(self.exp_avg), self.bucket.views(self.exp_avg_sq)))
        self._slot = slot

    def _sync_state(self, k):
        """The per-parameter state torch's Adam would hold for segment k (none before its first step)."""
        for p in self.seg_params[k]:
            if self.seg_steps[k] == 0:
                self.state.pop(p, None)
            else:
                m, v = self._views[self._slot[id(p)]]
                self.state[p] = {"step": self._seg_step_t[k], "exp_avg": m, "exp_avg_sq": v}

    def prepare(self, segments=None):
        """Host half: advance the step count of each segment in ``segments`` (default all) and upload the hyper-parameter
        blocks (one 16 * S byte H2D)."""
        group = self.param_groups[0]
        self._opt_called = True
        b1, b2 = group["betas"]
        for k in (range(len(self.bounds)) if segments is None else segments):
            self.seg_steps[k] += 1
            t = self.seg_steps[k]
            self._seg_step_t[k].fill_(float(t))
            self._seg_hyper_host[k, 0] = group["lr"] / (1.0 - b1 ** t)
            self._seg_hyper_host[k, 1] = math.sqrt(1.0 - b2 ** t)
            self._seg_hyper_host[k, 2] = group["lr"]
            if t == 1:
                self._sync_state(k)
        self._seg_hyper.copy_(self._seg_hyper_host)

    @torch.no_grad()
    def launch(self, max_norm=None, grad_scale=1.0, write_back_grad=False, segments=None):
        """Device half over ``segments`` (consecutive indices; default all): [norm of their gradient] + clip + Adam."""
        group = self.param_groups[0]
        b1, b2 = group["betas"]
        ks = list(range(len(self.bounds))) if segments is None else list(segments)
        if ks != list(range(ks[0], ks[-1] + 1)):
            raise ValueError("SegmentedAdam steps a run of consecutive segments, got %r" % (ks,))
        lo, hi = self.bounds[ks[0]][0], self.bounds[ks[-1]][1]
        clip = float(max_norm) if max_norm is not None else -1.0
        if clip > 0:
            _lib.call("xb_grad_sumsq", _lib.ptr(self.bucket.grad[lo:hi]), hi - lo, float(grad_scale),
                      _lib.ptr(self._norm), _lib.ptr(self._scratch))
        for k in ks:
            a, b = self.bounds[k]
            _lib.call("xb_adam_step", _lib.ptr(self.bucket.flat[a:b]), _lib.ptr(self.bucket.grad[a:b]),
                      _lib.ptr(self.exp_avg[a:b]), _lib.ptr(self.exp_avg_sq[a:b]), b - a, _lib.ptr(self._seg_hyper[k]),
                      float(b1), float(b2), float(group["eps"]), clip, _lib.ptr(self._norm), float(grad_scale),
                      1 if write_back_grad else 0)

    @torch.no_grad()
    def step(self, closure=None, max_norm=None, grad_scale=1.0, write_back_grad=False, segments=None):
        self.prepare(segments)
        self.launch(max_norm, grad_scale, write_back_grad, segments)

    def snapshot(self):
        return (self.bucket.flat.clone(), self.exp_avg.clone(), self.exp_avg_sq.clone(), list(self.seg_steps))

    def restore(self, snap):
        self.bucket.flat.copy_(snap[0])
        self.exp_avg.copy_(snap[1])
        self.exp_avg_sq.copy_(snap[2])
        self.seg_steps = list(snap[3])
        for k, t in enumerate(self.seg_steps):
            self._seg_step_t[k].fill_(float(t))
            self._sync_state(k)

    def load_state_dict(self, state_dict):
        """A torch.optim.Adam state_dict (the reference's checkpoints): moments and each segment's step count from the
        saved per-parameter state; a segment without saved state starts unstepped."""
        super().load_state_dict(state_dict)
        st = state_dict.get("state", {})
        pos_of = {id(p): i for i, p in enumerate(self.param_groups[0]["params"])}
        saved_ids = state_dict["param_groups"][0]["params"]
        for k, seg in enumerate(self.seg_params):
            pid = saved_ids[pos_of[id(seg[0])]]
            self.seg_steps[k] = int(float(st[pid]["step"])) if pid in st else 0
            if pid not in st:
                a, b = self.bounds[k]
                self.exp_avg[a:b].zero_()
                self.exp_avg_sq[a:b].zero_()
        self.restore((self.bucket.flat, self.exp_avg, self.exp_avg_sq, self.seg_steps))
