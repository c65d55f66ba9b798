"""One contiguous float32 bucket for a learner's parameters and gradients.

The reference leaves parameters as separate tensors and (for DQN / MARL models only) lets DistributedDataParallel
bucket their gradients (SURVEY.md section 2a).  Here every trainable parameter of the learner is re-homed into ONE
flat HBM array (``flat``) and its gradient into another (``grad``): ``p.data`` / ``p.grad`` become views, autograd
accumulates straight into the bucket, the multi-GPU step is a single NCCL all-reduce over ``grad``, and the
clip-norm + Adam step (K7) streams over the two arrays once."""
import torch

_ALIGN = 32  # elements (128 B): keeps every parameter view 128-byte aligned for cuDNN / cuBLAS vector loads


def cudnn_rnn_front(module):
    """The flat weights of the first ``nn.RNNBase`` inside ``module`` (or []).  cuDNN's RNN path uses the weights in place
    only when they sit, in ``_flat_weights`` order and back to back, at the START of their storage (ATen
    cudnn/RNN.cpp ``try_get_weight_buf``); anywhere else it re-packs them on every forward.  Passing this list as
    ``FlatBucket(..., front=)`` puts that one group at offset 0 of the bucket."""
    for m in module.modules():
        if isinstance(m, torch.nn.RNNBase):
            return [w for w in m._flat_weights if w is not None and w.requires_grad]
    return []


class FlatBucket:
    TAIL = 32   # float32 slots BEFORE the first gradient: per-update statistics ride in the same all-reduce as the gradient

    def __init__(self, params, front=()):
        """``front``: parameters to lay out first (see ``cudnn_rnn_front``); ``self.params`` keeps the caller's order."""
        seen, plist = set(), []
        for p in params:
            if p.requires_grad and id(p) not in seen:
                seen.add(id(p))
                plist.append(p)
        if not plist:
            raise ValueError("FlatBucket: no trainable parameters")
        dev = plist[0].device
        if dev.type != "cuda":
            raise RuntimeError("FlatBucket: parameters must live on a CUDA device (no CPU fallback)")
        self.params = plist
        first = [id(p) for p in front if id(p) in seen]
        layout = sorted(range(len(plist)), key=lambda i: (first.index(id(plist[i])) if id(plist[i]) in first
                                                          else len(first) + i))
        self.offsets, off = [0] * len(plist), 0
        for i in layout:
            p = plist[i]
            if p.dtype != torch.float32 or p.device != dev:
                raise ValueError("FlatBucket: all parameters must be float32 on one device")
            self.offsets[i] = off
            off += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
        self.numel = off
        self.flat = torch.zeros(off, dtype=torch.float32, device=dev)
        self.grad_all = torch.zeros(off + self.TAIL, dtype=torch.float32, device=dev)   # what a sharded learner all-reduces
        self.tail = self.grad_all[:self.TAIL]
        self.grad = self.grad_all[self.TAIL:]
        for p, o in zip(plist, self.offsets):
            v = self._view(self.flat, p, o)
            v.copy_(p.data)
            p.data = v
            p.grad = self._view(self.grad, p, o)

    @staticmethod
    def _view(buf, p, off):
        chunk = buf[off:off + p.numel()]
        if p.dim() == 4 and p.is_contiguous(memory_format=torch.channels_last) and not p.is_contiguous():
            o, i, h, w = p.shape
            return chunk.view(o, h, w, i).permute(0, 3, 1, 2)
        return chunk.view(p.shape)

    def views(self, buf):
        return [self._view(buf, p, o) for p, o in zip(self.params, self.offsets)]

    def zero_grad(self):
        self.grad.zero_()
        for p, o in zip(self.params, self.offsets):  # re-attach if someone set .grad to None
            if p.grad is None or p.grad.data_ptr() != self.grad.data_ptr() + 4 * o:
                p.grad = self._view(self.grad, p, o)


def target_bucket(target, live):
    """A target network's parameters re-homed into their own flat array, in the ``live`` bucket's parameter order and
    layout, so that one K7 ``xb_soft_update`` streams the Polyak update over the two arrays.  The target's parameters
    stay frozen (no gradient)."""
    params = list(target.parameters())
    bucket = FlatBucket([p.requires_grad_(True) for p in params])
    for p in params:
        p.requires_grad_(False)
        p.grad = None
    assert bucket.numel == live.numel and bucket.offsets == live.offsets
    return bucket
