"""ValueNorm - mirror of xuance/torch/utils/value_norm.py:6-75 (input_shape 1, norm_axes 1, beta 0.99999, no
per-element update).  Same parameter names (``running_mean``, ``running_mean_sq``, ``debiasing_term``), so checkpoints
interchange with the reference.  The state lives on the device and is updated there by ``xb_value_norm_update`` from
the moments ``xb_mappo_prepare`` leaves in a small float64 block; ``mean_std`` holds (mean, std) of the updated state
for the loss kernel.  No host synchronisation: the update is capturable in a CUDA graph."""
import numpy as np
import torch
import torch.nn as nn

from ... import _lib


class ValueNorm(nn.Module):
    def __init__(self, input_shape, norm_axes=1, beta=0.99999, per_element_update=False, epsilon=1e-5, device=None):
        super().__init__()
        if input_shape not in (1, (1,)) or norm_axes != 1 or per_element_update or epsilon != 1e-5:
            raise NotImplementedError("ValueNorm: only the scalar value normaliser of the MARL learners is on the hot path")
        self.input_shape, self.norm_axes, self.epsilon, self.beta = input_shape, norm_axes, epsilon, beta
        self.per_element_update = per_element_update
        self.running_mean = nn.Parameter(torch.zeros(input_shape, device=device), requires_grad=False)
        self.running_mean_sq = nn.Parameter(torch.zeros(input_shape, device=device), requires_grad=False)
        self.debiasing_term = nn.Parameter(torch.tensor(0.0, device=device), requires_grad=False)
        self.register_buffer("mean_std", torch.tensor([0.0, 1.0], device=device), persistent=False)

    def reset_parameters(self):
        with torch.no_grad():
            self.running_mean.zero_()
            self.running_mean_sq.zero_()
            self.debiasing_term.zero_()

    def state_pointers(self):
        """(running_mean, running_mean_sq, debiasing_term) device pointers, as xb_gae_scan_vn reads them."""
        return _lib.ptr(self.running_mean), _lib.ptr(self.running_mean_sq), _lib.ptr(self.debiasing_term)

    def update_from_block(self, block, rows_total):
        """ValueNorm.update on the targets whose (sum, sum of squares) are block[1:3] over ``rows_total`` rows."""
        _lib.call("xb_value_norm_update", *self.state_pointers(), _lib.ptr(block), int(rows_total), float(self.beta),
                  _lib.ptr(self.mean_std))

    # ---- host-side conveniences with the reference's semantics (not on the update path)
    def running_mean_var(self):
        d = self.debiasing_term.clamp(min=self.epsilon)
        mean, mean_sq = self.running_mean / d, self.running_mean_sq / d
        return mean, (mean_sq - mean ** 2).clamp(min=1e-2)

    @torch.no_grad()
    def update(self, input_vector):
        x = torch.as_tensor(input_vector, dtype=torch.float32, device=self.running_mean.device).reshape(-1).contiguous()
        block = torch.zeros(4, dtype=torch.float64, device=x.device)
        _lib.call("xb_mappo_prepare", _lib.ptr(x), _lib.ptr(x), x.numel(), _lib.ptr(block),
                  _lib.ptr(_lib.scratch(x.device)))
        self.update_from_block(block, x.numel())

    def normalize(self, input_vector):
        x = torch.as_tensor(input_vector, device=self.running_mean.device)
        mean, var = self.running_mean_var()
        return (x - mean) / torch.sqrt(var)

    def denormalize(self, input_vector):
        x = torch.as_tensor(input_vector, device=self.running_mean.device)
        mean, var = self.running_mean_var()
        return (x * torch.sqrt(var) + mean).cpu().numpy()
