"""Observation encoders (reference: xuance/torch/rl_models/representations/{mlp,cnn}.py).

``Basic_CNN`` / ``AC_CNN_Atari`` accept exactly what the reference accepts (uint8 / float NHWC arrays or
tensors -> ``x / 255.0`` -> float32 -> NCHW, cnn.py:45-50, 98-102) AND the two device-side fast inputs of this
repo: a CUDA uint8 tensor (converted by the K3 kernel, u8/255 correctly rounded, written straight in the layout
the convolutions run in) or a ``PreparedObs`` produced by the buffer's fused gather.  ``compute`` selects how the
convolution stack runs: 'fp32' (strict IEEE fp32, TF32 off - the reference's CPU arithmetic), 'tf32' (PyTorch's
default conv behaviour on GPUs), 'bf16' (autocast, channels-last)."""
import numpy as np
import torch
import torch.nn as nn

from ... import _lib
from ...common.memory_tools import PreparedObs
from .layers import cnn_block, mlp_block
from .outputs import RepresentationOutput


class Basic_Identical(nn.Module):
    def __init__(self, input_shape, device=None, **kwargs):
        super().__init__()
        assert len(input_shape) == 1
        self.output_shapes = {'state': (input_shape[0],)}
        self.device = device

    def forward(self, observations, **kwargs):
        return RepresentationOutput(embeddings=torch.as_tensor(observations, dtype=torch.float32, device=self.device))


class Basic_MLP(nn.Module):
    def __init__(self, input_shape, hidden_sizes, normalize=None, initialize=None, activation=None, device=None,
                 **kwargs):
        super().__init__()
        self.input_shape, self.hidden_sizes, self.device = input_shape, hidden_sizes, device
        self.output_shapes = {'state': (hidden_sizes[-1],)}
        layers, shape = [], input_shape
        for h in hidden_sizes:
            mlp, shape = mlp_block(shape[0], h, normalize, activation, initialize, device=device)
            layers.extend(mlp)
        self.model = nn.Sequential(*layers)

    def forward(self, observations, **kwargs):
        x = torch.as_tensor(observations, dtype=torch.float32, device=self.device)
        return RepresentationOutput(embeddings=self.model(x))


class _PixelEncoder(nn.Module):
    """Shared input handling for the two CNN encoders."""

    compute = "fp32"

    def set_compute(self, mode):
        assert mode in ("fp32", "fp32_cl", "tf32", "bf16", "tc")
        if mode == "tc":
            self._build_tc()
        self.compute = mode
        fmt = torch.channels_last if mode not in ("fp32", "tc") else torch.contiguous_format
        for m in self.model:
            if isinstance(m, nn.Conv2d):
                m.to(memory_format=fmt)
        return self

    def preferred_obs_format(self):
        """K3 output format this encoder consumes without any further copy."""
        if self.compute == "tc":
            return _lib.OBS_PLANE_RAW      # one exact bf16 plane of the uint8 pixels; the 1/255 lives in conv1's packed weights
        return {"fp32": _lib.OBS_F32_NCHW, "fp32_cl": _lib.OBS_F32_NHWC, "tf32": _lib.OBS_F32_NHWC,
                "bf16": _lib.OBS_BF16_NHWC}[self.compute]

    # ---- "tc" mode: the conv stack + hidden layer as K12 launches (split-bf16 wgmma GEMMs, float32 accumulation,
    # utils/tc_conv.py): forward, data gradients and weight gradients; pinned against float64 in tests/test_gpu_tc_conv.py.
    def _build_tc(self):
        import os
        from ..utils.tc_conv import TensorCoreNatureCNN, BoxNatureCNN, CudaBackend
        mods = list(self.model)
        convs, fc, i = [], None, 0
        while i + 1 < len(mods) and isinstance(mods[i], nn.Conv2d) and isinstance(mods[i + 1], nn.ReLU):
            convs.append(mods[i])
            i += 2
        rest = mods[i:]
        hidden = (len(rest) == 3 and isinstance(rest[0], nn.Flatten) and isinstance(rest[1], nn.Linear)
                  and isinstance(rest[2], nn.ReLU))                                     # AC_CNN_Atari, one hidden layer
        pooled = len(rest) == 2 and isinstance(rest[0], nn.AdaptiveMaxPool2d) and isinstance(rest[1], nn.Flatten)  # Basic_CNN
        if not convs or not (hidden or pooled):
            raise NotImplementedError("compute='tc' covers Conv2d+ReLU stacks followed by Flatten, Linear, ReLU "
                                      "(AC_CNN_Atari with one hidden layer) or by AdaptiveMaxPool2d(1,1), Flatten (Basic_CNN)")
        C, H, W = self.input_shape
        # padded-row activations + TMA boxes for the convolutions after the first when the stack has the NatureCNN shape
        # (XB_K12_BOX=0 / XB_K12_TMA=0 keep the gathered cp.async path for every convolution)
        cls = TensorCoreNatureCNN
        probe = BoxNatureCNN(convs, rest[1] if hidden else None, (H, W, C))
        if probe._box_ok() and os.environ.get("XB_K12_BOX", "1") != "0" and os.environ.get("XB_K12_TMA", "1") != "0":
            cls = BoxNatureCNN
        self._tc = cls(convs, rest[1] if hidden else None, (H, W, C), backend=CudaBackend(planes=getattr(self, "tc_planes", 3)))
        self._tc_pooled = pooled

    def _run_tc(self, observations):
        from ..utils import tc_conv
        P = self._tc.be.planes
        if isinstance(observations, np.ndarray) and observations.dtype == np.uint8:
            observations = torch.from_numpy(observations).to(self.device)
        if isinstance(observations, PreparedObs) and observations.fmt in (_lib.OBS_PLANES2, _lib.OBS_PLANES3, _lib.OBS_PLANE_RAW):
            planes = observations.tensor                                   # K3-P already produced [P, B, H, W, C]
        elif isinstance(observations, torch.Tensor) and observations.is_cuda and observations.dtype == torch.uint8 \
                and observations[0].numel() % 16 == 0:
            obs = observations.contiguous()                                # raw pixels -> one exact plane
            planes = torch.empty((1,) + tuple(obs.shape), dtype=torch.bfloat16, device=obs.device)
            _lib.call("xb_gather_obs_planes", _lib.ptr(obs), None, obs.shape[0], obs[0].numel(), 1, _lib.ptr(planes))
        else:
            x = self._as_input_f32_nhwc(observations)
            planes = tc_conv.split_bf16(x, P)
        B = planes.shape[1]
        z = tc_conv.tc_encode(self._tc, planes, B) if torch.is_grad_enabled() else self._tc.forward(planes, B, keep=False)
        if self._tc_pooled:         # [B*OY*OX, C] NHWC rows of the last convolution -> global max over the sites (cnn.py:47-48)
            z = z.view(B, -1, z.shape[-1]).amax(dim=1)
        return z

    def _as_input_f32_nhwc(self, observations):
        """float32 NHWC u8/255 for inputs that are neither a planes batch nor a CUDA uint8 tensor (host arrays, floats)."""
        if isinstance(observations, PreparedObs):
            x = observations.tensor if observations.fmt != _lib.OBS_F32_NCHW else observations.tensor.permute(0, 2, 3, 1)
            return x.float().contiguous()
        if isinstance(observations, np.ndarray):
            observations = torch.from_numpy(observations).to(self.device)
        return (observations / 255.0).to(dtype=torch.float32, device=self.device).contiguous()

    def _as_input(self, observations):
        fmt = self.preferred_obs_format()
        if isinstance(observations, PreparedObs):
            x = observations.tensor
            return x if observations.fmt == _lib.OBS_F32_NCHW else x.permute(0, 3, 1, 2)
        if isinstance(observations, torch.Tensor) and observations.is_cuda and observations.dtype == torch.uint8:
            obs = observations.contiguous()
            B, H, W, C = obs.shape
            if (H * W * C) % 16 == 0 and (fmt != _lib.OBS_F32_NCHW or (C == 4 and W % 4 == 0)):
                dt = torch.bfloat16 if fmt == _lib.OBS_BF16_NHWC else torch.float32
                shape = (B, C, H, W) if fmt == _lib.OBS_F32_NCHW else (B, H, W, C)
                out = torch.empty(shape, dtype=dt, device=obs.device)
                _lib.call("xb_gather_obs", _lib.ptr(obs), None, B, H, W, C, _lib.ptr(out), fmt)
                return out if fmt == _lib.OBS_F32_NCHW else out.permute(0, 3, 1, 2)
        # reference path (cnn.py:98-101): true division, float32, NHWC -> NCHW view
        if isinstance(observations, np.ndarray):
            observations = torch.from_numpy(observations).to(self.device)
        observations = observations / 255.0
        return torch.as_tensor(observations, dtype=torch.float32, device=self.device).permute((0, 3, 1, 2))

    def _run(self, x):
        if self.compute == "bf16":
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return self.model(x).float()
        if x.dtype != torch.float32:
            x = x.float()
        return self.model(x)


class Basic_CNN(_PixelEncoder):
    """cnn.py:11-50: conv stack (config initialiser) -> AdaptiveMaxPool2d(1,1) -> Flatten -> filters[-1] features."""

    def __init__(self, input_shape, kernels, strides, filters, normalize=None, initialize=None, activation=None,
                 device=None, **kwargs):
        super().__init__()
        self.input_shape = (input_shape[2], input_shape[0], input_shape[1])
        self.kernels, self.strides, self.filters = kernels, strides, filters
        self.device = device
        self.output_shapes = {'state': (filters[-1],)}
        layers, shape = [], self.input_shape
        for k, s, f in zip(kernels, strides, filters):
            cnn, shape = cnn_block(shape, f, k, s, normalize, activation, initialize, device)
            layers.extend(cnn)
        layers.append(nn.AdaptiveMaxPool2d((1, 1)))
        layers.append(nn.Flatten())
        self.model = nn.Sequential(*layers)

    def forward(self, observations, **kwargs):
        if self.compute == "tc":
            return RepresentationOutput(embeddings=self._run_tc(observations))
        return RepresentationOutput(embeddings=self._run(self._as_input(observations)))


class AC_CNN_Atari(_PixelEncoder):
    """cnn.py:53-102: conv stack + Flatten + FC hidden layers, orthogonal(gain sqrt 2) weights, zero biases.
    With the reference's padding rule the 84x84x4 NatureCNN flattens to 6400 features (SURVEY appendix B #14)."""

    def __init__(self, input_shape, kernels, strides, filters, normalize=None, initialize=None, activation=None,
                 device=None, fc_hidden_sizes=(), **kwargs):
        super().__init__()
        self.input_shape = (input_shape[2], input_shape[0], input_shape[1])
        self.kernels, self.strides, self.filters = kernels, strides, filters
        self.device = device
        self.fc_hidden_sizes = fc_hidden_sizes
        self.output_shapes = {'state': (fc_hidden_sizes[-1],)}
        layers, shape = [], self.input_shape
        for k, s, f in zip(kernels, strides, filters):
            cnn, shape = cnn_block(shape, f, k, s, None, activation, None, device)
            cnn[0] = self._init_layer(cnn[0])
            layers.extend(cnn)
        layers.append(nn.Flatten())
        shape = (int(np.prod(shape, dtype=np.int64)),)
        for h in fc_hidden_sizes:
            mlp, shape = mlp_block(shape[0], h, None, activation, None, device)
            mlp[0] = self._init_layer(mlp[0])
            layers.extend(mlp)
        self.model = nn.Sequential(*layers)

    @staticmethod
    def _init_layer(layer, gain=np.sqrt(2), bias=0.0):
        nn.init.orthogonal_(layer.weight, gain=gain)
        nn.init.constant_(layer.bias, bias)
        return layer

    def forward(self, observations, **kwargs):
        if self.compute == "tc":
            return RepresentationOutput(embeddings=self._run_tc(observations))
        return RepresentationOutput(embeddings=self._run(self._as_input(observations)))


REGISTRY_Representation = {
    "Basic_Identical": Basic_Identical,
    "Basic_MLP": Basic_MLP,
    "Basic_CNN": Basic_CNN,
    "AC_CNN_Atari": AC_CNN_Atari,
}
