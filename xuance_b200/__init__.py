"""xuance_b200 - H100-native rollout->update hot path behind the xuance.torch Agent / Learner / buffer API.

Host code is Python/PyTorch (device memory, streams, torch.distributed); every hot operation is a hand-written
sm_90a kernel reached through the C-ABI in include/xb200.h (libxb200.so, built in-tree by xuance_b200.build)."""
__version__ = "0.1.0"


def get_runner(*args, **kwargs):
    from .engine import get_runner as _g
    return _g(*args, **kwargs)
