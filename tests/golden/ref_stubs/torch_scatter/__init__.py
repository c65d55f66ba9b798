"""Import stub: ``torch_scatter.scatter_add`` on ``Tensor.index_add_``, enough for the reference's coordination graph
(xuance/torch/rl_models/heads/coordination_graph.py, learners/multi_agent_rl/dcg_learner.py) to run on a machine
without torch_scatter.  TEST INFRASTRUCTURE ONLY - used by tests/golden/make_golden_dcg.py; never imported by the
product package."""
import torch


def scatter_add(src, index, dim=-1, out=None, dim_size=None):
    """out[..., index[i], ...] += src[..., i, ...] along ``dim`` (index one-dimensional, as the reference passes it),
    summed in index order into zeros of ``dim_size`` rows."""
    dim = dim % src.dim()
    if out is None:
        shape = list(src.shape)
        shape[dim] = int(dim_size) if dim_size is not None else int(index.max()) + 1 if index.numel() else 0
        out = torch.zeros(shape, dtype=src.dtype, device=src.device)
    return out.index_add_(dim, index.long(), src)
