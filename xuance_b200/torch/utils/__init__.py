from .flat_bucket import FlatBucket
from .fused_adam import FusedAdam, SegmentedAdam
from .distributed import init_distributed_mode, allreduce_sum_, shard_bounds, stratified_minibatches, world
from .graphs import CapturedStep
from .value_norm import ValueNorm
