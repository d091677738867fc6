from . import hdf5  # noqa: F401
from .dataset import (  # noqa: F401
    ShardedPretrainingDataset, DistributedSampler, BatchedPretrainingLoader, HeldOutSet, mask_batch,
    segment_ids_and_input_mask)
