"""Data sharding across replica groups (reference: upstream torchft/data.py:24-77).

Fault tolerance keeps the WORLD elastic, so the dataset is sharded over the
*maximum* grid ``num_replica_groups x num_replicas``; when a replica group is down
its shard is simply skipped for those steps. For exactly-once semantics pair this
with a stateful dataloader checkpointed next to ``Manager.state_dict()``.
"""

from __future__ import annotations

from typing import Optional

import torch.distributed as dist
from torch.utils import data


class DistributedSampler(data.distributed.DistributedSampler):
    """Sampler for worker ``group_rank`` of replica group ``replica_rank``.

    global rank  = group_rank + num_replicas * replica_rank
    global world = num_replicas * num_replica_groups
    """

    def __init__(self, dataset: data.Dataset, replica_rank: int, num_replica_groups: int,
                 group_rank: Optional[int] = None, num_replicas: Optional[int] = None, **kwargs: object) -> None:
        if group_rank is None:
            group_rank = dist.get_rank()
        if num_replicas is None:
            num_replicas = dist.get_world_size()
        self.global_rank: int = group_rank + num_replicas * replica_rank
        self.global_world_size: int = num_replicas * num_replica_groups
        super().__init__(dataset, rank=self.global_rank, num_replicas=self.global_world_size, **kwargs)  # type: ignore[arg-type]
