"""Multi-GPU plumbing for the poser hot path: one process per GPU (torchrun), frames sharded contiguously across
ranks, NO data-path collective (every op of the path is per-sample: InstanceNorm / GroupNorm statistics, attention
and warps never cross frames; SURVEY.md section 8e).  The only optional collective is an all_gather of finished
frames for a caller that wants the whole sweep on every rank.  The reference has no counterpart for inference (its
only parallelism is DDP over the distillation batch, src/tha4/shion/core/training/distrib/distributed_trainer.py)."""
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist
from torch import Tensor

from tha4_b200.poser.poser import Poser


def shard_range(total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous [begin, end) slice of `total` items owned by `rank`; the first `total % world` ranks get one extra."""
    assert 0 <= rank < world and total >= 0
    base, extra = divmod(total, world)
    begin = rank * base + min(rank, extra)
    return begin, begin + base + (1 if rank < extra else 0)


class ShardedPoseSweep:
    """Runs a batch of poses of ONE character image through a poser, each rank handling its contiguous shard
    (a 512-pose sweep sharded across the GPUs of one box)."""

    def __init__(self, poser: Poser, rank: Optional[int] = None, world: Optional[int] = None, chunk: int = 16):
        self.poser = poser
        self.rank = dist.get_rank() if rank is None else rank
        self.world = dist.get_world_size() if world is None else world
        self.chunk = chunk

    def local_range(self, num_poses: int) -> Tuple[int, int]:
        return shard_range(num_poses, self.rank, self.world)

    def pose_local(self, image: Tensor, poses: Tensor, output_index: int = 0) -> Tensor:
        """Frames [n_local, 4, H, W] of this rank's shard of `poses` ([num_poses, 45], replicated on every rank)."""
        begin, end = self.local_range(poses.shape[0])
        frames: List[Tensor] = []
        for i in range(begin, end, self.chunk):
            p = poses[i:min(end, i + self.chunk)]
            img = image.unsqueeze(0).expand(p.shape[0], -1, -1, -1).contiguous() if image.dim() == 3 else image
            frames.append(self.poser.pose(img, p, output_index))
        if not frames:
            size = self.poser.get_image_size()
            return torch.empty((0, 4, size, size), dtype=self.poser.get_dtype(), device=poses.device)
        return torch.cat(frames, dim=0)

    def pose_all(self, image: Tensor, poses: Tensor, output_index: int = 0) -> Tensor:
        """All frames on every rank (one all_gather of padded shards; the only collective of the inference path)."""
        local = self.pose_local(image, poses, output_index)
        if self.world == 1:
            return local
        sizes = [shard_range(poses.shape[0], r, self.world) for r in range(self.world)]
        longest = max(e - b for b, e in sizes)
        padded = torch.zeros((longest,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        padded[:local.shape[0]] = local
        gathered = [torch.empty_like(padded) for _ in range(self.world)]
        dist.all_gather(gathered, padded)
        return torch.cat([g[:e - b] for g, (b, e) in zip(gathered, sizes)], dim=0)
