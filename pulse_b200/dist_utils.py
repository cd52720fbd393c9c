"""Multi-GPU plumbing: one process per GPU, `torch.distributed` (NCCL over NVLink / NVSwitch).

Replaces the Horovod calls the reference reaches through rl_games (SURVEY.md section 5):
  hvd.DistributedOptimizer gradient averaging (amp_agent.py:735-742)   -> average_gradients (one all-reduce on the flat bucket)
  hvd.sync_stats per epoch (common_agent.py:126-127)                    -> sync_running_stats
  hvd.average_value(kl) (amp_agent.py:508,524)                          -> average_scalar
  rank -> device / seed offset (run_hydra.py:117-131)                   -> rank_device_seed
The env axis is the only sharded axis (SURVEY 8e): rank r owns envs [r*N/G, (r+1)*N/G) and their MotionLib clips.
"""
from typing import Tuple

import torch
import torch.distributed as dist


def env_shard(total_envs: int, rank: int, world: int) -> Tuple[int, int]:
    """[start, stop) of the envs owned by `rank`; the remainder goes to the lowest ranks."""
    if not (0 <= rank < world):
        raise ValueError(f"rank {rank} outside world {world}")
    base, rem = divmod(total_envs, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def minibatches_per_rank(envs_per_rank: int, horizon: int, minibatch_size: int) -> int:
    """rl_games A2CBase: num_minibatches = batch_size // minibatch_size with the PER-RANK minibatch kept fixed."""
    batch = envs_per_rank * horizon
    if batch % minibatch_size:
        raise ValueError(f"per-rank batch {batch} is not a multiple of minibatch_size {minibatch_size}")
    return batch // minibatch_size


def rank_device_seed(base_seed: int, rank: int) -> Tuple[str, int]:
    """run_hydra.py:117-131: device cuda:rank, seed = base + rank."""
    return f"cuda:{rank}", base_seed + rank


def average_gradients(flat_grads: torch.Tensor, world: int) -> None:
    """One all-reduce (sum) + scale on the flat gradient buffer; NCCL's AVG op on GPUs."""
    if world <= 1:
        return
    if flat_grads.is_cuda:
        dist.all_reduce(flat_grads, op=dist.ReduceOp.AVG)
    else:  # gloo has no AVG
        dist.all_reduce(flat_grads, op=dist.ReduceOp.SUM)
        flat_grads.div_(world)


def average_scalar(x: torch.Tensor, world: int) -> torch.Tensor:
    if world > 1:
        average_gradients(x, world)
    return x


def sync_running_stats(mean: torch.Tensor, var: torch.Tensor, count: torch.Tensor, world: int) -> None:
    """HorovodWrapper.sync_stats [3P-memory]: all-reduce-average every running-statistics tensor once per epoch."""
    if world <= 1:
        return
    for t in (mean, var, count):
        average_gradients(t, world)


class ChainReducer:
    """Gradient averaging that OVERLAPS with the backward pass: the flat gradient buffer holds the actor, critic and discriminator slices
    back to back, and each network's backward chain runs on its own CUDA stream (ppo.PPOPolicy.train_minibatch) -- so each slice is
    all-reduced on ITS stream as soon as that chain has produced it, through its own communicator (one NCCL communicator serialises its
    collectives; three let the critic's and the discriminator's reductions run under the remaining GEMMs).  Only the reduction of the chain
    that finishes last is exposed.  Replaces the single 22 MB all-reduce after all chains joined (none of it overlapped) -- Horovod's DistributedOptimizer also reduces gradients as they become ready (amp_agent.py:735-742)."""

    def __init__(self, world: int, num_chains: int = 3):
        self.world = world
        self.groups = [None]
        if world > 1:
            for _ in range(num_chains - 1):        # every rank creates the groups in the same order
                self.groups.append(dist.new_group(ranks=list(range(world))))

    def reduce(self, grads_slice: torch.Tensor, chain: int) -> None:
        """Average `grads_slice` over the ranks on the CURRENT stream's timeline (chain 0 = default communicator)."""
        if self.world <= 1:
            return
        g = self.groups[chain % len(self.groups)]
        if grads_slice.is_cuda:
            dist.all_reduce(grads_slice, op=dist.ReduceOp.AVG, group=g)
        else:
            dist.all_reduce(grads_slice, op=dist.ReduceOp.SUM, group=g)
            grads_slice.div_(self.world)
