"""torchrun target (>= 2 GPUs): ops.whiten_advantages across data-parallel ranks against one whitening of every rank's
micro-batches in a single process.  Ranks hold different numbers of micro-batches of different widths.  Launched by
tests/test_gpu_whiten.py or by hand:
    torchrun --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29541 tests/dist_whiten.py
"""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from align_anything_b200 import ops  # noqa: E402

local = int(os.environ.get('LOCAL_RANK', '0'))
torch.cuda.set_device(local)
dev = torch.device('cuda', local)
dist.init_process_group('nccl', device_id=dev)
rank, world = dist.get_rank(), dist.get_world_size()
alone = [dist.new_group([r]) for r in range(world)]  # every rank creates every group, in the same order


def micro_batches(r):
    """Rank r's micro-batches: r + 1 of them, of different widths, with masked-out NaNs and rank-dependent means."""
    g = torch.Generator().manual_seed(100 + r)
    advs, masks = [], []
    for k in range(r + 1):
        B, W = 2 + k, 50 + 37 * r + 11 * k
        a = torch.randn(B, W, generator=g) * (1.0 + r) + 3.0 * r
        m = torch.rand(B, W, generator=g) < 0.6
        a[~m] = float('nan')
        advs.append(a.to(dev))
        masks.append(m.to(dev))
    return advs, masks


for dtype in (torch.float32, torch.bfloat16):
    mine = micro_batches(rank)
    got = ops.whiten_advantages([a.to(dtype) for a in mine[0]], mine[1])
    everyone = [micro_batches(r) for r in range(world)]
    all_advs = [a.to(dtype) for advs, _ in everyone for a in advs]
    all_masks = [m for _, masks in everyone for m in masks]
    dist.barrier()
    single = ops.whiten_advantages(all_advs, all_masks, group=alone[rank])
    first = sum(r + 1 for r in range(rank))
    for g, s in zip(got, single[first:first + rank + 1]):
        # the rank sums arrive through NCCL's reduction, the single process sums the slots in order: the fp64 totals
        # may differ in the last bits, the fp32 mean and rstd almost never
        d = (g.float() - s.float()).abs().max()
        tol = 1e-6 if dtype == torch.float32 else 8e-3
        assert float(d) <= tol * max(1.0, float(s.float().abs().max())), (dtype, float(d))
ops.check_status()
torch.cuda.synchronize()
dist.barrier()
if rank == 0:
    print(f'WHITEN DIST OK world={world}')
dist.destroy_process_group()
