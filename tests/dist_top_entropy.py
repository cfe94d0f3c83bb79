"""torchrun target (>= 2 GPUs): ops.entropy_quantile_threshold across data-parallel ranks against torch.quantile of every
rank's counted entropies concatenated.  The ranks hold different token counts, and the last rank counts none.
Launched by tests/test_gpu_top_entropy.py or by hand:
    torchrun --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29543 tests/dist_top_entropy.py
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


def rank_tokens(r):
    """Rank r's (B_r, K_r) entropies (ties, negative values, -0.0) and row_end; the last rank counts nothing."""
    g = torch.Generator().manual_seed(200 + r)
    B, K = 3 + 2 * r, 40 + 23 * r
    ent = torch.randint(-2, 9, (B, K), generator=g).float() * 0.375 + torch.rand(B, K, generator=g) * (r % 2)
    ent[0, 0] = -0.0
    row_end = torch.randint(1, K + 1, (B,), generator=g, dtype=torch.int32)
    if r == world - 1:
        row_end.zero_()
    return ent.to(dev), row_end.to(dev)


everyone = [rank_tokens(r) for r in range(world)]
values = torch.cat([e[torch.arange(e.size(1), device=dev) < re.unsqueeze(1)] for e, re in everyone])
ent, row_end = everyone[rank]
for q in (0.0, 0.3, 0.5, 0.8, 1.0):
    thr = ops.entropy_quantile_threshold(ent, row_end, q)
    want = torch.quantile(values, q)
    got = torch.stack([thr[0], want])
    allgot = [torch.empty_like(got) for _ in range(world)]
    dist.all_gather(allgot, got)
    for a in allgot:  # every rank holds the same threshold, and it is torch.quantile's
        assert float(a[0]) == float(want) and torch.equal(a[0].view(torch.int32), thr[0].view(torch.int32)), \
            (rank, q, float(a[0]), float(want))
torch.cuda.synchronize()
dist.barrier()
if rank == 0:
    print(f'TOP ENTROPY DIST OK world={world}')
dist.destroy_process_group()
