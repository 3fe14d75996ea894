"""Two (or more) processes, one GPU each: MaskedSyncBatchNorm1d over the peer exchange (CUDA IPC peer memory)
against the same layer over NCCL (torch.distributed.all_gather_into_tensor).  Both move the per-rank vectors
unchanged, so y, dx, the statistics, the running stats and dweight / dbias must be identical bit for bit.  Run:
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/sync_bn_check.py
Prints "sync_bn_check OK" on rank 0; exit code != 0 on any mismatch."""
import copy
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import spconv_b200.pytorch as spconv  # noqa: E402
from spconv_b200.pytorch import MaskedSyncBatchNorm1d, ops  # noqa: E402
from spconv_b200.pytorch.dist import PeerGroup  # noqa: E402


def run(bn, x, dy, nv, inds):
    xr = x.clone().requires_grad_(True)
    t = spconv.SparseConvTensor(xr, inds, [8, 8, 8], 1)
    t.num_valid = nv
    y = bn(t).features
    y.backward(dy)
    return [y.detach(), xr.grad, bn.weight.grad, bn.bias.grad, *bn.buffers()]


def main():
    rank = int(os.environ["RANK"])
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    peers = PeerGroup(capacity_bytes=1 << 20)
    for it, (c, dtype, m) in enumerate([(64, torch.float16, 5000), (12, torch.float32, 700), (128, torch.bfloat16, 0),
                                        (64, torch.float16, 1)]):
        g = torch.Generator(device=dev).manual_seed(100 * it + rank)
        valid = m * (rank + 1)                                    # rank 0 of the third case has no rows at all
        rows = valid + 37
        x = (torch.randn((rows, c), generator=g, device=dev) * 2 + 0.5).to(dtype)
        dy = torch.randn((rows, c), generator=g, device=dev).to(dtype)
        nv = torch.tensor([valid], dtype=torch.int32, device=dev)
        inds = torch.zeros((rows, 4), dtype=torch.int32, device=dev)
        base = MaskedSyncBatchNorm1d(c, momentum=None if it % 2 else 0.1).to(dev)
        with torch.no_grad():
            base.weight.uniform_(0.5, 1.5, generator=torch.Generator(device=dev).manual_seed(it))
        ops.set_peer_group(None)
        nccl = run(copy.deepcopy(base), x, dy, nv, inds)
        ops.set_peer_group(peers)
        peer = run(copy.deepcopy(base), x, dy, nv, inds)
        ops.set_peer_group(None)
        for i, (a, b) in enumerate(zip(nccl, peer)):
            if not torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8)):
                raise SystemExit(f"rank {rank} case {it}: result {i} differs between the NCCL and the peer route")
        stats = torch.cat([peer[4].float(), peer[5].float()])
        everyone = [torch.empty_like(stats) for _ in range(dist.get_world_size())]
        dist.all_gather(everyone, stats)
        if not all(torch.equal(e, everyone[0]) for e in everyone):
            raise SystemExit(f"case {it}: the running stats differ between ranks")
    torch.cuda.synchronize()
    if peers.error() != 0:
        raise SystemExit(f"rank {rank}: a peer exchange timed out")
    dist.barrier()
    peers.close()
    dist.destroy_process_group()
    if rank == 0:
        print("sync_bn_check OK")


if __name__ == "__main__":
    main()
