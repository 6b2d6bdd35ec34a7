"""world_size-2 gloo test of the multi-GPU sharding logic (host side): block partition, row shards,
and the single all-reduce at the Schur-assembly boundary.  The per-rank compute is the oracle
(reference getada chain) so the test runs without a GPU; on GPUs bench.py --shard runs the
same logic with the CUDA kernels and NCCL."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from helpers import ROOT, needs_reference
from sedumi_b200.host import cones, problems, setup, shard

sys.path.insert(0, os.path.join(ROOT, "oracle"))

needs_ref = needs_reference("test_shard_cpu", "getada3")


def test_partition_is_balanced_and_complete():
    s = [200] * 64
    parts = shard.partition_blocks(s, 8)
    assert sorted(sum(parts, [])) == list(range(64)) and all(len(p) == 8 for p in parts)
    parts = shard.partition_blocks([70, 35], 2)
    assert parts == [[0], [1]]
    parts = shard.partition_blocks([10, 50, 20, 49, 5], 2)
    loads = [sum(np.array([10, 50, 20, 49, 5])[p] ** 3) for p in parts]
    assert max(loads) / min(loads) < 1.2


def _worker(rank, world, port, out, compact):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import refpath
    import replay
    caller = os.environ["PYTEST_CURRENT_TEST"].rsplit(" (", 1)[0] + f"/rank{rank}"     # one record per rank
    with replay.context(caller):
        _assemble(rank, world, out, compact, refpath)
    replay.finish(caller)


def _assemble(rank, world, out, compact, refpath):
    raw = problems.synth_blockdiag_sdp(nblk=6, n=8, m=40, nlink=5, density=0.15, seed=3)
    At, b, c, K = cones.pretransfo(*raw)[:4]
    S = setup.build_setup(At, b, c, K, perm=np.arange(At.shape[1]))
    d = problems.scaling(K, "S1", seed=5)
    owned = shard.partition_blocks(K["s"], world)[rank]
    if compact:
        T, dr = shard.shard_compact(S, d, owned, rank)      # owner-computes cone: only this rank's PSD blocks
        assert list(T.K["s"]) == [K["s"][k] for k in owned]
    else:
        T, dr = shard.shard_setup(S, owned, rank), d
    udsqr, ADA, absd = refpath.RefHotPath(T).assemble(dr)
    vals = torch.from_numpy(ADA.data.copy())
    ab = torch.from_numpy(absd.ravel().copy())
    dist.all_reduce(vals)                       # the one collective of the path
    dist.all_reduce(ab)
    if rank == 0:
        _, full, absd_full = refpath.RefHotPath(S).assemble(d)
        out["ada"] = float(np.linalg.norm(vals.numpy() - full.data) / np.linalg.norm(full.data))
        out["absd"] = float(np.linalg.norm(ab.numpy() - absd_full.ravel()) / np.linalg.norm(absd_full))
    dist.barrier()
    dist.destroy_process_group()


@needs_ref
@pytest.mark.parametrize("compact", [False, True])
def test_sharded_assembly_equals_full_world2(compact):
    mgr = mp.Manager()
    out = mgr.dict()
    port = 29500 + (os.getpid() + 7 * int(compact)) % 2000
    mp.spawn(_worker, args=(2, port, out, compact), nprocs=2, join=True)
    assert out["ada"] <= 1e-12 and out["absd"] <= 1e-12
