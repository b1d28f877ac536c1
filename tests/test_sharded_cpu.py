"""Host-side logic of the multi-GPU path on CPU: world_size-2 gloo run of the table exchange + fold, checked against a
numpy model of the dictionary (no CUDA calls)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT, payload

M = np.uint32(0x9D6EF916)


def last_writer_table(data):
    """numpy model of what density_b200_shard_phase1 exports for a shard: touched<<16 | fingerprint of the last quad per bucket"""
    q = data[:data.size - data.size % 4].view(np.uint32)
    p = (q.astype(np.uint64) * np.uint64(M)).astype(np.uint32)
    h = (p >> np.uint32(16)).astype(np.int64)
    f = ((p & np.uint32(0xFFFE)) | (q >> np.uint32(31))).astype(np.int32)
    t = np.zeros(65536, np.int32)
    t[h] = f | 0x10000  # numpy assigns in order: the last writer wins
    return t


def _worker(rank, world, port, shards, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from density_b200 import sharded
    table = torch.from_numpy(last_writer_table(shards[rank]))
    gathered = sharded.gather_rows(table)
    carry = sharded.fold_tables(gathered, rank)
    q.put((rank, carry.numpy().copy()))
    dist.barrier()
    dist.destroy_process_group()


def test_gather_rows_and_fold_world2_gloo():
    world = 2
    data = payload("text", 2 * 65536, 4)
    shards = [data[:65536], data[65536:]]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, 29613, shards, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=120) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    init = np.zeros(65536, np.int32)
    init[0] = 0x10000
    assert (got[0] == init).all()
    t0 = last_writer_table(shards[0])
    want1 = np.where(t0 & 0x10000, t0, init)
    assert (got[1] == want1).all()


def test_fold_is_left_to_right():
    from density_b200 import sharded
    a = torch.zeros(65536, dtype=torch.int32); b = a.clone(); c = a.clone()
    a[5] = 0x10000 | 7; b[5] = 0x10000 | 9; c[6] = 0x10000 | 1
    g = torch.stack([a, b, c])
    assert sharded.fold_tables(g, 0)[0] == 0x10000 and sharded.fold_tables(g, 0)[5] == 0
    assert sharded.fold_tables(g, 1)[5] == (0x10000 | 7)
    assert sharded.fold_tables(g, 2)[5] == (0x10000 | 9)
    assert sharded.fold_tables(g, 3)[6] == (0x10000 | 1)
