"""Host-side logic of the sharded decode on CPU: the Python seam verdict on crafted seam words, and a world-2 gloo run of the
seam-word exchange (no CUDA calls)."""
import os
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT


def words(*rows):
    """rows of (first inc, last inc, not quiet, has blocks, size)"""
    return torch.tensor([[f, l, q, h, s & 0xFFFFFFFF, s >> 32, 0, 0] for f, l, q, h, s in rows], dtype=torch.int64).to(torch.int32)


def test_seam_verdict_quiet():
    from density_b200.sharded import seam_verdict
    flags, total, offsets = seam_verdict(words((1, 0, 0, 1, 1024), (0, 1, 0, 1, 512), (0, 0, 0, 1, 77)))
    assert flags == 0 and total == 1024 + 512 + 77
    assert offsets.tolist() == [0, 1024, 1536, 1613]


def test_seam_verdict_cross_seam_pair():
    from density_b200.sharded import seam_verdict
    assert seam_verdict(words((0, 1, 0, 1, 256), (1, 0, 0, 1, 256)))[0] == 1
    assert seam_verdict(words((0, 1, 0, 1, 256), (0, 1, 0, 1, 256)))[0] == 0
    assert seam_verdict(words((0, 0, 0, 1, 256), (0, 0, 1, 1, 256)))[0] == 1      # a piece that is not quiet


def test_seam_verdict_skips_empty_pieces():
    from density_b200.sharded import seam_verdict
    # an empty middle piece (no blocks) does not break the seam between the pieces around it
    assert seam_verdict(words((0, 1, 0, 1, 256), (0, 0, 0, 0, 0), (1, 0, 0, 1, 256)))[0] == 1
    flags, total, offsets = seam_verdict(words((0, 0, 0, 1, 256), (0, 0, 0, 0, 0), (1, 0, 0, 1, 300)))
    assert flags == 0 and total == 556 and offsets.tolist() == [0, 256, 256, 556]


def test_seam_verdict_sizes_beyond_4gib():
    from density_b200.sharded import seam_verdict
    big = (5 << 32) + 0xFFFFFF00
    flags, total, offsets = seam_verdict(words((0, 0, 0, 1, big), (0, 0, 0, 1, 3)))
    assert flags == 0 and total == big + 3 and offsets.tolist() == [0, big, big + 3]


def _worker(rank, world, port, rows, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from density_b200 import sharded
    mine = words(rows[rank])[0]
    gathered = sharded.gather_rows(mine)
    flags, total, offsets = sharded.seam_verdict(gathered)
    q.put((rank, gathered.numpy().copy(), flags, total, offsets.tolist()))
    dist.barrier()
    dist.destroy_process_group()


def test_seam_word_gather_rows_world2_gloo():
    world = 2
    rows = [(0, 1, 0, 1, 1 << 20), (1, 0, 0, 1, 4099)]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, 29617, rows, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict((r, rest) for r, *rest in (q.get(timeout=120) for _ in range(world)))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want = words(*rows).numpy()
    for r in range(world):
        g, flags, total, offsets = got[r]
        assert (g == want).all()
        assert flags == 1 and total == (1 << 20) + 4099 and offsets == [0, 1 << 20, (1 << 20) + 4099]
