"""Sharded Cheetah / Lion encode (needs an H100: pytest -m gpu): W shards of one input, run through the phase API on one device with
the library's folds, concatenate to exactly one cheetah_encode / lion_encode call whenever the seam verdict is 0, and the verdict
refuses what a later shard cannot encode alone."""
import ctypes

import numpy as np
import pytest

import oracle
import planted
from conftest import payload, splitmix_bytes

pytestmark = pytest.mark.gpu

CL = ("cheetah", "lion")
MIB = 1 << 20


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device; there is no CPU fallback")
    return torch


@pytest.fixture(scope="module")
def lib(torch_cuda):
    import density_b200
    return density_b200.load()


def _stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def encode_shards(torch, lib, alg, data, cuts):
    """The three shard phases of every shard on one device, the exchanges replaced by stacking the tables and folding them with
    density_b200_cl_table_init / _fold. Returns (pieces, (flags, total, offsets), seam words [world][8])."""
    from density_b200 import sharded
    aid = sharded.ALGS[alg]
    world = len(cuts) - 1
    ins, encs, tps, tcs, outs, sizes = [], [], [], [], [], []
    words = torch.zeros((world, 8), dtype=torch.int32, device="cuda")
    wp = lib.density_b200_cl_table_words(aid, sharded.CL_TABLE_P)
    wc = lib.density_b200_cl_table_words(aid, sharded.CL_TABLE_C)
    prev = None
    for r in range(world):
        d_in = torch.from_numpy(data[cuts[r]:cuts[r + 1]].copy()).cuda()
        e = sharded.ShardedCLEncoder(alg)
        tp = torch.empty(wp, dtype=torch.int32, device="cuda")
        rc = lib.density_b200_cl_shard_phase1(e._h, d_in.data_ptr(), d_in.numel(), int(r == world - 1),
                                              prev.data_ptr() if prev is not None else None, tp.data_ptr(), _stream(torch))
        assert rc == 0, lib.density_b200_last_error()
        if r == 0:
            prev = torch.zeros(1, dtype=torch.int32, device="cuda")
        if d_in.numel() >= 4:
            prev = d_in[d_in.numel() // 4 * 4 - 4:d_in.numel() // 4 * 4].clone().view(torch.int32)
        ins.append(d_in); encs.append(e); tps.append(tp)
    gp = torch.stack(tps)
    for r in range(world):
        carry = sharded.fold_cl_tables(alg, sharded.CL_TABLE_P, gp, r) if r > 0 else None
        tc = torch.empty(wc, dtype=torch.int32, device="cuda")
        rc = lib.density_b200_cl_shard_phase2(encs[r]._h, carry.data_ptr() if carry is not None else None, tc.data_ptr(), _stream(torch))
        assert rc == 0, lib.density_b200_last_error()
        tcs.append(tc)
    gc = torch.stack(tcs)
    for r in range(world):
        carry = sharded.fold_cl_tables(alg, sharded.CL_TABLE_C, gc, r) if r > 0 else None
        d_out = torch.zeros(getattr(lib, f"{alg}_safe_encode_buffer_size")(ins[r].numel()) + 64, dtype=torch.uint8, device="cuda")
        d_sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        rc = lib.density_b200_cl_shard_phase3(encs[r]._h, carry.data_ptr() if carry is not None else None, d_out.data_ptr(), d_out.numel(),
                                              d_sz.data_ptr(), words[r].data_ptr(), _stream(torch))
        assert rc == 0, lib.density_b200_last_error()
        outs.append(d_out); sizes.append(d_sz)
    torch.cuda.synchronize()
    verdict = sharded.seam_verdict(words)
    pieces = [outs[r][:int(sizes[r].item())].cpu().numpy() for r in range(world)]
    for e in encs:
        e.close()
    return pieces, verdict, words.cpu().numpy()


def single_call(torch, lib, alg, data):
    import density_b200
    d_in = torch.from_numpy(data.copy()).cuda()
    d_out = torch.zeros(getattr(lib, f"{alg}_safe_encode_buffer_size")(data.size) + 64, dtype=torch.uint8, device="cuda")
    d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    density_b200.encode_device(alg, d_in, d_out, d_sz)
    torch.cuda.synchronize()
    return d_out[:int(d_sz.item())].cpu().numpy()


def even_cuts(n, world, align=256):
    per = n // world // align * align
    return [r * per for r in range(world)] + [n]


def check_equal(torch, lib, alg, data, cuts, want=None):
    pieces, (flags, total, offsets), _ = encode_shards(torch, lib, alg, data, cuts)
    if want is None:
        want = oracle.encode(alg, data)
    assert flags == 0, (alg, cuts)
    cat = np.concatenate(pieces)
    assert total == want.size and cat.size == want.size and (cat == want).all(), (alg, cuts)
    return want


def text(n, first_page=0):
    from density_b200 import synth
    return synth.synth_text(n, first_page=first_page).numpy()


@pytest.mark.parametrize("alg", CL)
@pytest.mark.parametrize("world", range(1, 10))
def test_shards_equal_single_call_text(torch_cuda, lib, alg, world):
    data = text(3 * MIB + 1001)
    want = single_call(torch_cuda, lib, alg, data)
    assert (want == oracle.encode(alg, data)).all()
    check_equal(torch_cuda, lib, alg, data, even_cuts(data.size, world), want)


@pytest.mark.parametrize("alg", CL)
@pytest.mark.parametrize("world", [1, 2, 3, 5, 9])
def test_shards_equal_single_call_dickens_and_zeros(torch_cuda, lib, dickens200k, alg, world):
    check_equal(torch_cuda, lib, alg, dickens200k, even_cuts(dickens200k.size, world))
    z = np.zeros(MIB + 12, np.uint8)
    check_equal(torch_cuda, lib, alg, z, even_cuts(z.size, world))


@pytest.mark.parametrize("alg", CL)
def test_shards_cut_on_planted_positions(torch_cuda, lib, alg):
    """cl_corpus plants fresh contexts, context-0 quads, first chunk-map touches, (a, b) buckets and Lion contexts holding 4-6 values
    on both sides of every 16 KiB boundary: cut there (the context edge of every class, and cuts right before the first planted
    quad) and at odd multiples of 256 bytes."""
    data, manifest = planted.corpus("cl1")
    want = oracle.encode(alg, data)
    T = planted.TILE_BYTES
    for cuts in ([0, 5 * T, 6 * T, 7 * T, 8 * T, 9 * T, data.size],          # one seam in each of the five classes
                 [0, T, 3 * T + 256, 14 * T, 30 * T - 512, data.size],
                 [0, 2 * T, 2 * T, 24 * T, data.size]):                       # an empty shard in the middle
        check_equal(torch_cuda, lib, alg, data, cuts, want)


@pytest.mark.parametrize("alg", CL)
def test_empty_shards_and_tiny_last_shard(torch_cuda, lib, alg):
    data = text(MIB + 7, first_page=3)
    want = oracle.encode(alg, data)
    check_equal(torch_cuda, lib, alg, data, [0, 256 * 1000, 256 * 1000, MIB, MIB, data.size], want)
    check_equal(torch_cuda, lib, alg, data, [0, 256 * 2000, MIB, data.size], want)             # a 7-byte last shard
    # the stream start (and its cold-dictionary copy blocks) belongs to the first shard: with that shard empty it is refused
    assert encode_shards(torch_cuda, lib, alg, data, [0, 0, MIB, data.size])[1][0] != 0


@pytest.mark.parametrize("alg", CL)
def test_world1_equals_single_call_on_noise(torch_cuda, lib, alg):
    """The first shard runs the copy-map iteration like the single-device encoder: one shard equals one call, copy mode included."""
    for data in (splitmix_bytes(MIB + 3, 11), np.concatenate([text(512 * 1024), splitmix_bytes(256 * 1024, 4), text(512 * 1024 + 5, 7)])):
        check_equal(torch_cuda, lib, alg, data, [0, data.size])


@pytest.mark.parametrize("alg", CL)
def test_refusals(torch_cuda, lib, alg):
    torch = torch_cuda
    bb = 128 if alg == "cheetah" else 64
    t = text(2 * MIB, first_page=5)
    noise = splitmix_bytes(MIB, 12)
    # noise in a later shard: it would need copy mode
    d = np.concatenate([t[:MIB], noise])
    assert encode_shards(torch, lib, alg, d, [0, MIB, d.size])[1][0] != 0
    # one incompressible block on each side of a cut: the pair joins across the seam (one of them alone is fine)
    d = t.copy()
    d[MIB - bb:MIB] = noise[:bb]
    check_equal(torch, lib, alg, d, [0, MIB, d.size])
    d[MIB:MIB + bb] = noise[bb:2 * bb]
    assert encode_shards(torch, lib, alg, d, [0, MIB, d.size])[1][0] != 0
    # the first shard ends with a copy penalty pending: its last two blocks are incompressible, no block of it is copied for them,
    # and the single call copies the next shard's first block. Shard 0 refuses itself (seam word 2), whatever shard 1 holds.
    d = t.copy()
    d[MIB - 2 * bb:MIB] = noise[:2 * bb]
    _, (flags, _, _), words = encode_shards(torch, lib, alg, d, [0, MIB, d.size])
    assert flags != 0 and words[0][2] == 1 and words[0][1] == 1 and words[1][0] == 0 and words[1][2] == 0
    check_equal(torch, lib, alg, d, [0, d.size])
    check_equal(torch, lib, alg, d, [0, MIB + 4096, d.size])          # the copied block falls inside shard 0: copy mode in the first shard
    # the first shard ends inside a copy run
    d = np.concatenate([t[:MIB], noise[:64 * 1024], t[MIB:]])
    cut = MIB + 64 * 1024
    assert encode_shards(torch, lib, alg, d, [0, cut, d.size])[1][0] != 0
    check_equal(torch, lib, alg, d, [0, d.size])


@pytest.mark.parametrize("alg", CL)
def test_refused_when_first_shard_does_not_settle(torch_cuda, lib, alg):
    """With every stage of the copy-map iteration cut to one round (test hook) mixed data does not settle: the single-device path 1
    reports it with size 0, and the sharded encode refuses it (there is no in-order fallback on this path)."""
    import density_b200
    torch = torch_cuda
    data = payload("mixed", 2 * MIB + 5, 9)
    d_in = torch.from_numpy(data.copy()).cuda()
    d_out = torch.zeros(getattr(lib, f"{alg}_safe_encode_buffer_size")(data.size) + 64, dtype=torch.uint8, device="cuda")
    d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    lib.density_b200_test_set_stage_rounds(1)
    try:
        density_b200.encode_device(alg, d_in, d_out, d_sz, path=1)
        torch.cuda.synchronize()
        assert int(d_sz.item()) == 0, "the iteration settled: this input does not exercise the refusal"
        assert encode_shards(torch, lib, alg, data, [0, data.size])[1][0] != 0
        assert encode_shards(torch, lib, alg, data, [0, MIB, data.size])[1][0] != 0
    finally:
        lib.density_b200_test_set_stage_rounds(7)


def test_argument_checks(torch_cuda, lib):
    torch = torch_cuda
    from density_b200 import sharded
    assert not lib.density_b200_cl_shard_create(0) and not lib.density_b200_cl_shard_create(3)
    assert lib.density_b200_cl_table_words(0, 0) == 0 and lib.density_b200_cl_table_words(1, 2) == 0
    assert lib.density_b200_cl_table_words(1, 0) == 2 * 65536 and lib.density_b200_cl_table_words(2, 0) == 12 * 65536
    assert lib.density_b200_cl_table_words(1, 1) == lib.density_b200_cl_table_words(2, 1) == 3 * 65536
    t = torch.zeros(12 * 65536, dtype=torch.int32, device="cuda")
    assert lib.density_b200_cl_table_init(0, 0, t.data_ptr(), None) == 4
    assert lib.density_b200_cl_table_fold(1, 5, t.data_ptr(), t.data_ptr(), None) == 4
    e = sharded.ShardedCLEncoder("cheetah")
    d_in = torch.zeros(4096 + 8, dtype=torch.uint8, device="cuda")
    tc = torch.zeros(3 * 65536, dtype=torch.int32, device="cuda")
    assert lib.density_b200_cl_shard_phase2(e._h, None, tc.data_ptr(), None) == 4        # phase 1 not done
    assert lib.density_b200_cl_shard_phase1(e._h, d_in.data_ptr(), 1000, 0, None, t.data_ptr(), None) == 4   # not a multiple of 256
    assert lib.density_b200_cl_shard_phase1(e._h, d_in.data_ptr() + 2, 1024, 1, None, t.data_ptr(), None) == 4   # misaligned input
    assert lib.density_b200_cl_shard_phase1(e._h, d_in.data_ptr(), 1024, 1, None, None, None) == 4
    e.close()
    h = sharded.ShardedEncoder(torch.device("cuda"))
    d_out = torch.zeros(8192, dtype=torch.uint8, device="cuda")
    d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    d_fl = torch.zeros(1, dtype=torch.int32, device="cuda")
    for alg in (0, 3, -1):
        rc = lib.density_b200_encode_sharded_cl(h._h, alg, d_in.data_ptr(), 4096, d_out.data_ptr(), d_out.numel(), d_sz.data_ptr(),
                                                d_fl.data_ptr(), None, -1, None, 0, None)
        assert rc == 4
    rc = lib.density_b200_encode_sharded_cl(h._h, 1, d_in.data_ptr() + 1, 4096, d_out.data_ptr(), d_out.numel(), d_sz.data_ptr(),
                                            d_fl.data_ptr(), None, -1, None, 0, None)
    assert rc == 4
    h.close()


@pytest.mark.parametrize("alg", CL)
def test_encode_device_launch_counts_unchanged(torch_cuda, lib, alg):
    """The single-device run-parallel encoder (path 1: no in-order kernel behind it) keeps its launch sequence: 2 stages of the copy-map
    iteration (57 + 50 launches) up to 2 MiB, 4 stages (57 + 3 x 50) above, then sizes, scan (2), emit and the verdict."""
    import density_b200
    torch = torch_cuda
    for n, want in ((MIB + 5, 112), (3 * MIB + 5, 212)):
        data = text(n)
        d_in = torch.from_numpy(data).cuda()
        d_out = torch.zeros(getattr(lib, f"{alg}_safe_encode_buffer_size")(n) + 64, dtype=torch.uint8, device="cuda")
        d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
        density_b200.encode_device(alg, d_in, d_out, d_sz, path=1)
        torch.cuda.synchronize()
        before = lib.density_b200_kernel_launches()
        density_b200.encode_device(alg, d_in, d_out, d_sz, path=1)
        torch.cuda.synchronize()
        assert lib.density_b200_kernel_launches() - before == want
        assert (d_out[:int(d_sz.item())].cpu().numpy() == oracle.encode(alg, data)).all()


@pytest.mark.parametrize("alg", CL)
def test_encode_sharded_cl_cpp_entry_world1(torch_cuda, lib, alg):
    """density_b200_encode_sharded_cl with one rank (no NCCL): the piece and the gathered stream equal the single call, copy mode
    included, and the phase-level Python encoder agrees."""
    torch = torch_cuda
    from density_b200 import sharded
    h = sharded.ShardedEncoder(torch.device("cuda"))
    for data in (text(5 * MIB + 1021), np.concatenate([text(MIB), splitmix_bytes(100 * 1024, 2), text(77, 3)])):
        want = oracle.encode(alg, data)
        d_in = torch.from_numpy(data.copy()).cuda()
        d_out = torch.zeros(getattr(lib, f"{alg}_safe_encode_buffer_size")(data.size) + 64, dtype=torch.uint8, device="cuda")
        d_gather = torch.zeros(d_out.numel(), dtype=torch.uint8, device="cuda")
        d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
        d_fl = torch.ones(1, dtype=torch.int32, device="cuda")
        h.encode(d_in, d_out, d_sz, d_fl, gather_root=0, d_gather=d_gather, alg=alg)
        torch.cuda.synchronize()
        assert int(d_fl.item()) == 0 and int(d_sz.item()) == want.size == int(h.d_total.item())
        assert (d_out[:want.size].cpu().numpy() == want).all() and (d_gather[:want.size].cpu().numpy() == want).all()
        e = sharded.ShardedCLEncoder(alg)
        d_out.zero_()
        flags, total, _ = e.encode(d_in, d_out, d_sz, timing=True)
        assert flags == 0 and total == want.size and (d_out[:want.size].cpu().numpy() == want).all()
        assert len(e.phase_ms()) == 5
        e.close()
        ms = h.profile()                                   # the stages of this Cheetah / Lion call, not of an earlier Chameleon one
        assert len(ms) == 5 and all(v >= 0 for v in ms) and ms[0] > 0
    h.close()


def _nccl_worker(rank, world, port, alg, n_per_rank, q):
    import os, sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    import density_b200
    from density_b200 import sharded, synth
    enc = sharded.ShardedEncoder(dev)
    d_in = synth.synth_text(n_per_rank, device=dev, first_page=rank * (n_per_rank // synth.PAGE))
    cap = getattr(density_b200.load(), f"{alg}_safe_encode_buffer_size")(n_per_rank)
    d_out = torch.zeros(cap, dtype=torch.uint8, device=dev)
    d_gather = torch.zeros(world * cap, dtype=torch.uint8, device=dev) if rank == 0 else None
    d_sz = torch.zeros(1, dtype=torch.int64, device=dev)
    d_fl = torch.ones(1, dtype=torch.int32, device=dev)
    enc.encode(d_in, d_out, d_sz, d_fl, gather_root=0, d_gather=d_gather, alg=alg)
    torch.cuda.synchronize()
    total = int(enc.d_total.item())
    piece = d_out[:int(d_sz.item())].cpu().numpy()
    pe = sharded.ShardedCLEncoder(alg)                      # the phase-level path with torch.distributed exchanges
    d_out.zero_()
    fl2, _, _ = pe.encode(d_in, d_out, d_sz)
    piece2 = d_out[:int(d_sz.item())].cpu().numpy()
    q.put((rank, int(d_fl.item()), piece, total, d_gather[:total].cpu().numpy() if rank == 0 else None, fl2, piece2))
    dist.barrier()
    enc.close(); pe.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("alg", CL)
def test_encode_sharded_cl_two_ranks_nccl(torch_cuda, alg):
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from density_b200 import synth
    world, n_per = 2, 8 * MIB
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, world, 29733 + CL.index(alg), alg, n_per, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        r, *rest = q.get(timeout=600)
        got[r] = rest
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    want = oracle.encode(alg, synth.synth_text(world * n_per).numpy())
    assert all(got[r][0] == 0 and got[r][4] == 0 for r in range(world))
    for k in (1, 5):
        cat = np.concatenate([got[r][k] for r in range(world)])
        assert cat.size == want.size and (cat == want).all()
    assert got[0][2] == want.size and (got[0][3] == want).all()
