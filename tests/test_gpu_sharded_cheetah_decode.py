"""Sharded Cheetah decode (needs an H100: pytest -m gpu): the pieces of one Cheetah stream, run through the phase API on one device with
the library's folds, decode back to their shards byte for byte whenever the seam verdict is 0, and the verdict refuses what a piece
cannot decode alone (DESIGN.md section 5)."""
import ctypes

import numpy as np
import pytest

import oracle
import planted
from conftest import splitmix_bytes
from test_gpu_sharded_cl_encode import encode_shards, even_cuts, text

pytestmark = pytest.mark.gpu
CANARY = 0xA5

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


def _ptr(t):
    return t.data_ptr() if t.numel() else None


def decode_pieces(torch, lib, enc, cuts, caps=None):
    """Every phase of every piece enc[cuts[r]:cuts[r + 1]] on one device, the exchanges replaced by stacking the transfers and folding them
    with the library's init / fold entry points, for the whole round budget. Returns (decoded pieces, (flags, total, offsets), seam
    words [world][8], status [world][4]). Checks that nothing is written past any piece's cap."""
    from density_b200 import sharded
    world = len(cuts) - 1
    st = _stream(torch)
    wc, wp = lib.density_b200_cheetah_cmap_words(), lib.density_b200_cl_table_words(1, sharded.CL_TABLE_P)
    hs, ins, outs = [], [], []
    tc = torch.zeros((world, wc), dtype=torch.int32, device="cuda")
    for r in range(world):
        d_in = torch.from_numpy(np.ascontiguousarray(enc[cuts[r]:cuts[r + 1]])).cuda()
        cap = caps[r] if caps is not None else 16 * d_in.numel() + 256
        d_out = torch.full((max(cap, 1) + 64,), CANARY, dtype=torch.uint8, device="cuda")
        h = lib.density_b200_cheetah_decode_shard_create()
        assert h
        rc = lib.density_b200_cheetah_decode_shard_phase1(h, _ptr(d_in), d_in.numel(), d_out.data_ptr(), cap, int(r == 0), int(r == world - 1),
                                                          tc[r].data_ptr(), st)
        assert rc == 0, lib.density_b200_last_error()
        hs.append(h); ins.append(d_in); outs.append((d_out, cap))
    for r in range(world):
        carry = sharded.fold_cheetah_cmap(tc, r) if r > 0 else None
        assert lib.density_b200_cheetah_decode_shard_phase2(hs[r], carry.data_ptr() if carry is not None else None, st) == 0
    tp = torch.zeros((world, wp), dtype=torch.int32, device="cuda")
    words = torch.zeros((world, 4), dtype=torch.int32, device="cuda")
    for _ in range(lib.density_b200_cheetah_decode_round_budget()):
        for r in range(world):
            assert lib.density_b200_cheetah_decode_shard_round_walk(hs[r], tp[r].data_ptr(), words[r].data_ptr(), st) == 0
        for r in range(world):
            carry = sharded.fold_cl_tables("cheetah", sharded.CL_TABLE_P, tp, r) if r > 0 else None
            rc = lib.density_b200_cheetah_decode_shard_round_fold(hs[r], carry.data_ptr() if carry is not None else None, words.data_ptr(),
                                                                  world, r, st)
            assert rc == 0, lib.density_b200_last_error()
    seam = torch.zeros((world, 8), dtype=torch.int32, device="cuda")
    sizes = torch.zeros(world, dtype=torch.int64, device="cuda")
    for r in range(world):
        assert lib.density_b200_cheetah_decode_shard_phase3(hs[r], sizes[r:r + 1].data_ptr(), seam[r].data_ptr(), st) == 0
    torch.cuda.synchronize()
    status = []
    for r in range(world):
        s4 = (ctypes.c_uint32 * 4)()
        assert lib.density_b200_cheetah_decode_shard_status(hs[r], s4) == 0
        status.append(list(s4))
        lib.density_b200_cheetah_decode_shard_destroy(hs[r])
    for r, (d_out, cap) in enumerate(outs):
        assert bool((d_out[cap:] == CANARY).all()), f"piece {r} written past cap"
    verdict = sharded.seam_verdict(seam)
    pieces = [outs[r][0][:int(sizes[r].item())].cpu().numpy() for r in range(world)]
    return pieces, verdict, seam.cpu().numpy(), status


def piece_cuts(pieces):
    return [0] + list(np.cumsum([p.size for p in pieces]))


def check_round_trip(torch, lib, data, cuts):
    """encode the shards data[cuts[r]:cuts[r + 1]], decode the pieces, and the oracle's stream sliced at the same offsets"""
    pieces, (flags, _, _), _ = encode_shards(torch, lib, "cheetah", data, cuts)
    assert flags == 0, cuts
    enc = np.concatenate(pieces)
    want_enc = oracle.encode("cheetah", data)
    assert enc.size == want_enc.size and (enc == want_enc).all()
    pc = piece_cuts(pieces)
    got, (flags, total, offsets), _, status = decode_pieces(torch, lib, enc, pc)
    assert flags == 0, (cuts, status)
    assert total == data.size and list(offsets.numpy()) == list(cuts)
    for r in range(len(got)):
        assert got[r].size == cuts[r + 1] - cuts[r] and (got[r] == data[cuts[r]:cuts[r + 1]]).all(), (cuts, r)
    assert all(s[1] == 1 for s in status)
    return pc, status


@pytest.mark.parametrize("world", range(1, 10))
def test_pieces_decode_to_their_shards_text(torch_cuda, lib, world):
    data = text(3 * MIB + 1001)
    check_round_trip(torch_cuda, lib, data, even_cuts(data.size, world))


@pytest.mark.parametrize("world", [1, 2, 3, 5, 9])
def test_pieces_decode_to_their_shards_dickens_and_zeros(torch_cuda, lib, dickens200k, world):
    check_round_trip(torch_cuda, lib, dickens200k, even_cuts(dickens200k.size, world))
    z = np.zeros(MIB + 12, np.uint8)          # every piece starts behind a chain of predicted quads: its entry context comes from the rounds
    check_round_trip(torch_cuda, lib, z, even_cuts(z.size, world))


def test_interchange_single_call_and_oracle_slices(torch_cuda, lib):
    """The slices of one cheetah_encode call and of the oracle's stream at the piece-size prefix sums decode like the encoder's pieces."""
    import density_b200
    torch = torch_cuda
    data = text(2 * MIB + 333, first_page=2)
    cuts = [0, 256 * 1000, 256 * 3001, 256 * 6000, data.size]
    pc, _ = check_round_trip(torch, lib, data, cuts)
    d_in = torch.from_numpy(data.copy()).cuda()
    d_out = torch.zeros(lib.cheetah_safe_encode_buffer_size(data.size) + 64, dtype=torch.uint8, device="cuda")
    d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    density_b200.encode_device("cheetah", d_in, d_out, d_sz)
    torch.cuda.synchronize()
    single = d_out[:int(d_sz.item())].cpu().numpy()
    for enc in (single, oracle.encode("cheetah", data)):
        got, (flags, total, _), _, _ = decode_pieces(torch, lib, enc, pc)
        assert flags == 0 and total == data.size and (np.concatenate(got) == data).all()


def test_cut_on_planted_positions(torch_cuda, lib):
    data, _ = planted.corpus("cl1")
    T = planted.TILE_BYTES
    for cuts in ([0, 5 * T, 6 * T, 7 * T, 8 * T, 9 * T, data.size],
                 [0, T, 3 * T + 256, 14 * T, 30 * T - 512, data.size],
                 [0, 2 * T, 2 * T, 24 * T, data.size]):
        check_round_trip(torch_cuda, lib, data, cuts)


def test_piece_ends_empty_pieces_and_tiny_last_piece(torch_cuda, lib):
    torch = torch_cuda
    data = text(MIB + 7, first_page=3)
    check_round_trip(torch, lib, data, [0, 256 * 1000, 256 * 1000, MIB, MIB, data.size])     # empty pieces in the middle
    check_round_trip(torch, lib, data, [0, 256 * 2000, MIB, data.size])                      # a 7-byte last piece
    # a non-final piece whose last blocks start in its last 136 bytes (every non-final piece has some: the boundary walk leaves them to
    # the tail), and whose chunk-map and prediction writes the next piece reads: a shard that repeats the end of the one before it
    a = text(512 * 1024, first_page=9)
    d = np.concatenate([a, a[-64 * 1024:], text(64 * 1024 + 5, first_page=1)])
    check_round_trip(torch, lib, d, [0, a.size, a.size + 64 * 1024, d.size])
    check_round_trip(torch, lib, d, [0, a.size - 256, a.size + 256, d.size])


def _enc_and_cuts(data, shard_cuts):
    enc = oracle.encode("cheetah", data)
    return enc, [oracle.encode("cheetah", data[:c]).size if c < data.size else enc.size for c in shard_cuts]


def test_refusals(torch_cuda, lib):
    torch = torch_cuda
    t = text(2 * MIB, first_page=5)
    noise = splitmix_bytes(MIB, 12)
    # copy mode in piece 1: the slice of a text | noise | text single-call stream, cut in the text in front of the noise
    d = np.concatenate([t[:MIB], noise[:256 * 1024], t[MIB:]])
    enc, pc = _enc_and_cuts(d, [0, MIB - 64 * 1024, d.size])
    _, (flags, _, _), words, _ = decode_pieces(torch, lib, enc, pc)
    assert flags != 0 and words[1][2] == 1 and words[0][2] == 0
    got, (flags, _, _), _, _ = decode_pieces(torch, lib, enc, [0, enc.size])
    assert flags == 0 and (got[0] == d).all()
    # an incompressible block on each side of a seam: piece 0 is fine alone, the seam is not
    d = t.copy()
    d[MIB - 128:MIB + 128] = noise[:256]
    enc, pc = _enc_and_cuts(d, [0, MIB, d.size])
    _, (flags, _, _), words, _ = decode_pieces(torch, lib, enc, pc)
    assert flags != 0 and words[0][1] == 1 and words[1][0] == 1 and words[0][2] == 0
    # piece 0 ends with a copy penalty pending: its last two blocks are incompressible
    d = t.copy()
    d[MIB - 256:MIB] = noise[:256]
    enc, pc = _enc_and_cuts(d, [0, MIB, d.size])
    _, (flags, _, _), words, _ = decode_pieces(torch, lib, enc, pc)
    assert flags != 0 and words[0][2] == 1
    got, (flags, _, _), _, _ = decode_pieces(torch, lib, enc, [0, enc.size])     # one piece: copy mode is the first piece's to use
    assert flags == 0 and (got[0] == d).all()
    # piece 0 ends inside a copy run
    d = np.concatenate([t[:MIB], noise[:64 * 1024], t[MIB:]])
    enc, pc = _enc_and_cuts(d, [0, MIB + 64 * 1024, d.size])
    _, (flags, _, _), words, _ = decode_pieces(torch, lib, enc, pc)
    assert flags != 0 and words[0][2] == 1


def test_refused_when_the_rounds_do_not_settle(torch_cuda, lib):
    torch = torch_cuda
    data = text(3 * MIB + 1001)
    enc, pc = _enc_and_cuts(data, even_cuts(data.size, 3))
    lib.density_b200_test_set_decode_rounds(1)
    try:
        assert lib.density_b200_cheetah_decode_round_budget() == 1
        _, (flags, _, _), words, status = decode_pieces(torch, lib, enc, pc)
        assert flags != 0 and all(w[2] == 1 for w in words) and all(s[1] == 0 and s[3] == 1 for s in status)
    finally:
        lib.density_b200_test_set_decode_rounds(40)
    assert lib.density_b200_cheetah_decode_round_budget() == 40


def _decode_device(torch, data_enc, cap):
    import density_b200
    d_in = torch.from_numpy(data_enc.copy()).cuda()
    d_out = torch.zeros(max(cap, 4), dtype=torch.uint8, device="cuda")
    d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    density_b200.decode_device("cheetah", d_in, d_in.numel(), d_out, d_sz)
    torch.cuda.synchronize()
    return d_out[:int(d_sz.item())].cpu().numpy()


def test_damaged_pieces_refuse_or_match_decode_device(torch_cuda, lib):
    """Truncated and bit-flipped pieces, and a capacity one byte short: the pieces either refuse or decode, together, like decode_device
    of the whole damaged stream."""
    torch = torch_cuda
    data = text(MIB + 77, first_page=4)
    cuts = [0, 256 * 2048, data.size]
    enc, pc = _enc_and_cuts(data, cuts)
    rng = np.random.default_rng(5)
    for trial in range(8):
        e = enc.copy()
        if trial < 4:
            k = int(rng.integers(pc[1] // 2, e.size))
            e[k] ^= np.uint8(1 << int(rng.integers(0, 8)))
            p = list(pc)
        else:
            cut = int(rng.integers(1, 300))
            e = np.concatenate([enc[:pc[1] - cut], enc[pc[1]:]]) if trial < 6 else enc[:-cut]
            p = [0, pc[1] - cut, e.size] if trial < 6 else [0, pc[1], e.size]
        got, (flags, _, _), _, _ = decode_pieces(torch, lib, e, p)
        if flags == 0:
            want = _decode_device(torch, e, 16 * e.size + 256)
            cat = np.concatenate(got)
            assert cat.size == want.size and (cat == want).all(), trial
    # a capacity one byte short for the first piece: refused, nothing written past it
    caps = [cuts[1] - 1, 16 * (enc.size - pc[1]) + 256]
    _, (flags, _, _), words, _ = decode_pieces(torch, lib, enc, pc, caps)
    assert flags != 0 and words[0][2] == 1
    # and for the last piece
    caps = [16 * pc[1], data.size - cuts[1] - 1]
    _, (flags, _, _), words, _ = decode_pieces(torch, lib, enc, pc, caps)
    assert flags != 0 and words[1][2] == 1


def test_argument_checks_and_phase_order(torch_cuda, lib):
    torch = torch_cuda
    st = _stream(torch)
    h = lib.density_b200_cheetah_decode_shard_create()
    d_in = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(65536, dtype=torch.uint8, device="cuda")
    t = torch.zeros(3 * 65536, dtype=torch.int32, device="cuda")
    w = torch.zeros(8, dtype=torch.int32, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.density_b200_cheetah_cmap_words() == 3 * 65536
    assert lib.density_b200_cheetah_decode_shard_phase2(h, None, st) == 4                      # phase 1 not done
    assert lib.density_b200_cheetah_decode_shard_round_walk(h, None, w.data_ptr(), st) == 4
    assert lib.density_b200_cheetah_decode_shard_phase3(h, sz.data_ptr(), w.data_ptr(), st) == 4
    assert lib.density_b200_cheetah_decode_shard_phase1(h, d_in.data_ptr() + 1, 1024, d_out.data_ptr(), 65536, 1, 1, None, st) == 4
    assert lib.density_b200_cheetah_decode_shard_phase1(h, d_in.data_ptr(), 1024, d_out.data_ptr() + 2, 65536, 1, 1, None, st) == 4
    assert lib.density_b200_cheetah_decode_shard_phase1(h, None, 1024, d_out.data_ptr(), 65536, 1, 1, None, st) == 4
    assert lib.density_b200_cheetah_decode_shard_phase1(h, d_in.data_ptr(), 1024, d_out.data_ptr(), 65536, 1, 1, t.data_ptr(), st) == 0
    assert lib.density_b200_cheetah_decode_shard_round_walk(h, None, w.data_ptr(), st) == 4     # phase 2 not done
    assert lib.density_b200_cheetah_decode_shard_phase2(h, None, st) == 0
    assert lib.density_b200_cheetah_decode_shard_round_fold(h, None, w.data_ptr(), 1, 0, st) == 4   # its walk not done
    assert lib.density_b200_cheetah_decode_shard_round_walk(h, None, None, st) == 4
    assert lib.density_b200_cheetah_decode_shard_round_walk(h, None, w.data_ptr(), st) == 0
    assert lib.density_b200_cheetah_decode_shard_phase3(h, sz.data_ptr(), w.data_ptr(), st) == 4   # the round's fold not done
    assert lib.density_b200_cheetah_decode_shard_round_fold(h, None, w.data_ptr(), 1, 1, st) == 4  # rank >= world
    assert lib.density_b200_cheetah_decode_shard_round_fold(h, None, None, 1, 0, st) == 4
    assert lib.density_b200_cheetah_decode_shard_round_fold(h, None, w.data_ptr(), 1, 0, st) == 0
    assert lib.density_b200_cheetah_decode_shard_phase3(h, None, w.data_ptr(), st) == 4
    assert lib.density_b200_cheetah_decode_shard_phase3(h, sz.data_ptr(), w.data_ptr(), st) == 0
    assert lib.density_b200_cheetah_decode_shard_phase3(h, sz.data_ptr(), w.data_ptr(), st) == 4   # one phase 3 per phase 1
    torch.cuda.synchronize()
    lib.density_b200_cheetah_decode_shard_destroy(h)
    assert lib.density_b200_cheetah_cmap_init(None, st) == 4 and lib.density_b200_cheetah_cmap_fold(t.data_ptr(), None, st) == 4
    from density_b200 import sharded
    dec = sharded.ShardedDecoder(torch.device("cuda"))
    fl = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert lib.density_b200_decode_sharded_cheetah(dec._h, d_in.data_ptr() + 1, 1024, d_out.data_ptr(), 65536, sz.data_ptr(), fl.data_ptr(),
                                                   None, st) == 4
    assert lib.density_b200_decode_sharded_cheetah(dec._h, d_in.data_ptr(), 1024, d_out.data_ptr(), 65536, None, fl.data_ptr(), None, st) == 4
    with pytest.raises(ValueError):
        dec.decode(d_in, d_out, sz, fl, alg="lion")
    dec.close()


def test_decode_device_unchanged(torch_cuda, lib):
    """decode_device keeps its Cheetah launch sequence (9 boundary kernels, 5 + 40 x 3 rounds + 1 of the run-parallel decoder, the tail,
    the in-order kernel behind it) and its output, whatever the round-budget hook says."""
    import density_b200
    torch = torch_cuda
    data = text(3 * MIB + 5)
    enc = oracle.encode("cheetah", data)
    d_in = torch.from_numpy(enc).cuda()
    d_out = torch.zeros(data.size + 64, dtype=torch.uint8, device="cuda")
    d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    for k in (40, 1):
        lib.density_b200_test_set_decode_rounds(k)
        try:
            before = lib.density_b200_kernel_launches()
            density_b200.decode_device("cheetah", d_in, enc.size, d_out, d_sz)
            torch.cuda.synchronize()
            assert lib.density_b200_kernel_launches() - before == 137
        finally:
            lib.density_b200_test_set_decode_rounds(40)
        assert int(d_sz.item()) == data.size and (d_out[:data.size].cpu().numpy() == data).all()
        r4 = (ctypes.c_uint32 * 4)()
        assert lib.density_b200_cheetah_decode_rounds(r4) == 0 and r4[1] == 1 and r4[3] == 40


def test_cpp_entry_world1_and_python(torch_cuda, lib):
    """density_b200_decode_sharded_cheetah with one rank (no NCCL) and ShardedDecoder.decode(alg="cheetah") equal decode_device."""
    torch = torch_cuda
    from density_b200 import sharded
    dec = sharded.ShardedDecoder(torch.device("cuda"))
    for data in (text(5 * MIB + 1021), np.concatenate([text(MIB), splitmix_bytes(100 * 1024, 2), text(77, 3)]), np.zeros(MIB + 3, np.uint8)):
        enc = oracle.encode("cheetah", data)
        want = _decode_device(torch, enc, data.size + 64)
        assert (want == data).all()
        d_in = torch.from_numpy(enc.copy()).cuda()
        d_out = torch.zeros(data.size + 64, dtype=torch.uint8, device="cuda")
        d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
        d_fl = torch.ones(1, dtype=torch.int32, device="cuda")
        dec.decode(d_in, d_out, d_sz, d_fl, alg="cheetah")
        torch.cuda.synchronize()
        assert int(d_fl.item()) == 0 and int(d_sz.item()) == data.size == int(dec.d_total.item())
        assert (d_out[:data.size].cpu().numpy() == want).all()
        d_out.zero_()
        rc = lib.density_b200_decode_sharded_cheetah(dec._h, d_in.data_ptr(), d_in.numel(), d_out.data_ptr(), d_out.numel(), d_sz.data_ptr(),
                                                     d_fl.data_ptr(), None, _stream(torch))
        assert rc == 0
        torch.cuda.synchronize()
        assert int(d_fl.item()) == 0 and (d_out[:data.size].cpu().numpy() == want).all()
    dec.close()


def _nccl_worker(rank, world, port, n_per_rank, q):
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
    cap = density_b200.load().cheetah_safe_encode_buffer_size(n_per_rank)
    d_piece = torch.zeros(cap, dtype=torch.uint8, device=dev)
    d_sz = torch.zeros(1, dtype=torch.int64, device=dev)
    d_fl = torch.ones(1, dtype=torch.int32, device=dev)
    enc.encode(d_in, d_piece, d_sz, d_fl, alg="cheetah")
    torch.cuda.synchronize()
    fl_enc = int(d_fl.item())
    piece = d_piece[:int(d_sz.item())].clone()
    dec = sharded.ShardedDecoder(dev)
    d_out = torch.zeros(n_per_rank + 64, dtype=torch.uint8, device=dev)
    d_fl.fill_(1)
    dec.decode(piece, d_out, d_sz, d_fl, alg="cheetah")
    torch.cuda.synchronize()
    ok = int(d_sz.item()) == n_per_rank and bool((d_out[:n_per_rank] == d_in).all().item())
    q.put((rank, fl_enc, int(d_fl.item()), ok, int(dec.d_total.item())))
    dist.barrier()
    enc.close(); dec.close()
    dist.destroy_process_group()


def test_decode_sharded_cheetah_two_ranks_nccl(torch_cuda):
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, n_per = 2, 8 * MIB
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, world, 29741, n_per, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        r, *rest = q.get(timeout=600)
        got[r] = rest
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert all(got[r] == [0, 0, True, world * n_per] for r in range(world)), got
