"""Sharded Chameleon decode (needs an H100: pytest -m gpu): every piece of a sharded stream decodes back into its shard with the
dictionary carried in from the pieces before it, and the seam verdict refuses every stream it cannot decode piecewise."""
import ctypes

import numpy as np
import pytest

import oracle
import planted
from conftest import payload

pytestmark = pytest.mark.gpu

CANARY = 0xA5


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


def encode_pieces(torch, lib, data, cuts):
    """The shard phases of the encoder (as test_sharded_stream_equals_single_call): piece r of each shard data[cuts[r]:cuts[r+1]]."""
    from density_b200 import sharded
    world = len(cuts) - 1
    encs, tables, ins = [], [], []
    for r in range(world):
        d_in = torch.from_numpy(data[cuts[r]:cuts[r + 1]].copy()).cuda()
        t = torch.zeros(65536, dtype=torch.int32, device="cuda")      # an empty shard touches nothing and encodes to nothing
        e = sharded.ShardedChameleonEncoder()
        if d_in.numel():
            assert lib.density_b200_shard_phase1(e._h, d_in.data_ptr(), d_in.numel(), int(r == world - 1), t.data_ptr(), _stream(torch)) == 0
        encs.append(e); tables.append(t); ins.append(d_in)
    gathered = torch.stack(tables)
    pieces, flags = [], []
    for r in range(world):
        if not ins[r].numel():
            pieces.append(np.zeros(0, np.uint8)); flags.append(0); encs[r].close()
            continue
        carry = sharded.fold_tables(gathered, r) if r > 0 else None
        d_out = torch.zeros(lib.chameleon_safe_encode_buffer_size(ins[r].numel()) + 64, dtype=torch.uint8, device="cuda")
        d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
        d_fl = torch.zeros(1, dtype=torch.int32, device="cuda")
        assert lib.density_b200_shard_phase2(encs[r]._h, carry.data_ptr() if carry is not None else None, d_out.data_ptr(), d_out.numel(),
                                             d_sz.data_ptr(), d_fl.data_ptr(), _stream(torch)) == 0
        torch.cuda.synchronize()
        pieces.append(d_out[:int(d_sz.item())].cpu().numpy())
        flags.append(int(d_fl.item()))
        encs[r].close()
    return pieces, flags


def decode_pieces(torch, lib, pieces, caps, carry0=None):
    """The shard phases of the decoder, one handle per piece; the tables are stacked and folded as an all_gather would. Returns the
    decoded pieces (their first `size` bytes), the verdict (flags, total, offsets) and whether the canaries behind every cap held."""
    from density_b200 import sharded
    world = len(pieces)
    decs, tables, ins, outs = [], [], [], []
    for r in range(world):
        d_in = torch.from_numpy(np.ascontiguousarray(pieces[r])).cuda()
        d_out = torch.full((caps[r] + 64,), CANARY, dtype=torch.uint8, device="cuda")
        t = torch.empty(65536, dtype=torch.int32, device="cuda")
        d = sharded.ShardedChameleonDecoder()
        rc = lib.density_b200_decode_shard_phase1(d._h, d_in.data_ptr(), d_in.numel(), caps[r], int(r == world - 1), t.data_ptr(), _stream(torch))
        assert rc == 0, lib.density_b200_last_error()
        decs.append(d); tables.append(t); ins.append(d_in); outs.append(d_out)
    gathered = torch.stack(tables)
    words = torch.zeros((world, 8), dtype=torch.int32, device="cuda")
    sizes = []
    for r in range(world):
        carry = sharded.fold_tables(gathered, r) if r > 0 else carry0
        d_sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        rc = lib.density_b200_decode_shard_phase2(decs[r]._h, carry.data_ptr() if carry is not None else None, outs[r].data_ptr(),
                                                  d_sz.data_ptr(), words[r].data_ptr(), _stream(torch))
        assert rc == 0, lib.density_b200_last_error()
        sizes.append(d_sz)
    torch.cuda.synchronize()
    verdict = sharded.seam_verdict(words)
    canaries = all(bool((outs[r][caps[r]:] == CANARY).all()) for r in range(world))
    got = [outs[r][:int(sizes[r].item())].cpu().numpy() for r in range(world)]
    for d in decs:
        d.close()
    return got, verdict, canaries


def text(n):
    from density_b200 import synth
    return synth.synth_text(n).numpy()


def check_round_trip(torch, lib, data, cuts):
    pieces, eflags = encode_pieces(torch, lib, data, cuts)
    assert eflags == [0] * len(pieces)
    shards = [data[cuts[r]:cuts[r + 1]] for r in range(len(pieces))]
    got, (flags, total, offsets), canaries = decode_pieces(torch, lib, pieces, [max(4, s.size) for s in shards])
    assert flags == 0 and total == data.size and canaries
    assert list(offsets.tolist()) == cuts
    for r, s in enumerate(shards):
        assert got[r].size == s.size and (got[r] == s).all(), f"piece {r}"
    return pieces


MIB = 1 << 20
K = 256
ROUND_TRIP_CUTS = {
    "two": [0, 2 * MIB, 3 * MIB + 1001],
    "three": [0, MIB + 7 * K, 2 * MIB + 100 * K, 3 * MIB + 1001],
    "five": [0, 300 * K, 1 * MIB, 1 * MIB + 4096 * K // 4, 2 * MIB + 3 * K, 3 * MIB + 1001],
    "piece_256": [0, MIB, MIB + K, 3 * MIB + 1001],         # the middle piece is < 264 B: dec_tail decodes all of it
    "empty_middle": [0, MIB + 5 * K, MIB + 5 * K, 3 * MIB + 1001],
    "last_mod4_1": [0, 2 * MIB, 3 * MIB + 1],
    "last_mod4_2": [0, 2 * MIB, 3 * MIB + 2],
    "last_mod4_3": [0, 2 * MIB, 3 * MIB + 3],
    "empty_last": [0, MIB, 3 * MIB, 3 * MIB],
}


@pytest.mark.parametrize("name", sorted(ROUND_TRIP_CUTS))
def test_round_trip_through_the_phases(torch_cuda, lib, name):
    cuts = ROUND_TRIP_CUTS[name]
    check_round_trip(torch_cuda, lib, text(cuts[-1]), cuts)


def test_interchange_with_single_call_stream(torch_cuda, lib):
    """Slices of oracle.encode(whole) at the prefix sums of the piece sizes decode the same as the pieces themselves."""
    cuts = ROUND_TRIP_CUTS["five"]
    data = text(cuts[-1])
    pieces, _ = encode_pieces(torch_cuda, lib, data, cuts)
    whole = oracle.encode("chameleon", data)
    offs = np.cumsum([0] + [p.size for p in pieces])
    assert offs[-1] == whole.size
    slices = [whole[offs[r]:offs[r + 1]] for r in range(len(pieces))]
    got, (flags, total, _), canaries = decode_pieces(torch_cuda, lib, slices, [cuts[r + 1] - cuts[r] for r in range(len(pieces))])
    assert flags == 0 and total == data.size and canaries
    assert (np.concatenate(got) == data).all()


@pytest.mark.parametrize("seed", [1, 2])
def test_planted_seams(torch_cuda, lib, seed):
    """Cuts on the planted seams: the `copies_across_seam` quad is first written in the last block of a piece (the tail export) and
    read as a MAP in the next one; carried states of fp-0 quads, quad 0 and bucket 0 cross the seams, and across the empty piece a
    bucket's last writer is two pieces back."""
    n = 5 * MIB + 403
    seams = (MIB + 64 * K, 3 * MIB)
    data, manifest = planted.chameleon_corpus(n, seed, seams=seams)
    assert "copies_across_seam" in planted.classes(manifest)
    check_round_trip(torch_cuda, lib, data, [0, seams[0], seams[1], seams[1], n])


def test_tail_export_reaches_the_next_piece(torch_cuda, lib):
    """A quad written only by the tail of piece 0 and read as a MAP at the start of piece 1: decoding piece 1 needs the tail export."""
    data = text(2 * MIB)
    q = planted.quad_of(0x5A5A, 0x1234)
    cut = MIB
    data[cut - 16:cut + 16].view(np.uint32)[:] = q
    check_round_trip(torch_cuda, lib, data, [0, cut, 2 * MIB])


@pytest.mark.parametrize("kind", ["zeros", "text_quad0"])
def test_stream_start_identity(torch_cuda, lib, kind):
    """The encoder's stream-start table (bucket 0 touched, fingerprint 0) as the explicit carry-in of piece 0 decodes the same as NULL."""
    from density_b200 import sharded
    if kind == "zeros":
        data = np.zeros(MIB, np.uint8)
    else:
        data = text(MIB)
        data[400:404] = 0                  # the first MAP of bucket 0 reads the untouched bucket: quad 0
    enc = oracle.encode("chameleon", data)
    init = sharded.initial_table("cuda")
    for carry0 in (None, init):
        got, (flags, total, _), canaries = decode_pieces(torch_cuda, lib, [enc], [data.size], carry0=carry0)
        assert flags == 0 and total == data.size and canaries and (got[0] == data).all()


def _blocks(piece):
    """Block start offsets of a piece of whole encoded blocks (quiet: every block has a signature)."""
    offs, i = [], 0
    while i < piece.size:
        offs.append(i)
        sig = int.from_bytes(piece[i:i + 8].tobytes(), "little")
        i += 264 - 2 * bin(sig).count("1")
    assert i == piece.size
    return offs


def _refused(torch, lib, pieces, caps):
    got, (flags, _, _), canaries = decode_pieces(torch, lib, pieces, caps)
    assert flags != 0 and canaries


def test_refuses_copy_mode_pieces(torch_cuda, lib):
    data, _ = planted.chameleon_copy_corpus(3 * MIB + 5, 4)
    enc = oracle.encode("chameleon", data)
    _refused(torch_cuda, lib, [enc], [data.size])
    _refused(torch_cuda, lib, [enc, enc[:0]], [data.size, 4])


def test_refuses_incompressible_blocks_across_a_seam(torch_cuda, lib):
    n, cut = 2 * MIB, MIB
    data = text(n)
    rnd = np.random.default_rng(5).integers(0, 256, 512, dtype=np.uint8)
    data[cut - 256:cut + 256] = rnd
    pieces, _ = encode_pieces(torch_cuda, lib, data, [0, cut, n])
    # the encoder's pieces are not the single-call stream either: there the block after the pair is copied raw
    cat, whole = np.concatenate(pieces), oracle.encode("chameleon", data)
    assert cat.size != whole.size or not (cat == whole).all()
    _refused(torch_cuda, lib, pieces, [cut, n - cut])


def test_refuses_two_incompressible_blocks_at_the_end_of_a_piece(torch_cuda, lib):
    n, cut = 2 * MIB, MIB
    data = text(n)
    data[cut - 512:cut] = np.random.default_rng(6).integers(0, 256, 512, dtype=np.uint8)
    pieces, _ = encode_pieces(torch_cuda, lib, data, [0, cut, n])
    _refused(torch_cuda, lib, pieces, [cut, n - cut])


@pytest.mark.parametrize("damage", ["truncated", "flipped_signature", "cap_one_short"])
def test_refuses_damaged_pieces(torch_cuda, lib, damage):
    n, cut = 2 * MIB, MIB + 3 * K
    data = text(n)
    pieces, _ = encode_pieces(torch_cuda, lib, data, [0, cut, n])
    caps = [cut, n - cut]
    p0 = pieces[0].copy()
    if damage == "truncated":
        p0 = p0[:-2]
    elif damage == "flipped_signature":
        p0[_blocks(p0)[-1]] ^= 1
    else:
        caps[0] -= 1
    _refused(torch_cuda, lib, [p0, pieces[1]], caps)


def test_decode_sharded_world1_equals_decode_device(torch_cuda, lib):
    """density_b200_decode_sharded with one rank (no NCCL) equals decode_device; a noise stream is refused; encode_sharded and
    decode_sharded alternate on one handle."""
    torch = torch_cuda
    from density_b200 import sharded
    n = 5 * MIB + 1021
    data = text(n)
    h = sharded.ShardedEncoder(torch.device("cuda"))
    d_in = torch.from_numpy(data.copy()).cuda()
    cap_enc = lib.chameleon_safe_encode_buffer_size(n)
    d_enc = torch.zeros(cap_enc, dtype=torch.uint8, device="cuda")
    d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    d_fl = torch.ones(1, dtype=torch.int32, device="cuda")
    d_dec = torch.full((n + 64,), CANARY, dtype=torch.uint8, device="cuda")
    d_ref = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_tot = torch.zeros(1, dtype=torch.int64, device="cuda")
    d_ref_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    for _ in range(2):
        h.encode(d_in, d_enc, d_sz, d_fl)
        torch.cuda.synchronize()
        assert int(d_fl.item()) == 0
        m = int(d_sz.item())
        piece = d_enc[:m]
        d_fl.fill_(1)
        rc = lib.density_b200_decode_sharded(h._h, piece.data_ptr(), m, d_dec.data_ptr(), n, d_sz.data_ptr(), d_fl.data_ptr(),
                                             d_tot.data_ptr(), _stream(torch))
        assert rc == 0, lib.density_b200_last_error()
        rc = lib.density_b200_decode_device(0, piece.data_ptr(), m, d_ref.data_ptr(), n, d_ref_sz.data_ptr(), _stream(torch))
        assert rc == 0
        torch.cuda.synchronize()
        assert int(d_fl.item()) == 0 and int(d_sz.item()) == n == int(d_ref_sz.item()) and int(d_tot.item()) == n
        assert torch.equal(d_dec[:n], d_in) and torch.equal(d_ref, d_in) and bool((d_dec[n:] == CANARY).all())
    noise = payload("random", MIB, 3)
    enc = torch.from_numpy(oracle.encode("chameleon", noise)).cuda()
    d_fl.fill_(0)
    dec = sharded.ShardedDecoder(torch.device("cuda"))
    dec.decode(enc, d_dec[:MIB], d_sz, d_fl)
    torch.cuda.synchronize()
    assert int(d_fl.item()) != 0
    dec.close()
    h.close()


def test_decode_sharded_rejects_bad_arguments(torch_cuda, lib):
    torch = torch_cuda
    from density_b200 import sharded
    h = sharded.ShardedEncoder(torch.device("cuda"))
    buf = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    fl = torch.zeros(1, dtype=torch.int32, device="cuda")
    p, s = buf.data_ptr(), _stream(torch)
    assert lib.density_b200_decode_sharded(h._h, p + 1, 100, p + 2048, 1024, sz.data_ptr(), fl.data_ptr(), None, s) == 4
    assert lib.density_b200_decode_sharded(h._h, p, 100, p + 2050, 1024, sz.data_ptr(), fl.data_ptr(), None, s) == 4
    assert lib.density_b200_decode_sharded(h._h, p, 100, p + 2048, 1024, None, fl.data_ptr(), None, s) == 4
    d = sharded.ShardedChameleonDecoder()
    w = torch.zeros(8, dtype=torch.int32, device="cuda")
    assert lib.density_b200_decode_shard_phase2(d._h, None, p, sz.data_ptr(), w.data_ptr(), s) == 4      # phase 2 before phase 1
    t = torch.zeros(65536, dtype=torch.int32, device="cuda")
    assert lib.density_b200_decode_shard_phase1(d._h, p + 1, 100, 1024, 1, t.data_ptr(), s) == 4
    d.close()
    h.close()


def test_one_shot_decode_launch_count(torch_cuda, lib):
    """decode_device keeps its kernels: 9 boundary kernels, writer pass, carry fold, decode pass, tail and the queued in-order kernel."""
    torch = torch_cuda
    data = text(MIB)
    enc = torch.from_numpy(oracle.encode("chameleon", data)).cuda()
    out = torch.zeros(data.size, dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    before = lib.density_b200_kernel_launches()
    assert lib.density_b200_decode_device(0, enc.data_ptr(), enc.numel(), out.data_ptr(), data.size, sz.data_ptr(), _stream(torch)) == 0
    assert lib.density_b200_kernel_launches() - before == 14
    torch.cuda.synchronize()
    assert (out.cpu().numpy() == data).all()


def test_python_shard_decoder_world1(torch_cuda, lib):
    torch = torch_cuda
    from density_b200 import sharded
    data = text(MIB + 3)
    enc = torch.from_numpy(oracle.encode("chameleon", data)).cuda()
    out = torch.zeros(data.size, dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    d = sharded.ShardedChameleonDecoder()
    flags, total, offsets = d.decode(enc, out, sz)
    assert flags == 0 and total == data.size and offsets.tolist() == [0, data.size]
    assert (out.cpu().numpy() == data).all()
    d.close()


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
    h = sharded.ShardedEncoder(dev)
    dec = sharded.ShardedDecoder(dev)
    d_in = synth.synth_text(n_per_rank, device=dev, first_page=rank * (n_per_rank // synth.PAGE))
    d_enc = torch.zeros(density_b200.Chameleon.safe_encode_buffer_size(n_per_rank), dtype=torch.uint8, device=dev)
    d_sz = torch.zeros(1, dtype=torch.int64, device=dev)
    d_fl = torch.ones(1, dtype=torch.int32, device=dev)
    h.encode(d_in, d_enc, d_sz, d_fl)
    torch.cuda.synchronize()
    eflag = int(d_fl.item())
    piece = d_enc[:int(d_sz.item())]
    d_dec = torch.zeros(n_per_rank, dtype=torch.uint8, device=dev)
    d_fl.fill_(1)
    dec.decode(piece, d_dec, d_sz, d_fl)
    torch.cuda.synchronize()
    q.put((rank, eflag, int(d_fl.item()), int(dec.d_total.item()), bool(torch.equal(d_dec, d_in))))
    dist.barrier()
    dec.close(); h.close()
    dist.destroy_process_group()


def test_decode_sharded_two_ranks_nccl(torch_cuda, lib):
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, n_per = 2, 48 * MIB
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, world, 29733, n_per, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict((r, rest) for r, *rest in (q.get(timeout=600) for _ in range(world)))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for r in range(world):
        eflag, dflag, total, same = got[r]
        assert eflag == 0 and dflag == 0 and total == world * n_per and same
