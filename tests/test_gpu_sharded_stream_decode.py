"""Sharded decode of a stream without known cuts (needs an H100: pytest -m gpu): the device range maps equal the numpy model, every rank
finds where its piece starts, the located pieces decode back to the original, and the verdict refuses every stream it cannot decode
piecewise without writing past any cap."""
import ctypes

import numpy as np
import pytest

import oracle
import planted
from conftest import payload
from locate_model import CH, HALO, aligned_block_start, layout, model_maps, range_map, stream_blocks

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


def text(n):
    from density_b200 import synth
    return synth.synth_text(n).numpy()


def device_encode(torch, lib, data):
    """One chameleon_encode call on the device."""
    d_in = torch.from_numpy(data).cuda()
    out = torch.zeros(lib.chameleon_safe_encode_buffer_size(data.size), dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.density_b200_encode_device(0, d_in.data_ptr(), data.size, out.data_ptr(), out.numel(), sz.data_ptr(), _stream(torch)) == 0
    torch.cuda.synchronize()
    return out[:int(sz.item())].cpu().numpy()


def device_map(torch, lib, handle, buf, n_range, n_halo):
    d_in = torch.from_numpy(np.ascontiguousarray(buf[:n_range + n_halo])).cuda()
    m = torch.full((266,), -1, dtype=torch.int64, device="cuda")
    rc = lib.density_b200_decode_locate(handle._h, d_in.data_ptr(), n_range, n_halo, m.data_ptr(), _stream(torch))
    assert rc == 0, lib.density_b200_last_error()
    torch.cuda.synchronize()
    return m.cpu().numpy().view(np.uint64)


def decode_located(torch, lib, stream, lay, caps=None):
    """ShardedChameleonDecoder.decode_stream with the ranks simulated in sequence on one GPU: every rank's range map, the stacked maps
    (as the all_gather), locate_piece, then the shard phases on the located pieces. Returns the decoded pieces, the verdict, whether
    the canaries behind every cap held, and the located pieces."""
    from density_b200 import sharded
    world = len(lay)
    caps = caps or [2 * (n + h) for _, n, h in lay]
    decs, ins = [], []
    maps = []
    for o, n, h in lay:
        d = sharded.ShardedChameleonDecoder()
        d_in = torch.from_numpy(np.ascontiguousarray(stream[o:o + n + h])).cuda()
        m = torch.empty(266, dtype=torch.int64, device="cuda")
        rc = lib.density_b200_decode_locate(d._h, d_in.data_ptr(), n, h, m.data_ptr(), _stream(torch))
        assert rc == 0, lib.density_b200_last_error()
        decs.append(d); ins.append(d_in); maps.append(m)
    gathered = torch.stack(maps).cpu().numpy().view(np.uint64)
    located = [sharded.locate_piece(gathered, r) for r in range(world)]
    tables, outs = [], []
    for r in range(world):
        start, end, _, final = located[r]
        piece = ins[r][start:end]
        t = torch.empty(65536, dtype=torch.int32, device="cuda")
        d_out = torch.full((caps[r] + 64,), CANARY, dtype=torch.uint8, device="cuda")
        rc = lib.density_b200_decode_shard_phase1(decs[r]._h, piece.data_ptr(), piece.numel(), caps[r], final, t.data_ptr(), _stream(torch))
        assert rc == 0, lib.density_b200_last_error()
        tables.append(t); outs.append(d_out)
    gt = torch.stack(tables)
    words = torch.zeros((world, 8), dtype=torch.int32, device="cuda")
    sizes = []
    for r in range(world):
        carry = sharded.fold_tables(gt, r) if r > 0 else None
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
    return got, verdict, canaries, located


def check_round_trip(torch, lib, stream, data, lay):
    got, (flags, total, offsets), canaries, located = decode_located(torch, lib, stream, lay)
    assert flags == 0 and total == data.size and canaries
    for r, piece in enumerate(got):
        assert offsets[r] == 256 * located[r][2] or piece.size == 0
    out = np.concatenate(got) if got else np.zeros(0, np.uint8)
    assert out.size == data.size and (out == data).all()


def padded_for_short_last(data, stream_fn):
    """data with zero blocks appended until its stream's length mod 16 KiB lies in [1, 263]: the last range is shorter than a block and
    the stream ends inside the halo of the rank before. Each zero block adds 136 bytes, so the window is never stepped over."""
    base = data[:data.size // 256 * 256]
    for k in range(0, 200):
        d = np.concatenate([base, np.zeros(256 * k, np.uint8)])
        s = stream_fn(d)
        if 1 <= s.size % CH < HALO and s.size > 2 * CH:
            return d, s
    raise AssertionError("no padding found")


def layouts(stream):
    from density_b200 import sharded
    total = stream.size
    k = total // CH
    out = {f"ranges{w}": sharded.stream_ranges(total, w) for w in (2, 3, 5, 8)}
    if k >= 3:
        a = k // 3 * CH
        out["zero_middle"] = layout(total, [a, 0, 0, a, 0, total - 2 * a])
    starts, _ = stream_blocks(stream)
    b = aligned_block_start(starts)
    if b is not None:
        out["on_block_start"] = layout(total, [b, total - b])
    return out


def _check_all_layouts(torch, lib, stream, data):
    for name, lay in layouts(stream).items():
        check_round_trip(torch, lib, stream, data, lay)


# ---- 1. the device maps are the model's ------------------------------------------------------------------------------------------
def test_device_maps_equal_model(torch_cuda, lib):
    from density_b200 import sharded
    torch = torch_cuda
    s = oracle.encode("chameleon", text(3 * MIB + 5))
    h = sharded.ShardedChameleonDecoder()
    k = s.size // CH
    cases = [
        (s, 40 * CH, HALO),                              # full range, full halo
        (s[40 * CH:], s.size - 40 * CH, 0),              # the last range: a partial last chunk
        (s[:(k - 1) * CH + 100], (k - 1) * CH, 100),     # short halo: the stream ends inside it
        (s[:100], 100, 0),                               # a tiny stream
        (s[:100], 0, 100),                               # an empty range
        (s[CH:], CH * 70, HALO),                         # 70 chunks: two groups, the second short
    ]
    for buf, n, hl in cases:
        got = device_map(torch, lib, h, buf, n, hl)
        want = range_map(buf, n, hl)
        assert (got == want).all(), (n, hl)
    h.close()


# ---- 2. round trips ----------------------------------------------------------------------------------------------------------------
def test_round_trip_single_call_stream(torch_cuda, lib):
    data = text(5 * MIB + 403)
    s = device_encode(torch_cuda, lib, data)
    assert (s == oracle.encode("chameleon", data)).all()
    _check_all_layouts(torch_cuda, lib, s, data)


def test_round_trip_short_last_range(torch_cuda, lib):
    data, s = padded_for_short_last(text(2 * MIB + 17), lambda d: device_encode(torch_cuda, lib, d))
    k = s.size // CH
    for lay in (layout(s.size, [k * CH, s.size - k * CH]), layout(s.size, [(k - 1) * CH, CH, s.size - k * CH]),
                layout(s.size, [k * CH, 0, 0, s.size - k * CH])):
        check_round_trip(torch_cuda, lib, s, data, lay)


@pytest.mark.parametrize("n", [0, 1, 5, 200])
def test_round_trip_tiny_stream_world4(torch_cuda, lib, n):
    from density_b200 import sharded
    data = text(max(n, 1))[:n]
    s = oracle.encode("chameleon", data)
    assert s.size < HALO
    check_round_trip(torch_cuda, lib, s, data, sharded.stream_ranges(s.size, 4))


def test_round_trip_dickens(torch_cuda, lib, dickens200k):
    s = oracle.encode("chameleon", dickens200k)
    _check_all_layouts(torch_cuda, lib, s, dickens200k)


def test_round_trip_zeros_on_block_start(torch_cuda, lib):
    data = np.zeros(3 * MIB, np.uint8)
    s = oracle.encode("chameleon", data)
    assert "on_block_start" in layouts(s)
    _check_all_layouts(torch_cuda, lib, s, data)


@pytest.mark.parametrize("name", planted.QUIET)
def test_round_trip_planted_quiet(torch_cuda, lib, name):
    from density_b200 import sharded
    data, _ = planted.corpus(name)
    s = oracle.encode("chameleon", data)
    if data.size > 64 * MIB:
        check_round_trip(torch_cuda, lib, s, data, sharded.stream_ranges(s.size, 4))
    else:
        _check_all_layouts(torch_cuda, lib, s, data)


def test_python_decode_stream_world1(torch_cuda, lib):
    from density_b200 import sharded
    torch = torch_cuda
    data = text(MIB + 3)
    enc = torch.from_numpy(oracle.encode("chameleon", data)).cuda()
    out = torch.full((2 * enc.numel() + 64,), CANARY, dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    d = sharded.ShardedChameleonDecoder()
    flags, total, offsets, my_off = d.decode_stream(enc, enc.numel(), out[:2 * enc.numel()], sz)
    torch.cuda.synchronize()
    assert flags == 0 and total == data.size and my_off == 0 and offsets.tolist() == [0, data.size]
    assert (out[:data.size].cpu().numpy() == data).all() and bool((out[2 * enc.numel():] == CANARY).all())
    d.close()


# ---- 3. planted seams at the cuts --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [1, 2])
def test_planted_seams_at_cuts(torch_cuda, lib, seed):
    """Each range starts at the 16 KiB multiple just before the compressed offset of a planted seam block: the `copies_across_seam` quad
    is written by the previous piece's tail and read as a MAP after the cut; fp-0 quads, quad 0 and bucket 0 cross the cuts."""
    n = 5 * MIB + 403
    seams = (MIB + 64 * 1024, 3 * MIB)
    data, manifest = planted.chameleon_corpus(n, seed, seams=seams)
    assert "copies_across_seam" in planted.classes(manifest)
    s = oracle.encode("chameleon", data)
    starts, _ = stream_blocks(s)
    cuts = [int(starts[x // 256]) // CH * CH for x in seams]
    assert 0 < cuts[0] < cuts[1]
    check_round_trip(torch_cuda, lib, s, data, layout(s.size, [cuts[0], cuts[1] - cuts[0], s.size - cuts[1]]))
    check_round_trip(torch_cuda, lib, s, data, layout(s.size, [cuts[0], cuts[1] - cuts[0], 0, s.size - cuts[1]]))


# ---- 4. refusals and the invariant -------------------------------------------------------------------------------------------------
def check_invariant(torch, lib, stream, lay, caps=None):
    """Either the verdict is non-zero and every canary holds, or it is 0 and the output equals decode_device's byte for byte."""
    got, (flags, total, _), canaries, _ = decode_located(torch, lib, stream, lay, caps)
    assert canaries
    if flags:
        return flags
    cap = sum(g.size for g in got) + 64
    d_in = torch.from_numpy(np.ascontiguousarray(stream)).cuda()
    out = torch.zeros(max(cap, 4), dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.density_b200_decode_device(0, d_in.data_ptr(), stream.size, out.data_ptr(), out.numel(), sz.data_ptr(), _stream(torch)) == 0
    torch.cuda.synchronize()
    want = out[:int(sz.item())].cpu().numpy()
    cat = np.concatenate(got)
    assert total == want.size == cat.size and (cat == want).all()
    return flags


def test_invariant_truncated(torch_cuda, lib):
    from density_b200 import sharded
    s = oracle.encode("chameleon", text(2 * MIB + 77))
    for cut in (1, 2, 3, 100, 300):
        t = s[:-cut]
        for w in (1, 3):
            check_invariant(torch_cuda, lib, t, sharded.stream_ranges(t.size, w))


def test_invariant_flipped_signature_bits(torch_cuda, lib):
    from density_b200 import sharded
    s = oracle.encode("chameleon", text(2 * MIB + 77))
    starts, _ = stream_blocks(s)
    lay = sharded.stream_ranges(s.size, 3)
    before_cut = [int(starts[np.searchsorted(starts, o) - 1]) for o, _, _ in lay[1:]]
    rng = np.random.default_rng(9)
    for b in before_cut + [int(x) for x in rng.choice(starts, 4)]:
        for bit in (0, 63):
            t = s.copy()
            t[b + bit // 8] ^= 1 << (bit % 8)
            check_invariant(torch_cuda, lib, t, lay)


def test_invariant_cap_one_short(torch_cuda, lib):
    from density_b200 import sharded
    data = text(2 * MIB + 77)
    s = oracle.encode("chameleon", data)
    lay = sharded.stream_ranges(s.size, 3)
    got, (flags, _, _), _, _ = decode_located(torch_cuda, lib, s, lay)
    assert flags == 0
    for r in range(3):
        caps = [2 * (n + h) for _, n, h in lay]
        caps[r] = got[r].size - 1
        assert check_invariant(torch_cuda, lib, s, lay, caps) != 0


def test_refuses_copy_mode_noise_and_a_pair_across_a_cut(torch_cuda, lib):
    from density_b200 import sharded
    copy, _ = planted.chameleon_copy_corpus(3 * MIB + 5, 4)
    noise = payload("random", MIB, 3)
    for data in (copy, noise):
        s = oracle.encode("chameleon", data)
        for w in (1, 2, 3):
            assert check_invariant(torch_cuda, lib, s, sharded.stream_ranges(s.size, w)) != 0
    # two incompressible blocks, the first just before a 16 KiB multiple: the located cut falls between them
    data = text(2 * MIB)
    s = oracle.encode("chameleon", data)
    starts, _ = stream_blocks(s)
    i = int(np.nonzero((starts % CH >= CH - 200) & (starts > 4 * CH))[0][0])
    c = (int(starts[i]) // CH + 1) * CH
    data[256 * i:256 * i + 512] = np.random.default_rng(5).integers(0, 256, 512, dtype=np.uint8)
    s = oracle.encode("chameleon", data)
    assert int(stream_blocks(s)[0][i]) == int(starts[i])
    assert check_invariant(torch_cuda, lib, s, layout(s.size, [c, s.size - c])) != 0


# ---- 5-7. the C++ entry ------------------------------------------------------------------------------------------------------------
def test_decode_sharded_stream_world1_equals_decode_device(torch_cuda, lib):
    """The world-1 C++ entry equals decode_device; it alternates with encode_sharded and decode_sharded on one handle."""
    torch = torch_cuda
    from density_b200 import sharded
    n = 5 * MIB + 1021
    data = text(n)
    enc_h = sharded.ShardedEncoder(torch.device("cuda"))
    dec_h = sharded.ShardedDecoder(torch.device("cuda"))
    d_in = torch.from_numpy(data.copy()).cuda()
    d_enc = torch.zeros(lib.chameleon_safe_encode_buffer_size(n), dtype=torch.uint8, device="cuda")
    d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    d_fl = torch.ones(1, dtype=torch.int32, device="cuda")
    d_ref = torch.zeros(n, dtype=torch.uint8, device="cuda")
    d_ref_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    for _ in range(2):
        enc_h.encode(d_in, d_enc, d_sz, d_fl)
        torch.cuda.synchronize()
        m = int(d_sz.item())
        piece = d_enc[:m]
        cap = 2 * m
        d_dec = torch.full((cap + 64,), CANARY, dtype=torch.uint8, device="cuda")
        d_fl.fill_(1); dec_h.d_offset.fill_(-1)
        dec_h.decode_stream(piece, m, d_dec[:cap], d_sz, d_fl)
        assert lib.density_b200_decode_device(0, piece.data_ptr(), m, d_ref.data_ptr(), n, d_ref_sz.data_ptr(), _stream(torch)) == 0
        torch.cuda.synchronize()
        assert int(d_fl.item()) == 0 and int(d_sz.item()) == n == int(d_ref_sz.item()) == int(dec_h.d_total.item())
        assert int(dec_h.d_offset.item()) == 0
        assert torch.equal(d_dec[:n], d_ref) and torch.equal(d_ref, d_in) and bool((d_dec[cap:] == CANARY).all())
        d_fl.fill_(1)
        dec_h.decode(piece, d_dec[:n], d_sz, d_fl)
        torch.cuda.synchronize()
        assert int(d_fl.item()) == 0 and torch.equal(d_dec[:n], d_in)
    dec_h.close(); enc_h.close()


def test_decode_sharded_launch_count_unchanged(torch_cuda, lib):
    """density_b200_decode_sharded launches 18 kernels, as before the stream entry: 9 boundary kernels, writer pass, table export (2),
    fold, carry scan, decode pass, tail, seam words, verdict."""
    torch = torch_cuda
    from density_b200 import sharded
    data = text(MIB)
    enc = torch.from_numpy(oracle.encode("chameleon", data)).cuda()
    h = sharded.ShardedDecoder(torch.device("cuda"))
    out = torch.zeros(data.size, dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    fl = torch.ones(1, dtype=torch.int32, device="cuda")
    before = lib.density_b200_kernel_launches()
    h.decode(enc, out, sz, fl)
    assert lib.density_b200_kernel_launches() - before == 18
    before = lib.density_b200_kernel_launches()
    h.decode_stream(enc, enc.numel(), out, sz, fl)     # + the three locate kernels
    assert lib.density_b200_kernel_launches() - before == 21
    torch.cuda.synchronize()
    assert int(fl.item()) == 0 and (out.cpu().numpy() == data).all()
    h.close()


def test_output_offsets_beyond_4gib(torch_cuda, lib):
    """The 5.5 GiB Chameleon pair corpus of tests/big_streams.py (a stream of more than 2**32 + 2**28 bytes, every block distinct) in
    two ranges, the second starting past 2**32 bytes of stream: rank 1 locates its piece and writes its output above 2**32, and the
    decoded bytes equal the input."""
    import big_streams as bs
    torch = torch_cuda
    n = bs.SIZE["chameleon"]
    if torch.cuda.mem_get_info()[0] < 24 * (1 << 30):
        pytest.skip("needs 24 GiB of free device memory")
    data = bs.corpus("chameleon", n)
    stream, _ = bs.oracle_stream("chameleon", data)
    m = stream.size
    assert m > bs.STREAM_MIN
    r0 = ((1 << 32) // CH + 1) * CH
    lay = layout(m, [r0, m - r0])
    got, (flags, total, offsets), canaries, located = decode_located(torch, lib, stream, lay)
    del stream
    assert flags == 0 and total == n and canaries
    assert int(offsets[1]) > (1 << 32) and int(offsets[1]) == 256 * located[1][2]
    for r in range(2):
        assert got[r].size == int(offsets[r + 1] - offsets[r])
        off = bs.first_difference(got[r], data[int(offsets[r]):int(offsets[r + 1])])
        assert off is None, f"rank {r}: first difference at output byte {int(offsets[r]) + off}"


# ---- 8. two ranks over NCCL --------------------------------------------------------------------------------------------------------
def _nccl_worker(rank, world, port, n, q):
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
    lib = density_b200.load()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    d_data = synth.synth_text(n, device=dev)
    d_enc = torch.zeros(density_b200.Chameleon.safe_encode_buffer_size(n), dtype=torch.uint8, device=dev)
    d_sz = torch.zeros(1, dtype=torch.int64, device=dev)
    assert lib.density_b200_encode_device(0, d_data.data_ptr(), n, d_enc.data_ptr(), d_enc.numel(), d_sz.data_ptr(), stream) == 0
    torch.cuda.synchronize()
    m = int(d_sz.item())
    o, nr, hl = sharded.stream_ranges(m, world)[rank]
    d_in = d_enc[o:o + nr + hl].clone()
    dec = sharded.ShardedDecoder(dev)
    cap = 2 * (nr + hl)
    d_out = torch.zeros(cap, dtype=torch.uint8, device=dev)
    d_fl = torch.ones(1, dtype=torch.int32, device=dev)
    dec.decode_stream(d_in, nr, d_out, d_sz, d_fl)
    torch.cuda.synchronize()
    off, k = int(dec.d_offset.item()), int(d_sz.item())
    same = bool(torch.equal(d_out[:k], d_data[off:off + k]))
    pd = sharded.ShardedChameleonDecoder()
    d_out2 = torch.zeros(cap, dtype=torch.uint8, device=dev)
    flags, total, _, off2 = pd.decode_stream(d_in, nr, d_out2, d_sz)
    torch.cuda.synchronize()
    same2 = off2 == off and bool(torch.equal(d_out2[:k], d_out[:k]))
    q.put((rank, int(d_fl.item()), int(dec.d_total.item()), same, flags, total, same2, k))
    dist.barrier()
    pd.close(); dec.close()
    dist.destroy_process_group()


def test_decode_sharded_stream_two_ranks_nccl(torch_cuda, lib):
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, n = 2, 96 * MIB + 5
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, world, 29741, n, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict((r, rest) for r, *rest in (q.get(timeout=600) for _ in range(world)))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert sum(got[r][6] for r in range(world)) == n
    for r in range(world):
        flag, total, same, pflags, ptotal, same2, _ = got[r]
        assert flag == 0 and total == n and same and pflags == 0 and ptotal == n and same2


# ---- 9. argument checks (one rank only: a rank that returned before a collective would leave the others waiting in it) -----------
def test_decode_sharded_stream_rejects_bad_arguments(torch_cuda, lib):
    torch = torch_cuda
    from density_b200 import sharded
    h = sharded.ShardedDecoder(torch.device("cuda"))
    s = oracle.encode("chameleon", text(64 * 1024))
    buf = torch.zeros(4 * s.size + 4096, dtype=torch.uint8, device="cuda")
    buf[:s.size] = torch.from_numpy(s).cuda()
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    fl = torch.zeros(1, dtype=torch.int32, device="cuda")
    off = torch.zeros(1, dtype=torch.int64, device="cuda")
    p, st, n = buf.data_ptr(), _stream(torch), s.size
    o = p + s.size + 1024 - (s.size + 1024) % 4
    f = lib.density_b200_decode_sharded_stream
    assert f(h._h, p + 1, n - 1, 0, o, 2 * n, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 4     # misaligned d_in
    assert f(h._h, p, n, 0, o + 2, 2 * n, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 4        # misaligned d_out
    assert f(h._h, None, n, 0, o, 2 * n, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 4
    assert f(h._h, p, n, 0, None, 2 * n, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 4
    assert f(h._h, p, n, 0, o, 2 * n, None, off.data_ptr(), fl.data_ptr(), None, st) == 4
    assert f(h._h, p, n, 0, o, 2 * n, sz.data_ptr(), off.data_ptr(), None, None, st) == 4
    assert f(None, p, n, 0, o, 2 * n, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 4
    assert f(h._h, p, n - 10, 10, o, 2 * n, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 4     # the last rank has a halo
    assert f(h._h, p, n, 0, o, 2 * n, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 0           # and the good call works
    torch.cuda.synchronize()
    assert int(fl.item()) == 0 and int(sz.item()) == 64 * 1024 and int(off.item()) == 0
    d = sharded.ShardedChameleonDecoder()
    m = torch.zeros(266, dtype=torch.int64, device="cuda")
    assert lib.density_b200_decode_locate(d._h, p + 1, 100, 0, m.data_ptr(), st) == 4
    assert lib.density_b200_decode_locate(d._h, p, 100, 0, m.data_ptr() + 4, st) == 4
    assert lib.density_b200_decode_locate(d._h, p, 100, 0, None, st) == 4
    assert lib.density_b200_decode_locate(None, p, 100, 0, m.data_ptr(), st) == 4
    with pytest.raises(Exception):
        d.decode_stream(buf[:s.size], s.size - 10, buf[s.size + 1024:], sz)   # a halo on the last rank
    d.close()
    h.close()
