"""Sharded decode of streams without known cuts that have copy-mode blocks (needs an H100: pytest -m gpu). The device's protected range
maps equal the numpy model word for word; the ranks, simulated in sequence on one GPU through the phase API (prot_locate, the
composition, prot_enter, the rest of the protected phases), decode the oracle's stream byte for byte with a zero verdict, on streams
the quiet stream entries refuse; damaged streams and short caps refuse, never with wrong output, and nothing is written past cap."""
import ctypes
import functools

import numpy as np
import pytest

import oracle
import prot_locate_model as L
from conftest import payload

pytestmark = pytest.mark.gpu

CANARY = 0xA5
KIB, MIB = 1 << 10, 1 << 20
ALGS = ["chameleon", "cheetah"]


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


def _p(t):
    return t.data_ptr() if t is not None and t.numel() else None


@functools.lru_cache(maxsize=None)
def corpus(name, alg):
    """(data, oracle stream)"""
    from density_b200 import synth
    if name == "noise":
        data = payload("random", 2 * MIB + 77, 1)
    elif name == "synth_mixed":
        data = synth.synth_mixed(3 * MIB).numpy()
    else:
        data = synth.synth_text(3 * MIB).numpy()
        rnd = payload("random", 64 * KIB, 7)
        for i, lo in enumerate((100_000, 1_300_001, 2_700_003)):
            data[lo:lo + 5000] = rnd[i * 8192:i * 8192 + 5000]
    return data, oracle.encode(alg, data)


def shard_create(lib, alg):
    return lib.density_b200_decode_shard_create() if alg == "chameleon" else lib.density_b200_cheetah_decode_shard_create()


def shard_destroy(lib, alg, h):
    (lib.density_b200_decode_shard_destroy if alg == "chameleon" else lib.density_b200_cheetah_decode_shard_destroy)(h)


def launches(lib, fn, *args):
    """fn(*args) must return 0; the kernels it enqueued"""
    before = lib.density_b200_kernel_launches()
    rc = fn(*args)
    assert rc == 0, lib.density_b200_last_error()
    return lib.density_b200_kernel_launches() - before


def device_map(torch, lib, alg, h, buf):
    d_in, n, hl = buf
    m = torch.full((L.map_words(alg),), -1, dtype=torch.int32, device="cuda")
    fn = lib.density_b200_decode_prot_locate if alg == "chameleon" else lib.density_b200_cheetah_decode_prot_locate
    k = launches(lib, fn, h, _p(d_in), n, hl, m.data_ptr(), _stream(torch))
    assert k == (3 if n else 1), k                    # candidate rows, group rows, the head walks; an empty range: the identity
    return m


def decode_located(torch, lib, alg, stream, lay, caps=None):
    """The ranks of a sharded stream decode, in sequence on one GPU: every rank's protected range map, the stacked maps (the all-gather),
    density_b200_prot_locate_piece, then the protected phases of the located pieces from their entry candidates. Returns (flags, total,
    outs, located); checks that nothing is written past any cap."""
    from density_b200 import sharded as S
    world, st = len(lay), _stream(torch)
    caps = caps or [(2 if alg == "chameleon" else 16) * (n + h) for _, n, h in lay]
    hs = [shard_create(lib, alg) for _ in range(world)]
    ins = [torch.from_numpy(np.ascontiguousarray(stream[o:o + n + h])).cuda() for o, n, h in lay]
    maps = torch.stack([device_map(torch, lib, alg, hs[r], (ins[r], lay[r][1], lay[r][2])) for r in range(world)])
    located = [S.prot_locate_piece(maps.cpu().numpy().view(np.uint32), r, alg) for r in range(world)]
    outs = [torch.full((caps[r] + 64,), CANARY, dtype=torch.uint8, device="cuda") for r in range(world)]
    sizes = torch.full((world,), -1, dtype=torch.int64, device="cuda")
    seam = torch.zeros((world, 8), dtype=torch.int32, device="cuda")
    if located[0][5]:
        assert all(p == (0, 0, 0, 0, 0, 1) for p in located)
        for h in hs:
            shard_destroy(lib, alg, h)
        return 1, 0, [], located
    pieces = [ins[r][p[0]:p[1]] for r, p in enumerate(located)]
    if alg == "chameleon":
        tables = torch.zeros((world, 65536), dtype=torch.int32, device="cuda")
        for r, (start, end, final, first, cand, _) in enumerate(located):
            k = launches(lib, lib.density_b200_decode_shard_prot_enter, hs[r], _p(pieces[r]), end - start, caps[r], final, cand,
                         tables[r].data_ptr(), st)
            # the seed, the 9 boundary kernels (the candidate rows are the piece's own), the writer pass, the table export
            assert k == (1 + 9 + 1 + 2 if end > start else 1), (r, k)
        for r in range(world):
            carry = S.fold_tables(tables, r) if r > 0 else None
            rc = lib.density_b200_decode_shard_prot_phase2(hs[r], _p(carry), outs[r].data_ptr(), sizes[r:r + 1].data_ptr(), seam[r].data_ptr(), st)
            assert rc == 0, lib.density_b200_last_error()
    else:
        wc, wp = lib.density_b200_cheetah_cmap_words(), lib.density_b200_cl_table_words(1, S.CL_TABLE_P)
        tc = torch.zeros((world, wc), dtype=torch.int32, device="cuda")
        firsts = [bool(p[3]) for p in located]
        for r, (start, end, final, first, cand, _) in enumerate(located):
            k = launches(lib, lib.density_b200_cheetah_decode_shard_prot_enter, hs[r], _p(pieces[r]), end - start, outs[r].data_ptr(), caps[r],
                         first, final, cand, tc[r].data_ptr(), st)
            # the seed, the 9 boundary kernels, the end of the piece, unpack, chunk-map walk, the export; an empty piece: the identity map
            assert k == (1 + 9 + 1 + 2 + 1 if end > start else 2), (r, k)
        for r in range(world):
            carry = S.fold_cheetah_cmap(tc, r) if r > 0 and not firsts[r] else None
            assert lib.density_b200_cheetah_decode_shard_phase2(hs[r], _p(carry), st) == 0, lib.density_b200_last_error()
        tp = torch.zeros((world, wp), dtype=torch.int32, device="cuda")
        words = torch.zeros((world, 4), dtype=torch.int32, device="cuda")
        for _ in range(lib.density_b200_cheetah_decode_round_budget()):
            for r in range(world):
                assert lib.density_b200_cheetah_decode_shard_round_walk(hs[r], tp[r].data_ptr(), words[r].data_ptr(), st) == 0
            for r in range(world):
                carry = S.fold_cl_tables(1, S.CL_TABLE_P, tp, r) if r > 0 and not firsts[r] else None
                rc = lib.density_b200_cheetah_decode_shard_round_fold(hs[r], _p(carry), words.data_ptr(), world, r, st)
                assert rc == 0, lib.density_b200_last_error()
        for r in range(world):
            rc = lib.density_b200_cheetah_decode_shard_phase3(hs[r], sizes[r:r + 1].data_ptr(), seam[r].data_ptr(), st)
            assert rc == 0, lib.density_b200_last_error()
    torch.cuda.synchronize()
    for r in range(world):
        assert bool((outs[r][caps[r]:] == CANARY).all()), f"rank {r} wrote past cap"
        shard_destroy(lib, alg, hs[r])
    flags, total, _ = S.seam_verdict(seam)
    got = [outs[r][:max(int(sizes[r].item()), 0)].cpu().numpy() for r in range(world)]
    return flags, total, got, located


def check_round_trip(torch, lib, alg, stream, data, lay):
    flags, total, got, located = decode_located(torch, lib, alg, stream, lay)
    assert flags == 0 and total == data.size, (lay, located)
    out = np.concatenate(got)
    assert out.size == data.size and (out == data).all(), lay


def copy_mode_after(alg, stream, data, at):
    """the stream has a copy-mode block at or after stream offset `at`: the quiet stream entries refuse it once a range boundary lies in
    front of it (Chameleon refuses copy mode anywhere, Cheetah outside the range that holds the stream start)"""
    import protection as P
    tr = P.trace(alg, stream, data.size)
    return bool((tr.copied & (tr.off >= at)).any())


# ---- 1. the device maps are the model's ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", ALGS)
def test_device_maps_equal_model(torch_cuda, lib, alg):
    torch = torch_cuda
    h = shard_create(lib, alg)
    _, mixed = corpus("synth_mixed", alg)
    _, noise = corpus("noise", alg)
    U = L.RANGE_UNIT
    cases = [
        (mixed, 0, 4 * U, L.HALO),                         # the stream start (Cheetah's cold start), full halo
        (noise, 7 * U, 3 * U, L.HALO),                     # copy runs
        (mixed, 20 * U, 66 * U, L.HALO),                   # whole groups of 64 chunks and a short one: group jumps
        (mixed, mixed.size - 2 * U - 100, 2 * U, 100),     # a short halo: the stream ends inside it
        (mixed, mixed.size - 5000, 5000, 0),               # the last range
        (mixed, 3 * U, 0, L.HALO),                         # an empty range
    ]
    for s, o, n, hl in cases:
        assert o + n + hl <= s.size
        buf = np.ascontiguousarray(s[o:o + n + hl])
        got = device_map(torch, lib, alg, h, (torch.from_numpy(buf).cuda(), n, hl)).cpu().numpy().view(np.uint32)
        want = L.range_map(buf, n, hl, alg)
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, (o, n, hl, bad[:5], got[bad[:5]], want[bad[:5]])
    shard_destroy(lib, alg, h)


@pytest.mark.parametrize("alg", ALGS)
def test_heads_dropped_at_the_cap_refuse_never_lie(torch_cuda, lib, alg):
    """A range of zero bytes: every block reads as incompressible, and the walks from the 3200 candidates keep more than 256 distinct
    (offset, state, phase) heads alive after a chunk step (about 365 after the first; tests/prot_decode_model.py counts them), so the
    device drops heads (Chameleon in the first range, Cheetah, with 4 KiB chunks, in both). Every row of a dropped head is 0xFFFE, every
    other row is the exact walk's, and a composition that meets a dropped row refuses on every rank; one that does not locates what the
    model locates."""
    from density_b200 import sharded as S
    torch = torch_cuda
    U = L.RANGE_UNIT
    zeros = np.zeros(2 * U + 5000, np.uint8)
    lay = L.layout(zeros.size, [2 * U, None])
    h = [shard_create(lib, alg) for _ in lay]
    maps = np.stack([device_map(torch, lib, alg, h[r], (torch.from_numpy(zeros[o:o + n + hl].copy()).cuda(), n, hl))
                     .cpu().numpy().view(np.uint32) for r, (o, n, hl) in enumerate(lay)])
    want = L.stream_maps(zeros, lay, alg)
    assert not (want == L.NOEND).any()
    dropped = maps == L.NOEND
    assert dropped[0].any() and ((maps == want) | dropped).all()
    for r in range(len(lay)):
        got = S.prot_locate_piece(maps, r, alg)
        if got[5]:                                   # the path met a dropped row: refused, and only then
            assert got == (0, 0, 0, 0, 0, 1) and L.locate_piece(maps, r, alg)[5]
        else:
            assert got == L.locate_piece(want, r, alg)
    for x in h:
        shard_destroy(lib, alg, x)


# ---- 2. round trips at 1-8 pieces -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("name", ["noise", "synth_mixed", "text_bursts"])
def test_round_trip_phase_api(torch_cuda, lib, alg, name):
    from density_b200 import sharded as S
    data, s = corpus(name, alg)
    for world in (1, 2, 3, 5, 8):
        check_round_trip(torch_cuda, lib, alg, s, data, S.stream_ranges(s.size, world))
    U = L.RANGE_UNIT
    check_round_trip(torch_cuda, lib, alg, s, data, L.layout(s.size, [0, 5 * U, 0, 0, 17 * U, 0, None]))     # empty ranges
    assert copy_mode_after(alg, s, data, S.stream_ranges(s.size, 3)[1][0])


@pytest.mark.parametrize("alg", ALGS)
def test_round_trip_short_stream_and_short_last_halo(torch_cuda, lib, alg):
    from density_b200 import sharded as S
    for n in (0, 1, 200, 9000):
        data = payload("random", max(n, 1), 3)[:n]
        s = oracle.encode(alg, data)
        check_round_trip(torch_cuda, lib, alg, s, data, S.stream_ranges(s.size, 4))
    # noise whose stream ends 1 .. 263 bytes past a range boundary: the range before holds the stream end in its halo
    U = L.RANGE_UNIT
    noise = payload("random", 300 * KIB, 4)
    for n in range(200 * KIB, 300 * KIB, 256):
        s = oracle.encode(alg, noise[:n])
        if 1 <= s.size % U < L.HALO:
            break
    else:
        raise AssertionError("no short last range found")
    k = s.size // U
    for lay in (L.layout(s.size, [k * U, None]), L.layout(s.size, [(k - 1) * U, U, None]), L.layout(s.size, [k * U, 0, None])):
        check_round_trip(torch_cuda, lib, alg, s, noise[:n], lay)


# ---- 3. refusals --------------------------------------------------------------------------------------------------------------------
def _decode_device(torch, alg, enc, cap):
    import density_b200
    d_in = torch.from_numpy(np.ascontiguousarray(enc)).cuda()
    out = torch.zeros(max(cap, 4), dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    try:
        density_b200.decode_device(alg, d_in, enc.size, out, sz)
    except Exception:
        return None
    torch.cuda.synchronize()
    return out[:int(sz.item())].cpu().numpy()


@pytest.mark.parametrize("alg", ALGS)
def test_damaged_streams_and_short_caps_refuse_never_wrong(torch_cuda, lib, alg):
    from density_b200 import sharded as S
    torch = torch_cuda
    data, s = corpus("text_bursts", alg)
    lay = S.stream_ranges(s.size, 4)
    damaged = [s[:s.size - 1000], s[:s.size // 2 + 3]]
    rng = np.random.default_rng(5)
    for _ in range(3):
        bad = s.copy()
        bad[int(rng.integers(0, s.size))] ^= 1 << int(rng.integers(0, 8))
        damaged.append(bad)
    for bad in damaged:
        flags, total, got, _ = decode_located(torch, lib, alg, bad, S.stream_ranges(bad.size, 4), [2 * data.size] * 4)
        if flags == 0:                               # accepted: exactly what the stream decodes to on one device
            want = _decode_device(torch, alg, bad, 2 * data.size)
            assert want is not None and np.concatenate(got).size == want.size and (np.concatenate(got) == want).all()
    # a cap one byte short on one rank is refused
    flags, _, got, located = decode_located(torch, lib, alg, s, lay)
    sizes = [g.size for g in got]
    for r in range(4):
        if sizes[r]:
            caps = [max(z, 4) for z in sizes]
            caps[r] = sizes[r] - 1
            flags, _, _, _ = decode_located(torch, lib, alg, s, lay, caps)
            assert flags != 0, r


def test_prot_enter_rejects_bad_arguments(torch_cuda, lib):
    torch = torch_cuda
    h = lib.density_b200_decode_shard_create()
    d = torch.zeros(1024, dtype=torch.uint8, device="cuda")
    t = torch.zeros(65536, dtype=torch.int32, device="cuda")
    st = _stream(torch)
    assert lib.density_b200_decode_shard_prot_enter(h, d.data_ptr(), 1024, 4096, 1, 3200, t.data_ptr(), st) == 4
    assert lib.density_b200_decode_shard_prot_enter(h, d.data_ptr() + 1, 1022, 4096, 1, 0, t.data_ptr(), st) == 4
    assert lib.density_b200_decode_shard_prot_phase2(h, None, d.data_ptr(), d.data_ptr(), d.data_ptr(), st) == 4   # no phase 1 yet
    lib.density_b200_decode_shard_destroy(h)
    c = lib.density_b200_cheetah_decode_shard_create()
    assert lib.density_b200_cheetah_decode_shard_prot_enter(c, d.data_ptr(), 1024, d.data_ptr(), 1024, 1, 1, 3200, None, st) == 4
    lib.density_b200_cheetah_decode_shard_destroy(c)
    m = torch.zeros(8, dtype=torch.int32, device="cuda")
    assert lib.density_b200_decode_prot_locate(None, d.data_ptr(), 16, 0, m.data_ptr(), st) == 4


# ---- 4. the NCCL drivers at one rank ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", ALGS)
def test_driver_world_one_and_python(torch_cuda, lib, alg):
    """density_b200_decode_sharded[_cheetah]_stream_protected at world 1 (no collective) and ShardedChameleonDecoder's phase path equal
    the original bytes; the driver alternates with the quiet stream entry on one handle"""
    from density_b200 import sharded as S
    torch = torch_cuda
    data, s = corpus("noise", alg)
    d = S.ShardedDecoder(torch.device("cuda"))
    d_in = torch.from_numpy(np.ascontiguousarray(s)).cuda()
    cap = (2 if alg == "chameleon" else 16) * s.size
    out = torch.full((cap + 64,), CANARY, dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    fl = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    for _ in range(2):
        d.decode_stream_protected(d_in, s.size, out, sz, fl, alg=alg)
        torch.cuda.synchronize()
        assert int(fl.item()) == 0 and int(sz.item()) == data.size and int(d.d_offset.item()) == 0
        assert (out[:data.size].cpu().numpy() == data).all() and bool((out[cap:] == CANARY).all())
        d.decode_stream(d_in, s.size, out, sz, fl, alg=alg, range_offset=0)
        torch.cuda.synchronize()
        # the quiet Chameleon entry refuses noise; Cheetah's accepts copy mode in the range that holds the stream start
        assert (int(fl.item()) != 0) == (alg == "chameleon")
    with pytest.raises(ValueError):
        d.decode_stream_protected(d_in, s.size, out, sz, fl, alg="lion")
    with pytest.raises(ValueError):                    # a range longer than the buffer: no negative halo reaches the library
        d.decode_stream_protected(d_in, s.size + 2, out, sz, fl, alg=alg)
    d.close()
    if alg == "chameleon":
        dec = S.ShardedChameleonDecoder()
        flags, total, offsets, mine = dec.decode_stream_protected(d_in, s.size, out, sz)
        torch.cuda.synchronize()
        assert flags == 0 and total == data.size and mine == 0 and (out[:data.size].cpu().numpy() == data).all()
        dec.close()


# ---- 5. output offsets beyond 4 GiB ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", ALGS)
def test_output_offsets_beyond_4gib(torch_cuda, lib, alg):
    """The pair corpus of tests/big_streams.py with its noise bursts (a stream of more than 2**32 + 2**28 bytes, copy-mode blocks at
    stream offsets above 2**32) in two ranges, the second starting past 2**32 bytes of stream: its map header carries n_range above
    2**32 (rank 0's), rank 1 locates its piece in the copy-mode region's automaton state and writes its output above 2**32, and the
    decoded bytes equal the input."""
    import big_streams as bs
    torch = torch_cuda
    n = bs.SIZE[alg]
    if torch.cuda.mem_get_info()[0] < 24 * (1 << 30):
        pytest.skip("needs 24 GiB of free device memory")
    data = bs.corpus(alg, n, bursts=True)
    stream, copied = bs.oracle_stream(alg, data)
    m = stream.size
    assert m > bs.STREAM_MIN and copied > 0
    r0 = ((1 << 32) // L.RANGE_UNIT + 1) * L.RANGE_UNIT
    lay = L.layout(m, [r0, m - r0])
    flags, total, got, located = decode_located(torch, lib, alg, stream, lay, caps=[2 * (r + h) for _, r, h in lay])
    del stream
    assert flags == 0 and total == n, located
    assert located[0][3] == 1 and located[1][3] == 0 and located[1][2] == 1
    offsets = [0, got[0].size, got[0].size + got[1].size]
    assert offsets[1] > (1 << 32) and offsets[2] == n
    for r in range(2):
        off = bs.first_difference(got[r], data[offsets[r]:offsets[r + 1]])
        assert off is None, f"rank {r}: first difference at output byte {offsets[r] + off}"
