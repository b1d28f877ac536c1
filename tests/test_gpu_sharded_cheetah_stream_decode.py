"""Sharded decode of a Cheetah stream without known cuts (needs an H100: pytest -m gpu): the device range maps equal the numpy model (the
start range's row from the exact boundary walk, copy-mode blocks included), every rank finds where its piece starts, the located pieces
decode back to the original, and the verdict refuses every stream it cannot decode piecewise without writing past any cap."""
import ctypes

import numpy as np
import pytest

import oracle
import planted
from conftest import splitmix_bytes
from locate_model import layout
from locate_model_cheetah import HALO, RANGE, exact_walk, range_map

pytestmark = pytest.mark.gpu

CANARY = 0xA5
MIB = 1 << 20
WORDS = 142


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


def text(n, first_page=0):
    from density_b200 import synth
    return synth.synth_text(n, first_page=first_page).numpy()


def device_encode(torch, data):
    """One cheetah_encode call on the device."""
    import density_b200
    d_in = torch.from_numpy(data.copy()).cuda()
    out = torch.zeros(density_b200.load().cheetah_safe_encode_buffer_size(data.size) + 64, dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    density_b200.encode_device("cheetah", d_in, out, sz)
    torch.cuda.synchronize()
    return out[:int(sz.item())].cpu().numpy()


def decode_device(torch, enc, cap):
    import density_b200
    d_in = torch.from_numpy(np.ascontiguousarray(enc)).cuda()
    out = torch.zeros(max(cap, 4), dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    density_b200.decode_device("cheetah", d_in, enc.size, out, sz)
    torch.cuda.synchronize()
    return out[:int(sz.item())].cpu().numpy()


def device_map(torch, lib, h, buf, n_range, n_halo, offset):
    d_in = torch.from_numpy(np.ascontiguousarray(buf[:n_range + n_halo])).cuda()
    m = torch.full((WORDS,), -1, dtype=torch.int64, device="cuda")
    rc = lib.density_b200_cheetah_decode_locate(h, d_in.data_ptr() if d_in.numel() else None, n_range, n_halo, offset, m.data_ptr(), _stream(torch))
    assert rc == 0, lib.density_b200_last_error()
    torch.cuda.synchronize()
    return m.cpu().numpy().view(np.uint64)


def decode_located(torch, lib, stream, lay, caps=None):
    """ShardedDecoder.decode_stream(alg="cheetah") with the ranks simulated in sequence on one GPU: every rank's range map, the stacked
    maps (as the all_gather), locate_piece, then the piece phases on the located pieces with their is_first / is_last, the exchanges
    replaced by stacking the transfers and folding them with fold_cheetah_cmap / fold_cl_tables. Returns the decoded pieces, the
    verdict, whether the canaries behind every cap held, the located pieces and each piece's status words."""
    from density_b200 import sharded
    world = len(lay)
    st = _stream(torch)
    caps = caps or [16 * (n + h) for _, n, h in lay]
    hs, ins, maps = [], [], []
    for o, n, h in lay:
        hd = lib.density_b200_cheetah_decode_shard_create()
        assert hd
        d_in = torch.from_numpy(np.ascontiguousarray(stream[o:o + n + h])).cuda()
        m = torch.empty(WORDS, dtype=torch.int64, device="cuda")
        rc = lib.density_b200_cheetah_decode_locate(hd, d_in.data_ptr() if d_in.numel() else None, n, h, o, m.data_ptr(), st)
        assert rc == 0, lib.density_b200_last_error()
        hs.append(hd); ins.append(d_in); maps.append(m)
    gathered = torch.stack(maps).cpu().numpy().view(np.uint64)
    located = [sharded.locate_piece(gathered, r, alg="cheetah") for r in range(world)]
    wc, wp = lib.density_b200_cheetah_cmap_words(), lib.density_b200_cl_table_words(1, sharded.CL_TABLE_P)
    tc = torch.zeros((world, wc), dtype=torch.int32, device="cuda")
    outs = []
    for r in range(world):
        start, end, _, final, first = located[r]
        piece = ins[r][start:end]
        d_out = torch.full((caps[r] + 64,), CANARY, dtype=torch.uint8, device="cuda")
        rc = lib.density_b200_cheetah_decode_shard_phase1(hs[r], piece.data_ptr() if piece.numel() else None, piece.numel(), d_out.data_ptr(),
                                                          caps[r], first, final, tc[r].data_ptr(), st)
        assert rc == 0, lib.density_b200_last_error()
        outs.append(d_out)
    for r in range(world):
        carry = sharded.fold_cheetah_cmap(tc, r) if not located[r][4] else None
        assert lib.density_b200_cheetah_decode_shard_phase2(hs[r], carry.data_ptr() if carry is not None else None, st) == 0
    tp = torch.zeros((world, wp), dtype=torch.int32, device="cuda")
    words = torch.zeros((world, 4), dtype=torch.int32, device="cuda")
    for _ in range(lib.density_b200_cheetah_decode_round_budget()):
        for r in range(world):
            assert lib.density_b200_cheetah_decode_shard_round_walk(hs[r], tp[r].data_ptr(), words[r].data_ptr(), st) == 0
        for r in range(world):
            carry = sharded.fold_cl_tables("cheetah", sharded.CL_TABLE_P, tp, r) if not located[r][4] else None
            rc = lib.density_b200_cheetah_decode_shard_round_fold(hs[r], carry.data_ptr() if carry is not None else None, words.data_ptr(),
                                                                  world, r, st)
            assert rc == 0, lib.density_b200_last_error()
    seam = torch.zeros((world, 8), dtype=torch.int32, device="cuda")
    sizes = torch.full((world,), -1, dtype=torch.int64, device="cuda")
    for r in range(world):
        assert lib.density_b200_cheetah_decode_shard_phase3(hs[r], sizes[r:r + 1].data_ptr(), seam[r].data_ptr(), st) == 0
    torch.cuda.synchronize()
    status = []
    for r in range(world):
        s4 = (ctypes.c_uint32 * 4)()
        assert lib.density_b200_cheetah_decode_shard_status(hs[r], s4) == 0
        status.append(list(s4))
        lib.density_b200_cheetah_decode_shard_destroy(hs[r])
    verdict = sharded.seam_verdict(seam)
    canaries = all(bool((outs[r][caps[r]:] == CANARY).all()) for r in range(world))
    got = [outs[r][:int(sizes[r].item())].cpu().numpy() for r in range(world)]
    return got, verdict, canaries, located, status


def check_round_trip(torch, lib, stream, data, lay):
    got, (flags, total, offsets), canaries, located, status = decode_located(torch, lib, stream, lay)
    assert flags == 0 and total == data.size and canaries, lay
    for r, piece in enumerate(got):
        assert offsets[r] == 128 * located[r][2] or piece.size == 0
    assert all(s[1] == 1 for s in status)
    out = np.concatenate(got) if got else np.zeros(0, np.uint8)
    assert out.size == data.size and (out == data).all()


def padded_for_short_last(data):
    """data with zero blocks appended until its stream's length mod 16 KiB lies in [1, 135]: the last range is shorter than a block and
    the stream ends inside the halo of the rank before. Once the tables hold zeros a zero block is its 8-byte signature alone."""
    base = data[:data.size // 128 * 128]
    k = 16
    for _ in range(20):
        d = np.concatenate([base, np.zeros(128 * k, np.uint8)])
        s = oracle.encode("cheetah", d)
        r = s.size % RANGE
        if 1 <= r < 136 and s.size > 2 * RANGE:
            return d, s
        k += max(1, (64 - r) % RANGE // 8)
    raise AssertionError("no padding found")


def layouts(stream):
    from density_b200 import sharded
    total = stream.size
    k = total // RANGE
    out = {f"ranges{w}": sharded.stream_ranges(total, w) for w in (2, 3, 5, 8)}
    if k >= 3:
        a = k // 3 * RANGE
        out["zero_middle"] = layout(total, [a, 0, 0, a, 0, total - 2 * a])
        out["start_on_rank1"] = layout(total, [0, a, total - a])
    starts, _, _ = exact_walk(stream)
    on = starts[(starts >= RANGE) & (starts % RANGE == 0)]
    if on.size:
        out["on_block_start"] = layout(total, [int(on[0]), total - int(on[0])])
    return out


def _check_all_layouts(torch, lib, stream, data):
    for lay in layouts(stream).values():
        check_round_trip(torch, lib, stream, data, lay)


# ---- 1. the device maps are the model's ------------------------------------------------------------------------------------------
def test_device_maps_equal_model(torch_cuda, lib):
    torch = torch_cuda
    s = oracle.encode("cheetah", text(3 * MIB + 5))
    starts, copied, _ = exact_walk(s)
    assert copied.any() and int(starts[copied][-1]) < RANGE
    h = lib.density_b200_cheetah_decode_shard_create()
    o = 6 * RANGE
    cases = [
        (s[o:], 10 * RANGE, HALO, o),                    # a quiet range in the middle of the stream
        (s, RANGE, HALO, 0),                             # the start range: its cold-start copy-mode blocks are walked
        (s, 4096, HALO, 0),                              # a start range that ends inside the copy region
        (s, 80 * 4096, HALO, 0),                         # a start range over two groups
        (s[o:o + RANGE + 100], RANGE, 100, o),           # short halo: the stream ends inside it
        (s[:RANGE + 100], RANGE, 100, 0),                # the same on the start range
        (s[o:o + 100], 0, 100, o),                       # an empty range
        (s[:100], 0, 100, 0),                            # an empty range at offset 0 has no start row
        (s[:100], 100, 0, 0),                            # a tiny stream
        (s[RANGE:], 70 * 4096, HALO, RANGE),             # 70 chunks: two groups, the second short
    ]
    for buf, n, hl, off in cases:
        got = device_map(torch, lib, h, buf, n, hl, off)
        want = range_map(buf, n, hl, off)
        assert (got == want).all(), (n, hl, off, np.nonzero(got != want))
    lib.density_b200_cheetah_decode_shard_destroy(h)


# ---- 2. round trips ----------------------------------------------------------------------------------------------------------------
def test_round_trip_single_call_and_oracle_stream(torch_cuda, lib):
    data = text(5 * MIB + 403, first_page=3)
    s = device_encode(torch_cuda, data)
    o = oracle.encode("cheetah", data)
    assert s.size == o.size and (s == o).all()
    _check_all_layouts(torch_cuda, lib, s, data)


def test_round_trip_dickens_zeros_cl1(torch_cuda, lib, dickens200k):
    for data in (dickens200k, np.zeros(3 * MIB + 12, np.uint8), planted.corpus("cl1")[0]):
        _check_all_layouts(torch_cuda, lib, oracle.encode("cheetah", data), data)


def test_round_trip_zeros_on_block_start(torch_cuda, lib):
    data = np.zeros(3 * MIB, np.uint8)
    s = oracle.encode("cheetah", data)
    assert "on_block_start" in layouts(s)
    check_round_trip(torch_cuda, lib, s, data, layouts(s)["on_block_start"])


def test_round_trip_short_last_range(torch_cuda, lib):
    data, s = padded_for_short_last(text(MIB + 17, first_page=2))
    k = s.size // RANGE
    for lay in (layout(s.size, [k * RANGE, s.size - k * RANGE]), layout(s.size, [(k - 1) * RANGE, RANGE, s.size - k * RANGE]),
                layout(s.size, [k * RANGE, 0, 0, s.size - k * RANGE])):
        check_round_trip(torch_cuda, lib, s, data, lay)


@pytest.mark.parametrize("n", [0, 1, 5, 200, 3000])
def test_round_trip_tiny_stream_world4(torch_cuda, lib, n):
    """stream_ranges of a stream shorter than 16 KiB: ranks 0-2 are empty and the start piece is on rank 3."""
    from density_b200 import sharded
    data = text(max(n, 1))[:n]
    s = oracle.encode("cheetah", data)
    assert s.size < RANGE
    _, _, _, located, _ = decode_located(torch_cuda, lib, s, sharded.stream_ranges(s.size, 4))
    assert [p[4] for p in located] == [0, 0, 0, int(s.size > 0)]
    check_round_trip(torch_cuda, lib, s, data, sharded.stream_ranges(s.size, 4))


# ---- 3. refusals and the invariant -------------------------------------------------------------------------------------------------
def check_invariant(torch, lib, stream, lay, caps=None):
    """Either the verdict is non-zero and every canary holds, or it is 0 and the output equals decode_device's byte for byte."""
    got, (flags, total, _), canaries, _, _ = decode_located(torch, lib, stream, lay, caps)
    assert canaries
    if flags:
        return flags
    want = decode_device(torch, stream, sum(g.size for g in got) + 64)
    cat = np.concatenate(got)
    assert total == want.size == cat.size and (cat == want).all()
    return flags


def test_start_range_inside_the_cold_start_copy_region(torch_cuda, lib):
    """Noise in front of text: the cold-start copy region runs past the first 16 KiB. A start range that ends inside it is refused; the
    first 16 KiB multiple behind the copy region decodes."""
    torch = torch_cuda
    data = np.concatenate([splitmix_bytes(48 * 1024, 3), text(MIB, first_page=1)])
    s = oracle.encode("cheetah", data)
    starts, copied, _ = exact_walk(s)
    end_copy = int(starts[copied][-1]) + 128
    assert end_copy > 2 * RANGE
    assert check_invariant(torch, lib, s, layout(s.size, [RANGE, s.size - RANGE])) != 0
    c = (end_copy // RANGE + 1) * RANGE
    assert check_invariant(torch, lib, s, layout(s.size, [c, s.size - c])) == 0
    check_round_trip(torch, lib, s, data, layout(s.size, [c, RANGE, s.size - c - RANGE]))


def test_refuses_copy_mode_after_the_start_range_and_a_pair_across_a_cut(torch_cuda, lib):
    from density_b200 import sharded
    torch = torch_cuda
    t = text(2 * MIB, first_page=5)
    noise = splitmix_bytes(MIB, 12)
    d = np.concatenate([t[:MIB], noise[:256 * 1024], t[MIB:]])
    s = oracle.encode("cheetah", d)
    for w in (2, 3):
        assert check_invariant(torch, lib, s, sharded.stream_ranges(s.size, w)) != 0
    assert check_invariant(torch, lib, s, sharded.stream_ranges(s.size, 1)) == 0      # one piece: copy mode is the start piece's to use
    # a planted incompressible pair in range 1: the protection automaton copies the blocks behind it
    d = t.copy()
    p = t.size * 3 // 4 // 128 * 128
    d[p:p + 256] = noise[:256]
    s = oracle.encode("cheetah", d)
    lay = sharded.stream_ranges(s.size, 2)
    starts, copied, _ = exact_walk(s)
    assert copied[starts >= lay[1][0]].any()
    assert check_invariant(torch, lib, s, lay) != 0
    # two incompressible blocks, the first starting in the last 128 bytes before a 16 KiB multiple: the located cut falls between them
    s0 = oracle.encode("cheetah", t)
    starts, _, _ = exact_walk(s0)
    i = int(np.nonzero((starts % RANGE >= RANGE - 128) & (starts > 4 * RANGE))[0][0])
    c = (int(starts[i]) // RANGE + 1) * RANGE
    d = t.copy()
    d[128 * i:128 * i + 256] = noise[:256]
    s = oracle.encode("cheetah", d)
    assert int(exact_walk(s)[0][i]) == int(starts[i])
    assert check_invariant(torch, lib, s, layout(s.size, [c, s.size - c])) != 0


def test_invariant_truncated(torch_cuda, lib):
    from density_b200 import sharded
    s = oracle.encode("cheetah", text(2 * MIB + 77))
    for cut in (1, 2, 3, 100, 300):
        t = s[:-cut]
        for w in (1, 3):
            check_invariant(torch_cuda, lib, t, sharded.stream_ranges(t.size, w))


def test_invariant_flipped_signature_bits(torch_cuda, lib):
    from density_b200 import sharded
    s = oracle.encode("cheetah", text(2 * MIB + 77))
    starts, _, _ = exact_walk(s)
    lay = sharded.stream_ranges(s.size, 3)
    before_cut = [int(starts[np.searchsorted(starts, o) - 1]) for o, _, _ in lay[1:]]
    rng = np.random.default_rng(9)
    for b in before_cut + [int(x) for x in rng.choice(starts, 3)]:
        for bit in (0, 63):
            t = s.copy()
            t[b + bit // 8] ^= 1 << (bit % 8)
            check_invariant(torch_cuda, lib, t, lay)


def test_invariant_cap_one_short_and_cap_16x_on_zeros(torch_cuda, lib):
    from density_b200 import sharded
    data = text(2 * MIB + 77)
    s = oracle.encode("cheetah", data)
    lay = sharded.stream_ranges(s.size, 3)
    got, (flags, _, _), _, _, _ = decode_located(torch_cuda, lib, s, lay)
    assert flags == 0
    for r in range(3):
        caps = [16 * (n + h) for _, n, h in lay]
        caps[r] = got[r].size - 1
        assert check_invariant(torch_cuda, lib, s, lay, caps) != 0
    z = np.zeros(4 * MIB, np.uint8)
    s = oracle.encode("cheetah", z)
    lay = sharded.stream_ranges(s.size, 3)
    got, (flags, total, _), canaries, _, _ = decode_located(torch_cuda, lib, s, lay, [16 * (n + h) for _, n, h in lay])
    assert flags == 0 and canaries and total == z.size and not np.concatenate(got).any()


# ---- 4. the C++ entry --------------------------------------------------------------------------------------------------------------
def test_cpp_entry_world1_equals_decode_device_and_alternates(torch_cuda, lib):
    """The world-1 C++ entry equals decode_device and alternates with decode_sharded_cheetah on one handle; it adds exactly the 11
    locate kernels of the range that holds the stream start to the launches of decode_sharded_cheetah, which are unchanged."""
    torch = torch_cuda
    from density_b200 import sharded
    dec = sharded.ShardedDecoder(torch.device("cuda"))
    for data in (text(3 * MIB + 1021), np.concatenate([text(MIB), splitmix_bytes(100 * 1024, 2), text(77, 3)]), np.zeros(MIB + 3, np.uint8)):
        enc = oracle.encode("cheetah", data)
        want = decode_device(torch, enc, data.size + 64)
        assert (want == data).all()
        d_in = torch.from_numpy(enc.copy()).cuda()
        cap = 16 * enc.size
        d_out = torch.full((cap + 64,), CANARY, dtype=torch.uint8, device="cuda")
        d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
        d_fl = torch.ones(1, dtype=torch.int32, device="cuda")
        launches = []
        for k in range(2):
            d_fl.fill_(1); dec.d_offset.fill_(-1)
            torch.cuda.synchronize()
            before = lib.density_b200_kernel_launches()
            dec.decode_stream(d_in, enc.size, d_out[:cap], d_sz, d_fl, alg="cheetah", range_offset=0)
            torch.cuda.synchronize()
            launches.append(lib.density_b200_kernel_launches() - before)
            assert int(d_fl.item()) == 0 and int(d_sz.item()) == data.size == int(dec.d_total.item()) and int(dec.d_offset.item()) == 0
            assert (d_out[:data.size].cpu().numpy() == want).all() and bool((d_out[cap:] == CANARY).all())
            d_fl.fill_(1)
            before = lib.density_b200_kernel_launches()
            dec.decode(d_in, d_out[:cap], d_sz, d_fl, alg="cheetah")
            torch.cuda.synchronize()
            launches.append(lib.density_b200_kernel_launches() - before)
            assert int(d_fl.item()) == 0 and (d_out[:data.size].cpu().numpy() == want).all()
        # decode_sharded_cheetah on one rank: phase 1 (9 boundary kernels + 3), phase 2 (3), 40 rounds x 4, phase 3 (3), the verdict
        assert launches[1] == launches[3] == 179 and launches[0] == launches[2] == 179 + 11, launches
    dec.close()


def test_python_decode_stream_arguments(torch_cuda, lib):
    from density_b200 import sharded
    torch = torch_cuda
    dec = sharded.ShardedDecoder(torch.device("cuda"))
    d = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    fl = torch.zeros(1, dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError):
        dec.decode_stream(d, 4096, d, sz, fl, alg="cheetah")              # range_offset missing
    with pytest.raises(ValueError):
        dec.decode_stream(d, 4096, d, sz, fl, alg="lion", range_offset=0)
    dec.close()


# ---- 5. argument checks (one rank only: a rank that returned before a collective would leave the others waiting in it) -----------
def test_decode_sharded_cheetah_stream_rejects_bad_arguments(torch_cuda, lib):
    torch = torch_cuda
    from density_b200 import sharded
    h = sharded.ShardedDecoder(torch.device("cuda"))
    data = text(64 * 1024)
    s = oracle.encode("cheetah", data)
    buf = torch.zeros(20 * s.size + 4096, dtype=torch.uint8, device="cuda")
    buf[:s.size] = torch.from_numpy(s).cuda()
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    fl = torch.zeros(1, dtype=torch.int32, device="cuda")
    off = torch.zeros(1, dtype=torch.int64, device="cuda")
    p, st, n = buf.data_ptr(), _stream(torch), s.size
    o = p + s.size + 1024 - (s.size + 1024) % 4
    cap = 16 * n
    f = lib.density_b200_decode_sharded_cheetah_stream
    assert f(h._h, p + 1, n - 1, 0, 0, o, cap, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 4     # misaligned d_in
    assert f(h._h, p, n, 0, 0, o + 2, cap, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 4        # misaligned d_out
    assert f(h._h, None, n, 0, 0, o, cap, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 4
    assert f(h._h, p, n, 0, 0, None, cap, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 4
    assert f(h._h, p, n, 0, 0, o, cap, None, off.data_ptr(), fl.data_ptr(), None, st) == 4
    assert f(h._h, p, n, 0, 0, o, cap, sz.data_ptr(), off.data_ptr(), None, None, st) == 4
    assert f(None, p, n, 0, 0, o, cap, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 4
    assert f(h._h, p, n - 10, 10, 0, o, cap, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 4     # the last rank has a halo
    assert f(h._h, p, n, 0, 2, o, cap, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 4           # no range at offset 0
    assert f(h._h, p, n, 0, 0, o, cap, sz.data_ptr(), off.data_ptr(), fl.data_ptr(), None, st) == 0           # and the good call works
    torch.cuda.synchronize()
    assert int(fl.item()) == 0 and int(sz.item()) == data.size and int(off.item()) == 0
    assert (buf[o - p:o - p + data.size].cpu().numpy() == data).all()
    hd = lib.density_b200_cheetah_decode_shard_create()
    m = torch.zeros(WORDS, dtype=torch.int64, device="cuda")
    assert lib.density_b200_cheetah_decode_locate(hd, p + 1, 100, 0, 0, m.data_ptr(), st) == 4
    assert lib.density_b200_cheetah_decode_locate(hd, p, 100, 0, 0, m.data_ptr() + 4, st) == 4
    assert lib.density_b200_cheetah_decode_locate(hd, p, 100, 0, 0, None, st) == 4
    assert lib.density_b200_cheetah_decode_locate(None, p, 100, 0, 0, m.data_ptr(), st) == 4
    assert lib.density_b200_cheetah_decode_locate(hd, None, 100, 0, 0, m.data_ptr(), st) == 4
    lib.density_b200_cheetah_decode_shard_destroy(hd)
    h.close()


def test_output_offsets_beyond_4gib(torch_cuda, lib):
    """The 7.5 GiB Cheetah pair corpus of tests/big_streams.py (a stream of more than 2**32 + 2**28 bytes, every block distinct) in two
    ranges, the second starting past 2**32 bytes of stream: rank 1 locates its piece, carries the chunk map and the prediction rounds
    across the cut and writes its output above 2**32, and the decoded bytes equal the input."""
    import big_streams as bs
    torch = torch_cuda
    n = bs.SIZE["cheetah"]
    if torch.cuda.mem_get_info()[0] < 24 * (1 << 30):
        pytest.skip("needs 24 GiB of free device memory")
    data = bs.corpus("cheetah", n)
    stream, _ = bs.oracle_stream("cheetah", data)
    m = stream.size
    assert m > bs.STREAM_MIN
    r0 = ((1 << 32) // RANGE + 1) * RANGE
    lay = layout(m, [r0, m - r0])
    got, (flags, total, offsets), canaries, located, status = decode_located(torch, lib, stream, lay, caps=[2 * (r + h) for _, r, h in lay])
    del stream
    assert flags == 0 and total == n and canaries
    assert all(s[1] == 1 for s in status), status
    assert int(offsets[1]) > (1 << 32) and int(offsets[1]) == 128 * located[1][2]
    for r in range(2):
        assert got[r].size == int(offsets[r + 1] - offsets[r])
        off = bs.first_difference(got[r], data[int(offsets[r]):int(offsets[r + 1])])
        assert off is None, f"rank {r}: first difference at output byte {int(offsets[r]) + off}"


# ---- 6. two ranks over NCCL --------------------------------------------------------------------------------------------------------
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
    d_data = synth.synth_text(n, device=dev)
    d_enc = torch.zeros(density_b200.load().cheetah_safe_encode_buffer_size(n), dtype=torch.uint8, device=dev)
    d_sz = torch.zeros(1, dtype=torch.int64, device=dev)
    density_b200.encode_device("cheetah", d_data, d_enc, d_sz)
    torch.cuda.synchronize()
    m = int(d_sz.item())
    o, nr, hl = sharded.stream_ranges(m, world)[rank]
    d_in = d_enc[o:o + nr + hl].clone()
    dec = sharded.ShardedDecoder(dev)
    cap = 16 * (nr + hl)
    d_out = torch.zeros(cap, dtype=torch.uint8, device=dev)
    d_fl = torch.ones(1, dtype=torch.int32, device=dev)
    dec.decode_stream(d_in, nr, d_out, d_sz, d_fl, alg="cheetah", range_offset=o)
    torch.cuda.synchronize()
    off, k = int(dec.d_offset.item()), int(d_sz.item())
    same = bool(torch.equal(d_out[:k], d_data[off:off + k]))
    q.put((rank, int(d_fl.item()), int(dec.d_total.item()), same, k))
    dist.barrier()
    dec.close()
    dist.destroy_process_group()


def test_decode_sharded_cheetah_stream_two_ranks_nccl(torch_cuda, lib):
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, n = 2, 24 * MIB + 5
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, world, 29743, n, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = dict((r, rest) for r, *rest in (q.get(timeout=600) for _ in range(world)))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert sum(got[r][3] for r in range(world)) == n
    for r in range(world):
        flag, total, same, _ = got[r]
        assert flag == 0 and total == n and same
