"""The Chameleon seek index on an H100 (pytest -m gpu): density_b200_chameleon_index_build(_device) held byte for byte to
tests/chameleon_index_model.py, and density_b200_chameleon_decode_range_indexed(_device) held window by window to the oracle slice and to
the non-indexed range decode's {w, S, verdict}, with guard bytes on both sides of d_out (at odd addresses) and around d_result. Also:
only the piece between the two checkpoints is read, an index survives a trip through host memory, malformed streams, refused and
mismatched indexes, launch counts, stream order, the shared workspace, the synchronous forms and the Python forms.
tests/test_chameleon_index_cpu.py checks the model against the oracle."""
import ctypes

import numpy as np
import pytest

import chameleon_index_model as X
import oracle
import synth_streams as ss
from conftest import payload
from decoded_size_witness import MALFORMED, oracle_size
from test_gpu_decode_range import (BS, CANARY, CH, GROUP_BYTES, GIB, MIB, PAD, RES_CANARY, TILE, Case, _cur, corpus, decoded_size,  # noqa: F401
                                   edges, lib, torch_cuda, upload, window)

pytestmark = pytest.mark.gpu
EARG, EMALFORMED = 4, 3
LAUNCHES_INDEXED = 15          # the entry, phase 1 (10), phase 2 (3), the checked copy-out
LAUNCHES_BUILD_LOCATE = 4      # the candidate rows (2), the stride walk, the report


def build_launches(count):
    return LAUNCHES_BUILD_LOCATE + 14 * count      # per piece: its entry (but the first: table_init), phase 1 with export (12), a fold


def build(torch, lib, ptr, n, interval, stream=None, cap=None):
    """-> (rc, (bytes, S, verdict), the index's bytes on the device (a tensor of `bytes` bytes) or None)"""
    bound = lib.density_b200_chameleon_index_bytes(n, interval)
    cap = bound if cap is None else cap
    buf = torch.full((max(cap, 1) + 2 * PAD,), CANARY, dtype=torch.uint8, device="cuda")
    res = torch.full((5,), RES_CANARY, dtype=torch.int64, device="cuda")
    s = _cur(torch) if stream is None else ctypes.c_void_p(stream.cuda_stream)
    rc = lib.density_b200_chameleon_index_build_device(ptr, n, interval, buf.data_ptr() + PAD, cap, res.data_ptr() + 8, s)
    torch.cuda.synchronize()
    r = res.cpu().numpy().view(np.uint64)
    assert int(r[0]) == RES_CANARY and int(r[4]) == RES_CANARY
    got = tuple(int(x) for x in r[1:4])
    o = buf.cpu().numpy()
    assert (o[:PAD] == CANARY).all() and (o[PAD + got[0]:] == CANARY).all(), "the build wrote outside [d_index, d_index + bytes)"
    return rc, got, (buf[PAD:PAD + got[0]].clone() if rc == 0 else None), o[PAD:PAD + cap]


def indexed(torch, lib, ptr, n, index, first, length, align=1, room=None, index_len=None):
    """one indexed range decode, guards as test_gpu_decode_range.window -> (rc, (w, S, verdict), d_out's bytes)"""
    room = length if room is None else room
    out = torch.full((room + 2 * PAD,), CANARY, dtype=torch.uint8, device="cuda")
    res = torch.full((5,), RES_CANARY, dtype=torch.int64, device="cuda")
    il = index.numel() if index_len is None else index_len
    rc = lib.density_b200_chameleon_decode_range_indexed_device(ptr, n, index.data_ptr(), il, first, length, out.data_ptr() + PAD + align,
                                                                res.data_ptr() + 8, _cur(torch))
    torch.cuda.synchronize()
    r = res.cpu().numpy().view(np.uint64)
    assert int(r[0]) == RES_CANARY and int(r[4]) == RES_CANARY, "the call wrote outside its 24 result bytes"
    o = out.cpu().numpy()
    got = tuple(int(x) for x in r[1:4])
    if rc != 0:
        assert (r[1:4] == RES_CANARY).all() and (o == CANARY).all(), "a refused call wrote its result words or d_out"
        return rc, None, None
    w = got[0]
    assert (o[:PAD + align] == CANARY).all(), "wrote in front of d_out"
    assert (o[PAD + align + w:] == CANARY).all(), f"wrote behind d_out + w (w = {w})"
    return rc, got, o[PAD + align:PAD + align + room]


class IndexedCase(Case):
    """a stream on the device, its index at one interval (checked against the model when `model`), its witness"""

    def __init__(self, torch, lib, stream, interval, D=None, model=True):
        super().__init__(torch, lib, stream, D)
        self.interval = interval
        rc, got, self.index, _ = build(torch, lib, self.ptr, self.s.size, interval)
        assert rc == 0 and got[1:] == (self.size, 0), got
        self.host_index = self.index.cpu().numpy().tobytes()
        if model:
            want, _ = X.build(self.s, interval)
            assert self.host_index == want, f"the index at interval {interval} differs from the model"
        assert got[0] == len(self.host_index) <= lib.density_b200_chameleon_index_bytes(self.s.size, interval)

    def check(self, first, length, what="", align=1, room=None):
        room = length if room is None else room
        rc, got, o = indexed(self.torch, self.lib, self.ptr, self.s.size, self.index, first, length, align, room)
        assert rc == 0, f"{what}: rc {rc}"
        ref = window(self.torch, self.lib, self.ptr, self.s.size, first, length, align, room=room)
        assert got == ref[1], f"{what} [{first}, +{length}): {got}, non-indexed {ref[1]}"
        want = self.D[first:first + length]
        assert got[0] == want.size and (o[:want.size] == want).all(), f"{what} [{first}, +{length}): differs from the oracle slice"
        return got


# ---- the index --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["text", "mixed", "noise"])
def test_index_matches_the_model_and_windows_match_the_oracle(torch_cuda, lib, kind):
    n = 3 * MIB + 12345
    data = corpus(kind, n)
    enc = oracle.encode("chameleon", data)
    for interval in (256 * 1000, MIB, 16 * MIB):                   # interval >= S: no checkpoint
        c = IndexedCase(torch_cuda, lib, enc, interval, D=data)
        x = X.parse(c.host_index)
        assert (x["count"] == 0) == (interval > n)
        pts = [0, interval, 2 * interval, n // 2, n - 300, n - 1] + [interval * j for j in range(1, x["count"] + 1, 3)]
        for k, (first, length) in enumerate(edges(pts, n, lens=(1, 300, interval + 7))):
            c.check(first, length, f"{kind} / {interval}", align=k % 4, room=min(length, n + 16))
        for first, length in ((0, n), (5, 3 * interval + 11), (n, 5), (n + 99, 1)):
            c.check(first, length, f"{kind} / {interval} span", room=min(length, n + 16))


def test_golden_and_known_answer_streams(torch_cuda, lib, golden_inputs):
    from test_decode_range_cpu import KAT_INPUT
    kat = oracle.encode("chameleon", KAT_INPUT, cap=len(KAT_INPUT))
    c = IndexedCase(torch_cuda, lib, kat, 256)
    for first in range(len(KAT_INPUT) + 2):
        for length in (1, 2, 64, 200):
            c.check(first, length, "kat")
    for name, data in golden_inputs.items():
        if data.size > 2 * MIB or data.size < 1000:
            continue
        enc = oracle.encode("chameleon", data)
        for interval in (256 * 37, 64 << 10):
            c = IndexedCase(torch_cuda, lib, enc, interval, D=data)
            for k, (first, length) in enumerate(edges([0, interval, data.size // 2, data.size - 2], data.size, lens=(1, 999))):
                c.check(first, length, name, align=k % 4)


def test_seams_and_copy_mode_checkpoints(torch_cuda, lib):
    """windows at +-1 of checkpoints, blocks, tiles, decoder runs, boundary-row chunks and groups, and the tail, on a planted quiet
    corpus and on copy-mode data, with checkpoints every few blocks (many beside copy-mode episodes)"""
    import planted
    for name, interval in (("cham5", 256 * 251), ("copy3", 256 * 97)):
        data, _ = planted.corpus(name)
        enc = oracle.encode("chameleon", data)
        c = IndexedCase(torch_cuda, lib, enc, interval, D=data, model=data.size <= 4 * MIB)
        w = ss.walk("chameleon", enc)
        starts, S = w["starts"], data.size
        pts = [BS * k for k in (1, 63, 64, 65)] + [TILE * k for k in (1, 17)] + [interval * k for k in (1, 2, 5, 40)]
        pts += [BS * b for b in ss.seam_blocks("chameleon", enc.size, S, w["main_blocks"])[:4]]
        for edge in (CH, 7 * CH, GROUP_BYTES):
            b = int(np.searchsorted(starts, edge, side="right")) - 1
            if 0 <= b < len(starts):
                pts += [b * BS, (b + 1) * BS]
        pts += [BS * w["main_blocks"], S - 3]
        for first, length in edges(pts, S, lens=(1, 257, 3 * interval)):
            c.check(first, length, name, align=first % 4)


# ---- only the piece is read ---------------------------------------------------------------------------------------------------
def test_only_the_piece_is_read(torch_cuda, lib):
    torch = torch_cuda
    data = corpus("mixed", 4 * MIB + 7)
    enc = oracle.encode("chameleon", data)
    interval = 256 << 10
    c = IndexedCase(torch, lib, enc, interval, D=data, model=False)
    for first, length in ((0, 1000), (MIB + 5, 300000), (3 * MIB - 1, 2), (data.size - 1000, 5000)):
        p = X.plan(c.host_index, enc.size, first, length)
        poisoned = np.full(enc.size, 0x55, np.uint8)
        poisoned[p["off"]:p["end"]] = enc[p["off"]:p["end"]]
        d, ptr = upload(torch, poisoned)
        rc, got, o = indexed(torch, lib, ptr, enc.size, c.index, first, length)
        w = min(length, data.size - first)
        assert rc == 0 and got == (w, data.size, 0) and (o[:w] == data[first:first + w]).all()
        ho = np.full(length, CANARY, np.uint8)
        written = ctypes.c_uint64(0)
        hidx = np.frombuffer(c.host_index, np.uint8)
        assert lib.density_b200_chameleon_decode_range_indexed(poisoned.ctypes.data, enc.size, hidx.ctypes.data, hidx.size, first,
                                                               ho.ctypes.data, length, ctypes.byref(written)) == 0
        assert written.value == w and (ho[:w] == data[first:first + w]).all()


def test_index_round_trip_through_host_memory(torch_cuda, lib):
    torch = torch_cuda
    data = corpus("text", 2 * MIB + 3)
    enc = oracle.encode("chameleon", data)
    c = IndexedCase(torch, lib, enc, 128 << 10, D=data, model=False)
    saved = bytes(c.host_index)
    del c.index
    c.index = torch.from_numpy(np.frombuffer(saved, np.uint8).copy()).cuda()
    for first, length in ((0, 10), (MIB + 1, 70000), (data.size - 3, 3)):
        c.check(first, length, "reloaded")


# ---- malformed streams, refusals ------------------------------------------------------------------------------------------------
def test_malformed_streams_and_truncations(torch_cuda, lib):
    torch = torch_cuda
    s, _ = ss.build("chameleon", {"nbytes": 60000, "quiet": False, "copy_every": 23, "plant": False, "tail": (60, "raw2")}, 7)
    bad, _ = ss.build("chameleon", {"nbytes": 300000, "tail": (100, "map0")}, 26)
    verdicts = set()
    for stream in (s, bad):
        d, ptr = upload(torch, stream)
        for k in list(range(stream.size - 120, stream.size + 1, 7)) + [stream.size]:
            size, verdict = oracle_size("chameleon", stream[:k])
            assert decoded_size(torch, lib, ptr, k) == (size, verdict)
            rc, got, idx, raw = build(torch, lib, ptr, k, 256 * 23)
            verdicts.add(verdict)
            if verdict:
                assert rc == EMALFORMED and got == (0, 0, MALFORMED) and (raw == CANARY).all(), f"truncated at {k}"
            else:
                assert rc == 0 and got[1:] == (size, 0)
                want, _ = X.build(stream[:k], 256 * 23)
                assert idx.cpu().numpy().tobytes() == want
    assert verdicts == {0, MALFORMED}


def _corrupt(index, word=None, byte=None, value=0):
    a = np.frombuffer(index, np.uint8).copy()
    if word is not None:
        a[8 * word:8 * word + 8] = np.frombuffer(np.array([value], np.uint64).tobytes(), np.uint8)
    else:
        a[byte] = value
    return a


def _same_length(n):
    """a well-formed Chameleon stream of exactly n bytes that encodes noise, all copy-mode blocks (the input length found by bisection,
    then stepped: the raw tail of an input gives the encoded length a 1-byte resolution)"""
    from conftest import splitmix_bytes
    noise = splitmix_bytes(n + 4096, 5)
    lo, hi = 0, noise.size
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if oracle.encode("chameleon", noise[:mid]).size < n else (lo, mid)
    for L in range(hi, hi + 64):
        s = oracle.encode("chameleon", noise[:L])
        if s.size == n:
            return s
    raise AssertionError("no noise input encodes to exactly n bytes")


def test_refused_and_mismatched_indexes(torch_cuda, lib):
    torch = torch_cuda
    data = corpus("mixed", 2 * MIB + 11)
    enc = oracle.encode("chameleon", data)
    interval = 256 << 10
    c = IndexedCase(torch, lib, enc, interval, D=data, model=False)
    x = X.parse(c.host_index)
    assert x["count"] >= 3
    dir0 = 64
    cases = {
        "magic": _corrupt(c.host_index, word=0, value=1), "version": _corrupt(c.host_index, word=1, value=2),
        "n": _corrupt(c.host_index, word=2, value=enc.size + 2), "S small": _corrupt(c.host_index, word=3, value=x["main_blocks"] * 256 - 1),
        "S large": _corrupt(c.host_index, word=3, value=x["S"] + 10 ** 9), "main_blocks": _corrupt(c.host_index, word=4, value=10 ** 12),
        "interval": _corrupt(c.host_index, word=5, value=interval + 1), "interval 0": _corrupt(c.host_index, word=5, value=0),
        "count": _corrupt(c.host_index, word=6, value=x["count"] - 1), "bytes": _corrupt(c.host_index, word=7, value=x["bytes"] + 1),
        "offset order": _corrupt(c.host_index, word=(dir0 + 16) // 8, value=x["off"][0]),
        "offset past n": _corrupt(c.host_index, word=(dir0 + 32) // 8, value=enc.size + 2),
        "offset odd": _corrupt(c.host_index, word=dir0 // 8, value=x["off"][0] + 1),
        "candidate": _corrupt(c.host_index, word=(dir0 + 8) // 8, value=3200),
        "checkpoint past the main loop": _corrupt(c.host_index, word=5, value=interval * 64),
    }
    before = lib.density_b200_kernel_launches()
    for name, a in cases.items():
        idx = torch.from_numpy(a).cuda()
        for first, length in ((0, 100), (MIB, 100)):
            rc, got, o = indexed(torch, lib, c.ptr, enc.size, idx, first, length)
            assert rc == EARG, name
        written = ctypes.c_uint64(7)
        ho = np.full(100, CANARY, np.uint8)
        assert lib.density_b200_chameleon_decode_range_indexed(enc.ctypes.data, enc.size, a.ctypes.data, a.size, MIB, ho.ctypes.data, 100,
                                                               ctypes.byref(written)) == EARG, name
        assert written.value == 0 and (ho == CANARY).all()
    rc, _, _ = indexed(torch, lib, c.ptr, enc.size, c.index, 0, 100, index_len=c.index.numel() - 1)
    assert rc == EARG
    assert lib.density_b200_kernel_launches() == before, "a refused index ran a kernel"
    # a well-formed index of another stream of the same length whose structure differs: EMALFORMED, d_out untouched
    other = _same_length(enc.size)
    do, optr = upload(torch, other)
    rc, got, idx, _ = build(torch, lib, optr, other.size, interval)
    assert rc == 0
    for first in (0, MIB + 3, got[1] - 10):
        out = torch.full((1000 + 2 * PAD,), CANARY, dtype=torch.uint8, device="cuda")
        res = torch.zeros(3, dtype=torch.int64, device="cuda")
        assert lib.density_b200_chameleon_decode_range_indexed_device(c.ptr, enc.size, idx.data_ptr(), idx.numel(), first, 1000,
                                                                      out.data_ptr() + PAD, res.data_ptr(), _cur(torch)) == 0
        torch.cuda.synchronize()
        assert res.cpu().tolist() == [0, got[1], EMALFORMED] and bool((out == CANARY).all()), first
    # build refusals: a capacity one byte short, a bad interval, a misaligned d_index, n == 0; nothing enqueued
    buf = torch.zeros(c.index.numel() + 64, dtype=torch.uint8, device="cuda")
    res = torch.zeros(3, dtype=torch.int64, device="cuda")
    bound = lib.density_b200_chameleon_index_bytes(enc.size, interval)
    before = lib.density_b200_kernel_launches()
    for ptr, n, iv, d, cap in ((c.ptr, enc.size, interval, buf.data_ptr(), bound - 1), (c.ptr, enc.size, interval + 1, buf.data_ptr(), bound),
                               (c.ptr, enc.size, 0, buf.data_ptr(), bound), (c.ptr, enc.size, interval, buf.data_ptr() + 2, bound),
                               (c.ptr, 0, interval, buf.data_ptr(), bound), (c.ptr + 1, enc.size - 1, interval, buf.data_ptr(), bound)):
        assert lib.density_b200_chameleon_index_build_device(ptr, n, iv, d, cap, res.data_ptr(), _cur(torch)) == EARG
    torch.cuda.synchronize()
    assert lib.density_b200_kernel_launches() == before and not bool(buf.any())
    assert lib.density_b200_chameleon_index_bytes(enc.size, 255) == 0


# ---- launch counts, beyond 32 bits --------------------------------------------------------------------------------------------
def test_launch_counts(torch_cuda, lib):
    torch = torch_cuda
    data = corpus("text", 64 * MIB)
    enc = oracle.encode("chameleon", data)
    d, ptr = upload(torch, enc)
    for interval in (4 * MIB, 16 * MIB, 128 * MIB):
        before = lib.density_b200_kernel_launches()
        rc, got, idx, _ = build(torch, lib, ptr, enc.size, interval)
        count = X.parse(idx.cpu().numpy().tobytes())["count"]
        assert rc == 0 and lib.density_b200_kernel_launches() - before == build_launches(count), (interval, count)
    assert count == 0
    rc, got, idx, _ = build(torch, lib, ptr, enc.size, 4 * MIB)
    assert X.parse(idx.cpu().numpy().tobytes())["count"] == 15
    for first in (0, 17, 4 * MIB - 5, 31 * MIB, data.size - MIB, data.size - 1):
        before = lib.density_b200_kernel_launches()
        rc, got, o = indexed(torch, lib, ptr, enc.size, idx, first, MIB)
        w = min(MIB, data.size - first)
        assert rc == 0 and got == (w, data.size, 0) and (o[:w] == data[first:first + w]).all()
        assert lib.density_b200_kernel_launches() - before == LAUNCHES_INDEXED, first
    for first, length, extra in ((data.size, 5, 1), (data.size + 9, 5, 1), (7, 0, 0)):
        before = lib.density_b200_kernel_launches()
        rc, got, _ = indexed(torch, lib, ptr, enc.size, idx, first, length, room=8)
        assert rc == 0 and got == ((0, data.size, 0) if length else (0, 0, 0))
        assert lib.density_b200_kernel_launches() - before == extra


def test_window_past_2_32_in_a_stream_longer_than_2_32(torch_cuda, lib):
    import big_streams as bs
    from test_gpu_beyond_4gib import oracle_size as big_oracle_size, require_device, require_host
    torch = torch_cuda
    n = bs.SIZE["chameleon"]
    require_host(n + 2 * big_oracle_size("chameleon", n) + 2 * GIB)
    data = bs.corpus("chameleon", n)
    stream, _ = bs.oracle_stream("chameleon", data)
    require_device(torch, lib, stream.size + stream.size // 4 + 4 * GIB)
    d = torch.from_numpy(stream).cuda()
    m = stream.size
    del stream
    rc, got, idx, _ = build(torch, lib, d.data_ptr(), m, 256 * MIB)
    assert rc == 0 and got[1:] == (n, 0)
    for first, length in (((1 << 32) + 12345, MIB + 3), ((1 << 32) - 100, 300), (n - 2 * MIB - 1, 4 * MIB)):
        before = lib.density_b200_kernel_launches()
        rc, got, o = indexed(torch, lib, d.data_ptr(), m, idx, first, length, align=3)
        w = min(length, n - first)
        assert rc == 0 and got == (w, n, 0) and (o[:w] == data[first:first + w]).all(), (first, length)
        assert lib.density_b200_kernel_launches() - before == LAUNCHES_INDEXED
    del d, idx
    lib.density_b200_shutdown()
    torch.cuda.empty_cache()


# ---- interface ------------------------------------------------------------------------------------------------------------------
def test_stream_order_and_the_shared_workspace(torch_cuda, lib):
    """an encode, the index build and an indexed decode on one side stream with no host wait between the encode and the build; then
    indexed decodes on one stream and decode_device on another, back to back"""
    import density_b200
    from density_b200 import synth
    torch = torch_cuda
    data = synth.synth_mixed(6 * MIB + 3, device="cuda")
    want = oracle.encode("chameleon", data.cpu().numpy())
    d_enc = torch.zeros(density_b200.Chameleon.safe_encode_buffer_size(data.numel()) + 8, dtype=torch.uint8, device="cuda")
    d_size = torch.zeros(1, dtype=torch.int64, device="cuda")
    d_index = torch.zeros(lib.density_b200_chameleon_index_bytes(want.size, MIB), dtype=torch.uint8, device="cuda")
    res = torch.zeros(3, dtype=torch.int64, device="cuda")
    out = torch.zeros(MIB + 1, dtype=torch.uint8, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    density_b200.encode_device("chameleon", data, d_enc, d_size, stream=side)
    density_b200.index_build_device(d_enc, want.size, MIB, d_index, res, stream=side)
    blen = int(res[0].item())
    density_b200.decode_range_indexed_device(d_enc, want.size, d_index, blen, 3 * MIB - 1, out, res, stream=side)
    side.synchronize()
    assert res.cpu().tolist() == [MIB + 1, data.numel(), 0] and bool((out == data[3 * MIB - 1:4 * MIB]).all())
    ta = synth.synth_text(24 * MIB).numpy()
    a = oracle.encode("chameleon", ta)
    tb = synth.synth_mixed(8 * MIB).numpy()
    b = oracle.encode("chameleon", tb)
    da, pa = upload(torch, a)
    db, pb = upload(torch, b)
    rc, _, ia, _ = build(torch, lib, pa, a.size, 2 * MIB)
    win = torch.zeros(3 * MIB, dtype=torch.uint8, device="cuda")
    dout = torch.zeros(tb.size, dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    h1, h2 = ctypes.c_void_p(s1.cuda_stream), ctypes.c_void_p(s2.cuda_stream)
    for first in (0, 17 * MIB + 5):
        assert lib.density_b200_decode_device(0, pb, b.size, dout.data_ptr(), tb.size, sz.data_ptr(), h2) == 0
        assert lib.density_b200_chameleon_decode_range_indexed_device(pa, a.size, ia.data_ptr(), ia.numel(), first, 3 * MIB, win.data_ptr(),
                                                                      res.data_ptr(), h1) == 0
        assert lib.density_b200_decode_device(0, pb, b.size, dout.data_ptr(), tb.size, sz.data_ptr(), h2) == 0
        s1.synchronize(); s2.synchronize()
        assert res.cpu().tolist() == [3 * MIB, ta.size, 0] and (win.cpu().numpy() == ta[first:first + 3 * MIB]).all()
        assert int(sz.item()) == tb.size and (dout.cpu().numpy() == tb).all()
        dout.zero_(); win.zero_()


def test_synchronous_forms_and_python(torch_cuda, lib):
    import density_b200
    torch = torch_cuda
    C = density_b200.Chameleon
    data = payload("mixed", 700001, seed=9)
    enc = oracle.encode("chameleon", data)
    interval = 64 << 10
    want_index, _ = X.build(enc, interval)
    bound = lib.density_b200_chameleon_index_bytes(enc.size, interval)
    ilen = ctypes.c_uint64(0)
    written = ctypes.c_uint64(0)
    kinds, keep = [], []
    for off in (0, 1):                                                   # pageable, pinned and device buffers, at even and odd addresses
        h = np.zeros(enc.size + 1, np.uint8)
        h[off:off + enc.size] = enc
        pin = torch.empty(enc.size + 1, dtype=torch.uint8).pin_memory()
        pin.numpy()[off:off + enc.size] = enc
        d, p = upload(torch, enc, off)
        keep += [h, pin, d]
        kinds += [("pageable", h.ctypes.data + off), ("pinned", pin.data_ptr() + off), ("device", p)]
    for kind, src in kinds:
        for ikind in ("host", "device"):
            hi = np.full(bound + 3, CANARY, np.uint8)
            di = torch.full((bound + 3,), CANARY, dtype=torch.uint8, device="cuda")
            dst = hi.ctypes.data + 1 if ikind == "host" else di.data_ptr() + 1
            assert lib.density_b200_chameleon_index_build(src, enc.size, interval, dst, bound, ctypes.byref(ilen)) == 0, (kind, ikind)
            got = hi[1:1 + ilen.value] if ikind == "host" else di.cpu().numpy()[1:1 + ilen.value]
            assert got.tobytes() == want_index, (kind, ikind)
            for first, length in ((0, 1000), (123457, 70000), (data.size - 7, 100), (data.size + 3, 10)):
                w = min(length, max(data.size - first, 0))
                ho = np.full(length + 2, CANARY, np.uint8)
                do = torch.full((length + 2,), CANARY, dtype=torch.uint8, device="cuda")
                for dst_out, get in ((ho.ctypes.data + 1, lambda: ho), (do.data_ptr() + 1, lambda: do.cpu().numpy())):
                    written.value = 77
                    assert lib.density_b200_chameleon_decode_range_indexed(src, enc.size, dst, ilen.value, first, dst_out, length,
                                                                           ctypes.byref(written)) == 0, (kind, ikind, first)
                    o = get()
                    assert written.value == w and (o[1:1 + w] == data[first:first + w]).all(), (kind, ikind, first)
                    assert o[0] == CANARY and (o[1 + w:] == CANARY).all()
    idx = C.build_index(enc, interval=interval)
    assert isinstance(idx, bytes) and idx == want_index
    didx = C.build_index(torch.from_numpy(enc).cuda(), interval=interval)
    assert didx.is_cuda and didx.cpu().numpy().tobytes() == want_index
    out = np.zeros(4000, np.uint8)
    assert C.decode_range(enc, 5000, out, index=idx) == 4000 and (out == data[5000:9000]).all()
    t = torch.zeros(4000, dtype=torch.uint8, device="cuda")
    assert C.decode_range(torch.from_numpy(enc).cuda(), data.size - 1000, t, index=didx) == 1000
    assert (t[:1000].cpu().numpy() == data[-1000:]).all()
    assert C.decode_range(enc, 5000, out) == 4000                        # without an index, as before
    with pytest.raises(density_b200.DecodeError):
        C.build_index(enc[:7])
    with pytest.raises(ValueError):
        C.build_index(enc, interval=1000)
    with pytest.raises(density_b200.DensityB200Error):
        C.decode_range(enc, 0, out, index=idx[:-1])
