"""The Chameleon range decode on an H100 (pytest -m gpu): density_b200_chameleon_decode_range_device and _range, held window by window to
the oracle slice oracle.decode(...)[first:first + w], w = min(first + len, S) - first, with guard bytes on both sides of d_out (placed at
odd addresses) and around d_result, and to density_b200_decoded_size for S and the verdict. Encoded text, synth_mixed and noise; windows
at +-1 of block, tile, decoder-run and boundary-row chunk and group edges; streams no encoder writes and their truncations; the edge
windows; a window past 2^32 in a stream longer than 2^32 bytes; and the interface: launch counts, refused arguments, stream order, the
shared workspace, the synchronous variant, Python and host pointers. tests/test_decode_range_cpu.py checks the model behind it."""
import ctypes

import numpy as np
import pytest

import oracle
import planted
import synth_streams as ss
from conftest import payload, splitmix_bytes
from decoded_size_witness import MALFORMED, oracle_cap, oracle_size

pytestmark = pytest.mark.gpu
MIB, GIB = 1 << 20, 1 << 30
BS, CH, GROUP_BYTES = 256, 16384, 64 * 16384       # block; decode_bounds.cuh ChamT chunk and group of 64 chunks
TILE = 64 * BS                                     # chameleon_decode.cu: a tile is 64 blocks of output
RES_CANARY = 0x5A5A5A5A5A5A5A5A
CANARY = 0xA5
PAD = 64
LAUNCHES_LOCATE, LAUNCHES_FIRST_BLOCK, LAUNCHES_LATER = 4, 13, 26


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


def _cur(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def upload(torch, stream, offset=0):
    s = np.asarray(stream, np.uint8)
    buf = torch.zeros(s.size + offset + 2, dtype=torch.uint8, device="cuda")
    if s.size:
        buf[offset:offset + s.size] = torch.from_numpy(s.copy()).cuda()
    return buf, buf.data_ptr() + offset


def window(torch, lib, ptr, n, first, length, align=1, stream=None, room=None):
    """one range decode into d_out at an address `align` bytes past a 64-byte boundary, guards on both sides; `room`: the bytes
    allocated behind d_out when len is larger than any w -> (rc, (w, S, verdict), the len (room) bytes of d_out)"""
    room = length if room is None else room
    out = torch.full((room + 2 * PAD,), CANARY, dtype=torch.uint8, device="cuda")
    res = torch.full((5,), RES_CANARY, dtype=torch.int64, device="cuda")
    s = _cur(torch) if stream is None else ctypes.c_void_p(stream.cuda_stream)
    rc = lib.density_b200_chameleon_decode_range_device(ptr, n, first, length, out.data_ptr() + PAD + align, res.data_ptr() + 8, s)
    torch.cuda.synchronize()
    r = res.cpu().numpy().view(np.uint64)
    assert int(r[0]) == RES_CANARY and int(r[4]) == RES_CANARY, "the call wrote outside its 24 result bytes"
    o = out.cpu().numpy()
    got = tuple(int(x) for x in r[1:4])
    w = got[0]
    assert (o[:PAD + align] == CANARY).all(), "wrote in front of d_out"
    assert (o[PAD + align + w:] == CANARY).all(), f"wrote behind d_out + w (w = {w})"
    return rc, got, o[PAD + align:PAD + align + room]


def decoded_size(torch, lib, ptr, n):
    res = torch.zeros(2, dtype=torch.int64, device="cuda")
    assert lib.density_b200_decoded_size_device(0, ptr, n, res.data_ptr(), _cur(torch)) == 0
    torch.cuda.synchronize()
    return tuple(int(x) for x in res.cpu().numpy().view(np.uint64))


class Case:
    """a stream on the device and its witness: D, the oracle's decode (or the encoder's input), S and the verdict"""

    def __init__(self, torch, lib, stream, D=None):
        self.torch, self.lib = torch, lib
        self.s = np.asarray(stream, np.uint8)
        self.size, self.verdict = oracle_size("chameleon", self.s) if D is None else (D.size, 0)
        if D is None:
            D = oracle.decode("chameleon", self.s, oracle_cap(self.s.size)) if self.s.size and not self.verdict else np.zeros(0, np.uint8)
        self.D = D
        self.buf, self.ptr = upload(torch, self.s)

    def check(self, first, length, what="", align=1, room=None):
        rc, got, o = window(self.torch, self.lib, self.ptr, self.s.size, first, length, align, room=room)
        want = self.D[first:first + length] if not self.verdict else self.D[:0]
        wantS = (0, MALFORMED) if self.verdict else (self.size, 0)
        assert rc == 0, f"{what}: rc {rc}"
        assert got == (want.size,) + wantS, f"{what} [{first}, +{length}): got {got}, want {(want.size,) + wantS}"
        assert (o[:want.size] == want).all(), f"{what} [{first}, +{length}): window bytes differ from the oracle slice"
        return got


def edges(points, S, lens=(1, 3, 256, 4099)):
    for p in sorted(set(points)):
        for f in (p - 1, p, p + 1):
            if 0 <= f < S:
                for L in lens:
                    yield f, L
                yield max(f - 700, 0), f - max(f - 700, 0) + 1 + (f % 3)     # a window whose end is at f (+0..2)


# ---- encoded corpora ------------------------------------------------------------------------------------------------------------
def corpus(kind, n):
    from density_b200 import synth
    if kind == "text":
        return synth.synth_text(n).numpy()
    if kind == "mixed":
        return synth.synth_mixed(n).numpy()
    return splitmix_bytes(n, 11)


@pytest.mark.parametrize("kind", ["text", "mixed", "noise"])
def test_encoded_corpora(torch_cuda, lib, kind):
    n = 12 * MIB + 12345
    data = corpus(kind, n)
    enc, copied = oracle.encode("chameleon", data, return_copied=True)
    assert bool(copied) == (kind != "text")
    c = Case(torch_cuda, lib, enc, D=data)
    for k, (first, length) in enumerate([(0, MIB), (n // 2 - 77, MIB), (n - MIB, MIB), (n - MIB + 5, 2 * MIB), (n - 3, 3), (n - 1, 1),
                                         (n, 5), (n + 1000, 5), (300, 1), (5 * MIB + 129, 40000)]):
        c.check(first, length, kind, align=k % 4)


def test_seams(torch_cuda, lib):
    """first or end at +-1 of block, tile, decoder-run, boundary-row chunk and group edges, on a planted quiet corpus and on copy-mode
    data"""
    for name in ("cham5", "copy3"):
        data, _ = planted.corpus(name)
        enc = oracle.encode("chameleon", data)
        c = Case(torch_cuda, lib, enc, D=data)
        w = ss.walk("chameleon", enc)
        starts, S = w["starts"], data.size
        pts = [BS * k for k in (1, 2, 63, 64, 65, 1000)] + [TILE * k for k in (1, 2, 17)]
        pts += [BS * b for b in ss.seam_blocks("chameleon", enc.size, S, w["main_blocks"])[:6]]      # decode_device's run seams
        for edge in (CH, 2 * CH, 7 * CH, GROUP_BYTES, 2 * GROUP_BYTES):     # the block that holds a stream-chunk or group edge
            b = int(np.searchsorted(starts, edge, side="right")) - 1
            if 0 <= b < len(starts):
                pts += [b * BS, (b + 1) * BS]
        pts += [BS * w["main_blocks"], S - 3]
        for first, length in edges(pts, S):
            c.check(first, length, name, align=first % 4)


# ---- streams no encoder writes --------------------------------------------------------------------------------------------------
PLANS = {
    "cham_bad": ({"nbytes": 300000, "tail": (100, "map0")}, 26),
    "cham1": ({"nbytes": MIB, "tail": (16, "plain_end")}, 25),
    "cham4_copy": ({"nbytes": 4 * MIB, "quiet": False, "copy_every": 301, "cuts": (0.33, 0.66), "tail": (60, "raw2")}, 23),
    "cham_prot": ({"nbytes": 2 * MIB, "quiet": False, "prot_states": True, "tail": (138, "raw2")}, 24),
}


@pytest.mark.parametrize("name", list(PLANS))
def test_synthesized_streams(torch_cuda, lib, name):
    plan, seed = PLANS[name]
    s, m = ss.build("chameleon", plan, seed)
    c = Case(torch_cuda, lib, s)
    assert (c.size, c.verdict) == ((0, MALFORMED) if name.endswith("_bad") else (m["decoded_size"], 0))
    assert decoded_size(torch_cuda, lib, c.ptr, s.size) == (c.size, c.verdict)
    S = max(c.size, 300000)
    for first, length in edges([0, BS * 301, BS * 302, S // 3, S // 2 + 7, S - 300, S - 2], S, lens=(1, 257, 70000)):
        c.check(first, length, name, align=length % 4)


def test_truncations(torch_cuda, lib):
    """the last 300 byte offsets of a synthesized stream with copy-mode blocks and of an encoded one: S and the verdict are
    decoded_size's whatever the window"""
    torch = torch_cuda
    s, _ = ss.build("chameleon", {"nbytes": 60000, "quiet": False, "copy_every": 23, "plant": False, "tail": (60, "raw2")}, 7)
    enc = oracle.encode("chameleon", payload("mixed", 50000, seed=2))
    verdicts = set()
    for stream in (s, enc):
        full = Case(torch, lib, stream)
        for k in range(stream.size - 300, stream.size + 1):
            t = stream[:k]
            size, verdict = oracle_size("chameleon", t)
            for first, length in ((0, 1 << 40), (size // 2, 700), (max(size - 5, 0), 9)):
                rc, got, o = window(torch, lib, full.ptr, k, first, length, align=k % 4, room=min(length, size + 16))
                assert rc == 0 and got[1:] == decoded_size(torch, lib, full.ptr, k), f"truncated at {k}"
                assert got[1:] == (size, verdict)
                if verdict == 0 and got[0]:
                    ref = oracle.decode("chameleon", t, size)
                    assert (o[:got[0]] == ref[first:first + got[0]]).all(), f"truncated at {k}: [{first}, +{length})"
            verdicts.add(verdict)
    assert verdicts == {0, MALFORMED}


# ---- edge windows -----------------------------------------------------------------------------------------------------------------
def test_edge_windows_and_launch_counts(torch_cuda, lib):
    torch = torch_cuda
    data = corpus("mixed", 3 * MIB + 5)
    enc = oracle.encode("chameleon", data)
    c = Case(torch, lib, enc, D=data)
    S = data.size
    cases = [(0, 1, LAUNCHES_FIRST_BLOCK), (0, S, LAUNCHES_FIRST_BLOCK), (255, 2, LAUNCHES_FIRST_BLOCK), (256, 1, LAUNCHES_LATER),
             (S - 10, 10, LAUNCHES_LATER), (S - 10, 1 << 40, LAUNCHES_LATER), (S - 1, 2, LAUNCHES_LATER), (S, 1, 0), (S + 7, 9, 0),
             (~0 & ((1 << 64) - 1), 1, 0), (MIB, (1 << 64) - MIB, LAUNCHES_LATER)]
    c.check(0, 1)                                                                         # workspace allocated
    for first, length, extra in cases:
        before = lib.density_b200_kernel_launches()
        c.check(first, length, f"edge {first}", room=min(length, S + 16))
        assert lib.density_b200_kernel_launches() - before == LAUNCHES_LOCATE + extra, (first, length)
    for n, length in ((0, 5), (enc.size, 0), (0, 0)):                                      # no kernel, {0, 0, 0}
        before = lib.density_b200_kernel_launches()
        rc, got, _ = window(torch, lib, c.ptr if n else 0, n, 5, length)
        assert rc == 0 and got == (0, 0, 0) and lib.density_b200_kernel_launches() == before
    bad = Case(torch, lib, enc[:7])                                                       # a signature cut short: the locate step only
    before = lib.density_b200_kernel_launches()
    bad.check(0, 100, "malformed")
    assert lib.density_b200_kernel_launches() - before == LAUNCHES_LOCATE


def test_refused_arguments_enqueue_nothing(torch_cuda, lib):
    torch = torch_cuda
    enc = oracle.encode("chameleon", payload("text", 200000))
    buf, ptr = upload(torch, enc)
    out = torch.full((4096,), CANARY, dtype=torch.uint8, device="cuda")
    res = torch.full((4,), RES_CANARY, dtype=torch.int64, device="cuda")
    r = res.data_ptr() + 8
    before = lib.density_b200_kernel_launches()
    cases = [(None, enc.size, 0, 10, out.data_ptr(), r), (ptr, enc.size, 0, 10, None, r), (ptr, enc.size, 0, 10, out.data_ptr(), None),
             (ptr + 1, enc.size - 1, 0, 10, out.data_ptr(), r), (ptr, enc.size, 0, 10, out.data_ptr(), r + 4)]
    for p, n, first, length, o, rr in cases:
        assert lib.density_b200_chameleon_decode_range_device(p, n, first, length, o, rr, _cur(torch)) == 4, (p, n, o, rr)
    torch.cuda.synchronize()
    assert lib.density_b200_kernel_launches() == before
    assert (res.cpu().numpy().view(np.uint64) == RES_CANARY).all() and bool((out == CANARY).all())


# ---- beyond 32 bits ---------------------------------------------------------------------------------------------------------------
def test_window_past_2_32_in_a_stream_longer_than_2_32(torch_cuda, lib):
    import big_streams as bs
    from test_gpu_beyond_4gib import oracle_size as big_oracle_size, require_device, require_host
    torch = torch_cuda
    n = bs.SIZE["chameleon"]
    require_host(n + 2 * big_oracle_size("chameleon", n) + 2 * GIB)
    data = bs.corpus("chameleon", n)
    stream, _ = bs.oracle_stream("chameleon", data)
    assert stream.size > bs.STREAM_MIN
    require_device(torch, lib, stream.size + stream.size // 4 + 4 * GIB)
    d = torch.from_numpy(stream).cuda()
    m = stream.size
    del stream
    for first, length in (((1 << 32) + 12345, MIB + 3), (n - 2 * MIB - 1, 4 * MIB), ((1 << 32) - 100, 300)):
        rc, got, o = window(torch, lib, d.data_ptr(), m, first, length, align=3)
        w = min(length, n - first)
        assert rc == 0 and got == (w, n, 0), (first, length, got)
        assert (o[:w] == data[first:first + w]).all(), f"window at {first} differs"
    del d
    lib.density_b200_shutdown()
    torch.cuda.empty_cache()


# ---- interface --------------------------------------------------------------------------------------------------------------------
def test_stream_ordered_behind_an_encode(torch_cuda, lib):
    """the encode on a side stream and the range decode behind it on the same stream, with no host synchronisation in between"""
    import density_b200
    from density_b200 import synth
    torch = torch_cuda
    data = synth.synth_mixed(6 * MIB + 3, device="cuda")
    want = oracle.encode("chameleon", data.cpu().numpy())
    d_enc = torch.zeros(density_b200.Chameleon.safe_encode_buffer_size(data.numel()) + 8, dtype=torch.uint8, device="cuda")
    d_size = torch.zeros(1, dtype=torch.int64, device="cuda")
    out = torch.zeros(MIB + 1, dtype=torch.uint8, device="cuda")
    res = torch.zeros(3, dtype=torch.int64, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    density_b200.encode_device("chameleon", data, d_enc, d_size, stream=side)
    density_b200.decode_range_device(d_enc, want.size, 3 * MIB - 1, out, res, stream=side)
    side.synchronize()
    assert int(d_size.item()) == want.size
    assert res.cpu().tolist() == [MIB + 1, data.numel(), 0]
    assert bool((out == data[3 * MIB - 1:4 * MIB]).all())


def test_range_decode_and_decode_share_the_workspace(torch_cuda, lib):
    """range decodes on one stream and decode_device on another, enqueued back to back: every result is right"""
    from density_b200 import synth
    torch = torch_cuda
    ta = synth.synth_text(24 * MIB).numpy()
    a = oracle.encode("chameleon", ta)
    tb = synth.synth_mixed(8 * MIB).numpy()
    b = oracle.encode("chameleon", tb)
    da, pa = upload(torch, a)
    db, pb = upload(torch, b)
    res = torch.zeros(3, dtype=torch.int64, device="cuda")
    win = torch.zeros(3 * MIB, dtype=torch.uint8, device="cuda")
    out = torch.zeros(tb.size, dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    h1, h2 = ctypes.c_void_p(s1.cuda_stream), ctypes.c_void_p(s2.cuda_stream)
    for first in (0, 17 * MIB + 5):
        assert lib.density_b200_decode_device(0, pb, b.size, out.data_ptr(), tb.size, sz.data_ptr(), h2) == 0
        assert lib.density_b200_chameleon_decode_range_device(pa, a.size, first, 3 * MIB, win.data_ptr(), res.data_ptr(), h1) == 0
        assert lib.density_b200_decode_device(0, pb, b.size, out.data_ptr(), tb.size, sz.data_ptr(), h2) == 0
        s1.synchronize(); s2.synchronize()
        assert res.cpu().tolist() == [3 * MIB, ta.size, 0]
        assert (win.cpu().numpy() == ta[first:first + 3 * MIB]).all()
        assert int(sz.item()) == tb.size and (out.cpu().numpy() == tb).all()
        out.zero_(); win.zero_()


def test_synchronous_variant_python_and_host_pointers(torch_cuda, lib):
    import density_b200
    torch = torch_cuda
    C = density_b200.Chameleon
    data = payload("mixed", 300001, seed=9)
    enc = oracle.encode("chameleon", data)
    written = ctypes.c_uint64(0)
    for off in (0, 1):                                                    # host and device buffers, at even and odd addresses
        h = np.zeros(enc.size + 1, np.uint8)
        h[off:off + enc.size] = enc
        d, p = upload(torch, enc, off)
        for src in (h.ctypes.data + off, p):
            for first, length in ((0, 1000), (123457, 5000), (data.size - 7, 100), (data.size + 3, 10)):
                ho = np.full(length + 2, CANARY, np.uint8)
                do = torch.full((length + 2,), CANARY, dtype=torch.uint8, device="cuda")
                w = min(length, max(data.size - first, 0))
                for dst, get in ((ho.ctypes.data + 1, lambda: ho), (do.data_ptr() + 1, lambda: do.cpu().numpy())):
                    written.value = 77
                    assert lib.density_b200_chameleon_decode_range(src, enc.size, first, dst, length, ctypes.byref(written)) == 0
                    o = get()
                    assert written.value == w and (o[1:1 + w] == data[first:first + w]).all()
                    assert o[0] == CANARY and (o[1 + w:] == CANARY).all()
    out = np.zeros(4000, np.uint8)
    assert C.decode_range(enc, 5000, out) == 4000 and (out == data[5000:9000]).all()
    t = torch.zeros(4000, dtype=torch.uint8, device="cuda")
    assert C.decode_range(torch.from_numpy(enc).cuda(), data.size - 1000, t) == 1000
    assert (t[:1000].cpu().numpy() == data[-1000:]).all()
    assert C.decode_range(enc, data.size, out) == 0
    assert C.decode_range(b"", 0, out) == 0
    with pytest.raises(density_b200.DecodeError):
        C.decode_range(enc[:7], 0, out)                                   # a signature cut short
    assert lib.density_b200_chameleon_decode_range(enc.ctypes.data, enc.size, 0, out.ctypes.data, 10, None) == 4
