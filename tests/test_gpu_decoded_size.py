"""The decoded-size query on an H100 (pytest -m gpu): density_b200_decoded_size_device and density_b200_decoded_size for all three
algorithms, held case by case to the witness of tests/decoded_size_witness.py (the oracle's decode) and to decode itself: a size s means
decode_device with cap = s writes s bytes equal to the oracle's (a canary behind them holds) and with cap = s - 1 writes 0; a malformed
verdict means decode writes 0 at any capacity. Encoded corpora and the tail sweep, streams no encoder writes and their truncations,
copy-mode streams, sizes past 2^32, and the interface: launch counts, the 16 bytes written, refused arguments, stream order and the
shared workspace."""
import ctypes

import numpy as np
import pytest

import oracle
import synth_streams as ss
from conftest import ALGS, payload, splitmix_bytes
from decoded_size_witness import MALFORMED, oracle_cap, oracle_size
from lion_streams import TAIL_SWEEP

pytestmark = pytest.mark.gpu
ALG_ID = {"chameleon": 0, "cheetah": 1, "lion": 2}
MIB, GIB = 1 << 20, 1 << 30
RES_CANARY = 0x5A5A5A5A5A5A5A5A
CANARY = 0xA5
PAD = 64


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
    """a device copy of a host stream at `offset` bytes into its allocation -> (buffer, address)"""
    s = np.asarray(stream, np.uint8)
    buf = torch.zeros(s.size + offset + 2, dtype=torch.uint8, device="cuda")
    if s.size:
        buf[offset:offset + s.size] = torch.from_numpy(s.copy()).cuda()
    return buf, buf.data_ptr() + offset


def query(torch, lib, alg, d_in, n, stream=None):
    """-> (rc, (size, verdict)); checks that exactly the 16 bytes between two canary words were written"""
    res = torch.full((4,), RES_CANARY, dtype=torch.int64, device="cuda")
    s = _cur(torch) if stream is None else ctypes.c_void_p(stream.cuda_stream)
    rc = lib.density_b200_decoded_size_device(ALG_ID[alg], d_in, n, res.data_ptr() + 8, s)
    torch.cuda.synchronize()
    r = res.cpu().numpy().view(np.uint64)
    assert int(r[0]) == RES_CANARY and int(r[3]) == RES_CANARY, f"{alg}: the query wrote outside its 16 bytes"
    return rc, (int(r[1]), int(r[2]))


def query_host(torch, lib, alg, stream):
    buf, ptr = upload(torch, stream)        # buf keeps the allocation alive through the query
    rc, got = query(torch, lib, alg, ptr, np.asarray(stream).size)
    assert rc == 0
    return got


def decode(torch, lib, alg, d_in, n, cap):
    """decode_device into exactly `cap` bytes and a canary -> (size, output)"""
    out = torch.full((cap + PAD,), CANARY, dtype=torch.uint8, device="cuda")
    sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    rc = lib.density_b200_decode_device(ALG_ID[alg], d_in, n, out.data_ptr(), cap, sz.data_ptr(), _cur(torch))
    torch.cuda.synchronize()
    assert rc == 0
    assert bool((out[cap:] == CANARY).all()), f"{alg}: decode wrote past cap {cap}"
    return int(sz.item()), out[:cap]


def check_contract(torch, lib, alg, stream, what, want=None):
    """the query equals the witness, and decode agrees with the query at cap = s and s - 1 (or at any capacity when malformed)"""
    s = np.asarray(stream, np.uint8)
    want = oracle_size(alg, s) if want is None else want
    buf, ptr = upload(torch, s)
    rc, got = query(torch, lib, alg, ptr, s.size)
    assert rc == 0 and got == want, f"{alg} {what}: query {got} (rc {rc}), witness {want}"
    size, verdict = got
    if verdict == MALFORMED:
        assert decode(torch, lib, alg, ptr, s.size, oracle_cap(s.size))[0] == 0, f"{alg} {what}: decoded a malformed stream"
        return got
    if s.size == 0:
        return got
    m, out = decode(torch, lib, alg, ptr, s.size, size)
    assert m == size, f"{alg} {what}: decode at cap = {size} wrote {m}"
    if size:
        ref = oracle.decode(alg, s, size)
        assert ref.size == size and (out.cpu().numpy() == ref).all(), f"{alg} {what}: decoded bytes differ from the oracle"
        assert decode(torch, lib, alg, ptr, s.size, size - 1)[0] == 0, f"{alg} {what}: decode at cap = s - 1 did not fail"
    return got


# ---- encoded corpora --------------------------------------------------------------------------------------------------------------
def corpus(kind, n):
    from density_b200 import synth
    if kind == "text":
        return synth.synth_text(n).numpy()
    if kind == "mixed":
        return synth.synth_mixed(n).numpy()
    if kind == "dickens":
        return payload("text", n, seed=3)
    if kind == "zeros":
        return np.zeros(n, np.uint8)
    return splitmix_bytes(n, 11)


@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("kind", ["text", "mixed", "dickens", "zeros", "noise"])
def test_encoded_corpora(torch_cuda, lib, alg, kind):
    n = (6 * MIB if alg != "lion" else 2 * MIB) + 12345
    data = corpus(kind, n)
    enc, copied = oracle.encode(alg, data, return_copied=True)
    if kind in ("noise", "mixed"):
        assert copied, "copy-mode blocks expected"
    w = ss.walk(alg, enc)
    if kind == "noise":
        assert any(w["copy"]), "noise: the main loop should hold copy-mode blocks"
    check_contract(torch_cuda, lib, alg, enc, kind, want=(n, 0))


@pytest.mark.parametrize("alg", ALGS)
def test_cheetah_cold_start_and_tail_sweep(torch_cuda, lib, alg):
    """every length of TAIL_SWEEP behind a few blocks, five kinds: the size is the input length (Cheetah text starts in copy mode)"""
    for kind in ("text", "random", "zeros", "low", "mixed"):
        for L in TAIL_SWEEP:
            data = payload(kind, 7 * ss.BS[alg] + L, seed=L)
            enc = oracle.encode(alg, data)
            assert query_host(torch_cuda, lib, alg, enc) == (data.size, 0), f"{alg} {kind} {L}"
    text = corpus("text", MIB)
    enc, copied = oracle.encode(alg, text, return_copied=True)
    if alg == "cheetah":
        assert copied and ss.walk(alg, enc)["copy"][:4] != [False] * 4
    check_contract(torch_cuda, lib, alg, enc, "text 1 MiB", want=(text.size, 0))


@pytest.mark.parametrize("alg", ALGS)
def test_empty_stream(torch_cuda, lib, alg):
    before = lib.density_b200_kernel_launches()
    rc, got = query(torch_cuda, lib, alg, 0, 0)
    assert rc == 0 and got == (0, 0)
    buf, ptr = upload(torch_cuda, np.zeros(0, np.uint8))
    rc, got = query(torch_cuda, lib, alg, ptr, 0)
    assert rc == 0 and got == (0, 0)
    assert lib.density_b200_kernel_launches() == before, "n == 0 launches no kernel"


# ---- streams no encoder writes ------------------------------------------------------------------------------------------------
PLANS = {
    "cham_bad": ("chameleon", {"nbytes": 300000, "tail": (100, "map0")}, 26),
    "cham1": ("chameleon", {"nbytes": MIB, "tail": (16, "plain_end")}, 25),
    "cham4_copy": ("chameleon", {"nbytes": 4 * MIB, "quiet": False, "copy_every": 301, "cuts": (0.33, 0.66), "tail": (60, "raw2")}, 23),
    "cham_prot": ("chameleon", {"nbytes": 2 * MIB, "quiet": False, "prot_states": True, "tail": (138, "raw2")}, 24),
    "chee_bad": ("cheetah", {"nbytes": 300000, "p_pred": 0.5, "tail": (9, "map1")}, 38),
    "chee2_p99": ("cheetah", {"nbytes": 2 * MIB, "p_pred": 0.99, "tail": (100, "raw2")}, 35),
    "chee4_copy": ("cheetah", {"nbytes": 4 * MIB, "p_pred": 0.3, "quiet": False, "copy_every": 211, "cuts": (0.5,), "tail": (91, "raw3")}, 36),
    "chee_prot": ("cheetah", {"nbytes": 3 * MIB, "p_pred": 0.3, "quiet": False, "prot_states": True, "tail": (20, "clean")}, 37),
    "lion3_p5": ("lion", {"nbytes": 3 * MIB, "p_pred": 0.5, "cuts": tuple(k / 10 for k in range(1, 10)), "odd": True, "tail": (20, "raw2")}, 63),
    "lion2_p99": ("lion", {"nbytes": 2 * MIB, "p_pred": 0.99, "cuts": (0.5,), "odd": True, "tail": (13, "raw1")}, 65),
    "lion3_copy": ("lion", {"nbytes": 3 * MIB, "p_pred": 0.3, "quiet": False, "copy_every": 97, "cuts": (0.33, 0.66), "tail": (31, "raw3")}, 66),
    "lion_prot": ("lion", {"nbytes": 2 * MIB, "p_pred": 0.3, "quiet": False, "prot_states": True, "cuts": (0.2, 0.4, 0.6, 0.8),
                           "tail": (22, "clean")}, 67),
    "lion_bad": ("lion", {"nbytes": 200000, "p_pred": 0.5, "tail": (9, "map1")}, 68),
}


@pytest.mark.parametrize("name", list(PLANS))
def test_synthesized_streams(torch_cuda, lib, name):
    alg, plan, seed = PLANS[name]
    s, m = ss.build(alg, plan, seed)
    got = check_contract(torch_cuda, lib, alg, s, name)
    assert got == ((0, MALFORMED) if name.endswith("_bad") else (m["decoded_size"], 0))


@pytest.mark.parametrize("alg", ALGS)
def test_truncations(torch_cuda, lib, alg):
    """the last 300 byte offsets of a short synthesized stream with copy-mode blocks, and of an encoded one"""
    tail = (40, dict(ss.tail_lengths(alg))[40])
    s, _ = ss.build(alg, {"nbytes": 60000, "quiet": False, "copy_every": 23, "plant": False, "tail": tail}, 7)
    enc = oracle.encode(alg, payload("mixed", 50000, seed=2))
    verdicts = set()
    for stream in (s, enc):
        for k in range(stream.size - 300, stream.size + 1):
            verdicts.add(check_contract(torch_cuda, lib, alg, stream[:k], f"truncated at {k}")[1])
    assert verdicts == {0, MALFORMED}


# ---- beyond 32 bits ---------------------------------------------------------------------------------------------------------------
def test_cheetah_size_past_2_32(torch_cuda, lib):
    """Cheetah zeros: every block is an 8-byte signature of predicted quads (0xFF bytes) that decodes to 128 bytes. About 300 MiB of
    them decode to more than 2^32 bytes, reported exactly; no output buffer is allocated."""
    torch = torch_cuda
    small = oracle.encode("cheetah", np.zeros(128 * 9, np.uint8))
    assert (small == 0xFF).all() and small.size == 8 * 9
    n = 300 * MIB + 8 * 5
    d = torch.full((n,), 0xFF, dtype=torch.uint8, device="cuda")
    rc, got = query(torch, lib, "cheetah", d.data_ptr(), n)
    assert rc == 0 and got == (16 * n, 0) and got[0] > 1 << 32
    rc, got = query(torch, lib, "cheetah", d.data_ptr(), n - 3)          # a signature cut short: malformed
    assert rc == 0 and got == (0, MALFORMED)
    del d


def test_stream_longer_than_2_32(torch_cuda, lib):
    """the Chameleon corpus of tests/big_streams.py (5.5 GiB, a stream past 2^32 bytes), as the beyond-4 GiB decode tests use it"""
    import big_streams as bs
    from test_gpu_beyond_4gib import oracle_size as big_oracle_size, require_device, require_host
    torch = torch_cuda
    n = bs.SIZE["chameleon"]
    require_host(n + 2 * big_oracle_size("chameleon", n) + 2 * GIB)
    data = bs.corpus("chameleon", n)
    stream, _ = bs.oracle_stream("chameleon", data)
    del data
    assert stream.size > bs.STREAM_MIN
    require_device(torch, lib, stream.size + stream.size // 8 + 2 * GIB)
    d = torch.from_numpy(stream).cuda()
    m = stream.size
    del stream
    rc, got = query(torch, lib, "chameleon", d.data_ptr(), m)
    assert rc == 0 and got == (n, 0)
    del d
    lib.density_b200_shutdown()
    torch.cuda.empty_cache()


# ---- interface --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", ALGS)
def test_launch_count_and_refused_arguments(torch_cuda, lib, alg):
    torch = torch_cuda
    enc = oracle.encode(alg, payload("text", 200000))
    buf, ptr = upload(torch, enc)
    query(torch, lib, alg, ptr, enc.size)                                 # workspace allocated
    for n in (1, 5, enc.size):
        before = lib.density_b200_kernel_launches()
        assert query(torch, lib, alg, ptr, n)[0] == 0
        assert lib.density_b200_kernel_launches() - before == 4
    res = torch.full((4,), RES_CANARY, dtype=torch.int64, device="cuda")
    before = lib.density_b200_kernel_launches()
    cases = [(7, ptr, enc.size, res.data_ptr() + 8), (-1, ptr, enc.size, res.data_ptr() + 8),
             (ALG_ID[alg], ptr, enc.size, None), (ALG_ID[alg], None, enc.size, res.data_ptr() + 8),
             (ALG_ID[alg], ptr + 1, enc.size - 1, res.data_ptr() + 8), (ALG_ID[alg], ptr, enc.size, res.data_ptr() + 12)]
    for a, p, n, r in cases:
        assert lib.density_b200_decoded_size_device(a, p, n, r, _cur(torch)) == 4, (a, p, n, r)     # DENSITY_B200_EARG
    torch.cuda.synchronize()
    assert lib.density_b200_kernel_launches() == before
    assert (res.cpu().numpy().view(np.uint64) == RES_CANARY).all(), "a refused call wrote its result"


@pytest.mark.parametrize("alg", ALGS)
def test_stream_ordered_behind_an_encode(torch_cuda, lib, alg):
    """the encode and the query on a side stream, back to back with no host synchronisation: the query sees the encoded stream"""
    import density_b200
    from density_b200 import synth
    torch = torch_cuda
    data = synth.synth_text(4 * MIB + 3, device="cuda")
    want = oracle.encode(alg, data.cpu().numpy())
    d_enc = torch.zeros(density_b200.CODECS[alg].safe_encode_buffer_size(data.numel()) + 8, dtype=torch.uint8, device="cuda")
    d_size = torch.zeros(1, dtype=torch.int64, device="cuda")
    res = torch.zeros(2, dtype=torch.int64, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    density_b200.encode_device(alg, data, d_enc, d_size, stream=side)
    density_b200.decoded_size_device(alg, d_enc, want.size, res, stream=side)
    side.synchronize()
    assert int(d_size.item()) == want.size
    assert res.cpu().tolist() == [data.numel(), 0]


def test_query_and_decode_share_the_workspace(torch_cuda, lib):
    """a query on one stream and a decode on another, enqueued back to back: both results are right"""
    from density_b200 import synth
    torch = torch_cuda
    a = oracle.encode("chameleon", synth.synth_text(24 * MIB).numpy())
    text = synth.synth_mixed(8 * MIB).numpy()
    b = oracle.encode("cheetah", text)
    da, pa = upload(torch, a)
    db, pb = upload(torch, b)
    res_a = torch.zeros(2, dtype=torch.int64, device="cuda")
    res_b = torch.zeros(2, dtype=torch.int64, device="cuda")
    out = torch.zeros(text.size, dtype=torch.uint8, device="cuda")
    sz = torch.zeros(1, dtype=torch.int64, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    h1, h2 = ctypes.c_void_p(s1.cuda_stream), ctypes.c_void_p(s2.cuda_stream)
    for _ in range(2):
        assert lib.density_b200_decoded_size_device(0, pa, a.size, res_a.data_ptr(), h1) == 0
        assert lib.density_b200_decode_device(1, pb, b.size, out.data_ptr(), text.size, sz.data_ptr(), h2) == 0
        assert lib.density_b200_decoded_size_device(1, pb, b.size, res_b.data_ptr(), h2) == 0
        assert lib.density_b200_decoded_size_device(0, pa, a.size - 5, res_a.data_ptr(), h1) == 0
        s1.synchronize(); s2.synchronize()
        assert res_a.cpu().tolist() == list(oracle_size("chameleon", a[:-5]))
        assert res_b.cpu().tolist() == [text.size, 0]
        assert int(sz.item()) == text.size and (out.cpu().numpy() == text).all()
        res_a.zero_(); res_b.zero_(); out.zero_()


@pytest.mark.parametrize("alg", ALGS)
def test_synchronous_variant_and_python(torch_cuda, lib, alg):
    import density_b200
    torch = torch_cuda
    C = density_b200.CODECS[alg]
    data = payload("mixed", 300001, seed=9)
    enc = oracle.encode(alg, data)
    out = ctypes.c_uint64(0)
    for off in (0, 1):                                                    # host and device buffers, at even and odd addresses
        h = np.zeros(enc.size + 1, np.uint8)
        h[off:off + enc.size] = enc
        assert lib.density_b200_decoded_size(ALG_ID[alg], h.ctypes.data + off, enc.size, ctypes.byref(out)) == 0 and out.value == data.size
        d, p = upload(torch, enc, off)
        out.value = 0
        assert lib.density_b200_decoded_size(ALG_ID[alg], p, enc.size, ctypes.byref(out)) == 0 and out.value == data.size
    assert C.decoded_size(enc) == data.size
    assert C.decoded_size(torch.from_numpy(enc).cuda()) == data.size
    assert C.decode_bytes(enc) == data.tobytes()
    assert C.decode_bytes(enc, data.size) == data.tobytes()
    assert C.decode_bytes(b"") == b""
    bad = enc[:ss.SIG[alg] - 1]                                           # a signature cut short
    assert lib.density_b200_decoded_size(ALG_ID[alg], bad.ctypes.data, bad.size, ctypes.byref(out)) == MALFORMED
    with pytest.raises(density_b200.DecodeError):
        C.decoded_size(bad)
    with pytest.raises(density_b200.DecodeError):
        C.decode_bytes(bad)
    assert lib.density_b200_decoded_size(9, enc.ctypes.data, enc.size, ctypes.byref(out)) == 4
    assert lib.density_b200_decoded_size(ALG_ID[alg], enc.ctypes.data, enc.size, None) == 4
