"""Streams longer than 2^32 bytes through the parallel encoders and decoders, every byte compared (needs an H100: pytest -m gpu).

The kernels keep stream and output offsets in 64 bits next to 32-bit tile-, chunk- and block-relative quantities; one narrowing on
those paths corrupts output only past 4 GiB of stream. The inputs are the pair corpora of tests/big_streams.py at SIZE (5.5 / 7.5 /
7 GiB), whose streams are longer than 2^32 + 2^28 bytes (asserted on every stream). Encodes are compared with the oracle's stream and
decodes with the input, over the whole length, on the device; a mismatch names its first offset. Every output buffer carries a
canary behind its capacity.

Lion decode is not run at this size: lion_decode is the exact in-order kernel at 10-20 MB/s (include/density_b200.h), minutes per
GiB. The sharded decoders of a stream without known cuts are run past 2^32 in test_gpu_sharded_stream_decode.py and
test_gpu_sharded_cheetah_stream_decode.py.
"""
import ctypes

import numpy as np
import pytest

import big_streams as bs

pytestmark = pytest.mark.gpu

CANARY = 0xA5
PAD = 64
GIB = 1 << 30
ALG_ID = {"chameleon": 0, "cheetah": 1, "lion": 2}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device; there is no CPU fallback")
    return torch


@pytest.fixture(scope="module")
def lib(torch_cuda):
    import density_b200
    L = density_b200.load()
    yield L
    L.density_b200_shutdown()                        # the workspaces of these sizes are not for the modules that follow
    torch_cuda.cuda.empty_cache()


def host_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def require_host(nbytes):
    have = host_available()
    if have < nbytes:
        pytest.skip(f"needs {nbytes / GIB:.1f} GiB of available host memory ({have / GIB:.1f} GiB available)")


def require_device(torch, lib, nbytes):
    """Skip unless nbytes of device memory are free once the library's workspaces and torch's cache are released."""
    lib.density_b200_shutdown()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < nbytes:
        pytest.skip(f"needs {nbytes / GIB:.1f} GiB of free device memory ({free / GIB:.1f} GiB free)")


@pytest.fixture(scope="module")
def big():
    """big(alg, bursts=False) -> (input, oracle stream, copy-mode blocks) of the corpus at SIZE[alg]. Only the corpus asked for last
    is kept: each one is 10 to 20 GiB of host memory."""
    kept = {}

    def get(alg, bursts=False):
        key = (alg, bursts)
        if key not in kept:
            kept.clear()
            n = bs.SIZE[alg]
            require_host(n + 2 * oracle_size(alg, n) + 2 * GIB)
            data = bs.corpus(alg, n, bursts=bursts)
            stream, copied = bs.oracle_stream(alg, data)
            assert stream.size > bs.STREAM_MIN, f"{alg} stream of {stream.size} bytes: the corpus no longer reaches past 2^32"
            assert (copied > 0) == bursts
            kept[key] = (data, stream, copied)
        return kept[key]

    yield get
    kept.clear()


def oracle_size(alg, n):
    return int(n * (bs.RATIO[alg] + 0.01))


def canaried(torch, cap):
    buf = torch.empty(cap + PAD, dtype=torch.uint8, device="cuda")
    buf[cap:] = CANARY
    return buf


def canary_held(buf, cap):
    return bool((buf[cap:] == CANARY).all())


def assert_same(torch, got, want, what):
    """got: a device tensor; want: a host array uploaded for the comparison."""
    w = torch.from_numpy(want).cuda()
    off = bs.first_difference(got, w)
    del w
    assert off is None, f"{what}: first difference at byte {off} (0x{off:x}) of {want.size}"


def _stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def encode_device(torch, lib, alg, d_in, out, cap, path):
    """-> (rc, size) of density_b200_encode_device_path into out[:cap]; the size is -1 if the call was refused."""
    sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    rc = lib.density_b200_encode_device_path(ALG_ID[alg], d_in.data_ptr(), d_in.numel(), out.data_ptr(), cap, sz.data_ptr(),
                                             _stream(torch), path)
    torch.cuda.synchronize()
    return rc, int(sz.item())


def decode_device(torch, lib, alg, d_s, out, cap, path):
    sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    rc = lib.density_b200_decode_device_path(ALG_ID[alg], d_s.data_ptr(), d_s.numel(), out.data_ptr(), cap, sz.data_ptr(),
                                             _stream(torch), path)
    torch.cuda.synchronize()
    return rc, int(sz.item())


def encode_and_compare(torch, lib, big, alg, how, bursts=False):
    """Encode the corpus on the device by `how` (a path of density_b200_encode_device_path, or "symbol": <alg>_encode with device
    pointers) into exactly the safe encode size, and compare the whole stream with the oracle's."""
    data, stream, _ = big(alg, bursts)
    n, m = data.size, stream.size
    cap = getattr(lib, f"{alg}_safe_encode_buffer_size")(n)
    require_device(torch, lib, n + cap + m + n)          # input, output, the oracle stream to compare with, workspace
    d_in = torch.from_numpy(data).cuda()
    out = canaried(torch, cap)
    if how == "symbol":
        rc, got = 0, getattr(lib, f"{alg}_encode")(d_in.data_ptr(), n, out.data_ptr(), cap)
    else:
        rc, got = encode_device(torch, lib, alg, d_in, out, cap, how)
    del d_in
    assert rc == 0 and got == m, f"{alg} {how}: rc {rc}, {got} bytes, the oracle's stream has {m}"
    assert canary_held(out, cap)
    assert_same(torch, out[:m], stream, f"{alg} encode {how}")


def decode_and_compare(torch, lib, big, alg, path, bursts=False):
    """Decode the oracle stream on the device by `path` into exactly n bytes (plus a canary) and compare with the input."""
    data, stream, _ = big(alg, bursts)
    n, m = data.size, stream.size
    require_device(torch, lib, m + 2 * n + n)            # stream, output, the input to compare with, workspace
    d_s = torch.from_numpy(stream).cuda()
    out = canaried(torch, n)
    rc, got = decode_device(torch, lib, alg, d_s, out, n, path)
    del d_s
    assert rc == 0 and got == n, f"{alg} decode path {path}: rc {rc}, {got} bytes of {n}"
    assert canary_held(out, n)
    assert_same(torch, out[:n], data, f"{alg} decode path {path}")


def decode_status(lib):
    st = (ctypes.c_uint64 * 10)()
    assert lib.density_b200_decode_status(st) == 0
    return list(st)


def encode_status(lib):
    st = (ctypes.c_uint64 * 6)()
    assert lib.density_b200_encode_status(st) == 0
    return list(st)


# ---- Chameleon, 5.5 GiB of pairs: a 4.39 GiB stream -----------------------------------------------------------------------------
def test_chameleon_encode_fast_path(torch_cuda, lib, big):
    """Path 1, the segment-parallel fast path alone: every tile's output offset past 2^32 comes from the tile scan."""
    encode_and_compare(torch_cuda, lib, big, "chameleon", 1)
    assert lib.density_b200_last_encode_was_fast() == 1


@pytest.mark.parametrize("how", [0, "symbol"])
def test_chameleon_encode_auto_and_symbol(torch_cuda, lib, big, how):
    encode_and_compare(torch_cuda, lib, big, "chameleon", how)
    assert lib.density_b200_last_encode_was_fast() == 1


def test_chameleon_encode_exact_capacity(torch_cuda, lib, big):
    """cap = the stream's size (above 2^32) succeeds; one byte less gives size 0 and writes nothing behind cap."""
    torch = torch_cuda
    data, stream, _ = big("chameleon")
    n, m = data.size, stream.size
    require_device(torch, lib, n + m + m + n)
    d_in = torch.from_numpy(data).cuda()
    out = canaried(torch, m)
    rc, got = encode_device(torch, lib, "chameleon", d_in, out, m, 0)
    assert rc == 0 and got == m and canary_held(out, m)
    assert_same(torch, out[:m], stream, "chameleon encode, cap = stream size")
    out = canaried(torch, m - 1)
    rc, got = encode_device(torch, lib, "chameleon", d_in, out, m - 1, 0)
    assert (rc != 0 or got == 0) and canary_held(out, m - 1), f"cap one byte short: rc {rc}, {got} bytes"


@pytest.mark.parametrize("path", [1, 0])
def test_chameleon_decode(torch_cuda, lib, big, path):
    """Path 1 (parallel decoder only) and path 0 (with the in-order kernel queued behind). The status of the parallel decoder
    agrees with the stream: more than 2^24 main-loop blocks, the tail past 2^32 with fewer than 264 bytes left behind it."""
    decode_and_compare(torch_cuda, lib, big, "chameleon", path)
    data, stream, _ = big("chameleon")
    n, m = data.size, stream.size
    out_bytes, main_blocks, tail_off, nonquiet, error = decode_status(lib)[:5]
    assert (out_bytes, nonquiet, error) == (n, 0, 0)
    assert main_blocks > (1 << 24) and 0 <= n - 256 * main_blocks < 2 * 264
    assert (1 << 32) < tail_off <= m < tail_off + 264


@pytest.mark.parametrize("how", [0, "symbol"])
def test_chameleon_bursts_encode(torch_cuda, lib, big, how):
    """Copy-mode blocks past block 2^24 and stream offset 2^32: path 0 (fixed round budget, the in-order walk behind it) and
    chameleon_encode (path 4, the host keeps iterating the copy map)."""
    encode_and_compare(torch_cuda, lib, big, "chameleon", how, bursts=True)
    data, stream, _ = big("chameleon", True)
    s0 = bs.burst_ranges("chameleon", data.size)[0][0]
    # the blocks from the first burst on encode to at most the safe size of their bytes, so the burst starts past 2^32 of stream
    assert stream.size - lib.chameleon_safe_encode_buffer_size(data.size - s0) > (1 << 32)
    out_bytes, nonquiet, error, first_nonquiet, converged = encode_status(lib)[:5]
    assert (out_bytes, nonquiet, error) == (stream.size, 1, 0)
    assert first_nonquiet >= s0 // 256 > (1 << 24)
    if how == "symbol":
        assert converged == 1


def test_chameleon_bursts_decode(torch_cuda, lib, big):
    """Path 1 on a stream with copy-mode blocks past 2^32: the block boundaries come from the copy-aware walk (dec_seq_walk), whose
    block offsets carry the copy bit."""
    decode_and_compare(torch_cuda, lib, big, "chameleon", 1, bursts=True)
    st = decode_status(lib)
    assert st[0] == big("chameleon", True)[0].size and st[4] == 0
    assert st[6] != 0, "the stream has copy-mode blocks: the boundaries should come from the copy-aware walk"


def test_chameleon_host_buffers_encode(torch_cuda, lib, big):
    """chameleon_encode from pageable host memory: the pipelined path, 64 MiB chunks whose output offsets pass 2^32."""
    torch = torch_cuda
    data, stream, _ = big("chameleon")
    n, m = data.size, stream.size
    cap = lib.chameleon_safe_encode_buffer_size(n)
    require_host(m + GIB)
    require_device(torch, lib, 2 * m + 4 * GIB)
    out = np.empty(cap + PAD, np.uint8)                  # pages past the stream are never touched
    out[cap:] = CANARY
    got = lib.chameleon_encode(data.ctypes.data, n, out.ctypes.data, cap)
    assert got == m and (out[cap:] == CANARY).all()
    assert_same(torch, torch.from_numpy(out[:m]).cuda(), stream, "chameleon_encode, host buffers")


def test_chameleon_host_buffers_decode(torch_cuda, lib, big):
    torch = torch_cuda
    data, stream, _ = big("chameleon")
    n, m = data.size, stream.size
    require_host(n + GIB)
    require_device(torch, lib, 2 * n + m + n)
    out = np.empty(n + PAD, np.uint8)
    out[n:] = CANARY
    got = lib.chameleon_decode(stream.ctypes.data, m, out.ctypes.data, n)
    assert got == n and (out[n:] == CANARY).all()
    assert_same(torch, torch.from_numpy(out[:n]).cuda(), data, "chameleon_decode, host buffers")


# ---- Cheetah, 7.5 GiB of pairs: a 4.34 GiB stream ---------------------------------------------------------------------------------
@pytest.mark.parametrize("path", [1, 0])
def test_cheetah_encode(torch_cuda, lib, big, path):
    encode_and_compare(torch_cuda, lib, big, "cheetah", path)


@pytest.mark.parametrize("path", [1, 0])
def test_cheetah_decode(torch_cuda, lib, big, path):
    decode_and_compare(torch_cuda, lib, big, "cheetah", path)
    if path == 1:
        r = (ctypes.c_uint32 * 4)()
        assert lib.density_b200_cheetah_decode_rounds(r) == 0
        assert r[1] == 1, f"context rounds did not settle: {list(r)}"


# ---- Lion, 7 GiB of pairs: a 4.27 GiB stream ------------------------------------------------------------------------------------
def test_lion_encode(torch_cuda, lib, big):
    encode_and_compare(torch_cuda, lib, big, "lion", 1)
