"""The parallel Lion decoder on the GPU (needs an H100: pytest -m gpu): lion_decode, decode_device and decode_device_path with paths 0
and 1 run boundaries, unpack, the chunk-map passes and the prediction walk (cl_decode.cu); path 3 is the in-order kernel. Every output is
compared in full with the oracle, with a canary behind the capacity; the walk's counts with the CPU model's (tests/lion_walk_model.cpp)
and with the counts tests/lion_streams.py computes from the stream."""
import ctypes

import numpy as np
import pytest

import oracle
import lion_streams as ls
from conftest import payload
from lion_streams import TAIL_SWEEP

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


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return ls.build_model(tmp_path_factory.mktemp("lion_walk"))


def model_counts(L, enc, cap):
    return ls.run_model(L, enc, cap)[2]


def _stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def dev_decode(torch, lib, enc, cap, path, in_off=0, out_off=0, canary=64):
    """-> (rc, size, output bytes, canary bytes after cap) of density_b200_decode_device_path for Lion; views at byte offsets."""
    d_in = torch.zeros(enc.size + in_off + 1, dtype=torch.uint8, device="cuda")
    d_in[in_off:in_off + enc.size] = torch.from_numpy(np.ascontiguousarray(enc)).cuda()
    d_out = torch.full((out_off + cap + canary,), CANARY, dtype=torch.uint8, device="cuda")
    d_sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    rc = lib.density_b200_decode_device_path(2, d_in.data_ptr() + in_off, enc.size, d_out.data_ptr() + out_off, cap, d_sz.data_ptr(),
                                             _stream(torch), path)
    torch.cuda.synchronize()
    m = int(d_sz.item())
    out = d_out.cpu().numpy()
    return rc, m, out[out_off:out_off + max(m, 0)], out[out_off + cap:]


def stats(lib):
    s = (ctypes.c_uint64 * 4)()
    assert lib.density_b200_lion_decode_stats(s) == 0
    return tuple(s)


def first_diff(a, b):
    k = min(a.size, b.size)
    d = np.flatnonzero(a[:k] != b[:k])
    return int(d[0]) if d.size else k


def check_paths(torch, lib, data, paths=(0, 1), what=""):
    """decode the oracle stream of data into exactly data.size bytes on each path; returns the stream"""
    enc = oracle.encode("lion", data)
    for path in paths:
        rc, m, got, tail = dev_decode(torch, lib, enc, data.size, path)
        assert rc == 0 and m == data.size, (what, path, m)
        assert (got == data).all(), (what, path, first_diff(got, data))
        assert (tail == CANARY).all(), (what, path)
    return enc


KINDS = [("text", 200000), ("mixed", 150001), ("random", 40003), ("zeros", 600000), ("low", 70002), ("text", 1), ("text", 70),
         ("mixed", 3 * MIB + 5)]


@pytest.mark.parametrize("kind,nbytes", KINDS)
def test_paths_0_and_1(torch_cuda, lib, model, kind, nbytes):
    data = payload(kind, nbytes, seed=3)
    enc = check_paths(torch_cuda, lib, data, what=kind)
    assert stats(lib) == model_counts(model, enc, data.size)


def test_lion_decode_symbol_host_and_device(torch_cuda, lib, dickens200k):
    import density_b200
    torch = torch_cuda
    for data in (dickens200k, payload("mixed", 2 * MIB + 3, seed=8), np.frombuffer(b"test" * 31 + b"t", np.uint8)):
        enc = oracle.encode("lion", data)
        out = np.full(data.size + 64, CANARY, np.uint8)
        n = density_b200.Lion.decode(enc, out[:data.size])
        assert n == data.size and (out[:n] == data).all() and (out[data.size:] == CANARY).all()
        d_in = torch.from_numpy(enc).cuda()
        d_out = torch.full((data.size + 64,), CANARY, dtype=torch.uint8, device="cuda")
        n = lib.lion_decode(ctypes.c_void_p(d_in.data_ptr()), enc.size, ctypes.c_void_p(d_out.data_ptr()), data.size)
        got = d_out.cpu().numpy()
        assert n == data.size and (got[:n] == data).all() and (got[data.size:] == CANARY).all()


def test_decode_device_entry(torch_cuda, lib, model):
    """density_b200_decode_device (no path argument) runs the parallel decoder: its walk counts are the model's"""
    torch = torch_cuda
    data = payload("text", 300001, seed=6)
    enc = oracle.encode("lion", data)
    d_in = torch.from_numpy(enc).cuda()
    d_out = torch.full((data.size + 64,), CANARY, dtype=torch.uint8, device="cuda")
    sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    assert lib.density_b200_decode_device(2, d_in.data_ptr(), enc.size, d_out.data_ptr(), data.size, sz.data_ptr(), _stream(torch)) == 0
    torch.cuda.synchronize()
    got = d_out.cpu().numpy()
    assert int(sz.item()) == data.size and (got[:data.size] == data).all() and (got[data.size:] == CANARY).all()
    assert stats(lib) == model_counts(model, enc, data.size)


def test_stats_after_in_order_decode(torch_cuda, lib):
    """after a Lion decode on the in-order kernel (path 3, a misaligned buffer) the walk counts are not reported"""
    data = payload("text", 50000, seed=2)
    enc = oracle.encode("lion", data)
    for path, in_off in ((3, 0), (0, 1)):
        assert dev_decode(torch_cuda, lib, enc, data.size, 0)[1] == data.size
        stats(lib)
        assert dev_decode(torch_cuda, lib, enc, data.size, path, in_off)[1] == data.size
        s = (ctypes.c_uint64 * 4)()
        assert lib.density_b200_lion_decode_stats(s) != 0, (path, in_off)


def test_golden_digests(torch_cuda, lib, golden, golden_inputs):
    from conftest import sha256
    for name, data in golden_inputs.items():
        g = golden[name]["alg"]["lion"]
        enc = oracle.encode("lion", data)
        assert g["size"] == enc.size and g["sha256"] == sha256(enc), name
        for path in (0, 1):
            rc, m, got, tail = dev_decode(torch_cuda, lib, enc, data.size, path)
            assert rc == 0 and m == data.size and sha256(got) == golden[name]["input_sha256"] and (tail == CANARY).all(), (name, path)


@pytest.mark.parametrize("extra", TAIL_SWEEP)
def test_tail_sweep(torch_cuda, lib, dickens200k, extra):
    check_paths(torch_cuda, lib, dickens200k[:64 * 300 + extra], what=extra)
    check_paths(torch_cuda, lib, np.concatenate([np.zeros(64 * 33, np.uint8), dickens200k[:extra]]), what=extra)


def test_path0_equals_path3(torch_cuda, lib):
    for kind in ("text", "mixed", "random", "zeros", "low"):
        data = payload(kind, 1 * MIB + 77, seed=21)
        enc = oracle.encode("lion", data)
        r0 = dev_decode(torch_cuda, lib, enc, data.size, 0)
        r3 = dev_decode(torch_cuda, lib, enc, data.size, 3)
        assert r0[0] == r3[0] == 0 and r0[1] == r3[1] == data.size and (r0[2] == r3[2]).all() and (r0[2] == data).all(), kind


def test_walk_inputs(torch_cuda, lib, model):
    for name, data in ls.walk_inputs().items():
        enc = check_paths(torch_cuda, lib, data, what=name)
        s = stats(lib)
        assert s == model_counts(model, enc, data.size) == ls.walk_counts(enc, data), name
        assert s[1] > 0, name


def test_zero_fill_and_records(torch_cuda, lib):
    rng = np.random.default_rng(4)
    zf = np.concatenate([payload("text", 100000, 1), np.zeros(6 * MIB + 5, np.uint8), rng.integers(0, 256, 3000, dtype=np.uint8),
                         np.zeros(2 * MIB, np.uint8), payload("text", 50001, 2)])
    check_paths(torch_cuda, lib, zf, what="zero fill")
    assert stats(lib)[1] > (8 * MIB) // 4 - 100000
    for period in range(2, 41):
        check_paths(torch_cuda, lib, ls.records(period, 300000 + period), what=period)


@pytest.mark.parametrize("seed", range(8))
def test_random_flag_streams(torch_cuda, lib, model, seed):
    """well-formed streams no encoder writes: random flags at several densities of predicted quads, the protection automaton's copy-mode
    blocks where a decoder expects them, and raw tails of every kind"""
    s = ls.synth_stream(seed, 4000 + 997 * seed, tail_bytes=[0, 3, 40, 69, 70, 100, 5, 64][seed],
                        p_pred=[0.5, 0.9, 0.2, 0.7, 0.99, 0.5, 0.0, 0.35][seed])
    cap = ls.decode_cap(s)
    want = oracle.decode("lion", s, cap)
    for path in (0, 1):
        rc, m, got, tail = dev_decode(torch_cuda, lib, s, cap, path)
        assert rc == 0 and (tail == CANARY).all(), (seed, path)
        if path == 1 and want.size == 0:
            assert m == 0, seed                        # the walk never gives up; a malformed tail is reported by the tail kernel
            continue
        assert m == want.size and (got == want).all(), (seed, path, m, want.size, first_diff(got, want))
    if want.size:
        assert stats(lib) == model_counts(model, s, cap) == ls.walk_counts(s, want)


def test_capacity(torch_cuda, lib, dickens200k):
    data = dickens200k
    enc = oracle.encode("lion", data)
    for cap in (data.size - 1, data.size - 63, data.size - 64 * 5, 1000, 0):
        want = oracle.decode("lion", enc, max(cap, 1))
        for path in (0, 1, 3):
            rc, m, got, tail = dev_decode(torch_cuda, lib, enc, cap, path)
            assert rc == 0 and m == want.size == 0 and (tail == CANARY).all(), (cap, path)


def test_misaligned_buffers(torch_cuda, lib, dickens200k):
    """d_in not 2-byte or d_out not 4-byte aligned: the in-order kernel decodes (path 0 and path 1)"""
    data = dickens200k[:100003]
    enc = oracle.encode("lion", data)
    for in_off, out_off in ((1, 0), (0, 2), (3, 1)):
        for path in (0, 1):
            rc, m, got, tail = dev_decode(torch_cuda, lib, enc, data.size, path, in_off, out_off)
            assert rc == 0 and m == data.size and (got == data).all() and (tail == CANARY).all(), (in_off, out_off, path)


def test_truncated_and_corrupted(torch_cuda, lib, dickens200k):
    """what path 3 returns, on path 0; path 1 returns the same or size 0"""
    rng = np.random.default_rng(9)
    data = dickens200k[:120000]
    enc = oracle.encode("lion", data)
    cases = [enc[:k] for k in (1, 5, 6, 7, 69, 70, 71, 1000, enc.size // 2, enc.size - 1)]
    for _ in range(12):
        c = enc.copy()
        for i in rng.integers(0, c.size, 3):
            c[i] ^= np.uint8(1 << int(rng.integers(0, 8)))
        cases.append(c)
    for k, s in enumerate(cases):
        r3 = dev_decode(torch_cuda, lib, s, data.size, 3)
        want = oracle.decode("lion", s, data.size)
        assert r3[1] == want.size and (r3[2] == want).all(), k
        r0 = dev_decode(torch_cuda, lib, s, data.size, 0)
        assert r0[0] == 0 and r0[1] == r3[1] and (r0[2] == r3[2]).all() and (r0[3] == CANARY).all(), k
        r1 = dev_decode(torch_cuda, lib, s, data.size, 1)
        assert r1[1] in (0, r3[1]) and (r1[1] == 0 or (r1[2] == r3[2]).all()) and (r1[3] == CANARY).all(), k


def test_256_mib(torch_cuda, lib):
    from density_b200 import synth
    torch = torch_cuda
    for data in (synth.synth_mixed(256 * MIB), synth.synth_text(256 * MIB)):
        d_data = data.cuda()
        cap = lib.lion_safe_encode_buffer_size(data.numel())
        d_enc = torch.empty(cap, dtype=torch.uint8, device="cuda")
        sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        assert lib.density_b200_encode_device_path(2, d_data.data_ptr(), data.numel(), d_enc.data_ptr(), cap, sz.data_ptr(), _stream(torch), 0) == 0
        torch.cuda.synchronize()
        m = int(sz.item())
        enc = d_enc[:m].cpu().numpy()
        assert (enc == oracle.encode("lion", data.numpy())).all()
        d_out = torch.full((data.numel() + 64,), CANARY, dtype=torch.uint8, device="cuda")
        assert lib.density_b200_decode_device_path(2, d_enc.data_ptr(), m, d_out.data_ptr(), data.numel(), sz.data_ptr(), _stream(torch), 0) == 0
        torch.cuda.synchronize()
        assert int(sz.item()) == data.numel()
        assert bool(d_out[:data.numel()].equal(d_data)) and bool((d_out[data.numel():] == CANARY).all())
        del d_data, d_enc, d_out


def test_stream_beyond_4gib(torch_cuda, lib):
    """one stream longer than 2^32 + 2^28 bytes (the pair corpus of tests/big_streams.py with its noise bursts, so copy-mode blocks sit
    past 2^32 too), encoded on the device (its stream equals the oracle's: test_gpu_beyond_4gib.py) and decoded with path 0"""
    import big_streams as bs
    torch = torch_cuda
    n = bs.SIZE["lion"]
    lib.density_b200_shutdown()
    torch.cuda.empty_cache()
    need = n + int(n * (bs.RATIO["lion"] + 0.01)) + n + int(n * 0.9)
    if torch.cuda.mem_get_info()[0] < need:
        pytest.skip("not enough free device memory")
    data = torch.from_numpy(bs.corpus("lion", n, bursts=True)).cuda()
    cap = lib.lion_safe_encode_buffer_size(n)
    d_enc = torch.empty(cap, dtype=torch.uint8, device="cuda")
    sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    assert lib.density_b200_encode_device_path(2, data.data_ptr(), n, d_enc.data_ptr(), cap, sz.data_ptr(), _stream(torch), 0) == 0
    torch.cuda.synchronize()
    m = int(sz.item())
    assert m > bs.STREAM_MIN
    d_out = torch.empty(n + 64, dtype=torch.uint8, device="cuda")
    d_out[n:] = CANARY
    assert lib.density_b200_decode_device_path(2, d_enc.data_ptr(), m, d_out.data_ptr(), n, sz.data_ptr(), _stream(torch), 0) == 0
    torch.cuda.synchronize()
    assert int(sz.item()) == n
    off = bs.first_difference(d_out[:n], data)
    assert off is None, f"first difference at byte {off}"
    assert bool((d_out[n:] == CANARY).all())
    del data, d_enc, d_out
    lib.density_b200_shutdown()
    torch.cuda.empty_cache()
