"""Planted corpora (tests/planted.py) through every encode and decode path on the GPU (needs an H100: pytest -m gpu).

Every stream is compared byte for byte with oracle.encode and must decode back, on the GPU and with the oracle. Also: state carried
across calls (CodecInstance, the one-GPU shard path, a fixed call order in one process), output bounds and pointer alignment."""
import ctypes

import numpy as np
import pytest

import oracle
import planted
from planted import TILE_QUADS, corpus, quad_of, twin

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
    return density_b200.load()  # raises if the CUDA extension is missing


def _stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def dev_encode(torch, lib, alg, data, path, cap=None, canary=64, in_off=0, out_off=0):
    """-> (rc, size, stream bytes, canary bytes after cap). d_in / d_out may be views at byte offsets."""
    import density_b200
    cap = density_b200.CODECS[alg].safe_encode_buffer_size(data.size) if cap is None else cap
    d_in = torch.zeros(data.size + in_off, dtype=torch.uint8, device="cuda")
    d_in[in_off:] = torch.from_numpy(data).cuda()
    d_out = torch.full((out_off + cap + canary,), CANARY, dtype=torch.uint8, device="cuda")
    d_sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    rc = lib.density_b200_encode_device_path(density_b200.codec.ALG_IDS[alg], d_in.data_ptr() + in_off, data.size,
                                             d_out.data_ptr() + out_off, cap, d_sz.data_ptr(), _stream(torch), path)
    torch.cuda.synchronize()
    n = int(d_sz.item())
    out = d_out.cpu().numpy()
    return rc, n, out[out_off:out_off + max(n, 0)], out[out_off + cap:]


def dev_decode(torch, lib, alg, enc, n, path, canary=64, in_off=0, out_off=0):
    import density_b200
    d_in = torch.zeros(enc.size + in_off, dtype=torch.uint8, device="cuda")
    d_in[in_off:] = torch.from_numpy(enc).cuda()
    d_out = torch.full((out_off + n + canary,), CANARY, dtype=torch.uint8, device="cuda")
    d_sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    rc = lib.density_b200_decode_device_path(density_b200.codec.ALG_IDS[alg], d_in.data_ptr() + in_off, enc.size,
                                             d_out.data_ptr() + out_off, n, d_sz.data_ptr(), _stream(torch), path)
    torch.cuda.synchronize()
    m = int(d_sz.item())
    out = d_out.cpu().numpy()
    return rc, m, out[out_off:out_off + max(m, 0)], out[out_off + n:]


def first_diff(a, b):
    k = min(a.size, b.size)
    d = np.flatnonzero(a[:k] != b[:k])
    return int(d[0]) if d.size else k


def assert_stream(got_rc, got_n, got, want, what):
    assert got_rc == 0, what
    assert got_n == want.size and (got == want).all(), f"{what}: size {got_n} vs {want.size}, first differing byte {first_diff(got, want)}"


_want = {}


def want_stream(alg, name):
    if (alg, name) not in _want:
        _want[(alg, name)] = oracle.encode(alg, corpus(name)[0])
    return _want[(alg, name)]


# ---- Chameleon encode -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,path", [("cham33", 0), ("cham33", 1), ("cham5", 2), ("copy3", 0), ("copy3", 2)])
def test_chameleon_encode_device_paths(torch_cuda, lib, name, path):
    """encode_device paths 0 (auto), 1 (fast path only: quiet corpora) and 2 (protection-aware walk). The GPU stream decodes back
    with the oracle and on the GPU."""
    torch = torch_cuda
    data, _ = corpus(name)
    want = want_stream("chameleon", name)
    rc, n, got, tail = dev_encode(torch, lib, "chameleon", data, path)
    if path == 1:
        assert lib.density_b200_last_encode_was_fast() == 1
    assert_stream(rc, n, got, want, f"{name} path {path}")
    assert (tail == CANARY).all()
    assert (oracle.decode("chameleon", got, data.size) == data).all()
    rc, m, back, _ = dev_decode(torch, lib, "chameleon", got, data.size, 0)
    assert rc == 0 and m == data.size and (back == data).all()


def test_chameleon_encode_through_reference_symbols(torch_cuda, lib):
    """chameleon_encode with device pointers (33 MiB) and with host buffers of 129 MiB, which take the pipelined path in 64 MiB chunks
    with plantings on both sides of the 64 and 128 MiB seams."""
    torch = torch_cuda
    import density_b200
    C = density_b200.Chameleon
    data, _ = corpus("cham33")
    want = want_stream("chameleon", "cham33")
    d_in = torch.from_numpy(data).cuda()
    d_out = torch.zeros(C.safe_encode_buffer_size(data.size), dtype=torch.uint8, device="cuda")
    n = C.encode(d_in, d_out)
    assert n == want.size and (d_out[:n].cpu().numpy() == want).all(), first_diff(d_out[:n].cpu().numpy(), want)
    big, _ = corpus("cham129")
    want = want_stream("chameleon", "cham129")
    out = np.zeros(C.safe_encode_buffer_size(big.size), dtype=np.uint8)
    n = C.encode(big, out)
    assert n == want.size and (out[:n] == want).all(), first_diff(out[:n], want)


# ---- Chameleon decode -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,path", [("cham33", 0), ("cham33", 1), ("cham5", 3), ("copy3", 0), ("copy3", 1), ("copy3", 3)])
def test_chameleon_decode_device_paths(torch_cuda, lib, name, path):
    """decode_device paths 0, 1 and 3 on oracle streams; the output buffer is exactly n bytes, followed by a canary that must stay
    intact."""
    torch = torch_cuda
    data, _ = corpus(name)
    enc = want_stream("chameleon", name)
    rc, m, got, tail = dev_decode(torch, lib, "chameleon", enc, data.size, path)
    assert rc == 0 and m == data.size, (name, path, m)
    assert (got == data).all(), f"first differing byte {first_diff(got, data)}"
    assert (tail == CANARY).all(), "wrote past the output capacity"


# ---- Cheetah / Lion ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", ["cheetah", "lion"])
@pytest.mark.parametrize("name,path", [("cl1", 0), ("cl1", 1), ("cl1", 3), ("cl33", 0), ("cl33", 1)])
def test_cheetah_lion_encode_paths(torch_cuda, lib, alg, name, path):
    torch = torch_cuda
    data, _ = corpus(name)
    want = want_stream(alg, name)
    rc, n, got, tail = dev_encode(torch, lib, alg, data, path)
    if path == 1 and n == 0:
        pytest.fail("the run-parallel encoder's copy map did not settle on a planted corpus")
    assert_stream(rc, n, got, want, f"{alg} {name} path {path}")
    assert (tail == CANARY).all()
    assert (oracle.decode(alg, got, data.size) == data).all()


@pytest.mark.parametrize("name", ["cl1", "cl33"])
@pytest.mark.parametrize("path", [0, 1])
def test_cheetah_decode_paths(torch_cuda, lib, name, path):
    torch = torch_cuda
    data, _ = corpus(name)
    rc, m, got, tail = dev_decode(torch, lib, "cheetah", want_stream("cheetah", name), data.size, path)
    assert rc == 0 and m == data.size and (got == data).all(), first_diff(got, data)
    assert (tail == CANARY).all()


@pytest.mark.parametrize("name", ["cl1", "cl33"])
def test_lion_decode(torch_cuda, lib, name):
    """lion_decode (host buffers) and decode_device path 0, each into exactly n bytes followed by a canary."""
    torch = torch_cuda
    import density_b200
    data, _ = corpus(name)
    enc = want_stream("lion", name)
    out = np.full(data.size + 64, CANARY, dtype=np.uint8)
    assert density_b200.Lion.decode(enc, out[:data.size]) == data.size
    assert (out[:data.size] == data).all() and (out[data.size:] == CANARY).all()
    rc, m, got, tail = dev_decode(torch, lib, "lion", enc, data.size, 0)
    assert rc == 0 and m == data.size and (got == data).all() and (tail == CANARY).all()


# ---- state carried across calls ---------------------------------------------------------------------------------------------
def _continuation_pieces(alg):
    """Three pieces; each of the first two ends with a bucket's last writer being its fingerprint-0 member, a bit-31 twin or quad 0, and
    the next piece starts by touching that bucket."""
    data, _ = corpus("cham5" if alg == "chameleon" else "cl1")
    P = planted.Planter(data.size, 99, data.copy())     # its free buckets: untouched by the corpus, plantings included
    cuts = [P.nq // 3, 2 * P.nq // 3 + 1]
    for k, c in enumerate(cuts):
        h1, h2 = P.bucket(), P.bucket()
        a = quad_of(h2, P.fp())
        for j, v in enumerate([quad_of(h1, 0), twin(a), 0] if k == 0 else [0, quad_of(h1, 0), twin(a)]):
            P.put(c - 3 + j, v, "last_writer")
        for j, v in enumerate([quad_of(h1, P.fp()), a, quad_of(0, P.fp()), quad_of(h1, 0)]):
            P.put(c + j, v, "first_touch")
    b = P.data
    return [b[:4 * cuts[0]], b[4 * cuts[0]:4 * cuts[1]], b[4 * cuts[1]:]]


@pytest.mark.parametrize("alg", ["chameleon", "cheetah", "lion"])
def test_codec_instance_continuation_at_planted_seams(torch_cuda, lib, alg):
    import density_b200
    from density_b200.codec import CodecInstance
    pieces = _continuation_pieces(alg)
    ref, enc, dec = oracle.Codec(alg), CodecInstance(alg), CodecInstance(alg)
    streams = []
    for p in pieces:
        want = ref.encode(p)
        out = np.zeros(density_b200.CODECS[alg].safe_encode_buffer_size(p.size), dtype=np.uint8)
        n = enc.encode(p, out)
        assert n == want.size and (out[:n] == want).all(), (alg, p.size, first_diff(out[:n], want))
        streams.append(out[:n].copy())
    for p, s in zip(pieces, streams):
        back = np.zeros(p.size, dtype=np.uint8)
        assert dec.decode(s, back) == p.size and (back == p).all()
    enc.close(); dec.close()


def test_shard_phases_cut_at_planted_positions(torch_cuda, lib):
    """The one-GPU shard path (phase 1 on every shard, tables folded left to right, phase 2 with the carried-in dictionary), cut at
    a run start with planted edges and carried states, and 3 blocks into a tile of a later run."""
    torch = torch_cuda
    import density_b200
    from density_b200 import sharded
    data, _ = corpus("cham5")
    want = want_stream("chameleon", "cham5")
    runs = planted.cham_runs(data.size)
    cuts = [0, runs[3][0] * TILE_QUADS * 4, runs[9][0] * TILE_QUADS * 4 + 256 * 3 + 4 * TILE_QUADS, data.size]
    stream = _stream(torch)
    encs, tables, ins = [], [], []
    for r in range(3):
        d_in = torch.from_numpy(data[cuts[r]:cuts[r + 1]].copy()).cuda()
        t = torch.empty(65536, dtype=torch.int32, device="cuda")
        e = sharded.ShardedChameleonEncoder()
        assert lib.density_b200_shard_phase1(e._h, d_in.data_ptr(), d_in.numel(), int(r == 2), t.data_ptr(), stream) == 0
        encs.append(e); tables.append(t); ins.append(d_in)
    gathered = torch.stack(tables)
    pieces = []
    for r in range(3):
        carry = sharded.fold_tables(gathered, r) if r > 0 else None
        d_out = torch.zeros(density_b200.Chameleon.safe_encode_buffer_size(ins[r].numel()), dtype=torch.uint8, device="cuda")
        d_sz = torch.zeros(1, dtype=torch.int64, device="cuda")
        d_fl = torch.zeros(1, dtype=torch.int32, device="cuda")
        assert lib.density_b200_shard_phase2(encs[r]._h, carry.data_ptr() if carry is not None else None, d_out.data_ptr(),
                                             d_out.numel(), d_sz.data_ptr(), d_fl.data_ptr(), stream) == 0
        torch.cuda.synchronize()
        assert int(d_fl.item()) == 0
        pieces.append(d_out[:int(d_sz.item())].cpu().numpy())
    got = np.concatenate(pieces)
    assert got.size == want.size and (got == want).all(), first_diff(got, want)


def test_fixed_call_order_in_one_process(torch_cuda, lib):
    """40 MiB encode, 300 B, 1 MiB Cheetah, 40 MiB decode, 1 MiB Lion, the first 40 MiB again: state must not leak between calls through
    the cached workspace, the epoch-tagged tables, the double-buffered mailbox counters or a shrinking run count."""
    torch = torch_cuda
    big = planted.chameleon_corpus(40 * planted.MIB + 5, 7)[0]
    small = big[:300].copy()
    cl, _ = corpus("cl1")
    big_want = oracle.encode("chameleon", big)
    steps = [("enc", "chameleon", big, big_want), ("enc", "chameleon", small, oracle.encode("chameleon", small)),
             ("enc", "cheetah", cl, want_stream("cheetah", "cl1")), ("dec", "chameleon", big, big_want),
             ("enc", "lion", cl, want_stream("lion", "cl1")), ("enc", "chameleon", big, big_want)]
    for k, (op, alg, data, want) in enumerate(steps):
        if op == "enc":
            rc, n, got, _ = dev_encode(torch, lib, alg, data, 0)
            assert_stream(rc, n, got, want, f"step {k}: {alg} encode of {data.size} B")
        else:
            rc, m, got, _ = dev_decode(torch, lib, alg, want, data.size, 0)
            assert rc == 0 and m == data.size and (got == data).all(), f"step {k}: first differing byte {first_diff(got, data)}"


# ---- output bounds and pointer alignment ------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", ["chameleon", "cheetah", "lion"])
def test_encode_capacity_edges(torch_cuda, lib, alg):
    """cap = safe size, cap = the exact stream size (succeeds), cap = one byte less (fails, writes nothing past cap), through
    encode_device path 0 and through the reference symbol with host buffers."""
    torch = torch_cuda
    import density_b200
    C = density_b200.CODECS[alg]
    data = corpus("cham5")[0][:(1 << 20) + 7].copy()
    want = oracle.encode(alg, data)
    for cap in (C.safe_encode_buffer_size(data.size), want.size):
        rc, n, got, tail = dev_encode(torch, lib, alg, data, 0, cap=cap)
        assert_stream(rc, n, got, want, f"{alg} cap {cap}")
        assert (tail == CANARY).all(), f"{alg}: wrote past cap {cap}"
    rc, n, got, tail = dev_encode(torch, lib, alg, data, 0, cap=want.size - 1)
    assert rc != 0 or n == 0, f"{alg}: an encode into one byte less than the stream reported {n} bytes"
    assert (tail == CANARY).all(), f"{alg}: wrote past cap"
    out = np.full(want.size + 63, CANARY, dtype=np.uint8)
    with pytest.raises(density_b200.EncodeError):
        C.encode(data, out[:want.size - 1])
    assert (out[want.size - 1:] == CANARY).all()
    assert C.encode(data, out[:want.size]) == want.size and (out[:want.size] == want).all()


@pytest.mark.parametrize("alg", ["chameleon", "cheetah", "lion"])
def test_unaligned_pointers(torch_cuda, lib, alg):
    """d_in / d_out at byte offsets 1, 2 and 3 (api.cu: the parallel encoders need d_in 4-aligned and d_out 2-aligned, the parallel
    decoders d_in 2-aligned and d_out 4-aligned; other pointers take the in-order kernels, except that an encode into an odd d_out is
    rejected with DENSITY_B200_EARG). Through encode_device, decode_device and the reference symbols."""
    torch = torch_cuda
    import density_b200
    C = density_b200.CODECS[alg]
    data = corpus("cham5")[0][:70001 + 4 * TILE_QUADS].copy()
    want = oracle.encode(alg, data)
    for off in (0, 1, 2, 3):
        for in_off, out_off in ((off, 0), (0, off), (off, off)):
            rc, n, got, tail = dev_encode(torch, lib, alg, data, 0, in_off=in_off, out_off=out_off)
            if out_off % 2:
                assert rc == 4, (alg, in_off, out_off, rc)        # DENSITY_B200_EARG
                assert (tail == CANARY).all() and (got.size == 0)
            else:
                assert_stream(rc, n, got, want, f"{alg} encode d_in+{in_off} d_out+{out_off}")
            rc, m, back, tail = dev_decode(torch, lib, alg, want, data.size, 0, in_off=in_off, out_off=out_off)
            assert rc == 0 and m == data.size and (back == data).all(), (alg, in_off, out_off, m)
            assert (tail == CANARY).all()
        # the reference symbols with device pointers
        d_in = torch.zeros(data.size + off, dtype=torch.uint8, device="cuda")
        d_in[off:] = torch.from_numpy(data).cuda()
        d_out = torch.full((C.safe_encode_buffer_size(data.size) + off,), CANARY, dtype=torch.uint8, device="cuda")
        n = getattr(lib, f"{alg}_encode")(d_in.data_ptr() + off, data.size, d_out.data_ptr() + off, d_out.numel() - off)
        if off % 2:
            assert n == 0
        else:
            assert n == want.size and (d_out[off:off + n].cpu().numpy() == want).all(), (alg, off)
        d_enc = torch.zeros(want.size + off, dtype=torch.uint8, device="cuda")
        d_enc[off:] = torch.from_numpy(want).cuda()
        d_dec = torch.full((data.size + off + 64,), CANARY, dtype=torch.uint8, device="cuda")
        m = getattr(lib, f"{alg}_decode")(d_enc.data_ptr() + off, want.size, d_dec.data_ptr() + off, data.size)
        dec = d_dec.cpu().numpy()
        assert m == data.size and (dec[off:off + m] == data).all() and (dec[off + m:] == CANARY).all(), (alg, off)
