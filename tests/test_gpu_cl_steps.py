"""Collision steps (tests/cl_steps.py) through the run-parallel Cheetah and Lion encoders and decoders on the GPU (needs an H100:
pytest -m gpu): whole warp steps in one hash bucket and one context, at run edges, split across adjacent steps, in both halves of a Lion
step, behind copy-mode episodes and in the last partial step. Every stream equals oracle.encode byte for byte; every output buffer has a
64-byte canary behind its capacity.

The in-order kernel (path 3) gets the corpora of at most 4 MiB: it is one thread, and on cls33 it would take most of the file's time
without reaching any kernel the collision steps are aimed at."""
import ctypes

import numpy as np
import pytest

import cl_steps
import lion_streams
import oracle
from test_gpu_planted import CANARY, assert_stream, dev_decode, dev_encode, first_diff
from test_gpu_sharded_cheetah_decode import decode_pieces, piece_cuts
from test_gpu_sharded_cl_encode import encode_shards
from test_gpu_sharded_lion_decode import decode_lion_pieces

pytestmark = pytest.mark.gpu
ALGS = ("cheetah", "lion")
NAMES = ("cls1", "cls33", "cls_pure", "cls_copy")
SMALL = ("cls1", "cls_pure", "cls_copy")


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


_want = {}


def want(alg, name):
    if (alg, name) not in _want:
        _want[(alg, name)] = oracle.encode(alg, cl_steps.build(name)[0])
    return _want[(alg, name)]


@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("name", NAMES)
def test_encode_device_paths(torch_cuda, lib, alg, name):
    """encode_device paths 0 (auto), 1 (run-parallel only) and 3 (in-order kernel), then the exact capacity and one byte less"""
    data = cl_steps.build(name)[0]
    w = want(alg, name)
    for path in (0, 1, 3) if name in SMALL else (0, 1):
        rc, n, got, tail = dev_encode(torch_cuda, lib, alg, data, path)
        if path == 1 and n == 0:
            pytest.fail(f"{alg} {name}: the run-parallel encoder's copy map did not settle")
        assert_stream(rc, n, got, w, f"{alg} {name} path {path}")
        assert (tail == CANARY).all(), f"{alg} {name} path {path}: wrote past cap"
    rc, n, got, tail = dev_encode(torch_cuda, lib, alg, data, 0, cap=w.size)
    assert_stream(rc, n, got, w, f"{alg} {name} cap = stream size")
    assert (tail == CANARY).all()
    rc, n, got, tail = dev_encode(torch_cuda, lib, alg, data, 0, cap=w.size - 1)
    assert (rc != 0 or n == 0) and got.size == 0, f"{alg} {name}: an encode into one byte less than the stream reported {n} bytes"
    assert (tail == CANARY).all(), f"{alg} {name}: wrote past cap"


@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("name", NAMES)
def test_encode_synchronous_from_pageable_host_memory(alg, name, lib):
    """the synchronous reference symbol (path 4 inside) on pageable numpy buffers, with a canary behind the output"""
    import density_b200
    data = cl_steps.build(name)[0]
    w = want(alg, name)
    C = density_b200.CODECS[alg]
    out = np.full(C.safe_encode_buffer_size(data.size) + 64, CANARY, np.uint8)
    n = C.encode(data, out[:-64])
    assert n == w.size and (out[:n] == w).all(), f"{alg} {name}: first differing byte {first_diff(out[:n], w)}"
    assert (out[-64:] == CANARY).all()


@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("name", NAMES)
def test_decode_device_paths(torch_cuda, lib, alg, name):
    """decode_device paths 0, 1 and 3 of the oracle's stream; the Cheetah decoder's context rounds settle, the Lion decoder's walk counts
    equal lion_streams.walk_counts"""
    data = cl_steps.build(name)[0]
    enc = want(alg, name)
    for path in (0, 1, 3) if name in SMALL else (0, 1):
        rc, m, got, tail = dev_decode(torch_cuda, lib, alg, enc, data.size, path)
        assert rc == 0 and m == data.size, (alg, name, path, rc, m)
        assert (got == data).all(), f"{alg} {name} path {path}: first differing byte {first_diff(got, data)}"
        assert (tail == CANARY).all(), f"{alg} {name} path {path}: wrote past cap"
        if path == 1 and alg == "cheetah":
            r = (ctypes.c_uint32 * 4)()
            assert lib.density_b200_cheetah_decode_rounds(r) == 0
            assert r[1] == 1, f"{name}: the context rounds did not settle: {list(r)}"
        if path == 1 and alg == "lion":
            c = (ctypes.c_uint64 * 4)()
            assert lib.density_b200_lion_decode_stats(c) == 0
            assert tuple(c) == lion_streams.walk_counts(enc, data), (name, tuple(c))


def _cuts(name, k):
    """256-byte cuts on collision steps (step pairs start every 64 quads) and between the two halves of a split group"""
    data, man, _ = cl_steps.build(name)
    at = ("run_mid", "alt2", "halves", "pure", "after_copy")
    starts = sorted({p * 4 for p, v, c, w, r, *_ in man if r == "step" and p % 64 == 0 and w in at})
    split = sorted({(p + 16) * 4 for p, v, c, w, r, *_ in man if r == "step" and w == "split" and p % 32 == 16})
    pick = lambda xs, j: xs[(j * len(xs)) // (k + 1)] if xs else None
    cuts = {pick(starts, j) for j in range(1, k + 1)} | {pick(split, j) for j in range(1, k + 1)}
    cuts = sorted(c for c in cuts if c and 0 < c < data.size)
    return [0] + cuts + [data.size]


@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("name", SMALL)
def test_sharded_encode_and_decode_cut_at_collision_steps(torch_cuda, lib, alg, name):
    """the sharded encoder's shards cut on collision steps and inside split groups concatenate to the oracle's stream; the sharded
    decoders' pieces cut at the same places decode to their slices. Where a shard after the first holds copy-mode blocks, the
    protection-aware sharded paths run (the quiet ones refuse such shards)."""
    import test_gpu_sharded_cl_protected_encode as PE
    from test_gpu_sharded_cheetah_protected_decode import decode_prot_pieces
    data = cl_steps.build(name)[0]
    w = want(alg, name)
    cuts = _cuts(name, 3)
    assert len(cuts) >= 5, cuts
    _, copied = cl_steps.stream_flags(alg, w, data.size)
    prot = bool(copied[cuts[1] // cl_steps.BS[alg]:].any())
    pieces, (flags, total, _), words = (PE.encode_shards if prot else encode_shards)(torch_cuda, lib, alg, data, cuts)
    assert flags == 0, (alg, name, cuts, words)
    cat = np.concatenate(pieces)
    assert total == w.size and cat.size == w.size and (cat == w).all(), (alg, name, cuts, first_diff(cat, w))
    caps = [max(b - a, 4) for a, b in zip(cuts[:-1], cuts[1:])]
    if alg == "lion":
        flags, total, got, words, _, _ = decode_lion_pieces(torch_cuda, lib, pieces, caps, prot)
    elif prot:
        flags, total, got, _, words = decode_prot_pieces(torch_cuda, lib, pieces, caps)
    else:
        got, (flags, total, _), words, _ = decode_pieces(torch_cuda, lib, w, piece_cuts(pieces))
    assert flags == 0 and total == data.size, (alg, name, prot, words)
    for r in range(len(cuts) - 1):
        sl = data[cuts[r]:cuts[r + 1]]
        assert got[r].size == sl.size and (got[r] == sl).all(), (alg, name, r, first_diff(got[r], sl))


@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("name", SMALL)
def test_codec_instance_two_calls_cut_at_a_collision_step(torch_cuda, lib, alg, name):
    """CodecInstance encode in two calls, cut at a collision step, equals the oracle Codec's continuation, and decodes back in two calls"""
    import density_b200
    from density_b200.codec import CodecInstance
    data = cl_steps.build(name)[0]
    cut = _cuts(name, 1)[1]
    pieces = [data[:cut], data[cut:]]
    ref, enc, dec = oracle.Codec(alg), CodecInstance(alg), CodecInstance(alg)
    try:
        streams = []
        for p in pieces:
            w = ref.encode(p)
            out = np.full(density_b200.CODECS[alg].safe_encode_buffer_size(p.size) + 64, CANARY, np.uint8)
            n = enc.encode(p, out[:-64])
            assert n == w.size and (out[:n] == w).all(), (alg, name, cut, first_diff(out[:n], w))
            assert (out[-64:] == CANARY).all()
            streams.append(out[:n].copy())
        for p, s in zip(pieces, streams):
            back = np.full(p.size + 64, CANARY, np.uint8)
            assert dec.decode(s, back[:-64]) == p.size and (back[:-64] == p).all() and (back[-64:] == CANARY).all()
    finally:
        enc.close(); dec.close()
