"""CPU check of the sharded Cheetah decode PROTOCOL (DESIGN.md section 5): tests/cl_piece_model.cpp cuts one oracle-encoded stream into
pieces at the stream offsets of shard cuts, runs every piece's stages with the table logic the CUDA kernels share (cl_core.cuh) and
exchanges the chunk-map transfers once and the prediction transfers and round words in every round. The pieces must reproduce the
input, their carries must equal the in-order decoder's state at every cut, and the rounds must stay in the range of the single-device
scheme with the same total run count. The kernels themselves are checked on the GPU (tests/test_gpu_sharded_cheetah_decode.py)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import oracle
import planted
from conftest import payload

HERE = os.path.dirname(os.path.abspath(__file__))
RUN_BYTES = 16384          # stream bytes per run in the model (the kernels use 48 KiB): more runs, more seams inside every piece
MAX_ROUNDS = 40


def _compile(tmp_path_factory, name):
    so = str(tmp_path_factory.mktemp(name) / f"{name}.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(HERE, f"{name}.cpp"), "-o", so])
    return ctypes.CDLL(so)


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    L = _compile(tmp_path_factory, "cl_piece_model")
    L.cl_piece_model_decode.restype = ctypes.c_size_t
    L.cl_piece_model_decode.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint32,
                                        ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint32)]
    return L


@pytest.fixture(scope="module")
def single_model(tmp_path_factory):
    """the single-device scheme (tests/cl_model.cpp)"""
    L = _compile(tmp_path_factory, "cl_model")
    L.cl_model_decode.restype = ctypes.c_size_t
    L.cl_model_decode.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32,
                                  ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint32)]
    return L


def single_rounds(L, enc, size, nruns):
    out = np.zeros(size + 64, np.uint8)
    stats = (ctypes.c_uint32 * 4)()
    n = L.cl_model_decode(oracle.ALGS["cheetah"], enc.ctypes.data, enc.size, out.ctypes.data, size, nruns, MAX_ROUNDS, stats)
    assert n == size and stats[1] == 1
    return stats[0]


def run_model(L, enc, cuts, nruns=None, max_rounds=MAX_ROUNDS):
    """decode enc cut at the stream offsets `cuts` (0 .. enc.size); returns (decoded, stats): stats = {rounds, settled, verdict, refused
    pieces, chunk-map / prediction / context carries that differ from the in-order decoder at their cut, run walks}"""
    cuts = np.asarray(cuts, np.uint64)
    if nruns is None:
        nruns = [max(1, int(cuts[p + 1] - cuts[p]) // RUN_BYTES) for p in range(cuts.size - 1)]
    nr = np.asarray(nruns, np.uint32)
    cap = 16 * enc.size + 256
    out = np.zeros(cap, np.uint8)
    stats = (ctypes.c_uint32 * 8)()
    n = L.cl_piece_model_decode(enc.ctypes.data, enc.size, cuts.ctypes.data, cuts.size - 1, nr.ctypes.data, max_rounds, out.ctypes.data, cap, stats)
    return out[:n], list(stats), int(nr.sum())


def stream_cuts(data, shard_cuts, enc):
    """the stream offset of every shard cut: a prefix of a multiple of 256 bytes encodes to a prefix of the stream"""
    return [oracle.encode("cheetah", data[:c]).size if c < data.size else enc.size for c in shard_cuts]


def shard_cuts(n, world, seed, lo):
    """world shards of n bytes: non-final cuts at multiples of 256 in [lo, n), sorted, with an empty piece from 4 shards on"""
    if world == 1:
        return [0, n]
    rng = np.random.default_rng(seed)
    inner = sorted(int(c) * 256 for c in rng.integers(lo // 256, n // 256, world - 1))
    if world >= 4:
        inner[2] = inner[1]
    return [0] + inner + [n]


def inputs(dickens):
    yield "text", payload("text", 300001, 4), 16384
    yield "dickens200k", dickens, 16384
    yield "zeros", np.zeros(262144 + 77, np.uint8), 256
    yield "mixed", np.concatenate([payload("mixed", 60000, 9), payload("text", 240000, 2)]), 65536   # copy mode in piece 0 only
    yield "cl1", planted.corpus("cl1")[0], 16384


@pytest.mark.parametrize("world", range(1, 10))
def test_pieces_reproduce_the_input_and_carries_equal_in_order(model, single_model, dickens200k, world):
    for name, data, lo in inputs(dickens200k):
        enc = oracle.encode("cheetah", data)
        sc = shard_cuts(data.size, world, 1000 * world + len(name), lo)
        pc = stream_cuts(data, sc, enc)
        got, st, total_runs = run_model(model, enc, pc)
        assert st[1] == 1 and st[2] == 0, (name, sc, st)
        assert got.size == data.size and (got == data).all(), (name, sc)
        assert st[4:7] == [0, 0, 0], (name, sc, st)         # chunk map, prediction table, entry context at every cut
        # the single-device scheme over the same number of runs: the pieces run the same iteration, with "settled" known one round
        # late (it is read off the next round's gathered words) and the runs cut at the piece ends instead of evenly (up to 2 more
        # rounds on these inputs)
        single = single_rounds(single_model, enc, data.size, total_runs)
        assert st[0] <= single + 3, (name, sc, st[0], single)


def test_refusals(model):
    t = payload("text", 300000, 6)
    noise = np.random.default_rng(3).integers(0, 256, 65536, dtype=np.uint8)
    d = np.concatenate([t[:150016], noise, t[150016:]])
    enc = oracle.encode("cheetah", d)
    # copy mode in piece 1
    _, st, _ = run_model(model, enc, stream_cuts(d, [0, 131072, d.size], enc))
    assert st[2] == 1 and st[3] == 0b10
    # piece 0 ends inside the copy run the noise starts
    _, st, _ = run_model(model, enc, stream_cuts(d, [0, 150016 + 32768, d.size], enc))
    assert st[2] == 1 and st[3] & 1
    # too few rounds: the pieces decode fine with enough of them
    enc = oracle.encode("cheetah", t)
    cuts = stream_cuts(t, [0, 65536, 140032, t.size], enc)
    _, st, _ = run_model(model, enc, cuts, max_rounds=1)
    assert st[1] == 0 and st[2] == 1 and st[3] == 0
    got, st, _ = run_model(model, enc, cuts)
    assert st[1] == 1 and st[2] == 0 and (got == t).all()
