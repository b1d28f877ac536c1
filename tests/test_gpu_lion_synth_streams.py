"""Synthesized Lion streams (tests/synth_streams.py) through every single-device and sharded Lion decode path on an H100 (pytest -m gpu).
The answer is always oracle.decode("lion", stream, cap); every output buffer is exactly `cap` bytes followed by a 64-byte canary. The
streams hold what no encoder writes, placed on the parallel Lion decoder's own seams (the rows' lanes 0, 15, 16 and 31, rows with one
copy-mode block, chunk-map run and piece edges, the last main-loop quad and the first tail quad): MAP_A / MAP_B at unwritten or once-written
buckets followed by a predicted quad (its context is the explicit hash, not hash16(0)), predicted reads of lists never pushed, too short or
holding duplicates, more than five pushes in one row, self-mapping spans behind deep reads and across copy-mode blocks."""
import collections
import ctypes

import numpy as np
import pytest

import oracle
import lion_streams as ls
import synth_streams as ss
from test_gpu_sharded_lion_decode import decode_lion_pieces
from test_gpu_sharded_lion_decode_loopback import decode as loopback_decode
from test_gpu_sharded_loopback import env  # noqa: F401  (the loopback ranks' fixture)
from test_gpu_synth_streams import dev_decode, check, caps_of, pieces_at, CANARY
from test_synth_streams_cpu import lion_coverage, lion_cut_sets

pytestmark = pytest.mark.gpu
MIB = 1 << 20
ALG = "lion"


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
def sms(torch_cuda):
    return torch_cuda.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return ls.build_model(tmp_path_factory.mktemp("lion_walk"))


# (plan, seed): the 52 MiB stream gives the chunk-map passes 1056 runs (8 per SM of 132); streams at p_pred 0 .. 0.99, a copy-mode
# stream, the automaton driven into every reachable state, and a MAP with one byte left in the tail (malformed). Both parities of the
# main loop's block count.
PLANS = {
    "lion52": ({"nbytes": 52 * MIB, "p_pred": 0.2, "cuts": (0.3, 0.6), "odd": True, "tail": (45, "raw1")}, 61),
    "lion3_p0": ({"nbytes": 3 * MIB, "p_pred": 0.0, "cuts": tuple(k / 41 for k in range(1, 41)), "odd": False, "tail": (64, "clean")}, 62),
    "lion3_p5": ({"nbytes": 3 * MIB, "p_pred": 0.5, "cuts": tuple(k / 10 for k in range(1, 10)), "odd": True, "tail": (20, "raw2")}, 63),
    "lion2_p9": ({"nbytes": 2 * MIB, "p_pred": 0.9, "cuts": (0.3, 0.6), "odd": False, "tail": (40, "plain_end")}, 64),
    "lion2_p99": ({"nbytes": 2 * MIB, "p_pred": 0.99, "cuts": (0.5,), "odd": True, "tail": (13, "raw1")}, 65),
    "lion3_copy": ({"nbytes": 3 * MIB, "p_pred": 0.3, "quiet": False, "copy_every": 97, "cuts": (0.33, 0.66), "tail": (31, "raw3")}, 66),
    "lion_prot": ({"nbytes": 2 * MIB, "p_pred": 0.3, "quiet": False, "prot_states": True, "cuts": (0.2, 0.4, 0.6, 0.8),
                   "tail": (22, "clean")}, 67),
    "lion_bad": ({"nbytes": 200000, "p_pred": 0.5, "tail": (9, "map1")}, 68),
}
MALFORMED = ("lion_bad",)
QUIET = ("lion52", "lion3_p0", "lion3_p5", "lion2_p9", "lion2_p99")
_cache = {}


def case(name):
    """(stream, manifest, oracle output at an unbounded capacity)"""
    if name not in _cache:
        plan, seed = PLANS[name]
        s, m = ss.build(ALG, plan, seed)
        _cache[name] = (s, m, oracle.decode(ALG, s, 64 * s.size + 4096))
    return _cache[name]


def size_of(name):
    s, m, full = case(name)
    return full.size if full.size else m["decoded_size"]


def stats(lib):
    c = (ctypes.c_uint64 * 4)()
    assert lib.density_b200_lion_decode_stats(c) == 0
    return tuple(c)


def test_streams_carry_their_classes_on_the_decoders_seams(sms):
    """every class on every placement, the planted values where the oracle decodes them, the chunk-map runs the decoder picks for each
    stream, 1056 of them (or 8 per SM) on the large one, and main loops of both parities"""
    for name in PLANS:
        s, m, full = case(name)
        assert (full.size == 0) == (name in MALFORMED), name
        out = full if full.size else oracle.decode(ALG, s[:m["tail_off"]], 64 * s.size)
        assert out.size == m["decoded_size"], name
        q = out[:m["main_blocks"] * 64].view("<u4")
        for cls, b, qi, want in m["classes"]:
            assert want is None or int(q[qi]) == want, (name, cls, qi)
        assert ss.lion_dec_runs(s.size, m["main_blocks"], sms) == m["run_blocks"], name
    on, _ = lion_coverage([case(n)[:2] for n in PLANS])
    for k in ss.LION_PLACES:
        assert set(ss.LION_CLASSES) <= on[k], (k, set(ss.LION_CLASSES) - on[k])
    assert len(case("lion52")[1]["run_blocks"]) == min(sms * 8, 1056)
    assert {case(n)[1]["main_blocks"] % 2 for n in PLANS} == {0, 1}


# ---- single device ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(PLANS))
def test_paths(torch_cuda, lib, model, name):
    """paths 0 and 1 and decode_device at the decoded size, one byte and one block short and a capacity inside a chunk-map run; path 3 on
    the streams of 4 MiB or less. At the decoded size the walk's counts are the CPU model's and lion_streams.walk_counts'."""
    s, m, full = case(name)
    size = size_of(name)
    for cap in caps_of(ALG, size, m):
        want = oracle.decode(ALG, s, cap)
        for path in ((0, 1, None) if s.size > 4 * MIB else (0, 1, 3, None)):
            rc, got_m, got, tail = dev_decode(torch_cuda, lib, ALG, s, cap, path)
            assert rc == 0 and (tail == CANARY).all(), (name, cap, path)
            check(got_m, got, want, f"{name} cap {cap} path {path}")
            if path == 1 and cap == size and full.size:
                assert stats(lib) == ls.run_model(model, s, cap)[2] == ls.walk_counts(s, full), name


def test_reference_symbols_host_and_device(torch_cuda, lib):
    torch = torch_cuda
    for name in ("lion3_p5", "lion2_p99", "lion_bad"):
        s, m, full = case(name)
        size = full.size if full.size else 1 << 20
        out = np.full(size + 64, CANARY, np.uint8)
        n = lib.lion_decode(s.ctypes.data, s.size, out.ctypes.data, size)
        assert n == full.size and (out[:n] == full).all() and (out[size:] == CANARY).all(), name
        d_in = torch.from_numpy(s).cuda()
        d_out = torch.full((size + 64,), CANARY, dtype=torch.uint8, device="cuda")
        n = lib.lion_decode(ctypes.c_void_p(d_in.data_ptr()), s.size, ctypes.c_void_p(d_out.data_ptr()), size)
        got = d_out.cpu().numpy()
        assert n == full.size and (got[:n] == full).all() and (got[size:] == CANARY).all(), name


# ---- sharded, known cuts ------------------------------------------------------------------------------------------------------------------
def run_cuts(torch, lib, name, prot):
    s, m, full = case(name)
    n = 0
    for cuts in lion_cut_sets(m):
        pieces, caps = pieces_at(ALG, s, m, cuts, full)
        flags, total, outs = decode_lion_pieces(torch, lib, pieces, [max(c, 4) for c in caps], prot=prot)[:3]
        assert flags == 0, (name, prot, cuts)
        cat = np.concatenate(outs)
        check(cat.size, cat, full, f"{name} prot {prot} cuts {cuts}")
        n += 1
    return n


@pytest.mark.parametrize("name", QUIET)
def test_sharded_known_cuts_plain(torch_cuda, lib, name):
    """the plain piece path at the manifest's cuts, a chunk-map run seam, each side of a planted class, odd blocks (the piece's rows shift
    by one block), one-block and empty pieces: every cut set is accepted and exact"""
    assert run_cuts(torch_cuda, lib, name, False) >= 5


@pytest.mark.parametrize("name", ["lion3_p5", "lion3_copy", "lion_prot"])
def test_sharded_known_cuts_protected(torch_cuda, lib, name):
    """the protected piece path at the same cuts and, on the copy-mode streams, behind copy-mode episodes and at automaton targets"""
    assert run_cuts(torch_cuda, lib, name, True) >= 5


# ---- NCCL drivers through the loopback collective library -----------------------------------------------------------------------------
@pytest.mark.parametrize("prot", [False, True])
@pytest.mark.parametrize("world", [2, 5, 8])
def test_drivers_loopback(env, world, prot):  # noqa: F811
    """density_b200_decode_sharded_lion and _protected at W ranks on one stream cut at planted blocks"""
    name = "lion3_copy" if prot else "lion3_p5"
    s, m, full = case(name)
    planted = sorted({b for _, b, _, _ in m["classes"] if 0 < b < m["main_blocks"]})
    cuts = sorted({planted[(k * len(planted)) // world] for k in range(1, world)})
    pieces, caps = pieces_at(ALG, s, m, cuts, full)
    flags, total, outs = loopback_decode(env, pieces, [max(c, 4) for c in caps], prot)
    assert flags == 0 and total == full.size, (world, prot, cuts)
    cat = np.concatenate(outs)
    check(cat.size, cat, full, f"{name} W {world}")
