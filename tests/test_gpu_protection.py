"""Protection-automaton corpora (tests/protection.py) through every encode and decode path on the GPU (needs an H100: pytest -m gpu).

Every stream is compared byte for byte with oracle.encode and must decode back; every decode writes into exactly n bytes followed by
a canary. Where a corpus is meant for a parallel evaluation of the automaton, the test also checks that it ran rather than a fallback:
the converged copy map of Chameleon path 4, a non-zero size from the Cheetah / Lion run-parallel encoder (path 1), boundaries from
the in-order walk of the parallel Chameleon decoder, a settled Cheetah context iteration."""
import ctypes

import numpy as np
import pytest

import oracle
import protection as P
from test_gpu_planted import CANARY, assert_stream, dev_decode, dev_encode, first_diff

pytestmark = pytest.mark.gpu
MIB = 1 << 20
NAMES = ("seam_states", "chunk_entries", "seam_counts", "thresholds", "tails")
# corpora meant for the parallel automaton: every piece has copy-mode blocks and more than one segment
PARALLEL = ("seam_states", "chunk_entries", "seam_counts", "thresholds")


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


def _pieces(name, alg):
    for piece in P.corpus(name, alg):
        data, enc, tr = P.oracle_stream(name, alg, piece.label)
        yield piece.label, data, enc, tr


def _first_nonquiet(tr):
    """The second block of the first pair of consecutive incompressible blocks that some block follows (the block after it is copied;
    a pair that ends the stream copies nothing, and the stream is still quiet)."""
    k = np.flatnonzero(tr.inc[1:-1] & tr.inc[:-2])
    return int(k[0]) + 1 if k.size else None


def _main_blocks(enc, tr, alg):
    """Blocks of the decoder's main loop (codec.rs:88-100): those with at least SIG + BS stream bytes left."""
    return next((k for k in range(len(tr.off)) if enc.size - tr.off[k] < P.maxblk(alg)), len(tr.off))


def _status(lib, fn, n, ctype=ctypes.c_uint64):
    st = (ctype * n)()
    assert getattr(lib, fn)(st) == 0
    return list(st)


# ---- encode -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("path", [0, 1, 2, 3, 4])
def test_chameleon_encode_paths(torch_cuda, lib, name, path):
    """Paths 0 (auto), 2 (protection-aware walk), 3 (in-order kernel, pieces up to 1 MiB) and 4 (host-resumed iteration: the copy map
    must converge on the corpora meant for it). Path 1 (fast path only) must report the stream as not quiet, with its first
    non-quiet block the second block of the trace's first incompressible pair."""
    torch = torch_cuda
    for label, data, want, tr in _pieces(name, "chameleon"):
        if path == 3 and data.size > MIB:
            continue
        rc, n, got, tail = dev_encode(torch, lib, "chameleon", data, path)
        what = f"{name}/{label} path {path}"
        if path == 1:
            st = _status(lib, "density_b200_encode_status", 6)
            fb = _first_nonquiet(tr)
            if fb is not None:
                assert lib.density_b200_last_encode_was_fast() == 0, what
                assert st[1] == 1 and st[3] == fb, (what, st, fb)
            else:
                assert_stream(rc, n, got, want, what)
            continue
        assert_stream(rc, n, got, want, what)
        assert (tail == CANARY).all(), what
        if path == 4 and name in PARALLEL:
            assert _status(lib, "density_b200_encode_status", 6)[4] == 1, what


def test_chameleon_reference_symbol_device_pointers(torch_cuda, lib):
    torch = torch_cuda
    for name in NAMES:
        for label, data, want, tr in _pieces(name, "chameleon"):
            d_in = torch.from_numpy(data.copy()).cuda()
            cap = oracle.safe_encode_buffer_size("chameleon", data.size)
            d_out = torch.full((cap + 64,), CANARY, dtype=torch.uint8, device="cuda")
            n = lib.chameleon_encode(d_in.data_ptr(), data.size, d_out.data_ptr(), cap)
            out = d_out.cpu().numpy()
            assert n == want.size and (out[:n] == want).all(), (name, label, n, first_diff(out[:n], want))
            assert (out[cap:] == CANARY).all()


@pytest.mark.parametrize("alg", ["cheetah", "lion"])
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("path", [0, 1, 3, 4])
def test_cheetah_lion_encode_paths(torch_cuda, lib, alg, name, path):
    """Paths 0, 1 (run-parallel encoder only: a size of 0 means the copy map did not settle), 3 (in-order kernel, up to 1 MiB) and 4."""
    torch = torch_cuda
    for label, data, want, tr in _pieces(name, alg):
        if path == 3 and data.size > MIB:
            continue
        rc, n, got, tail = dev_encode(torch, lib, alg, data, path)
        what = f"{alg} {name}/{label} path {path}"
        if path == 1 and n == 0:
            pytest.fail(f"{what}: the run-parallel encoder's copy map did not settle")
        assert_stream(rc, n, got, want, what)
        assert (tail == CANARY).all(), what


# ---- decode -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg,path", [("chameleon", 0), ("chameleon", 1), ("chameleon", 3), ("cheetah", 0), ("cheetah", 1),
                                      ("cheetah", 3), ("lion", 0)])
@pytest.mark.parametrize("name", NAMES)
def test_decode_paths(torch_cuda, lib, alg, path, name):
    """Every stream decodes into exactly n bytes with the canary behind them intact. The parallel Chameleon decoder (path 1) must finish
    the stream itself with the boundaries of its in-order walk whenever copy mode starts inside its main loop; the parallel Cheetah decoder
    (path 1) must settle its context iteration."""
    torch = torch_cuda
    for label, data, enc, tr in _pieces(name, alg):
        rc, m, got, tail = dev_decode(torch, lib, alg, enc, data.size, path)
        what = f"{alg} {name}/{label} path {path}"
        assert rc == 0 and m == data.size, (what, rc, m)
        assert (got == data).all(), (what, first_diff(got, data))
        assert (tail == CANARY).all(), f"{what}: wrote past the output"
        h = _main_blocks(enc, tr, alg)
        if path == 1 and alg == "chameleon" and (tr.inc[1:h] & tr.inc[:h - 1]).any():      # copy mode starts in the main loop
            st = _status(lib, "density_b200_decode_status", 10)
            assert st[0] == data.size and st[6] != 0, (what, st)
        if path == 1 and alg == "cheetah":
            assert _status(lib, "density_b200_cheetah_decode_rounds", 4, ctypes.c_uint32)[1] != 0, what


# ---- the host pipeline ------------------------------------------------------------------------------------------------------
def test_pipelined_host_path(torch_cuda, lib):
    """96 MiB + 77 bytes of pageable host memory through chameleon_encode: the pipeline cuts at 64 MiB. An R block on either side of
    the cut keeps every chunk quiet; an R R pair across it needs copy mode and the whole-buffer path."""
    import density_b200
    C = density_b200.Chameleon
    for label, data, want, tr in _pieces("pipelined", "chameleon"):
        out = np.full(C.safe_encode_buffer_size(data.size) + 64, CANARY, dtype=np.uint8)
        n = C.encode(data, out[:-64])
        assert n == want.size and (out[:n] == want).all(), (label, n, first_diff(out[:n], want))
        assert (out[-64:] == CANARY).all()
        back = np.zeros(data.size, np.uint8)
        assert C.decode(want, back) == data.size and (back == data).all(), label


# ---- state carried across calls -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg", P.ALGS)
def test_codec_instance_after_a_piece_that_ends_in_copy_mode(torch_cuda, lib, alg):
    """A CodecInstance piece that ends in copy mode with start > 1, then a piece of text that repeats quads of the first: the protection
    state restarts with every call (codec.rs:75,85) while the dictionary carries over."""
    import density_b200
    from density_b200.codec import CodecInstance
    bld = P.Builder(alg, 80)
    bld.add("Z" * 30)
    b = next(b for b in range(bld.n + 40, bld.n + 60) if (2, 2, 1, b % 16) in P.reachable_states())
    bld.place(b, (2, 2, 1), "end_in_copy")
    bld.add("Z")
    assert bld.state()[0] == 1 and bld.state()[1] == 2
    first, _ = bld.realize()
    second = np.concatenate([first[:P.BS[alg] * 20], P.planted.base_text(50000 + 3)])
    ref, enc, dec = oracle.Codec(alg), CodecInstance(alg), CodecInstance(alg)
    streams = []
    for p in (first, second):
        want = ref.encode(p)
        out = np.zeros(density_b200.CODECS[alg].safe_encode_buffer_size(p.size), dtype=np.uint8)
        n = enc.encode(p, out)
        assert n == want.size and (out[:n] == want).all(), (alg, p.size, first_diff(out[:n], want))
        streams.append(out[:n].copy())
    tr = P.trace(alg, streams[0], first.size)
    assert tr.copied[-1] and tr.state[-1][0] >= 1 and tr.state[-1][1] >= 2
    for p, s in zip((first, second), streams):
        back = np.zeros(p.size, dtype=np.uint8)
        assert dec.decode(s, back) == p.size and (back == p).all()
    enc.close(); dec.close()


# ---- sharded Cheetah / Lion encode on one GPU ---------------------------------------------------------------------------------
def _shard_cases(alg):
    """The first shard ends in penalty 0 with start 2..6 and prev 0 / 1 (prev = 1 both after a copy run and after an encoded R), or with
    a penalty pending; the next shard starts with R or Z. Yields (end, next letter, cut in bytes, builder)."""
    B = P.BS[alg]
    reach = P.reachable_states()
    step = 256 // B                                               # non-final shards are multiples of 256 bytes
    ends = [(0, s, pv) for s in range(2, 7) for pv in (0, 1)] + [("R after", s) for s in range(2, 7)] + ["pending"]
    for end in ends:
        for nxt in "RZ":
            bld = P.Builder(alg, 90)
            bld.add("Z" * 200)
            cut = (bld.n + 60 + 16 * step - 1) // (16 * step) * (16 * step)
            if end == "pending":
                bld.add("Z" * (cut - 2 - bld.n)).add("RR")
            elif end[0] == "R after":                             # (0, s, 0) in front of the last block, an encoded R
                cut = next((k for k in range(cut, cut + 4096, step) if (0, end[1], 0, (k - 1) % 16) in reach), None)
                if cut is None:                                   # start 6 cannot be left by a block at that phase
                    continue
                bld.place(cut - 1, (0, end[1], 0), "shard_end")
                bld.add("R")
            else:
                cut = next(k for k in range(cut, cut + 4096, step) if end + (k % 16,) in reach)
                bld.place(cut, end, "shard_end")
            bld.add(nxt)
            bld.recover()
            bld.add("Z" * 300)
            yield end, nxt, cut * B, bld


@pytest.mark.parametrize("alg", ["cheetah", "lion"])
def test_sharded_cl_encode_seam_states(torch_cuda, lib, alg):
    """The verdict of the phase API equals the header's rule computed from the trace: refused when the first shard ends inside a copy
    run (its last block copied) or with a copy penalty pending, or when the seam joins two incompressible blocks, previous_incompressible
    at the end of the first shard counting as its last block being incompressible; otherwise the concatenation equals one call."""
    from test_gpu_sharded_cl_encode import encode_shards
    torch = torch_cuda
    n_ok = n_refused = 0
    for end, nxt, cut, bld in _shard_cases(alg):
        data, _ = bld.realize()
        want = oracle.encode(alg, data)
        tr = P.trace(alg, want, data.size)
        b = cut // P.BS[alg]
        in_copy = bool(tr.copied[b - 1]) or tr.state[b][0] > 0     # shard 0 ends inside a copy run or with a penalty pending
        joins = bool(tr.state[b][2] and tr.inc[b])     # previous_incompressible survives a copy run: it may end shard 0 set
        later_pair = bool((tr.inc[b + 1:] & tr.inc[b:-1]).any())
        refuse = in_copy or joins or later_pair
        pieces, (flags, total, _), _ = encode_shards(torch, lib, alg, data, [0, cut, data.size])
        assert (flags != 0) == refuse, (alg, end, nxt, flags)
        if not refuse:
            cat = np.concatenate(pieces)
            assert cat.size == want.size and (cat == want).all(), (alg, end, nxt, first_diff(cat, want))
            n_ok += 1
        else:
            n_refused += 1
    assert n_ok > 0 and n_refused > 0
