"""density_b200_cheetah_locate_piece (host only, no GPU): on the Cheetah range maps of a numpy model, every rank's piece starts at the
first block start at or after its range start, as an exact walk of the whole stream (copy-mode blocks included) finds it; layouts
that break the rules are refused on every rank."""
import ctypes

import numpy as np
import pytest

import oracle
import planted
from locate_model import layout
from locate_model_cheetah import HALO, NCAND, RANGE, TERM, WORDS, exact_walk, expected_piece, model_maps, quiet_after

EARG = 4


def _text(n):
    from density_b200 import synth
    return synth.synth_text(n).numpy()


STREAMS = {
    "dickens": lambda d: oracle.encode("cheetah", d),
    "text": lambda d: oracle.encode("cheetah", _text(3 * (1 << 20) + 5)),
    "zeros": lambda d: oracle.encode("cheetah", np.zeros(1 << 20, np.uint8)),
    "cl1": lambda d: oracle.encode("cheetah", planted.corpus("cl1")[0]),
}
_cache = {}


@pytest.fixture(params=sorted(STREAMS))
def stream(request, dickens200k):
    name = request.param
    if name not in _cache:
        s = STREAMS[name](dickens200k)
        starts, copied, tail = exact_walk(s)
        assert quiet_after(copied, starts, RANGE), "copy mode behind the first range: the candidate rows would not be the true walk"
        _cache[name] = (s, starts, tail)
    return _cache[name]


def check_layout(stream, starts, tail, lay):
    from density_b200 import sharded
    maps = model_maps(stream, lay)
    total = stream.size
    prev_end = 0
    for r, (o, n, h) in enumerate(lay):
        got = sharded.locate_piece(maps, r, alg="cheetah")
        assert got == expected_piece(starts, tail, total, o, n), f"rank {r} of {lay}"
        if got[1] > got[0]:                       # the pieces tile the stream
            assert o + got[0] == prev_end
            prev_end = o + got[1]
    assert prev_end == total
    assert sum(sharded.locate_piece(maps, r, alg="cheetah")[4] for r in range(len(lay))) == (1 if total and any(n for _, n, _ in lay) else 0)


def test_model_start_row_is_the_exact_walk(stream):
    """The start row of a range that ends inside the cold-start copy region (ranges of any length are allowed to the kernel): its exit
    and block count are those of the exact walk, copy-mode blocks counted."""
    from locate_model_cheetah import range_map
    s, starts, _ = stream
    for n_range in (2048, 4096, 6400, RANGE):
        m = range_map(s[:n_range + HALO], n_range, HALO, 0)
        k = int(np.searchsorted(starts, n_range))
        assert m[3 + 2 * NCAND] == 1 and m[4 + 2 * NCAND] == (starts[k] - n_range) // 2 and m[5 + 2 * NCAND] == k
        assert m[2:2 + 2 * NCAND:2].tolist() == list(range(NCAND)) and not m[3:3 + 2 * NCAND:2].any()


@pytest.mark.parametrize("world", range(1, 10))
def test_stream_ranges_pieces(stream, world):
    from density_b200 import sharded
    s, starts, tail = stream
    check_layout(s, starts, tail, sharded.stream_ranges(s.size, world))


def test_zero_length_middle_ranges(stream):
    s, starts, tail = stream
    a = max(1, s.size // RANGE // 3) * RANGE
    if 2 * a >= s.size:
        pytest.skip("stream shorter than three ranges")
    check_layout(s, starts, tail, layout(s.size, [a, 0, 0, a, 0, s.size - 2 * a]))
    check_layout(s, starts, tail, layout(s.size, [0, a, 0, s.size - a]))      # the start row on rank 1
    check_layout(s, starts, tail, layout(s.size, [0, 0, 0, s.size]))          # and on the last rank, which holds the whole stream


@pytest.mark.parametrize("last", [1, 2, 100, 263])
def test_last_range_shorter_than_a_block(stream, last):
    """The stream cut short so that the last range is `last` bytes: the walk of the rank before may end inside its halo."""
    s, _, _ = stream
    k = min(s.size // RANGE - 1, 10)
    if k < 1:
        pytest.skip("stream too short")
    t = s[:k * RANGE + last]
    starts, _, tail = exact_walk(t)
    check_layout(t, starts, tail, layout(t.size, [RANGE * (k // 2 + 1), RANGE * (k - k // 2 - 1), last]))
    check_layout(t, starts, tail, layout(t.size, [RANGE * k, last]))


def test_stream_ends_inside_a_halo(stream):
    """Every cut of the last 600 bytes, the start range included: the stream often ends inside the halo of the rank before, and the
    last pieces are empty."""
    s, _, _ = stream
    for k in (1, min(s.size // RANGE - 1, 4)):
        for extra in range(2, 600, 22):
            t = s[:k * RANGE + extra]
            starts, _, tail = exact_walk(t)
            check_layout(t, starts, tail, layout(t.size, [k * RANGE, 0, extra]) if extra < HALO else layout(t.size, [k * RANGE, extra]))


@pytest.mark.parametrize("n", [0, 1, 8, 100, 263])
def test_stream_shorter_than_a_block_world4(stream, n):
    """stream_ranges of a stream shorter than 16 KiB at world 4: ranks 0-2 are empty, the start row is on rank 3."""
    from density_b200 import sharded
    t = stream[0][:n]
    starts, _, tail = exact_walk(t)
    lay = sharded.stream_ranges(n, 4)
    assert all(r == 0 for _, r, _ in lay[:3])
    check_layout(t, starts, tail, lay)
    if n:
        assert sharded.locate_piece(model_maps(t, lay), 3, alg="cheetah")[4] == 1


def test_range_start_on_a_block_start():
    """A block starts exactly on a range start (zeros: 8-byte blocks), so a block of the rank before ends exactly at its range end."""
    s = oracle.encode("cheetah", np.zeros(1 << 20, np.uint8))
    starts, _, tail = exact_walk(s)
    assert (starts == 2 * RANGE).any() and (starts == 3 * RANGE).any()
    check_layout(s, starts, tail, layout(s.size, [2 * RANGE, RANGE, s.size - 3 * RANGE]))


@pytest.mark.parametrize("bad", ["offset", "range_not_chunk_multiple", "halo", "exit_index", "start_exit_index", "start_row_missing",
                                 "start_row_on_wrong_rank", "start_row_twice"])
def test_bad_layouts_are_refused(bad):
    from density_b200 import _lib
    s = oracle.encode("cheetah", _text(1 << 20))
    lay = layout(s.size, [0, 2 * RANGE, 3 * RANGE, s.size - 5 * RANGE])
    maps = model_maps(s, lay)
    S = 2 + 2 * NCAND
    if bad == "offset":
        maps[2][S] += 2
    elif bad == "range_not_chunk_multiple":
        maps[1][0] += 2
    elif bad == "halo":
        maps[2][1] = HALO - 2
    elif bad == "exit_index":
        maps[2][2 + 2 * 7] = NCAND
    elif bad == "start_exit_index":
        maps[1][S + 2] = NCAND
    elif bad == "start_row_missing":
        maps[1][S + 1] = 0
    elif bad == "start_row_on_wrong_rank":
        maps[1][S + 1] = 0
        maps[2][S + 1] = 1
    else:
        maps[0][S + 1] = 1
    lib = _lib.load()
    out = (ctypes.c_uint64 * 5)()
    m = np.ascontiguousarray(maps)
    for r in range(len(lay)):
        assert lib.density_b200_cheetah_locate_piece(m.ctypes.data, len(lay), r, out) == EARG, r
    assert lib.density_b200_cheetah_locate_piece(m.ctypes.data, len(lay), len(lay), out) == EARG
    assert lib.density_b200_cheetah_locate_piece(None, len(lay), 0, out) == EARG
    assert lib.density_b200_cheetah_locate_piece(m.ctypes.data, len(lay), 0, None) == EARG


def test_term_start_row_ends_the_stream():
    """A TERM start row: the start piece runs to the end of its halo, and every later piece is empty behind the stream end."""
    from density_b200 import sharded
    total = RANGE + 100
    maps = np.zeros((3, WORDS), np.uint64)
    for r, (o, n, h) in enumerate(layout(total, [RANGE, 0, 100])):
        maps[r][0], maps[r][1], maps[r][2 + 2 * NCAND] = n, h, o
        maps[r][2:2 + 2 * NCAND:2] = np.arange(NCAND, dtype=np.uint64)
        maps[r][3:2 + 2 * NCAND:2] = 7
    S = 2 + 2 * NCAND
    maps[0][S + 1], maps[0][S + 2], maps[0][S + 3] = 1, TERM, 9
    assert sharded.locate_piece(maps, 0, alg="cheetah") == (0, RANGE + 100, 0, 1, 1)
    assert sharded.locate_piece(maps, 1, alg="cheetah") == (0, 0, 9, 1, 0)
    assert sharded.locate_piece(maps, 2, alg="cheetah") == (0, 0, 9, 1, 0)
    maps[0][S + 2] = 5                                   # an exit into rank 2 (rank 1 is empty): rank 2 starts 10 bytes in
    maps[2][2 + 2 * 5] = TERM
    assert sharded.locate_piece(maps, 0, alg="cheetah") == (0, RANGE + 10, 0, 0, 1)
    assert sharded.locate_piece(maps, 2, alg="cheetah") == (10, 100, 9, 1, 0)
