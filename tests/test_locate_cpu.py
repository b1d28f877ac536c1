"""density_b200_locate_piece (host only, no GPU): on the range maps of a numpy model, every rank's piece starts at the first block
start at or after its range start, as a brute-force walk of the whole stream finds it; layouts that break the rules are refused."""
import numpy as np
import pytest

import oracle
import planted
from locate_model import CH, HALO, TERM, WORDS, aligned_block_start, expected_piece, layout, model_maps, stream_blocks

EARG = 4


def _text(n):
    from density_b200 import synth
    return synth.synth_text(n).numpy()


STREAMS = {
    "dickens": lambda d: oracle.encode("chameleon", d),
    "text": lambda d: oracle.encode("chameleon", _text(3 * (1 << 20) + 5)),
    "zeros": lambda d: oracle.encode("chameleon", np.zeros(1 << 20, np.uint8)),
    **{q: (lambda d, q=q: oracle.encode("chameleon", planted.corpus(q)[0])) for q in planted.QUIET},
}
_cache = {}


@pytest.fixture(params=sorted(STREAMS))
def stream(request, dickens200k):
    name = request.param
    if name not in _cache:
        s = STREAMS[name](dickens200k)
        _cache[name] = (s,) + stream_blocks(s)
    return _cache[name]


def check_layout(stream, starts, tail, lay):
    from density_b200 import sharded
    maps = model_maps(stream, lay)
    total = stream.size
    prev_end = 0
    for r, (o, n, h) in enumerate(lay):
        got = sharded.locate_piece(maps, r)
        assert got == expected_piece(starts, tail, total, o, n, h), f"rank {r} of {lay}"
        if got[1] > got[0]:                       # the pieces tile the stream
            assert o + got[0] == prev_end
            prev_end = o + got[1]
    assert prev_end == total


def test_stream_ranges():
    from density_b200 import sharded
    for total in (0, 1, 263, 264, CH, 5 * CH + 7, 10 ** 7):
        for world in range(1, 10):
            lay = sharded.stream_ranges(total, world)
            assert lay == layout(total, [n for _, n, _ in lay])
            assert all(n % CH == 0 for _, n, _ in lay[:-1])


def test_model_identity_on_empty_range():
    m = model_maps(np.zeros(100, np.uint8), [(0, 0, 100)])[0]
    assert m[2::2].tolist() == list(range(132)) and not m[3::2].any()


@pytest.mark.parametrize("world", range(1, 10))
def test_stream_ranges_pieces(stream, world):
    from density_b200 import sharded
    s, starts, tail = stream
    if s.size > (32 << 20) and world not in (2, 9):
        pytest.skip("large corpus: two worlds suffice")
    check_layout(s, starts, tail, sharded.stream_ranges(s.size, world))


def test_zero_length_middle_ranges(stream):
    s, starts, tail = stream
    a = max(1, s.size // CH // 3) * CH
    if 2 * a >= s.size:
        pytest.skip("stream shorter than three chunks")
    check_layout(s, starts, tail, layout(s.size, [a, 0, 0, a, 0, s.size - 2 * a]))
    check_layout(s, starts, tail, layout(s.size, [0, a, 0, s.size - a]))


@pytest.mark.parametrize("last", [1, 2, 100, 263])
def test_last_range_shorter_than_a_block(stream, last):
    """The stream cut short so that the last range is `last` bytes: the walk of the rank before may end inside its halo."""
    s, _, _ = stream
    k = min(s.size // CH - 1, 40)           # a prefix of a stream is a stream: the large corpora need not be walked whole each time
    if k < 1:
        pytest.skip("stream too short")
    t = s[:k * CH + last]
    starts, tail = stream_blocks(t)
    check_layout(t, starts, tail, layout(t.size, [CH * (k // 2), CH * (k - k // 2), last]))


@pytest.mark.parametrize("n", [0, 1, 8, 100, 263])
def test_stream_shorter_than_a_block_world4(stream, n):
    from density_b200 import sharded
    t = stream[0][:n]
    starts, tail = stream_blocks(t)
    check_layout(t, starts, tail, sharded.stream_ranges(n, 4))


def test_stream_ends_inside_a_halo(stream):
    """Every cut of the last 600 bytes: the stream often ends inside the halo of the rank before, and the last pieces are empty."""
    s, _, _ = stream
    k = min(s.size // CH - 1, 40)           # a prefix of a stream is a stream: the large corpora need not be walked whole each time
    if k < 1:
        pytest.skip("stream too short")
    for extra in range(2, 600, 22):
        t = s[:k * CH + extra]
        starts, tail = stream_blocks(t)
        check_layout(t, starts, tail, layout(t.size, [k * CH, 0, extra]) if extra < HALO else layout(t.size, [k * CH, extra]))


def test_range_start_on_a_block_start():
    """A block starts exactly on a range start, so a block of the rank before ends exactly at its range end (zeros: 136-byte blocks,
    every 17th chunk boundary)."""
    s = oracle.encode("chameleon", np.zeros(3 << 20, np.uint8))
    starts, tail = stream_blocks(s)
    b = aligned_block_start(starts)
    assert b is not None
    check_layout(s, starts, tail, layout(s.size, [b, s.size - b]))
    check_layout(s, starts, tail, layout(s.size, [b - CH, CH, 0, s.size - b]))


@pytest.mark.parametrize("bad", ["range_not_chunk_multiple", "halo_too_long", "halo_inconsistent", "halo_short", "exit_index"])
def test_bad_layouts_are_refused(bad):
    from density_b200 import _lib
    s = oracle.encode("chameleon", _text(1 << 20))
    lay = layout(s.size, [2 * CH, 3 * CH, s.size - 5 * CH])
    maps = model_maps(s, lay)
    if bad == "range_not_chunk_multiple":
        maps[0][0] += 2
    elif bad == "halo_too_long":
        maps[1][1] = HALO + 2
    elif bad == "halo_inconsistent":
        maps[2][1] = 2                          # the last rank has no halo
    elif bad == "halo_short":
        maps[0][1] = HALO - 2
    else:
        maps[1][2 + 2 * 7] = 132
    lib = _lib.load()
    out = (__import__("ctypes").c_uint64 * 4)()
    m = np.ascontiguousarray(maps)
    for r in range(3):
        assert lib.density_b200_locate_piece(m.ctypes.data, 3, r, out) == EARG
    assert lib.density_b200_locate_piece(m.ctypes.data, 3, 3, out) == EARG
    assert lib.density_b200_locate_piece(None, 3, 0, out) == EARG


def test_term_row_ends_the_stream():
    """A TERM row in a rank's map: its piece runs to the end of its halo, and every later piece is empty behind the stream end."""
    from density_b200 import sharded
    total = 2 * CH + 100
    maps = np.zeros((3, WORDS), np.uint64)
    for r, (o, n, h) in enumerate(layout(total, [CH, CH, 100])):
        maps[r][0], maps[r][1] = n, h
        maps[r][2::2] = np.arange(132, dtype=np.uint64)
        maps[r][3::2] = 7
    maps[1][2 + 2 * 3] = TERM
    maps[0][2] = 3
    assert sharded.locate_piece(maps, 0) == (0, CH + 6, 0, 0)
    assert sharded.locate_piece(maps, 1) == (6, CH + 100, 7, 1)
    assert sharded.locate_piece(maps, 2) == (0, 0, 14, 1)
