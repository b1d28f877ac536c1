"""The corpora of tests/big_streams.py at 64 MiB against the oracle (CPU only): the stream ratio the GPU tests size their inputs by,
the copy-mode blocks of each variant, the oracle round trip, and that the generator is deterministic and piecewise."""
import numpy as np
import pytest

import big_streams as bs
import oracle
from protection import trace

N = 64 << 20


@pytest.mark.parametrize("alg", bs.BLOCK)
def test_pair_corpus_ratio_quiet_and_round_trip(alg):
    data = bs.corpus(alg, N + 5)
    stream, copied = bs.oracle_stream(alg, data)
    assert abs(stream.size / data.size - bs.RATIO[alg]) < 0.01, stream.size / data.size
    assert copied == 0
    back = oracle.decode(alg, stream, data.size)
    assert back.size == data.size and np.array_equal(back, data)
    # at the GPU tests' size the ratio puts the stream past STREAM_MIN with room to spare (they assert it on the real stream)
    assert bs.SIZE[alg] * (bs.RATIO[alg] - 0.01) > bs.STREAM_MIN


def test_oracle_encode_into_too_small():
    data = bs.corpus("chameleon", 1 << 20)
    stream, _ = bs.oracle_stream("chameleon", data)
    out = np.empty(stream.size, np.uint8)
    assert bs.oracle_encode_into("chameleon", data, out)[0] == stream.size and np.array_equal(out, stream)
    assert bs.oracle_encode_into("chameleon", data, out[:-1])[0] == 0


def test_bursts_copy_mode_only_in_the_bursts():
    data = bs.corpus("chameleon", N + 5, bursts=True)
    stream, copied = bs.oracle_stream("chameleon", data)
    back = oracle.decode("chameleon", stream, data.size)
    assert back.size == data.size and np.array_equal(back, data)
    pairs = bs.corpus("chameleon", N + 5)
    ranges = bs.burst_ranges("chameleon", data.size)
    inside = np.zeros(data.size, bool)
    for s, e in ranges:
        inside[s:e] = True
        assert e - s == bs.BURST
    assert np.array_equal(data[~inside], pairs[~inside]) and not np.array_equal(data[inside], pairs[inside])
    assert all(e0 < s1 for (_, e0), (s1, _) in zip(ranges, ranges[1:]))
    t = trace("chameleon", stream, data.size)
    assert t.n_stream == stream.size and int(t.copied.sum()) == copied > 0
    blk = np.flatnonzero(t.copied)
    slack = 4 * bs.LAG * 2                            # blocks an episode may run past its burst (see big_streams)
    hit = np.zeros(blk.size, bool)
    for s, e in ranges:
        mine = (blk >= s // 256) & (blk < e // 256 + slack)
        assert mine.sum() > (e - s) // 256 // 2       # most of a burst's blocks are copied
        hit |= mine
    assert hit.all(), blk[~hit][:8]


@pytest.mark.parametrize("alg", bs.BLOCK)
@pytest.mark.parametrize("bursts", [False, True])
def test_generator_deterministic_and_piecewise(alg, bursts):
    n = bs.PIECE + 4099 if alg == "chameleon" else (5 << 20) + 3
    a = bs.corpus(alg, n, seed=5, bursts=bursts)
    assert np.array_equal(a, bs.corpus(alg, n, seed=5, bursts=bursts))
    assert not np.array_equal(a, bs.corpus(alg, n, seed=6, bursts=bursts))
    cuts = [0, 1, 7, 1000, 4096 + 3, n // 3, n // 2 + 5, n - 9, n]
    b = np.empty(n, np.uint8)
    for lo, hi in zip(cuts, cuts[1:]):
        bs.fill(alg, n, 5, bursts, b[lo:hi], lo)
    assert np.array_equal(a, b)
    # the layout: A blocks of fresh quads, B blocks repeating half the A block LAG pairs earlier and half their own, nothing but the bursts differs
    B = bs.BLOCK[alg]
    p = bs.corpus(alg, n, seed=5)
    k = n // (2 * B) - 1
    h = B // 2
    assert np.array_equal(p[(2 * k + 1) * B:(2 * k + 1) * B + h], p[2 * (k - bs.LAG) * B:2 * (k - bs.LAG) * B + h])
    assert np.array_equal(p[(2 * k + 1) * B + h:(2 * k + 2) * B], p[2 * k * B + h:(2 * k + 1) * B])
    assert np.array_equal(p[B:2 * B], p[:B])
    quads = p[:(4 << 20) // (2 * B) * 2 * B].reshape(-1, 2, B)[:, 0].reshape(-1).view(np.uint32)
    assert np.unique(quads).size > 0.999 * quads.size
