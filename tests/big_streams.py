"""Corpora whose compressed stream is longer than 2^32 bytes, and the oracle stream of them (numpy + the CPU oracle).

Text compresses too well to reach 2^32 bytes of stream at a size that fits on one GPU, and noise is copied raw by the protection
automaton. The pair corpus sits in between: the input is a sequence of pairs of blocks (256 / 128 / 64 bytes for Chameleon / Cheetah
/ Lion),

    A  fresh splitmix64 quads: every quad misses, the block is incompressible (signature + the block, raw)
    B  its first half repeats the first half of the A block LAG pairs earlier (of its own pair for the first LAG pairs), read from a
       tile of the encoders that lies before the block's own; its second half repeats the second half of its own pair's A block.
       Dictionary and prediction hits: compressible, and still compressible when the earlier A block was never encoded

so no two incompressible blocks are adjacent, the automaton never enters copy mode and the fast paths run end to end. Every A block
holds fresh values, so a byte written at the wrong offset, or a dictionary entry read from the wrong bucket, changes the output.
With `bursts` three 1 MiB stretches of noise in the last 3 * 64 MiB of the input put copy-mode blocks (and with them the copy-map
iteration of the encoders and the copy-aware boundary walk of the decoders) at block indices above 2^24 and stream offsets above 2^32
for the sizes in SIZE. A copy-mode block does not enter the dictionary, so a B block that repeated a copied A block whole would miss,
sit next to an incompressible A block and start copy mode again LAG pairs later: the episode would run on to the end of the input.
The half a B block takes from its own pair keeps it compressible, so an episode ends within a few hundred blocks of its burst.

Everything depends on (alg, nbytes, seed, bursts) alone, and `fill` builds any byte range without the bytes before it.
"""
import concurrent.futures
import ctypes
import os

import numpy as np

import oracle

BLOCK = {"chameleon": 256, "cheetah": 128, "lion": 64}
LAG = 37                                          # pairs between a B block and the A block it repeats (> 32 pairs: a 16 KiB tile)
BURST = 1 << 20
BURST_GAP = 64 << 20                              # burst starts: 3, 2 and 1 gaps before the end (at most a 40th of the input each)
BURST_SEED = 0x5EED_B0B5
GIB = 1 << 30
# stream bytes per input byte of the pair corpus (the oracle on 64 MiB), and input sizes whose stream is longer than STREAM_MIN
RATIO = {"chameleon": 0.788, "cheetah": 0.581, "lion": 0.625}
SIZE = {"chameleon": 11 * GIB // 2 + 5, "cheetah": 15 * GIB // 2 + 5, "lion": 7 * GIB + 5}
STREAM_MIN = (1 << 32) + (1 << 28)
PIECE = 64 << 20


def _splitmix(idx, seed):
    """splitmix64 of the counters idx (uint64 array), in place where it can."""
    with np.errstate(over="ignore"):
        z = idx * np.uint64(0x9E3779B97F4A7C15)
        z += np.uint64(seed)
        z ^= z >> np.uint64(30)
        z *= np.uint64(0xBF58476D1CE4E5B9)
        z ^= z >> np.uint64(27)
        z *= np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
    return z


def burst_ranges(alg, nbytes):
    """[(start, end)] byte ranges of the noise bursts of the bursts variant."""
    B, gap = BLOCK[alg], min(BURST_GAP, nbytes // 40)
    out = []
    for k in (3, 2, 1):
        s = max(0, nbytes - k * gap) // B * B
        out.append((s, min(s + BURST, nbytes)))
    return out


def fill(alg, nbytes, seed, bursts, out, lo):
    """Write bytes [lo, lo + out.size) of the corpus into out (uint8)."""
    B = BLOCK[alg]
    P = 2 * B
    hi = lo + out.size
    assert 0 <= lo <= hi <= nbytes
    if lo == hi:
        return out
    p0, p1 = lo // P, -(-hi // P)
    e0 = max(0, p0 - LAG)
    w = B // 8
    a = _splitmix(np.arange(e0 * w, p1 * w, dtype=np.uint64), seed).view(np.uint8).reshape(p1 - e0, B)
    k = np.arange(p0, p1)
    pairs = np.empty((p1 - p0, 2, B), np.uint8)
    pairs[:, 0] = a[p0 - e0:]
    pairs[:, 1, :B // 2] = a[np.where(k >= LAG, k - LAG, k) - e0, :B // 2]
    pairs[:, 1, B // 2:] = a[p0 - e0:, B // 2:]
    flat = pairs.reshape(-1)
    base = p0 * P
    if bursts:
        for s, e in burst_ranges(alg, nbytes):
            s2, e2 = max(s, base), min(e, p1 * P)
            if s2 < e2:
                noise = _splitmix(np.arange(s2 // 8, -(-e2 // 8), dtype=np.uint64), seed ^ BURST_SEED).view(np.uint8)
                flat[s2 - base:e2 - base] = noise[s2 % 8:s2 % 8 + e2 - s2]
    out[:] = flat[lo - base:hi - base]
    return out


def corpus(alg, nbytes, seed=0, bursts=False):
    """The whole corpus of nbytes, built PIECE bytes at a time (bounded temporaries) on up to 8 threads (numpy releases the GIL)."""
    out = np.empty(nbytes, np.uint8)
    with concurrent.futures.ThreadPoolExecutor(min(8, os.cpu_count() or 1)) as ex:
        list(ex.map(lambda lo: fill(alg, nbytes, seed, bursts, out[lo:lo + PIECE], lo), range(0, nbytes, PIECE)))
    return out


def first_difference(got, want, step=1 << 28):
    """None if got and want (both numpy arrays or both 1-D torch tensors) are equal, else the first offset at which they differ (the
    shorter length when one is a prefix of the other). Compared step bytes at a time, so the temporaries stay small."""
    n = min(got.shape[0], want.shape[0])
    for lo in range(0, n, step):
        a, b = got[lo:lo + step], want[lo:lo + step]
        if isinstance(a, np.ndarray):
            if not np.array_equal(a, b):
                return lo + int(np.argmax(a != b))
        elif not bool(a.equal(b)):
            return lo + int((a != b).to(dtype=a.dtype).argmax())
    return None if got.shape[0] == want.shape[0] else n


def oracle_encode_into(alg, data, out):
    """The oracle's stream of data, written straight into the preallocated uint8 buffer out (oracle.encode keeps a second copy).
    Returns (stream bytes, copy-mode blocks); the stream bytes are 0 when out is too small."""
    copied = ctypes.c_uint64(0)
    n = oracle.lib().oracle_encode_stats(oracle.ALGS[alg], data.ctypes.data, data.size, out.ctypes.data, out.size, ctypes.byref(copied))
    return n, copied.value


def oracle_stream(alg, data):
    """(stream, copy-mode blocks): the oracle's stream of data, a view of a buffer of the safe encode size whose pages past the
    stream are never touched."""
    out = np.empty(oracle.safe_encode_buffer_size(alg, data.size), np.uint8)
    m, copied = oracle_encode_into(alg, data, out)
    assert m > 0
    return out[:m], copied
