"""Numpy model of the range maps of density_b200_decode_locate, a brute-force block walk of a whole Chameleon stream, and the
layouts (range + halo per rank) the locate tests share. Blocks are taken as encoded blocks throughout (264 - 2 * popcount(signature)
bytes), as the candidate walks of the boundary kernels take them."""
import numpy as np

CH, HALO, NCAND, WORDS = 16384, 264, 132, 266
TERM = (1 << 64) - 1


class Sizes:
    """Encoded block size at an offset of a buffer."""

    def __init__(self, buf):
        self.buf = buf

    def __call__(self, p):
        return 264 - 2 * int.from_bytes(self.buf[p:p + 8].tobytes(), "little").bit_count()


def range_map(buf, n_range, n_halo):
    """The range map of buf[0 .. n_range + n_halo) (DENSITY_B200_LOCATE_MAP_WORDS u64), walking every candidate entry: a walk leaves
    the range at the first block start >= ceil(n_range / CH) * CH, and stops (TERM) at the first block with fewer than 264 bytes left."""
    n = n_range + n_halo
    lim = -(-n_range // CH) * CH
    size = Sizes(buf[:n])
    known = {}                               # offset -> (exit, blocks from there): the walks of different entries merge
    m = np.zeros(WORDS, np.uint64)
    m[0], m[1] = n_range, n_halo
    for c in range(NCAND):
        path, p = [], 2 * c
        while True:
            if p in known:
                ex, nb = known[p]
                break
            if p >= lim:
                ex, nb = (p - lim) // 2, 0
                break
            if p + HALO > n:
                ex, nb = TERM, 0
                break
            path.append(p)
            p += size(p)
        for k, q in enumerate(reversed(path)):
            known[q] = (ex, nb + k + 1)
        m[2 + 2 * c], m[3 + 2 * c] = ex, nb + len(path)
    return m


def stream_blocks(stream):
    """Main-loop block starts of a whole stream (codec.rs's main loop: at least 264 bytes left) and the offset where the tail starts."""
    size, starts, p = Sizes(stream), [], 0
    while p + HALO <= stream.size:
        starts.append(p)
        p += size(p)
    return np.array(starts, np.int64), p


def expected_piece(starts, tail, total, off, n_range, n_halo):
    """(start, end, blocks_before, is_final) of the range at `off`, from the whole-stream walk: the piece runs from the first block
    start at or after the range start to the first one at or after the range end (or to the stream end)."""
    before = int(np.searchsorted(starts, off))
    if tail < off:
        return 0, 0, len(starts), 1
    if n_range == 0:
        return 0, 0, before, int(off == total)
    q = int(starts[before]) if before < len(starts) else tail
    if tail < off + n_range:
        return q - off, total - off, before, 1
    k = int(np.searchsorted(starts, off + n_range))
    q2 = int(starts[k]) if k < len(starts) else tail
    return q - off, q2 - off, before, int(q2 == total)


def layout(total, n_ranges):
    """[(offset, n_range, n_halo)] for the given range lengths (which must sum to total)."""
    assert sum(n_ranges) == total
    out, off = [], 0
    for n in n_ranges:
        out.append((off, n, min(HALO, total - off - n)))
        off += n
    return out


def model_maps(stream, lay):
    return np.stack([range_map(stream[o:o + n + h], n, h) for o, n, h in lay])


def aligned_block_start(starts, lo=CH):
    """A main-loop block start (>= lo) on the 16 KiB grid, or None."""
    hit = starts[(starts >= lo) & (starts % CH == 0)]
    return int(hit[0]) if hit.size else None
