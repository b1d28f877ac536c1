"""Numpy model of the Cheetah range maps of density_b200_cheetah_decode_locate and an exact block walk of a whole Cheetah stream.

Candidate rows take every block as an encoded block (8 + 4 * plain + 2 * map bytes from the 2-bit signature, cld::cheetah_block_bytes),
as the candidate walks of the boundary kernels do. The start row and the whole-stream walk run codec.rs's main loop with the protection
automaton (tests/protection.py), copy-mode blocks taken as 128 raw bytes."""
import numpy as np

from protection import Protection

CH, HALO, NCAND, WORDS = 4096, 264, 68, 142     # boundary-walk chunk, halo of the layout, candidates, u64 per map
RANGE = 16384                                    # non-last ranges are multiples of this
MAXBLK, BS = 136, 128
TERM = (1 << 64) - 1
M55 = 0x5555555555555555


def block_bytes(buf, p):
    sig = int.from_bytes(buf[p:p + 8].tobytes(), "little")
    lo, hi = sig & M55, (sig >> 1) & M55
    return 8 + 4 * (~(lo | hi) & M55).bit_count() + 2 * (lo ^ hi).bit_count()


def candidate_rows(buf, n_range, n_halo):
    """[(exit or TERM, blocks)] of the 68 candidate entries of buf[0 .. n_range + n_halo): a walk leaves the range at the first block start
    >= ceil(n_range / CH) * CH, and stops (TERM) at the first block with fewer than 136 bytes left."""
    n = n_range + n_halo
    lim = -(-n_range // CH) * CH
    known, rows = {}, []
    for c in range(NCAND):
        path, p = [], 2 * c
        while True:
            if p in known:
                ex, nb = known[p]
                break
            if p >= lim:
                ex, nb = (p - lim) // 2, 0
                break
            if p + MAXBLK > n:
                ex, nb = TERM, 0
                break
            path.append(p)
            p += block_bytes(buf, p)
        for k, q in enumerate(reversed(path)):
            known[q] = (ex, nb + k + 1)
        rows.append((ex, nb + len(path)))
    return rows


def exact_walk(buf):
    """Main-loop block starts of a whole stream (codec.rs:88-100 with protection_state.rs: at least 136 bytes left; copy-mode blocks
    are 128 raw bytes), whether each is copied, and the offset where the tail starts."""
    n, ps, p = buf.size, Protection(), 0
    starts, copied = [], []
    while p + MAXBLK <= n:
        starts.append(p)
        probe = Protection(ps.penalty, ps.start, ps.prev, ps.counter)
        if probe.step(False):                       # copy mode does not depend on the block's own bit
            ps.step(False)
            copied.append(True)
            p += BS
        else:
            s = block_bytes(buf, p)
            ps.step(s >= BS)
            copied.append(False)
            p += s
    return np.array(starts, np.int64), np.array(copied, bool), p


def start_row(buf, n_range, n_halo):
    """(exit or TERM, blocks) of the exact walk of buf[0 .. n_range + n_halo) from the stream start, read off at n_range."""
    starts, _, tail = exact_walk(buf[:n_range + n_halo])
    k = int(np.searchsorted(starts, n_range))
    if k < starts.size:
        return (int(starts[k]) - n_range) // 2, k
    if tail >= n_range:
        return (tail - n_range) // 2, k
    return TERM, k


def range_map(buf, n_range, n_halo, range_offset):
    m = np.zeros(WORDS, np.uint64)
    m[0], m[1], m[2 + 2 * NCAND] = n_range, n_halo, range_offset
    if range_offset == 0 and n_range > 0:
        m[2:2 + 2 * NCAND:2] = np.arange(NCAND, dtype=np.uint64)          # the identity: the start range's candidate rows are void
        m[3 + 2 * NCAND] = 1
        m[4 + 2 * NCAND], m[5 + 2 * NCAND] = start_row(buf, n_range, n_halo)
    else:
        for c, (ex, nb) in enumerate(candidate_rows(buf, n_range, n_halo)):
            m[2 + 2 * c], m[3 + 2 * c] = ex, nb
    return m


def model_maps(stream, lay):
    return np.stack([range_map(stream[o:o + n + h], n, h, o) for o, n, h in lay])


def expected_piece(starts, tail, total, off, n_range):
    """(start, end, blocks_before, is_final, is_first) of the range at `off`, from the whole-stream exact walk: the piece runs from the
    first block start at or after the range start to the first one at or after the range end (or to the stream end)."""
    before = int(np.searchsorted(starts, off))
    first = int(off == 0 and n_range > 0)
    if tail < off:
        return 0, 0, len(starts), 1, 0
    if n_range == 0:
        return 0, 0, before, int(off == total), 0
    q = int(starts[before]) if before < len(starts) else tail
    if tail < off + n_range:
        return q - off, total - off, before, 1, first
    k = int(np.searchsorted(starts, off + n_range))
    q2 = int(starts[k]) if k < len(starts) else tail
    return q - off, q2 - off, before, int(q2 == total), first


def quiet_after(copied, starts, off):
    """No copy-mode block starts at or after stream offset `off` (the later ranges' candidate walks are then the true walk)."""
    return not copied[starts >= off].any()
