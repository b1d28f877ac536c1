"""CPU model of the decode-side protection transfer of a sharded Lion stream (numpy only; the twin of dec_prot_transfer<LionT> in
decode_bounds.cuh).

The head walk, the candidate encoding, the jump rule and the composition are those of prot_decode_model / prot_decode_model_cheetah;
only the geometry differs: the boundary walk's chunks are 4 KiB with 35 candidate entry offsets per chunk row (MAXBLK / 2), a block
decodes to 64 bytes, an encoded block takes at most 70 (6 signature bytes of 16 three-bit flags + 16 quads) and a copy-mode block 64
raw bytes."""
import numpy as np

import prot_decode_model_cheetah as _C
from prot_decode_model import HEAD_CAP, NCAND, NOEND, PROT_ESC, TERM, cand_index, cand_state, compose, sw_jump  # noqa: F401
from protection import CH as _CH, GROUP

CH = _CH["lion"]
BS = 64
SIG = 6
MAXBLK = 70
NC = MAXBLK // 2

# the bytes of the 16 three-bit flags of a Lion signature (flag 0: a 4-byte quad, 1-5: predicted, none, 6 and 7: a 2-byte hash)
_FLAG_BYTES = np.array([4, 0, 0, 0, 0, 0, 2, 2], np.int64)


def consumed_table(s):
    """bytes an encoded Lion block starting at offset o takes (6 + the sum over its 16 flags), for every o; signature bytes past the
    end read as 0"""
    s = np.concatenate([np.asarray(s, np.uint8), np.zeros(SIG, np.uint8)]).astype(np.uint64)
    o = np.arange(s.size - SIG + 1)
    sig = np.zeros(o.size, np.uint64)
    for i in range(SIG):
        sig |= s[o + i] << np.uint64(8 * i)
    total = np.full(o.size, SIG, np.int64)
    for k in range(16):
        total += _FLAG_BYTES[((sig >> np.uint64(3 * k)) & np.uint64(7)).astype(np.int64)]
    return total


class Rows(_C.Rows):
    """dec_chunk_walk<LionT>'s rows and dec_group_compose<LionT>'s group rows of one piece, computed on demand"""

    def __init__(self, cons, n):
        super().__init__(cons, n)
        self.nchunks = (n + CH - 1) // CH

    def chunk_row(self, c, e):
        """(exit index or TERM, blocks, flags {1 pair inside, 2 first incompressible, 4 last incompressible})"""
        key = (c, e)
        if key not in self.chunk:
            base, off, nb, pair, first, prev = c * CH, 2 * e, 0, 0, 0, 0
            while True:
                if off >= CH:
                    r = ((off - CH) >> 1, nb, pair | first << 1 | prev << 2)
                    break
                if base + off + MAXBLK > self.n:
                    r = (TERM, nb, 0)
                    break
                con = int(self.cons[base + off])
                inc = int(con >= BS)
                if nb == 0:
                    first = inc
                pair |= inc & prev
                prev = inc
                off += con
                nb += 1
            self.chunk[key] = r
        return self.chunk[key]


def _step(cons, n, off, st):
    """one block of codec.rs:88-98 (a non-final piece: every block is a main-loop block). None: the block does not fit the piece."""
    pen, start, prev, ph = st
    if ph == 0 and start > 1:
        start >>= 1
    ph = (ph + 1) & 15
    if pen > 0:
        pen = (pen - 1) & 0xFF
        if pen == 0:
            start = (start + 1) & 0xFF
        off += BS
    else:
        if off + SIG > n:
            return None
        con = int(cons[off])
        if con >= BS:
            if prev:
                pen = start
            prev = 1
        else:
            prev = 0
        off += con
    if off > n:
        return None
    return off, (pen, start, prev, ph)


def exact_walk(cons, n, st):
    """the in-order walk of a whole piece from state st: (end state, blocks) when it ends on the cut, else None"""
    off, nb = 0, 0
    while off < n:
        r = _step(cons, n, off, st)
        if r is None:
            return None
        off, st = r
        nb += 1
    return st, nb


def transfer(stream, head_cap=HEAD_CAP):
    """The transfer of a non-final piece (uint8 array) and the walk's statistics, as prot_decode_model_cheetah.transfer on the Lion
    geometry: (int array [NCAND], {"max_live", "heads", "capped"})."""
    s = np.asarray(stream, np.uint8)
    n = s.size
    out = np.full(NCAND, NOEND, np.int64)
    stats = {"max_live": 0, "heads": [], "capped": 0}
    if n == 0:
        out[:] = np.arange(NCAND)
        return out, stats
    cons = consumed_table(s)
    rows = Rows(cons, n)
    heads = {}                            # (offset, pen, start, prev, phase) -> candidates
    for c in range(NCAND):
        heads.setdefault((0,) + cand_state(c), []).append(c)
    for c in range(rows.nchunks):
        nxt = {}
        for key, cands in heads.items():
            off, st = key[0], key[1:]
            if off >= (c + 1) * CH:       # a group jump took it past this chunk
                nxt.setdefault(key, []).extend(cands)
                continue
            pen, start, prev, ph = st
            e = (off - c * CH) >> 1
            ended = None
            jumped = False
            if pen == 0 and c % GROUP == 0:
                ex, nb, fl = rows.group_row(c // GROUP, e)
                if ex != TERM and not (fl & 9) and not (prev and (fl & 2)):
                    start, ph = sw_jump(start, ph, nb)
                    off, st, jumped = (c + GROUP) * CH + 2 * ex, (0, start, (fl >> 2) & 1, ph), True
            if not jumped and pen == 0:
                ex, nb, fl = rows.chunk_row(c, e)
                if ex != TERM and not (fl & 1) and not (prev and (fl & 2)):
                    start, ph = sw_jump(start, ph, nb)
                    off, st, jumped = (c + 1) * CH + 2 * ex, (0, start, (fl >> 2) & 1, ph), True
            if not jumped:
                while off < min((c + 1) * CH, n):
                    r = _step(cons, n, off, st)
                    if r is None:
                        ended = NOEND
                        break
                    off, st = r
            if ended is None and off == n:
                ended = cand_index(*st)
            if ended is not None:
                out[cands] = ended
            else:
                nxt.setdefault((off,) + tuple(st), []).extend(cands)
        heads = nxt
        if head_cap is not None and len(heads) > head_cap:
            for key in list(heads)[head_cap:]:
                out[heads.pop(key)] = NOEND
                stats["capped"] += 1
        stats["heads"].append(len(heads))
        if c > 0 or rows.nchunks == 1:
            stats["max_live"] = max(stats["max_live"], len(heads))
    return out, stats
