"""CPU model of the decode-side protection transfer of a sharded Cheetah stream (numpy only; the twin of dec_prot_transfer<CheeT> in
decode_bounds.cuh).

The head walk is prot_decode_model's (the Chameleon twin), whose candidate encoding, jump rule and composition this module reuses; only
the geometry differs: the boundary walk's chunks are 4 KiB with 68 candidate entry offsets per chunk row (MAXBLK / 2), a block decodes
to 128 bytes, an encoded block takes at most 136 (8 signature bytes + 32 quads) and a copy-mode block 128 raw bytes."""
import numpy as np

from prot_decode_model import HEAD_CAP, NCAND, NOEND, PROT_ESC, TERM, cand_index, cand_state, compose, sw_jump  # noqa: F401
from protection import CH as _CH, GROUP

CH = _CH["cheetah"]
BS = 128
MAXBLK = 136
NC = MAXBLK // 2

# the bytes the four 2-bit flags of one signature byte add to an encoded block (flag 0: a 4-byte quad, 1 and 2: a 2-byte hash, 3: none)
_BYTE = np.array([sum((4, 2, 2, 0)[(v >> (2 * k)) & 3] for k in range(4)) for v in range(256)], np.int64)


def consumed_table(s):
    """bytes an encoded Cheetah block starting at offset o takes (8 + the sum over its 32 two-bit flags of {0: 4, 1: 2, 2: 2, 3: 0}), for
    every o; signature bytes past the end read as 0"""
    s = np.asarray(s, np.uint8)
    cs = np.concatenate([[0], np.cumsum(np.concatenate([_BYTE[s], np.full(8, _BYTE[0], np.int64)]))])
    o = np.arange(s.size + 1)
    return 8 + (cs[o + 8] - cs[o])


class Rows:
    """dec_chunk_walk<CheeT>'s rows and dec_group_compose<CheeT>'s group rows of one piece, computed on demand"""

    def __init__(self, cons, n):
        self.cons, self.n = cons, n
        self.nchunks = (n + CH - 1) // CH
        self.chunk, self.group = {}, {}

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

    def group_row(self, g, e):
        """(exit index or TERM, blocks, flags as chunk_row + 8 short last group)"""
        key = (g, e)
        if key not in self.group:
            idx, blocks, pair, first, last, have = e, 0, 0, 0, 0, False
            c0, c1 = g * GROUP, min(self.nchunks, (g + 1) * GROUP)
            for c in range(c0, c1):
                ex, nb, fl = self.chunk_row(c, idx)
                blocks += nb
                idx = ex
                if ex == TERM:
                    break
                if nb:
                    if not have:
                        first, have = (fl >> 1) & 1, True
                    else:
                        pair |= last & (fl >> 1) & 1
                    pair |= fl & 1
                    last = (fl >> 2) & 1
            fl = pair | first << 1 | last << 2 | (8 if c1 - c0 < GROUP else 0)
            self.group[key] = (idx, blocks, fl)
        return self.group[key]


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
        if off + 8 > n:
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
    """The transfer of a non-final piece (uint8 array) and the walk's statistics: (int array [NCAND], {"max_live": most live heads
    after the first chunk, "heads": live heads after every chunk step, "capped": candidates refused for the cap}). head_cap: the most
    heads kept after a merge step; the candidates of the heads beyond it get NOEND."""
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
