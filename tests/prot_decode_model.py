"""CPU model of the decode-side protection transfer of a sharded Chameleon stream (numpy only; the twin of dec_prot_transfer in
decode_bounds.cuh).

A piece of a sharded stream starts at a block boundary, but its decoder does not know the automaton state it is entered in, nor the
counter phase (revert_to_copy halves the penalty start on every 16th block of the STREAM, protection_state.rs:18-27). A decode
candidate is therefore (penalty 0..9, start 1..10, previous_incompressible, counter mod 16): 200 x 16 = 3200 of them, candidate 0 the
stream start. The transfer of a non-final piece says, for every candidate, where the boundary walk of codec.rs:88-100 (copy-mode
blocks included) leaves the piece: the candidate at its end when the walk ends exactly on the cut, PROT_ESC when that state is not a
candidate, NOEND when the walk overshoots the cut, stops short of it or reads a malformed block.

The walk follows HEADS, not candidates. A head is keyed by (offset, penalty, start, previous_incompressible, phase); heads that reach
the same key merge for good. All heads advance chunk by chunk (decode_bounds.cuh's 16 KiB chunks): a head with penalty 0 jumps a whole
group of 64 chunks, or a chunk, in O(1) from the candidate rows of dec_group_compose / dec_chunk_walk when the automaton provably stays
in encoded mode inside it (dec_seq_walk's rule); any other head walks its chunk block by block."""
import numpy as np

from protection import CH as _CH, GROUP

NCAND = 3200
PROT_ESC = 0xFFFF
NOEND = 0xFFFE
CH = _CH["chameleon"]
NC = 132                         # candidate entry offsets of a chunk row (MAXBLK / 2)
TERM = 0xFF
HEAD_CAP = 256                   # live heads kept after a chunk step (dec_prot_transfer's PT_CAP); the walk starts with 3200
_NS, _NP = 10, 10


def cand_index(pen, start, prev, phase):
    """(penalty, start, previous_incompressible, counter mod 16) -> decode candidate, PROT_ESC outside the set"""
    if pen >= _NP or start < 1 or start > _NS:
        return PROT_ESC
    return phase * 200 + (int(prev) * _NS + (start - 1)) * _NP + pen


def cand_state(c):
    """the inverse of cand_index"""
    pc = c % 200
    return (pc % _NP, (pc // _NP) % _NS + 1, pc // (_NP * _NS), c // 200)


def consumed_table(s):
    """bytes an encoded Chameleon block starting at offset o takes (264 - 2 popcount(signature)), for every o; signature bytes past
    the end read as 0"""
    s = np.asarray(s, np.uint8)
    bits = np.unpackbits(s[:, None], axis=1).sum(axis=1).astype(np.int64)
    cs = np.concatenate([[0], np.cumsum(np.concatenate([bits, np.zeros(8, np.int64)]))])
    o = np.arange(s.size + 1)
    return 264 - 2 * (cs[o + 8] - cs[o])


def sw_jump(start, phase, nb):
    """dec_seq_walk's jump over nb encoded blocks with penalty 0: the start halves on every 16th block"""
    k = (phase + nb + 15) // 16 - (phase + 15) // 16
    if start > 1:
        start = max(start >> min(k, 8), 1)
    return start, (phase + nb) & 15


class Rows:
    """dec_chunk_walk's rows and dec_group_compose's group rows of one piece, computed on demand"""

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
                if base + off + 264 > self.n:
                    r = (TERM, nb, 0)
                    break
                con = int(self.cons[base + off])
                inc = int(con >= 256)
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
        off += 256
    else:
        if off + 8 > n:
            return None
        con = int(cons[off])
        if con >= 256:
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


def compose(transfers, rank):
    """the candidate entering piece `rank`: the transfers of the pieces before it applied in order to candidate 0. Stops at the first
    PROT_ESC / NOEND, which it returns."""
    x = 0
    for r in range(rank):
        if x >= NCAND:
            break
        x = int(transfers[r][x])
    return x
