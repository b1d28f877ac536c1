"""CPU model of the protected range map of a stream without known cuts (numpy only; the twin of dec_prot_transfer<T, true> and
of prot_locate_walk in decode_bounds.cuh).

Rank r holds the stream bytes [o_r, o_r + n_range) of its RANGE and the next min(264, rest) bytes of its HALO. For every entry offset e
(2e bytes into the range: 132 of them for Chameleon, 68 for Cheetah) and every decode candidate c (prot_decode_model's encoding, 3200 of
them) the map holds where the exact boundary walk of codec.rs:88-100, copy-mode blocks included, leaves the range: the exit index x
(the first block start at or after n_range is n_range + 2x) and the candidate there, packed as x | cand << 8; TERM when the main loop
ends (fewer than MAXBLK bytes left) in front of n_range; PROT_ESC when the state there is not a candidate.

The model walks every (entry, candidate) exactly, as one lane each; lanes that reach the same (offset, state, phase) are merged, which
changes no lane's result. It has no head cap: the device refuses (NOEND) where it drops heads, which the composition turns into a refusal."""
import numpy as np

import prot_decode_model as CM
import prot_decode_model_cheetah as KM
from prot_decode_model import NCAND, NOEND, PROT_ESC, cand_index, cand_state  # noqa: F401

TERM = 0xFF
HDR = 4                                 # {n_range lo, hi, n_halo lo, hi}
RANGE_UNIT = 16384                      # non-last ranges are multiples of it
HALO = 264
# alg -> (consumed table, block bytes, MAXBLK, entry offsets)
GEOM = {"chameleon": (CM.consumed_table, 256, 264, 132), "cheetah": (KM.consumed_table, 128, 136, 68)}


def map_words(alg):
    return HDR + GEOM[alg][3] * NCAND


def _pack(pen, start, prev, ph):
    return pen | (start << 8) | (prev << 16) | (ph << 17)


def _row(off, st, n_range):
    """the map word of heads that reached off >= n_range in packed state st"""
    pen, start, ph = st & 0xFF, (st >> 8) & 0xFF, st >> 17
    pc = (ph * 200 + (((st >> 16) & 1) * 10 + (start - 1)) * 10 + pen).astype(np.int64)
    esc = (pen >= 10) | (start < 1) | (start > 10)
    return np.where(esc, PROT_ESC, ((off - n_range) >> 1) | (pc << 8))


def walk(cons, n_range, n, off, st, alg):
    """rows of lanes starting at offsets `off` in packed states `st` (int64 arrays), walked exactly over a range of n_range bytes
    followed by n - n_range halo bytes (cons: the consumed table of those n bytes)"""
    _, BS, MAXBLK, _ = GEOM[alg]
    key, lane = np.unique((off.astype(np.int64) << 21) | st, return_inverse=True)
    h_off, h_st = key >> 21, key & ((1 << 21) - 1)
    res = np.full(key.size, -1, np.int64)
    while True:
        live = np.nonzero(res < 0)[0]
        if live.size == 0:
            break
        o, s = h_off[live], h_st[live]
        out = o >= n_range
        res[live[out]] = _row(o[out], s[out], n_range)
        term = ~out & (o + MAXBLK > n)
        res[live[term]] = TERM
        go = ~out & ~term
        i, o, s = live[go], o[go], s[go]
        pen, start, prev, ph = s & 0xFF, (s >> 8) & 0xFF, (s >> 16) & 1, s >> 17
        start = np.where((ph == 0) & (start > 1), start >> 1, start)
        ph = (ph + 1) & 15
        copy = pen > 0
        pen = np.where(copy, (pen - 1) & 0xFF, pen)
        start = np.where(copy & (pen == 0), (start + 1) & 0xFF, start)
        con = cons[np.minimum(o, cons.size - 1)]
        inc = ~copy & (con >= BS)
        pen = np.where(inc & (prev == 1), start, pen)
        prev = np.where(copy, prev, inc.astype(np.int64))
        h_off[i] = o + np.where(copy, BS, con)
        h_st[i] = _pack(pen, start, prev, ph)
        # merge the live heads that met: every lane follows its head
        live = np.nonzero(res < 0)[0]
        k2, inv = np.unique((h_off[live] << 21) | h_st[live], return_inverse=True)
        if k2.size < live.size:
            done = np.nonzero(res >= 0)[0]
            remap = np.empty(h_off.size, np.int64)
            remap[done] = np.arange(done.size)
            remap[live] = done.size + inv
            h_off = np.concatenate([h_off[done], k2 >> 21])
            h_st = np.concatenate([h_st[done], k2 & ((1 << 21) - 1)])
            res = np.concatenate([res[done], np.full(k2.size, -1, np.int64)])
            lane = remap[lane]
    return res[lane]


def range_map(buf, n_range, n_halo, alg):
    """the protected range map of buf[:n_range + n_halo] (uint32 [map_words(alg)])"""
    cons_fn, _, _, nc = GEOM[alg]
    n = n_range + n_halo
    out = np.zeros(map_words(alg), np.uint32)
    out[:HDR] = [n_range & 0xFFFFFFFF, n_range >> 32, n_halo & 0xFFFFFFFF, n_halo >> 32]
    e = np.repeat(np.arange(nc, dtype=np.int64), NCAND)
    c = np.tile(np.arange(NCAND, dtype=np.int64), nc)
    if n_range == 0:
        rows = e | (c << 8)                   # an empty range passes its entry on
    else:
        pc = c % 200
        st = _pack(pc % 10, (pc // 10) % 10 + 1, pc // 100, c // 200)
        rows = walk(cons_fn(np.asarray(buf[:n], np.uint8)), n_range, n, 2 * e, st, alg)
    out[HDR:] = rows.astype(np.uint32)
    return out


def stream_maps(stream, lay, alg):
    """[world, map_words] maps of a layout [(offset, n_range, n_halo)] of one stream"""
    return np.stack([range_map(stream[o:o + n + h], n, h, alg) for o, n, h in lay])


def locate_piece(maps, rank, alg):
    """prot_locate_walk: (start, end, is_final, is_first, entry candidate, refused); ValueError on a bad layout or row"""
    nc = GEOM[alg][3]
    maps = np.asarray(maps, np.uint32).reshape(-1, map_words(alg))
    world = maps.shape[0]
    hdr = [(int(m[0]) | int(m[1]) << 32, int(m[2]) | int(m[3]) << 32) for m in maps]
    later = 0
    for r in range(world - 1, -1, -1):
        nr, nh = hdr[r]
        if r < world - 1 and nr % RANGE_UNIT:
            raise ValueError("a non-last range is not a multiple of 16384 bytes")
        if nh != min(later, HALO):
            raise ValueError("a halo is not min(264, the bytes of the later ranges)")
        later += nr
    out = [0] * 6
    idx, cand, started, ended = 0, 0, False, False
    for r in range(world):
        nr, nh = hdr[r]
        if ended or nr == 0:
            if r == rank:
                out[2] = int(ended or nh == 0)
            continue
        row = int(maps[r][HDR + idx * NCAND + cand])
        if row in (PROT_ESC, NOEND):
            return (0, 0, 0, 0, 0, 1)
        x = row & 0xFF
        if x == TERM:
            if row != TERM:
                raise ValueError("bad row")
            end, ended = nr + nh, True
        else:
            if x >= nc or (row >> 8) >= NCAND:
                raise ValueError("bad row")
            end = nr + 2 * x
        if 2 * idx > end or end > nr + nh:
            raise ValueError("bad row")
        if r == rank:
            out = [2 * idx, end, int(end == nr + nh), int(not started), cand, 0]
        if not ended:
            idx, cand = x, row >> 8
        started = True
    return tuple(out)


def layout(total, ranges):
    """[(offset, n_range, n_halo)] for explicit range lengths (the last takes the rest when it is None)"""
    out, off = [], 0
    for i, n in enumerate(ranges):
        n = total - off if n is None else n
        out.append((off, n, 0))
        off += n
    return [(o, n, min(HALO, total - o - n)) for o, n, _ in out]
