"""A CPU model of the Chameleon seek index (include/density_b200.h, "Chameleon seek index"; DESIGN §4h), byte for byte, and of the
piece an indexed range decode reads. Built from test_decode_range_cpu.py's walk model: every block start and the automaton state in
front of it (walk_all), the decode candidate of a state (candidate), and the writer pass (prefix_table), here kept in the shard table
format (bit 16 touched, low 16 bits the fingerprint) and folded checkpoint by checkpoint."""
import numpy as np

import planted
from test_decode_range_cpu import BS, candidate, walk_all

MAGIC = int.from_bytes(b"CHAMINDX", "little")
SNAPSHOT_WORDS = 65536


def max_count(n, interval):
    """density_b200_chameleon_index_bytes's checkpoint bound: the largest block count n bytes hold (bounds_layout: n / 136 + 2)"""
    return (n // 136 + 2 - 1) // (interval // BS)


def snapshots_at(count):
    return (64 + 16 * count + 255) // 256 * 256


def index_bytes(n, interval):
    if interval < BS or interval % BS:
        return 0
    c = max_count(n, interval)
    return snapshots_at(c) + c * SNAPSHOT_WORDS * 4


def build(stream, interval, m=None):
    """-> (index bytes, walk) or (None, walk) for a malformed stream"""
    s = np.asarray(stream, np.uint8)
    m = m or walk_all(s)
    if m["verdict"]:
        return None, m
    every, mb, starts, copy = interval // BS, m["main_blocks"], m["starts"], m["copy"]
    count = (mb - 1) // every if mb else 0
    raw = s.tobytes()
    table = np.zeros(SNAPSHOT_WORDS, np.uint32)
    table[0] = 0x10000                                   # density_b200_table_init: bucket 0 holds quad 0 (chameleon.rs:41)
    snaps, dir_ = [], []
    for b in range(count * every):
        if not copy[b]:
            pos = starts[b]
            sig = int.from_bytes(raw[pos:pos + 8], "little")
            pos += 8
            for k in range(64):
                if (sig >> k) & 1:
                    pos += 2
                else:
                    h, f = planted.hf(int.from_bytes(raw[pos:pos + 4], "little"))
                    table[h] = 0x10000 | f
                    pos += 4
        if (b + 1) % every == 0:
            snaps.append(table.copy())
            dir_.append((starts[b + 1], candidate(m["before"][b + 1])))
    total = snapshots_at(count) + count * SNAPSHOT_WORDS * 4
    out = bytearray(np.array([MAGIC, 1, s.size, m["S"], mb, interval, count, total], np.uint64).tobytes())
    for off, cand in dir_:
        out += np.array([off], np.uint64).tobytes() + np.array([cand, 0], np.uint32).tobytes()
    out += bytes(snapshots_at(count) - len(out))
    for t in snaps:
        out += t.tobytes()
    assert len(out) == total
    return bytes(out), m


def parse(index):
    x = np.frombuffer(index, np.uint8)
    hdr = x[:64].view(np.uint64)
    count = int(hdr[6])
    d = x[64:64 + 16 * count]
    offs = d.reshape(-1, 16)[:, :8].copy().view(np.uint64).ravel() if count else np.zeros(0, np.uint64)
    cands = d.reshape(-1, 16)[:, 8:12].copy().view(np.uint32).ravel() if count else np.zeros(0, np.uint32)
    return {"n": int(hdr[2]), "S": int(hdr[3]), "main_blocks": int(hdr[4]), "interval": int(hdr[5]), "count": count,
            "bytes": int(hdr[7]), "off": [int(v) for v in offs], "cand": [int(v) for v in cands]}


def snapshot(index, j):
    """snapshot j (checkpoint j = 1 .. C) as 65536 u32"""
    x = parse(index)
    at = snapshots_at(x["count"]) + (j - 1) * SNAPSHOT_WORDS * 4
    return np.frombuffer(index, np.uint32, SNAPSHOT_WORDS, at)


def plan(index, n, first, length):
    """the piece an indexed range decode reads for the window (decode_range.cu index_plan): None when first >= S or length == 0, else
    {a, b (None: final), off, end, skip, w, expect}"""
    x = parse(index)
    S, mb, every, count = x["S"], x["main_blocks"], x["interval"] // BS, x["count"]
    if first >= S or length == 0:
        return None
    w = min(length, S - first)
    k0, k1 = first // BS, (first + w - 1) // BS
    a, b = min(k0 // every, count), k1 // every + 1
    final = b > count or k1 >= mb or first + w == S
    off = x["off"][a - 1] if a else 0
    end = n if final else x["off"][b - 1]
    expect = S - a * every * BS if final else (b - a) * every * BS
    return {"a": a, "b": None if final else b, "off": off, "end": end, "skip": first - a * every * BS, "w": w, "expect": expect,
            "cand": x["cand"][a - 1] if a else 0}


def dictionary(table):
    """a shard table as decode_reference's dictionary: the quad of each touched bucket, 0 for an untouched one"""
    quads = [0] * 65536
    for h in np.nonzero(table & 0x10000)[0]:
        quads[int(h)] = int(planted.quad_of(int(h), int(table[h]) & 0xFFFF))
    return quads
