"""Lion streams for the tests of the parallel Lion decoder: the block structure of a stream read off the stream itself, the walk's
counts computed from it and from the decoded quads (independently of density_b200/csrc/lion_walk.cuh), well-formed streams with random
flags that no encoder writes, and inputs aimed at the prediction walk."""
import ctypes
import os
import subprocess

import numpy as np

BS, SIG = 64, 6
# extra bytes behind whole blocks: every tail length class of decode_partial_unit and of the main-loop exit (SIG + BS = 70)
TAIL_SWEEP = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 69, 70, 71, 127, 128, 129, 133, 134, 135, 191, 255]
HASH_MULT = 0x9D6EF916


def hash16(v):
    return ((int(v) * HASH_MULT) & 0xFFFFFFFF) >> 16


class Prot:
    """codec/protection_state.rs:9-47"""

    def __init__(self):
        self.pen, self.start, self.prev, self.counter = 0, 1, 0, 0

    def revert(self):
        if self.counter % 16 == 0 and self.start > 1:
            self.start >>= 1
        self.counter += 1
        return self.pen > 0

    def decay(self):
        self.pen = (self.pen - 1) & 0xFF
        if self.pen == 0:
            self.start = (self.start + 1) & 0xFF

    def update(self, inc):
        if inc:
            if self.prev:
                self.pen = self.start
            self.prev = 1
        else:
            self.prev = 0


def blocks(stream):
    """The main loop's blocks (codec.rs:88-100): a list of (copy, flags or None, explicit hashes of MAP quads by position)."""
    s = bytes(stream)
    n, idx, ps, out = len(s), 0, Prot(), []
    while n - idx >= SIG + BS:
        if ps.revert():
            out.append((True, None, None))
            idx += BS
            ps.decay()
            continue
        sig = int.from_bytes(s[idx:idx + SIG], "little")
        flags = [(sig >> (3 * k)) & 7 for k in range(16)]
        p, maps = idx + SIG, {}
        for k, f in enumerate(flags):
            if f == 0:
                p += 4
            elif f >= 6:
                maps[k] = s[p] | (s[p + 1] << 8)
                p += 2
        out.append((False, flags, maps))
        ps.update(p - idx >= BS)
        idx = p
    return out


def walk_counts(stream, decoded):
    """{encoded quads, predicted quads, table reads that waited on a predicted quad, rows} of the prediction walk over 32-quad rows
    (two blocks per row). A read waits on a predicted quad when a row needs the row-start list of a context c and no lane's context
    was c before the row's first table read: the first predicted lane at c has fewer than 5 pushes at c in front of it, or, with no
    predicted lane at c, the row has fewer than 5 pushes at c."""
    blk = blocks(stream)
    q = np.frombuffer(np.ascontiguousarray(decoded)[:len(blk) * BS].tobytes(), dtype="<u4")
    nrows = (len(blk) + 1) // 2
    quads = pred = dep = 0
    carry = 0
    for r in range(nrows):
        lanes = []                                      # (lane, predicted, hash) of the encoded lanes
        for half in range(2):
            b = 2 * r + half
            if b >= len(blk) or blk[b][0]:
                continue
            _, flags, maps = blk[b]
            for k, f in enumerate(flags):
                v = int(q[b * 16 + k])
                lanes.append((16 * half + k, 1 <= f <= 5, maps[k] if f >= 6 else hash16(v)))
        if not lanes:
            continue
        quads += len(lanes)
        pred += sum(1 for _, p, _ in lanes if p)
        ctx, known = [], []
        prev = None
        for i, (lane, p, h) in enumerate(lanes):
            inrow = prev is not None and prev[0] == lane - 1
            ctx.append(prev[2] if inrow else carry)
            known.append(not (inrow and prev[1]))
            prev = (lane, p, h)
        carry = lanes[-1][2]
        for c in set(ctx):
            at = [i for i in range(len(lanes)) if ctx[i] == c]
            if any(known[i] for i in at):
                continue
            first_pred = next((i for i in at if lanes[i][1]), None)
            pushes = sum(1 for i in at if not lanes[i][1] and (first_pred is None or i < first_pred))
            dep += pushes < 5
    return quads, pred, dep, nrows


def synth_stream(seed, nblocks, tail_bytes=0, p_pred=0.5):
    """A well-formed Lion stream with random flags, laid out block by block with the protection automaton as a decoder reads it
    (copy-mode blocks are 64 raw bytes), then `tail_bytes` raw bytes for the tail loop. Predicted flags are drawn with probability
    p_pred, MAP_A / MAP_B hashes and literals at random."""
    rng = np.random.default_rng(seed)
    ps, parts = Prot(), []
    for _ in range(nblocks):
        if ps.revert():
            parts.append(rng.integers(0, 256, BS, dtype=np.uint8).tobytes())
            ps.decay()
            continue
        flags = [int(rng.integers(1, 6)) if rng.random() < p_pred else int(rng.choice([0, 6, 7])) for _ in range(16)]
        sig = sum(f << (3 * k) for k, f in enumerate(flags))
        body = bytearray(sig.to_bytes(SIG, "little"))
        for f in flags:
            if f == 0:
                body += rng.integers(0, 256, 4, dtype=np.uint8).tobytes()
            elif f >= 6:
                body += rng.integers(0, 256, 2, dtype=np.uint8).tobytes()
        parts.append(bytes(body))
        ps.update(len(body) >= BS)
    parts.append(rng.integers(0, 256, tail_bytes, dtype=np.uint8).tobytes())
    return np.frombuffer(b"".join(parts), dtype=np.uint8).copy()


def decode_cap(stream):
    """An output capacity no Lion stream of this size can exceed (a 6-byte signature of predicted quads decodes to 64 bytes)."""
    return (len(stream) // SIG + 2) * BS


def records(period_quads, nbytes, seed=0):
    """Repeating records of `period_quads` quads with a counter field that changes every record: the contexts repeat with the period."""
    rng = np.random.default_rng(seed + period_quads)
    rec = rng.integers(0, 256, 4 * period_quads, dtype=np.uint8)
    reps = nbytes // rec.size + 1
    out = np.tile(rec, reps)
    out[::rec.size] = np.arange(reps, dtype=np.uint8)
    return out[:nbytes].copy()


def walk_inputs():
    """name -> input aimed at the walk: predicted chains across rows and blocks, copy-mode blocks between a predicted quad and its
    successor, contexts revisited at every depth inside one row, zero fill, records with periods from 2 to 40 quads."""
    rng = np.random.default_rng(5)
    d = {}
    words = rng.integers(0, 1 << 32, 6, dtype=np.uint64).astype("<u4")
    # a few values in a rotating order: predicted at depths 1-5 on one context, revisited within a row
    seq = np.concatenate([words[rng.permutation(6)[:5]] for _ in range(4000)])
    d["depths"] = seq.view(np.uint8).copy()
    # text with incompressible bursts: copy-mode blocks land between predicted quads and their successors
    base = np.tile(np.frombuffer(b"the quick brown fox jumps over the lazy dog. ", np.uint8), 3000)
    noisy = base.copy()
    for k in range(0, noisy.size - 400, 9000):
        noisy[k:k + 300] = rng.integers(0, 256, 300, dtype=np.uint8)
    d["text_bursts"] = noisy
    d["zeros_runs"] = np.concatenate([np.zeros(70001, np.uint8), rng.integers(0, 256, 5000, dtype=np.uint8), np.zeros(64 * 1024 + 3, np.uint8)])
    for p in (2, 3, 5, 7, 8, 16, 17, 24, 31, 32, 33, 40):
        d[f"records{p}"] = records(p, 40000 + p)
    return d


def build_model(directory):
    """tests/lion_walk_model.cpp built with g++ into `directory`, loaded with ctypes"""
    here = os.path.dirname(os.path.abspath(__file__))
    so = os.path.join(str(directory), "_lion_walk_model.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(here, "lion_walk_model.cpp"), "-o", so])
    L = ctypes.CDLL(so)
    L.lion_walk_model_decode.restype = ctypes.c_size_t
    L.lion_walk_model_decode.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_uint64)]
    return L


def run_model(L, enc, cap):
    """-> (decoded size, decoded bytes, walk counts) of the CPU model"""
    enc = np.ascontiguousarray(enc, dtype=np.uint8)
    out = np.zeros(cap + 64, np.uint8)
    c = (ctypes.c_uint64 * 4)()
    n = L.lion_walk_model_decode(enc.ctypes.data, enc.size, out.ctypes.data, cap, c)
    return n, out[:n], tuple(c)
