"""Planted corpora: text with chosen (hash, fingerprint) sentinels at chosen tile, region and run positions (numpy only).

The kernels go wrong in (hash, fingerprint) space and at positions relative to their tiles, warp regions and runs, not on
whatever values ordinary text happens to contain. Every generator here starts from the dickens fixture (compressible text, so
the Chameleon fast path is taken), plants sentinel quads at positions derived from the host code's run geometry and returns
`(bytes, manifest)`. The manifest is a list of `(quad index, quad, class)`; tests/test_planted_cpu.py checks that every class
is still planted where it says, so a later edit cannot silently drop coverage.

Planted buckets are taken from the buckets the base text never touches, so the state a sentinel meets (never touched, last
written in an earlier run by the same quad, by another member, by its bit-31 twin or by its fingerprint-0 member, ...) is the one
the generator chose, not an accident of the text.
"""
import os

import numpy as np

M = 0x9D6EF916                     # common.cuh HASH_MULT
M_HALF_INV = pow(M >> 1, -1, 1 << 32)
H100_SMS = 132
TILE_QUADS = 4096                  # a tile is 4096 quads (16 KiB) in all three algorithms
TILE_BYTES = 4 * TILE_QUADS
F6_REGION = 256                    # quads per warp region in cham_flag_pass6 / cham_decode_pass7
R1_REGION = 128                    # quads per warp region in the round-1 passes
ALL_ONES = 0xEE4FF4DD              # hash 0xFFFF, fingerprint 0xFFFF: record word 0xFFFFFFFF
FP0_HASHES = (1, 0x0FFF, 0x1000, 0x7FFF, 0x8000, 0xFFFF)
_DICKENS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dickens_200k.bin")


def hf(q):
    """(hash, fingerprint) of a quad or an array of quads (common.cuh: hash_prod / prod_hash / prod_fp)."""
    a = np.asarray(q, dtype=np.uint64)
    p = (a * np.uint64(M)) & np.uint64(0xFFFFFFFF)
    h, f = (p >> np.uint64(16)), (p & np.uint64(0xFFFE)) | (a >> np.uint64(31))
    if np.ndim(q) == 0:
        return int(h), int(f)
    return h.astype(np.int64), f.astype(np.int64)


def quad_of(h, f):
    """The quad with hash h and fingerprint f (common.cuh: quad_from_hf)."""
    p = ((h & 0xFFFF) << 16) | (f & 0xFFFE)
    return (((p >> 1) * M_HALF_INV) & 0x7FFFFFFF) | ((f & 1) << 31)


def twin(q):
    """Same product and hash; the fingerprints differ only in bit 0."""
    return q ^ 0x80000000


def cham_runs(nbytes, num_sms=H100_SMS):
    """Tile ranges of the Chameleon runs (chameleon_encode.cu: cham_pick_runs, run r covers [r*ntiles/nruns, (r+1)*ntiles/nruns))."""
    ntiles = ((nbytes + 255) // 256 + 63) // 64
    nruns = min(max(ntiles // 16, 1), num_sms)
    return [(r * ntiles // nruns, (r + 1) * ntiles // nruns) for r in range(nruns)]


def chee_runs(nbytes, num_sms=H100_SMS, per_sm=8):
    """Tile ranges of the Cheetah / Lion runs (cheetah_encode.cu: chee_pick_runs: ntiles / 2, at most 8 per SM, at least 64 once
    there are 64 tiles; run r covers [r*ntiles/nruns, (r+1)*ntiles/nruns))."""
    ntiles = ((nbytes + 127) // 128 + 127) // 128
    r = min(ntiles // 2, num_sms * per_sm)
    if r < 64 <= ntiles:
        r = 64
    r = max(r, 1)
    return [(k * ntiles // r, (k + 1) * ntiles // r) for k in range(r)]


def base_text(nbytes):
    """The dickens fixture repeated to nbytes (200,003 B is not a multiple of 4, so the quads of every copy differ)."""
    return np.resize(np.fromfile(_DICKENS, dtype=np.uint8), nbytes)


class Planter:
    """Quads of a base buffer plus a pool of buckets the base never touches."""

    def __init__(self, nbytes, seed, data=None):
        self.nbytes = nbytes
        self.data = base_text(nbytes) if data is None else data
        self.nq = nbytes // 4
        self.q = self.data[:self.nq * 4].view(np.uint32)      # a view: planting writes the bytes
        self.rng = np.random.default_rng(seed)
        used = np.zeros(65536, bool)
        for k in range(4):                                     # the text's quads at every byte phase
            m = (nbytes - k) // 4
            if m > 0:
                used[hf(self.data[k:k + 4 * m].view(np.uint32))[0]] = True
        used[list(FP0_HASHES) + [0]] = True                    # planted on purpose, never handed out as fresh
        free = np.flatnonzero(~used)
        self.free = list(self.rng.permutation(free))
        self.free_set = set(int(x) for x in free)
        self.manifest = {}

    def bucket(self):
        """A bucket nothing has touched yet."""
        h = int(self.free.pop())
        self.free_set.discard(h)
        return h

    def take(self, h):
        """Claim a specific free bucket (False if it is not free)."""
        if h not in self.free_set:
            return False
        self.free_set.discard(h)
        self.free.remove(h)
        return True

    def fp(self):
        """A random fingerprint that is neither 0 nor 0xFFFF / 0xFFFE."""
        return int(self.rng.integers(1, 0xFFFE))

    def put(self, pos, value, cls):
        if 0 <= pos < self.nq:
            self.q[pos] = value
            self.manifest[pos] = (int(value), cls)

    def result(self):
        return self.data, sorted((p, v, c) for p, (v, c) in self.manifest.items())


# ---- Chameleon --------------------------------------------------------------------------------------------------------------
EDGE_OFFS = (0, 1, 127, 128, 255, 256, 257, 511, 2047, 2048, 3839, 3840, 4094, 4095)   # tile position 0 / 4095, region starts and ends


def _edge_value(P, k):
    """Sentinel values for tile and region edges, cycling through the value classes."""
    c = k % 7
    if c == 0:
        return quad_of(FP0_HASHES[(k // 7) % len(FP0_HASHES)], 0), "fp0_fixed"
    if c == 1:
        return quad_of(P.bucket(), 0), "fp0_fresh"
    if c == 2:
        return 0, "quad0"
    if c == 3:
        return quad_of(0, P.fp()), "bucket0_member"
    if c == 4:
        return ALL_ONES, "all_ones"
    if c == 5:
        return quad_of(P.bucket(), 0xFFFF if k & 1 else 0xFFFE), "fp_ffff_fffe"
    return twin(quad_of(P.bucket(), P.fp())), "twin_fresh"


def _carried_state(P, prev_pos, pos, k):
    """A bucket last written before `pos` (at prev_pos: an earlier run) in one of the chosen ways, then touched at pos."""
    h = P.bucket()
    f = P.fp()
    a = quad_of(h, f)
    c = k % 6
    if c == 0:
        P.put(prev_pos, a, "carry_same"); P.put(pos, a, "carry_same")
    elif c == 1:
        P.put(prev_pos, quad_of(h, P.fp()), "carry_other"); P.put(pos, a, "carry_other")
    elif c == 2:
        P.put(prev_pos, twin(a), "carry_twin"); P.put(pos, a, "carry_twin")
    elif c == 3:
        P.put(prev_pos, quad_of(h, 0), "carry_fp0_writer"); P.put(pos, a, "carry_fp0_writer")
    elif c == 4:
        P.put(prev_pos, a, "carry_to_fp0"); P.put(pos, quad_of(h, 0), "carry_to_fp0")
    else:
        P.put(prev_pos, quad_of(h, 0), "carry_fp0_same"); P.put(pos, quad_of(h, 0), "carry_fp0_same")


def _slot_buckets(P, nb, stride=4096):
    """nb free buckets s, s + stride, s + 2*stride, ...: the same f6 mailbox slot (hh & 4095) for stride 4096."""
    for s in P.rng.permutation(stride):
        hs = [int(s) + k * stride for k in range(nb)]
        if all(h < 65536 and h in P.free_set for h in hs):
            for h in hs:
                P.take(h)
            return hs
    raise RuntimeError("no free slot")


def _alias_tiles(P, a, b, class_list):
    """Aliasing and capacity edges in tiles a + 3 .. a + 12 of the run [a, b) (text alone does not overflow there)."""
    T = lambda t, off: t * TILE_QUADS + off
    if b - a < 14:
        return
    # 4, 5 and 6 distinct buckets with dirty members in one mailbox slot, all with one fingerprint, so that a lookup that confuses
    # the buckets of a slot finds an equal fingerprint; the same quads again in the next tile (hits)
    for nb, base in ((4, 100), (5, 1300), (6, 2500)):
        f = P.fp()
        qs = [quad_of(h, f) for h in _slot_buckets(P, nb)]
        for k, v in enumerate(qs):
            P.put(T(a + 4, base + 41 * k), v, f"slot_{nb}_buckets")
            P.put(T(a + 5, base + 37 * k + 3), v, f"slot_{nb}_buckets_again")
    # tiles a + 6 .. a + 9 test exact capacities: their text is replaced by one quad that is a hit (it closes tile a + 5), so the
    # planted members are the only records of the tile
    z = quad_of(P.bucket(), P.fp())
    P.put(T(a + 5, 4000), z, "filler")
    P.q[T(a + 6, 0):T(a + 10, 0)] = z
    # one bucket with exactly 20 / 21 dirty members that are not one run (alternating values, 193 quads apart)
    for t, nm in ((a + 6, 20), (a + 7, 21)):
        h = P.bucket()
        x, y = quad_of(h, P.fp()), quad_of(h, 0)
        for k in range(nm):
            P.put(T(t, 60 + 193 * k), x if k % 2 == 0 else y, f"bucket_{nm}_members")
    # exactly 16 / 17 entries in one overflow mailbox (slot & 63): two slots s and s + 64, 4 mailbox entries each, the rest overflow
    for t, (n1, n2) in ((a + 8, (12, 12)), (a + 9, (12, 13))):
        while True:
            s = int(P.rng.integers(0, 4096 - 64))
            if s in P.free_set and s + 64 in P.free_set:
                P.take(s); P.take(s + 64)
                break
        for h, nm, off in ((s, n1, 50), (s + 64, n2, 2100)):
            x, y = quad_of(h, P.fp()), twin(quad_of(h, P.fp()))
            for k in range(nm):
                P.put(T(t, off + 151 * k), x if k % 2 == 0 else y, f"overflow_{n1 - 4 + n2 - 4}_entries")
    # decoder mark map (hh & 8191) and round-1 side tables (hh & 8191 encode, hh & 4095 decode): readers of h ^ 0x2000 / h ^ 0x1000
    # (written in an earlier tile) among writers of h
    t = a + 10
    for j in range(6):
        h0, h1, h2 = _slot_buckets(P, 3, stride=0x1000)
        r1, r2 = quad_of(h1, P.fp()), quad_of(h2, 0)
        P.put(T(a + 3, 700 + 10 * j), r1, "alias_reader_setup")
        P.put(T(a + 3, 705 + 10 * j), r2, "alias_reader_setup")
        base = 200 + 600 * j
        P.put(T(t, base), quad_of(h0, P.fp()), "alias_writer")
        P.put(T(t, base + 1), r1, "alias_reader")
        P.put(T(t, base + 130), quad_of(h0, 0), "alias_writer")
        P.put(T(t, base + 131), r2, "alias_reader")
        P.put(T(t, base + 300), r1, "alias_reader")
    # a round-1 class list (hh >> 11) past 128 entries: 140 first touches of one class in one tile (every fourth such run: the
    # free buckets would run out)
    if not class_list:
        return
    cls = int(P.rng.integers(0, 32))
    pool = [h for h in range(cls << 11, (cls + 1) << 11) if h in P.free_set][:140]
    for k, h in enumerate(pool):
        P.take(h)
        P.put(T(a + 11, 20 + 29 * k), quad_of(h, 0 if k % 3 == 0 else P.fp()), "class_list_140")
    # runs of equal copies across region (128, 256) and tile boundaries
    x = quad_of(P.bucket(), 0)
    for off in range(124, 133):
        P.put(T(a + 12, off), x, "copies_across_region")
    y = quad_of(P.bucket(), P.fp())
    for off in range(250, 262):
        P.put(T(a + 12, off), y, "copies_across_region")
    z = ALL_ONES
    for off in range(-4, 4):
        P.put(T(a + 12, off), z, "copies_across_tile")


def chameleon_corpus(nbytes, seed, num_sms=H100_SMS, seams=()):
    """Chameleon corpus for the run-parallel fast path. Plants, in every run of `cham_runs(nbytes)`:
    sentinels at the edge positions of the first three tiles (which take f6_replay on text) and of the last tile; buckets carried
    in from the previous run in every chosen state; aliasing and capacity edges in tiles 4..12; runs of equal copies across
    region, tile and run boundaries. Also the stream's first quad, the last partial tile and the last 264 bytes (dec_tail). `seams`
    adds the same carried-state plantings around further byte offsets (the 64 MiB chunk seams of the host pipeline). The aliasing
    and capacity tiles go into every fourth run, so that the free buckets suffice."""
    P = Planter(nbytes, seed)
    runs = cham_runs(nbytes, num_sms)
    T = lambda t, off: t * TILE_QUADS + off
    k = 0
    for r, (a, b) in enumerate(runs):
        for t in sorted({a, a + 1, a + 2, b - 1}):
            if t >= b:
                continue
            for off in EDGE_OFFS:
                if r % 4 == 1 and t == a and off < 4:
                    continue                                   # the copies across the run boundary live there
                v, c = _edge_value(P, k)
                P.put(T(t, off), v, c + ("_run_first_tiles" if t < a + 3 else "_run_last_tile"))
                k += 1
        if r > 0:
            pa = runs[r - 1][1] - 1                            # last tile of the previous run
            for j in range(12):
                _carried_state(P, T(pa, 1000 + 200 * j + (j % 3)), T(a, 600 + 211 * j + (j % 4)), k)
                k += 1
            # written earlier in the same tile by another member, then the planted quad
            for j in range(4):
                h = P.bucket()
                P.put(T(a + min(1, b - a - 1), 300 + 800 * j), quad_of(h, P.fp()), "same_tile_other")
                P.put(T(a + min(1, b - a - 1), 300 + 800 * j + 5 + j * 60), quad_of(h, 0) if j % 2 else twin(quad_of(h, P.fp())), "same_tile_other")
            # the all-ones record word as the first quad of a tile that resolves through the mailboxes, right after another member
            # of bucket 0xFFFF: a miss, never the continuation of a run
            for t in (a + 4, b - 1):
                if a + 4 < b:
                    P.put(T(t - 1, 4000), quad_of(0xFFFF, P.fp()), "all_ones_tile_start_miss")
                    P.put(T(t, 0), ALL_ONES, "all_ones_tile_start_miss")
            if b - a >= 14:                                    # fp-0 last writer in one tile, read again in a later tile of the run
                for j in range(4):
                    x = quad_of(P.bucket(), 0)
                    P.put(T(a + 3, 1500 + 7 * j), x, "fp0_reread_later_tile")
                    P.put(T(b - 1, 1700 + 7 * j), x, "fp0_reread_later_tile")
            if r % 4 == 1:
                x = quad_of(P.bucket(), 0) if r % 8 == 1 else ALL_ONES
                for off in range(-3, 3):
                    P.put(T(a, off), x, "copies_across_run")
        if r % 4 == 2:
            _alias_tiles(P, a, b, r % 16 == 2)
    for s in seams:
        s4 = s // 4
        for j in range(16):
            _carried_state(P, s4 - 3000 + 150 * j, s4 + 40 + 97 * j, j)
        x = quad_of(P.bucket(), 0)
        for off in range(-3, 3):
            P.put(s4 + off, x, "copies_across_seam")
    P.put(0, quad_of(FP0_HASHES[seed % len(FP0_HASHES)], 0), "stream_first")
    nq = P.nq
    last_tile = (nq - 1) // TILE_QUADS
    for j, off in enumerate((0, 1, 255, 256)):
        v, c = _edge_value(P, j)
        P.put(T(last_tile, off), v, "last_partial_tile")
    for j in range(1, 67, 5):                                  # the last 264 bytes: decoded by dec_tail
        v, c = _edge_value(P, j)
        P.put(nq - j, v, "stream_tail")
    return P.result()


def chameleon_copy_corpus(nbytes, seed, every=1 << 16):
    """Chameleon corpus with copy mode: every `every` bytes a 512-byte random burst (two incompressible 256-byte blocks, so the
    block after it is copied raw) with planted sentinels right before it and inside the copied block. A quad planted inside the
    copied block is planted again after it: its first encoded occurrence must still be a miss, because copied blocks never touch
    the dictionary. Not quiet: the stream takes the protection-aware path."""
    data = base_text(nbytes)
    rng = np.random.default_rng(seed + 1000)
    bursts = range(every - every % 256, nbytes - 4096, every)
    for B in bursts:
        data[B:B + 512] = rng.integers(0, 256, 512, dtype=np.uint8)
    P = Planter(nbytes, seed, data)
    for k, B in enumerate(bursts):
        b4 = B // 4
        for j in range(1, 5):
            v, c = _edge_value(P, k * 4 + j)
            P.put(b4 - j, v, "before_burst")
        x = quad_of(P.bucket(), 0 if k % 2 else P.fp())
        P.put(b4 + 128 + 3, x, "inside_copy_block")          # block B + 512 is copied raw
        P.put(b4 + 128 + 64 + 7, x, "after_copy_block_miss")  # first encoded occurrence: a miss
        P.put(b4 + 128 + 64 + 9, x, "after_copy_block_hit")
        v, c = _edge_value(P, k)
        P.put(b4 + 128 + 64, v, "after_burst")
    return P.result()


# ---- Cheetah / Lion ---------------------------------------------------------------------------------------------------------
def cl_corpus(nbytes, seed):
    """Cheetah / Lion corpus: runs start on 16 KiB tile boundaries (one tile per run at 1 MiB, two at 33 MiB on an H100), so
    every 16 KiB boundary b gets one of: quad 0 as the first quad of a fresh prediction context; quad 0 after context 0; quad_of(h, 0)
    as the first chunk-map touch of bucket h; a bucket left at (a, b) before the seam, then a, b, the twin of a and a third value;
    a context holding 4, 5 or 6 distinct values before the seam, then hits at depths 0..4 and a miss after it."""
    P = Planter(nbytes, seed)
    ntiles = (P.nq + TILE_QUADS - 1) // TILE_QUADS
    for t in range(1, ntiles):
        b = t * TILE_QUADS
        c = t % 5
        if c == 0:
            P.put(b - 1, quad_of(P.bucket(), P.fp()), "fresh_context")
            P.put(b, 0, "quad0_fresh_context")
        elif c == 1:
            P.put(b - 1, quad_of(0, P.fp()), "context0")
            P.put(b, 0, "quad0_after_context0")
            P.put(b + 1, 0, "quad0_after_context0")
        elif c == 2:
            h = P.bucket()
            P.put(b, quad_of(h, 0), "fp0_first_touch")
            P.put(b + 2, quad_of(h, 0), "fp0_first_touch")
        elif c == 3:
            h = P.bucket()
            xa, xb, xc = quad_of(h, P.fp()), quad_of(h, 0), quad_of(h, P.fp())
            P.put(b - 3, xb, "chunk_ab_before")
            P.put(b - 2, xa, "chunk_ab_before")
            for j, v in enumerate((xa, xb, twin(xa), xc)):
                P.put(b + j, v, "chunk_ab_after")
        else:
            m = 4 + (t // 5) % 3
            z = quad_of(P.bucket(), P.fp())
            vs = [quad_of(P.bucket(), 0 if j == 0 else P.fp()) for j in range(m)]
            for j, v in enumerate(vs):
                P.put(b - 2 * m + 2 * j, z, f"lion_ctx{m}_before")
                P.put(b - 2 * m + 2 * j + 1, v, f"lion_ctx{m}_before")
            after = vs[::-1][:5] + [vs[0] if m == 6 else quad_of(P.bucket(), P.fp())]
            for j, v in enumerate(after):
                P.put(b + 2 * j, z, f"lion_ctx{m}_after")
                P.put(b + 2 * j + 1, v, f"lion_ctx{m}_after")
    return P.result()


def classes(manifest):
    out = {}
    for p, v, c in manifest:
        out.setdefault(c, []).append(p)
    return out


# ---- the named corpora the tests share ----------------------------------------------------------------------------------------
MIB = 1 << 20
CORPORA = {
    # >= 33 MiB: 132 runs x 16 tiles, every run of an H100; the last tile is partial (300 quads + 3 bytes)
    "cham33": lambda: chameleon_corpus(33 * MIB + 1203, 1),
    "cham5": lambda: chameleon_corpus(5 * MIB + 402, 2),
    # >= 129 MiB host buffers take the pipelined path in 64 MiB chunks: plantings on both sides of the 64 and 128 MiB seams
    "cham129": lambda: chameleon_corpus(129 * MIB + 7, 3, seams=(64 * MIB, 128 * MIB)),
    "copy3": lambda: chameleon_copy_corpus(3 * MIB + 5, 4),
    "cl1": lambda: cl_corpus(MIB + 13, 5),
    "cl33": lambda: cl_corpus(33 * MIB + 66, 6),
}
QUIET = ("cham33", "cham5", "cham129")
_cache = {}


def corpus(name):
    """(bytes, manifest) of a named corpus, built once per process."""
    if name not in _cache:
        _cache[name] = CORPORA[name]()
    return _cache[name]
