"""Protection-automaton corpora: streams that put chosen automaton states on the seams the parallel kernels cut at (numpy only).

The protection automaton (protection_state.rs:1-47) is a state machine (copy_penalty, copy_penalty_start, previous_incompressible,
counter). No kernel runs it in order: the encoders evaluate it per segment of PSEG blocks and settle the seams afterwards
(chameleon_encode.cu: prot_iterate), the decoders jump whole chunks and groups of the stream (decode_bounds.cuh: dec_seq_walk) and
hand the state to the in-order tail. The corpora here are sequences of block LETTERS whose incompressible bit does not depend on the
dictionary, so that a breadth-first search over the automaton decides which state lands on which seam:

    Z  compressible padding: pairs of fresh quads (plain, then a dictionary hit), a fixed encoded size ZSIZE below BS
    R  fresh quads, never seen before: every quad plain, SIG + BS bytes, incompressible
    P  threshold block "T+": encoded size exactly BS (incompressible)
    M  threshold block "T-": encoded size exactly BS - 2 (not incompressible)
    S  a Z block that writes a fresh quad q into the dictionary
    D  a threshold block holding the q of the last S: T+ when that S was copied (q is a miss), T- when it was encoded (q is a hit)

Every letter has a known encoded size, so the stream layout follows from the letters alone (`Builder`). `trace` parses an oracle
stream block by block and runs the automaton on it: the tests compare the two, so a corpus that stops meaning what its manifest says
fails on the CPU.
"""
import collections
import functools

import numpy as np

import oracle
import planted

ALGS = ("chameleon", "cheetah", "lion")
BS = {"chameleon": 256, "cheetah": 128, "lion": 64}
SIG = {"chameleon": 8, "cheetah": 8, "lion": 6}
FLAG_BITS = {"chameleon": 1, "cheetah": 2, "lion": 3}
CH = {"chameleon": 16384, "cheetah": 4096, "lion": 4096}            # decode_bounds.cuh: chunk bytes of ChamT / CheeT / LionT
GROUP = 64                                                          # decode_bounds.cuh: chunks per group
PSEG = 256                                                          # chameleon_encode.cu: blocks per automaton segment
TILE_BLOCKS = {"chameleon": 64, "cheetah": 128, "lion": 256}        # 16 KiB tiles of the encoders
CANON = (0, 1, 0)                                                   # (penalty, start, previous_incompressible) of protection_state.rs:9-16
MIB = 1 << 20


def maxblk(alg):
    return BS[alg] + SIG[alg]


def min_jump_blocks(alg):
    """The fewest blocks a chunk the decoder jumps can hold: it enters at most MAXBLK - 2 bytes into the chunk, and a jumped chunk
    has no two incompressible blocks in a row, so its blocks alternate at best between SIG + BS and BS - 2 bytes."""
    n, got = 0, maxblk(alg) - 2
    while got < CH[alg]:
        got += maxblk(alg) if n % 2 == 0 else BS[alg] - 2
        n += 1
    return n


# ---- the automaton ------------------------------------------------------------------------------------------------------------
class Protection:
    """protection_state.rs:9-47 with codec.rs:35-37,68 folded into one step per block."""

    def __init__(self, penalty=0, start=1, prev=0, counter=0):
        self.penalty, self.start, self.prev, self.counter = penalty, start, int(prev), counter

    def key(self):
        return (self.penalty, self.start, self.prev)

    def step(self, inc):
        """One block; `inc` is its incompressible bit if it is encoded. Returns True when the block is copied."""
        if (self.counter & 15) == 0 and self.start > 1:
            self.start >>= 1
        self.counter += 1
        if self.penalty > 0:
            self.penalty -= 1
            if self.penalty == 0:
                self.start += 1
            return True
        if inc:
            if self.prev:
                self.penalty = self.start
            self.prev = 1
        else:
            self.prev = 0
        return False


def _successors(st):
    """(penalty, start, prev, counter % 16) -> [(next state, inc bit or None for a copied block)]"""
    p, s, prev, c = st
    if c == 0 and s > 1:
        s >>= 1
    c = (c + 1) & 15
    if p > 0:
        p -= 1
        if p == 0:
            s += 1
        return [((p, s, prev, c), None)]
    return [((0, s, 0, c), 0), ((s if prev else 0, s, 1, c), 1)]


@functools.lru_cache(maxsize=None)
def _bfs(phase):
    """Shortest inc words from the canonical state at counter phase `phase`: state -> (distance, parent state, inc bit)."""
    root = (0, 1, 0, phase)
    seen = {root: (0, None, None)}
    queue = collections.deque([root])
    while queue:
        st = queue.popleft()
        for nxt, bit in _successors(st):
            if nxt not in seen:
                seen[nxt] = (seen[st][0] + 1, st, bit)
                queue.append(nxt)
    return seen


def reachable_states():
    """Every (penalty, start, prev, counter % 16) reachable from the initial state (counter 0), choosing each encoded block's
    incompressible bit freely."""
    return set(_bfs(0))


def seam_states():
    """The (penalty, start, prev) that can occur in front of a block whose index is a multiple of 16 (every encoder seam)."""
    return sorted({s[:3] for s in reachable_states() if s[3] == 0})


@functools.lru_cache(maxsize=None)
def word_to(target, index):
    """The shortest letter word (R for incompressible, Z otherwise and for copied blocks) that, started from the canonical state
    right after len(word) blocks before `index`, leaves the automaton in `target` = (penalty, start, prev) in front of block `index`."""
    best = None
    for ph in range(16):
        tab = _bfs(ph)
        key = target + (index & 15,)
        if key in tab and (best is None or tab[key][0] < best[0]):
            best = (tab[key][0], ph)
    if best is None:
        raise ValueError(f"state {target} is not reachable at counter phase {index & 15}")
    tab = _bfs(best[1])
    st, word = target + (index & 15,), []
    while tab[st][1] is not None:
        _, parent, bit = tab[st]
        word.append("R" if bit == 1 else "Z")
        st = parent
    return "".join(reversed(word))


# ---- round 0 and the relaxation rounds of prot_iterate (chameleon_encode.cu) ---------------------------------------------------
def _walk(inc, b0, b1, st):
    ps = Protection(*st, counter=b0)
    for b in range(b0, b1):
        ps.step(bool(inc[b]))
    return ps.key()


def prot_rounds(inc, pseg=PSEG):
    """Round 0 (every segment from the canonical state) and the relaxation rounds, each re-evaluating a segment from the outgoing
    state its predecessor had after the previous round (a chain of L non-canonical seams settles after at most L such rounds; the
    kernel's chaotic reads can only be faster). Returns (segments whose outgoing state is not canonical after round 0, number of
    relaxation rounds until no incoming state changes)."""
    nb = len(inc)
    nseg = (nb + pseg - 1) // pseg
    seg = [(s * pseg, min((s + 1) * pseg, nb)) for s in range(nseg)]
    ins = [CANON] * nseg
    outs = [_walk(inc, a, b, CANON) for a, b in seg]
    bad = sum(o != CANON for o in outs)
    rounds = 0
    while True:
        new_in = [CANON] + outs[:-1]
        if new_in == ins:
            return bad, rounds
        rounds += 1
        outs = [outs[s] if new_in[s] == ins[s] else _walk(inc, seg[s][0], seg[s][1], new_in[s]) for s in range(nseg)]
        ins = new_in


# ---- letters as bytes ---------------------------------------------------------------------------------------------------------
ZSIZE = {"chameleon": 200, "cheetah": 104, "lion": 54}
# threshold recipes: (fresh plain quads, "x x" pairs, "x x x" triples). A pair is plain + dictionary hit (Cheetah / Lion: MAP_A),
# a triple adds a PREDICTED quad (0 bytes) in Cheetah / Lion. Sizes: SIG + 4 f + 6 p + 6 g (+ 0 for the raw tail).
T_PLUS = {"chameleon": [(56, 4, 0)], "cheetah": [(24, 4, 0), (27, 1, 1)], "lion": [(10, 3, 0), (13, 0, 1)]}
T_MINUS = {"chameleon": [(54, 5, 0)], "cheetah": [(22, 5, 0), (25, 2, 1)], "lion": [(8, 4, 0), (11, 1, 1)]}


class Blocks:
    """Bytes of the letters for one algorithm. Fresh quads are random 32-bit values that are never 0, so they are misses in the
    zero-initialised dictionary and predictions as well."""

    def __init__(self, alg, seed):
        self.alg, self.nq = alg, BS[alg] // 4
        self.rng = np.random.default_rng(seed)
        self.next = 1 + (seed << 26)
        self.last_hash = -1
        self.q = None
        self.nt = 0

    def fresh(self, k):
        """k quads no earlier call returned (a bijection of a counter: random draws would repeat after ~2^16 quads)."""
        x = np.arange(self.next, self.next + k, dtype=np.uint64)
        self.next += k
        x = (x * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)
        x ^= x >> np.uint64(15)
        x = (x * np.uint64(0x85EBCA77)) & np.uint64(0xFFFFFFFF)
        x ^= x >> np.uint64(13)
        return x.astype(np.uint32)

    def _assemble(self, units):
        """Quads of (value, repeats) units. A value whose hash equals the previous quad's is replaced by a fresh one: the previous
        quad's prediction context would then hold it and its repeat would be PREDICTED (Cheetah / Lion) instead of a MAP hit."""
        vals = np.array([v for v, _ in units], np.uint32)
        while True:
            h = ((vals.astype(np.uint64) * np.uint64(planted.M)) & np.uint64(0xFFFFFFFF)) >> np.uint64(16)
            prev = np.concatenate([[self.last_hash], h[:-1].astype(np.int64)])
            bad = np.flatnonzero(h.astype(np.int64) == prev)
            if bad.size == 0:
                break
            vals[bad[0]] = self.fresh(1)[0]          # one at a time: a replacement changes the next unit's predecessor
        self.last_hash = int(h[-1])
        out = np.repeat(vals, [k for _, k in units])
        assert out.size == self.nq
        return out.view(np.uint8)

    def z_run(self, m):
        """m Z blocks at once: the same units as m calls of block("Z"), with the hash rule of _assemble applied to the whole run."""
        vals = self.fresh(m * self.nq // 2)
        mul, mask = np.uint64(planted.M), np.uint64(0xFFFFFFFF)
        while True:
            h = (((vals.astype(np.uint64) * mul) & mask) >> np.uint64(16)).astype(np.int64)
            prev = np.concatenate([[self.last_hash], h[:-1]])
            bad = np.flatnonzero(h == prev)
            if bad.size == 0:
                break
            bad = bad[np.concatenate([[True], np.diff(bad) > 1])]    # no two neighbours at once: each fix changes the next predecessor
            vals[bad] = self.fresh(bad.size)
        self.last_hash = int(h[-1])
        return np.repeat(vals, 2).view(np.uint8)

    def _recipe(self, f, p, g, extra=()):
        units = [1] * f + [2] * p + [3] * g + [0] * len(extra)
        units = [units[i] for i in self.rng.permutation(len(units))]
        vals = self.fresh(len(units))
        ex = list(extra)
        return self._assemble([(ex.pop(), 1) if u == 0 else (v, u) for u, v in zip(units, vals)])

    def block(self, letter):
        if letter == "R":
            return self._assemble([(v, 1) for v in self.fresh(self.nq)])
        if letter in "ZS":
            b = self._assemble([(v, 2) for v in self.fresh(self.nq // 2)])
            if letter == "S":
                self.q = b[:4].view(np.uint32)[0]
            return b
        self.nt += 1
        if letter in "PM":
            rs = (T_PLUS if letter == "P" else T_MINUS)[self.alg]
            return self._recipe(*rs[self.nt % len(rs)])
        assert letter == "D" and self.q is not None
        f, p, g = T_PLUS[self.alg][0]
        return self._recipe(f - 1, p, g, extra=[self.q])


class Builder:
    """A letter sequence with its layout: the automaton over the letters' bits, every block's stream offset and copy status."""

    def __init__(self, alg, seed):
        self.alg, self.seed = alg, seed
        self.letters, self.offs, self.copied, self.states = [], [], [], []
        self.ps = Protection()
        self.off = 0
        self.s_copied = False
        self.manifest = []

    @property
    def n(self):
        return len(self.letters)

    def state(self):
        return self.ps.key()

    def size(self, letter, copied):
        B = BS[self.alg]
        if copied:
            return B
        return {"Z": ZSIZE[self.alg], "S": ZSIZE[self.alg], "R": B + SIG[self.alg], "P": B, "M": B - 2,
                "D": B if self.s_copied else B - 2}[letter]

    def inc(self, letter):
        return {"Z": 0, "S": 0, "M": 0, "R": 1, "P": 1, "D": int(self.s_copied)}[letter]

    def add(self, word):
        for L in word:
            self.states.append((self.ps.key(), self.ps.counter))
            c = self.ps.step(self.inc(L))
            self.offs.append(self.off)
            self.off += self.size(L, c)
            if L == "S":
                self.s_copied = c
            self.letters.append(L)
            self.copied.append(c)
        return self

    def recover(self):
        """Z blocks until the automaton is canonical again (at least one)."""
        self.add("Z")
        while self.state() != CANON:
            self.add("Z")
        return self

    def mark(self, cls, **info):
        """The next block gets class `cls`."""
        self.manifest.append((self.n, cls, info))

    def place(self, b, target, cls, **info):
        """The automaton in state `target` in front of block b (padding with Z from here)."""
        w = word_to(target, b)
        assert b - len(w) >= self.n, (b, len(w), self.n)
        self.add("Z" * (b - len(w) - self.n)).add(w)
        assert self.state() == target
        self.mark(cls, state=target, **info)

    def place_in_window(self, target, lo, hi, phase=None, chunk_ok=lambda c: True, cls=None, **info):
        """The automaton in state `target` in front of the next block, whose stream offset o satisfies lo <= o - c*CH < hi for a
        chunk c with chunk_ok(c) (and block index % 16 == phase). The padding is Z blocks, k of them swapped for M (T-, same
        automaton step, BS - 2 - ZSIZE bytes more) to reach the window. Returns the chunk."""
        A, C = self.alg, CH[self.alg]
        z, dz = ZSIZE[A], BS[A] - 2 - ZSIZE[A]
        assert self.state() == CANON and hi - lo > dz
        for e in range(self.n + 1, self.n + 100000):
            if phase is not None and e % 16 != phase:
                continue
            try:
                w = word_to(target, e)
            except ValueError:
                continue
            npad = e - len(w) - self.n
            if npad < 0:
                continue
            sim = Builder(A, 0)
            sim.ps = Protection(counter=e - len(w))
            sim.add(w)
            base = self.off + npad * z + sim.off
            c = max(-(-(base - hi + 1) // C), self.off // C + 1)
            while c * C + lo <= base + npad * dz:
                if chunk_ok(c):
                    k = max(0, -(-(c * C + lo - base) // dz))
                    if k <= npad and lo <= base + k * dz - c * C < hi:
                        self.add("M" * k + "Z" * (npad - k)).add(w)
                        assert self.state() == target and lo <= self.off - c * C < hi
                        if cls:
                            self.mark(cls, state=target, chunk=c, phase=e % 16, **info)
                        return c
                c += 1
        raise RuntimeError("no window found")

    def realize(self, last_len=None):
        """(bytes, manifest); `last_len` cuts the last block to that many bytes. Runs of Z blocks are made as one array."""
        blk = Blocks(self.alg, self.seed)
        parts, i, n = [], 0, self.n
        while i < n:
            j = i
            while j < n and self.letters[j] == "Z":
                j += 1
            if j > i:
                parts.append(blk.z_run(j - i))
                i = j
            else:
                parts.append(blk.block(self.letters[i]))
                i += 1
        data = np.concatenate(parts)
        if last_len is not None:
            data = data[:(self.n - 1) * BS[self.alg] + last_len]
        return data, list(self.manifest)


# ---- the oracle stream, block by block ----------------------------------------------------------------------------------------
def _payload_bytes(alg, sig, nq):
    """Payload bytes of nq quads under signature `sig` (algorithms/*: plain 4, hit / MAP_A / MAP_B 2, PREDICTED 0)."""
    fb = FLAG_BITS[alg]
    flags = [(sig >> (fb * i)) & ((1 << fb) - 1) for i in range(nq)]
    if alg == "chameleon":
        return sum(2 if f else 4 for f in flags)
    if alg == "cheetah":
        return sum((4, 2, 2, 0)[f] for f in flags)
    return sum((4, 0, 0, 0, 0, 0, 2, 2)[f] for f in flags)


Trace = collections.namedtuple("Trace", "off copied inc size state counter n_stream")


def trace(alg, stream, n):
    """Parse an oracle stream of n input bytes block by block (codec.rs:34-70): per block its stream offset, whether it is copied,
    whether it is incompressible (encoded and at least BS bytes), its encoded size and the automaton state (penalty, start, prev)
    and counter in front of it. The automaton runs on the parsed bits."""
    B, S = BS[alg], SIG[alg]
    s = np.asarray(stream, np.uint8)
    nb = (n + B - 1) // B
    off = np.zeros(nb, np.int64)
    copied = np.zeros(nb, bool)
    inc = np.zeros(nb, bool)
    size = np.zeros(nb, np.int64)
    state, counter = [], []
    ps = Protection()
    o = 0
    for b in range(nb):
        blen = min(B, n - b * B)
        state.append(ps.key())
        counter.append(ps.counter)
        off[b] = o
        probe = Protection(ps.penalty, ps.start, ps.prev, ps.counter)
        if probe.step(False):                       # copy mode does not depend on the block's own bit
            ps.step(False)
            copied[b] = True
            size[b] = blen
        else:
            sig = int.from_bytes(bytes(s[o:o + S]), "little")
            size[b] = S + _payload_bytes(alg, sig, blen // 4) + blen % 4
            inc[b] = size[b] >= B
            ps.step(bool(inc[b]))
        o += int(size[b])
    return Trace(off, copied, inc, size, state, counter, o)


Piece = collections.namedtuple("Piece", "label data manifest builder")


# ---- named corpora -----------------------------------------------------------------------------------------------------------
def seam_states_corpus(alg):
    """Each of the seam states at PSEG seams, at tile seams and at run seams (planted.cham_runs / chee_runs on 132 SMs). Z padding
    in between returns the automaton to the canonical state. Manifest: (block, "seam", {state, kinds})."""
    nbytes = {"chameleon": 8 * MIB + 100, "cheetah": 2 * MIB + 50, "lion": MIB + 30}[alg]
    B = BS[alg]
    nblocks = (nbytes + B - 1) // B
    tb = TILE_BLOCKS[alg]
    runs = planted.cham_runs(nbytes) if alg == "chameleon" else planted.chee_runs(nbytes)
    run_seams = {a * (planted.TILE_BYTES // B) for a, _ in runs[1:]}

    def kinds(b):
        k = set()
        if b % PSEG == 0:
            k.add("pseg")
        if b % tb == 0 and (tb == PSEG or b % PSEG):     # tile seams inside a segment where the tiles are shorter
            k.add("tile")
        if b in run_seams:
            k.add("run")
        return k

    todo = {k: list(seam_states()) for k in ("run", "tile", "pseg")}
    bld = Builder(alg, {"chameleon": 11, "cheetah": 12, "lion": 13}[alg])
    step = min(tb, 64)
    for b in range(step, nblocks - 200, step):
        ks = kinds(b)
        kind = next((k for k in ("run", "tile", "pseg") if k in ks and todo[k]), None)
        if kind is None:
            continue
        nxt_run = min([r for r in run_seams if r > b] or [nblocks])
        if kind != "run" and todo["run"] and nxt_run - b < 160:
            continue
        st = todo[kind][0]
        if b - len(word_to(st, b)) < bld.n:
            continue
        for k in ks:
            if st in todo[k]:
                todo[k].remove(st)
        bld.place(b, st, "seam", kinds=tuple(sorted(ks)))
        bld.recover()
    assert not any(todo.values()), {k: len(v) for k, v in todo.items()}
    bld.add("Z" * (nblocks - bld.n))
    return [Piece("seam_states", *bld.realize(nbytes - (nblocks - 1) * B), bld)]


def chunk_entries_corpus(alg):
    """The decoder's geometry (CH stream bytes per chunk, GROUP chunks per group). At chunk and group entries (the first block
    starting in the chunk): penalty 0 with start 2..6 at every counter phase the padding allows (the chunk is then jumped with
    sw_jump's halving count); prev = 1 followed by an incompressible first block (the chunk must be walked); and a copy-mode block
    that straddles a chunk seam for each penalty 1..6. A chunk of Z padding holds at least 3 multiples of 16 blocks, so start <= 6
    always leaves such a jump as 1. An off-by-one in the halving count can only show in Cheetah's 4 KiB chunks (short_jump below);
    Chameleon (at least 63 blocks in a jumped 16 KiB chunk) and Lion (at least 62 in 4 KiB) have no chunk in which it could."""
    bld = Builder(alg, {"chameleon": 21, "cheetah": 22, "lion": 23}[alg])
    bld.add("Z" * 20)
    B = BS[alg]
    reach = reachable_states()
    for s in range(2, 7):
        bld.place_in_window((0, s, 0), 0, ZSIZE[alg], chunk_ok=lambda c: c % GROUP == 0, cls="group_start", start=s)
        bld.recover()
        for ph in range(16):
            if (0, s, 0, ph) not in reach:
                continue
            bld.place_in_window((0, s, 0), 0, ZSIZE[alg], phase=ph, cls="chunk_start", start=s)
            bld.recover()
    for s in (1, 2, 3):
        for group in (False, True):
            bld.place_in_window((0, s, 1), 0, ZSIZE[alg], chunk_ok=(lambda c: c % GROUP == 0) if group else (lambda c: True),
                                cls="forced_walk", group=group)
            bld.add("R")
            bld.recover()
    for p in range(1, 7):
        cands = sorted((len(word_to(st[:3], st[3])), st[:3]) for st in reach if st[0] == p)
        bld.place_in_window(cands[0][1], -B + 2, -1, cls="copy_straddle", penalty=p)
        bld.recover()
    if alg == "cheetah":
        # the one case in which sw_jump's halving count shows (test_protection_cpu.test_where_the_halving_count_shows): start 4..6
        # entering at counter phase 0 a chunk of exactly 31 blocks, which holds two multiples of 16 blocks (start ends at 1) where a
        # count shifted by one block sees one (start 2..3). R and M alternating from an entry at least 30 bytes into the chunk give
        # 31 blocks without two incompressible blocks in a row, so the chunk is jumped; the R that opens the next chunk pairs with
        # the last R and copies as many blocks as the jump left in `start`.
        for s in (4, 5, 6):
            c = bld.place_in_window((0, s, 0), 30, ZSIZE[alg], phase=0, cls="short_jump", start=s)
            k = 0
            while bld.off < (c + 1) * CH[alg]:
                bld.add("RM"[k % 2])
                k += 1
            bld.add("RR")
            bld.recover()
    bld.add("Z" * 40)
    return [Piece("chunk_entries", *bld.realize(), bld)]


def _seam_count_builder(alg, nseams, seed):
    """nseams segments whose outgoing state after round 0 is not canonical: an R R pair right before the segment's end (the
    copy penalty runs into the next segment). Plus a burst inside one segment that settles before its end."""
    bld = Builder(alg, seed)
    bld.add("Z" * 100 + "RR").recover()
    nseg = max(nseams, 1) + 2
    for s in range(1, nseg):
        bld.add("Z" * (s * PSEG - 2 - bld.n))
        if s <= nseams:
            bld.mark("bad_seam", segment=s - 1)
            bld.add("RR")
        bld.recover()
    bld.add("Z" * (nseg * PSEG + 17 - bld.n))
    return bld


def chain_builder(alg, length, seed):
    """`length` consecutive segments of incompressible blocks in Z padding: round 0 leaves every one of their outgoing states
    non-canonical and each depends on the state it is entered with, so `prot_rounds` needs `length` relaxation rounds, more than
    prot_iterate's PROT_FAST_ROUNDS = 4. That is proved for the round-by-round restatement only: prot_iterate reads its predecessor's
    state with __ldcg within a round (chameleon_encode.cu), so a segment may see a value written in the same round and settle sooner
    (the chain's segments sit in neighbouring lanes of one warp, which run in step). No diagnostic of the library says which of the
    relaxation, the candidate tables or the in-order fix-up settled a stream (density_b200_prot_debug counts copy-map changes per
    fixed-point round), so the GPU tests check the stream and the converged copy map, not the path taken."""
    bld = Builder(alg, seed)
    bld.add("Z" * (2 * PSEG))
    bld.mark("chain", length=length)
    bld.add("R" * (length * PSEG))
    bld.recover()
    bld.add("Z" * (PSEG + 3))
    return bld


def seam_counts_corpus(alg):
    out = []
    for k in (0, 1, 8, 9):
        bld = _seam_count_builder(alg, k, 30 + k)
        out.append(Piece(f"seams{k}", *bld.realize(), bld))
    for L in (5, 8):
        bld = chain_builder(alg, L, 40 + L)
        out.append(Piece(f"chain{L}", *bld.realize(), bld))
    return out


def thresholds_builder(alg, control=False):
    """T+ T+, T+ T-, T- T+, T+ R and R T+ pairs and D blocks, each once inside a segment and once across a PSEG or tile seam. A D
    block follows R R S: its S is copied, D is T+, and the pair (D, R) copies the block after it, which round 0 (nothing copied: S
    encoded, D = T-) does not. `control`: the R R in front of every S are Z Z, so S is encoded and D is T-."""
    bld = Builder(alg, {"chameleon": 51, "cheetah": 52, "lion": 53}[alg])
    bld.add("Z" * 30)
    tb = min(TILE_BLOCKS[alg], PSEG // 2)
    k = 0
    for pair in ("PP", "PM", "MP", "PR", "RP"):
        for at_seam in (False, True):
            if at_seam:                     # the pair's second block opens a segment (even k) or a tile inside one (odd k)
                unit = PSEG if k % 2 == 0 else tb
                b = (bld.n // PSEG + 1) * PSEG + (0 if unit == PSEG else tb)
                k += 1
                bld.add("Z" * (b - 1 - bld.n))
            bld.mark("pair_" + pair, seam=at_seam)
            bld.add(pair)
            bld.recover()
            bld.add("Z" * 20)
    for at_seam in (False, True, True):
        if at_seam:
            bld.add("Z" * ((bld.n // PSEG + 1) * PSEG - 3 - bld.n))
        bld.add("ZZ" if control else "RR")
        bld.mark("S")
        bld.add("S")
        bld.mark("D", seam=at_seam)
        bld.add("DR")
        bld.recover()
        bld.add("Z" * 30)
    return bld


def tails_builders(alg):
    """Streams that end in copy mode or with a penalty pending, for last-block lengths 1, 2, 3, 4, 5, BS - 1 and BS, with the decoder's
    main / tail handover (the first block with fewer than SIG + BS stream bytes left) right before, on and right after a copy-mode
    block:  end_copy  ... R R X      the last block is copied (handover on it)
            end_run   ... R R X X    start 2: the last two blocks are copied
            pending   ... R R        the last block is the second of an incompressible pair (pending when it is incompressible)
            after     ... R P X      P is exactly BS: with a last block under SIG bytes the handover is on P, the copy after it
            encoded   ... R R X Z    the copy-mode block is the last one of the main loop
    Yields (label, builder, last block length)."""
    B = BS[alg]
    for L in (1, 2, 3, 4, 5, B - 1, B):
        for kind, tail in (("end_copy", "RRZ"), ("end_run", None), ("pending", "RR"), ("after", "RPZ"), ("encoded", "RRZZ")):
            bld = Builder(alg, 60 + L)
            bld.add("Z" * (40 + L % 16))
            if tail is None:
                bld.place(bld.n + 20, (2, 2, 1), "end_run_pair")
                tail = "ZZ"
            bld.mark("tail_" + kind, last_len=L)
            bld.add(tail)
            yield f"{kind}_{L}", bld, L


def pipelined_builders():
    """Chameleon only, 96 MiB + a few bytes through the host pipeline (64 MiB chunks): an R only as the last block of the first chunk,
    an R only as the first block of the second chunk, and an R R pair straddling the cut."""
    B = BS["chameleon"]
    cut = 64 * MIB // B
    nblocks = 96 * MIB // B + 1
    for kind, at in (("last_of_first", ("R", cut - 1)), ("first_of_second", ("R", cut)), ("pair_across", ("RR", cut - 1))):
        bld = Builder("chameleon", 70 + len(kind))
        bld.add("Z" * (at[1] - 40))
        bld.add("Z" * 40)
        bld.mark("pipelined_" + kind, cut=cut)
        bld.add(at[0])
        bld.recover()
        bld.add("Z" * (nblocks - bld.n))
        yield kind, bld, 77


def thresholds_pieces(alg):
    bld = thresholds_builder(alg)
    return [Piece("thresholds", *bld.realize(), bld)]


def tails_pieces(alg):
    return [Piece(label, *bld.realize(L), bld) for label, bld, L in tails_builders(alg)]


def pipelined_pieces(alg):
    assert alg == "chameleon"
    return [Piece(label, *bld.realize(L), bld) for label, bld, L in pipelined_builders()]


# name -> alg -> [Piece(label, bytes, manifest, builder)]; every corpus exists for every algorithm except `pipelined` (Chameleon only)
CORPORA = {
    "seam_states": seam_states_corpus,
    "chunk_entries": chunk_entries_corpus,
    "seam_counts": seam_counts_corpus,
    "thresholds": thresholds_pieces,
    "tails": tails_pieces,
    "pipelined": pipelined_pieces,
}
_cache = {}


def corpus(name, alg):
    """[Piece(label, bytes, manifest, builder)] of a named corpus, built once per process."""
    if (name, alg) not in _cache:
        _cache[(name, alg)] = CORPORA[name](alg)
    return _cache[(name, alg)]


_encoded = {}


def oracle_stream(name, alg, label):
    """(bytes, oracle stream, trace) of one piece of a named corpus."""
    key = (name, alg, label)
    if key not in _encoded:
        data = next(p.data for p in corpus(name, alg) if p.label == label)
        enc = oracle.encode(alg, data)
        _encoded[key] = (data, enc, trace(alg, enc, data.size))
    return _encoded[key]
