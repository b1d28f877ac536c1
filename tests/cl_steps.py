"""Collision steps for the run-parallel Cheetah and Lion encoders: whole 32-quad warp steps in one hash bucket (numpy only).

chee_pass_p, chee_pass_c and lion_pass_p (density_b200/csrc/cheetah_encode.cu) decide inside one 32-quad step with __match_any_sync
groups, a rank loop per group and first-lane / last-lane ownership of the run's table entries; the folds then resolve the accesses a run
left undecided against the state carried in. Text rarely puts more than one value of one bucket into a step. A COLLISION STEP here is
32 quads of one bucket h (lanes 1-31 then share context h as well), or of two buckets, alternating (two 16-lane context groups) or one
per 16-lane half (one per Lion block). Its values follow one of PATTERNS, and the bucket's state in front of it is one of STATES:

  fresh       untouched before the step
  one / two   one value / two values (a, b) accessed earlier in the same run
  pred        context h written earlier in the run with the value of lane 1 (bucket g): a predicted hit from the run's table
  prev_two / prev_pred   the same, but only in an earlier run: the folds resolve the step's first accesses (u1, u2 from one step)
  list5 / prev_list5     (the undecided patterns) context h holds five values c4..c0 of bucket g, written earlier in the run / in an
                         earlier run; the odd lanes (bucket g, context h) make five undecided accesses and miss a full list

Collision steps go at the first, middle and last step of every run of `planted.chee_runs` (H100 geometry), at a group split across steps
s and s + 1 (s + 1 even, so a 256-byte cut falls between the halves), at two-bucket steps, at the last partial step of the stream and
behind copy-mode episodes; bucket 0 (quad 0 and quad_of(0, f)) goes at the stream start and later. Buckets come from the Planter's
pool of buckets the base text never touches, and every step is preceded by a LEAD quad of a fresh bucket, so the state in front of every
planted quad is the one the generator chose.

`build(name)` returns (bytes, manifest, planted buckets). A manifest entry is (quad index, quad, class, position, role, step, intent):
role "step", "prefix" (the state planted in front) or "lead"; intent (Cheetah flag, Lion flag) is what the planting is for (the MAP_B of
an ab chain, the PREDICTED of a pred state, the Lion depth of a cycle, the five undecided accesses of undec5, ...; None where a value has
no purpose of its own, MISS for "not predicted"). tests/test_cl_steps_cpu.py asserts the intents against the oracle's stream, so a later
edit cannot silently drop what a planting is for. `intended(alg, data, manifest, buckets, copied)` restates the two codecs in order over
the planted buckets and contexts, a consistency check of every planted flag.
"""
import numpy as np

import planted
from lion_streams import Prot
from planted import MIB, TILE_QUADS, Planter, hf, quad_of, twin

STEP = 32
PATTERNS = ("a1", "ab", "abc", "cyc4", "alpha5", "cyc6", "abba", "twin", "fp0", "alpha32")
ALPHABET = {"a1": 1, "ab": 2, "abc": 3, "cyc4": 4, "alpha5": 5, "cyc6": 6, "abba": 2, "twin": 1, "fp0": 2, "alpha32": 32}
STATES = ("fresh", "one", "two", "pred", "prev_two", "prev_pred")
LIST_PATTERNS = ("undec5", "undec_rep")
LIST_STATES = ("list5", "prev_list5")
CLASSES = [f"{p}.{s}" for p in PATTERNS for s in STATES] + [f"{p}.{s}" for p in LIST_PATTERNS for s in LIST_STATES]
SINGLE = ("run_first", "split", "run_mid", "run_last")
COPY = -1                                            # intended flag of a quad in a copy-mode block


def _same_run(state):
    return state in ("one", "two", "pred", "list5")


MISS = -2                                            # intent: a Lion quad that is not predicted (any flag but 1-5)


def _pattern_intent(pat, seq, j):
    """(Cheetah flag, Lion flag) the j-th value of one bucket's sequence in a step is meant to get from the in-step values in front of it
    (None: no intent); from j = 2 on the value's nearest lower lane of its context group holds seq[j - 1] in every layout"""
    if j < 2:
        return None, None
    same = seq[j] == seq[j - 1]
    if pat == "a1":
        return 3, 1                                  # predicted by the nearest lower lane
    if pat in ("ab", "twin"):
        return (2, 2) if j >= 3 else (None, None)    # MAP_B chain; Lion depth 1
    if pat in ("abc", "cyc4", "alpha5", "cyc6"):
        L = ALPHABET[pat]
        return 0, ((L if L < 6 else 0) if j >= L + 1 else None)      # Lion: depth L - 1; the sixth value misses a full list
    if pat == "alpha32":
        return 0, 0
    if pat == "abba":
        return (3, 1) if same else ((2, 2) if j >= 5 else (None, None))
    if pat == "fp0":
        if j % 2:
            return (2, 2) if j >= 3 else (None, None)  # the fingerprint-0 member from the MAP_B slot; Lion depth 1
        return 0, (3 if j >= 6 else None)
    return None, None


UNDEC = {   # per value of the context-h group: the sequence over c0..c4 (in the list of h) and new values n0..n2, and the Lion flags
    "undec5": (["c4", "n0", "c2", "c3", "n1", "c0", "c1", "n0", "c4", "c2", "n2", "c3", "c0", "n1", "c1", "c4"],
               [1, MISS, 4, 4, MISS, MISS]),   # five undecided accesses (depth 0, miss, depth 3, depth 3, miss), a miss on a full list
    "undec_rep": (["n0", "c3", "n0", "c1", "c4", "n1", "c2", "c0", "n2", "c3", "n1", "c4", "c1", "n0", "c2", "c0"],
                  [MISS, 3, 2, 5, 4]),         # n0 again inside the undecided stretch: a local hit at depth 1
}


class _Gen:
    def __init__(self, P):
        self.P, self.man, self.S, self.sid = P, {}, {0}, 0
        self.deps = {}                                # step -> quads planted by other steps that its intents rely on

    def bucket(self):
        h = self.P.bucket()
        self.S.add(h)
        return h

    def put(self, pos, v, cls, where, role, want=(None, None)):
        assert 0 <= pos < self.P.nq and pos not in self.man, (pos, cls, where)
        self.P.q[pos] = v
        self.man[pos] = (int(v), cls, where, role, self.sid, want)

    def fps(self, n):
        """n distinct even fingerprints other than 0 (their bit-0 twins stay unused unless a pattern asks for them)"""
        return [2 * int(x) for x in self.P.rng.choice(np.arange(1, 0x7FFF), n, replace=False)]

    def seq(self, pat, h, n, values=None):
        """(values of n lanes, alphabet)"""
        a = values or [quad_of(h, f) for f in self.fps(ALPHABET[pat])]
        if pat == "abba":
            cyc = [a[0], a[1], a[1], a[0]]
        elif pat == "twin":
            cyc = [a[0], twin(a[0])]
        elif pat == "fp0":
            cyc = [a[0], quad_of(h, 0), a[1], quad_of(h, 0)]
        else:
            cyc = a
        return [cyc[k % len(cyc)] for k in range(n)], a

    def new(self, h):
        return quad_of(h, self.fps(1)[0] | 1)         # odd fingerprints: never one of an alphabet's values

    def lead(self, pos, where):
        if pos >= 0 and pos not in self.man:          # a planted quad in front is as good a context: the last step of the run before
            self.put(pos, quad_of(self.bucket(), self.fps(1)[0]), "lead", where, "lead")

    def step(self, p, n, cls, where, same_at, prev_at, layout="one"):
        """a collision step of class `cls` on quads p .. p + n - 1; its prefixes at same_at (same run) or prev_at (an earlier run). The
        prediction and list states take the alternating layout: a context h can only keep a planted value that is not of bucket h (the
        quad behind an h-quad always writes context h), so the odd lanes (bucket g) are the ones in context h."""
        pat, state = cls.split(".")
        base = state.replace("prev_", "")
        at = same_at if _same_run(state) else prev_at
        if base in ("pred", "list5"):
            layout = "alt2"
        self.sid += 1
        self.lead(p - 1, where)
        if layout == "one":
            lanes_of = [list(range(n))]
        elif layout == "alt2":
            lanes_of = [list(range(0, n, 2)), list(range(1, n, 2))]
        else:                                         # halves
            lanes_of = [list(range(min(16, n))), list(range(16, n))]
        lanes_of = [x for x in lanes_of if x]
        hs = [self.bucket() for _ in lanes_of]
        if pat in UNDEC:                              # w0 c0 w1 c1 .. w4 c4: context h holds c4 c3 c2 c1 c0 (h = hs[0], c of bucket g = hs[1])
            names, lflags = UNDEC[pat]
            h, g = hs
            vals = {f"c{k}": quad_of(g, f) for k, f in enumerate(self.fps(5))}
            vals.update({f"n{k}": self.new(g) for k in range(3)})
            for k in range(5):
                self.put(at + 2 * k, self.new(h), cls, where, "prefix")
                self.put(at + 2 * k + 1, vals[f"c{k}"], cls, where, "prefix")
            for j, l in enumerate(lanes_of[0]):
                self.put(p + l, self.new(h), cls, where, "step")
            for j, l in enumerate(lanes_of[1]):
                nm = names[j]
                want = (3 if pat == "undec5" and j == 0 else None, lflags[j] if j < len(lflags) else None)
                self.put(p + l, vals[nm], cls, where, "step", want)
            return
        seqs = [self.seq(pat, h, len(lanes)) for h, lanes in zip(hs, lanes_of)]
        if base == "pred":                            # x of bucket h, then the value of lane 1 (bucket g): context h predicts lane 1
            self.put(at, self.new(hs[0]), cls, where, "prefix")
            self.put(at + 1, seqs[1][0][0], cls, where, "prefix")
        for k, (h, lanes, (vals, alphabet)) in enumerate(zip(hs, lanes_of, seqs)):
            if base == "one":
                self.put(at - 20 * k, alphabet[0], cls, where, "prefix")
            elif base == "two":
                self.put(at - 20 * k, alphabet[1] if len(alphabet) > 1 else self.new(h), cls, where, "prefix")
                self.put(at - 20 * k + 3, alphabet[0], cls, where, "prefix")
            for j, (l, v) in enumerate(zip(lanes, vals)):
                want = _pattern_intent(pat, vals, j)
                if j == 0 and base == "fresh":
                    want = (0, 0)
                elif j == 0 and base in ("one", "two"):
                    want = (1, 6)                     # MAP_A of the value known in front (resolved by the fold for prev_two)
                elif j == 1 and base == "two" and len(alphabet) > 1 and v == alphabet[1]:
                    want = (2, 7)                     # MAP_B of the other value (prev_two: u2 of the same step as u1)
                elif j == 0 and base == "pred" and k == 1:
                    want = (3, 1)                     # predicted from the run's table entry (prev_pred: from chee_fold_p through u1)
                self.put(p + l, v, cls, where, "step", want)

    def zero_step(self, p, n, where):
        """bucket 0: quad 0 and two members quad_of(0, f): the stream start's zero lists and (quad 0, quad 0) chunk map"""
        f1, f2 = self.fps(2)
        F1, F2 = quad_of(0, f1), quad_of(0, f2)
        base = [0, 0, F1, 0, F2, 0, F1, F2, F2, 0, 0, F1]
        # at the stream start: quad 0 predicted twice (pred 0 / five zeros), F1 PLAIN, then quad 0 from the chunk map's b slot (MAP_B) and
        # from Lion's list at depth 1
        wants = [(3, 1), (3, 1), (0, 0), (2, 2)] if p == 0 else []
        self.sid += 1
        self.lead(p - 1, where)
        for l in range(n):
            self.put(p + l, base[l % len(base)], "bucket0", where, "step", wants[l] if l < len(wants) else (None, None))


class _Cycle:
    """the classes in order, per position, skipping those a position cannot hold"""

    def __init__(self):
        self.k = {}

    def next(self, where, ok):
        while True:
            k = self.k.get(where, 0)
            self.k[where] = k + 1
            c = CLASSES[k % len(CLASSES)]
            if ok(c.split(".")[1]):
                return c


def steps_corpus(nbytes, seed, bucket0_later=False):
    """dickens text with collision steps at every run's first, split, middle, two-bucket and last step and at the last partial step;
    bucket 0 at the stream start (and, with bucket0_later, not before the middle of run 1)"""
    P = Planter(nbytes, seed)
    G, C = _Gen(P), _Cycle()
    nq = P.nq
    runs = [(a * TILE_QUADS, min(b * TILE_QUADS, nq)) for a, b in planted.chee_runs(nbytes)]
    tail0 = nq // STEP * STEP
    for r, (S, E) in enumerate(runs):
        last = (E - 1) // STEP * STEP if E < nq else tail0 - STEP
        mid = S + (E - S) // 2 // 64 * 64
        spots = [("run_first", S), ("split", S + 1008), ("run_mid", mid), ("alt2" if r % 2 else "halves", S + 3328), ("run_last", last)]
        for k, (where, p) in enumerate(spots):
            if r == 0 and where == "run_first":
                if not bucket0_later:
                    G.zero_step(0, STEP, "stream_start")
                continue
            if r == 1 and where == "run_mid" and bucket0_later:
                G.zero_step(p, STEP, "bucket0_later")
                continue
            ok = lambda st: (r > 0 or not st.startswith("prev")) and (where != "run_first" or not _same_run(st))
            cls = C.next(where, ok)
            layout = where if where in ("alt2", "halves") else "one"
            G.step(p, STEP, cls, where, p - 200, S - 1000 - 100 * k, layout)
    if nq > tail0:                                    # the last partial step
        S = runs[-1][0]
        G.step(tail0, nq - tail0, C.next("tail", lambda st: st in ("fresh", "two", "prev_two")), "tail", tail0 - 200, S - 1500)
    return P.data, _entries(G)


# mostly-PLAIN patterns between mostly-hit ones: a Cheetah block of 30 PLAIN quads is incompressible, and two of them in a row would hide
# the next block in copy mode; "pred" is a two-bucket step whose lane 1 is the quad that followed the last quad of lane 0's bucket
PURE_ORDER = ("abc", "a1", "cyc4", "ab", "alpha5", "abba", "pred", "cyc6", "twin", "alpha32", "fp0", "pred", "a1", "ab")


def pure_corpus(nbytes, seed, pool=4096):
    """only collision steps: every step is one or two buckets of a pool of `pool` buckets, each with 32 values, so every step has large
    groups and states carried from step to step and run to run; bucket 0 joins from the middle of the stream on. The "pred" steps are
    predicted at lane 1 from the table entry of lane 0's bucket, written in the same run or (through chee_fold_p) in an earlier one."""
    rng = np.random.default_rng(seed)
    data = np.zeros(nbytes, np.uint8)
    P = Planter(nbytes, seed, data)
    P.free = [int(x) for x in rng.permutation(np.arange(1, 65536))]
    P.free_set = set(P.free)
    G = _Gen(P)
    hs = [G.bucket() for _ in range(pool)]
    vals = {h: [quad_of(h, f) for f in G.fps(32)] for h in hs}
    hq = lambda x: ((x * planted.M) & 0xFFFFFFFF) >> 16
    succ = {}                                        # bucket -> the quad that followed its last quad (what its context predicts)
    nq = P.nq
    k = 0
    for p in range(0, nq, STEP):
        n = min(STEP, nq - p)
        pat = PURE_ORDER[k % len(PURE_ORDER)]
        G.sid += 1
        if p == nq // 2 // STEP * STEP:
            G.zero_step(p, n, "bucket0_later")
        elif pat == "pred" and n == STEP:
            while True:
                h = hs[int(rng.integers(pool))]
                if h in succ and hq(succ[h][1]) not in (h, 0) and hq(int(P.q[p - 1])) != h:
                    break
            G.deps[G.sid] = [succ[h][0] - 1, succ[h][0]]
            y = succ[h][1]
            g = hq(y)
            other = next(v for v in vals[g] if v != y)
            for l in range(n):
                if l % 2 == 0:
                    G.put(p + l, vals[h][(l // 2) % 2], "ab.pure_pred", "alt2", "step")
                else:
                    G.put(p + l, (y, other)[(l // 2) % 2], "ab.pure_pred", "alt2", "step", (3, None) if l == 1 else (None, None))
        else:
            pat = "a1" if pat == "pred" else pat
            where = ("pure", "alt2", "pure", "halves")[k % 4]
            lanes_of = [list(range(n))] if where == "pure" else ([list(range(0, n, 2)), list(range(1, n, 2))] if where == "alt2" else
                                                                [list(range(min(16, n))), list(range(16, n))])
            for h, lanes in zip(rng.choice(hs, 2, replace=False).tolist(), lanes_of):
                if not lanes:
                    continue
                v = vals[h][int(rng.integers(32)):] + vals[h]
                seq, _ = G.seq(pat, h, len(lanes), v[:32] if pat == "alpha32" else v[:ALPHABET[pat]])
                for j, (l, x) in enumerate(zip(lanes, seq)):
                    c, lf = _pattern_intent(pat, seq, j)
                    lf = None if pat == "alpha32" else lf     # the pool's values recur: Lion lists may still hold them
                    G.put(p + l, x, f"{pat}.pure", "tail" if n < STEP else where, "step", (c, lf))
        for i in range(max(p, 1), p + n):
            succ[hq(int(P.q[i - 1]))] = (i, int(P.q[i]))
        k += 1
    return P.data, _entries(G)


def copy_corpus(nbytes, seed, every=32 << 10):
    """dickens text with a 512-byte incompressible burst every `every` bytes, and collision steps (and Lion halves) at 0 .. 14 steps
    behind each burst: the copy-mode episodes the bursts start end in front of some of them, and in the middle of a Lion step in front of
    others. The burst quads are random members of buckets the text uses, so the planted buckets stay fresh."""
    data = planted.base_text(nbytes)
    P = Planter(nbytes, seed, data)
    used = np.flatnonzero(~np.isin(np.arange(65536), list(P.free_set)))
    used = used[used != 0]
    G, C = _Gen(P), _Cycle()
    rng = np.random.default_rng(seed + 5)
    for j, B in enumerate(range(every, nbytes - every, every)):
        b4 = B // 4
        n = 128
        hs, fs = rng.choice(used, n), rng.integers(1, 0xFFFE, n)
        P.q[b4:b4 + n] = [quad_of(int(h), int(f)) for h, f in zip(hs, fs)]
        for s in range(8):
            p = b4 + n + 2 * STEP * s + (16 if (j + s) % 3 == 2 else 0)     # some start in the middle of a step: a Lion half
            cls = C.next("after_copy", lambda st: st in ("fresh", "one", "two", "pred", "list5"))
            G.step(p, STEP, cls, "after_copy", b4 - 400 - 40 * s, None, "halves" if s % 4 == 3 else "one")
    G.zero_step(nbytes // 4 // 2 // STEP * STEP, STEP, "bucket0_later")
    return P.data, _entries(G)


def _entries(G):
    return sorted((p, *e) for p, e in G.man.items()), sorted(G.S), G.deps


CORPORA = {
    "cls1": lambda: steps_corpus(MIB + 13, 21),
    "cls33": lambda: steps_corpus(33 * MIB + 66, 22),     # 1056 runs on an H100; the last step is 16 quads + 2 bytes
    "cls_pure": lambda: pure_corpus(4 * MIB + 30, 23),    # the last step is 7 quads + 2 bytes
    "cls_copy": lambda: copy_corpus(2 * MIB + 5, 24),
}
_cache = {}


def build(name):
    """(bytes, manifest, planted buckets) of a named corpus, built once per process"""
    if name not in _cache:
        data, (man, S, deps) = CORPORA[name]()
        _cache[name] = (data, man, S, deps)
    return _cache[name][:3]


def checked_intents(alg, name, flags):
    """[(manifest entry, flag in the stream, intended flag)] of the entries with an intent whose step (its quads, its prefix, its lead and
    the quads it relies on) is not in copy mode: copy-mode blocks take quads out of the context chain and the tables"""
    build(name)
    data, man, S, deps = _cache[name]
    got = flags[[e[0] for e in man]]
    dirty = {e[5] for e, g in zip(man, got) if g == COPY}
    dirty |= {sid for sid, ps in deps.items() if (flags[ps] == COPY).any()}
    k = 0 if alg == "cheetah" else 1
    return [(e, int(g), e[6][k]) for e, g in zip(man, got) if e[6][k] is not None and e[5] not in dirty]


def meets(flag, want):
    return flag not in (1, 2, 3, 4, 5) and flag != COPY if want == MISS else flag == want


# ---- reading a stream back, and the flags the plantings are meant to get ------------------------------------------------------------
BS = {"cheetah": 128, "lion": 64}
SIGB = {"cheetah": 8, "lion": 6}
FB = {"cheetah": 2, "lion": 3}
PAY = {"cheetah": (4, 2, 2, 0), "lion": (4, 0, 0, 0, 0, 0, 2, 2)}


def stream_flags(alg, enc, nbytes):
    """(flag per quad, COPY in copy-mode blocks; copy mode per block) of a Cheetah / Lion stream of `nbytes` input bytes: every block of
    the encoder's loop (codec.rs:34-80), the protection automaton replayed as the encoder runs it. Raises if the stream does not end
    where the last block does."""
    bs, sb, fb = BS[alg], SIGB[alg], FB[alg]
    qpb = bs // 4
    nblocks = (nbytes + bs - 1) // bs
    by12 = np.array(PAY[alg])[(np.arange(1 << 12)[:, None] >> (fb * np.arange(12 // fb))[None, :]) & ((1 << fb) - 1)].sum(axis=1).tolist()
    buf = bytes(np.asarray(enc, np.uint8))
    ng = (fb * qpb + 11) // 12                        # 12-bit groups per signature; the flags past nqb in them read as PLAIN
    ps, idx = Prot(), 0
    copied = np.zeros(nblocks, bool)
    sigs = np.zeros(nblocks, np.uint64)
    for b in range(nblocks):
        blen = min(bs, nbytes - b * bs)
        if ps.revert():
            copied[b] = True
            idx += blen
            ps.decay()
            continue
        sig = int.from_bytes(buf[idx:idx + sb], "little")
        nqb = blen // 4
        s = sig & ((1 << (fb * nqb)) - 1)
        sz = sb + sum(by12[(s >> (12 * k)) & 4095] for k in range(ng)) - (ng * 12 // fb - nqb) * PAY[alg][0] + (blen & 3)
        sigs[b] = sig
        idx += sz
        ps.update(blen == bs and sz >= bs)
    assert idx == len(buf), (alg, idx, len(buf))
    sh = (fb * np.arange(qpb, dtype=np.uint64))[None, :]
    fl = ((sigs[:, None] >> sh) & np.uint64((1 << fb) - 1)).astype(np.int8)
    fl[copied] = COPY
    return fl.reshape(-1)[:nbytes // 4], copied


def intended(alg, data, manifest, S, copied):
    """The flag of every manifest entry (Cheetah 0 PLAIN, 1 MAP_A, 2 MAP_B, 3 PREDICTED; Lion 0 PLAIN, 1-5 PREDICTED at depth 0-4,
    6 MAP_A, 7 MAP_B; COPY in a copy-mode block), given the copy map: cheetah.rs:121-150 / lion.rs:209-271 in order, over the quads whose
    context or bucket is planted only, plus every quad of the unplanted contexts at which a planted value occurs a second time."""
    nq = data.size // 4
    q = data[:nq * 4].view(np.uint32)
    h = hf(q)[0]
    qpb = BS[alg] // 4
    enc = ~np.repeat(copied, qpb)[:nq]
    idx = np.flatnonzero(enc)
    ctx = np.zeros(nq, np.int64)
    ctx[idx[1:]] = h[idx[:-1]]
    Ss = set(int(x) for x in S)
    extra = set()                                     # unplanted contexts that meet a planted value again: simulated in full
    while True:
        keys = np.array(sorted(Ss | extra))
        sel = idx[(np.isin(h, keys) | np.isin(ctx, keys))[idx]]
        flag, more = _inorder(alg, sel, q[sel].tolist(), h[sel].tolist(), ctx[sel].tolist(), Ss, Ss | extra)
        if not more:
            break
        extra |= more
    return np.array([COPY if not enc[p] else flag[p] for p, *_ in manifest], np.int8)


def _inorder(alg, sel, ql, hl, cl, Ss, known):
    """flags of the selected quads; the unplanted contexts at which a planted value occurs again (their tables are not simulated)"""
    tab, cmap, seen, flag, more = {}, {}, {0}, {}, set()   # quad 0 is in every untouched context
    for i, v, hb, c in zip(sel.tolist(), ql, hl, cl):
        code = 0
        if c in known:
            if alg == "cheetah":
                code = 3 if tab.get(c, 0) == v else 0
                tab[c] = v
            else:
                L = tab.setdefault(c, [0, 0, 0, 0, 0])
                if v in L:
                    k = L.index(v)
                    code = k + 1
                    del L[k]
                else:
                    L.pop()
                L.insert(0, v)
        elif v in seen:
            more.add(c)
        if hb in Ss:
            seen.add(v)
            if code == 0:
                a, b = cmap.get(hb, (0, 0))                 # the chunk map starts as (quad 0, quad 0) (cheetah.rs:52)
                if v == a:
                    code = 1 if alg == "cheetah" else 6
                else:
                    code = (2 if alg == "cheetah" else 7) if v == b else 0
                    cmap[hb] = (v, a)
        flag[i] = code
    return flag, more
