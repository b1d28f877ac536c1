"""CPU model of the sharded Cheetah / Lion encode (cheetah_encode.cu: the run tables, the shard transfers, their composition and the
folds with a carry-in), checked against an in-order model of the encoders' tables: for cuts at multiples of 256 bytes, the state folded
from the shard transfers equals the in-order tables at the cut, and the flags the runs resolve from it equal the in-order flags.
Copy mode is left out: the algebra is the same on the encoded quads, and only the first shard, which has no carry-in, may use it."""
import numpy as np
import pytest

import planted
from conftest import GOLDEN_DIR, splitmix_bytes

M = 0x9D6EF916
INV = 0x10000                       # FP_INVALID: a fingerprint that matches nothing


def hf(q):
    p = (q * M) & 0xFFFFFFFF
    return p >> 16, (p & 0xFFFE) | (q >> 31)


def quads(data):
    return [int(v) for v in data[:data.size // 4 * 4].view(np.uint32)]


# ---- in-order model (cheetah.rs:121-150, lion.rs:209-271 without the protection automaton) ---------------------------------------
def inorder(lion, qs, stop):
    """flags per quad (('P', depth) / 'A' / 'B' / 'plain') and the tables after quad `stop` for every stop: {stop: (P, C)}."""
    pred, chunk, ctx, flags, snaps = {}, {}, 0, [], {}
    stops = set(stop)
    for i, q in enumerate(qs):
        if i in stops:
            snaps[i] = (dict(pred), dict(chunk))
        lst = pred.get(ctx, [0] * 5 if lion else 0)
        hit = None
        if lion:
            if q in lst:
                hit = lst.index(q)
                pred[ctx] = [q] + lst[:hit] + lst[hit + 1:]
            else:
                pred[ctx] = [q] + lst[:4]
        else:
            hit = 0 if lst == q else None
            pred[ctx] = q
        h, f = hf(q)
        if hit is not None:
            flags.append(("P", hit))
        else:
            a, b = chunk.get(h, (0, 0) if h == 0 else (INV, INV))
            flags.append("A" if f == a else "B" if f == b else "plain")
            if f != a:
                chunk[h] = (f, a)
        ctx = h
    if len(qs) in stops:
        snaps[len(qs)] = (dict(pred), dict(chunk))
    return flags, snaps


# ---- run tables (pass P / pass C of one run) --------------------------------------------------------------------------------------
def run_pass_p(lion, qs, lo, hi, ctx0):
    """per context: Cheetah {last quad, index of the first (undecided) access}; Lion {local list, indices of the undecided accesses}.
    Returns (table, local flags {i: flag})."""
    tab, flags, ctx = {}, {}, ctx0
    for i in range(lo, hi):
        q = qs[i]
        if lion:
            loc, und = tab.setdefault(ctx, ([], []))
            if q in loc:
                k = loc.index(q)
                flags[i] = ("P", k)
                loc.insert(0, loc.pop(k))
            else:
                if len(loc) < 5:
                    und.append(i)
                loc.insert(0, q)
                del loc[5:]
        else:
            if ctx in tab:
                if tab[ctx][0] == q:
                    flags[i] = ("P", 0)
                tab[ctx] = (q, tab[ctx][1])
            else:
                tab[ctx] = (q, i)
        ctx = hf(q)[0]
    return tab, flags


def run_pass_c(qs, lo, hi, predicted):
    """per bucket on the not-predicted quads: (T, a, b, u1, u2) as chee_pass_c keeps it"""
    tab, flags = {}, {}
    for i in range(lo, hi):
        if i in predicted:
            continue
        h, v = hf(qs[i])
        T, a, b, u1, u2 = tab.get(h, (0, 0, 0, None, None))
        if T == 0:
            tab[h] = (1, v, 0, i, None)
        elif T == 1:
            if v == a:
                flags[i] = "A"
            else:
                tab[h] = (2, v, a, u1, i)
        else:
            if v == a:
                flags[i] = "A"
            else:
                if v == b:
                    flags[i] = "B"
                tab[h] = (2, v, a, u1, u2)
    return tab, flags


# ---- transfers: run -> transfer, compose (lion_t_compose, chunk_t_compose), stream-start states -----------------------------------
def lion_compose(x, y):
    """x then y; a transfer is (local list, undecided values); a concrete list is (list of 5, [])"""
    lit, und = list(x[0]), list(x[1])
    for k, v in enumerate(y[1]):
        vis = 5 - k
        lim = min(len(lit), vis)
        if v in lit[:lim]:
            lit.pop(lit[:lim].index(v))
        elif len(lit) < vis:
            und.append(v)
    return list(y[0]) + lit[:5 - len(y[0])], und


def chunk_compose(x, y):
    T, a, b = x
    T2, a2, b2 = y
    if T2 == 0:
        return x
    if T2 == 2:
        return y
    if T == 0:
        return (1, a2, 0)
    return (T, a, b) if a2 == a else (2, a2, a)


def p_init(lion):
    return ([0] * 5, []) if lion else 0


def c_init(h):
    return (2, 0, 0) if h == 0 else (2, INV, INV)


# ---- fold with a carry-in (chee_fold_p / lion_fold_p / chee_fold_c): resolve a run's undecided accesses, carry the state on --------
def fold_p_run(lion, qs, tab, carry, flags):
    """carry: {ctx: concrete state}; updates carry and flags in place"""
    for ctx, e in tab.items():
        if lion:
            loc, und = e
            c = list(carry.get(ctx, p_init(True)[0]))
            for k, i in enumerate(und):
                vis = 5 - k
                if qs[i] in c[:vis]:
                    j = c[:vis].index(qs[i])
                    flags[i] = ("P", k + j)
                    c.pop(j)
                    c.append(c[-1] if c else 0)
            carry[ctx] = list(loc) + c[:5 - len(loc)]
        else:
            q, i = e
            if qs[i] == carry.get(ctx, 0):
                flags[i] = ("P", 0)
            carry[ctx] = q


def fold_c_run(qs, tab, carry, flags):
    for h, (T, a, b, u1, u2) in tab.items():
        a0, b0 = carry.get(h, c_init(h)[1:])
        v1 = hf(qs[u1])[1]
        if v1 == a0:
            flags[u1] = "A"
            bafter = b0
        else:
            if v1 == b0:
                flags[u1] = "B"
            bafter = a0
        if T == 2:
            if hf(qs[u2])[1] == bafter:
                flags[u2] = "B"
            carry[h] = (a, b)
        elif v1 != a0:
            carry[h] = (v1, a0)


def run_cuts(lo, hi, k):
    """k uneven runs over [lo, hi)"""
    n = hi - lo
    pts = sorted({lo + n * j * j // (k * k) for j in range(k)} | {hi})
    return list(zip(pts[:-1], pts[1:])) if n else []


def sharded_model(lion, qs, qcuts, nruns=3):
    """the three phases of every shard and the two folds; returns (flags, carry-ins per shard as {ctx: state}, {h: (a, b)})"""
    W = len(qcuts) - 1
    flags = {}
    runs = [run_cuts(qcuts[r], qcuts[r + 1], nruns) for r in range(W)]
    # phase 1: ctx0 from the previous shard's last quad, run tables, the shard's P transfer composed over its runs
    tabs_p, tp = [], []
    for r in range(W):
        shard_tabs = []
        for lo, hi in runs[r]:
            ctx0 = hf(qs[lo - 1])[0] if lo > 0 else 0      # the previous quad, in this shard or (across the cut) in the one before
            tab, fl = run_pass_p(lion, qs, lo, hi, ctx0)
            flags.update(fl)
            shard_tabs.append(tab)
        t = {}
        for tab in shard_tabs:
            for ctx, e in tab.items():
                if lion:
                    y = (list(e[0]), [qs[i] for i in e[1]])
                    t[ctx] = lion_compose(t.get(ctx, ([], [])), y)
                else:
                    t[ctx] = e[0]
        tabs_p.append(shard_tabs)
        tp.append(t)
    # exchange + fold P, then phase 2: predictions final, pass C, the C transfer
    carries_p, tabs_c, tc = [], [], []
    for r in range(W):
        carry = {}
        for s in range(r):
            for ctx, y in tp[s].items():
                carry[ctx] = (lion_compose((carry.get(ctx, p_init(True)[0]), []), y)[0]) if lion else y
        carries_p.append(dict((k, list(v) if lion else v) for k, v in carry.items()))
        for tab in tabs_p[r]:
            fold_p_run(lion, qs, tab, carry, flags)
        predicted = {i for i, f in flags.items() if f[0] == "P"}
        shard_tabs, t = [], {}
        for lo, hi in runs[r]:
            tab, fl = run_pass_c(qs, lo, hi, predicted)
            flags.update(fl)
            shard_tabs.append(tab)
            for h, (T, a, b, _, _) in tab.items():
                t[h] = chunk_compose(t.get(h, (0, 0, 0)), (T, a, b))
        tabs_c.append(shard_tabs)
        tc.append(t)
    # exchange + fold C, phase 3: chunk-map flags final
    carries_c = []
    for r in range(W):
        carry = {}
        for s in range(r):
            for h, y in tc[s].items():
                carry[h] = chunk_compose((2,) + carry.get(h, c_init(h)[1:]), y)[1:]
        carries_c.append(dict(carry))
        for tab in tabs_c[r]:
            fold_c_run(qs, tab, carry, flags)
    out = [flags.get(i, "plain") for i in range(len(qs))]
    return out, carries_p, carries_c


def check(lion, data, cuts):
    qs = quads(data)
    qcuts = [c // 4 for c in cuts[:-1]] + [len(qs)]
    want_flags, snaps = inorder(lion, qs, qcuts)
    flags, carries_p, carries_c = sharded_model(lion, qs, qcuts)
    assert flags == want_flags
    for r in range(len(qcuts) - 1):
        P, C = snaps[qcuts[r]]
        for ctx in set(P) | set(carries_p[r]):
            start = [0] * 5 if lion else 0
            assert carries_p[r].get(ctx, start) == P.get(ctx, start), (r, ctx)
        for h in set(C) | set(carries_c[r]):
            assert carries_c[r].get(h, c_init(h)[1:]) == C.get(h, c_init(h)[1:]), (r, h)


def even(n, w):
    per = n // w // 256 * 256
    return [r * per for r in range(w)] + [n]


def dickens(n):
    return np.fromfile(f"{GOLDEN_DIR}/dickens_200k.bin", dtype=np.uint8)[:n]


@pytest.mark.parametrize("lion", [False, True], ids=["cheetah", "lion"])
@pytest.mark.parametrize("world", range(1, 10))
def test_fold_equals_inorder_dickens(lion, world):
    d = dickens(48 * 1024 + 3)
    check(lion, d, even(d.size, world))


@pytest.mark.parametrize("lion", [False, True], ids=["cheetah", "lion"])
def test_fold_equals_inorder_text_zeros_empty(lion):
    from density_b200 import synth
    t = synth.synth_text(40 * 1024 + 5).numpy()
    for w in (2, 4, 7):
        check(lion, t, even(t.size, w))
    z = np.zeros(8 * 1024, np.uint8)
    check(lion, z, [0, 256, 4096, z.size])
    check(lion, t, [0, 0, 4096, 4096, 4096, 30 * 1024, t.size])          # empty shards
    check(lion, t, [0, t.size - 5, t.size])                                 # a tiny last shard


@pytest.mark.parametrize("lion", [False, True], ids=["cheetah", "lion"])
def test_fold_equals_inorder_planted(lion):
    """cuts on the 16 KiB boundaries where cl_corpus plants its sentinels, and 256 bytes away from them"""
    data, _ = planted.cl_corpus(10 * planted.TILE_BYTES + 13, 5)
    T = planted.TILE_BYTES
    check(lion, data, [0] + [t * T for t in range(1, 10)] + [data.size])
    check(lion, data, [0, 3 * T - 256, 4 * T + 256, 6 * T, data.size])


def test_lion_undecided_accesses_hit_duplicate_zeros():
    """The stream-start list is five zeros: a shard whose context-0 accesses are 0 and small values, cut so that they are undecided in
    the shard's runs, must remove ONE zero per hit (dedupe-and-concatenate would be wrong)."""
    rng = np.random.default_rng(3)
    head = dickens(4096)
    tail = rng.choice(np.array([0, 0, 0, 7, 9, 11], np.uint32), 2048).astype(np.uint32).view(np.uint8)
    data = np.concatenate([head, tail, dickens(8192)[4096:]])
    qs = quads(data)
    n0 = sum(1 for i in range(1024, 1024 + 2048) if qs[i - 1] == 0 and qs[i] == 0)
    assert n0 > 100
    for cuts in ([0, 4096, data.size], [0, 4096, 4096 + 256, 4096 + 1024, data.size], [0, 4352, 8192, data.size]):
        check(True, data, cuts)
    # the composition itself: two zeros taken from the carried five zeros leave three
    assert lion_compose(([0] * 5, []), ([0, 7], [7, 0])) == ([0, 7, 0, 0, 0], [])
    assert lion_compose(([], []), ([0, 7], [7, 0])) == ([0, 7], [7, 0])
    assert lion_compose(([0, 9], [9, 0]), ([0, 7], [7, 0]))[0] == [0, 7, 9]


def test_noise_shards_fold_too():
    d = np.concatenate([dickens(8192), splitmix_bytes(4096, 1), dickens(16384)[8192:]])
    for lion in (False, True):
        check(lion, d, [0, 8192, 12288, d.size])
