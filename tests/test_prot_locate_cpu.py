"""The protected range maps of a stream without known cuts and their composition (CPU only).

tests/prot_locate_model.py models dec_prot_transfer's range map (every entry offset x every decode candidate, walked exactly with the
copy-mode blocks) and prot_locate_walk. Composed from (entry 0, candidate 0), the maps must give at every cut the oracle stream's true
block boundary and automaton state (protection.trace), also where a cut falls inside a copy run or with a penalty pending, at many
counter phases, and on Cheetah's cold start. density_b200_prot_locate_piece is checked against the model on the same maps."""
import ctypes
import functools

import numpy as np
import pytest

import oracle
import prot_locate_model as L
import protection as P
from conftest import payload

ALGS = ["chameleon", "cheetah"]
NAMES = ["noise", "synth_mixed", "text_bursts", "feedback"]
KIB = 1024


@functools.lru_cache(maxsize=None)
def corpus(name, alg):
    """(data, oracle stream, trace)"""
    from density_b200 import synth
    if name == "noise":
        data = payload("random", 600 * KIB + 77, 1)
    elif name == "synth_mixed":
        data = synth.synth_mixed(1 << 20).numpy()
    elif name == "text_bursts":
        data = synth.synth_text(1 << 20).numpy()
        rnd = payload("random", 64 * KIB, 7)
        for i, lo in enumerate((100_000, 300_001, 700_003)):
            data[lo:lo + 3000] = rnd[i * 8192:i * 8192 + 3000]
    else:
        from test_gpu_sharded_protected_encode import _feedback_input
        data = _feedback_input()
    enc = oracle.encode(alg, data)
    return data, enc, P.trace(alg, enc, data.size)


def true_candidate(tr, b):
    return L.cand_index(*tr.state[b], tr.counter[b] % 16)


def cut_kind(tr, b):
    """'run': the cut falls inside a copy run (blocks b - 1 and b copied); 'pending': a penalty is pending in front of block b (it is
    copied, the one before it encoded); 'plain' otherwise"""
    if tr.state[b][0] > 0:
        return "run" if b > 0 and tr.copied[b - 1] else "pending"
    return "plain"


def interesting_cuts(tr, total, alg, most=8):
    """range boundaries (multiples of 16 KiB) inside copy runs and with a penalty pending, at as many counter phases as there are,
    then plain ones"""
    maxblk = L.GEOM[alg][2]
    kinds = {"run": {}, "pending": {}, "plain": {}}
    for k in range(1, (total - 2 * maxblk) // L.RANGE_UNIT + 1):
        b = int(np.searchsorted(tr.off, k * L.RANGE_UNIT))
        if b >= len(tr.off):
            break
        kinds[cut_kind(tr, b)].setdefault(tr.counter[b] % 16, k)
    ks = list(kinds["run"].values())[:most // 2] + list(kinds["pending"].values())[:most // 2]
    return sorted(set(ks + list(kinds["plain"].values())[:max(0, most - len(ks))]))[:most]


def layout_at(total, ks):
    bounds = [0] + [k * L.RANGE_UNIT for k in ks]
    return L.layout(total, [b - a for a, b in zip(bounds, bounds[1:])] + [None])


def check_layout(enc, tr, lay, alg):
    """every rank's located piece starts on the trace's block boundary, in its state; the pieces tile the stream"""
    maps = L.stream_maps(enc, lay, alg)
    pos = 0
    final_seen = False
    for r, (o, n, h) in enumerate(lay):
        start, end, final, first, cand, refused = L.locate_piece(maps, r, alg)
        assert not refused
        if end == start:
            continue
        assert not final_seen
        assert o + start == pos, (r, o + start, pos)
        b = int(np.searchsorted(tr.off, pos))
        assert tr.off[b] == pos and cand == true_candidate(tr, b), (r, cand, tr.state[b], tr.counter[b])
        assert first == (pos == 0)
        pos = o + end
        final_seen = bool(final)
    assert final_seen and pos == tr.n_stream
    return maps


@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("name", NAMES)
def test_composed_maps_are_the_in_order_automaton_at_every_cut(name, alg):
    data, enc, tr = corpus(name, alg)
    ks = interesting_cuts(tr, enc.size, alg)
    assert len(ks) >= 3
    kinds = [(cut_kind(tr, b), tr.counter[b] % 16) for b in (int(np.searchsorted(tr.off, k * L.RANGE_UNIT)) for k in ks)]
    print(f"{name}/{alg}: cuts {kinds}")
    if name == "noise":
        assert len({ph for k, ph in kinds if k == "run"}) >= 3
    check_layout(enc, tr, layout_at(enc.size, ks), alg)


def scalar_row(cons, n_range, n, off, st, alg):
    """one (entry, candidate) walked alone, block by block: codec.rs:88-100 with protection_state.rs"""
    _, BS, MAXBLK, _ = L.GEOM[alg]
    pen, start, prev, ph = st
    while True:
        if off >= n_range:
            c = L.cand_index(pen, start, prev, ph)
            return L.PROT_ESC if c == L.PROT_ESC else ((off - n_range) >> 1) | (c << 8)
        if off + MAXBLK > n:
            return L.TERM
        if ph == 0 and start > 1:
            start >>= 1
        ph = (ph + 1) & 15
        if pen:
            pen -= 1
            if not pen:
                start += 1
            off += BS
        else:
            con = int(cons[off])
            if con >= BS:
                if prev:
                    pen = start
                prev = 1
            else:
                prev = 0
            off += con


@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("name,at,n_range,n_halo", [("noise", 5, 2, L.HALO), ("synth_mixed", 0, 2, L.HALO), ("text_bursts", 6, 1, 10),
                                                    ("noise", 0, 0, 0)])
def test_every_row_equals_its_own_in_order_walk(name, at, n_range, n_halo, alg):
    """merging lanes changes no row: a sample of (entry, candidate) rows, each walked alone; a short halo and a tail: TERM rows"""
    _, enc, _ = corpus(name, alg)
    o = at * L.RANGE_UNIT
    n_range = n_range * L.RANGE_UNIT if n_range else enc.size - o     # 0: the rest of the stream
    buf = enc[o:o + n_range + n_halo]
    m = L.range_map(buf, n_range, n_halo, alg)
    cons = L.GEOM[alg][0](buf)
    nc = L.GEOM[alg][3]
    rng = np.random.default_rng(at)
    lanes = {(0, 0), (nc - 1, L.NCAND - 1)} | {(int(e), int(c)) for e, c in zip(rng.integers(0, nc, 300), rng.integers(0, L.NCAND, 300))}
    for e, c in sorted(lanes):
        want = scalar_row(cons, n_range, n_range + n_halo, 2 * e, L.cand_state(c), alg)
        assert m[L.HDR + e * L.NCAND + c] == want, (e, c)
    if n_halo < L.HALO:
        assert (m[L.HDR:] == L.TERM).any()


@pytest.mark.parametrize("alg", ALGS)
def test_empty_ranges_short_stream_and_short_last_halo(alg):
    _, enc, tr = corpus("synth_mixed", alg)
    # empty ranges around and between the pieces
    check_layout(enc, tr, L.layout(enc.size, [0, 2 * L.RANGE_UNIT, 0, 0, 3 * L.RANGE_UNIT, 0, None]), alg)
    # a stream shorter than world x 16 KiB: every range but the last is empty
    from density_b200 import synth
    small = synth.synth_mixed(9000).numpy()
    s = oracle.encode(alg, small)
    from density_b200 import sharded
    check_layout(s, P.trace(alg, s, small.size), sharded.stream_ranges(s.size, 4), alg)
    # the stream ends inside the halo of the range before the last: its last range is shorter than a block
    k = enc.size // L.RANGE_UNIT
    cut = enc.size - L.RANGE_UNIT * k
    part = enc[:L.RANGE_UNIT * (k - 1) + 100] if cut >= L.HALO else enc
    n = part.size
    lay = L.layout(n, [L.RANGE_UNIT * (k - 1), None])
    assert lay[0][2] == 100 or part is enc
    maps = L.stream_maps(part, lay, alg)
    pieces = [L.locate_piece(maps, r, alg) for r in range(2)]
    assert not any(p[5] for p in pieces) and pieces[1][2] == 1
    if pieces[0][2]:                                   # the first piece takes the tail, the last range is behind the stream end
        assert pieces[0][1] == n and pieces[1][:2] == (0, 0)
    else:                                              # Cheetah: a block may still start in the 100 bytes
        assert pieces[0][1] == lay[1][0] + pieces[1][0] and lay[1][0] + pieces[1][1] == n


@pytest.mark.parametrize("alg", ALGS)
def test_a_refused_row_refuses_every_rank_never_a_wrong_seed(alg):
    _, enc, tr = corpus("noise", alg)
    lay = layout_at(enc.size, interesting_cuts(tr, enc.size, alg, most=3))
    maps = check_layout(enc, tr, lay, alg)
    path = [L.locate_piece(maps, r, alg) for r in range(len(lay))]
    for bad in (L.NOEND, L.PROT_ESC):           # a head dropped at the cap / a state outside the candidates, on the path at range 1
        m = maps.copy()
        m[1, L.HDR + path[1][0] // 2 * L.NCAND + path[1][4]] = bad
        for r in range(len(lay)):
            assert L.locate_piece(m, r, alg) == (0, 0, 0, 0, 0, 1)
    # a row off the path changes nothing
    m = maps.copy()
    m[1, L.HDR + ((path[1][0] // 2 + 1) % L.GEOM[alg][3]) * L.NCAND] = L.NOEND
    assert [L.locate_piece(m, r, alg) for r in range(len(lay))] == path


@pytest.mark.parametrize("alg", ALGS)
def test_a_flipped_signature_bit_locates_what_the_in_order_walk_reads(alg):
    """the maps are the exact walk of the bytes they are given: on a damaged stream they locate the cuts the in-order decoder would
    read, so the pieces decode exactly as the stream does on one device (which refuses it or not); no seed from another walk"""
    _, enc, tr = corpus("synth_mixed", alg)
    bad = enc.copy()
    b = int(np.searchsorted(tr.off, L.RANGE_UNIT + 5000))
    bad[int(tr.off[b]) + 1] ^= 0x10                        # a bit of a signature in range 1 (block b is encoded in synth_mixed or not)
    lay = L.layout(bad.size, [2 * L.RANGE_UNIT, 3 * L.RANGE_UNIT, None])
    maps = L.stream_maps(bad, lay, alg)
    cons = L.GEOM[alg][0](bad)
    _, BS, MAXBLK, _ = L.GEOM[alg]
    starts, states = {}, {}
    off, st = 0, (0, 1, 0, 0)
    while off + MAXBLK <= bad.size:                        # the in-order main loop over the damaged bytes
        starts[off] = L.cand_index(*st)
        pen, start, prev, ph = st
        if ph == 0 and start > 1:
            start >>= 1
        ph = (ph + 1) & 15
        if pen:
            pen -= 1
            start += pen == 0
            off += BS
        else:
            con = int(cons[off])
            pen = start if con >= BS and prev else pen
            prev = int(con >= BS)
            off += con
        st = (pen, start, prev, ph)
    for r, (o, n, h) in enumerate(lay):
        start, end, final, first, cand, refused = L.locate_piece(maps, r, alg)
        if refused:
            continue
        if end > start:
            assert starts.get(o + start) == cand, r


def _lib_piece(lib, maps, rank, alg):
    m = np.ascontiguousarray(maps, np.uint32)
    out = (ctypes.c_uint64 * 6)()
    rc = lib.density_b200_prot_locate_piece(0 if alg == "chameleon" else 1, m.ctypes.data, m.shape[0], rank, out)
    return rc, tuple(int(v) for v in out)


@pytest.mark.parametrize("alg", ALGS)
def test_library_composition_equals_the_model_and_checks_the_layout(alg):
    import density_b200
    lib = density_b200.load()
    _, enc, tr = corpus("text_bursts", alg)
    lay = L.layout(enc.size, [0, 3 * L.RANGE_UNIT, 0, 2 * L.RANGE_UNIT, 0, None])
    maps = check_layout(enc, tr, lay, alg)
    from density_b200 import sharded
    for r in range(len(lay)):
        rc, got = _lib_piece(lib, maps, r, alg)
        assert rc == 0 and got == L.locate_piece(maps, r, alg) == sharded.prot_locate_piece(maps, r, alg)
    m = maps.copy()
    m[1, L.HDR + 0] = L.NOEND                              # (entry 0, candidate 0) of the first non-empty range
    assert all(_lib_piece(lib, m, r, alg) == (0, (0, 0, 0, 0, 0, 1)) for r in range(len(lay)))
    bad_layouts = []
    m = maps.copy(); m[1, 0] += 2; bad_layouts.append(m)             # a non-last range that is not a multiple of 16 KiB
    m = maps.copy(); m[2, 2] = 7; bad_layouts.append(m)              # a halo that is not min(264, the later bytes)
    m = maps.copy(); m[1, L.HDR] = 200; bad_layouts.append(m)        # an exit index beyond the entry offsets, on the path
    m = maps.copy(); m[1, L.HDR] = 0xFF | (3 << 8); bad_layouts.append(m)   # a TERM row with a candidate
    for m in bad_layouts:
        for r in (0, len(lay) - 1):
            rc, _ = _lib_piece(lib, m, r, alg)
            assert rc == 4, lib.density_b200_last_error()   # DENSITY_B200_EARG
            with pytest.raises(ValueError):
                L.locate_piece(m, r, alg)
    assert _lib_piece(lib, maps, len(lay), alg)[0] == 4
    assert lib.density_b200_prot_locate_piece(2, maps.ctypes.data, 1, 0, (ctypes.c_uint64 * 6)()) == 4
