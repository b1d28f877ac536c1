"""The protection-automaton corpora (tests/protection.py) mean what their manifests say (no GPU).

Every piece is encoded with the oracle and parsed block by block (protection.trace); the parse must agree with the oracle and with the
layout the corpus was built from, and every manifest class must be where it says: the seam states on PSEG, tile and run seams, the
decoder's chunk and group entries, the number of non-canonical seams prot_iterate meets after its round 0, threshold blocks of exactly
BS and BS - 2 bytes, D blocks that flip with their S, streams that end in copy mode. The breadth-first search facts the corpora rest on
are checked too."""
import numpy as np
import pytest

import oracle
import protection as P
from protection import BS, CH, GROUP, PSEG, SIG, TILE_BLOCKS

NAMES = ("seam_states", "chunk_entries", "seam_counts", "thresholds", "tails")
CASES = [(n, a) for n in NAMES for a in P.ALGS] + [("pipelined", "chameleon")]


def _traced(name, alg):
    out = []
    for piece in P.corpus(name, alg):
        enc, copied = oracle.encode(alg, piece.data, return_copied=True)
        out.append((piece, enc, copied, P.trace(alg, enc, piece.data.size)))
    return out


def test_bfs_facts():
    """306 states (penalty, start, prev, counter % 16) are reachable; start and penalty never exceed 6, so the candidate-state tables
    of prot_iterate (PC_NS = PC_NP = 10 in chameleon_encode.cu) hold every state of a real stream; 28 states can sit in front of a
    block whose index is a multiple of 16 (every PSEG, tile and run seam), and a segment of 256 incompressible blocks maps them to 3."""
    reach = P.reachable_states()
    assert len(reach) == 306
    assert max(s[1] for s in reach) == 6 and max(s[0] for s in reach) == 6
    assert all(s[0] < 10 and 1 <= s[1] <= 10 for s in reach)
    seams = P.seam_states()
    assert len(seams) == 28 and P.CANON in seams
    noise = np.ones(PSEG, bool)
    assert len({P._walk(noise, 0, PSEG, s) for s in seams}) == 3
    for s in seams:                                     # the words the corpora use reach their target
        for b in (PSEG, PSEG + 64):
            w = P.word_to(s, b)
            ps = P.Protection(counter=b - len(w))
            for L in w:
                ps.step(L == "R")
            assert ps.key() == s and ps.counter == b


@pytest.mark.parametrize("name,alg", CASES)
def test_trace_agrees_with_the_oracle_and_the_layout(name, alg):
    """Copied blocks as counted by the oracle, the last block ending at the stream's end, the oracle round trip, and the letters'
    layout (offsets, copy map, automaton states) equal to the parse."""
    for piece, enc, copied, tr in _traced(name, alg):
        what = (name, alg, piece.label)
        assert tr.copied.sum() == copied, what
        assert tr.n_stream == enc.size, what
        assert (oracle.decode(alg, enc, piece.data.size) == piece.data).all(), what
        bld = piece.builder
        assert (tr.off == np.array(bld.offs)).all(), (what, int(np.flatnonzero(tr.off != np.array(bld.offs))[0]))
        assert (tr.copied == np.array(bld.copied)).all(), what
        assert tr.state == [s for s, _ in bld.states], what


def _entry(tr, b, c, alg):
    """Block b is the first block starting in chunk c."""
    return tr.off[b] >= c * CH[alg] > tr.off[b - 1] and tr.off[b] - c * CH[alg] < P.maxblk(alg)


def _flags(alg, enc, tr, b):
    fb = P.FLAG_BITS[alg]
    sig = int.from_bytes(bytes(enc[tr.off[b]:tr.off[b] + SIG[alg]]), "little")
    return [(sig >> (fb * i)) & ((1 << fb) - 1) for i in range(BS[alg] // 4)]


@pytest.mark.parametrize("alg", P.ALGS)
def test_seam_states_manifest(alg):
    (piece, enc, _, tr), = _traced("seam_states", alg)
    got = {"pseg": set(), "tile": set(), "run": set()}
    runs = P.planted.cham_runs(piece.data.size) if alg == "chameleon" else P.planted.chee_runs(piece.data.size)
    run_seams = {a * (P.planted.TILE_BYTES // BS[alg]) for a, _ in runs[1:]}
    for b, cls, info in piece.manifest:
        assert tr.state[b] == info["state"], (b, info)
        for k in info["kinds"]:
            assert {"pseg": b % PSEG == 0, "tile": b % TILE_BLOCKS[alg] == 0, "run": b in run_seams}[k], (b, k)
            got[k].add(info["state"])
    for k, states in got.items():
        assert states == set(P.seam_states()), (k, len(states))


@pytest.mark.parametrize("alg", P.ALGS)
def test_chunk_entries_manifest(alg):
    (piece, enc, _, tr), = _traced("chunk_entries", alg)
    phases, groups, straddle, forced, short = {}, set(), set(), set(), set()
    for b, cls, info in piece.manifest:
        c = info["chunk"]
        assert tr.state[b] == info["state"], (b, cls, info)
        if cls in ("chunk_start", "group_start", "forced_walk"):
            assert _entry(tr, b, c, alg), (b, cls, info)
            assert tr.counter[b] % 16 == info["phase"]
        if cls == "chunk_start":
            phases.setdefault(info["start"], set()).add(info["phase"])
        elif cls == "group_start":
            assert c % GROUP == 0
            groups.add(info["start"])
        elif cls == "forced_walk":
            assert tr.state[b][2] == 1 and tr.inc[b] and tr.copied[b + 1]
            forced.add(info["group"])
        elif cls == "short_jump":
            nb = int(np.searchsorted(tr.off, (c + 1) * CH[alg])) - b
            assert nb == 31 and tr.counter[b] % 16 == 0 and not tr.copied[b:b + nb + 1].any()
            assert not (tr.inc[b + 1:b + nb] & tr.inc[b:b + nb - 1]).any()
            assert tr.state[b + nb][1] == 1 and tr.copied[b + nb + 1]          # two halvings; the R R behind copies one block
            short.add(info["start"])
        elif cls == "copy_straddle":
            assert tr.copied[b] and tr.off[b] < c * CH[alg] < tr.off[b] + BS[alg]
            straddle.add(tr.state[b][0])
    reach = P.reachable_states()
    for s in range(2, 7):
        assert phases[s] == {ph for ph in range(16) if (0, s, 0, ph) in reach}, (s, sorted(phases[s]))
    assert groups == set(range(2, 7)) and forced == {False, True} and straddle == set(range(1, 7))
    assert short == ({4, 5, 6} if alg == "cheetah" else set())


def _jump_model(shift=0, dk=0):
    """test_models_cpu._sw_jump with the window of counted multiples of 16 shifted by `shift` blocks and `dk` halvings more."""
    def jump(ps, nb, last_inc):
        c = ps.counter + shift
        k = max(0, (c + nb + 15) // 16 - (c + 15) // 16 + dk)
        if ps.start > 1:
            ps.start = max(1, ps.start >> min(k, 8))
        ps.counter += nb
        ps.prev = last_inc
    return jump


OFF_BY_ONE = {"window+1": (1, 0), "window-1": (-1, 0), "k+1": (0, 1), "k-1": (0, -1)}


def _start_after(jump, s, ph, nb):
    from test_models_cpu import _Protection
    ps = _Protection(0, s, False, ph)
    jump(ps, nb, False)
    return ps.start


@pytest.mark.parametrize("alg", P.ALGS)
def test_where_the_halving_count_shows(alg):
    """Every reachable state with penalty 0, entering a chunk of any block count a jumped chunk can have: where does an off-by-one in
    sw_jump's halving count change the start it leaves? Nowhere for Chameleon and Lion (at least 63 and 61 blocks per jumped chunk:
    start <= 6 ends at 1 either way). For Cheetah (at least 31 blocks) a window shifted back by one block or one halving more never
    shows; a window shifted forward shows only for start 4..6 entering a 31-block chunk at counter phase 0, and one halving fewer
    shows there too: the short_jump entries of the chunk-entry corpus."""
    from test_models_cpu import _sw_jump
    n0 = P.min_jump_blocks(alg)
    shows = {m: set() for m in OFF_BY_ONE}
    for p, s, prev, ph in P.reachable_states():
        if p:
            continue
        for nb in range(n0, n0 + 64):
            want = _start_after(_sw_jump, s, ph, nb)
            for m, (sh, dk) in OFF_BY_ONE.items():
                if _start_after(_jump_model(sh, dk), s, ph, nb) != want:
                    shows[m].add((s, ph, nb))
    if alg != "cheetah":
        assert not any(shows.values()), {m: sorted(v)[:3] for m, v in shows.items()}
        return
    assert n0 == 31
    corpus_entries = {(s, 0, 31) for s in (4, 5, 6)}
    assert shows["window-1"] == set() and shows["k+1"] == set()
    assert shows["window+1"] == corpus_entries and corpus_entries <= shows["k-1"]


@pytest.mark.parametrize("mutant", ["window+1", "k-1"])
def test_chunk_entries_catch_an_off_by_one_halving_count(mutant):
    """The Cheetah chunk-entry corpus replayed through a jump model whose halving count is off by one fails: the start it leaves is
    wrong at the next chunk entry, and the R R there copies the wrong number of blocks."""
    (piece, enc, _, tr), = _traced("chunk_entries", "cheetah")
    with pytest.raises(AssertionError):
        replay_seq_walk("cheetah", enc, tr, _jump_model(*OFF_BY_ONE[mutant]))


def _round0_bits(bld):
    """Incompressible bits with nothing copied (prot_iterate's round 0): a D block is T- then, its S being encoded."""
    return np.array([L in "RP" for L in bld.letters])


@pytest.mark.parametrize("alg", P.ALGS)
def test_seam_counts_manifest(alg):
    """Exactly 0, 1, 8 and 9 segments with a non-canonical outgoing state after round 0 (9 takes the candidate evaluation at once), and
    chains of 5 and 8 noise segments that the relaxation needs 5 and 8 rounds for: more than prot_iterate's PROT_FAST_ROUNDS = 4."""
    for piece, enc, _, tr in _traced("seam_counts", alg):
        bad, rounds = P.prot_rounds(_round0_bits(piece.builder))
        if piece.label.startswith("seams"):
            k = int(piece.label[5:])
            assert bad == k, (piece.label, bad)
            assert tr.copied.sum() > 0
            for b, cls, info in piece.manifest:
                assert tr.state[(info["segment"] + 1) * PSEG] != P.CANON
        else:
            L = int(piece.label[5:])
            assert (bad, rounds) == (L, L), (piece.label, bad, rounds)
            assert rounds + 1 > 4


@pytest.mark.parametrize("alg", P.ALGS)
def test_thresholds_manifest(alg):
    """T+ is exactly BS bytes (incompressible), T- exactly BS - 2; for Cheetah and Lion T+ is reached both with and without PREDICTED
    quads. A D block is T+ behind a copied S and T- in the control copy, where the S is encoded; only behind the copied S does it make
    the blocks after it copied (which the copy map's round 0, with S encoded, does not see)."""
    (piece, enc, _, tr), = _traced("thresholds", alg)
    B = BS[alg]
    want = {"P": B, "M": B - 2, "R": B + SIG[alg]}
    routes = set()
    seams = 0
    for b, cls, info in piece.manifest:
        if cls.startswith("pair_"):
            for k, L in enumerate(cls[5:]):
                assert not tr.copied[b + k] and tr.size[b + k] == want[L], (b, cls, k)
                assert tr.inc[b + k] == (L != "M")
                if L == "P" and alg != "chameleon":
                    f = _flags(alg, enc, tr, b + k)
                    pred = sum(1 for x in f if (x == 3 if alg == "cheetah" else 1 <= x <= 5))
                    routes.add(pred > 0)
            if info["seam"]:
                assert (b + 1) % min(TILE_BLOCKS[alg], PSEG // 2) == 0
                seams += 1
    assert seams == 5
    if alg != "chameleon":
        assert routes == {False, True}
    ctrl = P.thresholds_builder(alg, control=True)
    cdata, _ = ctrl.realize()
    cenc = oracle.encode(alg, cdata)
    ctr = P.trace(alg, cenc, cdata.size)
    ds = [b for b, cls, _ in piece.manifest if cls == "D"]
    assert len(ds) == 3
    for b in ds:
        assert tr.copied[b - 1] and not tr.copied[b] and tr.size[b] == B and tr.inc[b] and tr.copied[b + 1:b + 3].any(), b
        assert not ctr.copied[b - 1] and ctr.size[b] == B - 2 and not ctr.inc[b] and not ctr.copied[b + 1:b + 3].any(), b


@pytest.mark.parametrize("alg", P.ALGS)
def test_tails_manifest(alg):
    """Every last-block length, streams ending in copy mode and with a penalty pending, and the decoder's main / tail handover (first
    block with fewer than SIG + BS stream bytes left) one block before, on and one block after a copy-mode block."""
    B = BS[alg]
    rel, ends = set(), set()
    for piece, enc, _, tr in _traced("tails", alg):
        n = piece.data.size
        nb = len(tr.off)
        L = n - (nb - 1) * B
        (b, cls, info), = [m for m in piece.manifest if m[1].startswith("tail_")]
        kind = cls[5:]
        assert L == info["last_len"]
        h = next((k for k in range(nb) if enc.size - tr.off[k] < P.maxblk(alg)), nb)
        copies = np.flatnonzero(tr.copied)
        assert copies.size > 0 or kind == "pending"
        rel.update(int(c) - h for c in copies if abs(int(c) - h) <= 1)
        if kind in ("end_copy", "end_run"):
            assert tr.copied[-1]
            ends.add("copy")
        if kind == "end_run":
            assert tr.copied[-2] and tr.state[-2][1] >= 2
        if kind == "pending":
            assert tr.inc[-2] and not tr.copied[-1]
            if tr.inc[-1]:
                ends.add("pending")
        if kind == "after" and L < SIG[alg]:
            assert h == nb - 2 and tr.size[h] == B and tr.copied[-1]
    assert rel == {-1, 0, 1} and ends == {"copy", "pending"}


def test_pipelined_manifest():
    """The R blocks sit on either side of the host pipeline's 64 MiB cut and the pair across it copies the first block after it."""
    for piece, enc, _, tr in _traced("pipelined", "chameleon"):
        (b, cls, info), = piece.manifest
        cut = info["cut"]
        assert piece.data.size > 96 * P.MIB
        rs = np.flatnonzero(tr.inc)
        if cls.endswith("last_of_first"):
            assert list(rs) == [cut - 1] and tr.copied.sum() == 0
        elif cls.endswith("first_of_second"):
            assert list(rs) == [cut] and tr.copied.sum() == 0
        else:
            assert list(rs) == [cut - 1, cut] and list(np.flatnonzero(tr.copied)) == [cut + 1]


# ---- the decoder's boundary walk replayed through the models of test_models_cpu ---------------------------------------------------
def replay_seq_walk(alg, enc, tr, jump):
    """dec_seq_walk (decode_bounds.cuh) on the parsed stream: entering a group or a chunk with penalty 0 and no incompressible pair
    inside it (nor across the entry), the whole group / chunk is jumped with `jump` (the model of sw_jump); any other chunk is walked
    block by block. Returns the number of jumps; asserts that the replayed state equals the parse at every chunk entry and at the
    handover to the tail."""
    from test_models_cpu import _Protection
    C, MB = CH[alg], P.maxblk(alg)
    n = enc.size
    nb_main = next((k for k in range(len(tr.off)) if n - tr.off[k] < MB), len(tr.off))
    nchunks = (n + C - 1) // C
    first = np.searchsorted(tr.off[:nb_main], np.arange(nchunks + 1) * C)   # first main block starting in each chunk

    def span(c0, c1):
        """(blocks, jumpable, last bit) of the blocks starting in chunks [c0, c1), as dec_chunk_walk / dec_group_compose see them."""
        b0, b1 = first[c0], first[min(c1, nchunks)]
        if b1 >= nb_main:                     # the chunk reaches the tail region: its row ends in TERM, never jumped
            return b1 - b0, False, False
        if b1 == b0 or tr.copied[b0:b1].any():
            return b1 - b0, False, False
        inc = tr.inc[b0:b1]
        return b1 - b0, not (inc[1:] & inc[:-1]).any(), bool(inc[-1])

    ps = _Protection()
    b, c, jumps = 0, 0, 0
    while b < nb_main:
        c = int(tr.off[b] // C)
        assert (ps.penalty, ps.start, int(ps.prev)) == tr.state[b] and ps.counter == tr.counter[b], (b, c)
        done = False
        for c1 in ((c // GROUP + 1) * GROUP, c + 1) if c % GROUP == 0 else (c + 1,):
            if c1 > nchunks:
                continue
            nb, ok, last = span(c, c1)
            if ok and ps.penalty == 0 and not (ps.prev and tr.inc[b]) and first[min(c1, nchunks)] < nb_main:
                jump(ps, nb, last)
                b += nb
                jumps += 1
                done = True
                break
        if done:
            continue
        while b < nb_main and tr.off[b] < (c + 1) * C:
            copied = ps.revert_to_copy()
            assert copied == tr.copied[b], b
            if copied:
                ps.penalty -= 1
                if ps.penalty == 0:
                    ps.start += 1
            else:
                ps.update(bool(tr.inc[b]))
            b += 1
    if nb_main < len(tr.off):
        assert (ps.penalty, ps.start, int(ps.prev)) == tr.state[nb_main] and ps.counter == tr.counter[nb_main]
    return jumps


@pytest.mark.parametrize("alg", P.ALGS)
def test_chunk_entries_replayed_through_the_jump_model(alg):
    """The chunk-entry corpus through the jump model of sw_jump (test_models_cpu._sw_jump): every chunk and group entry state and the
    state handed to the tail equal the parse."""
    from test_models_cpu import _sw_jump
    for name in ("chunk_entries", "tails", "thresholds"):
        for piece, enc, _, tr in _traced(name, alg):
            jumps = replay_seq_walk(alg, enc, tr, _sw_jump)
            if name == "chunk_entries":
                assert jumps > 50
