"""The protection state carried across the pieces of a sharded Cheetah decode with copy-mode blocks (CPU only).

tests/prot_decode_model_cheetah.py models dec_prot_transfer<CheeT>: 4 KiB chunks, 68 entry offsets per chunk row, 128-byte
blocks of at most 136 bytes. Composed from the stream start, the transfers must give exactly the in-order automaton of the oracle's
Cheetah stream (protection.trace) at every cut: the state and the block count mod 16. The corpora are those of the sharded protected
Cheetah encode: noise, synth_mixed, text with noise bursts at the cuts, the seam cases of every automaton state, and copy decisions
that feed each other across shards. The head walk keeps at most PT_CAP = 256 heads; the test records how many stay live."""
import functools

import numpy as np
import pytest

import oracle
import prot_decode_model_cheetah as M
import protection as P
from conftest import payload

ALG = "cheetah"
BS = P.BS[ALG]
MIB = 1 << 20


def _text(n, first_page=0):
    from density_b200 import synth
    return synth.synth_text(n, first_page=first_page).numpy()


def _bursts():
    data = _text(MIB, first_page=5)
    rnd = payload("random", 64 * 1024, 7)
    cuts = [1000 * 256, 2001 * 256, 3001 * 256]
    for i, c in enumerate(cuts):                    # a burst ending at the cut, one straddling it, one starting at it
        lo = [c - 2048, c - 1024, c][i]
        data[lo:lo + 2048] = rnd[i * 8192:i * 8192 + 2048]
    return data, [0] + cuts + [data.size]


def _feedback():
    """the input of the protected CL encode tests whose copy decisions feed each other across shards"""
    t = _text(MIB, first_page=1)
    blob = payload("random", 40 * 256, 9)
    data = np.concatenate([t[:100 * 256], blob, t[100 * 256:600 * 256], blob, t[600 * 256:]])
    return data, [0] + [u * 256 for u in (137, 300, 620, 900)] + [data.size]


@functools.lru_cache(maxsize=None)
def corpora():
    from density_b200 import synth
    noise = payload("random", MIB // 2 + 77, 1)
    mixed = synth.synth_mixed(MIB).numpy()
    out = [(noise, [0, 300 * 256, 1111 * 256, noise.size]), (mixed, [0, 1111 * 256, 2003 * 256, 3001 * 256, mixed.size]), _bursts(),
           _feedback()]
    res = []
    for data, cuts in out:
        enc = oracle.encode(ALG, data)
        res.append((data, cuts, enc, P.trace(ALG, enc, data.size)))
    return res


NAMES = ["noise", "synth_mixed", "text_bursts", "feedback"]


def true_candidate(tr, b):
    """the decode candidate in front of block b of the traced stream"""
    return M.cand_index(*tr.state[b], tr.counter[b] % 16)


def _kind(tr, b):
    """"pending": the cut falls between an incompressible pair and the copy run it starts; "run": the cut falls inside a copy run"""
    if tr.state[b][0] > 0 and not tr.copied[b - 1]:
        return "pending"
    return "run" if tr.copied[b] and tr.copied[b - 1] else None


def cut_blocks(tr, cuts):
    """the corpus' cuts plus, for every counter phase, a block with a penalty pending in front of it and one inside a copy run (the
    first and a middle one of each kind that exist), all as block indices in the stream"""
    nb = len(tr.off)
    want = {c // BS for c in cuts[1:-1]}
    for ph in range(16):
        pend = [b for b in range(ph or 16, nb, 16) if _kind(tr, b) == "pending"]
        run = [b for b in range(ph or 16, nb, 16) if _kind(tr, b) == "run"]
        for kind in (pend, run):
            if kind:
                want.update({kind[0], kind[len(kind) // 2]})
    return [0] + sorted(b for b in want if 0 < b < nb) + [nb]


def offset(tr, b):
    return int(tr.off[b]) if b < len(tr.off) else tr.n_stream


def check_cuts(enc, tr, blocks):
    """the composed transfers at every cut of `blocks` are the traced automaton; returns the most live heads of any piece"""
    transfers, max_live = [], 0
    for r, (a, b) in enumerate(zip(blocks[:-2], blocks[1:-1])):
        piece = enc[offset(tr, a):offset(tr, b)]
        T, stats = M.transfer(piece)
        transfers.append(T)
        max_live = max(max_live, stats["max_live"])
        x = M.compose(transfers, r + 1)
        assert x == true_candidate(tr, b), (r, b, x, tr.state[b], tr.counter[b])
        # the piece walked in order from the composed state ends on the cut after exactly its blocks, in the same state
        st = M.cand_state(M.compose(transfers, r))
        end = M.exact_walk(M.consumed_table(piece), piece.size, st)
        assert end is not None and end[1] == b - a and M.cand_index(*end[0]) == x
    return max_live


def test_the_cheetah_geometry():
    assert (M.CH, M.BS, M.MAXBLK, M.NC) == (4096, 128, 136, 68) and P.CH[ALG] == 4096 and P.BS[ALG] == M.BS
    sig = np.array([0b11100100] * 8, np.uint8)           # flags 0, 1, 2, 3 in every byte: 4 + 2 + 2 + 0 per byte
    assert M.consumed_table(sig)[0] == 8 + 8 * 8
    assert M.consumed_table(np.zeros(8, np.uint8))[0] == 8 + 32 * 4 and M.consumed_table(np.full(8, 255, np.uint8))[0] == 8
    # the size of every block of an oracle stream, copy-mode blocks aside
    data = _text(64 * 1024, first_page=2)
    enc = oracle.encode(ALG, data)
    tr = P.trace(ALG, enc, data.size)
    cons = M.consumed_table(enc)
    full = [b for b in range(len(tr.off)) if not tr.copied[b] and (b + 1) * BS <= data.size]
    assert full and all(cons[tr.off[b]] == tr.size[b] for b in full)


@pytest.mark.parametrize("k", range(len(NAMES)), ids=NAMES)
def test_composed_transfers_are_the_in_order_automaton_at_every_cut(k):
    data, cuts, enc, tr = corpora()[k]
    assert tr.copied.any()
    blocks = cut_blocks(tr, cuts)
    assert len(blocks) > 3
    kinds = {(tr.counter[b] % 16, _kind(tr, b)) for b in blocks[1:-1]}
    if k < 2:          # noise and mixed data have cuts with a penalty pending and cuts inside a copy run at every counter phase
        assert all((ph, kind) in kinds for ph in range(16) for kind in ("pending", "run")), sorted(kinds, key=str)
    max_live = check_cuts(enc, tr, blocks)
    print(f"{NAMES[k]}: {len(blocks) - 1} pieces, at most {max_live} live heads after a piece's first chunk")
    assert max_live <= M.HEAD_CAP


def test_every_seam_case():
    """the seam cases of every automaton state a shard may end in, with the next shard starting incompressible or not"""
    from test_gpu_protection import _shard_cases
    n, max_live = 0, 0
    for end, nxt, cut, bld in _shard_cases(ALG):
        data, _ = bld.realize()
        enc = oracle.encode(ALG, data)
        tr = P.trace(ALG, enc, data.size)
        max_live = max(max_live, check_cuts(enc, tr, [0, cut // BS, len(tr.off)]))
        n += 1
    assert n >= 20 and max_live <= M.HEAD_CAP


@pytest.mark.parametrize("k", [0, 1, 3], ids=[NAMES[i] for i in (0, 1, 3)])
def test_every_candidate_equals_its_own_in_order_walk(k):
    """merging heads and jumping chunks and groups changes no candidate's result: a sample of candidates, each walked alone"""
    data, cuts, enc, tr = corpora()[k]
    b0, b1 = cuts[1] // BS, cuts[2] // BS
    piece = enc[offset(tr, b0):offset(tr, b1)]
    T, _ = M.transfer(piece)
    cons = M.consumed_table(piece)
    rng = np.random.default_rng(k)
    for c in sorted({0, 1, 199, 200, 3199, true_candidate(tr, b0)} | set(rng.integers(0, M.NCAND, 120).tolist())):
        end = M.exact_walk(cons, piece.size, M.cand_state(c))
        want = M.NOEND if end is None else M.cand_index(*end[0])
        assert T[c] == want, (c, M.cand_state(c), T[c], want)


@pytest.mark.parametrize("k", [0, 2], ids=[NAMES[0], NAMES[2]])
def test_a_cut_that_is_not_a_block_boundary_does_not_end_on_the_cut(k):
    data, cuts, enc, tr = corpora()[k]
    b0, b1 = cuts[1] // BS, cuts[2] // BS
    x = true_candidate(tr, b0)
    for delta in (-2, -1, 1, 2, 100):
        T, _ = M.transfer(enc[offset(tr, b0):offset(tr, b1) + delta])
        assert T[x] == M.NOEND, delta


def test_head_cap_refuses_never_lies():
    data, cuts, enc, tr = corpora()[0]
    piece = enc[offset(tr, cuts[1] // BS):offset(tr, cuts[2] // BS)]
    full, _ = M.transfer(piece)
    capped, stats = M.transfer(piece, head_cap=8)
    assert stats["capped"] > 0
    assert ((capped == full) | (capped == M.NOEND)).all()
    assert (capped == M.NOEND).sum() > (full == M.NOEND).sum()
