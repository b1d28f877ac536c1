"""The protection state carried across the pieces of a sharded Chameleon decode with copy-mode blocks (CPU only).

tests/prot_decode_model.py models the head walk of dec_prot_transfer: each non-final piece exports, for every decode candidate
(automaton state and counter phase), the candidate at its end or PROT_ESC / NOEND. Composed from the stream start, the transfers
must give exactly the in-order automaton of the oracle's stream (protection.trace) at every cut: the state and the block count mod
16. The corpora are those of the sharded protected encode: noise, synth_mixed, text with noise bursts at the cuts, automaton states
on the cuts, copy decisions that feed each other across shards."""
import functools

import numpy as np
import pytest

import oracle
import prot_decode_model as M
import protection as P


@functools.lru_cache(maxsize=None)
def corpora():
    from test_gpu_sharded_loopback import _protected_corpora
    out = []
    for data, cuts in _protected_corpora():
        enc = oracle.encode("chameleon", data)
        out.append((data, cuts, enc, P.trace("chameleon", enc, data.size)))
    return out


NAMES = ["noise", "synth_mixed", "text_bursts", "states_on_cuts", "feedback"]


def true_candidate(tr, b):
    """the decode candidate in front of block b of the traced stream"""
    return M.cand_index(*tr.state[b], tr.counter[b] % 16)


def cut_blocks(tr, cuts):
    """the corpus' cuts plus, for every counter phase, a block with a penalty pending in front of it and one inside a copy run (the
    first block that exists of each kind), all as block indices in the stream"""
    nb = len(tr.off)
    want = {c // 256 for c in cuts[1:-1]}
    for ph in range(16):
        pend = [b for b in range(ph, nb, 16) if tr.state[b][0] > 0]
        if pend:
            want.add(pend[0])
            if len(pend) > 1:
                want.add(pend[len(pend) // 2])
        quiet = [b for b in range(ph, nb, 16) if tr.state[b][0] == 0 and tr.state[b][1] > 1]
        if quiet:
            want.add(quiet[0])
    return [0] + sorted(b for b in want if 0 < b < nb) + [nb]


def offset(tr, b):
    return int(tr.off[b]) if b < len(tr.off) else tr.n_stream


@pytest.mark.parametrize("k", range(len(NAMES)), ids=NAMES)
def test_composed_transfers_are_the_in_order_automaton_at_every_cut(k):
    data, cuts, enc, tr = corpora()[k]
    blocks = cut_blocks(tr, cuts)
    assert len(blocks) > 3
    transfers, max_live = [], 0
    for r, (a, b) in enumerate(zip(blocks[:-2], blocks[1:-1])):
        T, stats = M.transfer(enc[offset(tr, a):offset(tr, b)])
        transfers.append(T)
        max_live = max(max_live, stats["max_live"])
        x = M.compose(transfers, r + 1)
        assert x == true_candidate(tr, b), (r, b, x, tr.state[b], tr.counter[b])
        # the piece walked in order from the composed state ends on the cut after exactly its blocks, in the same state
        st = M.cand_state(M.compose(transfers, r))
        end = M.exact_walk(M.consumed_table(enc[offset(tr, a):offset(tr, b)]), offset(tr, b) - offset(tr, a), st)
        assert end is not None and end[1] == b - a and M.cand_index(*end[0]) == x
    print(f"{NAMES[k]}: {len(blocks) - 1} pieces, at most {max_live} live heads after a piece's first chunk")
    assert max_live <= M.HEAD_CAP


@pytest.mark.parametrize("k", [0, 1, 4], ids=[NAMES[i] for i in (0, 1, 4)])
def test_every_candidate_equals_its_own_in_order_walk(k):
    """merging heads and jumping chunks and groups changes no candidate's result: a sample of candidates, each walked alone"""
    data, cuts, enc, tr = corpora()[k]
    b0, b1 = cuts[1] // 256, cuts[2] // 256
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
    b0, b1 = cuts[1] // 256, cuts[2] // 256
    x = true_candidate(tr, b0)
    for delta in (-2, -1, 1, 2, 100):
        T, _ = M.transfer(enc[offset(tr, b0):offset(tr, b1) + delta])
        assert T[x] == M.NOEND, delta


def test_head_cap_refuses_never_lies():
    data, cuts, enc, tr = corpora()[0]
    piece = enc[offset(tr, cuts[1] // 256):offset(tr, cuts[2] // 256)]
    full, _ = M.transfer(piece)
    capped, stats = M.transfer(piece, head_cap=8)
    assert stats["capped"] > 0
    assert ((capped == full) | (capped == M.NOEND)).all()
    assert (capped == M.NOEND).sum() > (full == M.NOEND).sum()


def test_empty_piece_is_the_identity_and_candidate_zero_is_the_stream_start():
    T, _ = M.transfer(np.zeros(0, np.uint8))
    assert (T == np.arange(M.NCAND)).all()
    assert M.cand_state(0) == (0, 1, 0, 0) and M.cand_index(0, 1, 0, 0) == 0
    for c in range(M.NCAND):
        assert M.cand_index(*M.cand_state(c)) == c
