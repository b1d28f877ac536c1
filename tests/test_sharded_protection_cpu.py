"""The automaton state carried over the cuts of a sharded Chameleon encode with copy mode (CPU only).

Each shard exports its transfer: for every candidate state entering it (penalty 0..9, start 1..10, previous_incompressible), the
state at its end, or PROT_ESC. density_b200.sharded.compose_prot_transfers (the twin of cham_prot_enter_k) composes the transfers of
the shards before a rank from the stream start. Walking each shard from the composed state must give exactly the in-order automaton:
the same state at every cut and the same copy map, whatever the cuts (any block index, not only multiples of 16)."""
import numpy as np
import pytest

from density_b200 import sharded as S
from protection import Protection, reachable_states


def transfer(inc, first_block):
    """What cham_prot_seg_k / _groups_k / _transfer_k compute for one shard: entry c = the candidate at the shard end when entered in
    candidate c, the automaton counting blocks from the shard's first global block."""
    out = np.zeros(S.PROT_TRANSFER_WORDS, dtype=np.int64)
    for c in range(S.PROT_TRANSFER_WORDS):
        ps = Protection(*S.prot_state(c), counter=first_block)
        for bit in inc:
            ps.step(bool(bit))
        out[c] = S.prot_candidate(ps.key())
    return out


def in_order(inc):
    """The automaton over the whole stream: (copy map, state in front of every block and after the last)."""
    ps, cm, states = Protection(), [], []
    for bit in inc:
        states.append(ps.key())
        cm.append(ps.step(bool(bit)))
    states.append(ps.key())
    return np.array(cm, dtype=bool), states


def sharded(inc, cuts):
    """Transfers of every shard, the composed incoming states, and the copy map walked shard by shard from them."""
    T = np.stack([transfer(inc[a:b], a) for a, b in zip(cuts[:-1], cuts[1:])])
    cm, ins = [], []
    for r, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        x = S.compose_prot_transfers(T, r)
        ins.append(x)
        assert x != S.PROT_ESC
        ps = Protection(*S.prot_state(x), counter=a)
        cm.extend(ps.step(bool(bit)) for bit in inc[a:b])
    return np.array(cm, dtype=bool), ins, T


def check(inc, cuts):
    want_cm, want_states = in_order(inc)
    cm, ins, _ = sharded(inc, cuts)
    assert (cm == want_cm).all(), cuts
    for r, a in enumerate(cuts[:-1]):
        assert S.prot_state(ins[r]) == want_states[a], (r, a)


def _sequences():
    rng = np.random.default_rng(11)
    yield "random 0.5", (rng.random(3000) < 0.5).astype(np.uint8)
    yield "random 0.9", (rng.random(3000) < 0.9).astype(np.uint8)
    yield "long runs", np.concatenate([np.ones(700), np.zeros(300), np.ones(1000), np.zeros(5), np.ones(400)]).astype(np.uint8)
    yield "alternating pairs", np.tile([1, 1, 0, 0], 700).astype(np.uint8)
    yield "pairs and singles", np.tile([1, 1, 0, 1, 0, 0, 1], 400).astype(np.uint8)
    bursts = np.zeros(3000, np.uint8)
    for b in rng.integers(0, 2990, 60):
        bursts[b:b + rng.integers(2, 9)] = 1
    yield "bursts in quiet data", bursts


@pytest.mark.parametrize("name,inc", list(_sequences()), ids=[n for n, _ in _sequences()])
def test_composed_transfers_equal_the_in_order_automaton(name, inc):
    rng = np.random.default_rng(len(name))
    n = inc.size
    for world in (2, 3, 5, 9):
        for _ in range(4):
            cuts = [0] + sorted(rng.choice(np.arange(1, n), world - 1, replace=False).tolist()) + [n]
            check(inc, cuts)


def test_every_reachable_seam_state_with_a_penalty_pending_at_the_cut():
    """Cuts right after the first and the second block of a pair, inside a copy run and right after it, at every counter phase."""
    inc = np.tile(np.array([0] * 13 + [1, 1] + [0] * 6 + [1] * 9 + [0] * 3, np.uint8), 5)
    _, states = in_order(inc)
    seen = set()
    for a in range(1, inc.size):
        check(inc, [0, a, inc.size])
        seen.add(states[a] + (a % 16,))
    assert any(s[0] > 0 for s in seen) and any(s[2] == 1 for s in seen)
    assert seen <= reachable_states()


def test_empty_shards_are_the_identity():
    inc = (np.random.default_rng(3).random(900) < 0.6).astype(np.uint8)
    assert (transfer(inc[:0], 123) == np.arange(S.PROT_TRANSFER_WORDS)).all()
    check(inc, [0, 0, 300, 300, 300, 701, 900, 900])


def test_a_path_that_leaves_the_candidates_is_esc():
    """Entering a one-block shard in (0, 10, 1) at a counter that does not halve the start, an incompressible block sets penalty 10:
    outside the candidates. The transfer says PROT_ESC, and so does every composition through it."""
    t1 = transfer(np.array([1], np.uint8), 5)
    c = S.prot_candidate((0, 10, 1))
    assert t1[c] == S.PROT_ESC
    assert t1[S.prot_candidate((0, 3, 1))] == S.prot_candidate((3, 3, 1))
    t0 = np.arange(S.PROT_TRANSFER_WORDS)
    t0[0] = c
    T = np.stack([t0, t1, np.arange(S.PROT_TRANSFER_WORDS)])
    assert S.compose_prot_transfers(T, 1) == c
    assert S.compose_prot_transfers(T, 2) == S.PROT_ESC
    assert S.compose_prot_transfers(T, 3) == S.PROT_ESC
    assert S.prot_state(S.PROT_ESC) is None


def test_candidate_encoding_round_trips():
    for c in range(S.PROT_TRANSFER_WORDS):
        assert S.prot_candidate(S.prot_state(c)) == c
    assert S.prot_candidate((0, 1, 0)) == 0
    assert S.prot_candidate((10, 10, 0)) == S.PROT_ESC and S.prot_candidate((0, 11, 1)) == S.PROT_ESC
