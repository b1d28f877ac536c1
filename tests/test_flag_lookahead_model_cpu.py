"""The three-barrier variant of the flag-pass tile protocol (tools/proto_tile_protocol_v6.py, `overlap=True`; DESIGN.md section 9):
phase A of a tile reads the dictionary while the previous tile's phase D writes it, and takes the pre-tile value of the buckets D
writes from that tile's mailboxes. The flags and the dictionary must equal the in-order walk, with the same dirty members and the
same overflow tiles as the four-barrier tile. No GPU needed."""
import os

import numpy as np
import pytest

import planted
from planted import TILE_QUADS, corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cases():
    d = np.fromfile(os.path.join(ROOT, "tests", "golden", "dickens_200k.bin"), np.uint8)
    text = d[:160000].view(np.uint32).copy()
    rng = np.random.default_rng(5)
    hot = np.concatenate([text[:6000], np.tile(text[100:108], 1500), text[6000:20000]])      # one short phrase repeated across tiles
    low = rng.integers(0, 3, 30000, dtype=np.uint32) * 0x01010101                               # few buckets, fingerprint-0 members
    return {"dickens": text, "hot": hot, "low": low}


def _check(q, seed):
    from tools import proto_tile_protocol_v6 as m6
    want, want_tab = m6.reference_flags(q)
    four, three = {}, {}
    m6.flag_pass(q, seed=seed, stats=four, overlap=False)
    got, tab, touched = m6.flag_pass(q, seed=seed, stats=three, overlap=True)
    assert (got == want).all(), int((got != want).sum())
    assert {int(b): int(tab[b]) for b in np.flatnonzero(touched)} == want_tab
    assert three["dirty"] == four["dirty"] and three["tile_overflow"] == four["tile_overflow"]
    return three


@pytest.mark.parametrize("name", ["dickens", "hot", "low"])
@pytest.mark.parametrize("seed", [1, 2])
def test_lookahead_tile_protocol_equals_the_in_order_walk(name, seed):
    st = _check(_cases()[name], seed)
    assert st["early"] >= 1


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_lookahead_tile_protocol_on_a_planted_run(seed):
    data, _ = corpus("cham5")
    q = data[:data.size // 4 * 4].view(np.uint32)
    a, _b = planted.cham_runs(data.size)[2]
    st = _check(q[a * TILE_QUADS:(a + 14) * TILE_QUADS], seed)
    assert st["stale"] >= 1
