"""The Chameleon seek index without a GPU: tests/chameleon_index_model.py's index held to the oracle. For every checkpoint pair
(c_a, c_b), synth_streams.decode_reference of the piece stream[off(c_a):off(c_b)], entered in c_a's candidate state with snapshot c_a's
dictionary, must give the oracle's D[256 c_a I : 256 c_b I], and the final piece stream[off(c_a):] gives D[256 c_a I:]. That is the
size the indexed range decode's checked copy-out requires of phase 2, so these tests pin that rule as well. Windows are planned as the
library plans them (chameleon_index_model.plan) and held to the oracle slice. tests/test_gpu_chameleon_index.py holds the library's
index to this model byte for byte."""
import numpy as np
import pytest

import chameleon_index_model as X
import oracle
import synth_streams as ss
from conftest import payload
from decoded_size_witness import MALFORMED, oracle_cap, oracle_size
from test_decode_range_cpu import ALG, BS, KAT_INPUT, _copy_stream, blocks


class Indexed:
    """a stream, its oracle decode, its model index at one interval, and the piece decodes by (a, b) (computed once each)"""

    def __init__(self, stream, interval, m=None):
        self.s = np.asarray(stream, np.uint8)
        self.interval = interval
        self.size, self.verdict = oracle_size(ALG, self.s)
        self.D = oracle.decode(ALG, self.s, oracle_cap(self.s.size)).tobytes() if self.s.size else b""
        self.index, self.m = X.build(self.s, interval, m)
        self.pieces = {}
        if self.index is not None:
            assert len(self.index) <= X.index_bytes(self.s.size, interval)
            x = X.parse(self.index)
            assert (x["S"], x["n"], x["bytes"]) == (self.size, self.s.size, len(self.index))
            every = interval // BS
            assert x["count"] * every < max(x["main_blocks"], 1) and x["off"] == sorted(set(x["off"]))
            assert all(c < 3200 for c in x["cand"])

    def piece(self, a, b):
        """decode_reference of the piece from checkpoint a to checkpoint b (None: the stream end)"""
        if (a, b) not in self.pieces:
            x = X.parse(self.index)
            off = x["off"][a - 1] if a else 0
            end = self.s.size if b is None else x["off"][b - 1]
            k = a * (self.interval // BS)
            state = {"a": X.dictionary(X.snapshot(self.index, a))} if a else None
            self.pieces[(a, b)] = ss.decode_reference(ALG, self.s[off:end], 1 << 40, state=state, prot=self.m["before"][k])
        return self.pieces[(a, b)]

    def check_pairs(self):
        """every checkpoint pair, and every checkpoint to the stream end"""
        c, every = X.parse(self.index)["count"], self.interval // BS
        for a in range(c + 1):
            for b in list(range(a + 1, c + 1)) + [None]:
                got = self.piece(a, b)
                lo, hi = a * every * BS, (self.size if b is None else b * every * BS)
                assert got == self.D[lo:hi], f"pieces ({a}, {b}) at interval {self.interval}: differs from the oracle"

    def check(self, first, length, what=""):
        want = self.D[first:first + length]
        p = X.plan(self.index, self.s.size, first, length)
        if p is None:
            assert not want or length == 0, what
            return p
        got = self.piece(p["a"], p["b"])
        assert len(got) == p["expect"], f"{what}: the piece decodes to {len(got)} bytes, the index promises {p['expect']}"
        assert got[p["skip"]:p["skip"] + p["w"]] == want, f"{what} [{first}, +{length}): differs from the oracle slice"
        return p


def test_known_answer_and_golden_fixtures(golden_inputs):
    kat = Indexed(oracle.encode(ALG, KAT_INPUT, cap=len(KAT_INPUT)), 256)
    kat.check_pairs()
    for first in range(len(KAT_INPUT) + 2):
        for length in range(0, len(KAT_INPUT) + 3):
            kat.check(first, length, "kat")
    for name, data in golden_inputs.items():
        if data.size > 1 << 20:
            continue
        enc = oracle.encode(ALG, data)
        for interval in (256 * 97, 64 << 10, 1 << 30):
            g = Indexed(enc, interval)
            g.check_pairs() if X.parse(g.index)["count"] < 12 else None
            S = g.size
            for first in (0, 255, 256, interval - 1, interval, interval + 1, S // 2, S - 257, S - 1, S):
                for length in (1, 300, interval + 1):
                    if first >= 0:
                        g.check(first, length, f"{name} / {interval}")


@pytest.mark.parametrize("interval", [256, 512])
def test_every_window_of_a_short_stream(interval):
    data = payload("mixed", 1100 + 3, seed=4)
    st = Indexed(oracle.encode(ALG, data), interval)
    assert X.parse(st.index)["count"] >= 1
    st.check_pairs()
    finals = set()
    for first in range(st.size + 2):
        for length in range(0, st.size + 2 - first + 1):
            p = st.check(first, length, "short")
            finals.add(None if p is None else p["b"] is None)
    assert finals == {None, True, False}


@pytest.mark.parametrize("interval", [256, 512, 256 * 3])
def test_checkpoints_in_and_beside_copy_mode_blocks_on_every_counter_phase(interval):
    st = _copy_stream()
    ix = Indexed(st.s, interval, st.m)
    starts, copy, before = blocks(ix.s)
    x = X.parse(ix.index)
    every = interval // BS
    ks = [j * every for j in range(1, x["count"] + 1)]
    assert {before[k][3] for k in ks} == set(range(16)) or every % 2 == 0
    assert any(copy[k] for k in ks) and any(before[k][0] > 0 for k in ks) and any(before[k][2] for k in ks)
    # windows across the checkpoints next to copy-mode blocks, pending penalties and incompressible pairs
    picks = [k for k in ks if copy[k] or copy[k - 1] or before[k][0] > 0 or before[k][2]]
    for k in picks[:12] + picks[-12:]:
        for first, length in ((k * BS - 1, 2), (k * BS, BS), (k * BS + 9, 3 * interval), ((k - 1) * BS + 5, 700)):
            ix.check(first, length, f"checkpoint block {k}")
    for a in range(0, x["count"] + 1, max(1, x["count"] // 9)):
        ix.piece(a, a + 1 if a + 1 <= x["count"] else None)


@pytest.mark.parametrize("r", [1, 2, 3])
def test_windows_in_the_raw_tail(r):
    data = payload("text", 256 * 9 + 40 + r, seed=r)
    st = Indexed(oracle.encode(ALG, data), 512)
    st.check_pairs()
    S = st.size
    for first in range(S - r - 9, S + 2):
        for length in (1, 2, 3, 4, 9, 300):
            st.check(first, length, f"raw tail {r}")


def test_synthesized_and_truncated_streams():
    s, m = ss.build(ALG, {"nbytes": 60000, "quiet": False, "copy_every": 23, "plant": False, "tail": (60, "raw2")}, 7)
    full = Indexed(s, 256 * 23)
    assert full.size == m["decoded_size"] and full.index is not None
    full.check_pairs()
    verdicts = set()
    for k in range(s.size - 40, s.size + 1, 3):
        t = Indexed(s[:k], 256 * 23)
        verdicts.add(t.verdict)
        assert (t.index is None) == (t.verdict == MALFORMED)
        if t.index is not None:
            for first, length in ((0, 1 << 40), (t.size // 2, 700), (max(t.size - 5, 0), 9)):
                t.check(first, length, f"truncated at {k}")
    assert verdicts == {0, MALFORMED}


def test_index_bytes_bound_and_refused_intervals():
    for n in (1, 135, 136, 137, 4096, 1 << 20):
        for interval in (256, 512, 1 << 24):
            c = X.max_count(n, interval)
            assert X.index_bytes(n, interval) == X.snapshots_at(c) + c * 262144
    for bad in (0, 1, 255, 257, 1000):
        assert X.index_bytes(1 << 20, bad) == 0
