"""The Chameleon range decode without a GPU: a Python model of its locate step and of the state it carries into the window, held to the
oracle. The witness of a window [first, first + len) is oracle.decode(...)[first:first + w], w = min(first + len, S) - first.

The model (`locate`) is what decode_range.cu computes: every block start and the automaton state in front of it (the main loop from
synth_streams.walk, the tail loop walked here), the decoded size S and the verdict (decoded_size_witness.model_size), the window's
blocks k0 = first / 256 and k1, the offsets of k0 and k1 + 1, the decode candidate in front of k0 and whether the window's piece runs to
the stream end. The state is checked against tests/protection.py's automaton; the prefix's last-writer dictionary (`prefix_table`, the
writer pass: the last PLAIN quad of each bucket in blocks [0, k0), copy-mode blocks skipped) and that state, carried into
synth_streams.decode_reference on the suffix stream[off(k0):], must reproduce the window at offset first - 256 k0 of its output. The
whole suffix is decoded, because the main loop's exit depends on the bytes left in the stream. tests/test_gpu_decode_range.py holds
the library to the oracle slice."""
import numpy as np
import pytest

import oracle
import protection as P
import synth_streams as ss
from conftest import payload
from decoded_size_witness import MALFORMED, model_size, oracle_cap, oracle_size

ALG = "chameleon"
BS = 256
KAT_INPUT = b"test" * 31 + b"t"   # lib.rs:19


def blocks(stream):
    """every block the decoder enters, main loop and tail loop: (starts, copy bits, state in front (penalty, start, prev, counter % 16))"""
    s = np.asarray(stream, np.uint8)
    n = s.size
    w = ss.walk(ALG, s)
    starts, copy, before = list(w["starts"]), list(w["copy"]), list(w["before"])
    ps = ss._Prot(*w["state"])
    idx = w["tail_off"]
    while n - idx > 0:                                         # codec.rs:102-123: the last block may be cut short
        before.append((ps.penalty, ps.start, ps.prev, ps.counter & 15))
        starts.append(idx)
        if ps.step_copy():
            copy.append(True)
            if n - idx <= BS:
                break
            idx += BS
            continue
        copy.append(False)
        if n - idx < 8:
            break
        consumed = 8 + 256 - 2 * bin(int.from_bytes(s[idx:idx + 8].tobytes(), "little")).count("1")
        if idx + consumed >= n:
            break
        idx += consumed
        ps.step_update(consumed >= BS)
    return starts, copy, before


def candidate(state):
    pen, start, prev, phase = state
    return phase * 200 + (prev * 10 + start - 1) * 10 + pen


def walk_all(stream):
    """what the locate step walks once per stream: S, the verdict, every block and the main loop's block count"""
    s = np.asarray(stream, np.uint8)
    S, verdict = model_size(ALG, s)
    starts, copy, before = blocks(s)
    return {"n": s.size, "S": S, "verdict": verdict, "starts": starts, "copy": copy, "before": before,
            "main_blocks": ss.walk(ALG, s)["main_blocks"]}


def locate(m, first, length):
    """the locate step on walk_all's result m for the window [first, first + length)"""
    S, starts, before = m["S"], m["starts"], m["before"]
    r = {"S": S, "verdict": m["verdict"], "w": 0}
    if m["verdict"] or first >= S or length == 0:
        return r
    w = min(length, S - first)
    k0, k1 = first // BS, (first + w - 1) // BS
    final = first + w == S or k1 >= m["main_blocks"]
    r.update(w=w, k0=k0, k1=k1, final=final, off0=starts[k0], off1=m["n"] if final or k1 + 1 == len(starts) else starts[k1 + 1],
             state=before[k0], cand=candidate(before[k0]))
    return r


def prefix_table(stream, starts, copy, k0):
    """the writer pass of the piece [0, off(k0)): the last PLAIN quad of every bucket (chameleon.rs:55-60); MAP quads and copy-mode
    blocks write nothing"""
    s = np.asarray(stream, np.uint8).tobytes()
    tab = [0] * 65536
    for b in range(k0):
        if copy[b]:
            continue
        pos = starts[b]
        sig = int.from_bytes(s[pos:pos + 8], "little")
        pos += 8
        for k in range(64):
            if (sig >> k) & 1:
                pos += 2
            else:
                q = int.from_bytes(s[pos:pos + 4], "little")
                tab[ss.hash16(q)] = q
                pos += 4
    return tab


def automaton_state(starts, copy, k0):
    """protection.py's automaton over the blocks in front of k0, from their encoded sizes; checks the copy bits on the way"""
    ps = P.Protection()
    for b in range(k0):
        inc = not copy[b] and starts[b + 1] - starts[b] >= BS
        assert ps.step(inc) == copy[b], f"block {b}: the copy bit differs from the automaton's"
    return ps.penalty, ps.start, ps.prev, ps.counter & 15


class Stream:
    """a stream, its oracle decode, and the model's suffix decodes by k0 (computed once per k0)"""

    def __init__(self, stream):
        self.s = np.asarray(stream, np.uint8)
        self.size, self.verdict = oracle_size(ALG, self.s)
        self.D = oracle.decode(ALG, self.s, oracle_cap(self.s.size)).tobytes() if self.s.size else b""
        self.m = walk_all(self.s)
        self.suffix = {}

    def check(self, first, length, what=""):
        r = locate(self.m, first, length)
        assert (r["S"], r["verdict"]) == (self.size, self.verdict), f"{what}: S / verdict"
        want = self.D[first:first + length] if not self.verdict else b""
        assert r["w"] == len(want), f"{what} [{first}, +{length}): w {r['w']}, oracle slice {len(want)}"
        if not r["w"]:
            return r
        k0 = r["k0"]
        starts, copy = self.m["starts"], self.m["copy"]
        assert r["off0"] == starts[k0] and (r["final"] or r["off1"] in starts + [self.s.size])
        if k0 not in self.suffix:
            st = automaton_state(starts, copy, k0)
            assert st == r["state"], f"{what}: block {k0}: walk state {r['state']}, automaton {st}"
            assert st in P.reachable_states() and r["cand"] < 3200
            tab = prefix_table(self.s, starts, copy, k0)
            self.suffix[k0] = ss.decode_reference(ALG, self.s[r["off0"]:], 1 << 40, state={"a": tab}, prot=st)
        got = self.suffix[k0][first - k0 * BS:first - k0 * BS + r["w"]]
        assert got == want, f"{what} [{first}, +{length}): the suffix decode differs from the oracle slice"
        return r


def windows_around(S, points, lens=(1, 2, 255, 256, 257, 600)):
    for p in points:
        for f in (p - 1, p, p + 1):
            if 0 <= f <= S + 1:
                for L in lens:
                    yield f, L


def test_known_answer_and_golden_fixtures(golden_inputs):
    kat = Stream(oracle.encode(ALG, KAT_INPUT, cap=len(KAT_INPUT)))
    for first in range(len(KAT_INPUT) + 2):
        for length in range(1, len(KAT_INPUT) + 3):
            kat.check(first, length, "kat")
    for name, data in golden_inputs.items():
        if data.size > 2 << 20:
            continue
        g = Stream(oracle.encode(ALG, data))
        S = g.size
        for first, length in windows_around(S, (0, 256, 4096 * 7, S // 2, S - 256, S - 3, S)):
            g.check(first, length, name)


def test_every_window_of_a_short_stream():
    """every first in [0, S + 1] and every len in [1, S + 1 - first] of a stream with a tail of raw bytes"""
    data = payload("mixed", 1100 + 3, seed=4)
    st = Stream(oracle.encode(ALG, data))
    assert st.size == data.size
    finals = set()
    for first in range(st.size + 2):
        for length in range(1, st.size + 2 - first + 1):
            finals.add(st.check(first, length, "short").get("final"))
    assert finals == {None, True, False}


def _copy_stream():
    """noise between text: copy-mode blocks, pending penalties and incompressible pairs in the main loop"""
    from density_b200 import synth
    data = np.concatenate([synth.synth_text(40000).numpy(), payload("random", 30000, seed=8), synth.synth_text(30000).numpy(),
                           payload("random", 9000, seed=9), synth.synth_text(7001).numpy()])
    enc, copied = oracle.encode(ALG, data, return_copied=True)
    assert copied
    return Stream(enc)


def test_windows_on_every_counter_phase():
    st = _copy_stream()
    starts, copy, before = blocks(st.s)
    phases = set()
    for k0 in range(100, 132):
        for k1 in (k0, k0 + 5, k0 + 16 + (k0 % 16)):
            first, end = k0 * BS + (k0 % 3), k1 * BS + 256 - (k1 % 5)
            r = st.check(first, end - first, "phases")
            phases.add((before[k0][3], before[k1][3]))
    assert {a for a, _ in phases} == set(range(16)) and {b for _, b in phases} == set(range(16))


def test_windows_in_and_across_copy_mode_blocks_and_pending_penalties():
    st = _copy_stream()
    starts, copy, before = blocks(st.s)
    copied = [b for b in range(len(copy)) if copy[b]]
    pending = [b for b in range(len(copy)) if before[b][0] > 0]
    incpair = [b for b in range(1, len(copy)) if before[b][2] and not copy[b]]
    assert copied and pending and incpair
    picks = sorted(set(copied[:6] + copied[-6:] + pending[:6] + pending[-6:] + incpair[:6] + incpair[-6:]))
    for b in picks:
        for first, length in ((b * BS, BS), (b * BS + 7, 3), (b * BS - 1, 2), (b * BS + 255, 2 * BS + 3), ((b - 2) * BS + 11, 5 * BS)):
            if first >= 0:
                st.check(first, length, f"block {b}")
    assert any(before[b][0] > 0 and copy[b] for b in picks)


@pytest.mark.parametrize("r", [1, 2, 3])
def test_windows_in_the_raw_tail(r):
    """an input of 8 m + r bytes ends in an r-byte raw tail (decode_partial_unit)"""
    data = payload("text", 256 * 9 + 40 + r, seed=r)
    st = Stream(oracle.encode(ALG, data))
    S = st.size
    assert S == data.size
    for first in range(S - r - 9, S + 2):
        for length in (1, 2, 3, 4, 9, 300):
            st.check(first, length, f"raw tail {r}")


def test_synthesized_and_truncated_streams():
    """streams no encoder writes (synth_streams.build) and their truncations: S and the verdict are decoded_size's, a window a slice"""
    s, m = ss.build(ALG, {"nbytes": 60000, "quiet": False, "copy_every": 23, "plant": False, "tail": (60, "raw2")}, 7)
    full = Stream(s)
    assert (full.size, full.verdict) == (m["decoded_size"], 0)
    for first, length in windows_around(full.size, (0, 256 * 23, 256 * 46 + 5, full.size - 300, full.size - 1)):
        full.check(first, length, "synth")
    verdicts = set()
    for k in range(s.size - 40, s.size + 1, 3):
        t = Stream(s[:k])
        verdicts.add(t.verdict)
        for first, length in ((0, 1 << 40), (t.size // 2, 700), (max(t.size - 5, 0), 9)):
            r = t.check(first, length, f"truncated at {k}")
            if t.verdict == MALFORMED:
                assert r["w"] == 0 and r["S"] == 0
    assert verdicts == {0, MALFORMED}
