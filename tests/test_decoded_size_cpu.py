"""The witness of the decoded-size query, without a GPU: the oracle's decode (with the one rule that tells a malformed stream from one
that decodes to nothing) and a Python walk of the tail loop's control flow must agree on size and verdict, and the size must be what the
in-order Python decoder (synth_streams.decode_reference) writes. Streams: the reference's known-answer vectors and the golden fixtures,
every truncation of short streams, every tail length the main loop's exit rule leaves, the synthesized plans that no encoder writes
(the malformed ones included) and copy-mode streams. tests/test_gpu_decoded_size.py holds the library to this witness."""
import numpy as np
import pytest

import oracle
import synth_streams as ss
from conftest import ALGS, payload, splitmix_bytes
from decoded_size_witness import MALFORMED, model_size, oracle_size

MIB = 1 << 20
KAT_INPUT = b"test" * 31 + b"t"   # lib.rs:19


def agree(alg, stream, what, reference=True):
    """reference: also run the (slow) in-order Python decoder"""
    s = np.asarray(stream, np.uint8)
    want = oracle_size(alg, s)
    assert model_size(alg, s) == want, f"{alg} {what}: model {model_size(alg, s)} oracle {want}"
    if reference:
        ref = ss.decode_reference(alg, s, 1 << 40)
        assert len(ref) == want[0], f"{alg} {what}: decode_reference wrote {len(ref)} bytes, witness {want}"
    return want


@pytest.mark.parametrize("alg", ALGS)
def test_known_answers_and_golden_fixtures(alg, golden_inputs):
    enc = oracle.encode(alg, KAT_INPUT, cap=len(KAT_INPUT))     # the reference's own buffer size (lib.rs:24,46,68)
    assert agree(alg, enc, "kat") == (len(KAT_INPUT), 0)
    for name, data in golden_inputs.items():
        if data.size > 2 * MIB:
            continue
        enc = oracle.encode(alg, data)
        assert agree(alg, enc, name) == (data.size, 0), name


@pytest.mark.parametrize("alg", ALGS)
def test_empty_and_one_signature(alg):
    assert agree(alg, np.zeros(0, np.uint8), "empty") == (0, 0)
    sb = ss.SIG[alg]
    for first in range(1 << ss.FB[alg]):                       # one signature: PLAIN first decodes to nothing, the others do not
        s = np.zeros(sb, np.uint8)
        s[0] = first
        got = agree(alg, s, f"signature {first}")
        if first == 0:
            assert got == (0, 0)
        else:
            assert got != (0, 0)


@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("kind", ["text", "random", "mixed", "zeros"])
def test_every_truncation_of_short_streams(alg, kind):
    data = payload(kind, 1500 + 37 * ALGS.index(alg), seed=5)
    enc = oracle.encode(alg, data)
    verdicts = set()
    for k in range(enc.size + 1):
        verdicts.add(agree(alg, enc[:k], f"{kind} truncated at {k}")[1])
    assert agree(alg, enc, kind) == (data.size, 0)
    if kind != "zeros":
        assert verdicts == {0, MALFORMED}


@pytest.mark.parametrize("alg", ALGS)
def test_every_tail_length(alg):
    for L, end in ss.tail_lengths(alg):
        s, m = ss.build(alg, {"nbytes": 12000, "plant": False, "tail": (L, end)}, 100 + L)
        got = agree(alg, s, f"tail {L} {end}")
        if got[1] == 0:
            assert got[0] == m["decoded_size"], (L, end)


# the malformed plans of tests/test_gpu_synth_streams.py and tests/test_gpu_lion_synth_streams.py, and the shapes of their copy-mode and
# Lion plans at a size the Python walks take in seconds
PLANS = {
    "cham_bad": ("chameleon", {"nbytes": 300000, "tail": (100, "map0")}, 26),
    "cham_copy": ("chameleon", {"nbytes": 300000, "quiet": False, "copy_every": 31, "cuts": (0.33, 0.66), "tail": (60, "raw2")}, 23),
    "chee_bad": ("cheetah", {"nbytes": 300000, "p_pred": 0.5, "tail": (9, "map1")}, 38),
    "chee_prot": ("cheetah", {"nbytes": 300000, "p_pred": 0.3, "quiet": False, "prot_states": True, "tail": (20, "clean")}, 37),
    "lion_p5": ("lion", {"nbytes": 200000, "p_pred": 0.5, "cuts": tuple(k / 10 for k in range(1, 10)), "odd": True, "tail": (20, "raw2")}, 63),
    "lion_p99": ("lion", {"nbytes": 200000, "p_pred": 0.99, "cuts": (0.5,), "odd": True, "tail": (13, "raw1")}, 65),
    "lion_copy": ("lion", {"nbytes": 200000, "p_pred": 0.3, "quiet": False, "copy_every": 97, "cuts": (0.33, 0.66), "tail": (31, "raw3")}, 66),
    "lion_prot": ("lion", {"nbytes": 200000, "p_pred": 0.3, "quiet": False, "prot_states": True, "cuts": (0.2, 0.4, 0.6, 0.8),
                           "tail": (22, "clean")}, 67),
    "lion_bad": ("lion", {"nbytes": 200000, "p_pred": 0.5, "tail": (9, "map1")}, 68),
}


@pytest.mark.parametrize("name", list(PLANS))
def test_synthesized_plans(name):
    alg, plan, seed = PLANS[name]
    s, m = ss.build(alg, plan, seed)
    got = agree(alg, s, name)
    if name.endswith("_bad"):
        assert got == (0, MALFORMED)
    else:
        assert got == (m["decoded_size"], 0) and got[0] > m["main_blocks"] * ss.BS[alg]
    if "copy" in name or "prot" in name:
        assert m["copy_blocks"]
    for k in range(max(0, s.size - 300), s.size):                 # the last 300 byte offsets
        agree(alg, s[:k], f"{name} truncated at {k}", reference=False)


@pytest.mark.parametrize("alg", ALGS)
def test_copy_mode_tail(alg):
    """noise: the stream ends in copy mode, the last copy-mode block shorter than a block"""
    for n in (5 * ss.BS[alg] + 3, 40 * ss.BS[alg] + 1, 40 * ss.BS[alg]):
        data = splitmix_bytes(n, n)
        enc, copied = oracle.encode(alg, data, return_copied=True)
        assert copied
        assert agree(alg, enc, f"noise {n}") == (n, 0)
