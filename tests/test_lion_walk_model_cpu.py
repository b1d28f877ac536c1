"""CPU check of the parallel Lion decoder's prediction walk: tests/lion_walk_model.cpp runs the row algorithm of
density_b200/csrc/lion_walk.cuh (the one the walk kernel runs) on 32 emulated lanes over oracle-encoded streams and must reproduce the
input byte for byte; its counts must equal the ones tests/lion_streams.py computes from the stream's flags and the decoded quads.
The kernels themselves are checked on the GPU (tests/test_gpu_lion_decode.py)."""
import numpy as np
import pytest

import oracle
import lion_streams as ls
from conftest import payload
from lion_streams import TAIL_SWEEP


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return ls.build_model(tmp_path_factory.mktemp("lion_walk"))


def run(L, enc, cap):
    return ls.run_model(L, enc, cap)


def check(L, data, counts=True):
    enc = oracle.encode("lion", data)
    n, got, c = run(L, enc, data.size)
    assert n == data.size and (got == data).all()
    if counts:
        assert c == ls.walk_counts(enc, data), (c, ls.walk_counts(enc, data))
    return c


@pytest.mark.parametrize("kind,nbytes", [("text", 200000), ("mixed", 150001), ("random", 40003), ("zeros", 60000), ("low", 70002),
                                         ("text", 127), ("text", 129), ("zeros", 5), ("low", 1)])
def test_walk_reproduces_the_input(model, kind, nbytes):
    check(model, payload(kind, nbytes, seed=11))


@pytest.mark.parametrize("period", [2, 3, 5, 6, 7, 8, 11, 16, 24, 31, 32, 33, 40])
def test_records(model, period):
    """repeating records (24-byte records are period 6): contexts come back every `period` quads, inside one row and across rows"""
    check(model, ls.records(period, 30000 + period))


def test_walk_inputs(model):
    for name, data in ls.walk_inputs().items():
        c = check(model, data)
        assert c[1] > 0, name


def test_known_answer_and_dickens(model, golden_inputs, dickens200k):
    for name in ("kat", "dickens_65539", "zeros_1m", "splitmix_1m_seed1", "mixed_280004"):
        check(model, golden_inputs[name], counts=name != "zeros_1m" and name != "splitmix_1m_seed1")
    c = check(model, dickens200k)
    assert c[0] > 0 and 0 < c[1] < c[0]


@pytest.mark.parametrize("extra", TAIL_SWEEP)
def test_tail_lengths(model, dickens200k, extra):
    check(model, dickens200k[:64 * 200 + extra], counts=False)
    check(model, np.concatenate([np.zeros(64 * 33, np.uint8), dickens200k[:extra]]), counts=False)


def test_counts_on_large_inputs(model):
    """counts that do not come from the walk's own bookkeeping, on inputs where reads that wait on a predicted quad do happen"""
    from density_b200 import synth
    for data in (synth.synth_text(1 << 20).numpy(), synth.synth_mixed(1 << 20).numpy()):
        enc = oracle.encode("lion", data)
        n, got, c = run(model, enc, data.size)
        assert n == data.size and (got == data).all()
        assert c == ls.walk_counts(enc, data)
        assert c[2] > 0


@pytest.mark.parametrize("seed", range(6))
def test_random_flag_streams(model, seed):
    """well-formed streams that no encoder writes (random flags laid out with the protection automaton) against the oracle"""
    s = ls.synth_stream(seed, 300 + 37 * seed, tail_bytes=[0, 5, 40, 69, 70, 100][seed], p_pred=[0.5, 0.9, 0.2, 0.7, 0.99, 0.5][seed])
    cap = ls.decode_cap(s)
    want = oracle.decode("lion", s, cap)
    n, got, c = run(model, s, cap)
    assert n == want.size and (got == want).all()
    if n:
        assert c == ls.walk_counts(s, got)


def test_truncated_and_capacity(model, dickens200k):
    data = dickens200k[:50000]
    enc = oracle.encode("lion", data)
    for cut in (1, 5, 6, 7, 100, enc.size // 2, enc.size - 1):
        want = oracle.decode("lion", enc[:cut], data.size)
        n, got, _ = run(model, enc[:cut], data.size)
        assert n == want.size and (got == want).all(), cut
    for cap in (data.size - 1, data.size - 64, 100):
        assert run(model, enc, cap)[0] == oracle.decode("lion", enc, cap).size == 0
