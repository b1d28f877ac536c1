"""CPU checks of the corpus planted at the run-parallel Cheetah decoder's own run seams (tests/cl_decode_seams.py) and of the decoder
scheme on it (tests/cl_model.cpp): every class is planted where the decoder cuts and confirmed in the oracle stream, the model decodes
every corpus exactly at the decoder's run count and at others, and a stretch of one repeated quad needs one round per run it covers, so
that past 40 runs the round budget runs out. The kernels are compared with these numbers on the GPU
(tests/test_gpu_cheetah_decode_rounds.py)."""
import numpy as np
import pytest

import oracle
import cl_decode_seams as cds
from conftest import payload

MIB = 1 << 20


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return cds.build_model(tmp_path_factory.mktemp("cl_model"))


_corpora = {}


@pytest.fixture(scope="module", params=[(132, 8), (114, 1)], ids=["132sms", "114sms_1per_sm"])
def corpus(request):
    """The 12 MiB corpus at an H100 SXM's default geometry (130 runs, one per 48 KiB of stream) and at an H100 PCIe's with one run per
    SM, where the SM cap binds (114 runs): different seams."""
    if request.param not in _corpora:
        sms, per_sm = request.param
        _corpora[request.param] = cds.cl_decode_corpus(12 * MIB + 77, 3, num_sms=sms, per_sm=per_sm)
    return request.param, _corpora[request.param]


def test_geometry_mirror():
    """cd_pick_runs: one run per 48 KiB of stream, at most SMs x runs per SM, at least one; run r starts at block r * blocks / nruns."""
    assert cds.pick_runs(0, 132) == 1 and cds.pick_runs(48 * 1024 - 1, 132) == 1 and cds.pick_runs(48 * 1024, 132) == 1
    assert cds.pick_runs(2 * 48 * 1024, 132) == 2
    assert cds.pick_runs(10 ** 9, 132) == 1056 and cds.pick_runs(10 ** 9, 114) == 912 and cds.pick_runs(10 ** 9, 114, 1) == 114
    assert cds.cd_runs(7 * 48 * 1024, 100, 132) == [0, 14, 28, 42, 57, 71, 85]
    assert [cds.pick_runs(oracle.encode("cheetah", cds.zeros(k)).size, 132) for k in (39, 40, 41)] == [39, 40, 41]


@pytest.mark.parametrize("kind,n", [("text", 200000), ("mixed", 300001), ("random", 50003), ("zeros", 70000), ("low", 90002)])
def test_walk_matches_the_model(model, kind, n):
    """The Python block walk and the model's boundary stage agree on where the main loop stops."""
    data = payload(kind, n, seed=5)
    enc = oracle.encode("cheetah", data)
    w = cds.Walk(enc)
    out, st = cds.model_decode(model, enc, data.size, 3)
    assert st["main_blocks"] == w.main_blocks and (out == data).all()
    assert enc.size - w.tail_off < 136 and (w.kind == cds.COPY).any() == w.copy.any()


def test_manifest(corpus):
    """Every class is planted at 8 or more seams and every planting has, in the oracle stream, the kinds its class needs (the quad in
    front of a seam predicted, copy blocks on both sides of it, ...), at the seams of the oracle stream itself. Every variant of every
    class is among them."""
    (sms, per_sm), (data, enc, manifest, starts) = corpus
    w, now = cds.seams(enc, sms, per_sm)
    assert now == starts
    if per_sm != 8:
        assert len(starts) == sms * per_sm < cds.pick_runs(enc.size, sms)       # the SM cap decides the seams
    by = {}
    for cls, t, var, chk in manifest:
        by.setdefault(cls, []).append((t, var, chk))
        assert 0 < t < len(starts)
        assert cds.confirmed(w, chk), (cls, t, var, [(q, e, w.kind_of(q)) for q, e in chk if not cds.KIND_OK[e](w.kind_of(q))])
    assert sorted(by) == sorted(cds.CLASSES)
    assert all(len(v) >= 8 for v in by.values()), {k: len(v) for k, v in by.items()}
    variants = {cls: {var for _, var, _ in v} for cls, v in by.items()}
    assert variants["self_stretch"] == set(cds.STRETCH)      # lengths 2, 31, 32, 33, 95 from seam - 1, - 16, - 31, - 32
    assert variants["pred_exit"] == {"lane0", "lane31"}
    assert variants["late_snapshot"] == {2, 3} and variants["cmap_carried"] == {1, 3}
    assert variants["in_step_writers"] == set(cds.IN_STEP) and variants["snap_passthrough"] == {0, 1}
    for _, D, chk in by["late_snapshot"]:                    # a predicted quad per link exit, per link start and the reader
        assert len([q for q, e in chk if e == "P"]) == 2 * D - 1


def test_model_decodes_the_corpus(model, corpus):
    """At the decoder's run count for this geometry, and at 1, 7 and 64 runs."""
    _, (data, enc, manifest, starts) = corpus
    for nruns in (len(starts), 1, 7, 64):
        out, st = cds.model_decode(model, enc, data.size, nruns)
        assert st["settled"] == 1 and st["nruns"] == nruns, (nruns, st)
        assert out.size == data.size and (out == data).all(), nruns
        assert st["queued"] == st["walks"] - nruns           # a settled stream: every queued walk ran
    assert st["rounds"] >= 3                                  # the late snapshots: round 2 or 3 rewalks


@pytest.mark.parametrize("nruns", [1, 2, 3, 5, 8, 13])
def test_rounds_grow_one_per_run_on_zeros(model, nruns):
    """Every quad of zeros is predicted at context 0: run r's entry context is unknown until run r - 1 has settled."""
    data = np.zeros(MIB + 5000, np.uint8)
    enc = oracle.encode("cheetah", data)
    out, st = cds.model_decode(model, enc, data.size, nruns)
    assert st["settled"] == 1 and st["rounds"] == nruns and (out == data).all(), st


@pytest.mark.parametrize("k,rounds,settled", [(39, 39, 1), (40, 40, 1), (41, 40, 0)])
def test_round_budget_edge_on_zeros(model, k, rounds, settled):
    """At the decoder's own run count, zeros settle in exactly one round per run: 40 runs in the last round of the budget, 41 not."""
    data = cds.zeros(k)
    enc = oracle.encode("cheetah", data)
    nruns = cds.pick_runs(enc.size, 132)
    assert nruns == k
    out, st = cds.model_decode(model, enc, data.size, nruns)
    assert (st["rounds"], st["settled"]) == (rounds, settled), st
    if settled:
        assert (out == data).all() and st["queued"] == st["walks"] - nruns
    else:
        assert out.size == 0 and st["queued"] == st["walks"] - nruns + st["last_queued"] and st["last_queued"] > 0


@pytest.mark.parametrize("name", ["zero_hole", "spaces"])
def test_long_repeated_stretches_exhaust_the_budget(model, name):
    """36 MiB of zeros between text, and 36 MiB of spaces, do not settle within 40 rounds at the decoder's run count."""
    data = getattr(cds, name)()
    enc = oracle.encode("cheetah", data)
    out, st = cds.model_decode(model, enc, data.size, cds.pick_runs(enc.size, 132))
    assert st["settled"] == 0 and st["rounds"] == 40 and out.size == 0, st
    out, st = cds.model_decode(model, enc, data.size, 8)      # fewer runs than rounds: exact
    assert st["settled"] == 1 and (out == data).all()
