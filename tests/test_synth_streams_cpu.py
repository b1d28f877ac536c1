"""Synthesized Chameleon and Cheetah streams (tests/synth_streams.py) on the CPU: every stream parses back to its manifest and every class
is where the manifest says, with the flag it was planted with and the value it must decode to; the plain in-order decoder and the oracle
agree on every stream at every capacity the GPU tests use; the CPU formulations of the parallel decoders (the decode-pass model, the
Cheetah round model, the range maps of the located paths) give the oracle's answer on them."""
import collections

import numpy as np
import pytest

import oracle
import cl_decode_seams as cds
import planted
import synth_streams as ss

# the small streams of the CPU checks: (alg, plan, seed)
SMALL = [
    ("chameleon", {"nbytes": 700000, "cuts": (0.15, 0.3, 0.45, 0.6, 0.8)}, 1),
    ("chameleon", {"nbytes": 200000, "quiet": False, "copy_every": 97, "tail": (150, "raw2")}, 2),
    ("chameleon", {"nbytes": 6000000, "quiet": False, "prot_states": True, "tail": (37, "raw1")}, 3),
    ("cheetah", {"nbytes": 600000, "p_pred": 0.5, "cuts": (0.1, 0.25, 0.4, 0.5, 0.6, 0.75, 0.9)}, 4),
    ("cheetah", {"nbytes": 150000, "p_pred": 0.0, "quiet": False, "copy_every": 61, "tail": (60, "map0")}, 5),
    ("cheetah", {"nbytes": 150000, "p_pred": 0.2, "tail": (71, "raw3")}, 6),
    ("cheetah", {"nbytes": 100000, "p_pred": 0.9, "tail": (100, "plain_end")}, 7),
    ("cheetah", {"nbytes": 80000, "p_pred": 0.99, "tail": (9, "map1")}, 8),
    ("cheetah", {"nbytes": 2000000, "p_pred": 0.3, "quiet": False, "prot_states": True}, 9),
]
CHAM_CLASSES = {"map_unwritten", "map_unwritten_fixed", "map_bucket0_before_write", "map_bucket0_after_write", "bucket0_write",
                "plain_same_value", "plain_same_value_reader", "plain_twin", "plain_twin_reader", "map_fp0_written_same_tile",
                "map_fp0_written_earlier_tile", "map_fp0_written_earlier_run", "map_fp0_written_earlier_piece", "pileup_4", "pileup_5",
                "pileup_20", "pileup_21"}
CHEE_CLASSES = {"mapa_unwritten", "mapb_unwritten", "mapa_written_once_earlier_run", "mapa_written_once_earlier_piece",
                "mapb_written_once_earlier_run", "mapb_twice_earlier_run", "mapb_written_once_earlier_piece", "mapb_twice_earlier_piece",
                "pred_unwritten_context", "pred_context0", "pred_self_chain", "pred_chain_through_context0"}
_cache = {}


def stream(i):
    if i not in _cache:
        alg, plan, seed = SMALL[i]
        _cache[i] = ss.build(alg, plan, seed)
    return _cache[i]


def caps(alg, m, size):
    """the capacities of the GPU tests: exact, one byte short, one block short, and one that ends inside a tile of a decoder run"""
    bs = ss.BS[alg]
    mid = (size // 2) // (64 * bs) * (64 * bs) + 17 * bs + 100
    return [size, size - 1, size - bs, min(mid, size - 1)]


@pytest.mark.parametrize("i", range(len(SMALL)))
def test_stream_parses_back_to_its_manifest(i):
    alg = SMALL[i][0]
    s, m = stream(i)
    w = ss.walk(alg, s)
    assert w["main_blocks"] == m["main_blocks"] and w["tail_off"] == m["tail_off"] and w["state"] == m["state"]
    assert [b for b, c in enumerate(w["copy"]) if c] == [b for b in m["copy_blocks"] if b < w["main_blocks"]]
    assert list(m["block_offsets"][:w["main_blocks"]]) == w["starts"]
    for B, st in m["prot_targets"]:
        assert w["before"][B] == st, (B, st, w["before"][B])
    if SMALL[i][1].get("quiet", True):
        assert not m["copy_blocks"]
    else:
        assert m["copy_blocks"]


@pytest.mark.parametrize("i", range(len(SMALL)))
def test_classes_are_where_the_manifest_says(i):
    """every planted quad has its flag in the stream and decodes (oracle) to the value its class says"""
    alg = SMALL[i][0]
    s, m = stream(i)
    out = oracle.decode(alg, s[:m["tail_off"]], 64 * s.size + 4096)         # the main loop alone: a malformed tail decodes to size 0
    assert out.size >= m["main_blocks"] * ss.BS[alg]
    quads = out[:m["main_blocks"] * ss.BS[alg]].view("<u4")
    for cls, b, qi, expect in m["classes"]:
        fl = ss.flags_of(alg, s, m, b)[qi % ss.QPB[alg]]
        assert fl == m["planted_flags"][qi], (cls, b, qi)
        if expect is not None:
            assert int(quads[qi]) == expect, (cls, qi, hex(int(quads[qi])), hex(expect))


PLACES = {"chameleon": {"run_first", "run_last", "piece_first", "piece_last", "tile_first", "tile_last", "region_first", "region_last",
                        "after_copy"},
          "cheetah": {"run_first", "run_last", "piece_first", "piece_last", "after_copy"}}


def test_every_class_is_present_at_every_placement():
    seen, places = collections.defaultdict(set), collections.defaultdict(set)
    for i in range(len(SMALL)):
        alg = SMALL[i][0]
        s, m = stream(i)
        seen[alg].update(c for c, *_ in m["classes"])
        places[alg].update(k for k, v in m["placements"].items() if v)
        planted_at = {qi for _, _, qi, _ in m["classes"]}
        assert all(q in planted_at for v in m["placements"].values() for q in v)
    assert CHAM_CLASSES <= seen["chameleon"], CHAM_CLASSES - seen["chameleon"]
    assert CHEE_CLASSES <= seen["cheetah"], CHEE_CLASSES - seen["cheetah"]
    for alg in PLACES:
        assert PLACES[alg] <= places[alg], (alg, PLACES[alg] - places[alg])


@pytest.mark.parametrize("i", range(len(SMALL)))
def test_plantings_sit_on_the_runs_of_the_decoding_capacity(i):
    """the decoder's runs at the capacities the streams are decoded with that are not capacity errors (the decoded size, one byte and
    one block less) are the runs the plantings were placed at; the run edges carry classes"""
    alg = SMALL[i][0]
    s, m = stream(i)
    size = m["decoded_size"]
    full = oracle.decode(alg, s, 64 * s.size + 4096)
    assert size == (full.size or oracle.decode(alg, s[:m["tail_off"]], 64 * s.size).size)
    for cap in (size, size - 1, size - ss.BS[alg]):
        if alg == "chameleon":
            runs = [ss.TILE_BLOCKS * t0 for t0, _ in ss.cham_dec_runs(s.size, cap, m["main_blocks"])]
        else:
            runs = ss.cheetah_dec_runs(s.size, m["main_blocks"])
        assert runs == m["run_blocks"], cap
    if len(m["run_blocks"]) > 1:
        on_seams = {q // ss.QPB[alg] for q in m["placements"].get("run_first", [])}
        assert on_seams and on_seams <= set(m["run_blocks"])


def test_prot_targets_cover_every_reachable_state():
    import protection as P
    for i in (2, 8):
        _, m = stream(i)
        assert {st for _, st in m["prot_targets"]} == P.reachable_states()


@pytest.mark.parametrize("i", range(len(SMALL)))
def test_reference_decoder_equals_oracle(i):
    """the plain decoder and the oracle agree, at every capacity the GPU tests use; the automaton streams are compared on their first
    MiB or so, cut at a main-loop block start"""
    alg = SMALL[i][0]
    s, m = stream(i)
    if s.size > 3 * (1 << 19):
        s = s[:m["starts"][int(np.searchsorted(m["starts"], 1 << 20))]]
    full = oracle.decode(alg, s, 64 * s.size + 4096)
    ref = ss.decode_reference(alg, s, 64 * s.size + 4096)
    assert len(ref) == full.size and ref == full.tobytes()
    if full.size:
        for cap in caps(alg, None, full.size)[1:]:
            want = oracle.decode(alg, s, cap)
            got = ss.decode_reference(alg, s, cap)
            assert len(got) == want.size == 0, cap                   # every cap below the size is a capacity error


@pytest.mark.parametrize("alg", ss.ALGS)
def test_every_tail_length(alg):
    """every tail length 0 .. SIG + BS - 1 behind a short stream, with and without a copy penalty pending: the plain decoder and the
    oracle agree, and the malformed ends (a signature cut short, a MAP with 0 or 1 byte left) decode to size 0"""
    ends = collections.Counter()
    for L, end in ss.tail_lengths(alg):
        for plan in ({"nbytes": 3000, "tail": (L, end)}, {"nbytes": 3000, "quiet": False, "copy_every": 5, "copy_at_end": L % 2 == 0, "tail": (L, end)}):
            s, m = ss.build(alg, dict(plan, plant=False), L)
            ends[m["tail_class"]] += 1
            want = oracle.decode(alg, s, 64 * s.size + 4096)
            got = ss.decode_reference(alg, s, 64 * s.size + 4096)
            assert got == want.tobytes(), (L, end, m["tail_class"])
            malformed = m["tail_class"] in ("tail_short_signature", "tail_map0", "tail_map1")
            assert (want.size == 0) == malformed, (L, end, m["tail_class"], want.size)
    assert set(ends) >= {"tail_empty", "tail_copy_pending", "tail_short_signature", "tail_clean", "tail_plain_end", "tail_raw1", "tail_raw2",
                         "tail_raw3", "tail_map0", "tail_map1"}, ends


def test_codec_instance_second_call():
    """a codec instance decoding two synthesized streams in a row: the second meets the first one's dictionary"""
    for alg in ss.ALGS:
        s1, _ = ss.build(alg, {"nbytes": 60000}, 11)
        s2, _ = ss.build(alg, {"nbytes": 60000}, 12)
        ref, st = oracle.Codec(alg), {}
        for s in (s1, s2):
            want = ref.decode(s, 64 * s.size)
            assert ss.decode_reference(alg, s, 64 * s.size, st) == want.tobytes()


def test_decode_pass_model():
    """tools/proto_tile_protocol_v6.decode_pass on the (is_plain, payload) sequence of the small Chameleon streams (copy-mode blocks
    left out: they neither read nor write the dictionary) against the plain decoder"""
    from tools import proto_tile_protocol_v6 as v6
    for i in (0, 1):
        s, m = stream(i)
        is_plain, payload, keep = [], [], []
        ref = np.frombuffer(ss.decode_reference("chameleon", s[:m["tail_off"]], 64 * s.size)[:m["main_blocks"] * 256], "<u4")
        for b in range(m["main_blocks"]):
            if b in m["copy_blocks"]:
                continue
            keep.append(b)
            fl = ss.flags_of("chameleon", s, m, b)
            o = m["starts"][b] + ss.SIG
            for f in fl:
                is_plain.append(f == ss.PLAIN)
                n = 4 if f == ss.PLAIN else 2
                payload.append(int.from_bytes(s[o:o + n].tobytes(), "little"))
                o += n
        is_plain, payload = np.array(is_plain), np.array(payload, np.uint64)
        stats = {}
        got, dic = v6.decode_pass(is_plain, payload, stats=stats)
        want = ref.reshape(-1, 64)[keep].reshape(-1)
        assert (got == want).all(), (i, int((got != want).sum()))
        assert dic == v6.decode_reference(is_plain, payload)[1]
        if not m["copy_blocks"] and any(c == "pileup_21" for c, *_ in m["classes"]):   # (without copy blocks the model's tiles are the kernel's)
            assert stats["overflow"] >= 1                           # the 21-writer pile-up sends its tile to the in-order replay


@pytest.fixture(scope="module")
def cl_model(tmp_path_factory):
    return cds.build_model(tmp_path_factory.mktemp("cl_model"))


@pytest.mark.parametrize("i", [i for i, c in enumerate(SMALL) if c[0] == "cheetah"])
def test_cheetah_round_model(cl_model, i):
    """tests/cl_model.cpp (the run-parallel Cheetah decoder's scheme on the CPU, sharing cl_core.cuh with the kernels) at 1 run, 5 runs
    and the H100 run count: exact whenever its rounds settle within the budget, and settled at 1 run"""
    s, m = stream(i)
    size = m["decoded_size"]
    want = oracle.decode("cheetah", s, size)
    for nruns in (1, 5, cds.pick_runs(s.size, planted.H100_SMS)):
        out, st = cds.model_decode(cl_model, s, size, nruns)
        assert st["main_blocks"] == m["main_blocks"], (nruns, st)
        if nruns == 1:
            assert st["settled"], st
        if st["settled"]:
            assert out.size == want.size and (out == want).all(), (nruns, st)
