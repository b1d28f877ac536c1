"""Synthesized Chameleon, Cheetah and Lion streams (tests/synth_streams.py) on the CPU: every stream parses back to its manifest and every class
is where the manifest says, with the flag it was planted with and the value it must decode to; the plain in-order decoder and the oracle
agree on every stream at every capacity the GPU tests use; the CPU formulations of the parallel decoders (the decode-pass model, the
Cheetah round model, the range maps of the located paths) give the oracle's answer on them. The Lion walk models
(tests/lion_walk_model.cpp, tests/lion_piece_model.cpp), which compile density_b200/csrc/lion_walk.cuh itself, are checked against the
plain decoder, which shares no code with them."""
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
    ("lion", {"nbytes": 400000, "p_pred": 0.5, "cuts": tuple(k / 25 for k in range(1, 25)), "odd": True, "tail": (40, "raw2")}, 51),
    ("lion", {"nbytes": 300000, "p_pred": 0.3, "quiet": False, "copy_every": 41, "odd": False, "tail": (30, "clean")}, 52),
    ("lion", {"nbytes": 150000, "p_pred": 0.9, "cuts": (0.2, 0.45, 0.7), "odd": False, "tail": (26, "plain_end")}, 53),
    ("lion", {"nbytes": 1500000, "p_pred": 0.3, "quiet": False, "prot_states": True, "cuts": tuple(k / 10 for k in range(1, 10)),
              "tail": (63, "raw3")}, 54),
    ("lion", {"nbytes": 100000, "p_pred": 0.99, "odd": True, "tail": (9, "map1")}, 55),
]
LION = [i for i, c in enumerate(SMALL) if c[0] == "lion"]
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


# the lane (quad index mod 32) of a row, or of a block (mod 16), every quad of a placement sits on
LION_LANES = {"lane_0": (32, 0), "lane_15": (32, 15), "lane_16": (32, 16), "lane_31": (32, 31), "copy_row_lane_16": (32, 16),
              "after_copy_row_lane_0": (32, 0), "after_copy": (16, 0), "run_first": (16, 0), "run_last": (16, 15), "piece_first": (16, 0),
              "piece_last": (16, 15)}


def lion_coverage(streams):
    """{placement: Lion classes planted on it} and every class name noted, over (stream, manifest) pairs; every quad of a placement sits
    on its lane, and the quads behind copy-mode episodes follow the last copy-mode block"""
    on, names = collections.defaultdict(set), set()
    for _, m in streams:
        at = collections.defaultdict(set)
        for c, _, qi, _ in m["classes"]:
            at[qi].add(ss.lion_class(c)); names.add(c)
        copy = set(m["copy_blocks"])
        for k, v in m["placements"].items():
            mod, lane = LION_LANES[k]
            for x in v:
                assert x % mod == lane, (k, x)
                if "copy" in k:
                    assert x // 16 - 1 in copy and x // 16 not in copy, (k, x)
                    assert (k == "copy_row_lane_16") == ((x // 16 - 1) % 2 == 0) or k == "after_copy", (k, x)
                on[k] |= at[x]
    return on, names


def test_every_lion_class_is_on_every_placement():
    """every Lion class on the rows' lanes 0, 15, 16 and 31, lane 16 of a row whose first block is copy mode, lane 0 of a row behind one
    whose second block is, chunk-map run and piece edges and behind copy-mode episodes; the variants of the chunk-map writes, the self-map
    spans across a block, a row and copy-mode blocks, the stream start, and the predicted first tail quad behind a MAP at an unwritten
    bucket"""
    on, names = lion_coverage([stream(i) for i in LION])
    for k in ss.LION_PLACES:
        assert set(ss.LION_CLASSES) <= on[k], (k, set(ss.LION_CLASSES) - on[k])
    for cls in ("mapb_written_once", "mapb_twice"):
        assert {f"{cls}_{w}" for w in ("same_row", "earlier_row", "earlier_run", "earlier_piece")} <= names, cls
    assert {"map_unwritten_ctx_mapa", "map_unwritten_ctx_mapb_once", "map_unwritten_ctx_main_last", "self_span_cross_15_16",
            "self_span_cross_row", "self_span_cut_by_copy", "self_span_then_depth_1", "pred_chain_context0_stream_start"} <= names
    assert {SMALL[i][1]["odd"] for i in LION if "odd" in SMALL[i][1]} == {True, False}
    assert {stream(i)[1]["main_blocks"] % 2 for i in LION} == {0, 1}
    for i in LION:
        s, m = stream(i)
        out = oracle.decode("lion", s, 64 * s.size + 4096)
        if m["tail_expect"] is not None and out.size:                  # (not behind a malformed tail)
            q, want = m["tail_expect"]
            assert q == m["main_blocks"] * 16 and int(out[4 * q:4 * q + 4].view("<u4")[0]) == want, i


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
        elif alg == "lion":
            runs = ss.lion_dec_runs(s.size, m["main_blocks"])
        else:
            runs = ss.cheetah_dec_runs(s.size, m["main_blocks"])
        assert runs == m["run_blocks"], cap
    if len(m["run_blocks"]) > 1:
        on_seams = {q // ss.QPB[alg] for q in m["placements"].get("run_first", [])}
        assert on_seams and on_seams <= set(m["run_blocks"])


def test_prot_targets_cover_every_reachable_state():
    import protection as P
    for i in (2, 8, LION[3]):
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
            o = m["starts"][b] + ss.SIG["chameleon"]
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


# ---- Lion: the walk models against the plain decoder ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lion_walk_model(tmp_path_factory):
    import lion_streams as ls
    return ls.build_model(tmp_path_factory.mktemp("lion_walk"))


@pytest.mark.parametrize("i", LION)
def test_lion_walk_model_equals_the_plain_decoder(lion_walk_model, i):
    """tests/lion_walk_model.cpp (boundaries, unpack, chunk map, the walk of lion_walk.cuh, the tail) gives the plain decoder's bytes at the
    decoded size and every capacity below it is refused; its counts are the ones lion_streams.walk_counts reads off the stream"""
    import lion_streams as ls
    s, m = stream(i)
    if s.size > 3 * (1 << 19):
        s = s[:m["starts"][int(np.searchsorted(m["starts"], 1 << 20))]]
    size = m["decoded_size"] if s.size == stream(i)[0].size else 64 * s.size
    want = ss.decode_reference("lion", s, size)
    n, got, c = ls.run_model(lion_walk_model, s, size)
    assert n == len(want) and got.tobytes() == want, (i, n, len(want))
    if n:
        assert c == ls.walk_counts(s, got), (c, ls.walk_counts(s, got))
        for cap in (n - 1, n - 64):
            assert ls.run_model(lion_walk_model, s, cap)[0] == 0
    else:                                                            # a malformed tail: the main loop alone
        main = s[:m["tail_off"]]
        want = ss.decode_reference("lion", main, 64 * s.size)
        n, got, c = ls.run_model(lion_walk_model, main, len(want))
        assert n == len(want) > 0 and got.tobytes() == want and c == ls.walk_counts(main, got)


@pytest.fixture(scope="module")
def lion_piece_model(tmp_path_factory):
    import ctypes
    import os
    import subprocess
    so = os.path.join(str(tmp_path_factory.mktemp("lion_piece")), "lion_piece_model.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++",
                           os.path.join(os.path.dirname(os.path.abspath(__file__)), "lion_piece_model.cpp"), "-o", so])
    L = ctypes.CDLL(so)
    L.lion_piece_model_check.restype = ctypes.c_long
    L.lion_piece_model_check.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_uint64)]
    return L


def lion_cut_sets(m):
    """the manifest's cuts, chunk-map run seams, each side of planted classes, odd blocks, one-block and empty pieces, the blocks behind
    copy-mode episodes and automaton targets"""
    mb = m["main_blocks"]
    planted_blocks = sorted({b for _, b, _, _ in m["classes"]})
    pick = lambda xs, f: xs[int(f * (len(xs) - 1))] if xs else mb // 2
    seams = m["run_blocks"][1:]
    sets = [list(m["cut_blocks"]), [pick(seams, 0.5)], [pick(seams, 0.2), pick(seams, 0.7)],
            [pick(planted_blocks, 0.3), pick(planted_blocks, 0.3) + 1, pick(planted_blocks, 0.6)],
            [mb // 3 | 1, (mb // 2) | 1], [mb // 4, mb // 4 + 1, mb // 4 + 1, mb // 2]]
    after_copy = [b + 1 for b in m["copy_blocks"] if b + 1 < mb and b + 1 not in m["copy_blocks"]]
    if after_copy:
        sets.append(after_copy[1::max(1, len(after_copy) // 5)][:5])
    if m["prot_targets"]:
        sets.append([B for B, _ in m["prot_targets"][::max(1, len(m["prot_targets"]) // 7)]][:7])
    return [sorted(c for c in cs if 0 < c < mb) for cs in sets if cs]


@pytest.mark.parametrize("i", LION)
def test_lion_piece_model_at_the_planted_cuts(lion_piece_model, i):
    """tests/lion_piece_model.cpp: the walk relayed piece by piece (every piece laid out in rows of its own) equals the whole walk at the
    manifest's cuts and the cut sets of the GPU tests"""
    from test_sharded_lion_decode_cpu import walk_pieces
    s, m = stream(i)
    for cuts in lion_cut_sets(m):
        nb, counts = walk_pieces(lion_piece_model, s, [0] + cuts + [m["main_blocks"]])
        assert nb == m["main_blocks"], (i, cuts)
        assert counts[0] == counts[4] and counts[1] == counts[5], (i, cuts, counts)
