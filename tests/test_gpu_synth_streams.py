"""Synthesized Chameleon and Cheetah streams (tests/synth_streams.py) through every single-device and sharded decode path on an H100
(pytest -m gpu). The answer is always oracle.decode(alg, stream, cap); every output buffer is exactly `cap` bytes followed by a 64-byte
canary. The streams hold what no encoder writes: MAPs at buckets never written or written only by their fingerprint-0 member, PLAIN
rewrites of the value a bucket holds, twins, pile-ups, MAP_B swaps of empty slots, predicted reads of contexts never written, placed at
the decoders' own tile, region, run and piece seams and behind copy-mode episodes."""
import ctypes

import numpy as np
import pytest

import oracle
import cl_decode_seams as cds
import synth_streams as ss
from test_gpu_sharded_decode import decode_pieces as cham_pieces
from test_gpu_sharded_protected_decode import decode_prot_pieces as cham_prot_pieces
from test_gpu_sharded_cheetah_decode import decode_pieces as chee_pieces
from test_gpu_sharded_cheetah_protected_decode import decode_prot_pieces as chee_prot_pieces
from test_gpu_sharded_lion_decode import decode_lion_pieces
import test_gpu_sharded_stream_decode as cham_located
import test_gpu_sharded_cheetah_stream_decode as chee_located
import test_gpu_sharded_stream_protected_decode as prot_located

pytestmark = pytest.mark.gpu
CANARY = 0xA5
MIB = 1 << 20
ALG_ID = {"chameleon": 0, "cheetah": 1, "lion": 2}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device; there is no CPU fallback")
    return torch


@pytest.fixture(scope="module")
def lib(torch_cuda):
    import density_b200
    return density_b200.load()


@pytest.fixture(scope="module")
def sms(torch_cuda):
    return torch_cuda.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return cds.build_model(tmp_path_factory.mktemp("cl_model"))


# (alg, plan, seed): quiet and copy-mode streams of both algorithms, all with well-formed tails except the two small "bad" ones. At its
# decoded size (about 37 MB) the 27 MiB Chameleon stream gives the decoder its full 132 runs.
PLANS = {
    "cham27": ("chameleon", {"nbytes": 27 * MIB, "cuts": (0.3, 0.55), "tail": (201, "raw1")}, 21),
    "cham4": ("chameleon", {"nbytes": 4 * MIB, "cuts": (0.2, 0.5, 0.8), "tail": (100, "raw2")}, 22),
    "cham4_copy": ("chameleon", {"nbytes": 4 * MIB, "quiet": False, "copy_every": 301, "cuts": (0.33, 0.66), "tail": (60, "raw2")}, 23),
    "cham_prot": ("chameleon", {"nbytes": 6 * MIB, "quiet": False, "prot_states": True, "tail": (138, "raw2")}, 24),
    "cham1": ("chameleon", {"nbytes": MIB, "tail": (16, "plain_end")}, 25),
    "cham_bad": ("chameleon", {"nbytes": 300000, "tail": (100, "map0")}, 26),
    "chee24_p2": ("cheetah", {"nbytes": 24 * MIB, "p_pred": 0.2, "cuts": (0.4, 0.7), "tail": (77, "raw1")}, 31),
    "chee4_p0": ("cheetah", {"nbytes": 4 * MIB, "p_pred": 0.0, "cuts": (0.25, 0.5, 0.75), "tail": (64, "clean")}, 32),
    "chee4_p5": ("cheetah", {"nbytes": 4 * MIB, "p_pred": 0.5, "cuts": (0.5,), "tail": (10, "raw2")}, 33),
    "chee4_p9": ("cheetah", {"nbytes": 4 * MIB, "p_pred": 0.9, "cuts": (0.3, 0.6), "tail": (40, "plain_end")}, 34),
    "chee2_p99": ("cheetah", {"nbytes": 2 * MIB, "p_pred": 0.99, "tail": (100, "raw2")}, 35),
    "chee4_copy": ("cheetah", {"nbytes": 4 * MIB, "p_pred": 0.3, "quiet": False, "copy_every": 211, "cuts": (0.5,), "tail": (91, "raw3")}, 36),
    "chee_prot": ("cheetah", {"nbytes": 3 * MIB, "p_pred": 0.3, "quiet": False, "prot_states": True, "tail": (20, "clean")}, 37),
    "chee_bad": ("cheetah", {"nbytes": 300000, "p_pred": 0.5, "tail": (9, "map1")}, 38),
}
MALFORMED = ("cham_bad", "chee_bad")
CHAM_CLASSES = {"map_unwritten", "map_unwritten_fixed", "map_bucket0_before_write", "map_bucket0_after_write", "bucket0_write",
                "plain_same_value", "plain_twin", "map_fp0_written_same_tile", "map_fp0_written_earlier_tile", "map_fp0_written_earlier_run",
                "map_fp0_written_earlier_piece", "pileup_4", "pileup_5", "pileup_20", "pileup_21"}
CHEE_CLASSES = {"mapa_unwritten", "mapb_unwritten", "mapa_written_once_earlier_run", "mapa_written_once_earlier_piece",
                "mapb_written_once_earlier_run", "mapb_twice_earlier_run", "mapb_written_once_earlier_piece", "mapb_twice_earlier_piece",
                "pred_unwritten_context", "pred_context0", "pred_self_chain", "pred_chain_through_context0"}
PLACES = {"chameleon": {"run_first", "run_last", "piece_first", "piece_last", "tile_first", "tile_last", "region_first", "region_last",
                        "after_copy"},
          "cheetah": {"run_first", "run_last", "piece_first", "piece_last", "after_copy"}}
_cache = {}


def case(name):
    """(alg, stream, manifest, oracle output at an unbounded capacity)"""
    if name not in _cache:
        alg, plan, seed = PLANS[name]
        s, m = ss.build(alg, plan, seed)
        full = oracle.decode(alg, s, 64 * s.size + 4096)
        _cache[name] = (alg, s, m, full)
    return _cache[name]


def caps_of(alg, size, m):
    """exact, one byte short, one block short, and a capacity that ends inside a tile in the middle of a decoder run"""
    bs = ss.BS[alg]
    mid = (size // 2) // (64 * bs) * (64 * bs) + 17 * bs + 100
    return [size, size - 1, size - bs, min(mid, size - 1)]


def _stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def dev_decode(torch, lib, alg, enc, cap, path):
    """-> (rc, size, output, canary) of density_b200_decode_device_path (path None: density_b200_decode_device)"""
    d_in = torch.from_numpy(np.ascontiguousarray(enc)).cuda()
    d_out = torch.full((cap + 64,), CANARY, dtype=torch.uint8, device="cuda")
    d_sz = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    if path is None:
        rc = lib.density_b200_decode_device(ALG_ID[alg], d_in.data_ptr(), enc.size, d_out.data_ptr(), cap, d_sz.data_ptr(), _stream(torch))
    else:
        rc = lib.density_b200_decode_device_path(ALG_ID[alg], d_in.data_ptr(), enc.size, d_out.data_ptr(), cap, d_sz.data_ptr(),
                                                 _stream(torch), path)
    torch.cuda.synchronize()
    m = int(d_sz.item())
    out = d_out.cpu().numpy()
    return rc, m, out[:max(m, 0)], out[cap:]


def first_diff(a, b):
    k = min(a.size, b.size)
    d = np.flatnonzero(a[:k] != b[:k])
    return int(d[0]) if d.size else k


def check(got_m, got, want, what):
    assert got_m == want.size and (got == want).all(), f"{what}: size {got_m} vs {want.size}, first differing byte {first_diff(got, want)}"


def cham_status(lib):
    s = (ctypes.c_uint64 * 10)()
    assert lib.density_b200_decode_status(s) == 0
    return list(s)


def chee_rounds(lib):
    r = (ctypes.c_uint32 * 4)()
    assert lib.density_b200_cheetah_decode_rounds(r) == 0
    return list(r)


def test_streams_carry_their_classes_on_the_decoders_seams(sms):
    """the streams of this file hold every class and every placement, well-formed tails where they should, and the plantings sit on
    the decoder's runs at every capacity the tests decode with that is not a capacity error: the decoded size, one byte and one block
    less (bounds_layout bounds the block count by the capacity, so the run count follows it)"""
    seen, places = {"chameleon": set(), "cheetah": set()}, {"chameleon": set(), "cheetah": set()}
    for name in PLANS:
        alg, s, m, full = case(name)
        assert (full.size == 0) == (name in MALFORMED), name
        assert m["decoded_size"] == (full.size or oracle.decode(alg, s[:m["tail_off"]], 64 * s.size).size)
        seen[alg].update(c for c, *_ in m["classes"])
        places[alg].update(k for k, v in m["placements"].items() if v)
        size = m["decoded_size"]
        for cap in (size, size - 1, size - ss.BS[alg]):
            runs = [ss.TILE_BLOCKS * t0 for t0, _ in ss.cham_dec_runs(s.size, cap, m["main_blocks"], sms)] if alg == "chameleon" else \
                ss.cheetah_dec_runs(s.size, m["main_blocks"], sms)
            assert runs == m["run_blocks"], (name, cap)
    assert len(case("cham27")[2]["run_blocks"]) == min(sms, 132)
    assert CHAM_CLASSES <= seen["chameleon"], CHAM_CLASSES - seen["chameleon"]
    assert CHEE_CLASSES <= seen["cheetah"], CHEE_CLASSES - seen["cheetah"]
    for alg in PLACES:
        assert PLACES[alg] <= places[alg], (alg, PLACES[alg] - places[alg])


# ---- a. single device --------------------------------------------------------------------------------------------------------------
CHAM = [k for k in PLANS if PLANS[k][0] == "chameleon"]
CHEE = [k for k in PLANS if PLANS[k][0] == "cheetah"]


@pytest.mark.parametrize("name", CHAM)
def test_chameleon_paths(torch_cuda, lib, name):
    """paths 0 and 1 (and 3 on the smaller streams) and decode_device at every capacity class: the oracle's answer; the status of the
    parallel decoder reports the manifest's main loop"""
    torch = torch_cuda
    alg, s, m, full = case(name)
    size = full.size if full.size else oracle.decode(alg, s[:m["tail_off"]], 64 * s.size).size
    for cap in caps_of(alg, size, m):
        want = oracle.decode(alg, s, cap)
        for path in ((0, 1, None) if s.size > 5 * MIB else (0, 1, 3, None)):
            if path == 3 and cap != size:
                continue
            rc, got_m, got, tail = dev_decode(torch, lib, alg, s, cap, path)
            assert rc == 0 and (tail == CANARY).all(), (name, cap, path)
            check(got_m, got, want, f"{name} cap {cap} path {path}")
            if path == 1 and cap == size:
                st = cham_status(lib)
                assert st[1] == m["main_blocks"] and st[2] == m["tail_off"], (st, m["main_blocks"], m["tail_off"])
                # copy-mode blocks: the boundaries come from the in-order walk, which clears the non-quiet bit once it has them
                assert st[3] == 0 and bool(st[6]) == bool(m["copy_blocks"]), st
                assert (st[4] != 0) == (full.size == 0), st          # error: the malformed tails (dec_tail gives up)
                if st[6]:                                    # the in-order walk's automaton behind the main loop
                    assert (st[7], st[8], st[9]) == tuple(m["state"][:3]), (st, m["state"])
                else:                                        # quiet: only the last main-loop block's incompressible bit
                    assert st[5] == m["state"][2], (st, m["state"])


@pytest.mark.parametrize("name", CHEE)
def test_cheetah_paths(torch_cuda, lib, sms, model, name):
    """paths 0 and 3 and decode_device give the oracle's answer; path 1 gives it exactly when the CPU model of the rounds settles, size 0
    otherwise, and its rounds, settled flag and queued walks are the model's"""
    torch = torch_cuda
    alg, s, m, full = case(name)
    size = full.size if full.size else oracle.decode(alg, s[:m["tail_off"]], 64 * s.size).size
    nruns = cds.pick_runs(s.size, sms)
    for cap in caps_of(alg, size, m):
        want = oracle.decode(alg, s, cap)
        for path in ((0, None) if s.size > 5 * MIB or PLANS[name][1].get("p_pred", 0) >= 0.9 else (0, 3, None)):
            rc, got_m, got, tail = dev_decode(torch, lib, alg, s, cap, path)
            assert rc == 0 and (tail == CANARY).all(), (name, cap, path)
            check(got_m, got, want, f"{name} cap {cap} path {path}")
        rc, got_m, got, tail = dev_decode(torch, lib, alg, s, cap, 1)
        assert rc == 0 and (tail == CANARY).all()
        if cap == size:
            r = chee_rounds(lib)
            mo, st = cds.model_decode(model, s, cap, nruns)
            assert (r[0], r[1], r[2]) == (st["rounds"], st["settled"], st["queued"]), (name, r, st)
            if st["settled"] and want.size:
                check(got_m, got, want, f"{name} path 1")
                assert mo.size == want.size and (mo == want).all()
            else:
                assert got_m == 0, name
        else:
            assert got_m == 0, (name, cap)


@pytest.mark.parametrize("alg", ["chameleon", "cheetah"])      # Lion: tests/test_gpu_lion_synth_streams.py
def test_reference_symbols_host_and_device(torch_cuda, lib, alg):
    torch = torch_cuda
    for name in [k for k in PLANS if PLANS[k][0] == alg and PLANS[k][1]["nbytes"] <= 4 * MIB and k not in MALFORMED][:2] + \
            [k for k in MALFORMED if PLANS[k][0] == alg]:
        _, s, m, full = case(name)
        size = full.size if full.size else 1 << 20
        out = np.full(size + 64, CANARY, np.uint8)
        n = getattr(lib, f"{alg}_decode")(s.ctypes.data, s.size, out.ctypes.data, size)
        assert n == full.size and (out[:n] == full).all() and (out[size:] == CANARY).all(), name
        d_in = torch.from_numpy(s).cuda()
        d_out = torch.full((size + 64,), CANARY, dtype=torch.uint8, device="cuda")
        n = getattr(lib, f"{alg}_decode")(ctypes.c_void_p(d_in.data_ptr()), s.size, ctypes.c_void_p(d_out.data_ptr()), size)
        got = d_out.cpu().numpy()
        assert n == full.size and (got[:n] == full).all() and (got[size:] == CANARY).all(), name


@pytest.mark.parametrize("alg", ss.ALGS)
def test_codec_instance_two_streams(torch_cuda, lib, alg):
    """a codec instance decodes two synthesized streams in a row like oracle.Codec: the second meets the first one's dictionary"""
    from density_b200.codec import CodecInstance
    s1, _ = ss.build(alg, {"nbytes": MIB, "tail": (0, "clean")}, 41)
    s2, _ = ss.build(alg, {"nbytes": MIB, "tail": (0, "clean")}, 42)
    ref, dec = oracle.Codec(alg), CodecInstance(alg)
    try:
        for s in (s1, s2):
            want = ref.decode(s, 64 * s.size)
            out = np.full(want.size + 64, CANARY, np.uint8)
            assert dec.decode(s, out[:want.size]) == want.size
            assert (out[:want.size] == want).all() and (out[want.size:] == CANARY).all()
    finally:
        dec.close()


@pytest.mark.parametrize("alg", ss.ALGS)
def test_second_call_of_a_codec_instance_one_shot(torch_cuda, lib, alg):
    """the second call of an oracle.Codec is encoded against a warm dictionary; the one-shot paths decode it from a fresh one, so its MAPs
    name buckets this stream never wrote"""
    from conftest import payload
    enc = oracle.Codec(alg)
    enc.encode(payload("text", 3 * MIB, seed=5))
    s = enc.encode(payload("text", 3 * MIB + 11, seed=6))
    size = 3 * MIB + 11
    want = oracle.decode(alg, s, size)
    for path in (0, 1, 3, None):
        rc, m, got, tail = dev_decode(torch_cuda, lib, alg, s, size, path)
        assert rc == 0 and (tail == CANARY).all()
        if alg == "cheetah" and path == 1 and m == 0:
            continue
        check(m, got, want, f"{alg} path {path}")


# ---- d. sharded, known cuts -------------------------------------------------------------------------------------------------------
def pieces_at(alg, s, m, cut_blocks, full):
    """the stream cut at main-loop block starts; each piece's capacity is what its blocks decode to (the last piece: the rest)"""
    offs = [0] + [m["starts"][b] for b in cut_blocks] + [s.size]
    bs = ss.BS[alg]
    sizes = [(b1 - b0) * bs for b0, b1 in zip([0] + cut_blocks, cut_blocks)]
    sizes.append(full.size - sum(sizes))
    return [s[offs[r]:offs[r + 1]] for r in range(len(offs) - 1)], sizes


def cut_sets(alg, s, m, sms):
    """cuts at the manifest's piece cuts, on a decoder run seam, right before and after planted classes, one-block and empty pieces"""
    seams = m["run_blocks"][1:]
    planted_blocks = sorted({b for _, b, _, _ in m["classes"]})
    mb = m["main_blocks"]
    pick = lambda xs, f: xs[int(f * (len(xs) - 1))] if xs else mb // 2
    sets = [list(m["cut_blocks"]) or [mb // 2], [pick(seams, 0.5)], [pick(planted_blocks, 0.3), pick(planted_blocks, 0.3) + 1],
            [pick(seams, 0.2), pick(seams, 0.2) + 1, pick(seams, 0.7)], [mb // 3, mb // 3, 2 * mb // 3]]
    after_copy = [b + 1 for b in m["copy_blocks"] if b + 1 < mb and b + 1 not in m["copy_blocks"]]
    out = [sorted(c for c in cs if 0 < c < mb) for cs in sets]
    return [c for c in out if c], after_copy


# Cheetah streams whose sharded decode must settle within the round budget (few predicted quads); at higher predicted densities a cut
# set may be refused when the rounds do not settle, and whatever is accepted must be exact
MUST_SETTLE = ("chee4_p0", "chee24_p2", "chee4_copy", "chee_prot")


def quiet_pieces(torch, lib, alg, s, pieces, caps):
    """(decoded pieces, verdict flags) of the quiet sharded driver of alg"""
    caps = [max(c, 4) for c in caps]
    if alg == "chameleon":
        got, (flags, _, _), canaries = cham_pieces(torch, lib, pieces, caps)
        assert canaries
    else:
        pc = [0] + list(np.cumsum([p.size for p in pieces]))
        got, (flags, _, _), _, _ = chee_pieces(torch, lib, np.concatenate(pieces), pc, caps=caps)
    return got, flags


@pytest.mark.parametrize("name", ["cham4", "cham27", "chee4_p0", "chee4_p5", "chee24_p2"])
def test_sharded_known_cuts_quiet(torch_cuda, lib, sms, name):
    torch = torch_cuda
    alg, s, m, full = case(name)
    sets, _ = cut_sets(alg, s, m, sms)
    accepted = 0
    for cuts in sets:
        pieces, caps = pieces_at(alg, s, m, cuts, full)
        got, flags = quiet_pieces(torch, lib, alg, s, pieces, caps)
        if flags == 0:
            accepted += 1
            cat = np.concatenate(got)
            check(cat.size, cat, full, f"{name} cuts {cuts}")
        else:
            assert alg == "cheetah" and name not in MUST_SETTLE, (name, cuts, flags)
    assert accepted >= 1 or name not in MUST_SETTLE, name


@pytest.mark.parametrize("name", ["cham4_copy", "chee4_copy"])
def test_quiet_paths_refuse_copy_mode(torch_cuda, lib, sms, name):
    """a stream with copy-mode blocks is refused by the quiet sharded paths when a piece after the first needs copy mode; the quiet
    Chameleon path refuses it whole too, the Cheetah one lets the first piece use copy mode (and must then be exact)"""
    alg, s, m, full = case(name)
    for cuts in ([], [m["main_blocks"] // 2]):
        pieces, caps = pieces_at(alg, s, m, cuts, full)
        got, flags = quiet_pieces(torch_cuda, lib, alg, s, pieces, caps)
        if alg == "cheetah" and not cuts:
            assert flags == 0, name
            check(got[0].size, got[0], full, f"{name} whole")
        else:
            assert flags != 0, (name, cuts)


@pytest.mark.parametrize("name", ["cham4_copy", "cham_prot", "chee4_copy", "chee_prot"])
def test_sharded_known_cuts_protected(torch_cuda, lib, sms, name):
    torch = torch_cuda
    alg, s, m, full = case(name)
    if not full.size:
        s = s[:m["tail_off"]]
        full = oracle.decode(alg, s, 64 * s.size)
    sets, after_copy = cut_sets(alg, s, m, sms)
    if after_copy:
        sets.append([after_copy[len(after_copy) // 2]])
    sets.append([B for B, _ in m["prot_targets"][::max(1, len(m["prot_targets"]) // 7)]][:7])
    for cuts in sets:
        cuts = sorted(c for c in cuts if 0 < c < m["main_blocks"])
        if not cuts:
            continue
        pieces, caps = pieces_at(alg, s, m, cuts, full)
        caps = [max(c, 4) for c in caps]
        if alg == "chameleon":
            flags, total, got, _ = cham_prot_pieces(torch, lib, pieces, caps)
        else:
            flags, total, got, _, _ = chee_prot_pieces(torch, lib, pieces, caps)
        if flags == 0:
            cat = np.concatenate(got)
            check(cat.size, cat, full, f"{name} cuts {cuts}")
        else:
            assert alg == "cheetah" and name not in MUST_SETTLE, (name, cuts, flags)


@pytest.mark.parametrize("prot", [False, True])
@pytest.mark.parametrize("seed", range(3))
def test_sharded_lion_synth_streams(torch_cuda, lib, seed, prot):
    """the sharded Lion decoder, plain and protected, on well-formed Lion streams with random flags (lion_streams.synth_stream), cut at
    main-loop block starts: one-block, empty and ordinary pieces, W = 1 .. 5"""
    import lion_streams as ls
    s = ls.synth_stream(100 + seed, 3000 + 500 * seed, p_pred=(0.5, 0.9, 0.2)[seed])
    full = oracle.decode("lion", s, ls.decode_cap(s))
    assert full.size
    offs, idx = [], 0
    for copy, flags, _ in ls.blocks(s):
        offs.append(idx)
        idx += ls.BS if copy else ls.SIG + sum(4 if f == 0 else 2 if f >= 6 else 0 for f in flags)
    nb = len(offs)
    accepted = 0
    for cut_blocks in ([], [nb // 2], [nb // 3, nb // 3 + 1, 2 * nb // 3], [5, 5, nb // 2, nb - 3]):
        cuts = [0] + [offs[b] for b in cut_blocks] + [s.size]
        caps = [(b1 - b0) * ls.BS for b0, b1 in zip([0] + cut_blocks, cut_blocks)]
        caps.append(full.size - sum(caps))
        pieces = [s[cuts[r]:cuts[r + 1]] for r in range(len(cuts) - 1)]
        flags, total, outs = decode_lion_pieces(torch_cuda, lib, pieces, [max(c, 4) for c in caps], prot=prot)[:3]
        if flags == 0 or not cut_blocks:
            assert flags == 0, (seed, prot, cut_blocks)
            accepted += 1
            cat = np.concatenate(outs)
            check(cat.size, cat, full, f"lion seed {seed} prot {prot} cuts {cut_blocks}")
    assert accepted >= 1


# ---- e. sharded, unknown cuts ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cham4", "chee4_p0", "cham4_copy", "chee4_copy"])
def test_located_pieces(torch_cuda, lib, name):
    """the located paths cut the stream at byte ranges (equal ranges of 2, 3, 5 and 8 ranks, empty middle ranges, a range that starts on
    a block start): each rank finds where its piece starts; the pieces decode to the oracle's output. Quiet streams through the quiet
    located paths, copy-mode streams through the protected one."""
    torch = torch_cuda
    alg, s, m, full = case(name)
    quiet = not m["copy_blocks"]
    if quiet:
        lays = (cham_located if alg == "chameleon" else chee_located).layouts(s)
    else:
        import prot_locate_model as L
        k, U = s.size // L.RANGE_UNIT, L.RANGE_UNIT
        lays = {"two": L.layout(s.size, [k // 2 * U, None]), "five": L.layout(s.size, [k // 5 * U, k // 3 * U, 0, U, None]),
                "eight": L.layout(s.size, [k // 8 * U] * 7 + [None])}
    for key, lay in lays.items():
        if quiet and alg == "chameleon":
            got, (flags, total, _), canaries, _ = cham_located.decode_located(torch, lib, s, lay)
            assert canaries
        elif quiet:
            got, (flags, total, _), canaries, _, _ = chee_located.decode_located(torch, lib, s, lay)
            assert canaries
        else:
            flags, total, got, _ = prot_located.decode_located(torch, lib, alg, s, lay)
        if flags == 0:
            cat = np.concatenate(got) if got else np.zeros(0, np.uint8)
            check(cat.size, cat, full, f"{name} {key}")
        else:
            assert alg == "cheetah" and name not in MUST_SETTLE, (name, key, flags)
