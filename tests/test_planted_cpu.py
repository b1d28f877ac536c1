"""The planted corpora (tests/planted.py) on the CPU: the (hash, fingerprint) inverse, the run geometry, the manifest, the oracle
and the single-run tile protocol models of tools/proto_tile_protocol_v6.py. No GPU needed."""
import numpy as np
import pytest

import oracle
import planted
from planted import TILE_QUADS, corpus, hf, quad_of, twin


def test_quad_of_inverts_hash_and_fingerprint():
    rng = np.random.default_rng(11)
    h = rng.integers(0, 1 << 16, 100000, dtype=np.uint64)
    f = rng.integers(0, 1 << 16, 100000, dtype=np.uint64)
    q = quad_of(h, f)
    h2, f2 = hf(q)
    assert (h2 == h.astype(np.int64)).all() and (f2 == f.astype(np.int64)).all()
    qs = rng.integers(0, 1 << 32, 100000, dtype=np.uint64)
    assert (quad_of(*hf(qs)) == qs).all()
    assert quad_of(0, 0) == 0 and quad_of(0xFFFF, 0xFFFF) == 0xEE4FF4DD == planted.ALL_ONES
    x = quad_of(0x1234, 0x5678)
    assert hf(twin(x)) == (0x1234, 0x5679)
    assert ((x * planted.M) & 0xFFFFFFFF) == ((twin(x) * planted.M) & 0xFFFFFFFF)   # same product


def test_run_geometry_on_an_h100():
    runs = planted.cham_runs(33 * planted.MIB)
    assert len(runs) == 132 and all(b - a == 16 for a, b in runs)
    assert planted.cham_runs(5 * planted.MIB + 402)[-1][1] == 321 and len(planted.cham_runs(5 * planted.MIB + 402)) == 20
    assert planted.cham_runs(300) == [(0, 1)]
    one = planted.chee_runs(planted.MIB + 13)
    assert len(one) == 64 and one[0] == (0, 1) and one[-1] == (63, 65)
    big = planted.chee_runs(33 * planted.MIB + 66)
    assert len(big) == 132 * 8 and {b - a for a, b in big} == {2, 3}
    assert len(planted.chee_runs(40 * 16384)) == 20


REQUIRED = {
    "cham33": ["stream_first", "stream_tail", "last_partial_tile", "copies_across_run", "copies_across_tile", "copies_across_region",
               "same_tile_other", "fp0_reread_later_tile", "all_ones_tile_start_miss", "alias_writer", "alias_reader", "class_list_140", "bucket_20_members", "bucket_21_members",
               "overflow_16_entries", "overflow_17_entries", "slot_4_buckets", "slot_5_buckets", "slot_6_buckets"]
              + [f"carry_{c}" for c in ("same", "other", "twin", "fp0_writer", "to_fp0", "fp0_same")]
              + [f"{v}_{w}" for v in ("fp0_fixed", "fp0_fresh", "quad0", "bucket0_member", "all_ones", "fp_ffff_fffe", "twin_fresh")
                 for w in ("run_first_tiles", "run_last_tile")],
    "cham129": ["copies_across_seam", "carry_same", "carry_twin", "carry_to_fp0", "stream_tail"],
    "copy3": ["before_burst", "inside_copy_block", "after_copy_block_miss", "after_copy_block_hit", "after_burst"],
    "cl1": ["quad0_fresh_context", "quad0_after_context0", "fp0_first_touch", "chunk_ab_before", "chunk_ab_after"]
           + [f"lion_ctx{m}_{w}" for m in (4, 5, 6) for w in ("before", "after")],
}
REQUIRED["cham5"] = REQUIRED["cham33"]
REQUIRED["cl33"] = REQUIRED["cl1"]


@pytest.mark.parametrize("name", sorted(planted.CORPORA))
def test_manifest_holds(name):
    data, man = corpus(name)
    q = data[:data.size // 4 * 4].view(np.uint32)
    pos = np.array([p for p, v, c in man])
    val = np.array([v for p, v, c in man], dtype=np.uint64)
    assert (q[pos].astype(np.uint64) == val).all()
    cls = planted.classes(man)
    missing = [c for c in REQUIRED[name] if c not in cls]
    assert not missing, missing
    nq = q.size
    if name.startswith("cham"):
        runs = planted.cham_runs(data.size)
        starts = {a * TILE_QUADS for a, b in runs}
        assert man[0][:2] == (0, quad_of(hf(man[0][1])[0], 0)) and hf(man[0][1])[1] == 0      # the stream's first quad: fp 0
        assert all(p >= nq - 66 for p in cls["stream_tail"])                                   # the last 264 bytes
        assert any(p - 3 in starts or p + 3 in starts for p in cls["copies_across_run"])
        offs = {p % TILE_QUADS for c in cls if c.endswith("_run_first_tiles") for p in cls[c]}
        assert {0, 127, 128, 255, 256, 4095} <= offs
        firsts = {p // TILE_QUADS for c in cls if c.endswith("_run_first_tiles") for p in cls[c]}
        assert {a + k for a, b in runs for k in range(3)} <= firsts                             # the first three tiles of every run
        lasts = {p // TILE_QUADS for c in cls if c.endswith("_run_last_tile") for p in cls[c]}
        assert {b - 1 for a, b in runs[:-1]} <= lasts
        # fingerprint-0 quads in buckets other than 0, all-ones record words, twins
        h, f = hf(val)
        assert ((f == 0) & (h != 0)).sum() > 500 and (val == planted.ALL_ONES).sum() > 100 and ((f == 0xFFFE).sum() > 50)
    if name == "cham129":
        for s in (64 * planted.MIB // 4, 128 * planted.MIB // 4):
            assert s - 1 in cls_pos(cls, "copies_across_seam") and s in cls_pos(cls, "copies_across_seam")
    if name.startswith("cl"):
        b = [p for p in cls["quad0_fresh_context"]]
        assert b and all(p % TILE_QUADS == 0 for p in b)


def cls_pos(cls, c):
    return set(cls[c])


@pytest.mark.parametrize("name", sorted(planted.CORPORA))
def test_corpus_round_trips_through_the_oracle(name):
    data, man = corpus(name)
    for alg in ("chameleon", "cheetah", "lion"):
        enc, copied = oracle.encode(alg, data, return_copied=True)
        assert (oracle.decode(alg, enc, data.size) == data).all(), alg
        if alg == "chameleon":
            if name in planted.QUIET:
                assert copied == 0, "meant for the fast path: must stay quiet"
            elif name == "copy3":
                assert copied >= 40


def _run_piece(name, run):
    data, man = corpus(name)
    q = data[:data.size // 4 * 4].view(np.uint32)
    a, b = planted.cham_runs(data.size)[run]
    return q, a, b


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_flag_pass_model_on_planted_run(seed):
    """cham_flag_pass6's protocol on the first 14 tiles of a run with aliasing and capacity plantings: the flags and the dictionary
    equal the in-order walk, and the mailboxes overflow exactly where intended (21 members of one bucket, 17 overflow entries)."""
    from tools import proto_tile_protocol_v6 as m6
    q, a, b = _run_piece("cham5", 2)
    piece = q[a * TILE_QUADS:(a + 14) * TILE_QUADS]
    want, want_tab = m6.reference_flags(piece)
    stats = {}
    got, tab, touched = m6.flag_pass(piece, seed=seed, stats=stats)
    assert (got == want).all(), int((got != want).sum())
    assert {int(k): int(tab[k]) for k in np.flatnonzero(touched)} == want_tab
    ov = stats["tile_overflow"]
    assert ov[4] is False and ov[5] is False                   # 4, 5, 6 buckets in one mailbox slot fit
    assert ov[6] is False and ov[7] is True                    # 20 members fit, 21 overflow
    assert ov[8] is False and ov[9] is True                    # 16 overflow entries fit, 17 overflow
    assert not any(ov[10:14])


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_decode_pass_model_on_planted_run(seed):
    """cham_decode_pass7's protocol on the same tiles, on the flag / payload sequence the in-order encoder makes from the stream start:
    mark-map aliases make suspects only, and the writers-only mailboxes overflow where intended."""
    from tools import proto_tile_protocol_v6 as m6
    q, a, b = _run_piece("cham5", 2)
    flags, _ = m6.reference_flags(q[:(a + 14) * TILE_QUADS])
    hit = (flags == 1) | ((flags == 2) & (q[:flags.size] == 0))
    lo = a * TILE_QUADS
    piece, is_plain = q[lo:lo + 14 * TILE_QUADS], ~hit[lo:]
    h, _f = hf(piece)
    payload = np.where(is_plain, piece.astype(np.uint64), h.astype(np.uint64))
    want, want_dic = m6.decode_reference(is_plain, payload)
    stats = {}
    got, dic = m6.decode_pass(is_plain, payload, seed=seed, stats=stats)
    assert (got == want).all(), int((got != want).sum())
    assert dic == want_dic
    ov = stats["tile_overflow"]
    assert ov[6] is False and ov[7] is True
    assert ov[8] is False and ov[9] is True
    assert not any(ov[10:14])
