"""Collision steps (tests/cl_steps.py) on the CPU: the manifest, the flags the plantings get in the oracle's stream, the run-decomposition
prototypes and the lane-level model of the encoders' flag passes (tests/cl_step_model.py). No GPU needed."""
import collections

import numpy as np
import pytest

import cl_step_model as M
import cl_steps
import oracle
import planted
from cl_steps import CLASSES, COPY, SINGLE
from tools import proto_cheetah_runs, proto_lion_runs

ALGS = ("cheetah", "lion")
_flags = {}


def oracle_flags(alg, name):
    """(flag per quad, copy mode per block) of the oracle's stream"""
    if (alg, name) not in _flags:
        data = cl_steps.build(name)[0]
        _flags[(alg, name)] = cl_steps.stream_flags(alg, oracle.encode(alg, data), data.size)
    return _flags[(alg, name)]


@pytest.mark.parametrize("name", sorted(cl_steps.CORPORA))
def test_manifest_holds(name):
    data, man, S = cl_steps.build(name)
    q = data[:data.size // 4 * 4].view(np.uint32)
    pos = np.array([p for p, *_ in man])
    assert (q[pos] == np.array([v for _, v, *_ in man], np.uint32)).all()
    steps = [(p, v, c, w) for p, v, c, w, r, *_ in man if r == "step"]
    h = planted.hf(np.array([v for _, v, _, _ in steps], np.uint32))[0]
    assert set(h.tolist()) <= set(S)
    at = collections.defaultdict(set)                     # class -> positions
    for p, v, c, w in steps:
        at[c].add(w)
    nq = q.size
    tail = nq // 32 * 32
    if name in ("cls1", "cls33"):
        runs = [a * planted.TILE_QUADS for a, b in planted.chee_runs(data.size)]
        firsts = {p for p, v, c, w in steps if w == "run_first"}
        assert set(runs[1:]) <= firsts                    # run 0 opens with bucket 0
        assert {p for p, v, c, w in steps if w == "stream_start"} == set(range(32))
        assert any(w == "split" and p % 32 == 16 and (p // 32 + 1) % 2 == 0 for p, v, c, w in steps)
        assert {p for p, v, c, w in steps if w == "tail"} == set(range(tail, nq)) and 0 < nq - tail < 32 and data.size % 4
        if name == "cls33":                               # every class at every position that can hold it
            for c in CLASSES:
                same_run = c.split(".")[1] in ("one", "two", "pred", "list5")
                want = set(SINGLE) | {"alt2", "halves"}
                if same_run:
                    want.discard("run_first")
                assert want <= at[c], (c, want - at[c])
        else:
            assert len(at) >= len(CLASSES)
    elif name == "cls_pure":
        assert {p for p, v, c, w in steps} == set(range(nq)) and 0 < nq - tail < 32 and data.size % 4
        assert {"pure", "alt2", "halves", "tail", "bucket0_later"} <= {w for *_, w in steps}
    else:
        assert {"after_copy", "bucket0_later"} <= {w for *_, w in steps}
        assert len(at) >= len(CLASSES) // 2


@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("name", sorted(cl_steps.CORPORA))
def test_plantings_get_their_flags_in_the_oracle_stream(alg, name):
    """Every planted quad has, in the oracle's stream, the flag the in-order restatement over the planted buckets gives it (a consistency
    check of the whole corpus), and the copy corpus puts collision quads right behind copy-mode episodes."""
    data, man, S = cl_steps.build(name)
    fl, copied = oracle_flags(alg, name)
    want = cl_steps.intended(alg, data, man, S, copied)
    got = fl[[p for p, *_ in man]]
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, [(man[i], int(got[i]), int(want[i])) for i in bad[:5]]
    step = np.array([e[4] == "step" for e in man])
    n = collections.Counter(got[step].tolist())
    assert n[COPY] < step.sum() // (3 if name == "cls_copy" else 8), n
    if alg == "cheetah":
        assert min(n[0], n[1], n[2], n[3]) > step.sum() // 200, n
    else:
        assert min(n[k] for k in range(8)) > 0, n
    if name == "cls_copy":                                # collision quads right behind a copied block, and Lion steps with one half copied
        bq = cl_steps.BS[alg] // 4
        behind = [e[0] for e, f in zip(man, got) if e[4] == "step" and f != COPY and e[0] % bq == 0 and copied[e[0] // bq - 1]]
        assert len(behind) >= 20, len(behind)
        if alg == "lion":
            half = [e[0] for e in man if e[4] == "step" and e[0] % 32 == 16 and copied[e[0] // 16 - 1] and not copied[e[0] // 16]]
            assert len(half) >= 5, len(half)


# (class, algorithm) -> flags its steps are planted for, beyond those of its pattern: the first accesses of the states
PURPOSES = {
    ("ab.pred", "cheetah"): {3}, ("ab.prev_pred", "cheetah"): {3},           # predicted from the run's table / through chee_fold_p
    ("abc.two", "cheetah"): {1, 2}, ("abc.prev_two", "cheetah"): {1, 2},     # MAP_A then MAP_B (prev_two: u1 and u2 of one step)
    ("abc.pred", "lion"): {1}, ("abc.prev_pred", "lion"): {1},
    ("undec5.list5", "lion"): {1, 4, cl_steps.MISS}, ("undec5.prev_list5", "lion"): {1, 4, cl_steps.MISS},
    ("undec_rep.prev_list5", "lion"): {2, 3, 4, 5}, ("undec5.prev_list5", "cheetah"): {3},
    ("bucket0", "cheetah"): {3, 0, 2}, ("bucket0", "lion"): {1, 0, 2},       # the stream start: pred 0, five zeros, (quad 0, quad 0)
}


@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("name", sorted(cl_steps.CORPORA))
def test_plantings_get_their_intended_flags(alg, name):
    """Every planting with an intent in the manifest gets it in the oracle's stream (steps that copy mode touches excepted), and every
    class still has checked intents, at every position in cls33, with the flags its state is planted for (PURPOSES)"""
    fl, copied = oracle_flags(alg, name)
    chk = cl_steps.checked_intents(alg, name, fl)
    bad = [(e[:5], g, w) for e, g, w in chk if not cl_steps.meets(g, w)]
    assert not bad, (len(bad), bad[:5])
    got = collections.defaultdict(set)
    for e, g, w in chk:
        got[e[2]].add(w)
    where = collections.defaultdict(set)
    for e, g, w in chk:
        where[e[2]].add(e[3])
    if name in ("cls1", "cls33"):
        need = [c for c in CLASSES if not (alg == "cheetah" and c.startswith("undec_rep"))]
        assert not [c for c in need if c not in got], [c for c in need if c not in got]
        for (c, a), flags in PURPOSES.items():
            if a == alg:
                assert flags <= got[c], (c, flags - got[c])
    if name == "cls33":
        for c in need:
            want = set(SINGLE) | {"alt2", "halves"}
            if c.split(".")[1] in ("one", "two", "pred", "list5"):
                want.discard("run_first")
            assert want <= where[c], (c, want - where[c])
    if name == "cls_pure" and alg == "cheetah":
        assert len([1 for e, g, w in chk if e[2] == "ab.pure_pred" and w == 3]) > 100
    assert len(chk) > 1000


@pytest.mark.parametrize("nruns", [1, 5, 64])
def test_run_prototypes_reproduce_the_oracle(nruns):
    """tools/proto_cheetah_runs.py and proto_lion_runs.py on cls1 and on a cut of cls_pure"""
    for name, cut in (("cls1", None), ("cls_pure", 96 << 10)):
        data = cl_steps.build(name)[0]
        if cut:
            data = data[:cut + 3].copy()
        for alg, proto in (("cheetah", proto_cheetah_runs), ("lion", proto_lion_runs)):
            got = proto.encode(data, nruns)[0]
            want = oracle.encode(alg, data)
            assert got.size == want.size and (got == want).all(), (alg, name, nruns)


MODEL_CASES = [("cls1", None), ("cls_pure", 256 << 10), ("cls_copy", 512 << 10)]


def _model_input(name, cut, alg):
    data = cl_steps.build(name)[0]
    if cut:
        data = data[:cut + 3].copy()
    fl, copied = cl_steps.stream_flags(alg, oracle.encode(alg, data), data.size)
    return data, fl, copied


@pytest.mark.parametrize("alg", ALGS)
@pytest.mark.parametrize("nruns", [1, 3, 8])
def test_step_model_reproduces_the_oracle(alg, nruns):
    """the lane-level model gives the oracle's flag for every quad, and the corpora reach the branches the collision steps are aimed at:
    the T 0 -> 1 -> 2 path and MAP_B inside one step, u1 and u2 of one step resolved by the fold, the stream start's (quad 0, quad 0)
    chunk map, and for Lion hits at every depth from in-step predecessors and from the fold, five undecided accesses in one step and
    misses while the local list is full"""
    cnt = collections.Counter()
    for name, cut in MODEL_CASES:
        data, fl, copied = _model_input(name, cut, alg)
        got = M.flags(alg, data, copied, nruns, counts=cnt)
        bad = np.flatnonzero(got != fl)
        assert bad.size == 0, (name, bad[:5].tolist(), got[bad[:5]].tolist(), fl[bad[:5]].tolist())
    need = ["c_map_b_in_step", "c_t0_t1_t2_in_step", "c_fold_u1_u2_one_step", "c_fold_bucket0_initial"]
    if alg == "cheetah":
        need += ["p_hit_in_warp", "p_hit_table", "p_miss_in_warp_multi_value"] + (["p_hit_fold", "c_fold_u2_map_b"] if nruns > 1 else [])
    else:
        need += [f"l_depth{k}_in_step" for k in range(5)] + ["l_undecided5_one_step", "l_miss_full", "half_step_copied"]
        need += [f"l_fold_depth{k}" for k in range(5)] + ["c_fold_u2_map_b"] if nruns > 1 else []
    assert all(cnt[k] > 0 for k in need), {k: cnt[k] for k in need}


@pytest.mark.parametrize("fault,alg,case", [("chee_c_first_lane_writes", "cheetah", 1), ("lion_undecided_cap4", "lion", 1),
                                            ("fold_c_invalid_bucket0", "cheetah", 0), ("chee_p_last_lane_u1", "cheetah", 1)])
def test_step_model_notices_each_fault(fault, alg, case):
    """each one-line change to the model's rules makes it differ from the oracle: on the cut of cls_pure, which has no text, except the
    initial chunk map of bucket 0, planted at cls1's stream start"""
    name, cut = MODEL_CASES[case]
    data, fl, copied = _model_input(name, cut, alg)
    got = M.flags(alg, data, copied, 3, faults=[fault])
    assert (got != fl).any(), f"{fault}: the model still matches the oracle on {name}"
