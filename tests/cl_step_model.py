"""A lane-level restatement of the run-parallel Cheetah and Lion encoders' flag passes (density_b200/csrc/cheetah_encode.cu), in plain Python.

One 32-quad step of chee_pass_p, chee_pass_c<BPS> and lion_pass_p: the active lanes are grouped by key as __match_any_sync groups them
(contexts in the prediction passes, buckets in the chunk-map pass); inside a group the lanes go in rank order (the rank loop), the
group's first lane takes its state from the run's table entry as it stood at the start of the step and every other lane from its nearest
lower lane; the first lane owns the first-access slot (u1), the last lane writes the entry. Then chee_fold_p, chee_fold_c and lion_fold_p
walk the runs in order per context / bucket and resolve what each run left undecided against the state carried in, which starts as
pred = 0 everywhere, the chunk map (quad 0, quad 0) (FP_INVALID for every bucket but 0) and five zeros per Lion list.

`flags(alg, data, copied, nruns)` gives the flag of every quad (Cheetah 0-3, Lion 0-7, -1 in copy-mode blocks) for a given copy map.
`counts` tallies the branches the collision steps (tests/cl_steps.py) are aimed at. `faults` switches on one of FAULTS, a one-line change
to one rule, so that a test can show the comparison with the oracle notices it.
"""
import collections

import numpy as np

from planted import hf

TILE_BLOCKS = 128                                    # cheetah_encode.cu TILE_B: 128 steps of 32 quads per tile
FP_INVALID = 0x10000
FAULTS = ("chee_c_first_lane_writes", "lion_undecided_cap4", "fold_c_invalid_bucket0", "chee_p_last_lane_u1")


def run_steps(nbytes, nruns):
    """[s0, s1) in 32-quad steps of every run (run_block_begin, Cheetah and Lion alike)"""
    nsteps = (nbytes + 127) // 128
    ntiles = (nsteps + TILE_BLOCKS - 1) // TILE_BLOCKS
    b = [(r * ntiles // nruns) * TILE_BLOCKS for r in range(nruns + 1)]
    return [(b[r], min(b[r + 1], nsteps)) for r in range(nruns)]


def flags(alg, data, copied, nruns, faults=(), counts=None):
    faults = set(faults)
    assert faults <= set(FAULTS), faults
    cnt = collections.Counter() if counts is None else counts
    nq = data.size // 4
    q = data[:nq * 4].view(np.uint32)
    h, f = hf(q)
    ql, hl, fl = q.tolist(), h.tolist(), f.tolist()
    bpq = 32 if alg == "cheetah" else 16                 # quads per block
    bps = 32 // bpq                                      # blocks per step
    cp = np.asarray(copied, bool).tolist()
    nsteps = (data.size + 127) // 128
    act = []                                             # active lanes of every step (step_active_lanes, and the quads that exist)
    for s in range(nsteps):
        n = max(0, min(32, nq - 32 * s))
        m = [l < n for l in range(32)]
        for k in range(bps):
            b = bps * s + k
            if b >= len(cp) or cp[b]:
                m[k * bpq:(k + 1) * bpq] = [False] * bpq
                if any(m):
                    cnt["half_step_copied"] += 1
        act.append(m)
    runs = run_steps(data.size, nruns)
    P = [0] * nq                                         # Cheetah: 1 predicted; Lion: depth + 1
    if alg == "cheetah":
        ents = [_chee_pass_p(ql, hl, act, s0, s1, _ctx0(hl, cp, bpq, s0 * bps, nq), P, faults, cnt) for s0, s1 in runs]
        _chee_fold_p(ql, ents, P, cnt)
    else:
        ents = [_lion_pass_p(ql, hl, act, s0, s1, _ctx0(hl, cp, bpq, s0 * bps, nq), P, faults, cnt) for s0, s1 in runs]
        _lion_fold_p(ql, ents, P, cnt)
    code = [0] * nq                                      # 1 MAP_A, 2 MAP_B
    entc = [_chee_pass_c(fl, hl, act, P, s0, s1, code, faults, cnt) for s0, s1 in runs]
    _chee_fold_c(fl, entc, code, faults, cnt)
    out = np.full(nq, -1, np.int8)
    for s, m in enumerate(act):
        for l in range(32):
            if m[l]:
                i = 32 * s + l
                if alg == "cheetah":
                    out[i] = 3 if P[i] else code[i]
                else:
                    out[i] = P[i] if P[i] else (5 + code[i] if code[i] else 0)
    return out


def _ctx0(hl, cp, bpq, b, nq):
    """chee_ctx0 / lion_ctx0: the hash of the last quad of the last encoded block before the run, 0 if there is none"""
    while b > 0:
        b -= 1
        if cp[b]:
            continue
        i = b * bpq + bpq - 1
        return hl[i] if i < nq else 0
    return 0


def _groups(keys, m):
    """__match_any_sync over the active lanes: key -> its lanes in lane order"""
    g = {}
    for l in range(32):
        if m[l]:
            g.setdefault(keys[l], []).append(l)
    return g


def _contexts(hl, m, q0, last_h):
    """the context of every active lane (the hash of the nearest active lane below it, else what the run carries) and the new carry"""
    ctx, c = [0] * 32, last_h
    for l in range(32):
        if m[l]:
            ctx[l] = c
            c = hl[q0 + l]
    return ctx, c


# ---- Cheetah predictions ------------------------------------------------------------------------------------------------------------
def _chee_pass_p(ql, hl, act, s0, s1, last_h, P, faults, cnt):
    ent = {}                                             # ctx -> (last quad, u1)
    for s in range(s0, s1):
        m = act[s]
        if not any(m):
            continue
        q0 = 32 * s
        ctx, last_h = _contexts(hl, m, q0, last_h)
        for c, lanes in _groups(ctx, m).items():
            e = ent.get(c)
            first = lanes[0]
            if e is not None and e[0] == ql[q0 + first]:
                P[q0 + first] = 1
                cnt["p_hit_table"] += 1
            for a, b in zip(lanes, lanes[1:]):          # every other lane: its nearest lower lane of the group
                if ql[q0 + a] == ql[q0 + b]:
                    P[q0 + b] = 1
                    cnt["p_hit_in_warp"] += 1
                elif len({ql[q0 + x] for x in lanes}) > 1:
                    cnt["p_miss_in_warp_multi_value"] += 1
            owner = lanes[-1] if "chee_p_last_lane_u1" in faults else first
            u1 = e[1] if e is not None else q0 + owner  # the first lane owns the first-access slot
            ent[c] = (ql[q0 + lanes[-1]], u1)           # the last lane leaves its quad
    return ent


def _chee_fold_p(ql, ents, P, cnt):
    keys = sorted(set().union(*ents))
    for c in keys:
        carry = 0                                        # cheetah.rs:53
        for ent in ents:
            e = ent.get(c)
            if e is None:
                continue
            i = e[1]
            if ql[i] == carry:
                P[i] = 1
                cnt["p_hit_fold" if carry else "p_hit_fold_zero"] += 1
            carry = e[0]


# ---- Lion predictions -----------------------------------------------------------------------------------------------------------------
def _lion_pass_p(ql, hl, act, s0, s1, last_h, P, faults, cnt):
    ent = {}                                             # ctx -> [local list, m, cold slots (quad indices of the undecided accesses)]
    cap = 4 if "lion_undecided_cap4" in faults else 5
    for s in range(s0, s1):
        m = act[s]
        if not any(m):
            continue
        q0 = 32 * s
        ctx, last_h = _contexts(hl, m, q0, last_h)
        for c, lanes in _groups(ctx, m).items():
            e = ent.get(c)
            if e is None:
                e = ent[c] = [[0, 0, 0, 0, 0], 0, [0] * 5]
            lst, mm, cold = e
            und = 0
            for rank, l in enumerate(lanes):
                v = ql[q0 + l]
                k = next((j for j in range(mm) if lst[j] == v), 5)   # first local depth holding v
                if k < 5:
                    P[q0 + l] = k + 1
                    if rank > 0:
                        cnt[f"l_depth{k}_in_step"] += 1
                    lst = [v] + lst[:k] + lst[k + 1:]
                else:
                    if mm < cap:                         # undecided: depends on the carried-in list
                        cold[mm] = q0 + l
                        mm += 1
                        und += 1
                    elif mm == 5:
                        cnt["l_miss_full"] += 1
                    lst = [v] + lst[:4]
            if und == 5:
                cnt["l_undecided5_one_step"] += 1
            e[0], e[1] = lst, mm
    return ent


def _lion_fold_p(ql, ents, P, cnt):
    keys = sorted(set().union(*ents))
    for c in keys:
        car = [0, 0, 0, 0, 0]                            # lion.rs:64-72
        for ent in ents:
            e = ent.get(c)
            if e is None:
                continue
            lst, mf, cold = e
            for k in range(mf):
                v = ql[cold[k]]
                vis = car[:5 - k]
                if v in vis:
                    j = vis.index(v)
                    P[cold[k]] = k + j + 1
                    cnt[f"l_fold_depth{k + j}"] += 1
                    del car[j]
                    car.append(0)                       # keeps the list five long; the tail is never visible again
            car = (lst[:mf] + car)[:5]


# ---- chunk map (both algorithms) ----------------------------------------------------------------------------------------------------------
def _chee_pass_c(fl, hl, act, P, s0, s1, code, faults, cnt):
    ent = {}                                             # bucket -> (a, b, T, u1, u2)
    first_writes = "chee_c_first_lane_writes" in faults
    for s in range(s0, s1):
        m0 = act[s]
        q0 = 32 * s
        m = [m0[l] and not P[q0 + l] for l in range(32)]
        if not any(m):
            continue
        keys = [hl[q0 + l] if m[l] else 0 for l in range(32)]
        for hb, lanes in _groups(keys, m).items():
            a, b, T, u1, u2 = ent.get(hb, (0, 0, 0, -1, -1))
            T0 = T
            states = []
            for l in lanes:
                i, v = q0 + l, fl[q0 + l]
                if T == 0:                               # first touch in the run: decided by the fold
                    u1, a, b, T = i, v, 0, 1
                elif T == 1:
                    if v == a:
                        code[i] = 1
                    else:                                # MAP_B iff v == the (unknown) carried b: decided by the fold
                        u2, b, a, T = i, a, v, 2
                else:
                    if v == a:
                        code[i] = 1
                    else:
                        if v == b:
                            code[i] = 2
                            if l != lanes[0]:
                                cnt["c_map_b_in_step"] += 1
                        b, a = a, v
                states.append((a, b, T, u1, u2))
            if T0 == 0 and T == 2 and u1 // 32 == u2 // 32 == s and len(set(fl[q0 + l] for l in lanes)) >= 3:
                cnt["c_t0_t1_t2_in_step"] += 1
            ent[hb] = states[0] if first_writes else states[-1]
    return ent


def _chee_fold_c(fl, ents, code, faults, cnt):
    keys = sorted(set().union(*ents))
    bad0 = "fold_c_invalid_bucket0" in faults
    for hb in keys:
        a0 = FP_INVALID if (hb or bad0) else 0           # the chunk map starts as (quad 0, quad 0): only bucket 0 holds it
        b0 = a0
        for ent in ents:
            e = ent.get(hb)
            if e is None:
                continue
            a, b, T, i1, i2 = e
            v1 = fl[i1]
            if v1 == a0:
                code[i1] = 1
                bafter = b0
            else:
                if v1 == b0:
                    code[i1] = 2
                bafter = a0
            if hb == 0 and a0 == 0 and b0 == 0:
                cnt["c_fold_bucket0_initial"] += 1
            if T == 2:
                if fl[i2] == bafter:
                    code[i2] = 2
                    cnt["c_fold_u2_map_b"] += 1
                if i1 // 32 == i2 // 32:
                    cnt["c_fold_u1_u2_one_step"] += 1
                a0, b0 = a, b
            elif v1 != a0:
                a0, b0 = v1, a0
