"""The run geometry of the run-parallel Cheetah decoder (density_b200/csrc/cl_decode.cu), the block walk of a Cheetah stream, and a corpus
planted at the decoder's run seams (numpy, the oracle and tests/cl_model.cpp).

The decoder cuts its runs in BLOCK space of the stream's main loop: run r starts at block r * main_blocks / nruns, with
nruns = max(1, min(stream bytes / 48 KiB, SMs * runs per SM)) (cd_pick_runs, run_step_begin). Every main-loop block, copy-mode or not,
decodes to 32 quads, so run r's first quad is quad 32 * its first block. These seams are not the encoder's 16 KiB tile seams
(tests/planted.py): they move with the stream, so cl_decode_corpus works them out from the oracle stream and plants again until they
stop moving.

The corpus plants, at the decoder's seams, the situations the cross-run code of the decoder exists for (one class per planting, cycled
over the seams); its manifest says, per planting, which quads must be predicted, encoded or copied in the stream, and
tests/test_cl_decode_seams_cpu.py checks that against the walk.
"""
import ctypes
import os
import subprocess

import numpy as np

import oracle
import planted
from planted import Planter, quad_of, twin

HERE = os.path.dirname(os.path.abspath(__file__))
RUN_STREAM_BYTES = 48 << 10        # cd_pick_runs: a run per 48 KiB of stream
MAX_ROUNDS = 40                    # cl_decode.cu MAX_ROUNDS
BS, SB = 128, 8                    # Cheetah block and signature bytes
K_PLAIN, K_MAP_A, K_MAP_B, K_PRED = 0, 1, 2, 3
COPY = 4                           # kind of every quad of a copy-mode block (walk())
CLASSES = ("pred_exit", "self_stretch", "snap_passthrough", "late_snapshot", "in_step_writers", "cmap_carried", "copy_at_seam")


# ---- the model ------------------------------------------------------------------------------------------------------------------
def build_model(dirpath):
    """tests/cl_model.cpp compiled into dirpath (a directory of this session's own: two sessions must not share one file)."""
    so = os.path.join(str(dirpath), "cl_model.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", os.path.join(HERE, "cl_model.cpp"), "-o", so])
    L = ctypes.CDLL(so)
    L.cl_model_decode_stats.restype = ctypes.c_size_t
    L.cl_model_decode_stats.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_uint32, ctypes.c_uint32,
                                        ctypes.POINTER(ctypes.c_uint32)]
    return L


def model_decode(L, enc, size, nruns, max_rounds=MAX_ROUNDS):
    """(decoded bytes, stats): stats = {rounds, settled, main_blocks, walks, queued, last_queued, nruns} (cl_model_decode_stats)."""
    out = np.zeros(size + 64, np.uint8)
    s = (ctypes.c_uint32 * 7)()
    n = L.cl_model_decode_stats(enc.ctypes.data, enc.size, out.ctypes.data, size, nruns, max_rounds, s)
    keys = ("rounds", "settled", "main_blocks", "walks", "queued", "last_queued", "nruns")
    return out[:n], dict(zip(keys, list(s)))


# ---- geometry and block walk ------------------------------------------------------------------------------------------------------
def pick_runs(stream_bytes, num_sms, per_sm=8):
    """cl_decode.cu cd_pick_runs."""
    return max(1, min(stream_bytes // RUN_STREAM_BYTES, num_sms * per_sm))


def cd_runs(stream_bytes, main_blocks, num_sms, per_sm=8):
    """The first main-loop block of every decoder run (cd_pick_runs, run_step_begin)."""
    nruns = pick_runs(stream_bytes, num_sms, per_sm)
    return [r * main_blocks // nruns for r in range(nruns)]


class Walk:
    """The main loop of a Cheetah stream (codec.rs:88-100: blocks while at least 136 stream bytes are left, with the protection
    automaton of protection_state.rs): per block its offset and copy mode, per quad its kind (K_* or COPY)."""

    def __init__(self, enc):
        buf = enc.tobytes()
        n = len(buf)
        M = 0x5555555555555555
        pen, start, prev, counter = 0, 1, 0, 0
        offs, copy, sigs = [], [], []
        idx = 0
        while n - idx >= SB + BS:
            if (counter & 15) == 0 and start > 1:        # revert_to_copy
                start >>= 1
            counter += 1
            if pen > 0:
                offs.append(idx); copy.append(True); sigs.append(0)
                idx += BS
                pen = (pen - 1) & 0xFF                      # decay
                if pen == 0:
                    start = (start + 1) & 0xFF
                continue
            sig = int.from_bytes(buf[idx:idx + SB], "little")
            lo, hi = sig & M, (sig >> 1) & M
            nplain = 32 - (lo | hi).bit_count()
            npred = (lo & hi).bit_count()
            sz = SB + 4 * nplain + 2 * (32 - nplain - npred)
            offs.append(idx); copy.append(False); sigs.append(sig)
            idx += sz
            if sz >= BS:                                    # update
                if prev:
                    pen = start
                prev = 1
            else:
                prev = 0
        self.main_blocks = len(offs)
        self.tail_off = idx
        self.offsets = np.array(offs, np.uint64)
        self.copy = np.array(copy, bool)
        s = np.array(sigs, np.uint64)
        self.kind = ((s[:, None] >> (2 * np.arange(32, dtype=np.uint64))[None, :]) & np.uint64(3)).astype(np.uint8).reshape(-1)
        self.kind.reshape(-1, 32)[self.copy] = COPY

    def kind_of(self, q):
        """Kind of quad q of the decoded main part (None past it)."""
        return int(self.kind[q]) if 0 <= q < self.kind.size else None


def seams(enc, num_sms, per_sm=8):
    w = Walk(enc)
    return w, cd_runs(enc.size, w.main_blocks, num_sms, per_sm)


# ---- the corpus -------------------------------------------------------------------------------------------------------------------
class _Seams:
    """Planter plus the manifest of the seam classes: per planting (class, seam, [(quad, expected kind)])."""

    def __init__(self, P, S):
        self.P, self.S, self.checks = P, S, []

    def fresh(self, fp=None):
        return quad_of(self.P.bucket(), self.P.fp() if fp is None else fp)

    def put(self, pos, v, cls):
        assert 0 <= pos < self.P.nq
        self.P.put(pos, v, cls)


def _pred_exit(Z, t, v):
    """Run t-1 ends in a predicted quad, so run t's entry context is unknown until a round has produced it. v even: run t's first
    quad is predicted (lane 0); v odd: its first predicted quad is lane 31 of its first step."""
    S = Z.S[t]
    a, b, c = Z.fresh(), Z.fresh(), Z.fresh()
    for j, x in enumerate((a, b, c)):                        # primes pred[h(a)] = b, pred[h(b)] = c inside run t-1
        Z.put(S - 300 + j, x, "pred_exit")
    Z.put(S - 2, a, "pred_exit"); Z.put(S - 1, b, "pred_exit")
    chk = [(S - 1, "P")]
    if v % 2 == 0:
        Z.put(S, c, "pred_exit")
        chk.append((S, "P"))
    else:
        h = Z.P.bucket()                                     # 31 distinct members of one bucket: none predicted, the last one again is
        us = [quad_of(h, Z.P.fp()) for _ in range(31)]
        for j, u in enumerate(us):
            Z.put(S + j, u, "pred_exit")
        Z.put(S + 31, us[-1], "pred_exit")
        chk += [(S + j, "N") for j in range(31)] + [(S + 31, "P")]
    return chk


STRETCH = [(L, o) for L in (2, 31, 32, 33, 95) for o in (-1, -16, -31, -32)]


def _self_stretch(Z, t, v):
    """L predicted copies of one quad (its hash maps its context onto itself) from seam + o on: the span logic of cd_pred_walk, up to
    p == 31, across a step boundary and the run boundary. The two copies in front of them write the prediction they read."""
    S = Z.S[t]
    L, o = STRETCH[v % len(STRETCH)]
    x = Z.fresh(0 if v % 3 == 0 else None)
    for j in range(-2, L):
        Z.put(S + o + j, x, "self_stretch")
    return [(S + o - 2, "N"), (S + o - 1, "N")] + [(S + o + j, "P") for j in range(L)]


def _snap_passthrough(Z, t, v):
    """Context h(y) is written only in run t-2; run t-1 never writes it; run t's first quad reads it as a predicted quad."""
    S0, S = Z.S[t - 1], Z.S[t]
    y, z = Z.fresh(), Z.fresh(0 if v % 2 else None)
    Z.put(S0 - 100, y, "snap_passthrough"); Z.put(S0 - 99, z, "snap_passthrough")
    Z.put(S - 1, y, "snap_passthrough"); Z.put(S, z, "snap_passthrough")
    return [(S0 - 100, "N"), (S0 - 99, "N"), (S - 1, "N"), (S, "P")]


def _late_snapshot(Z, t, D):
    """A chain of D runs: run t-D ends in a predicted quad; every link j = t-D+1 .. t-1 opens with a predicted quad p_j read at that exit
    context, then writes pred[h(p_j)] = w_j, a write the rounds make known only once run j's entry context is known; links other than
    the last end again in a predicted quad (w_j at context h(p_j)). Run t's entry context is known from the stream, and a predicted quad
    in its first step reads pred[h(p_{t-1})]: run t's snapshot there changes after run t has read it, so only its read set makes it
    dirty again (round 2 for D = 2, round 3 for D = 3)."""
    S = Z.S
    chk = []
    a, b, p = Z.fresh(), Z.fresh(), Z.fresh()
    e = S[t - D + 1]                                         # end of the base run t-D
    for j, x in enumerate((a, b, p)):                        # pred[h(a)] = b, pred[h(b)] = p
        Z.put(e - 300 + j, x, "late_snapshot")
    Z.put(e - 2, a, "late_snapshot"); Z.put(e - 1, b, "late_snapshot")
    chk += [(e - 1, "P")]
    for j in range(t - D + 1, t):
        w = Z.fresh()
        Z.put(S[j], p, "late_snapshot"); Z.put(S[j] + 1, w, "late_snapshot")
        chk += [(S[j], "P"), (S[j] + 1, "N")]
        if j < t - 1:
            nxt = Z.fresh()
            Z.put(S[j] + 2, nxt, "late_snapshot")            # pred[h(w)] = next link's first quad
            Z.put(S[j + 1] - 2, p, "late_snapshot"); Z.put(S[j + 1] - 1, w, "late_snapshot")
            chk += [(S[j] + 2, "N"), (S[j + 1] - 2, "N"), (S[j + 1] - 1, "P")]
            p = nxt
        else:
            f = Z.fresh()
            Z.put(S[t] - 1, f, "late_snapshot")               # run t's entry context is in the stream
            Z.put(S[t] + 5, p, "late_snapshot"); Z.put(S[t] + 6, w, "late_snapshot")
            chk += [(S[t] - 1, "N"), (S[t] + 5, "N"), (S[t] + 6, "P")]
    return chk


IN_STEP = ((2, 3, 6, 7, 10, 11), (20, 21, 24, 25, 30, 31), (0, 1, 4, 5, 8, 9))


def _in_step_writers(Z, t, v):
    """Two writers of context h(y), then a predicted reader of it, all in run t's first step (the ballot of the latest earlier
    writer), and a reader in the next step (the last writer's store)."""
    S = Z.S[t]
    y, u1, u2 = Z.fresh(), Z.fresh(), Z.fresh(0 if v % 2 else None)
    if v % 4 == 3:
        u2 = twin(u1)
    o = IN_STEP[v % len(IN_STEP)]
    for pos, x in zip(o, (y, u1, y, u2, y, u2)):
        Z.put(S + pos, x, "in_step_writers")
    Z.put(S + 40, y, "in_step_writers"); Z.put(S + 41, u2, "in_step_writers")
    return [(S + o[1], "N"), (S + o[3], "N"), (S + o[5], "P"), (S + 41, "P")]


def _cmap_carried(Z, t, v):
    """A bucket left at (A, B) in run t-1 (v odd: in run t-3, untouched since); run t opens with MAP_A, MAP_B, MAP_B, PLAIN, MAP_B:
    carried slots 0 and 1, two swaps, and a carried value read through the slot a push shifted it to."""
    S = Z.S[t]
    h = Z.P.bucket()
    c = v // 2
    A = quad_of(h, 0) if c % 3 == 0 else quad_of(h, Z.P.fp())
    B = twin(A) if c % 3 == 1 else quad_of(h, Z.P.fp())
    C = quad_of(h, 0) if c % 3 == 2 else twin(B) if c % 3 == 0 else quad_of(h, Z.P.fp())
    at = (Z.S[t - 2] if v % 2 else S) - 50
    Z.put(at, B, "cmap_carried"); Z.put(at + 1, A, "cmap_carried")
    for j, x in enumerate((A, B, A, C, A)):
        Z.put(S + j, x, "cmap_carried")
    return [(S, "A"), (S + 1, "B"), (S + 2, "B"), (S + 3, "L"), (S + 4, "B")]


def _prot_sim(b0, nblocks):
    """Copy mode of blocks b0 .. b0 + nblocks - 1 when they are all incompressible and the automaton enters them quiet (start 1)."""
    pen, start, prev, out = 0, 1, 0, []
    for b in range(b0, b0 + nblocks):
        if (b & 15) == 0 and start > 1:
            start >>= 1
        if pen > 0:
            out.append(True)
            pen -= 1
            if pen == 0:
                start += 1
            continue
        out.append(False)
        if prev:
            pen = start
        prev = 1
    return out


def _copy_at_seam(Z, t, v, rng):
    """An incompressible burst placed so that copy-mode blocks sit on both sides of the seam (cd_ctx_init walks back over them,
    cd_pred_walk skips them). Its quads are random members of buckets the text uses (the fresh ones stay fresh)."""
    s = Z.S[t] // 32
    for back in (5, 8, 9, 4, 6, 7, 10, 11, 12):
        b0 = s - back
        sim = _prot_sim(b0, back + 3)
        if sim[back - 1] and sim[back]:
            break
    else:
        raise RuntimeError("no burst start puts copy blocks on both sides of the seam")
    q0, q1 = 32 * b0, 32 * (s + 3)
    hs = rng.choice(Z.P.used, q1 - q0)
    vals = np.array([quad_of(int(h), int(f)) for h, f in zip(hs, rng.integers(1, 0xFFFE, q1 - q0))], np.uint32)
    Z.P.q[q0:q1] = vals
    for j in (32 * (s - 1), 32 * s):
        Z.P.manifest[j] = (int(Z.P.q[j]), "copy_at_seam")
    return [(32 * (s - 1), "C"), (32 * s + 31, "C")]


WIDTH = {"pred_exit": 1, "self_stretch": 2, "snap_passthrough": 2, "late_snapshot": None, "in_step_writers": 1, "cmap_carried": None,
         "copy_at_seam": 1}


def _plant(nbytes, seed, starts):
    P = Planter(nbytes, seed)
    P.used = np.flatnonzero(~np.isin(np.arange(65536), list(P.free_set)))
    rng = np.random.default_rng(seed + 77)
    Z = _Seams(P, [32 * b for b in starts])
    manifest = []
    k, i, ns = 1, 0, 0                                       # seam 0 is the stream start; ns: stretches planted so far
    while True:
        cls = CLASSES[i % len(CLASSES)]
        v = i // len(CLASSES)
        w = WIDTH[cls] or (2 + v % 2 if cls == "late_snapshot" else 1 + 2 * (v % 2))
        t = k + w - 1 if cls != "cmap_carried" else max(k + w - 1, 3)
        if t >= len(starts) or Z.S[t] + 200 >= P.nq:
            break
        if cls == "pred_exit":
            manifest.append((cls, t, "lane0" if v % 2 == 0 else "lane31", _pred_exit(Z, t, v)))
        elif cls == "self_stretch":                           # one stretch at each of its seams: every (length, start) in a 12 MiB corpus
            for u in (t - 1, t):
                manifest.append((cls, u, STRETCH[ns % len(STRETCH)], _self_stretch(Z, u, ns)))
                ns += 1
        elif cls == "snap_passthrough":
            manifest.append((cls, t, v % 2, _snap_passthrough(Z, t, v)))
        elif cls == "late_snapshot":
            manifest.append((cls, t, w, _late_snapshot(Z, t, w)))
        elif cls == "in_step_writers":
            manifest.append((cls, t, IN_STEP[v % len(IN_STEP)], _in_step_writers(Z, t, v)))
        elif cls == "cmap_carried":
            manifest.append((cls, t, 1 + 2 * (v % 2), _cmap_carried(Z, t, v)))
        else:
            manifest.append((cls, t, None, _copy_at_seam(Z, t, v, rng)))
        k, i = t + 1, i + 1
    return P.data, manifest


def cl_decode_corpus(nbytes, seed, num_sms=planted.H100_SMS, per_sm=8):
    """Dickens text planted at the seams of the run-parallel Cheetah decoder for `num_sms` SMs. Returns (bytes, oracle stream, manifest,
    first block of every run): manifest = [(class, seam index, variant, [(quad, expected kind: P predicted, N encoded and not predicted,
    A MAP_A, B MAP_B, L PLAIN, C copy mode)])]. Variants: pred_exit "lane0" / "lane31" (where run t's first predicted quad sits),
    self_stretch (length, start relative to the seam), late_snapshot the chain depth D, cmap_carried how many runs back the bucket was
    left, in_step_writers the lanes of the writers and readers. Planting moves the stream size a little, so the seams are worked out again from the new stream
    and the base planted again until they stop moving."""
    enc = oracle.encode("cheetah", planted.base_text(nbytes))
    _, starts = seams(enc, num_sms, per_sm)
    for _ in range(6):
        data, manifest = _plant(nbytes, seed, starts)
        enc = oracle.encode("cheetah", data)
        _, new = seams(enc, num_sms, per_sm)
        if new == starts:
            return data, enc, manifest, starts
        starts = new
    raise RuntimeError("the decoder's seams did not settle")


KIND_OK = {"P": lambda k: k == K_PRED, "N": lambda k: k is not None and k < K_PRED, "A": lambda k: k == K_MAP_A,
           "B": lambda k: k == K_MAP_B, "L": lambda k: k == K_PLAIN, "C": lambda k: k == COPY}


def confirmed(walk, chk):
    """The quads of one planting have the kinds the class needs in the stream."""
    return all(KIND_OK[e](walk.kind_of(q)) for q, e in chk)


# ---- the repeated-quad inputs of the round-budget edge ------------------------------------------------------------------------------
MIB = 1 << 20


def zeros(nruns_wanted):
    """Zeros whose Cheetah stream gives the decoder exactly nruns_wanted runs: every 128-byte block is 32 predicted quads, an 8-byte
    signature (16:1), so 768 KiB of zeros are 48 KiB of stream, one run."""
    return np.zeros(nruns_wanted * 16 * RUN_STREAM_BYTES + 5000, np.uint8)


def zero_hole():
    t = planted.base_text(6 * MIB)
    return np.concatenate([t[:3 * MIB], np.zeros(36 * MIB, np.uint8), t[3 * MIB:]])


def spaces():
    return np.full(36 * MIB, 0x20, np.uint8)
