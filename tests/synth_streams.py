"""Chameleon and Cheetah streams that no encoder writes, laid out block by block (numpy only), and a plain in-order decoder.

An encoder only ever names dictionary states it has just verified: a Chameleon MAP names a bucket that holds its quad, a Cheetah MAP_B
reads a slot 1 that holds the quad, a PREDICTED quad reads a context whose prediction is the quad. The decoders accept any well-formed
stream, so these generators write the others too: MAPs at buckets that were never written (they decode to 0), at buckets written only
by their fingerprint-0 member, PLAIN quads that rewrite the value their bucket holds, twins written back to back, pile-ups of one bucket
in one tile, MAP_B swaps of empty slots, predicted reads of contexts never written, self-mapping predicted chains, and every tail the
main loop's exit rule leaves (codec.rs:88-123).

`build(alg, plan, seed)` returns `(stream, manifest)`. Random content never touches a reserved pool of buckets (and bucket 0 and
planted.FP0_HASHES), so the state a planted quad meets is the one the generator chose. Classes go on the first and last quads of tiles,
warp regions and decoder runs (the geometry mirrors below), of the pieces a plan names, and on the block after a copy-mode episode.
The manifest records the main loop's block starts, copy-mode blocks, tail offset and automaton state, and per planting
(class, block, quad index, expected decoded value); tests/test_synth_streams_cpu.py checks that every class is still where it says.

`decode_reference` restates codec.rs:82-126, protection_state.rs, chameleon.rs:55-68,103-135 and cheetah.rs:67-103,152-185 in plain
Python: an independent witness for the oracle on streams it was never pinned on.
"""
import collections

import numpy as np

import planted
import protection as P
from planted import FP0_HASHES, quad_of, twin

ALGS = ("chameleon", "cheetah", "lion")
BS = {"chameleon": 256, "cheetah": 128, "lion": 64}
SIG = {"chameleon": 8, "cheetah": 8, "lion": 6}     # signature bytes (lion.rs:325)
QPB = {"chameleon": 64, "cheetah": 32, "lion": 16}  # quads per block
FB = {"chameleon": 1, "cheetah": 2, "lion": 3}      # flag bits
PLAIN, MAP, MAP_A, MAP_B, PRED = 0, 1, 1, 2, 3      # Chameleon: 0 PLAIN, 1 MAP; Cheetah: 0 PLAIN, 1 MAP_A, 2 MAP_B, 3 PREDICTED
NBYTES = {0: 4, 1: 2, 2: 2, 3: 0}
L_PA, L_PB, L_PC, L_PD, L_PE, L_MAP_A, L_MAP_B = 1, 2, 3, 4, 5, 6, 7   # Lion (lion.rs:18-27): 0 PLAIN, 1-5 PREDICTED_A..E, 6 MAP_A, 7 MAP_B
PAYLOAD = {"chameleon": (4, 2, 2, 0), "cheetah": (4, 2, 2, 0), "lion": (4, 0, 0, 0, 0, 0, 2, 2)}   # payload bytes per flag
M32 = 0xFFFFFFFF
TILE_BLOCKS = 64                                    # chameleon_decode.cu: a tile is 4096 quads = 64 blocks
MIN_BLOCK = {"chameleon": 136, "cheetah": 8}        # decode_bounds.cuh bounds_layout: smallest encoded block
D7_MB_CAP, D7_SEC_CAP = 4, 16                       # chameleon_decode.cu: mailbox slot and overflow capacity
FIXED_UNWRITTEN = tuple(FP0_HASHES) + (0xFFFF,)     # never written in any stream here (0xFFFF is in FP0_HASHES too)


def hash16(q):
    a = np.asarray(q, dtype=np.uint64)
    h = ((a * np.uint64(planted.M)) & np.uint64(M32)) >> np.uint64(16)
    return int(h) if np.ndim(q) == 0 else h.astype(np.int64)


# ---- geometry mirrors ---------------------------------------------------------------------------------------------------------
def cham_dec_runs(stream_bytes, cap, main_blocks, num_sms=planted.H100_SMS):
    """Tile ranges [t0, t1) of the Chameleon decoder's runs: dec_pick_runs on bounds_layout's maxblocks (an upper bound of the block
    count from the stream size and the capacity), the tiles of the real block count split evenly (cham_decode_pass7)."""
    maxblocks = min(stream_bytes // MIN_BLOCK["chameleon"] + 2, cap // BS["chameleon"] + 2)
    nruns = min(max(((maxblocks + 63) // 64) // 16, 1), num_sms)
    ntiles = (main_blocks + TILE_BLOCKS - 1) // TILE_BLOCKS
    return [(r * ntiles // nruns, (r + 1) * ntiles // nruns) for r in range(nruns)]


def cheetah_dec_runs(stream_bytes, main_blocks, num_sms=planted.H100_SMS):
    """First main-loop block of every run of the Cheetah decoder (tests/cl_decode_seams.py: cd_pick_runs, run_step_begin)."""
    import cl_decode_seams as cds
    return cds.cd_runs(stream_bytes, main_blocks, num_sms)


def lion_dec_runs(stream_bytes, main_blocks, num_sms=planted.H100_SMS):
    """First main-loop block of every run of the Lion decoder's chunk-map passes: run r starts at row r * nrows // nruns of the rows of
    two blocks (cd_pick_runs, run_step_begin on cd_steps<LionT>)"""
    import cl_decode_seams as cds
    nruns, nrows = cds.pick_runs(stream_bytes, num_sms), (main_blocks + 1) // 2
    return [2 * (r * nrows // nruns) for r in range(nruns)]


def seam_blocks(alg, stream_bytes, cap, main_blocks, num_sms=planted.H100_SMS):
    """First block of every decoder run after the first."""
    if alg == "lion":
        return sorted(set(lion_dec_runs(stream_bytes, main_blocks, num_sms)[1:]))
    if alg == "chameleon":
        return sorted({t0 * TILE_BLOCKS for t0, _ in cham_dec_runs(stream_bytes, cap, main_blocks, num_sms)[1:]})
    return sorted(set(cheetah_dec_runs(stream_bytes, main_blocks, num_sms)[1:]))


# ---- the plain in-order decoder -------------------------------------------------------------------------------------------------
def decode_reference(alg, stream, cap, state=None, prot=None):
    """codec.rs:82-126 with chameleon.rs / cheetah.rs / lion.rs, quad by quad. Returns the decoded bytes (empty on a malformed stream or when
    the output would pass `cap`, as the C ABI maps both to 0). `state` (a dict, optional) is the codec instance's dictionary carried
    in and updated, as `Codec::decode` on a reused instance (codec.rs:16,82). `prot` (penalty, start, previous_incompressible,
    counter): the automaton to start from instead of protection_state.rs:9-16 (to decode the tail behind a known main loop)."""
    s = bytes(stream)
    n, idx = len(s), 0
    bs, qpb, fb, sb = BS[alg], QPB[alg], FB[alg], SIG[alg]
    st = state if state is not None else {}
    cm = st.setdefault("a", [0] * 65536)
    cb = st.setdefault("b", [0] * 65536) if alg != "chameleon" else None
    pred = st.setdefault("pred", [0] * 65536) if alg == "cheetah" else None
    lists = st.setdefault("lists", {}) if alg == "lion" else None       # context -> [next_a .. next_e] (lion.rs:41-48), absent: zeros
    out = bytearray()
    ps = _Prot(*prot) if prot is not None else _Prot()

    class Bad(Exception):
        pass

    def rd(k):
        nonlocal idx
        if n - idx < k:
            raise Bad
        v = int.from_bytes(s[idx:idx + k], "little")
        idx += k
        return v

    def one(flag):
        """one quad (decode_plain / decode_map*; decode_predicted)"""
        if alg == "chameleon":
            if flag == PLAIN:
                q = rd(4)
                cm[hash16(q)] = q
                return q
            return cm[rd(2)]
        if alg == "lion":
            return lion(flag)
        if flag == PLAIN:
            q = rd(4); h = hash16(q)
            cb[h] = cm[h]; cm[h] = q
        elif flag == MAP_A:
            h = rd(2); q = cm[h]
        elif flag == MAP_B:
            h = rd(2); q = cb[h]
            cb[h] = cm[h]; cm[h] = q
        else:
            q = pred[st.get("last", 0)]
            st["last"] = hash16(q)
            return q
        pred[st.get("last", 0)] = q
        st["last"] = h
        return q

    def lion(flag):
        """lion.rs:84-186 and :286: the list of the context last_hash, then last_hash = the quad's hash (explicit for MAP_A / MAP_B)"""
        last = st.get("last", 0)
        L = lists.get(last, [0] * 5)
        if flag == PLAIN:
            q = rd(4); h = hash16(q)
            cb[h] = cm[h]; cm[h] = q
            L = [q] + L[:4]                                         # shift_predictions
        elif flag == L_MAP_A:
            h = rd(2); q = cm[h]
            L = [q] + L[:4]
        elif flag == L_MAP_B:
            h = rd(2); q = cb[h]
            cb[h] = cm[h]; cm[h] = q
            L = [q] + L[:4]
        else:                                                       # PREDICTED_A..E: slot k to the front
            k = flag - 1
            q = L[k]; h = hash16(q)
            L = [q] + L[:k] + L[k + 1:]
        lists[last] = L
        st["last"] = h
        return q

    def block(tail):
        """one encoded block; True when the stream ended inside it (decode_partial_unit)"""
        sig = rd(sb)
        unit = 8 if alg == "chameleon" else 4
        for _ in range(qpb * 4 // unit):
            full = not tail or n - idx >= unit
            for _ in range(unit // 4):
                f = sig & ((1 << fb) - 1)
                sig >>= fb
                if not full and f == PLAIN:
                    r = n - idx
                    if r < 4:
                        out.extend(s[idx:])
                        return True
                out.extend(one(f).to_bytes(4, "little"))
        return False

    try:
        while n - idx >= sb + bs:
            mark = idx
            if ps.step_copy():
                out.extend(s[idx:idx + bs]); idx += bs
                continue
            block(False)
            ps.step_update(idx - mark >= bs)
        while n - idx > 0:
            mark = idx
            if ps.step_copy():
                if n - idx > bs:
                    out.extend(s[idx:idx + bs]); idx += bs
                    continue
                out.extend(s[idx:]); idx = n
                break
            if block(True):
                break
            ps.step_update(idx - mark >= bs)
    except Bad:
        return b""
    if len(out) > cap:
        return b""
    return bytes(out)


class _Prot(P.Protection):
    """protection_state.rs split as codec.rs calls it: revert_to_copy (+ decay when copying), then update after an encoded block."""

    def step_copy(self):
        if (self.counter & 15) == 0 and self.start > 1:
            self.start >>= 1
        self.counter += 1
        if self.penalty > 0:
            self.penalty -= 1
            if self.penalty == 0:
                self.start += 1
            return True
        return False

    def step_update(self, inc):
        if inc:
            if self.prev:
                self.penalty = self.start
            self.prev = 1
        else:
            self.prev = 0


# ---- reading a stream's main loop back --------------------------------------------------------------------------------------------
def walk(alg, stream):
    """The main loop of `stream` (codec.rs:88-100): block starts, copy-mode blocks, tail offset and the automaton state behind it, and
    the automaton state in front of every block (penalty, start, previous_incompressible, counter % 16)."""
    s = np.asarray(stream, np.uint8)
    n, bs, fb, sb = s.size, BS[alg], FB[alg], SIG[alg]
    size_of = {f: NBYTES[f] if alg == "cheetah" else (4 if f == 0 else 2) for f in range(4)}
    if alg == "lion":                                                # payload bytes of 4 flags (12 signature bits) at once
        f4 = (np.arange(4096)[:, None] >> (3 * np.arange(4))[None, :]) & 7
        by12 = np.array(PAYLOAD["lion"])[f4].sum(axis=1).tolist()
        buf = s.tobytes()
    ps = _Prot()
    starts, copy, before = [], [], []
    idx = 0
    while n - idx >= sb + bs:
        before.append((ps.penalty, ps.start, ps.prev, ps.counter & 15))
        starts.append(idx)
        if ps.step_copy():
            copy.append(True)
            idx += bs
            continue
        if alg == "lion":
            sig = int.from_bytes(buf[idx:idx + sb], "little")
            sz = sb + by12[sig & 4095] + by12[(sig >> 12) & 4095] + by12[(sig >> 24) & 4095] + by12[sig >> 36]
        else:
            sig = int.from_bytes(s[idx:idx + sb].tobytes(), "little")
            sz = sb + sum(size_of[(sig >> (fb * k)) & ((1 << fb) - 1)] for k in range(QPB[alg]))
        copy.append(False)
        idx += sz
        ps.step_update(sz >= bs)
    return {"starts": starts, "copy": copy, "main_blocks": len(starts), "tail_off": idx, "before": before,
            "state": (ps.penalty, ps.start, ps.prev, ps.counter)}


# ---- the generator ----------------------------------------------------------------------------------------------------------------
class _Gen:
    def __init__(self, alg, nblocks, seed, plan):
        self.alg, self.nb, self.plan = alg, nblocks, plan
        self.q = QPB[alg]
        self.rng = np.random.default_rng(seed)
        rng = self.rng
        perm = rng.permutation(np.arange(1, 65536))
        self.pool = [int(h) for h in perm[~np.isin(perm, FIXED_UNWRITTEN)][:12000]]                                      # reserved: fresh buckets for the plantings
        self.reserved = np.zeros(65536, bool)
        self.reserved[self.pool] = True
        self.reserved[list(FIXED_UNWRITTEN) + [0]] = True
        self.free_h = np.flatnonzero(~self.reserved)
        self.planted = {}                                             # flat quad -> (flag, value)
        self.manifest = []                                            # (class, block, quad, expected value or None)
        self.forced_inc = {}                                          # block -> bool
        self._random_content()

    def fresh(self):
        return self.pool.pop()

    def fp(self):
        return int(self.rng.integers(1, 0xFFFE))

    def _random_quads(self, k):
        """k random quads whose hashes random content may use"""
        v = self.rng.integers(1, 1 << 32, k, dtype=np.uint64)
        while True:
            bad = self.reserved[hash16(v)]
            if not bad.any():
                return v.astype(np.uint32)
            v[bad] = self.rng.integers(1, 1 << 32, int(bad.sum()), dtype=np.uint64)

    def _random_content(self):
        rng, nb, q, alg = self.rng, self.nb, self.q, self.alg
        p = self.plan
        if alg == "chameleon":
            # every PLAIN count from 0 to 59 (block sizes 136 .. 254; 60 and more are incompressible, codec.rs:98)
            k = rng.integers(p.get("min_plain", 0), p.get("max_plain", 59) + 1, nb)
            rank = np.argsort(rng.random((nb, q)), axis=1).argsort(axis=1)
            F = np.where(rank < k[:, None], PLAIN, MAP).astype(np.int8)
        elif alg == "lion":
            pp = p.get("p_pred", 0.5)
            u = rng.random((nb, q))
            plain_share = rng.random(nb)[:, None] * 0.6
            depth = rng.integers(L_PA, L_PE + 1, (nb, q))
            F = np.where(u < pp, depth, np.where(rng.random((nb, q)) < plain_share, PLAIN,
                                                 np.where(rng.random((nb, q)) < 0.5, L_MAP_A, L_MAP_B))).astype(np.int8)
        else:
            pp = p.get("p_pred", 0.5)
            u = rng.random((nb, q))
            plain_share = rng.random(nb)[:, None] * 0.6              # block sizes from 8 to about 100 bytes at every density
            F = np.where(u < pp, PRED, np.where(rng.random((nb, q)) < plain_share, PLAIN,
                                                np.where(rng.random((nb, q)) < 0.5, MAP_A, MAP_B))).astype(np.int8)
        V = np.zeros((nb, q), np.uint32)
        flat_f, flat_v = F.reshape(-1), V.reshape(-1)
        pl = np.flatnonzero(flat_f == PLAIN)
        flat_v[pl] = self._random_quads(pl.size)
        mp = np.flatnonzero((flat_f == MAP) | (flat_f == MAP_B)) if alg == "cheetah" else \
            np.flatnonzero(flat_f >= L_MAP_A) if alg == "lion" else np.flatnonzero(flat_f == MAP)
        # a MAP names, with probability 0.6, the bucket of one of the last 64 PLAIN quads (in-tile readers of a written bucket), otherwise
        # any bucket random content may use
        k = np.searchsorted(pl, mp) - rng.integers(1, 65, mp.size)
        recent = (k >= 0) & (rng.random(mp.size) < 0.6)
        h = self.free_h[rng.integers(0, self.free_h.size, mp.size)]
        h[recent] = hash16(flat_v[pl[k[recent]]])
        flat_v[mp] = h.astype(np.uint32)
        self.F, self.V = F, V

    # plantings: flag and payload (PLAIN: the quad, MAP*: the hash) at a flat quad index
    def put(self, qi, flag, value):
        if 0 <= qi < self.nb * self.q:
            self.planted[qi] = (flag, int(value) & M32)

    def note(self, cls, qi, expect=None):
        if 0 <= qi < self.nb * self.q:
            self.manifest.append((cls, qi // self.q, qi, expect))

    def apply(self):
        F, V = self.F.copy(), self.V.copy()
        f, v = F.reshape(-1), V.reshape(-1)
        for qi, (fl, val) in self.planted.items():
            f[qi], v[qi] = fl, val
        return F, V

    def sizes(self, F):
        nbytes = np.array(PAYLOAD[self.alg], np.int64)
        return SIG[self.alg] + nbytes[F.astype(np.int64)].sum(axis=1)

    def force(self, F, b, inc):
        """make block b incompressible (all PLAIN) or not (all MAP / MAP_A), planted quads kept"""
        row = F[b]
        keep = np.array([(b * self.q + k) in self.planted for k in range(self.q)])
        if inc:
            row[~keep] = PLAIN
        else:
            row[~keep & (row == PLAIN)] = L_MAP_A if self.alg == "lion" else MAP

    def layout(self, tail_spec):
        """-> (stream bytes, copy flags per block, block offsets, automaton after the last block)"""
        F, V = self.apply()
        alg, nb, q, bs = self.alg, self.nb, self.q, BS[self.alg]
        for b, inc in self.forced_inc.items():
            self.force(F, b, inc)
        # forced blocks: new values for the quads that are not planted
        fl, vl = F.reshape(-1), V.reshape(-1)
        for b, inc in self.forced_inc.items():
            if inc:
                fresh = [i for i in range(b * q, (b + 1) * q) if i not in self.planted]
                vl[fresh] = self._random_quads(len(fresh))
            else:
                idx = [i for i in range(b * q, (b + 1) * q) if i not in self.planted]
                if alg != "chameleon":
                    fl[idx] = L_MAP_A if alg == "lion" else MAP_A
                vl[idx] = self.free_h[self.rng.integers(0, self.free_h.size, len(idx))].astype(np.uint32)
        sz = self.sizes(F)
        if alg == "lion":
            self._lion_blocks(F, V, sz, tail_spec)
        if self.plan.get("quiet", True):
            inc = sz >= bs
            for b in np.flatnonzero(inc[1:] & inc[:-1]) + 1:          # no two incompressible blocks in a row: no copy mode
                if inc[b - 1] and inc[b] and b not in self.forced_inc:
                    row = F[b]
                    cand = [k for k in range(q) if row[k] == PLAIN and (b * q + k) not in self.planted]
                    while sz[b] >= bs and cand:
                        k = cand.pop()
                        row[k] = L_MAP_A if alg == "lion" else MAP_A
                        V[b, k] = self.free_h[0]
                        sz[b] -= 2
                    inc[b] = sz[b] >= bs
        ps = _Prot()
        copy = np.zeros(nb, bool)
        for b in range(nb):
            if ps.step_copy():
                copy[b] = True
                sz[b] = bs
                continue
            ps.step_update(sz[b] >= bs)
        off = np.zeros(nb + 1, np.int64)
        np.cumsum(sz, out=off[1:])
        body = np.zeros(int(off[-1]), np.uint8)
        # signatures
        enc = ~copy
        fb, sb = FB[alg], SIG[alg]
        sig = np.zeros(nb, np.uint64)
        for k in range(q):
            sig |= F[:, k].astype(np.uint64) << np.uint64(fb * k)
        so = off[:-1][enc]
        for i in range(sb):
            body[so + i] = ((sig[enc] >> np.uint64(8 * i)) & np.uint64(0xFF)).astype(np.uint8)
        # payloads
        nbytes = np.array(PAYLOAD[alg], np.int64)[F.astype(np.int64)]
        nbytes[copy] = 0
        qoff = off[:-1, None] + sb + np.cumsum(nbytes, axis=1) - nbytes
        for width in (4, 2):
            m = nbytes == width
            o, val = qoff[m], V[m].astype(np.uint64)
            for i in range(width):
                body[o + i] = ((val >> np.uint64(8 * i)) & np.uint64(0xFF)).astype(np.uint8)
        # copy-mode blocks: raw bytes
        cb = np.flatnonzero(copy)
        if cb.size:
            raw = self.rng.integers(0, 256, (cb.size, bs), dtype=np.uint8)
            body[(off[cb][:, None] + np.arange(bs)).reshape(-1)] = raw.reshape(-1)
        self.F_final, self.V_final, self.copy = F, V, copy
        tail, tcls = self._tail_lion(tail_spec, ps) if alg == "lion" else self._tail(tail_spec, ps)
        return np.concatenate([body, tail]), copy, off, tcls

    def _lion_blocks(self, F, V, sz, tail_spec):
        """Lion: no block outside forced_inc is incompressible, so copy mode sits only where the plan forces it and plantings cannot move
        it; the last block is long enough that, with a tail of 6 .. 69 bytes behind it, it stays in the main loop (codec.rs:88), so the
        last main-loop quad is the last generated one"""
        q, nb = self.q, self.nb
        for b in np.flatnonzero(sz >= BS["lion"]):
            if b in self.forced_inc:
                continue
            for k in range(q):
                if sz[b] < BS["lion"]:
                    break
                if F[b, k] == PLAIN and (b * q + k) not in self.planted:
                    F[b, k] = L_MAP_A; V[b, k] = self.free_h[0]; sz[b] -= 2
        L = tail_spec[0]
        b = nb - 1
        if SIG["lion"] <= L < SIG["lion"] + BS["lion"] and b not in self.forced_inc:
            for k in range(q):
                if sz[b] >= SIG["lion"] + BS["lion"] - L:
                    break
                if F[b, k] != PLAIN and (b * q + k) not in self.planted:
                    sz[b] += 4 - PAYLOAD["lion"][F[b, k]]
                    F[b, k] = PLAIN; V[b, k] = self._random_quads(1)[0]

    def _tail_lion(self, spec, ps):
        """_tail for Lion: one block of 16 quads whose first quad is PREDICTED_A where it fits (it reads the list of the main loop's last
        context), then
        PLAIN, MAP_A / MAP_B and PREDICTED_A..E quads in random order, and the end asked for"""
        L, end = spec
        rng, q, sb = self.rng, self.q, SIG["lion"]
        if L == 0:
            return np.zeros(0, np.uint8), "tail_empty"
        if ps.penalty > 0:
            return rng.integers(0, 256, L, dtype=np.uint8), "tail_copy_pending"
        if L < sb:
            return rng.integers(0, 256, L, dtype=np.uint8), "tail_short_signature"
        r_end = {"clean": 0, "plain_end": 0, "raw1": 1, "raw2": 2, "raw3": 3, "map0": 0, "map1": 1}[end]
        term = {"clean": None, "plain_end": PLAIN, "raw1": PLAIN, "raw2": PLAIN, "raw3": PLAIN, "map0": L_MAP_A, "map1": L_MAP_B}[end]
        D = L - sb - r_end
        slots = q if term is None else q - 1
        lead = D // 2 - (slots - 1) <= D // 4                         # room for the leading PREDICTED_A (not in the longest tails)
        slots -= lead
        lo, hi = max(0, D // 2 - slots), D // 4
        if D % 2 or lo > hi:
            raise ValueError(f"tail {L} {end} does not fit one block")
        p = int(rng.integers(lo, hi + 1))
        m = D // 2 - 2 * p
        npred = slots - p - m if term is None else int(rng.integers(0, slots - p - m + 1))
        body = [PLAIN] * p + [int(f) for f in rng.integers(L_MAP_A, L_MAP_B + 1, m)] + [int(f) for f in rng.integers(L_PA, L_PE + 1, npred)]
        rng.shuffle(body)
        flags = [L_PA] * lead + body
        if term is not None:
            flags.append(term)
            flags += [int(f) for f in rng.integers(0, 8, q - len(flags))]
        sig = sum(f << (3 * k) for k, f in enumerate(flags))
        out = bytearray(sig.to_bytes(sb, "little"))
        for f in body:
            if f == PLAIN:
                out += int(self._random_quads(1)[0]).to_bytes(4, "little")
            elif f >= L_MAP_A:
                out += int(rng.integers(0, 65536)).to_bytes(2, "little")
        out += rng.integers(0, 256, r_end, dtype=np.uint8).tobytes()
        assert len(out) == L, (L, end, len(out))
        return np.frombuffer(bytes(out), np.uint8), "tail_" + end

    def _tail(self, spec, ps):
        """spec = (length, end): the bytes after the main loop. end: "clean" (the last quad's payload ends the stream), "plain_end" (a
        PLAIN flag with 0 bytes left), "raw1".."raw3" (a PLAIN flag with 1-3 bytes left: raw bytes out), "map0" / "map1" (a MAP with 0 or 1
        byte left: malformed, size 0). With a copy penalty pending the tail is raw bytes (codec.rs:103-110)."""
        L, end = spec
        rng, alg, q = self.rng, self.alg, self.q
        if L == 0:
            return np.zeros(0, np.uint8), "tail_empty"
        if ps.penalty > 0:
            return rng.integers(0, 256, L, dtype=np.uint8), "tail_copy_pending"
        if L < SIG[alg]:
            return rng.integers(0, 256, L, dtype=np.uint8), "tail_short_signature"
        D = L - SIG[alg]
        r_end = {"clean": 0, "plain_end": 0, "raw1": 1, "raw2": 2, "raw3": 3, "map0": 0, "map1": 1}[end]
        term = {"clean": None, "plain_end": PLAIN, "raw1": PLAIN, "raw2": PLAIN, "raw3": PLAIN, "map0": MAP_A, "map1": MAP_A}[end]
        D -= r_end
        assert D % 2 == 0, (L, end)
        slots = q if term is None else q - 1
        npred = min(int(rng.integers(0, 6)), max(0, slots - D // 2 + D // 4)) if alg == "cheetah" else 0
        lo, hi = max(0, D // 2 - (slots - npred)), D // 4
        if term is None and alg == "chameleon":
            lo = hi = None if D < 2 * q or D > 4 * q else (D - 2 * q) // 2
        if lo is None or lo > hi:
            raise ValueError(f"tail {L} {end} does not fit one block")
        if term is None and alg == "cheetah":
            # exactly q quads: p PLAIN, m MAP, the rest PREDICTED
            p = int(rng.integers(0, D // 4 + 1))
            while D - 4 * p > 2 * (q - p):
                p += 1
            m = (D - 4 * p) // 2
            if p + m > q:
                raise ValueError(f"tail {L} {end} does not fit one block")
            flags = [PLAIN] * p + [MAP_A] * m + [PRED] * (q - p - m)
        else:
            p = int(rng.integers(lo, hi + 1))
            m = D // 2 - 2 * p
            flags = [PLAIN] * p + [MAP] * m + ([PRED] * npred if alg == "cheetah" else [])
            flags = flags[:slots] if term is not None else flags
            assert len(flags) <= slots
        rng.shuffle(flags)
        if term is not None:
            flags = flags + [term]
            flags += [int(f) for f in rng.integers(0, 1 << FB[alg], q - len(flags))]
        if alg == "chameleon" and term is not None:
            flags = [MAP if f == MAP_A else f for f in flags]
        sig = sum(int(f) << (FB[alg] * k) for k, f in enumerate(flags))
        out = bytearray(sig.to_bytes(SIG[alg], "little"))
        used = 0
        for f in flags:
            if used == D:
                break
            if f == PLAIN:
                out += int(self._random_quads(1)[0]).to_bytes(4, "little"); used += 4
            elif f in (MAP, MAP_B) or (alg == "cheetah" and f == MAP_A):
                out += int(rng.integers(0, 65536)).to_bytes(2, "little"); used += 2
        out += rng.integers(0, 256, r_end, dtype=np.uint8).tobytes()
        assert len(out) == L, (L, end, len(out))
        return np.frombuffer(bytes(out), np.uint8), "tail_" + end


# ---- plantings ----------------------------------------------------------------------------------------------------------------------
class _Planter:
    """The classes at chosen quads; every class checks that the quads it needs are still free."""

    def __init__(self, g, runs_q, cuts_q, copy):
        self.g, self.runs_q, self.cuts_q, self.copy = g, runs_q, cuts_q, copy         # first quad of every decoder run / of every piece after the first
        self.bucket0 = None
        self.turn = collections.Counter()                             # per class: how many times it was planted (cycles its variants)

    def free(self, *qs):
        g = self.g
        return all(0 <= x < g.nb * g.q and x not in g.planted and (x // g.q) not in g.forced_inc and not self.copy[x // g.q]
                   for x in qs)

    def earlier(self, qi, how):
        """a quad in front of qi: in its tile, an earlier tile, an earlier decoder run or an earlier piece; -> (quad, where it is),
        falling back to an earlier tile where the asked one does not exist"""
        tq = TILE_BLOCKS * 64
        if how == "same_tile" and qi % tq >= 8:
            return qi - 5, how
        if how == "earlier_run":
            prev = [r for r in self.runs_q if r <= qi]
            if len(prev) >= 2:
                return prev[-2] + 37, how
        if how == "earlier_piece":
            prev = [c for c in self.cuts_q if c <= qi]
            if prev:
                return prev[-1] - 41, how
        return (qi - tq - 7, "earlier_tile") if qi >= tq + 7 else (qi - 3, "same_tile")

    def cham(self, qi, k):
        g = self.g
        c = k % 7
        if c == 0 and self.free(qi):
            g.put(qi, MAP, g.fresh()); g.note("map_unwritten", qi, 0)
        elif c == 1 and self.free(qi):
            g.put(qi, MAP, FIXED_UNWRITTEN[(k // 7) % len(FIXED_UNWRITTEN)]); g.note("map_unwritten_fixed", qi, 0)
        elif c == 2:
            ask = ("same_tile", "earlier_tile", "earlier_run", "earlier_piece")[self.turn["fp0"] % 4]
            w, how = self.earlier(qi, ask)
            if self.free(w, qi) and w < qi:
                self.turn["fp0"] += how == ask                       # a variant stays asked for until it could be placed
                h = g.fresh()
                g.put(w, PLAIN, quad_of(h, 0)); g.put(qi, MAP, h)
                g.note("map_fp0_written_" + how, qi, quad_of(h, 0))
        elif c == 3 and self.free(qi):
            g.put(qi, MAP, 0)
            after = self.bucket0 is not None and qi > self.bucket0[0]
            g.note("map_bucket0_" + ("after_write" if after else "before_write"), qi, self.bucket0[1] if after else 0)
        elif c == 4 and self.free(qi - 3, qi, qi + 1):
            h = g.fresh(); x = quad_of(h, 0 if k % 2 else g.fp())
            g.put(qi - 3, PLAIN, x); g.put(qi, PLAIN, x); g.put(qi + 1, MAP, h)
            g.note("plain_same_value", qi, x); g.note("plain_same_value_reader", qi + 1, x)
        elif c == 5 and self.free(qi - 1, qi, qi + 1):
            h = g.fresh(); x = quad_of(h, g.fp() if k % 2 else 0)
            g.put(qi - 1, PLAIN, x); g.put(qi, PLAIN, twin(x)); g.put(qi + 1, MAP, h)
            g.note("plain_twin", qi, twin(x)); g.note("plain_twin_reader", qi + 1, twin(x))
        elif c == 6 and self.free(qi):
            g.put(qi, MAP, g.fresh()); g.note("map_unwritten", qi, 0)

    def pileup(self, t, n):
        """n PLAIN quads of one bucket in tile t (alternating a member and the fingerprint-0 member), each read back by a MAP at once and
        93 quads later: the mailbox slot holds D7_MB_CAP, its overflow area D7_SEC_CAP more"""
        g = self.g
        base = t * TILE_BLOCKS * 64
        qs = [base + 60 + 193 * j for j in range(n)]
        if not self.free(*[x + d for x in qs for d in (0, 1, 93)]):
            return
        h = g.fresh()
        vals = (quad_of(h, g.fp()), quad_of(h, 0))
        for j, x in enumerate(qs):
            v = vals[j % 2]
            g.put(x, PLAIN, v); g.put(x + 1, MAP, h); g.put(x + 93, MAP, h)
            g.note(f"pileup_{n}", x + 1, v); g.note(f"pileup_{n}", x + 93, v)

    def chee(self, qi, k, seam=False):
        g = self.g
        c = k % 7
        if c == 0 and self.free(qi):
            g.put(qi, MAP_A, g.fresh()); g.note("mapa_unwritten", qi, 0)
        elif c == 1 and self.free(qi, qi + 1):
            h = g.fresh()
            g.put(qi, MAP_B, h); g.put(qi + 1, MAP_A, h)
            g.note("mapb_unwritten", qi, 0); g.note("mapb_unwritten", qi + 1, 0)
        elif c in (2, 3):
            ask = ("earlier_run", "earlier_piece", "same_tile")[self.turn[c] % 3]
            w, how = self.earlier(qi, ask)
            if self.free(w, qi, qi + 1) and w < qi:
                self.turn[c] += how == ask
                h = g.fresh(); x = quad_of(h, 0 if k % 3 == 0 else g.fp())
                g.put(w, PLAIN, x)
                if c == 2:
                    g.put(qi, MAP_A, h); g.note("mapa_written_once_" + how, qi, x)
                else:
                    g.put(qi, MAP_B, h); g.put(qi + 1, MAP_B, h)
                    g.note("mapb_written_once_" + how, qi, 0); g.note("mapb_twice_" + how, qi + 1, x)
        elif c == 4 and self.free(qi - 1, qi, qi + 1):
            g.put(qi - 1, MAP_A, g.fresh()); g.put(qi, PRED, 0); g.put(qi + 1, PRED, 0)
            g.note("pred_unwritten_context", qi, 0); g.note("pred_context0", qi + 1, None)
        elif c == 5:
            L = (2, 31, 33, 40)[(k // 7) % 4]
            s0 = qi - 1 if seam else qi
            if self.free(*range(s0 - 2, s0 + L)):
                x = quad_of(g.fresh(), 0 if k % 2 else g.fp())
                g.put(s0 - 2, PLAIN, x); g.put(s0 - 1, PLAIN, x)
                for j in range(L):
                    g.put(s0 + j, PRED, 0)
                    g.note("pred_self_chain", s0 + j, x)
        elif c == 6 and self.free(qi - 2, qi - 1, qi, qi + 1):
            g.put(qi - 2, MAP_A, g.fresh()); g.put(qi - 1, PRED, 0)
            for j in (0, 1):
                g.put(qi + j, PRED, 0)
            g.note("pred_chain_through_context0", qi, None)


# ---- Lion plantings -----------------------------------------------------------------------------------------------------------------
LION_CLASSES = ("map_unwritten_ctx", "mapb_written_once", "mapb_twice", "pred_unwritten_depth_k", "pred_short_list", "pred_duplicates",
                "six_pushes_then_pred", "self_span_after_depth_k", "pred_chain_context0")
LION_PLACES = ("lane_0", "lane_15", "lane_16", "lane_31", "copy_row_lane_16", "after_copy_row_lane_0", "run_first", "run_last",
               "piece_first", "piece_last", "after_copy")


def lion_class(name):
    """the class a noted Lion quad belongs to (its variant suffix dropped)"""
    return next((c for c in LION_CLASSES if name.startswith(c)), name)


def _lion_sim(seq, st):
    """The values of a planted Lion sequence [(flag, payload)]: every bucket and context it names is fresh (never touched by random
    content), so lion.rs decodes it from empty state. The context in front of the sequence, and context 0 (random content reads and pushes
    it), are unknown: a predicted read there is None. st ({"cm": {h: [a, b]}, "lists": {ctx: list}}) carries state between sequences."""
    cm, lists = st.setdefault("cm", {}), st.setdefault("lists", {})
    ctx, out = None, []
    for flag, pay in seq:
        L = lists.get(ctx, [0] * 5) if ctx else None
        if flag == PLAIN:
            q = pay; h = hash16(q)
            a, _ = cm.get(h, (0, 0)); cm[h] = (q, a)
        elif flag == L_MAP_A:
            h = pay; q = cm.get(h, (0, 0))[0]
        elif flag == L_MAP_B:
            h = pay; a, b = cm.get(h, (0, 0)); q = b; cm[h] = (b, a)
        else:
            k = flag - 1
            if L is None:
                out.append(None); ctx = None
                continue
            q = L[k]; h = hash16(q)
            lists[ctx] = [q] + L[:k] + L[k + 1:]
            out.append(q); ctx = h
            continue
        if L is not None:
            lists[ctx] = [q] + L[:4]
        out.append(q); ctx = h
    return out


class _LionPlanter:
    """The Lion classes as sealed sequences: a MAP_A at a fresh bucket in front (its value 0 goes to the random context before it) and one
    behind (the random quad after the sequence pushes into a fresh context), so random content never reads or writes the lists and chunk
    map slots a sequence uses, and _lion_sim gives every value. A sequence runs over consecutive encoded quads: copy-mode blocks between
    them leave last_hash as it is (codec.rs:89-92)."""

    def __init__(self, g, runs_q, cuts_q, copy):
        self.g, self.runs_q, self.cuts_q, self.copy = g, runs_q, cuts_q, copy
        self.turn = collections.Counter()                             # per class: plantings placed (cycles its variants)
        self.miss = collections.Counter()                             # per class: plantings that did not fit (moves on to other variants)

    def free(self, qs):
        """in the main loop, not planted, not copy mode"""
        g = self.g
        return all(0 <= x < g.nb * g.q and x not in g.planted and not self.copy[x // g.q] for x in qs)

    def keeps_forced(self, pos, flags):
        """the blocks forced compressible stay compressible (at most 10 PLAIN quads planted in one), the blocks forced incompressible stay
        incompressible (the planted quads carry at most 6 payload bytes less than PLAIN quads: 70 - 6 = 64 bytes)"""
        g, q = self.g, self.g.q
        new = collections.defaultdict(list)
        for x, f in zip(pos, flags):
            if (x // q) in g.forced_inc:
                new[x // q].append(f)
        for b, fs in new.items():
            fs = fs + [g.planted[b * q + k][0] for k in range(q) if (b * q + k) in g.planted]
            if g.forced_inc[b] and sum(4 - PAYLOAD["lion"][f] for f in fs) > 6:
                return False
            if not g.forced_inc[b] and sum(f == PLAIN for f in fs) > 10:
                return False
        return True

    def span(self, e, nb, na):
        """nb encoded quads in front of e, e and na behind it (copy-mode blocks skipped), or None"""
        g, pos = self.g, []
        x = e
        while len(pos) < nb:
            x -= 1
            if x < 0:
                return None
            if not self.copy[x // g.q]:
                pos.insert(0, x)
        pos.append(e)
        x = e
        while len(pos) < nb + 1 + na:
            x += 1
            if x >= g.nb * g.q:
                return None
            if not self.copy[x // g.q]:
                pos.append(x)
        return pos

    def seal(self):
        return (L_MAP_A, self.g.fresh(), None)

    def place(self, seq, k0, e, pre=None):
        """seq = [(flag, payload, note or None)] with seq[k0] at quad e; pre = (sequence, first quad): an earlier sequence (a chunk-map
        write) that must end in front of seq. Returns the positions or None when a quad is taken or a forced block would change."""
        pos = self.span(e, k0, len(seq) - 1 - k0)
        if pos is None or not self.free(pos) or not self.keeps_forced(pos, [f for f, _, _ in seq]):
            return None
        st = {}
        if pre is not None:
            pseq, w = pre
            ppos = self.span(w, 0, len(pseq) - 1) if w >= 0 else None
            if ppos is None or ppos[-1] >= pos[0] or not self.free(ppos) or \
                    not self.keeps_forced(ppos + pos, [f for f, _, _ in pseq] + [f for f, _, _ in seq]):
                return None
            for x, (f, v, _) in zip(ppos, pseq):
                self.g.put(x, f, v)
            _lion_sim([(f, v) for f, v, _ in pseq], st)
        vals = self.vals = _lion_sim([(f, v) for f, v, _ in seq], st)
        for x, (f, v, note), val in zip(pos, seq, vals):
            self.g.put(x, f, 0 if v is None else v)
            if note:
                self.g.note(note, x, val)
        return pos

    def earlier(self, s0, how):
        """the first quad of a chunk-map write in front of quad s0: in its row, an earlier row, an earlier chunk-map run or an earlier
        piece; -> (quad, where), an earlier row where the asked one does not exist"""
        if how == "same_row" and s0 % 32 >= 5:
            return s0 - s0 % 32, how
        if how == "earlier_run":
            prev = [r for r in self.runs_q if r <= s0]
            if len(prev) >= 2:
                return prev[-2] + 37, how
        if how == "earlier_piece":
            prev = [c for c in self.cuts_q if c <= s0]
            if prev:
                return prev[-1] - 97, how                            # clear of the classes planted on the cut's two sides
        return s0 - 32 - 7, "earlier_row"

    def plant(self, cls, e, at_read=False):
        """plant `cls` with its key quad at e (at_read: for the MAP classes, the predicted read behind the MAP at e); True when it was
        placed"""
        g, t = self.g, self.turn[cls] + self.miss[cls]
        fresh = g.fresh
        val = lambda: quad_of(fresh(), g.fp())
        if cls == "map_unwritten_ctx":                               # the next quad's context is the explicit hash, not hash16(0)
            h, y = fresh(), val()
            if t % 2 == 0:
                seq = [self.seal(), (L_MAP_A, h, None), (PLAIN, y, None), (L_MAP_A, h, "map_unwritten_ctx_mapa")]
            else:
                seq = [self.seal(), (PLAIN, quad_of(h, g.fp()), None), (PLAIN, y, None), (L_MAP_B, h, "map_unwritten_ctx_mapb_once")]
            ok = self.place(seq + [(L_PA, None, "map_unwritten_ctx_next"), self.seal()], 3 + at_read, e)
        elif cls in ("mapb_written_once", "mapb_twice"):
            h, y = fresh(), val()
            x = quad_of(h, g.fp())
            write = [self.seal(), (PLAIN, x, None), (PLAIN, y, None), self.seal()]
            if cls == "mapb_written_once":
                seq, km = [(L_MAP_B, h, None), (L_PA, None, "mapb_written_once_next"), self.seal()], 0
            else:
                seq, km = [(L_MAP_B, h, None), (L_MAP_B, h, None), (L_PB, None, "mapb_twice_next"), self.seal()], 1
            k0 = km + at_read
            pos = self.span(e, k0, 0)
            if pos is None:
                return False
            ok = None
            for j in range(4):                                       # the variant asked for, else the others in turn
                w, how = self.earlier(pos[0], ("same_row", "earlier_row", "earlier_run", "earlier_piece")[(t + j) % 4])
                seq[km] = (L_MAP_B, h, cls + "_" + how)
                ok = self.place(seq, k0, e, (write, w))
                if ok:
                    break
        elif cls == "pred_unwritten_depth_k":
            ok = self.place([self.seal(), (L_PB + t % 4, None, cls), (L_PA, None, None), self.seal()], 1, e)
        elif cls == "pred_short_list":                               # depth k, j <= k pushes
            k = 1 + t % 4
            c, seq = fresh(), []
            seq.append((L_MAP_A, c, None))
            for _ in range(1 + (t // 4) % k):
                seq += [(PLAIN, val(), None), (L_MAP_A, c, None)]
            seq.append((L_PA + k, None, cls))
            ok = self.place(seq + [self.seal()], len(seq) - 1, e)
        elif cls == "pred_duplicates":                               # MAP_A of bucket c at context c: pushes its value, keeps context c
            c = fresh()
            x, z = quad_of(c, g.fp()), quad_of(c, g.fp() ^ 0x5A5A)
            seq = [self.seal(), (PLAIN, x, None), (L_MAP_A, c, None), (L_MAP_A, c, None), (PLAIN, z, None),     # list c: z x x
                   (L_PC, None, "pred_duplicates_c"), (L_MAP_A, c, None), (L_PD, None, "pred_duplicates_d"), (L_MAP_A, c, None),
                   (L_PE, None, "pred_duplicates_e"), self.seal()]
            ok = self.place(seq, 5, e)
        elif cls == "six_pushes_then_pred":                          # quads of bucket c keep the context at c
            c, n = fresh(), 6 + t % 2
            seq = [(L_MAP_A, c, None)] + [(PLAIN, quad_of(c, 1 + 97 * j + t % 89), None) for j in range(n)]
            seq.append((L_PC + t % 3, None, cls))
            ok = self.place(seq + [self.seal()], n + 1, e)
        elif cls == "self_span_after_depth_k":                       # x at depth k of context hash16(x), read, then PREDICTED_A on x
            k, R = 1 + t % 4, (2, 5, 14, 30)[(t // 4) % 4]
            c = fresh()
            x = quad_of(c, g.fp())
            seq = [self.seal(), (PLAIN, x, None), (PLAIN, x, None)]
            for _ in range(k):
                seq += [(PLAIN, val(), None), (L_MAP_A, c, None)]
            k0 = len(seq)
            seq.append((L_PA + k, None, cls))
            seq += [(L_PA, None, "self_span_run")] * R + [(L_PB, None, "self_span_then_depth_1"), self.seal()]
            ok = self.place(seq, k0, e)
            if ok:
                for i in range(k0, k0 + R + 1):                     # where the run crosses a block, a row or a copy-mode block
                    a, b = ok[i], ok[i + 1]
                    where = "cut_by_copy" if b - a > 1 else "cross_15_16" if a % 32 == 15 else "cross_row" if a % 32 == 31 else None
                    if where:
                        g.note("self_span_" + where, b, self.vals[i + 1])
        elif cls == "pred_chain_context0":                           # the context after an unwritten read is 0
            ok = self.place([self.seal(), (L_PB + t % 4, None, "pred_chain_context0"), (L_PA, None, "pred_chain_context0_after"),
                             (L_PC, None, "pred_chain_context0_after"), self.seal()], 1, e)
        else:
            raise ValueError(cls)
        if ok:
            self.turn[cls] += 1
        else:
            self.miss[cls] += 1
        return bool(ok)

    def copy_episode(self, b, a):
        """blocks b - 2 and b - 1 (forced incompressible, in front of the copy-mode blocks b .. a - 1) planted with quads of one bucket c
        behind a MAP_A at c: the context stays c and its list holds the last five; the last quad in front of the copy run, PREDICTED_E,
        reads one of them (hash c: a self-map) and the first quads behind it continue the span across the copy-mode blocks. -> True when
        it was placed"""
        g, q = self.g, self.g.q
        lo, e = (b - 2) * q - 1, a * q
        if b < 3 or not all(g.forced_inc.get(x) is True for x in (b - 2, b - 1)) or not self.free([lo]) or \
                any((x in g.planted) for x in range(lo, b * q)) or not self.free(range(e, e + 4)):
            return None
        c = g.fresh()
        xs = [quad_of(c, 1 + 131 * j) for j in range(2 * q - 1)]
        seq = [(L_MAP_A, c)] + [(PLAIN, x) for x in xs] + [(L_PE, None), (L_PA, None), (L_PA, None), (L_PB, None), (L_MAP_A, g.fresh())]
        pos = list(range(lo, b * q)) + [e, e + 1, e + 2, e + 3]
        if not self.keeps_forced(pos, [f for f, _ in seq]):
            return False
        vals = _lion_sim(seq, {})
        for x, (f, v), val, note in zip(pos, seq, vals, [None] * (2 * q) + ["self_span_cut_by_copy_depth_4", "self_span_cut_by_copy",
                                                                           "self_span_cut_by_copy", "self_span_then_depth_1", None]):
            g.put(x, f, 0 if v is None else v)
            if note:
                g.note(note, x, val)
        return True

    def stream_start(self):
        """predicted quads at the stream start: context 0 with empty lists, so they decode to 0"""
        if self.free(range(4)):
            for x, f in enumerate((L_PA, L_PC, L_PE)):
                self.g.put(x, f, 0); self.g.note("pred_chain_context0_stream_start", x, 0)
            self.g.put(3, L_MAP_A, self.g.fresh())

    def main_end(self, nb):
        """the last main-loop quad a MAP_A at a never-written bucket h whose list holds y: the tail's first quad (PREDICTED_A) reads y
        from the walk's last context h (not hash16(0)). -> (quad of the tail's first quad, y) or None"""
        g = self.g
        h, y = g.fresh(), quad_of(g.fresh(), g.fp())
        e = nb * g.q - 1
        if self.place([self.seal(), (L_MAP_A, h, None), (PLAIN, y, None), (L_MAP_A, h, "map_unwritten_ctx_main_last")], 3, e):
            return e + 1, y
        return None


def _plant_lion(g, run_blocks, cut_blocks, copy, main_blocks, tail_spec):
    """the Lion classes, each in turn on every placement kind (rows' lanes 0, 15, 16 and 31, rows with one copy-mode block, chunk-map run
    edges, piece edges, behind copy-mode episodes); -> ({quad: placements}, tail expectation or None)"""
    q, nb = g.q, g.nb
    pl = _LionPlanter(g, [b * q for b in run_blocks], [b * q for b in cut_blocks], copy)
    kinds = {k: [] for k in LION_PLACES if "copy" not in k}
    nrows = (nb + 1) // 2
    for li, lane in enumerate((0, 15, 16, 31)):
        for j in range(48):
            kinds[f"lane_{lane}"].append(min(nrows - 1, (j * nrows) // 48 + 3 + 7 * li) * 32 + lane)
    for b in run_blocks[1:]:
        kinds["run_first"].append(b * q); kinds["run_last"].append(b * q - 1)
    for b in cut_blocks:
        kinds["piece_first"].append(b * q); kinds["piece_last"].append(b * q - 1)
    place = {}
    for k, qs in kinds.items():
        for x in qs:
            place.setdefault(x, set()).add(k)
    pl.stream_start()
    tail = None
    if main_blocks == nb and SIG["lion"] <= tail_spec[0] <= SIG["lion"] + 4 * (q - 1):             # a tail with a leading PREDICTED_A
        tail = pl.main_end(nb)
    ci = collections.Counter({k: nb for k in LION_PLACES})              # streams start the classes at different turns
    for i in range(max(len(v) for v in kinds.values())):
        order = list(kinds)[i % len(kinds):] + list(kinds)[:i % len(kinds)]
        if i % 2:                                                    # the two sides of a seam take turns at coming first
            order = [k.replace("_first", "_x").replace("_last", "_first").replace("_x", "_last") for k in order]
        for k in order:
            if i < len(kinds[k]) and 0 < kinds[k][i] < nb * q - 48:
                if pl.plant(LION_CLASSES[ci[k] % len(LION_CLASSES)], kinds[k][i]):
                    ci[k] += 1
    # copy-mode episodes: the first quad behind one (lane 16 of a row whose first block is copy mode, lane 0 of a row behind one whose
    # second block is) takes its context from the walk's carry across the copy-mode blocks. It holds a class's key quad (for the MAP
    # classes the predicted read behind the MAP, which is the last quad in front of the copy run), or, at every third episode, a
    # self-map span across the copy-mode blocks.
    for k, b in enumerate(np.flatnonzero(copy[1:] & ~copy[:-1]) + 1):
        a = int(b)
        while a < nb and copy[a]:
            a += 1
        if a + 2 >= nb:
            continue
        where = ("after_copy", "copy_row_lane_16" if (a - 1) % 2 == 0 else "after_copy_row_lane_0")
        if k % 3 == 2:
            ok = pl.copy_episode(int(b), a)
        else:
            ok = pl.plant(LION_CLASSES[ci[where[1]] % len(LION_CLASSES)], a * q, at_read=True)
            ci[where[1]] += ok
        if ok:
            place.setdefault(a * q, set()).update(where)
    return place, tail


def _drive_automaton(g, seams, nblocks):
    """force incompressible / compressible blocks so that the automaton is in a chosen state in front of chosen blocks: a state at every
    decoder run seam, then every reachable state once; each word (protection.word_to) follows 64 compressible blocks that take the
    automaton back to its initial state"""
    states = sorted(P.reachable_states())
    at_seams = []
    for s in seams:
        ph = [x for x in states if x[3] == s % 16]
        at_seams.append((s, ph[len(at_seams) % len(ph)]))
    targets, k, cur = [], 0, 0
    while True:
        st = states[k % len(states)]
        B = cur + 64 + 8
        while True:
            B += (st[3] - B) % 16
            word = P.word_to(st[:3], B)
            if B - len(word) - 64 >= cur:
                break
            B += 16
        if B >= nblocks - 40:
            break
        targets.append((B, st)); k += 1; cur = B + 1
    taken, out = set(), []
    for B, st in targets + at_seams:                                 # the seams where they do not collide with the sweep
        word = P.word_to(st[:3], B)
        lo = B - len(word) - 64
        if lo < 0 or any(x in taken for x in range(lo, B + 1)) or B >= nblocks - 2:
            continue
        for x in range(lo, B - len(word)):
            g.forced_inc[x] = False
        for j, c in enumerate(word):
            g.forced_inc[B - len(word) + j] = c == "R"
        taken.update(range(lo, B + 1))
        out.append((B, st))
    return sorted(out)


def _plant(g, alg, run_blocks, cut_blocks, copy, nbytes, cap, main_blocks, num_sms):
    """plant the classes on the edges of the geometry the decoder uses for (nbytes, cap); returns {quad: placements}"""
    q, nblocks = g.q, g.nb
    pl = _Planter(g, [b * q for b in run_blocks], [b * q for b in cut_blocks], copy)
    place = {}

    def at(quad, kind):
        place.setdefault(quad, set()).add(kind)

    for b in run_blocks[1:]:
        at(b * q, "run_first"); at(b * q - 1, "run_last")
    for b in cut_blocks:
        at(b * q, "piece_first"); at(b * q - 1, "piece_last")
    runs = None
    if alg == "chameleon":
        runs = cham_dec_runs(nbytes, cap, main_blocks, num_sms)
        tq = TILE_BLOCKS * q
        for t0, t1 in runs:
            for t in sorted({t0, t0 + 1, t1 - 1}):
                at(t * tq, "tile_first"); at(t * tq + tq - 1, "tile_last")
                at(t * tq + 256, "region_first"); at(t * tq + 15 * 256, "region_first")
                at(t * tq + 255, "region_last"); at(t * tq + 4 * 256 - 1, "region_last")
    for b in np.flatnonzero(copy):
        if b + 1 < nblocks and not copy[b + 1]:
            at(int(b + 1) * q, "after_copy")
    edges = sorted(e for e in place if 0 < e < nblocks * q - 64 and not copy[e // q])
    mid = edges[len(edges) // 2] if edges else 0
    if alg == "chameleon" and pl.free(mid + 2):
        x = quad_of(0, g.fp())
        g.put(mid + 2, PLAIN, x)
        pl.bucket0 = (mid + 2, x)
        g.note("bucket0_write", mid + 2, x)
    for k, e in enumerate(edges):
        if alg == "chameleon":
            pl.cham(e, k)
        else:
            pl.chee(e, k, seam=(e // q) in run_blocks and e % q == 0)
    if runs:
        t0, t1 = runs[len(runs) // 2]
        for j, n in enumerate((D7_MB_CAP, D7_MB_CAP + 1, D7_MB_CAP + D7_SEC_CAP, D7_MB_CAP + D7_SEC_CAP + 1)):
            if t0 + 2 + j < t1 - 1:
                pl.pileup(t0 + 2 + j, n)
    return place


def decoded_size(alg, stream, w):
    """what the stream decodes to: the main loop's blocks and the tail decoded behind them (0 for a malformed tail); the main loop alone
    when the tail is malformed, which is the capacity the tests decode such a stream with"""
    tail = stream[w["tail_off"]:]
    st = w["state"]
    t = len(decode_reference(alg, tail, 1 << 40, prot=(st[0], st[1], st[2], st[3]))) if tail.size else 0
    return w["main_blocks"] * BS[alg] + t


def _geometry(alg, nbytes, cap, main_blocks, num_sms):
    if alg == "chameleon":
        runs = cham_dec_runs(nbytes, cap, main_blocks, num_sms)
        return [t0 * TILE_BLOCKS for t0, _ in runs], runs
    if alg == "lion":
        return lion_dec_runs(nbytes, main_blocks, num_sms), None
    return cheetah_dec_runs(nbytes, main_blocks, num_sms), None


def build(alg, plan, seed):
    """A stream of `plan["nbytes"]` bytes or so. plan keys: quiet (default True: no two incompressible blocks in a row, no copy mode),
    p_pred (Cheetah, Lion: share of PREDICTED flags), tail = (length, end) (see _Gen._tail), copy_every (force an incompressible pair every
    that many blocks), prot_states (drive the automaton into every reachable state at chosen blocks, decoder run seams included),
    cuts (fractions of the block count: piece cuts whose edges get plantings), plant (default True), num_sms, odd (Lion: the parity of
    the block count).
    The plantings sit on the decoder's runs at the capacity the stream decodes to (decoded_size: the tests decode with it, one byte
    and one block less, which give the same runs). Returns (stream, manifest): manifest = {main_blocks, tail_off, state, starts,
    copy_blocks, cut_blocks, run_blocks (first block of every decoder run), decoded_size, classes: [(class, block, quad, expected value
    or None)], placements: {edge kind: [quads that carry a class]}, prot_targets: [(block, state)], tail_class, tail_expect (Lion: the
    first tail quad and the value it decodes to, a predicted read of the main loop's last context)}."""
    num_sms = plan.get("num_sms", planted.H100_SMS)
    q = QPB[alg]
    avg = {"chameleon": 8 + 128 + 59, "cheetah": 8 + 0.3 * 32 * 4 * (1 - plan.get("p_pred", 0.5)) + 0.7 * 32 * 2 * (1 - plan.get("p_pred", 0.5)),
           "lion": 6 + 0.3 * 16 * 4 * (1 - plan.get("p_pred", 0.5)) + 0.7 * 16 * 2 * (1 - plan.get("p_pred", 0.5))}
    nblocks = max(4, int(plan["nbytes"] / avg[alg]))
    if "odd" in plan:                                                # Lion: the parity of the block count (a last row of one block)
        nblocks += nblocks % 2 != plan["odd"]
    tail = plan.get("tail", (0, "clean"))
    geo = None                                                       # decoder run seams the plantings are placed at
    for _ in range(6):
        g = _Gen(alg, nblocks, seed, plan)
        cut_blocks = sorted({int(f * nblocks) for f in plan.get("cuts", ())})
        prot_targets = []
        if plan.get("copy_every"):
            for b in range(plan["copy_every"], nblocks - 8, plan["copy_every"]):
                g.forced_inc[b] = g.forced_inc[b + 1] = True
        if plan.get("copy_at_end"):                                  # the tail is entered with a copy penalty pending
            g.forced_inc[nblocks - 2] = g.forced_inc[nblocks - 1] = True
        if plan.get("prot_states") and geo is not None:
            prot_targets = _drive_automaton(g, geo[1:], nblocks)
        place, tail_expect = {}, None
        if geo is not None and plan.get("plant", True):
            stream, copy, _, _ = g.layout(tail)
            w = walk(alg, stream)
            if alg == "lion":
                place, tail_expect = _plant_lion(g, geo, cut_blocks, copy, w["main_blocks"], tail)
            else:
                place = _plant(g, alg, geo, cut_blocks, copy, stream.size, decoded_size(alg, stream, w), w["main_blocks"], num_sms)
        stream, copy, off, tcls = g.layout(tail)
        w = walk(alg, stream)
        size = decoded_size(alg, stream, w)
        # the decoder's runs at the capacity the stream is decoded with (bounds_layout bounds the block count by it)
        new = _geometry(alg, stream.size, size, w["main_blocks"], num_sms)[0]
        if new == geo or not (plan.get("plant", True) or plan.get("prot_states")):
            break
        geo = new
    else:
        raise RuntimeError("the decoder's run seams did not settle")
    copy_blocks = [int(b) for b in np.flatnonzero(copy)]
    classes = [(c, b, qi, e) for c, b, qi, e in g.manifest if not copy[b] and b < w["main_blocks"]]
    planted_at = {qi for _, _, qi, _ in classes}
    placements = {}
    for quad, kinds in place.items():
        if quad in planted_at:
            for k in kinds:
                placements.setdefault(k, []).append(quad)
    return stream, {"alg": alg, "main_blocks": w["main_blocks"], "tail_off": w["tail_off"], "state": w["state"], "starts": w["starts"],
                    "copy_blocks": copy_blocks, "cut_blocks": cut_blocks, "classes": classes, "prot_targets": prot_targets,
                    "tail_class": tcls, "block_offsets": off[:-1], "nblocks": nblocks, "decoded_size": size,
                    "run_blocks": geo if geo is not None else new, "placements": placements,
                    "planted_flags": {qi: fl for qi, (fl, _) in g.planted.items()}, "tail_expect": tail_expect}


def flags_of(alg, stream, manifest, block):
    """the flags of an encoded main-loop block"""
    o = manifest["starts"][block]
    sig = int.from_bytes(np.asarray(stream[o:o + SIG[alg]]).tobytes(), "little")
    fb = FB[alg]
    return [(sig >> (fb * k)) & ((1 << fb) - 1) for k in range(QPB[alg])]


def _fits(alg, L, end):
    if L < SIG[alg]:
        return True
    D = L - SIG[alg] - {"clean": 0, "plain_end": 0, "raw1": 1, "raw2": 2, "raw3": 3, "map0": 0, "map1": 1}[end]
    if D % 2 or D < 0:
        return False
    q = QPB[alg]
    if alg == "lion":
        return D // 2 - (q - (end != "clean")) <= D // 4
    if end == "clean":
        return (2 * q <= D <= 4 * q) if alg == "chameleon" else D <= 4 * q
    return D // 2 - (q - 1) <= D // 4


def tail_lengths(alg):
    """every tail length 0 .. SIG[alg] + BS - 1, each with an end that fits it (the ends in turn)"""
    ends = ("clean", "plain_end", "raw1", "raw2", "raw3", "map0", "map1")
    out = []
    for L in range(SIG[alg] + BS[alg]):
        ok = [e for e in ends if _fits(alg, L, e)] or ["clean"]
        out.append((L, ok[(L // 2) % len(ok)]))
    return out
