"""Python model of the round-2 Chameleon flag pass `cham_flag_pass6` (chameleon_encode.cu): write / verify / mailbox, per 4096-quad tile,
one run with an unknown carried-in dictionary (first touches of a bucket are reported as "unresolved", exactly like the kernel's
unresolved list). Checked against the in-order dictionary walk of chameleon.rs:86-101 by tests/test_models_cpu.py.

  A  every quad reads old = tab[h]; misser <=> old != f (fingerprint 0 on a never-touched bucket: misser too)
  B  missers store f — racy: ANY one of the missers of a bucket may win (the model picks a pseudo-random one)
  C  hit members read again: unchanged -> flag 1. Dirty members = missers + hit members whose bucket changed; records in stream
     order; a record equal to the record before it whose quad is also right before it in the stream, in the same 256-quad
     region (the records of one warp), is dropped (flag 1); the others go to the mailbox of their slot (low 12 hash bits,
     4 entries) or, from the fifth on, to one of 64 overflow mailboxes (16 entries); a 17th entry => the whole tile is replayed
     in order instead (`replay`)
  D  per record: predecessor = entry of my bucket with the largest smaller record index -> flag = its fingerprint == mine; none ->
     touched ? pre-tile fingerprint == mine : unresolved; the member without a successor stores the bucket's final fingerprint

`overlap=True` models a three-barrier tile that was built and measured slower (DESIGN.md section 9): when the tile before this
one exists and did not overflow, phase A of this tile runs during that tile's phase D, while D writes the dictionary. A bucket with an
entry in the previous tile's mailboxes is *stale*: D is writing it. Its value after D is the fingerprint of the bucket's entry with
the largest record index (D writes exactly that), so a stale member takes its pre-tile value, touched, from the mailbox and the
record; both are read-only during D. Every other bucket is written neither by B nor by D of the previous tile, so the dictionary
read during D is its pre-tile value. The model gives the other buckets the dictionary as it stood when D began: a bucket that D did
write would read a wrong value there. After the first tile of the run and after an overflow tile, A runs after the barrier. The
dirty members, the mailboxes and the overflow tiles are those of the four-barrier tile (`overlap=False`, the kernel).
"""
import numpy as np

M = 0x9D6EF916
TILE = 4096
MB_SLOTS, MB_CAP, SEC_SLOTS, SEC_CAP = 4096, 4, 64, 16
REGION = 256                                   # quads per warp: a warp compacts and deposits its own records


def hf(q):
    p = (q.astype(np.uint64) * M) & 0xFFFFFFFF
    return (p >> 16).astype(np.int64), ((p & 0xFFFE) | (q.astype(np.uint64) >> 31)).astype(np.int64)


def reference_flags(q):
    """In-order walk. 0 miss, 1 hit, 2 first touch of the bucket (decided by the carry-in: the kernel's unresolved list)."""
    h, f = hf(q)
    tab = {}
    out = np.zeros(q.size, np.uint8)
    for i in range(q.size):
        k, v = int(h[i]), int(f[i])
        if k not in tab:
            out[i] = 2
        else:
            out[i] = 1 if tab[k] == v else 0
        tab[k] = v
    return out, tab


def _mailbox_last(mb, sec, rec, hs, b):
    """Record index of the last member of bucket b in a tile's mailboxes (the one D lets write the bucket), or None."""
    slot = b & (MB_SLOTS - 1)
    cand = list(mb.get(slot, []))
    if len(cand) >= MB_CAP:
        cand += sec.get(slot & (SEC_SLOTS - 1), [])
    same = [c for c in cand if int(hs[rec[c]]) == b]
    return max(same) if same else None


def flag_pass(q, seed=1, stats=None, overlap=False):
    rng = np.random.default_rng(seed)
    h, f = hf(q)
    tab = np.zeros(65536, np.int64)            # fingerprints
    touched = np.zeros(65536, bool)            # tab != 0 or the touched bit
    out = np.zeros(q.size, np.uint8)
    early = None                               # A of this tile ran during the previous tile's D: what it could read there
    for t0 in range(0, q.size, TILE):
        hs, fs = h[t0:t0 + TILE], f[t0:t0 + TILE]
        n = hs.size
        if early is None:
            old = tab[hs].copy()
            old_t = touched[hs].copy()
            nstale = 0
        else:
            tab_d, touched_d, pmb, psec, prec, phs, pfs = early
            old = tab_d[hs].copy()
            old_t = touched_d[hs].copy()
            nstale = 0
            for b in np.unique(hs):
                k = _mailbox_last(pmb, psec, prec, phs, int(b))
                if k is not None:                  # stale: the previous D writes this bucket; its last record says with what
                    sel = hs == b
                    old[sel] = pfs[prec[k]]
                    old_t[sel] = True
                    nstale += int(sel.sum())
        miss = (old != fs) | ((fs == 0) & (old == 0) & ~old_t)
        # B: racy publish
        pub = tab.copy()
        for b in np.unique(hs[miss]):
            cands = fs[miss & (hs == b)]
            pub[b] = cands[rng.integers(cands.size)]
        # C
        dirty = miss | (pub[hs] != fs)
        flags = np.where(dirty, 0, 1).astype(np.uint8)
        rec = np.flatnonzero(dirty)            # stream order == record index order
        dropped = np.zeros(rec.size, bool)
        for k in range(1, rec.size):
            i, j = rec[k], rec[k - 1]
            if i == j + 1 and i // REGION == j // REGION and hs[i] == hs[j] and fs[i] == fs[j]:
                dropped[k] = True
                flags[i] = 1
        mb, sec, overflow = {}, {}, False
        for k in range(rec.size):              # arrival order does not matter: the record index orders the entries
            if dropped[k]:
                continue
            slot = int(hs[rec[k]]) & (MB_SLOTS - 1)
            lst = mb.setdefault(slot, [])
            if len(lst) < MB_CAP:
                lst.append(k)
            else:
                l2 = sec.setdefault(slot & (SEC_SLOTS - 1), [])
                if len(l2) < SEC_CAP:
                    l2.append(k)
                else:
                    overflow = True
        if stats is not None:
            stats["tiles"] = stats.get("tiles", 0) + 1
            stats["overflow"] = stats.get("overflow", 0) + int(overflow)
            stats["dirty"] = stats.get("dirty", 0) + int(rec.size)
            stats["early"] = stats.get("early", 0) + int(early is not None)
            stats["stale"] = stats.get("stale", 0) + nstale
            stats.setdefault("tile_overflow", []).append(overflow)   # per tile, in stream order
            # records (dropped ones included) of each warp's region: the trip count of the deposit and D loops is ceil(count / 32)
            stats.setdefault("warp_records", []).append(np.bincount(rec // REGION, minlength=TILE // REGION))
        early = None
        if overflow:
            # replay: restore the pre-tile values of the dirty buckets, walk the dirty members in stream order
            cur, cur_t = tab, touched
            for k in range(rec.size):
                cur[hs[rec[k]]] = old[rec[k]]
            for k in range(rec.size):
                i = rec[k]
                b, v = int(hs[i]), int(fs[i])
                if not cur_t[b]:
                    flags[i] = 2
                else:
                    flags[i] = 1 if cur[b] == v else 0
                cur[b] = v
                cur_t[b] = True
        else:
            if overlap:                         # the next tile's A sees the dictionary as D begins, and these mailboxes
                early = (pub.copy(), touched.copy(), mb, sec, rec, hs, fs)
            newtab = pub                        # clean buckets: unchanged; dirty buckets: written once below
            for k in range(rec.size):
                if dropped[k]:
                    continue
                i = rec[k]
                b, v = int(hs[i]), int(fs[i])
                slot = b & (MB_SLOTS - 1)
                cand = list(mb.get(slot, []))
                if len(mb.get(slot, [])) >= MB_CAP:
                    cand += sec.get(slot & (SEC_SLOTS - 1), [])
                same = [c for c in cand if int(hs[rec[c]]) == b]
                lower = [c for c in same if c < k]
                later = any(c > k for c in same)
                if lower:
                    flags[i] = 1 if int(fs[rec[max(lower)]]) == v else 0
                elif old_t[i]:
                    flags[i] = 1 if int(old[i]) == v else 0
                else:
                    flags[i] = 2
                if not later:
                    newtab[b] = v
                    touched[b] = True
            tab = newtab
        out[t0:t0 + n] = flags
    return out, tab, touched


# ------------------------------------------------------------------------------------------------------------------------------
# Decode side: `cham_decode_pass7` (chameleon_decode.cu). A tile's quads are writers (PLAIN: value in the stream, written to the
# dictionary at hash(value)) or readers (MAP: 16-bit hash in the stream, value = the latest PLAIN quad of that bucket, 0 if none).
#   A  readers read the pre-tile dictionary            B  writers store their fingerprint (racy) and raise a byte of a HASHED mark map
#   C  a reader whose mark byte is clear is final (no writer of its bucket in this tile); the others are suspects
#   D  a suspect takes the writer with the largest smaller stream index in its bucket (mailboxes hold writers only), else its pre-tile
#      value; the writer without a successor leaves the bucket's final value; mailbox overflow => in-order replay of the tile
MARK_N = 8192


def decode_reference(is_plain, payload):
    """In order: payload = quad for PLAIN, hash for MAP. Returns the quads."""
    d = {}
    out = np.zeros(is_plain.size, np.uint64)
    for i in range(is_plain.size):
        if is_plain[i]:
            q = int(payload[i])
            d[(q * M & 0xFFFFFFFF) >> 16] = q
            out[i] = q
        else:
            out[i] = d.get(int(payload[i]), 0)
    return out, d


def decode_pass(is_plain, payload, seed=1, stats=None):
    rng = np.random.default_rng(seed)
    dic = {}                                   # bucket -> quad (the kernel keeps fingerprints; quad_from_hf is a bijection per bucket)
    out = np.zeros(is_plain.size, np.uint64)
    for t0 in range(0, is_plain.size, TILE):
        pl, pay = is_plain[t0:t0 + TILE], payload[t0:t0 + TILE]
        n = pl.size
        hk = np.where(pl, ((pay.astype(np.uint64) * M) & 0xFFFFFFFF) >> 16, pay).astype(np.int64)
        pre = [dic.get(int(hk[i])) for i in range(n)]              # phase A (readers)
        widx = np.flatnonzero(pl)
        mark = np.zeros(MARK_N, bool)
        mark[hk[widx] & (MARK_N - 1)] = True                       # phase B (the racy stores themselves are never read back by the model:
        #                                                            a suspect never trusts the dictionary, a clean reader's bucket is unwritten)
        res = np.zeros(n, np.uint64)
        suspects = []
        for i in range(n):                                          # phase C
            if pl[i]:
                res[i] = pay[i]
            elif not mark[int(hk[i]) & (MARK_N - 1)]:
                res[i] = pre[i] if pre[i] is not None else 0
            else:
                suspects.append(i)
        recs = sorted(list(widx) + suspects)                        # record index order == stream order
        ridx = {i: k for k, i in enumerate(recs)}
        mb, sec, overflow = {}, {}, False
        for i in widx:
            slot = int(hk[i]) & (MB_SLOTS - 1)
            lst = mb.setdefault(slot, [])
            if len(lst) < MB_CAP:
                lst.append(ridx[i])
            else:
                l2 = sec.setdefault(slot & (SEC_SLOTS - 1), [])
                if len(l2) < SEC_CAP:
                    l2.append(ridx[i])
                else:
                    overflow = True
        if stats is not None:
            stats["overflow"] = stats.get("overflow", 0) + int(overflow)
            stats["suspects"] = stats.get("suspects", 0) + len(suspects)
            stats.setdefault("tile_overflow", []).append(overflow)
        if overflow:                                                # d7_replay: records in order, "written so far in this tile" bitmap
            seen = {}
            for i in recs:
                b = int(hk[i])
                if pl[i]:
                    seen[b] = int(pay[i])
                else:
                    res[i] = seen[b] if b in seen else (pre[i] if pre[i] is not None else 0)
            dic.update(seen)
        else:
            for i in recs:                                          # phase D
                b = int(hk[i])
                slot = b & (MB_SLOTS - 1)
                cand = list(mb.get(slot, []))
                if len(mb.get(slot, [])) >= MB_CAP:
                    cand += sec.get(slot & (SEC_SLOTS - 1), [])
                same = [c for c in cand if int(hk[recs[c]]) == b]
                k = ridx[i]
                if pl[i]:
                    if not any(c > k for c in same):
                        dic[b] = int(pay[i])
                else:
                    lower = [c for c in same if c < k]
                    res[i] = int(pay[recs[max(lower)]]) if lower else (pre[i] if pre[i] is not None else 0)
        out[t0:t0 + n] = res
    return out, dic


if __name__ == "__main__":
    # Records per tile and overflow tiles per run of the flag pass on the bench text (1 GiB of synth_text, the runs of an H100),
    # with the four-barrier tile and with the three-barrier one: `python -m tools.proto_tile_protocol_v6 [runs...]`
    import sys
    from density_b200 import synth
    nbytes, nsm = 1 << 30, 132
    ntiles = nbytes // (TILE * 4)
    nruns = min(max(ntiles // 16, 1), nsm)
    for r in [int(a) for a in sys.argv[1:]] or [0, 77]:
        t0, t1 = r * ntiles // nruns, (r + 1) * ntiles // nruns
        data = synth.synth_text(t1 * TILE * 4).numpy()[t0 * TILE * 4:]
        q = data.view(np.uint32)
        want, _ = reference_flags(q)
        for overlap in (False, True):
            st = {}
            got, _, _ = flag_pass(q, seed=1, stats=st, overlap=overlap)
            assert (got == want).all()
            print(f"run {r} ({st['tiles']} tiles) {'three' if overlap else 'four'} barriers: records/tile {st['dirty'] / st['tiles']:.1f}, "
                  f"stale members/tile {st['stale'] / st['tiles']:.1f}, tiles with an early A {st['early']}, overflow tiles {st['overflow']}", flush=True)
