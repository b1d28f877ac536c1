// chameleon_encode.cu — Chameleon encode for sm_90a.
//
// Replaces /root/reference/src/algorithms/chameleon/chameleon.rs:86-101 (encode_quad) driven by
// /root/reference/src/codec/codec.rs:34-80 (encode_block / encode), bit-exactly.
//
// The reference walks the stream once with ONE 65,536-entry dictionary that every quad reads and (on a
// miss) writes, so flag i depends on the most recent earlier quad with the same 16-bit hash. This file
// turns that into a data-parallel computation:
//
//   flag_i = 1  <=>  the previous quad in the same hash bucket (in stream order, skipping copy-mode blocks)
//                    equals quad_i; an empty bucket behaves as "holds quad 0".
//
// Pass 1  cham_flag_pass6     one persistent CTA per SM; CTA r owns the contiguous run r of the stream, keeps the run's
//                             dictionary in shared memory as 16-bit fingerprints and walks the run in tiles of 4096 quads
//                             (write / verify / mailbox; see the section comment above the kernel). First touches of a bucket
//                             inside a run cannot know the dictionary carried in from earlier runs; they are recorded in an
//                             "unresolved" list.
//         cham_carry_scan     per-bucket left fold of the runs' last-writer tables -> carry-in table per run.
//         cham_resolve        patches the unresolved flags from the carry-in tables.
//         cham_tile_sizes     per-block output sizes -> per-tile byte counts; detects whether the reference's
//                             protection automaton (codec/protection_state.rs) could ever have fired.
//         scan kernels        exclusive scan of the tile byte counts.
// Pass 2  cham_emit           re-reads the input, writes signatures + 2/4-byte payload at the scanned offsets.
//
// If two consecutive blocks are incompressible the automaton may switch to copy mode, which removes blocks
// from the dictionary history. That case is handled by cham_protected_pass: an exact, in-order,
// protection-aware single-CTA walk (also the device-side checker for the fast path in the tests).
#include <cstdio>
#include "common.cuh"
#include "encode_internal.cuh"

namespace dns {
namespace cham {

// ------------------------------------------------------------------------------------------------------
// Pass 1: flag pass. Write -> verify -> resolve the dirty members through a per-tile mailbox.
//
// One persistent CTA per run: run r owns tiles [r * tiles_total / nruns, (r + 1) * tiles_total / nruns) of the stream and keeps the
// run's dictionary in shared memory as 16-bit fingerprints (128 KiB, see common.cuh), starting empty. Outputs:
//   sigw_g       the flag bits of every block of the run, 2 x u32 per block (low half first);
//   unres        per run, up to 65536 (quad index in the run, hash | fp << 16): the quads whose bucket the run had not touched yet.
//                They cannot know the dictionary carried in from earlier runs, so their flag is left 0 for cham_resolve to patch;
//   unres_count  per run, the length of that list;
//   final_tab    per run, 65536 x (touched << 16 | fp): the run's last-writer table, folded by cham_carry_scan.
// With `copymap`, the quads of copy-mode blocks neither read nor write the dictionary (codec.rs:35-37); with `gate`, the kernel runs
// only while the protection iteration is still open. Per 4096-quad tile:
//   A  every quad reads the pre-tile dictionary: old != f => misser.                                                    (barrier)
//   B  missers store their fingerprint (racy on purpose).                                                              (barrier)
//   C  hit members read again: unchanged => no misser in my bucket => flag 1, final. Everything else -- the missers and the hit
//      members of a bucket some misser wrote to -- is a *dirty member* (~10 % of the quads on text). Each warp compacts its dirty
//      members in stream order into its record region (ballot + popc) and then, one record per lane, drops the record's index into the
//      mailbox of its bucket: 4096 slots (low 12 hash bits) x 4 entries of 16 bits (high 4 hash bits | record index); fifth and later
//      members of a slot go to 64 shared overflow mailboxes of 16 entries. A record equal to the record before it whose quad is also
//      right before it in the stream (a run of equal quads) is a hit on that quad and changes nothing: it is dropped here, so a run
//      of equal quads costs one mailbox entry.                                                                          (barrier)
//   D  one record per lane again: the slot's entries with my bucket give my predecessor (largest smaller index: region order is
//      stream order) => flag = predecessor's fingerprint == mine, or the pre-tile value when there is none; the member without a
//      successor stores the bucket's final fingerprint. First touches of a bucket inside the run go to the unresolved list.  (barrier)
// Clean buckets are never written and every dirty bucket is written once in D, so the dictionary after D is the sequential one.
// Phases A-D do the same work in every warp whatever the data; an overflow mailbox that would need a 17th entry (~20 dirty
// members of one bucket inside one tile that are not one run) sends the tile to f6_replay: the in-order replay of the dirty members,
// one bucket class per warp (exact for any input; on text, the first three tiles of every run, whose dictionary starts empty).
// ------------------------------------------------------------------------------------------------------
constexpr int TILE_Q = 4096;                           // quads per tile = 16 KiB = 64 blocks
__device__ __forceinline__ bool bit_test(const uint32_t* bm, uint32_t i) { return (bm[i >> 5] >> (i & 31)) & 1u; }

constexpr int F6_THREADS = 512, F6_QPT = 8;           // 16 warps, 8 quads per thread: one tile = TILE_Q quads
constexpr int F6_NW = F6_THREADS / 32, F6_WQ = 32 * F6_QPT;   // warps; quads (= record region size) per warp
static_assert(F6_THREADS * F6_QPT == TILE_Q, "tile geometry");
constexpr int F6_MB_SLOTS = 4096, F6_MB_CAP = 4;      // mailboxes: slot = low 12 hash bits
constexpr int F6_SEC_SLOTS = 64, F6_SEC_CAP = 16;      // overflow mailboxes shared by the slots with the same low 6 bits
#ifdef DNS_PHASE_TIMING
__device__ long long g_f6_ph[8];
#define F6_PH(k) { if (threadIdx.x == 0 && blockIdx.x == 77) { long long tn = clock64(); g_f6_ph[k] += tn - f6_tprev; f6_tprev = tn; } }
#define F6_PH_DECL long long f6_tprev = clock64();
#else
#define F6_PH(k)
#define F6_PH_DECL
#endif
constexpr uint32_t F6_TOUCHED = 1u << 12, F6_DROPPED = 1u << 13;   // record.y: pos (12) | touched << 12 | dropped << 13 | pre-tile fingerprint << 16
struct Flag6Smem {
    uint16_t tab[65536];          // fingerprint of the last quad seen in each bucket
    uint32_t vbit[2048];          // "bucket touched" for the one case tab cannot express (fingerprint 0)
    uint2 rec[TILE_Q];            // warp w: records [128 w, 128 w + cnt[w]) in stream order. x = hash | fp << 16, y see above
    union {
        uint16_t mb[F6_MB_SLOTS][F6_MB_CAP];
        uint2 stage[F6_NW][64];   // fallback only (the mailboxes are void then): per-warp staging of the replayed records
    };
    uint32_t mbcnt[2][F6_MB_SLOTS / 4];   // entry counts, 8 bits per slot; double buffered (the idle half is cleared during the tile)
    __align__(16) uint32_t sec[F6_SEC_SLOTS][F6_SEC_CAP];
    uint32_t seccnt[2][F6_SEC_SLOTS];
    uint32_t sigw[2][TILE_Q / 32];
    uint32_t cnt[32];             // records per warp (F6_NW used)
    uint32_t unres_count;
    uint32_t overflow;
};
static_assert(sizeof(Flag6Smem) <= 227 * 1024, "flag pass shared memory");

// Append the lanes with `pred` set to the run's unresolved list (warp-aggregated; all 32 lanes call).
__device__ __forceinline__ void f6_append_unres(bool pred, uint32_t qidx_in_run, uint32_t hf, uint32_t* s_count, uint2* __restrict__ unres_run) {
    const uint32_t m = __ballot_sync(0xFFFFFFFFu, pred);
    if (m == 0) return;
    uint32_t base = 0;
    if ((threadIdx.x & 31) == 0) base = atomicAdd(s_count, (uint32_t)__popc(m));
    base = __shfl_sync(0xFFFFFFFFu, base, 0);
    if (pred) {
        const uint32_t idx = base + __popc(m & lanemask_lt());
        if (idx < 65536u) unres_run[idx] = make_uint2(qidx_in_run, hf);
    }
}

// Fallback: in-order replay of the tile's dirty members, exact for any input. Buckets of different classes (hash >> 12) never interact,
// so warp w replays the members of class w: every warp first restores the pre-tile value of the dirty buckets of its own region (each
// record carries it); then each warp reads all regions in stream order, stages the records of its class (ballot + popc) and walks them
// 32 per step (match_any for members of the same bucket inside a step). All threads of the CTA call.
static_assert(F6_NW == 16, "one warp per bucket class hash >> 12");
__device__ __forceinline__ void f6_replay_step(Flag6Smem& S, const uint2* stage, uint32_t n, uint32_t buf, uint32_t run_q0,
                                               uint2* __restrict__ unres_run) {
    const uint32_t lane = threadIdx.x & 31;
    const bool valid = lane < n;
    uint2 r = make_uint2(0, 0);
    if (valid) r = stage[lane];
    const uint32_t hh = r.x & 0xFFFFu, ff = r.x >> 16, pos = r.y & 0xFFFu;
    uint32_t cur = 0;
    if (valid) cur = S.tab[hh];
    const uint32_t grp = __match_any_sync(0xFFFFFFFFu, valid ? hh : 0x10000u + lane);
    const uint32_t lower = grp & lanemask_lt();
    const uint32_t fprev = __shfl_sync(0xFFFFFFFFu, ff, lower ? 31 - __clz(lower) : 0);
    bool touched = true, hit;
    if (lower) hit = fprev == ff;
    else {
        if (cur == 0) touched = bit_test(S.vbit, hh);
        hit = touched && cur == ff;
    }
    if (valid && (grp & lanemask_gt()) == 0) {
        S.tab[hh] = (uint16_t)ff;
        if (ff == 0) atomicOr(&S.vbit[hh >> 5], 1u << (hh & 31));
    }
    if (valid && hit) atomicOr(&S.sigw[buf][pos >> 5], 1u << (pos & 31));
    f6_append_unres(valid && !touched, run_q0 + pos, r.x, &S.unres_count, unres_run);
    __syncwarp();
}

__device__ __noinline__ void f6_replay(Flag6Smem& S, uint32_t buf, uint32_t run_q0, uint2* __restrict__ unres_run) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    {
        const uint32_t n = S.cnt[warp];
        const uint2* __restrict__ myrec = S.rec + warp * F6_WQ;
        #pragma unroll 1
        for (uint32_t i = lane; i < n; i += 32) {
            const uint2 r = myrec[i];
            S.tab[r.x & 0xFFFFu] = (uint16_t)(r.y >> 16);
        }
    }
    __syncthreads();   // every dirty bucket holds its pre-tile value
    uint2* __restrict__ stage = S.stage[warp];   // < 32 staged records carried between steps + one region step
    uint32_t ns = 0;
    #pragma unroll 1
    for (uint32_t w = 0; w < (uint32_t)F6_NW; ++w) {
        const uint32_t n = S.cnt[w];
        const uint2* __restrict__ rg = S.rec + w * F6_WQ;
        #pragma unroll 1
        for (uint32_t i0 = 0; i0 < n; i0 += 32) {
            const uint32_t i = i0 + lane;
            uint2 r = make_uint2(0, 0);
            if (i < n) r = rg[i];
            const bool mine = i < n && ((r.x & 0xFFFFu) >> 12) == warp;
            const uint32_t m = __ballot_sync(0xFFFFFFFFu, mine);
            if (mine) stage[ns + __popc(m & lanemask_lt())] = r;
            ns += __popc(m);
            if (ns >= 32) {
                __syncwarp();
                f6_replay_step(S, stage, 32, buf, run_q0, unres_run);
                const uint2 rest = stage[32 + lane];
                __syncwarp();
                if (lane < ns - 32) stage[lane] = rest;
                ns -= 32;
                __syncwarp();
            }
        }
    }
    __syncwarp();
    if (ns) f6_replay_step(S, stage, ns, buf, run_q0, unres_run);
}

// One tile. GENERIC: the tile is partial or has copy-mode blocks (`validmask` bit j: my sub-row j quad takes part).
template <bool GENERIC>
__device__ __forceinline__ void f6_tile(Flag6Smem& S, const uint32_t (&q)[F6_QPT], uint32_t validmask, uint32_t buf, uint32_t run_q0,
                                        uint2* __restrict__ unres_run) {
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t pos0 = warp * F6_WQ + lane;
    uint32_t h[F6_QPT], f[F6_QPT], old[F6_QPT];
    uint32_t missmask = 0;
    F6_PH_DECL
    // the other half of the mailbox counters: last read before the previous tile's final barrier
#pragma unroll
    for (int k = 0; k < F6_MB_SLOTS / 4 / F6_THREADS; ++k) S.mbcnt[buf ^ 1u][tid + k * F6_THREADS] = 0;
    if (tid < F6_SEC_SLOTS) S.seccnt[buf ^ 1u][tid] = 0;
    // ---- A
#pragma unroll
    for (int j = 0; j < F6_QPT; ++j) {
        // prod_hash / prod_fp written as multiplies, so they issue on the FMA pipe beside the integer ALU work (p is even)
        const uint32_t p = hash_prod(q[j]);
        h[j] = __umulhi(p, 0x10000u);
        f[j] = __umulhi(q[j], 2u) + (p - h[j] * 0x10000u);
        old[j] = S.tab[h[j]];
    }
    uint32_t fmin = f[0];
#pragma unroll
    for (int j = 0; j < F6_QPT; ++j) {
        bool miss = old[j] != f[j];
        if (GENERIC) miss = miss && ((validmask >> j) & 1u);
        if (miss) missmask |= 1u << j;
        fmin = min(fmin, f[j]);
    }
    if (fmin == 0) {   // fingerprint 0 is also what an untouched bucket shows: "equal" is a hit only if the bucket was touched (rare path)
#pragma unroll
        for (int j = 0; j < F6_QPT; ++j)
            if (f[j] == 0 && old[j] == 0 && (!GENERIC || ((validmask >> j) & 1u)) && !bit_test(S.vbit, h[j])) missmask |= 1u << j;
    }
    __syncthreads();   // S1: every read of the pre-tile dictionary precedes the publishes
    F6_PH(0)
    // ---- B
#pragma unroll
    for (int j = 0; j < F6_QPT; ++j)
        if (missmask & (1u << j)) S.tab[h[j]] = (uint16_t)f[j];
    __syncthreads();   // S2
    F6_PH(1)
    // ---- C
    uint32_t clean[F6_QPT], base = 0;
    uint2* __restrict__ myrec = S.rec + warp * F6_WQ;
    const uint32_t ltmask = lanemask_lt();
#pragma unroll
    for (int j = 0; j < F6_QPT; ++j) {
        // straight-line: the re-read and the record store are predicated, the record words are formed whether or not they are stored
        const bool miss = (missmask >> j) & 1u;
        uint32_t now = f[j];
        if (!miss) now = S.tab[h[j]];
        bool dirty = miss || now != f[j];
        if (GENERIC) dirty = dirty && ((validmask >> j) & 1u);
        const uint32_t db = __ballot_sync(0xFFFFFFFFu, dirty);
        clean[j] = GENERIC ? __ballot_sync(0xFFFFFFFFu, !dirty && ((validmask >> j) & 1u)) : ~db;
        const uint2 rv = make_uint2(f[j] * 0x10000u + h[j], old[j] * 0x10000u + (pos0 + 32 * j));
        const uint32_t k = base + __popc(db & ltmask);
        if (dirty) myrec[k] = rv;
        base += __popc(db);
    }
    if (lane == 0) {
#pragma unroll
        for (int j = 0; j < F6_QPT; j += 4)
            *reinterpret_cast<uint4*>(&S.sigw[buf][warp * F6_QPT + j]) = make_uint4(clean[j], clean[j + 1], clean[j + 2], clean[j + 3]);
        S.cnt[warp] = base;
    }
    __syncwarp();
    // deposit: one record per lane (region order == stream order, so the record index orders the members of a bucket). A record
    // equal to the record right before it whose quad is also right before it in the stream (a run of equal quads) is a hit on that
    // quad and changes nothing: it is dropped here (flag 1), so a run costs one mailbox entry.
    uint2 r0 = make_uint2(0, 0);
    bool drop0 = false;
    {
        #pragma unroll 1
        for (uint32_t i0 = 0; i0 < base; i0 += 32) {
            const uint32_t i = i0 + lane;
            const bool valid = i < base;
            uint2 r = make_uint2(0xFFFFFFFFu, 0), pr = r;   // pr: the record before mine (its x and position are never rewritten)
            __syncwarp();                               // the previous step's flag writes precede these reads
            if (valid) r = myrec[i];
            if (valid && i != 0) pr = myrec[i - 1];
            __syncwarp();                               // ... and these reads precede this step's flag writes
            // "bucket touched before this tile": the pre-tile fingerprint, or the touched bit when that is 0 (stable until phase D)
            uint32_t tch = r.y >> 16;
            if (valid && tch == 0) tch = S.vbit[(r.x & 0xFFFFu) >> 5] & (1u << (r.x & 31u));
            if (valid && tch != 0) r.y |= F6_TOUCHED;
            const bool drop = valid && i != 0 && pr.x == r.x && (((pr.y + 1u) ^ r.y) & 0xFFFu) == 0;
            if (i0 == 0) { r0 = r; drop0 = drop; }
            if (drop) {
                const uint32_t pos = r.y & 0xFFFu;
                atomicOr(&S.sigw[buf][pos >> 5], 1u << (pos & 31));
                if (i0) myrec[i].y = r.y | F6_DROPPED;
            } else if (valid) {
                if (i0 && (r.y & F6_TOUCHED)) myrec[i].y = r.y;
                const uint32_t hh = r.x & 0xFFFFu, slot = hh & (F6_MB_SLOTS - 1), sh = (slot & 3u) * 8u;
                const uint32_t k = (atomicAdd(&S.mbcnt[buf][slot >> 2], 1u << sh) >> sh) & 0xFFu;
                if (k < (uint32_t)F6_MB_CAP) S.mb[slot][k] = (uint16_t)(((hh >> 12) << 12) | (warp * F6_WQ + i));
                else {      // fifth and later members of a slot: the shared overflow mailboxes (full hash | record index)
                    const uint32_t s2 = slot & (F6_SEC_SLOTS - 1);
                    const uint32_t k2 = atomicAdd(&S.seccnt[buf][s2], 1u);
                    if (k2 < (uint32_t)F6_SEC_CAP) S.sec[s2][k2] = (hh << 12) | (warp * F6_WQ + i);
                    else S.overflow = 1;
                }
            }
        }
    }
    __syncthreads();   // S3: records, counts, clean flags and mailboxes complete; nobody reads the published values any more
    F6_PH(2)
#ifdef DNS_PHASE_TIMING
    if (threadIdx.x == 0 && blockIdx.x == 77) { g_f6_ph[6] += S.overflow; uint32_t tot = 0; for (int w = 0; w < F6_NW; ++w) tot += S.cnt[w]; g_f6_ph[7] += tot; }
#endif
    if (S.overflow) {
        f6_replay(S, buf, run_q0, unres_run);
    } else {
        // ---- D
        #pragma unroll 1
        for (uint32_t i0 = 0; i0 < base; i0 += 32) {     // warp-uniform trip count
            const uint32_t i = i0 + lane;
            bool valid = i < base;
            uint2 r = r0;
            if (i0) r = valid ? myrec[i] : make_uint2(0, 0);
            if (i0 ? (r.y & F6_DROPPED) != 0 : drop0) valid = false;
            const uint32_t hh = r.x & 0xFFFFu, ff = r.x >> 16, pos = r.y & 0xFFFu, slot = hh & (F6_MB_SLOTS - 1);
            const uint32_t myidx = warp * F6_WQ + i;
            bool later = false, hit = false, unres = false;
            if (valid) {
                const uint32_t n = (S.mbcnt[buf][slot >> 2] >> ((slot & 3u) * 8u)) & 0xFFu;   // >= 1: my own entry
                const uint2 e2 = *reinterpret_cast<const uint2*>(&S.mb[slot][0]);
                const uint32_t me = (hh & 0xF000u) | myidx;
                // An entry e of my bucket is earlier than me exactly when me - e - 1 < myidx, and the latest of them has the
                // smallest such value; it is later exactly when e - me - 1 < 0xFFF - myidx. An entry of another bucket of the slot
                // meets neither, and an unused entry is replaced by my own, which meets neither.
                const uint32_t ea = e2.x & 0xFFFFu, eb = n > 1 ? e2.x >> 16 : me, ec = n > 2 ? e2.y & 0xFFFFu : me,
                               ed = n > 3 ? e2.y >> 16 : me;
                const uint32_t dmin = min(min(me - ea - 1u, me - eb - 1u), min(me - ec - 1u, me - ed - 1u));
                const uint32_t umin = min(min(ea - me - 1u, eb - me - 1u), min(ec - me - 1u, ed - me - 1u));
                int best = dmin < myidx ? (int)(myidx - 1u - dmin) : -1;
                later = umin < 0xFFFu - myidx;
                if (n > (uint32_t)F6_MB_CAP) {
                    const uint32_t s2 = slot & (F6_SEC_SLOTS - 1);
                    const uint32_t n2 = S.seccnt[buf][s2];     // <= F6_SEC_CAP here (else the tile overflowed)
                    const uint32_t mine = (hh << 12) | myidx;
                    #pragma unroll 1
                    for (uint32_t t4 = 0; t4 < n2; t4 += 4) {
                        const uint4 e4 = *reinterpret_cast<const uint4*>(&S.sec[s2][t4]);
                        const uint32_t ev[4] = {e4.x, e4.y, e4.z, e4.w};
#pragma unroll
                        for (int t = 0; t < 4; ++t) {
                            const uint32_t e = ev[t];
                            if (t4 + t < n2 && ((e ^ mine) & 0xFFFFF000u) == 0) {
                                if (e < mine) best = max(best, (int)(e & 0xFFFu));
                                later |= e > mine;
                            }
                        }
                    }
                }
                if (best >= 0) hit = (S.rec[best].x >> 16) == ff;
                else if (r.y & F6_TOUCHED) hit = (r.y >> 16) == ff;
                else unres = true;
                if (!later) {
                    S.tab[hh] = (uint16_t)ff;
                    if (ff == 0) atomicOr(&S.vbit[hh >> 5], 1u << (hh & 31));
                }
                if (hit) atomicOr(&S.sigw[buf][pos >> 5], 1u << (pos & 31));
            }
            f6_append_unres(unres, run_q0 + pos, r.x, &S.unres_count, unres_run);
        }
    }
    __syncthreads();   // S4: dictionary and flags of the tile final
    F6_PH(3)
}

__global__ void __launch_bounds__(F6_THREADS, 1)
cham_flag_pass6(const uint32_t* __restrict__ in, uint64_t nquads, uint32_t tiles_total, uint32_t nruns,
                uint32_t* __restrict__ sigw_g, uint2* __restrict__ unres, uint32_t* __restrict__ unres_count,
                uint32_t* __restrict__ final_tab, const uint8_t* __restrict__ copymap, const Status* __restrict__ gate)
{
    if (gate && !(gate->nonquiet && !gate->converged)) return;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Flag6Smem& S = *reinterpret_cast<Flag6Smem*>(smem_raw);
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t run = blockIdx.x;
    const uint64_t t_begin = (uint64_t)run * tiles_total / nruns;
    const uint64_t t_end = (uint64_t)(run + 1) * tiles_total / nruns;
    uint2* __restrict__ unres_run = unres + (size_t)run * 65536;
    const uint32_t pos0 = warp * F6_WQ + lane;
    const uint32_t ntile_run = (uint32_t)(t_end - t_begin);
    const uint64_t q_begin = t_begin * TILE_Q;
    const uint64_t q_end64 = (t_end * TILE_Q < nquads) ? t_end * TILE_Q : nquads;
    const uint32_t run_quads = q_begin < q_end64 ? (uint32_t)(q_end64 - q_begin) : 0u;
    const uint32_t* __restrict__ rin = in + q_begin;
    uint32_t* __restrict__ rsig = sigw_g + t_begin * (TILE_Q / 32);
    const uint8_t* __restrict__ rcm = copymap ? copymap + t_begin * 64 : nullptr;
    {
        const uint4 z = make_uint4(0, 0, 0, 0);
        uint4* t4 = reinterpret_cast<uint4*>(S.tab);
        #pragma unroll 1
        for (uint32_t i = tid; i < 65536 * 2 / 16; i += F6_THREADS) t4[i] = z;
        #pragma unroll 1
        for (uint32_t i = tid; i < 2048; i += F6_THREADS) S.vbit[i] = 0;
        #pragma unroll 1
        for (uint32_t i = tid; i < F6_MB_SLOTS / 4; i += F6_THREADS) { S.mbcnt[0][i] = 0; S.mbcnt[1][i] = 0; }
        if (tid < F6_SEC_SLOTS) { S.seccnt[0][tid] = 0; S.seccnt[1][tid] = 0; }
        if (tid == 0) { S.unres_count = 0; S.overflow = 0; }
    }
    __syncthreads();
    // Register ring of the next two tiles' quads: a tile's loads are issued two tiles before it runs, so they have two tiles' time to
    // arrive (every warp of the CTA issues its loads in the same burst, right after the tile's last barrier).
    uint32_t nxt[F6_QPT], nxt2[F6_QPT];
#pragma unroll
    for (int j = 0; j < F6_QPT; ++j) {
        nxt[j] = (pos0 + 32 * j < run_quads) ? ld_stream_u32(rin + pos0 + 32 * j) : 0u;
        nxt2[j] = (TILE_Q + pos0 + 32 * j < run_quads) ? ld_stream_u32(rin + TILE_Q + pos0 + 32 * j) : 0u;
    }
    // The 64-bit addressing and the bounds are set up once: a tile is whole exactly when lt < nfull, and the pointers advance by a tile.
    const uint32_t nfull = run_quads / TILE_Q;
    const uint32_t* __restrict__ np = rin + 2 * TILE_Q + pos0;    // my quads of the tile two ahead
    uint32_t* __restrict__ sp = rsig + tid;                         // my word of the tile's flags
    #pragma unroll 1
    for (uint32_t lt = 0; lt < ntile_run; ++lt, np += TILE_Q, sp += TILE_Q / 32) {
        uint32_t q[F6_QPT];
        const uint32_t run_q0 = lt * TILE_Q;
        const uint32_t buf = lt & 1u;
#pragma unroll
        for (int j = 0; j < F6_QPT; ++j) { q[j] = nxt[j]; nxt[j] = nxt2[j]; }
        if (lt + 2 < nfull) {
#pragma unroll
            for (int j = 0; j < F6_QPT; ++j) nxt2[j] = ld_stream_u32(np + 32 * j);
        } else {
            const uint32_t nleft = run_q0 + 2u * TILE_Q < run_quads ? run_quads - run_q0 - 2u * TILE_Q : 0u;
#pragma unroll
            for (int j = 0; j < F6_QPT; ++j) nxt2[j] = (pos0 + 32 * j < nleft) ? ld_stream_u32(np + 32 * j) : 0u;
        }
        if (lt < nfull && !rcm) {
            f6_tile<false>(S, q, (1u << F6_QPT) - 1u, buf, run_q0, unres_run);
        } else {
            const uint32_t left = run_q0 < run_quads ? run_quads - run_q0 : 0u;
            uint32_t validmask = 0, cp = 0;
            if (rcm) {
#pragma unroll
                for (int b = 0; b < F6_WQ / 64; ++b) cp |= (rcm[lt * 64 + warp * (F6_WQ / 64) + b] ? 1u : 0u) << b;
            }
#pragma unroll
            for (int j = 0; j < F6_QPT; ++j)
                if (pos0 + 32 * j < left && !((cp >> (j >> 1)) & 1u)) validmask |= 1u << j;
            f6_tile<true>(S, q, validmask, buf, run_q0, unres_run);
        }
        if (tid < TILE_Q / 32) *sp = S.sigw[buf][tid];
        if (tid == 0) S.overflow = 0;      // read by everybody before the tile's final barrier; next written after two more barriers
    }
    #pragma unroll 1
    for (uint32_t i = tid; i < 65536; i += F6_THREADS) {
        const uint32_t v = S.tab[i];
        const uint32_t tch = (v != 0 || bit_test(S.vbit, i)) ? 0x10000u : 0u;
        final_tab[(size_t)run * 65536 + i] = v | tch;
    }
    if (tid == 0) unres_count[run] = S.unres_count < 65536u ? S.unres_count : 65536u;
#ifdef DNS_PHASE_TIMING
    if (tid == 0 && run == 77 && ntile_run) { const long long nt = ntile_run;
        printf("f6 run %u tiles %lld cycles/tile: A %lld B %lld C+deposit %lld D+S4 %lld  overflow tiles %lld dirty/tile %lld\n", run, nt, g_f6_ph[0] / nt, g_f6_ph[1] / nt,
               g_f6_ph[2] / nt, g_f6_ph[3] / nt, g_f6_ph[6], g_f6_ph[7] / nt);
        for (int k = 0; k < 8; ++k) g_f6_ph[k] = 0; }
#endif
}

// ------------------------------------------------------------------------------------------------------
// carry-in tables: carry[r] = state of the dictionary before run r (as touched<<16 | fp)
// `init` = state before run 0 (NULL: the stream start, where only bucket 0 "holds quad 0").
// ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool gate_open(const Status* g) { return !g || (g->nonquiet && !g->converged); }

__global__ void cham_carry_scan(const uint32_t* __restrict__ final_tab, const uint32_t* __restrict__ init, int init_untouched,
                                uint32_t nruns, uint32_t* __restrict__ carry, uint32_t* __restrict__ table_out,
                                const Status* __restrict__ gate = nullptr) {
    if (!gate_open(gate)) return;
    uint32_t hb = blockIdx.x * blockDim.x + threadIdx.x;
    if (hb >= 65536) return;
    uint32_t c = init ? init[hb] : ((hb == 0 && !init_untouched) ? 0x10000u : 0u);
    for (uint32_t r = 0; r < nruns; ++r) {
        if (carry) carry[(size_t)r * 65536 + hb] = c;
        uint32_t v = final_tab[(size_t)r * 65536 + hb];
        if (v & 0x10000u) c = v;
    }
    if (table_out) table_out[hb] = c;
}

__global__ void cham_resolve(const uint2* __restrict__ unres, const uint32_t* __restrict__ unres_count,
                             const uint32_t* __restrict__ carry, uint32_t tiles_total, uint32_t nruns,
                             uint32_t* __restrict__ sigw_g, const Status* __restrict__ gate = nullptr) {
    if (!gate_open(gate)) return;
    const uint32_t run = blockIdx.y;
    const uint32_t n = unres_count[run];
    const uint64_t run_q0 = ((uint64_t)run * tiles_total / nruns) * TILE_Q;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        uint2 e = unres[(size_t)run * 65536 + i];
        uint32_t c = carry[(size_t)run * 65536 + (e.y & 0xFFFFu)];
        if ((c & 0x10000u) && (c & 0xFFFFu) == (e.y >> 16)) {
            uint64_t gq = run_q0 + e.x;
            atomicOr(&sigw_g[gq >> 5], 1u << (gq & 31));
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// Exact protection-aware walk (single CTA, one warp walks the blocks in order).
// Handles every input; used when the fast path reports `nonquiet`, and as the device-side checker.
// `start_state`: dictionary before the first block (NULL = stream start).
// ------------------------------------------------------------------------------------------------------
struct ProtSmem {
    uint16_t tab[65536];
    uint32_t vbit[2048];
};

__global__ void __launch_bounds__(1024, 1)
cham_protected_pass(const uint32_t* __restrict__ in, uint64_t nbytes, const Status* __restrict__ status, int only_if_nonquiet,
                    uint32_t* __restrict__ sigw_g, uint8_t* __restrict__ copymap) {
    if (only_if_nonquiet && !(status->nonquiet && !status->converged)) return;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    ProtSmem& S = *reinterpret_cast<ProtSmem*>(smem_raw);
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    {
        uint4 z = make_uint4(0, 0, 0, 0);
        uint4* t4 = reinterpret_cast<uint4*>(S.tab);
        for (uint32_t i = tid; i < 65536 * 2 / 16; i += blockDim.x) t4[i] = z;
        for (uint32_t i = tid; i < 2048; i += blockDim.x) S.vbit[i] = (i == 0) ? 1u : 0u;  // bucket 0 "holds quad 0"
    }
    __syncthreads();
    if (tid >= 32) return;

    const uint64_t nquads = nbytes / 4;
    const uint64_t nblocks = (nbytes + 255) / 256;
    Protection ps; ps.init();
    // register double buffer of the block's 64 quads (2 per lane)
    uint32_t n0 = 0, n1 = 0;
    if (nblocks) {
        if (lane < nquads) n0 = in[lane];
        if (32 + lane < nquads) n1 = in[32 + lane];
    }
    for (uint64_t b = 0; b < nblocks; ++b) {
        const uint32_t q0 = n0, q1 = n1;
        {
            uint64_t g = (b + 1) * 64 + lane;
            n0 = (b + 1 < nblocks && g < nquads) ? in[g] : 0u;
            n1 = (b + 1 < nblocks && g + 32 < nquads) ? in[g + 32] : 0u;
        }
        const uint64_t bq0 = b * 64;
        const uint32_t nq = (uint32_t)((nquads - bq0 < 64) ? (nquads - bq0) : 64);  // quads in this block (may be 0)
        if (ps.revert_to_copy()) {
            if (lane == 0) { copymap[b] = 1; sigw_g[2 * b] = 0; sigw_g[2 * b + 1] = 0; }
            ps.decay();
            continue;
        }
        uint32_t sig[2];
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const uint32_t q = half ? q1 : q0;
            const bool valid = half * 32 + lane < nq;
            const uint32_t p = hash_prod(q);
            uint32_t hh = valid ? prod_hash(p) : 0x10000u + lane;
            const uint32_t ff = prod_fp(p, q);
            uint32_t cur = 0; bool touched = false;
            if (valid) { cur = S.tab[hh]; touched = cur != 0 || bit_test(S.vbit, hh); }
            const uint32_t grp = __match_any_sync(0xFFFFFFFFu, hh);
            const uint32_t lower = grp & lanemask_lt();
            const int pl = lower ? 31 - __clz(lower) : 0;
            const uint32_t fprev = __shfl_sync(0xFFFFFFFFu, ff, pl);
            const bool hit = valid && (lower ? (fprev == ff) : (touched && cur == ff));
            const bool is_last = (grp & lanemask_gt()) == 0;
            if (valid && is_last && (lower || !hit)) {
                S.tab[hh] = (uint16_t)ff;
                if (ff == 0) atomicOr(&S.vbit[hh >> 5], 1u << (hh & 31));
            }
            sig[half] = __ballot_sync(0xFFFFFFFFu, hit);
            __syncwarp();
        }
        if (lane == 0) { copymap[b] = 0; sigw_g[2 * b] = sig[0]; sigw_g[2 * b + 1] = sig[1]; }
        const uint32_t hits = __popc(sig[0]) + __popc(sig[1]);
        const uint32_t tailb = (b == nblocks - 1) ? (uint32_t)(nbytes & 3) : 0u;
        const uint32_t out_sz = 8 + 4 * nq - 2 * hits + tailb;
        ps.update(out_sz >= 256);  // codec.rs:68
    }
}

// ------------------------------------------------------------------------------------------------------
// Parallel evaluation of the protection automaton (codec/protection_state.rs:18-47) over the block sequence.
//
// The copy map M (which blocks are in copy mode) is the fixed point of  M -> automaton(incompressible bits of the blocks
// that M leaves encoded, computed with M's copy-mode blocks hidden from the dictionary).  Iteration: M0 = nothing copied
// (the plain fast path), M(k+1) = automaton(flags(M(k))); when M(k+1) == M(k) the flags computed under M(k) are the
// reference's (induction over the block index: agreeing up to block b means the same dictionary and the same automaton
// state before b). The automaton itself is evaluated per segment of PSEG blocks from the canonical state
// (penalty 0, start 1, previous_incompressible false) in parallel; the seams are then settled by relaxation rounds (prot_iterate) and
// re-evaluates only the segments whose true incoming state differs (inside / right after incompressible regions).
// ------------------------------------------------------------------------------------------------------
constexpr int PSEG = 256;

// inc[b] = "block b, when encoded, is incompressible" (8 + 256 - 2*hits >= 256, codec.rs:68), refreshed after every flag pass for
// the blocks that pass encoded; blocks hidden by the copy map keep their last known value (from a pass in which they were
// encoded), which is what makes the iteration converge in 1-2 rounds: the bit hardly depends on the dictionary details.
__device__ __forceinline__ uint32_t prot_pack(const Protection& ps) { return ps.copy_penalty | (ps.copy_penalty_start << 8) | (ps.previous_incompressible << 16); }
// Walk the blocks [b0, b1) from state `ps`; writes the copy map and leaves the outgoing state in `ps`.
__device__ __forceinline__ void prot_walk(Protection& ps, const uint8_t* __restrict__ inc, uint64_t b0, uint64_t b1, uint8_t* __restrict__ cm) {
    for (uint64_t b = b0; b < b1; ++b) {
        if (ps.revert_to_copy()) { cm[b] = 1; ps.decay(); }
        else { cm[b] = 0; ps.update(__ldcg(&inc[b]) != 0); }
    }
}
// One launch per fixed-point round does the whole automaton step on a persistent grid with software grid barriers:
//   refresh the incompressible bits -> chaotic relaxation over the segments (segment s is re-evaluated whenever the outgoing
//   state of segment s-1 differs from the incoming state it was last evaluated with; a chain of L consecutive segments with
//   non-canonical seams settles after L rounds) -> in-order fix-up by one CTA if PROT_ROUNDS rounds were not enough
//   -> compare the new copy map with the one the flags were computed under -> converged / commit.
constexpr int PROT_ROUNDS = 48, PROT_FAST_ROUNDS = 4;   // relaxation rounds before the candidate evaluation when only a few seams are not canonical
constexpr int PI_THREADS = 1024;

// Exact evaluation in one shot for ordinary data: the automaton state at a segment seam is (penalty, start, previous_incompressible)
// with small penalty and start in practice (start halves every 16 blocks and grows by one per copy-mode episode: it hovers around 3-4
// even on pure noise). So every segment is walked from EVERY candidate state (PC_NC of them), which gives its transfer table
// candidate -> candidate (or PC_ESC when the walk ends outside the candidate set); the tables are composed per group of PC_GROUP
// segments, the group tables in order by one thread from the canonical state, the true incoming states are handed back down, and
// each segment is walked once more from its true state, now writing the copy map. No relaxation rounds, whatever the data. A true
// path that meets PC_ESC (never seen) falls back to the relaxation below.
constexpr uint32_t PC_NS = 10, PC_NP = 10, PC_NC = 2 * PC_NS * PC_NP, PC_ESC = 0xFFFFu, PC_GROUP = 128;
__host__ __device__ __forceinline__ size_t prot_table_elems(uint64_t nseg) {     // u16 elements behind the 2 (nseg + 1) state words
    const uint64_t ngrp = (nseg + PC_GROUP - 1) / PC_GROUP;
    return (size_t)(2 * (ngrp + 2) + nseg * PC_NC + ngrp * PC_NC + 64);
}
__device__ __forceinline__ void pc_decode(uint32_t c, Protection& ps) {
    ps.copy_penalty = c % PC_NP; ps.copy_penalty_start = (c / PC_NP) % PC_NS + 1u; ps.previous_incompressible = c / (PC_NP * PC_NS);
}
__device__ __forceinline__ uint32_t pc_encode(const Protection& ps) {
    if (ps.copy_penalty >= PC_NP || ps.copy_penalty_start < 1u || ps.copy_penalty_start > PC_NS) return PC_ESC;
    return (ps.previous_incompressible * PC_NS + (ps.copy_penalty_start - 1u)) * PC_NP + ps.copy_penalty;
}

__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int nctas, unsigned int& epoch) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(counter, 1u);
        const unsigned int target = (epoch + 1) * nctas;
        while (atomicAdd(counter, 0u) < target) { __nanosleep(64); }
        __threadfence();
    }
    ++epoch;
    __syncthreads();
}

// diagnostics of the last iteration: per fixed-point round {first block whose copy status changed, number of such blocks}
__device__ unsigned long long g_prot_dbg[16][2];

__global__ void __launch_bounds__(PI_THREADS)
prot_iterate(const uint32_t* __restrict__ sigw_g, uint64_t nbytes, uint64_t nblocks, uint32_t nseg, Status* __restrict__ st, int it,
             uint8_t* __restrict__ inc, uint8_t* __restrict__ cm_old, uint8_t* __restrict__ cm_new,
             uint32_t* __restrict__ in_state, uint32_t* __restrict__ out_state, uint16_t* __restrict__ ptab) {
    if (!gate_open(st)) return;                       // uniform over the grid: read before anybody modifies `converged`
    __shared__ uint32_t s_state[1024], s_in[1024];
    __shared__ uint8_t s_inc[PSEG], s_cm[PSEG];
    __shared__ uint32_t s_cur, s_redo;
    const uint32_t tid = threadIdx.x;
    const uint64_t gtid = (uint64_t)blockIdx.x * PI_THREADS + tid, gsz = (uint64_t)gridDim.x * PI_THREADS;
    unsigned int epoch = 0;
    unsigned int* bar = &st->barrier[it & 7];

    // (1) incompressible bits of the blocks that were encoded in the pass just finished
    if (sigw_g)   // Chameleon: derive the bits from the signatures; other codecs pass sigw_g == nullptr and fill `inc` themselves
        for (uint64_t b = gtid; b < nblocks; b += gsz)
            if (!(it && cm_old[b])) inc[b] = (nbytes - b * 256 >= 256) && (__popc(sigw_g[2 * b]) + __popc(sigw_g[2 * b + 1]) <= 4);
    if (gtid == 0) { st->relax_changed[0] = 0; st->relax_changed[1] = 0; st->iter_changed = 0; st->pad2[0] = 0; }
    if (gtid < 16 && it == 0) { g_prot_dbg[gtid][0] = ~0ull; g_prot_dbg[gtid][1] = 0; }
    grid_barrier(bar, gridDim.x, epoch);

    // (2) phase 0: round 0 evaluates every segment from the canonical state and counts the seams that are not canonical. None: done
    //     (text). A few (bursts inside text): relaxation rounds (segment s is re-evaluated whenever the outgoing state of segment s-1
    //     changed), at most PROT_FAST_ROUNDS. Many (mixed data, noise: a chain of L non-canonical seams needs L rounds), or not settled:
    //     the candidate-state evaluation (2a). Phase 1, only if that met PC_ESC: the remaining relaxation rounds.
    bool settled = false;
    int round = 0;
    for (int phase = 0; phase < 2 && !settled; ++phase) {
    const int limit = (phase == 0 && ptab) ? PROT_FAST_ROUNDS : PROT_ROUNDS;
    for (; round < limit; ++round) {
        for (uint64_t s = gtid; s < nseg; s += gsz) {
            const uint32_t new_in = (s && round) ? __ldcg(&out_state[s - 1]) : (1u << 8);   // L2 read: written by other SMs during this kernel
            if (round > 0 && new_in == in_state[s]) continue;
            Protection ps;
            ps.copy_penalty = new_in & 0xFFu; ps.copy_penalty_start = (new_in >> 8) & 0xFFu; ps.previous_incompressible = (new_in >> 16) & 1u;
            ps.counter = s * PSEG;
            const uint64_t b1 = ((s + 1) * PSEG < nblocks) ? (s + 1) * PSEG : nblocks;
            prot_walk(ps, inc, s * PSEG, b1, cm_new);
            in_state[s] = new_in;
            out_state[s] = prot_pack(ps);
            if (round > 0) st->relax_changed[round & 1] = 1;
            else if (prot_pack(ps) != (1u << 8)) atomicAdd(&st->pad2[0], 1u);
        }
        grid_barrier(bar, gridDim.x, epoch);
        if (round == 0 && phase == 0 && ptab) {
            const unsigned int bad = *((volatile unsigned int*)&st->pad2[0]);      // uniform over the grid
            if (bad == 0) { settled = true; break; }
            if (bad > 8u) { round = 1; break; }                                     // straight to the candidate evaluation
        }
        if (round > 0) {
            const bool changed = *((volatile unsigned int*)&st->relax_changed[round & 1]) != 0;
            if (!changed) { settled = true; break; }
        }
        if (gtid == 0) st->relax_changed[(round + 1) & 1] = 0;      // the flag of the next round (nobody reads it before the next barrier)
        grid_barrier(bar, gridDim.x, epoch);
    }
    // (2a) candidate-state evaluation (see PC_NC above)
    if (phase == 0 && !settled && ptab) {
        const uint32_t ngrp = (nseg + PC_GROUP - 1) / PC_GROUP;
        uint32_t* gin = reinterpret_cast<uint32_t*>(ptab);                   // incoming candidate of every group, then the final state
        uint16_t* T = ptab + 2 * (ngrp + 2);
        uint16_t* GT = T + (size_t)nseg * PC_NC;
        for (uint64_t idx = gtid; idx < (uint64_t)nseg * PC_NC; idx += gsz) {
            const uint64_t s = idx / PC_NC;
            Protection ps; pc_decode((uint32_t)(idx % PC_NC), ps);
            ps.counter = s * PSEG;
            const uint64_t b1 = ((s + 1) * PSEG < nblocks) ? (s + 1) * PSEG : nblocks;
            uint64_t b = s * PSEG;
            for (; b + 16 <= b1; b += 16) {                       // 16 incompressible bytes per L2 load (segments start 256-byte aligned)
                const uint4 v = __ldcg(reinterpret_cast<const uint4*>(inc + b));
                const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int k = 0; k < 16; ++k) {
                    if (ps.revert_to_copy()) ps.decay();
                    else ps.update(((w[k >> 2] >> ((k & 3) * 8)) & 0xFFu) != 0);
                }
            }
            for (; b < b1; ++b) {
                if (ps.revert_to_copy()) ps.decay();
                else ps.update(__ldcg(&inc[b]) != 0);
            }
            T[idx] = (uint16_t)pc_encode(ps);
        }
        grid_barrier(bar, gridDim.x, epoch);
        for (uint64_t idx = gtid; idx < (uint64_t)ngrp * PC_NC; idx += gsz) {
            const uint32_t g = (uint32_t)(idx / PC_NC);
            uint32_t x = (uint32_t)(idx % PC_NC);
            const uint32_t s1 = ((g + 1) * PC_GROUP < nseg) ? (g + 1) * PC_GROUP : nseg;
            for (uint32_t s = g * PC_GROUP; s < s1 && x != PC_ESC; ++s) x = __ldcg(&T[(size_t)s * PC_NC + x]);
            GT[idx] = (uint16_t)x;
        }
        grid_barrier(bar, gridDim.x, epoch);
        if (gtid == 0) {
            uint32_t x = 0;                                                  // canonical state: penalty 0, start 1, not incompressible
            for (uint32_t g = 0; g < ngrp; ++g) { gin[g] = x; if (x != PC_ESC) x = __ldcg(&GT[(size_t)g * PC_NC + x]); }
            gin[ngrp] = x;
        }
        grid_barrier(bar, gridDim.x, epoch);
        if (__ldcg(&gin[ngrp]) != PC_ESC) {                                  // uniform over the grid
            for (uint64_t g = gtid; g < ngrp; g += gsz) {
                uint32_t x = __ldcg(&gin[g]);
                const uint32_t s1 = ((g + 1) * PC_GROUP < nseg) ? (uint32_t)((g + 1) * PC_GROUP) : nseg;
                for (uint32_t s = (uint32_t)g * PC_GROUP; s < s1; ++s) { in_state[s] = x; x = __ldcg(&T[(size_t)s * PC_NC + x]); }
            }
            grid_barrier(bar, gridDim.x, epoch);
            for (uint64_t s = gtid; s < nseg; s += gsz) {
                Protection ps; pc_decode(__ldcg(&in_state[s]), ps);
                ps.counter = s * PSEG;
                const uint64_t b1 = ((s + 1) * PSEG < nblocks) ? (s + 1) * PSEG : nblocks;
                prot_walk(ps, inc, s * PSEG, b1, cm_new);
            }
            grid_barrier(bar, gridDim.x, epoch);
            settled = true;
        }
    }

    }   // phase

    // (3) pathologically long incompressible stretches: finish in order (one CTA; a stored result stands when it was computed
    //     from the true incoming state)
    if (!settled) {
        if (blockIdx.x == 0) {
            if (tid == 0) s_cur = 1u << 8;
            for (uint32_t s0 = 0; s0 < nseg; s0 += 1024) {
                __syncthreads();
                for (uint32_t i = tid; i < 1024 && s0 + i < nseg; i += PI_THREADS) { s_state[i] = __ldcg(&out_state[s0 + i]); s_in[i] = __ldcg(&in_state[s0 + i]); }
                __syncthreads();
                const uint32_t cnt = (nseg - s0 < 1024u) ? (nseg - s0) : 1024u;
                uint32_t i = 0;
                while (i < cnt) {
                    if (tid == 0) {
                        uint32_t cur = s_cur;
                        while (i < cnt && cur == s_in[i]) { cur = s_state[i]; ++i; }
                        s_cur = cur;
                        s_redo = (i < cnt) ? i : 0xFFFFFFFFu;
                    }
                    __syncthreads();
                    const uint32_t r = s_redo;
                    if (r == 0xFFFFFFFFu) break;
                    const uint64_t b0 = (uint64_t)(s0 + r) * PSEG;
                    const uint32_t nb = (uint32_t)((nblocks - b0 < (uint64_t)PSEG) ? (nblocks - b0) : PSEG);
                    if (tid < nb) s_inc[tid] = __ldcg(&inc[b0 + tid]);
                    __syncthreads();
                    if (tid == 0) {
                        Protection ps; const uint32_t c = s_cur;
                        ps.copy_penalty = c & 0xFFu; ps.copy_penalty_start = (c >> 8) & 0xFFu; ps.previous_incompressible = (c >> 16) & 1u; ps.counter = b0;
                        for (uint32_t k = 0; k < nb; ++k) {
                            if (ps.revert_to_copy()) { s_cm[k] = 1; ps.decay(); }
                            else { s_cm[k] = 0; ps.update(s_inc[k] != 0); }
                        }
                        s_cur = prot_pack(ps);
                    }
                    __syncthreads();
                    if (tid < nb) cm_new[b0 + tid] = s_cm[tid];
                    i = r + 1;
                    __syncthreads();
                }
            }
        }
        grid_barrier(bar, gridDim.x, epoch);
    }

    // (4) fixed point reached?
    {
        bool diff = false;
        unsigned long long first = ~0ull; unsigned int nd = 0;
        for (uint64_t b = gtid; b < nblocks; b += gsz)
            if (__ldcg(&cm_new[b]) != (it ? cm_old[b] : 0)) { diff = true; ++nd; if (b < first) first = b; }
        if (diff) {
            atomicOr(&st->iter_changed, 1u);
            if (it >= 0 && it < 16) { atomicAdd(&g_prot_dbg[it][1], (unsigned long long)nd); atomicMin(&g_prot_dbg[it][0], first); }   // diagnostics
        }
    }
    grid_barrier(bar, gridDim.x, epoch);
    const bool converged = *((volatile unsigned int*)&st->iter_changed) == 0;
    if (!converged || it == 0)
        for (uint64_t b = gtid; b < nblocks; b += gsz) cm_old[b] = __ldcg(&cm_new[b]);
    grid_barrier(bar, gridDim.x, epoch);
    if (gtid == 0 && converged) st->converged = 1;
}

// ------------------------------------------------------------------------------------------------------
// per-tile output sizes + quiet check. One warp per tile (64 blocks, 2 per lane).
// ------------------------------------------------------------------------------------------------------
// encoded block: 8-byte signature + 4 bytes per plain quad + 2 per mapped quad + 1..3 raw tail bytes (codec.rs:39-68);
// copy-mode block: the raw bytes (codec.rs:36).
__device__ __forceinline__ uint32_t block_out_bytes(uint64_t b, uint64_t nbytes, uint32_t hits, bool copied) {
    const uint64_t boff = b * 256;
    const uint32_t blen = (uint32_t)((nbytes - boff < 256) ? (nbytes - boff) : 256);
    return copied ? blen : 8 + blen - 2 * hits;
}

__global__ void cham_tile_sizes(const uint32_t* __restrict__ sigw_g, const uint8_t* __restrict__ copymap, uint64_t nbytes,
                                uint64_t nblocks, uint32_t ntiles, int use_copymap_if_nonquiet, int check_quiet, int assume_prev_inc,
                                Status* __restrict__ status, uint32_t* __restrict__ tile_bytes) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t tile = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (tile >= ntiles) return;
    if (use_copymap_if_nonquiet && !check_quiet && !status->nonquiet) return;   // quiet input: the sizes of the first pass stand
    const bool use_cm = copymap && (!use_copymap_if_nonquiet || status->nonquiet);
    uint32_t sum = 0, incm[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const uint64_t b = (uint64_t)tile * 64 + k * 32 + lane;
        uint32_t sz = 0; bool inc = false;
        if (b < nblocks) {
            const bool copied = use_cm && copymap[b];
            const uint32_t hits = __popc(sigw_g[2 * b]) + __popc(sigw_g[2 * b + 1]);
            sz = block_out_bytes(b, nbytes, hits, copied);
            inc = !copied && sz >= 256 && (nbytes - b * 256 >= 256);
        }
        sum += sz;
        incm[k] = __ballot_sync(0xFFFFFFFFu, inc);
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, d);
    if (lane == 0) tile_bytes[tile] = sum;
    if (check_quiet && lane == 0) {
        // adjacent incompressible pair anywhere => the automaton's copy_penalty would become non-zero
        bool prev = assume_prev_inc != 0;  // shard seam: the previous shard's last block is unknown here
        if (tile > 0) {
            const uint64_t b = (uint64_t)tile * 64 - 1;
            const uint32_t hits = __popc(sigw_g[2 * b]) + __popc(sigw_g[2 * b + 1]);
            prev = (8 + 256 - 2 * hits) >= 256;
        }
        const uint64_t m = ((uint64_t)incm[1] << 32) | incm[0];
        const uint64_t pairs = m & ((m << 1) | (prev ? 1ull : 0ull));
        if (pairs) {
            atomicOr(&status->nonquiet, 1u);
            atomicMin(&status->first_nonquiet_block, (unsigned long long)tile * 64 + (__ffsll((long long)pairs) - 1));
        }
    }
}

// ------------------------------------------------------------------------------------------------------
// exclusive scan of tile_bytes: groups of SCAN_G tiles
// ------------------------------------------------------------------------------------------------------
constexpr int SCAN_T = 1024;
constexpr int SCAN_PER = 4;
constexpr int SCAN_G = SCAN_T * SCAN_PER;  // tiles per group

__device__ __forceinline__ uint64_t block_exclusive_scan_u64(uint64_t v, uint64_t* s_warp, uint64_t* total) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint64_t u = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= (uint32_t)d) incl += u; }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint64_t w = (lane < (blockDim.x >> 5)) ? s_warp[lane] : 0;
        uint64_t wi = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint64_t u = __shfl_up_sync(0xFFFFFFFFu, wi, d); if (lane >= (uint32_t)d) wi += u; }
        s_warp[lane] = wi - w;
        if (lane == 31) s_warp[32] = wi;
    }
    __syncthreads();
    if (total) *total = s_warp[32];
    return incl - v + s_warp[warp];
}

__global__ void __launch_bounds__(SCAN_T) scan_groups_local(const uint32_t* __restrict__ tile_bytes, uint32_t ntiles,
                                                           uint32_t* __restrict__ tile_local, uint64_t* __restrict__ group_total) {
    __shared__ uint64_t s_warp[33];
    const uint32_t base = blockIdx.x * SCAN_G + threadIdx.x * SCAN_PER;
    uint32_t v[SCAN_PER]; uint64_t sum = 0;
#pragma unroll
    for (int k = 0; k < SCAN_PER; ++k) { v[k] = (base + k < ntiles) ? tile_bytes[base + k] : 0u; sum += v[k]; }
    uint64_t tot;
    uint64_t ex = block_exclusive_scan_u64(sum, s_warp, &tot);
#pragma unroll
    for (int k = 0; k < SCAN_PER; ++k) { if (base + k < ntiles) tile_local[base + k] = (uint32_t)ex; ex += v[k]; }
    if (threadIdx.x == 0) group_total[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(SCAN_T) scan_group_totals(const uint64_t* __restrict__ group_total, uint32_t ngroups,
                                                           uint64_t* __restrict__ group_off, Status* __restrict__ status,
                                                           uint64_t cap, uint64_t* __restrict__ d_out_size) {
    __shared__ uint64_t s_warp[33];
    __shared__ uint64_t s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < ngroups; base += SCAN_T) {
        uint32_t i = base + threadIdx.x;
        uint64_t v = (i < ngroups) ? group_total[i] : 0;
        uint64_t tot;
        uint64_t ex = block_exclusive_scan_u64(v, s_warp, &tot);
        if (i < ngroups) group_off[i] = s_carry + ex;
        __syncthreads();
        if (threadIdx.x == 0) s_carry += tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        uint64_t total = s_carry;
        if (total > cap) { status->error = 2; total = 0; }  // DENSITY_B200_ECAPACITY
        status->out_bytes = total;
        if (d_out_size) *d_out_size = total;
    }
}

// ------------------------------------------------------------------------------------------------------
// Pass 2: emit. One CTA (256 threads) per tile of 64 blocks. Pure tile movement: 128-bit streaming loads of the 16 KiB input tile,
// the tile's piece of the stream (<= 16.5 KiB) is assembled in shared memory at its final byte layout, and leaves as ONE bulk
// asynchronous copy shared -> global (cp.async.bulk, the TMA engine's 1-D mode) for the 16-byte aligned middle plus a few 2-byte
// stores for the ragged edges (the stream is only 2-byte aligned: block sizes are even, codec.rs:39-68).
// ------------------------------------------------------------------------------------------------------
constexpr int EM_THREADS = 256;
constexpr int EM_STAGE = 64 * 264 + 32;   // largest tile (64 all-plain blocks) + alignment slack

__device__ __forceinline__ uint4 ld_stream_u128(const uint32_t* p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ void bulk_store_smem_to_global(void* gdst, const void* ssrc, uint32_t bytes) {   // 16-byte aligned, bytes % 16 == 0
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(ssrc);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");    // generic-proxy writes to shared memory -> visible to the async proxy
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" :: "l"(gdst), "r"(s), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // shared memory must stay valid until it has been read
}

// The quads of one thread: 4 consecutive quads of block `bl`, starting at quad k of the block. FULL: the tile has 64 whole blocks.
template <bool FULL>
__device__ __forceinline__ void emit_quads(uint8_t* __restrict__ st, const uint32_t* s_off, const uint32_t* s_sig, const uint8_t* s_copied,
                                           const uint4 v, uint32_t u, uint32_t nvalid_tile /* quads of this tile that exist */) {
    const uint32_t bl = u >> 4, k = (u & 15u) * 4;
    const uint32_t qs[4] = {v.x, v.y, v.z, v.w};
    uint32_t nv = 4;                                                   // how many of my four quads exist
    if (!FULL) { const uint32_t first = u * 4; nv = nvalid_tile > first ? (nvalid_tile - first < 4 ? nvalid_tile - first : 4u) : 0u; }
    uint8_t* p = st + s_off[bl];
    if (s_copied[bl]) {                                                // copy-mode block: raw bytes (codec.rs:36)
        p += 4 * k;
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (FULL || (uint32_t)j < nv) { st_u16(p + 4 * j, qs[j] & 0xFFFFu); st_u16(p + 4 * j + 2, qs[j] >> 16); }
        return;
    }
    const uint32_t lo = s_sig[2 * bl], hi = s_sig[2 * bl + 1];
    if (k == 0 && (FULL || nv > 0 || true)) {                          // signature, 8 bytes LE at the block start (codec.rs:24-26,40-41,67)
        st_u16(p, lo & 0xFFFFu); st_u16(p + 2, lo >> 16); st_u16(p + 4, hi & 0xFFFFu); st_u16(p + 6, hi >> 16);
    }
    const uint32_t word = k < 32 ? lo : hi, kk = k & 31u;
    const uint32_t before = (k < 32 ? 0u : (uint32_t)__popc(lo)) + __popc(word & ((1u << kk) - 1u));
    const uint32_t fl = word >> kk;
    p += 8 + 4 * k - 2 * before;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (FULL || (uint32_t)j < nv) {
            const bool hit = (fl >> j) & 1u;
            const uint32_t hsh = prod_hash(hash_prod(qs[j]));
            st_u16(p, hit ? hsh : (qs[j] & 0xFFFFu));                  // chameleon.rs:97-98 / :92-93
            if (!hit) st_u16(p + 2, qs[j] >> 16);
            p += hit ? 2 : 4;
        }
    }
}

template <bool AL16>
__global__ void __launch_bounds__(EM_THREADS)
cham_emit(const uint32_t* __restrict__ in, uint64_t nbytes, uint64_t nblocks, const uint32_t* __restrict__ sigw_g,
          const uint8_t* __restrict__ copymap, int use_copymap_if_nonquiet, const Status* __restrict__ status,
          const uint32_t* __restrict__ tile_local, const uint64_t* __restrict__ group_off, uint8_t* __restrict__ out) {
    if (status->error) return;
    __shared__ __align__(16) uint8_t s_stage[EM_STAGE];
    __shared__ uint32_t s_off[65];
    __shared__ uint32_t s_sig[128];
    __shared__ uint8_t s_copied[64];
    __shared__ uint32_t s_wsum[2];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tile = blockIdx.x;
    const bool use_cm = copymap && (!use_copymap_if_nonquiet || status->nonquiet);
    const uint64_t tile_off = group_off[tile / SCAN_G] + tile_local[tile];
    const uint64_t nquads = nbytes / 4;
    const uint64_t tq0 = (uint64_t)tile * 4096;
    const bool full = tq0 + 4096 <= nquads;                            // 64 whole blocks (CTA-uniform)
    const uint32_t nvalid_tile = full ? 4096u : (uint32_t)(nquads > tq0 ? nquads - tq0 : 0);
    // all input loads of this thread first: 4 x 16 bytes, consecutive threads read consecutive 16-byte pieces
    uint4 qv[4];
    if (AL16 && full) {
#pragma unroll
        for (int i = 0; i < 4; ++i) qv[i] = ld_stream_u128(in + tq0 + 4u * (i * EM_THREADS + tid));
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t r = 4u * (i * EM_THREADS + tid);
            const uint32_t* g = in + tq0 + r;
            qv[i].x = (r + 0 < nvalid_tile) ? ld_stream_u32(g + 0) : 0u;
            qv[i].y = (r + 1 < nvalid_tile) ? ld_stream_u32(g + 1) : 0u;
            qv[i].z = (r + 2 < nvalid_tile) ? ld_stream_u32(g + 2) : 0u;
            qv[i].w = (r + 3 < nvalid_tile) ? ld_stream_u32(g + 3) : 0u;
        }
    }

    const uint64_t b_first = (uint64_t)tile * 64;
    const uint32_t nb_tile = (uint32_t)((nblocks - b_first < 64) ? (nblocks - b_first) : 64);
    if (tid < 64) {
        const uint64_t b = b_first + tid;
        uint32_t sz = 0, lo = 0, hi = 0; bool copied = false;
        if (tid < nb_tile) {
            copied = use_cm && copymap[b];
            lo = sigw_g[2 * b]; hi = sigw_g[2 * b + 1];
            sz = block_out_bytes(b, nbytes, __popc(lo) + __popc(hi), copied);
        }
        s_sig[2 * tid] = lo; s_sig[2 * tid + 1] = hi; s_copied[tid] = copied;
        uint32_t incl = sz;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= (uint32_t)d) incl += u; }
        if (lane == 31) s_wsum[warp] = incl;
        s_off[tid + 1] = incl;  // provisional (warp-local)
    }
    __syncthreads();
    if (tid >= 32 && tid < 64) s_off[tid + 1] += s_wsum[0];
    if (tid == 0) s_off[0] = 0;
    __syncthreads();

    // the tile's bytes sit in s_stage at the same offset modulo 16 as in the output, so that whole 16-byte lines can leave as they are
    uint8_t* const gdst = out + tile_off;
    const uint32_t a = (uint32_t)(reinterpret_cast<uintptr_t>(gdst) & 15u);
    uint8_t* const st = s_stage + a;
    if (full) {
#pragma unroll
        for (int i = 0; i < 4; ++i) emit_quads<true>(st, s_off, s_sig, s_copied, qv[i], i * EM_THREADS + tid, 4096u);
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t u = i * EM_THREADS + tid;
            if ((u >> 4) < nb_tile) emit_quads<false>(st, s_off, s_sig, s_copied, qv[i], u, nvalid_tile);
        }
        // 1..3 raw tail bytes after the last quad of the final block (codec.rs:58-61; copy mode: the rest of the raw block)
        if ((nbytes & 3u) && b_first + nb_tile == nblocks && tid < (uint32_t)(nbytes & 3u)) {
            const uint64_t b = nblocks - 1;
            const uint32_t bl = nb_tile - 1;
            const uint32_t blen = (uint32_t)(nbytes - b * 256);
            const uint32_t nq = blen >> 2;
            const uint32_t at = s_copied[bl] ? (blen & ~3u) : 8 + 4 * nq - 2 * (__popc(s_sig[2 * bl]) + __popc(s_sig[2 * bl + 1]));
            st[s_off[bl] + at + tid] = reinterpret_cast<const uint8_t*>(in)[b * 256 + (blen & ~3u) + tid];
        }
    }
    __syncthreads();

    const uint32_t total = s_off[nb_tile];                              // bytes of this tile
    const uint32_t end = a + total;
    const uint32_t mid_lo = a ? 16u : 0u;                               // s_stage offsets of the 16-byte aligned middle [mid_lo, mid_hi)
    const uint32_t mid_hi = end & ~15u;
    const bool have_mid = mid_hi > mid_lo;
    uint8_t* const gbase = gdst - a;                                    // 16-byte aligned
    if (have_mid && tid == 0) bulk_store_smem_to_global(gbase + mid_lo, s_stage + mid_lo, mid_hi - mid_lo);
    // ragged edges: [a, head_hi) in front of the middle and [mid_hi, end) behind it (everything when there is no aligned middle)
    const uint32_t head_hi = have_mid ? mid_lo : end;
    if (tid >= 32 && tid < 64) {
        for (uint32_t o = a + 2 * (tid - 32); o < head_hi; o += 64) {
            if (o + 2 <= head_hi) st_u16(gbase + o, *reinterpret_cast<const uint16_t*>(s_stage + o));
            else gbase[o] = s_stage[o];
        }
    }
    if (have_mid && tid >= 64 && tid < 96) {
        for (uint32_t o = mid_hi + 2 * (tid - 64); o < end; o += 64) {
            if (o + 2 <= end) st_u16(gbase + o, *reinterpret_cast<const uint16_t*>(s_stage + o));
            else gbase[o] = s_stage[o];
        }
    }
}

__global__ void cham_status_accumulate_k(const Status* __restrict__ st, uint32_t* __restrict__ flag) {
    if (st->nonquiet || st->error) *flag = 1;
}
__global__ void cham_table_init_k(uint32_t* __restrict__ t) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 65536) t[i] = (i == 0) ? 0x10000u : 0u;  // stream start: bucket 0 "holds quad 0" (chameleon.rs:41,89-91)
}
__global__ void cham_table_fold_k(uint32_t* __restrict__ acc, const uint32_t* __restrict__ next) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 65536) { uint32_t v = next[i]; if (v & 0x10000u) acc[i] = v; }
}

// the dictionary as the reference keeps it (one quad per bucket, zero = never written unless it is bucket 0) <-> touched | fingerprint
__global__ void cham_quads_to_table_k(const uint32_t* __restrict__ quads, uint32_t* __restrict__ t) {
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= 65536) return;
    const uint32_t v = quads[h];
    const uint32_t p = hash_prod(v);
    t[h] = (prod_hash(p) == h) ? (0x10000u | prod_fp(p, v)) : 0u;   // a slot only ever holds a quad of its own bucket (chameleon.rs:95) or the initial 0
}
__global__ void cham_table_into_quads_k(const uint32_t* __restrict__ t, uint32_t* __restrict__ quads) {
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= 65536) return;
    const uint32_t v = t[h];
    if (v & 0x10000u) quads[h] = quad_from_hf(h, v & 0xFFFFu);
}

// carry-in dictionary of shard `rank` = left fold of the last-writer tables of the shards before it over the stream-start state
// (one kernel for the whole fold; `tables` = [world][65536] as gathered over NVLink)
__global__ void cham_rank_fold_k(const uint32_t* __restrict__ tables, uint32_t rank, uint32_t* __restrict__ carry) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 65536) return;
    uint32_t c = (i == 0) ? 0x10000u : 0u;            // stream start: bucket 0 "holds quad 0" (chameleon.rs:41,89-91)
    for (uint32_t r = 0; r < rank; ++r) { const uint32_t v = tables[(size_t)r * 65536 + i]; if (v & 0x10000u) c = v; }
    carry[i] = c;
}
// what a shard tells the others after its phase 2: {first block incompressible, last block incompressible, not quiet or error, 0, size}
__global__ void cham_seam_words_k(const uint32_t* __restrict__ sigw_g, uint64_t nbytes, uint64_t nblocks, const Status* __restrict__ st,
                                  const uint64_t* __restrict__ d_out_size, uint32_t* __restrict__ words /* 8 x u32 */) {
    if (threadIdx.x || blockIdx.x) return;
    auto inc = [&](uint64_t b) { return (nbytes - b * 256 >= 256) && (__popc(sigw_g[2 * b]) + __popc(sigw_g[2 * b + 1]) <= 4); };
    words[0] = nblocks ? (inc(0) ? 1u : 0u) : 0u;
    words[1] = nblocks ? (inc(nblocks - 1) ? 1u : 0u) : 0u;
    words[2] = (nblocks && (st->nonquiet || st->error)) ? 1u : 0u;
    words[3] = nblocks ? 1u : 0u;                        // the shard has blocks at all
    const uint64_t sz = *d_out_size;
    words[4] = (uint32_t)sz; words[5] = (uint32_t)(sz >> 32); words[6] = 0; words[7] = 0;
}
// all ranks evaluate the same thing: the stream is quiet iff every shard is and no seam joins two incompressible blocks
// (protection_state.rs:38-43 across the cut); also the stream length and this rank's offset in it
__global__ void cham_seam_verdict_k(const uint32_t* __restrict__ all_words, uint32_t world, uint32_t rank, uint32_t* __restrict__ d_flags,
                                    uint64_t* __restrict__ d_total, uint64_t* __restrict__ d_sizes /* world + 1: offsets */) {
    if (threadIdx.x || blockIdx.x) return;
    uint32_t bad = 0, prev_inc = 0; uint64_t off = 0;
    for (uint32_t r = 0; r < world; ++r) {
        const uint32_t* w = all_words + 8 * r;
        if (w[2]) bad = 1;
        if (w[3]) { if (prev_inc && w[0]) bad = 1; prev_inc = w[1]; }
        if (d_sizes) d_sizes[r] = off;
        off += (uint64_t)w[4] | ((uint64_t)w[5] << 32);
    }
    if (d_sizes) d_sizes[world] = off;
    if (d_flags) *d_flags = bad;
    if (d_total) *d_total = off;
    (void)rank;
}

// ------------------------------------------------------------------------------------------------------
// Sharded copy-map iteration (include/density_b200.h density_b200_shard_prot_*, DESIGN.md section 5). Each shard runs the rounds of
// prot_iterate's fixed point on its own blocks, with the automaton state carried over the cuts: per round it exports its TRANSFER
// (candidate state at the shard start -> candidate state at the shard end, or PC_ESC; the candidates of pc_encode), every shard composes
// the transfers of the shards before it from the canonical state, walks its blocks from that true incoming state and reports round words
// {blocks whose copy status changed, met PC_ESC, the iteration had settled before this round, 0}. The verdict over all shards' words is
// the same on every shard: settled when no block changed anywhere and no path met PC_ESC. ps->first_block makes `counter` global:
// revert_to_copy halves the start on every 16th block of the STREAM, and shards start at any block.
// The kernels serve every codec: Chameleon refreshes the incompressible bits from its signatures inside cham_prot_seg_k (sigw_g), Cheetah
// and Lion pass sigw_g == nullptr with the bits already refreshed by their tile-size kernels; blocks are 256, 128 or 64 bytes.
// ------------------------------------------------------------------------------------------------------
constexpr uint32_t PROT_REFUSED = 16;   // Status::error of a shard whose iteration did not settle (or met PC_ESC): nothing is emitted

__global__ void cham_put_u64_k(uint64_t* __restrict__ p, uint64_t v) { if (threadIdx.x == 0 && blockIdx.x == 0) *p = v; }
__global__ void cham_prot_start_k(Status* __restrict__ st, ProtShard* __restrict__ ps, uint64_t first_block, const uint64_t* __restrict__ lengths,
                                  uint32_t rank, uint32_t block_bytes) {
    if (threadIdx.x || blockIdx.x) return;
    if (lengths) { uint64_t o = 0; for (uint32_t r = 0; r < rank; ++r) o += lengths[r]; first_block = o / block_bytes; }
    *ps = ProtShard{};
    ps->first_block = first_block;
    ps->stage_ok = 1;
    st->nonquiet = 1;        // the copy map is always in force on this path: every round's kernels run until the global verdict closes them
    st->converged = 0;
}

// segment s: refresh the incompressible bits of its blocks (prot_iterate step 1), then walk it from every candidate state at once, one
// candidate per thread; the paths merge quickly (the start halves every 16 blocks, a penalty decays), and once they all agree one thread
// walks the rest of the segment.
__global__ void __launch_bounds__(PSEG)
cham_prot_seg_k(const uint32_t* __restrict__ sigw_g, uint64_t nbytes, uint64_t nblocks, uint32_t nseg, const Status* __restrict__ st, int it,
                uint8_t* __restrict__ inc, const uint8_t* __restrict__ cm_old, const ProtShard* __restrict__ ps, uint16_t* __restrict__ T) {
    if (!gate_open(st)) return;
    __shared__ uint8_t s_inc[PSEG];
    __shared__ uint32_t s_ref;
    const uint32_t tid = threadIdx.x;
    for (uint32_t seg = blockIdx.x; seg < nseg; seg += gridDim.x) {   // a bounded grid: the settled rounds launch it for nothing
    const uint64_t b0 = (uint64_t)seg * PSEG;
    const uint32_t nb = (uint32_t)((nblocks - b0 < (uint64_t)PSEG) ? (nblocks - b0) : PSEG);
    if (tid < nb) {
        const uint64_t b = b0 + tid;
        if (sigw_g && !(it && cm_old[b])) inc[b] = (nbytes - b * 256 >= 256) && (__popc(sigw_g[2 * b]) + __popc(sigw_g[2 * b + 1]) <= 4);
        s_inc[tid] = inc[b];
    }
    __syncthreads();
    Protection p; pc_decode(tid < PC_NC ? tid : 0u, p);
    p.counter = ps->first_block + b0;
    uint32_t k = 0;
    while (k < nb) {                                               // CTA-uniform
        const uint32_t k1 = (k + 16 < nb) ? k + 16 : nb;
        for (; k < k1; ++k) { if (p.revert_to_copy()) p.decay(); else p.update(s_inc[k] != 0); }
        if (tid == 0) s_ref = prot_pack(p);
        __syncthreads();
        if (__syncthreads_and(prot_pack(p) == s_ref)) break;
    }
    if (k < nb) {
        if (tid == 0) {
            for (; k < nb; ++k) { if (p.revert_to_copy()) p.decay(); else p.update(s_inc[k] != 0); }
            s_ref = pc_encode(p);
        }
        __syncthreads();
        if (tid < PC_NC) T[(size_t)seg * PC_NC + tid] = (uint16_t)s_ref;
    } else if (tid < PC_NC) {
        T[(size_t)seg * PC_NC + tid] = (uint16_t)pc_encode(p);
    }
    __syncthreads();                                               // s_inc and s_ref are reused by the next segment
    }
}

// group tables (as prot_iterate's GT) and the shard's transfer: the group tables composed in order for every candidate
__global__ void cham_prot_groups_k(uint32_t nseg, const Status* __restrict__ st, const uint16_t* __restrict__ T, uint16_t* __restrict__ GT) {
    if (!gate_open(st)) return;
    const uint32_t ngrp = (nseg + PC_GROUP - 1) / PC_GROUP;
    const uint64_t idx = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (uint64_t)ngrp * PC_NC) return;
    const uint32_t g = (uint32_t)(idx / PC_NC);
    uint32_t x = (uint32_t)(idx % PC_NC);
    const uint32_t s1 = ((g + 1) * PC_GROUP < nseg) ? (g + 1) * PC_GROUP : nseg;
    for (uint32_t s = g * PC_GROUP; s < s1 && x != PC_ESC; ++s) x = T[(size_t)s * PC_NC + x];
    GT[idx] = (uint16_t)x;
}
__global__ void cham_prot_transfer_k(uint32_t nseg, const Status* __restrict__ st, const uint16_t* __restrict__ GT, uint32_t* __restrict__ out) {
    if (!gate_open(st)) return;
    const uint32_t c = threadIdx.x;
    if (c >= PC_NC) return;
    const uint32_t ngrp = (nseg + PC_GROUP - 1) / PC_GROUP;
    uint32_t x = c;                                                // an empty shard is the identity
    for (uint32_t g = 0; g < ngrp && x != PC_ESC; ++g) x = GT[(size_t)g * PC_NC + x];
    out[c] = x;
}

// settle, 1: the true incoming state (the transfers of the shards before `rank` composed from the canonical state), the incoming state
// of every group, and this round's words (written whether or not the gate is open, so that every gathered word is this round's)
__global__ void cham_prot_enter_k(const uint32_t* __restrict__ all_transfers, uint32_t rank, uint32_t nseg, const Status* __restrict__ st,
                                  const uint16_t* __restrict__ GT, uint32_t* __restrict__ gin, ProtShard* __restrict__ ps,
                                  uint32_t* __restrict__ words) {
    if (threadIdx.x || blockIdx.x) return;
    const bool open = gate_open(st);
    words[0] = 0; words[1] = 0; words[2] = open ? 0u : 1u; words[3] = 0;
    if (!open) return;
    uint32_t x = 0;                                                // canonical state: penalty 0, start 1, not incompressible
    for (uint32_t r = 0; r < rank && x != PC_ESC; ++r) x = all_transfers[(size_t)r * PC_NC + x];
    ps->in_state = x;
    const uint32_t ngrp = (nseg + PC_GROUP - 1) / PC_GROUP;
    for (uint32_t g = 0; g < ngrp; ++g) { gin[g] = x; if (x != PC_ESC) x = GT[(size_t)g * PC_NC + x]; }
    gin[ngrp] = x;
    if (x == PC_ESC) words[1] = 1;
}
// settle, 2: the incoming state of every segment
__global__ void cham_prot_seams_k(uint32_t nseg, const Status* __restrict__ st, const uint16_t* __restrict__ T, const uint32_t* __restrict__ gin,
                                  uint32_t* __restrict__ in_state) {
    if (!gate_open(st)) return;
    const uint32_t ngrp = (nseg + PC_GROUP - 1) / PC_GROUP;
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= ngrp || gin[ngrp] == PC_ESC) return;
    uint32_t x = gin[g];
    const uint32_t s1 = ((g + 1) * PC_GROUP < nseg) ? (g + 1) * PC_GROUP : nseg;
    for (uint32_t s = g * PC_GROUP; s < s1; ++s) { in_state[s] = x; x = T[(size_t)s * PC_NC + x]; }
}
// settle, 3: every segment walked from its true incoming state writes the new copy map; the blocks whose status changed are counted
// against the committed map, or in round 0 against the empty one unless `warm` (the map the round's flags were computed under is then
// the committed one from the start)
__global__ void cham_prot_walk_k(uint64_t nblocks, uint32_t nseg, const Status* __restrict__ st, int it, int warm, const uint8_t* __restrict__ inc,
                                 const uint8_t* __restrict__ cm_old, uint8_t* __restrict__ cm_new, const uint32_t* __restrict__ in_state,
                                 const uint32_t* __restrict__ gin, ProtShard* __restrict__ ps, uint32_t* __restrict__ words) {
    if (!gate_open(st)) return;
    const uint32_t ngrp = (nseg + PC_GROUP - 1) / PC_GROUP;
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= nseg || gin[ngrp] == PC_ESC) return;
    Protection p; pc_decode(in_state[s], p);
    const uint64_t b0 = (uint64_t)s * PSEG, b1 = (b0 + PSEG < nblocks) ? b0 + PSEG : nblocks;
    p.counter = ps->first_block + b0;
    prot_walk(p, inc, b0, b1, cm_new);
    uint32_t nd = 0;
    for (uint64_t b = b0; b < b1; ++b) nd += cm_new[b] != ((it || warm) ? cm_old[b] : 0);
    if (nd) {
        atomicAdd(&words[0], nd);
        if (it < 16) atomicAdd(&ps->changed[it], nd);
    }
}

// all_words: [world][stride] round words, {changed, met PC_ESC, ...} at the front of every row
__device__ __forceinline__ void prot_round_verdict(const uint32_t* all_words, uint32_t world, uint32_t stride, bool& changed, bool& esc) {
    changed = false; esc = false;
    for (uint32_t r = 0; r < world; ++r) { changed |= all_words[stride * r] != 0; esc |= all_words[stride * r + 1] != 0; }
}
// the global commit of a round, 1: cm_old <- cm_new unless the map settled (as prot_iterate step 4; round 0 always commits)
__global__ void cham_prot_commit_k(const uint32_t* __restrict__ all_words, uint32_t world, uint32_t stride, uint64_t nblocks, const Status* __restrict__ st,
                                   int it, uint8_t* __restrict__ cm_old, const uint8_t* __restrict__ cm_new) {
    if (!gate_open(st)) return;
    bool changed, esc;
    prot_round_verdict(all_words, world, stride, changed, esc);
    if (esc || !(changed || it == 0)) return;
    for (uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; b < nblocks; b += (uint64_t)gridDim.x * blockDim.x) cm_old[b] = cm_new[b];
}
// 2: the verdict closes the gate of every later kernel when the map has settled, or when a path met PC_ESC (the shard is then refused)
__global__ void cham_prot_verdict_k(const uint32_t* __restrict__ all_words, uint32_t world, uint32_t stride, Status* __restrict__ st, int it,
                                    ProtShard* __restrict__ ps) {
    if (threadIdx.x || blockIdx.x || !gate_open(st)) return;
    bool changed, esc;
    prot_round_verdict(all_words, world, stride, changed, esc);
    if (esc) { ps->esc = 1; st->converged = 1; }
    else if (!changed) { ps->settled = 1; ps->rounds = (uint32_t)it + 1; st->converged = 1; }
}
// finish: a shard whose iteration did not settle, or whose own staged iteration did not (Cheetah / Lion: the shard at the stream start), is
// refused (nothing is emitted: the emit kernels return on an error)
__global__ void cham_prot_finish_k(Status* __restrict__ st, const ProtShard* __restrict__ ps) {
    if (threadIdx.x || blockIdx.x) return;
    if (!ps->settled || !ps->stage_ok) st->error = PROT_REFUSED;
}
// the seam words of the layout of cham_seam_words_k: incompressible blocks may meet at a cut here, so words 0 and 1 stay 0; word 2 = refused
// or error (the size is then 0)
__global__ void cham_prot_seam_words_k(uint64_t nblocks, const Status* __restrict__ st, uint64_t* __restrict__ d_out_size, uint32_t* __restrict__ words) {
    if (threadIdx.x || blockIdx.x) return;
    const uint64_t sz = (nblocks && !st->error) ? *d_out_size : 0;
    *d_out_size = sz;
    words[0] = 0; words[1] = 0; words[2] = st->error ? 1u : 0u; words[3] = nblocks ? 1u : 0u;
    words[4] = (uint32_t)sz; words[5] = (uint32_t)(sz >> 32); words[6] = 0; words[7] = 0;
}

}  // namespace cham

// ------------------------------------------------------------------------------------------------------
// host-side launch sequence
// ------------------------------------------------------------------------------------------------------
using namespace cham;

size_t cham_workspace_bytes(size_t nbytes, int nruns_max, ChamLayout* L) {
    const uint64_t nblocks = (nbytes + 255) / 256;
    const uint64_t ntiles = (nblocks + 63) / 64;
    const uint64_t ngroups = (ntiles + SCAN_G - 1) / SCAN_G;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
    L->status = take(sizeof(Status));
    L->sigw = take((ntiles * 64 * 2 + 64 + 256) * sizeof(uint32_t));   // + one 64-block tile: the flag pass works in 128-block tiles
    L->copymap = take(ntiles * 64 + 64 + 128);
    L->copymap2 = take(ntiles * 64 + 64 + 128);
    L->seg_state = take(prot_state_bytes(ntiles * 64 / PSEG + 2));
    L->incb = take(ntiles * 64 + 64);
    L->tile_bytes = take((ntiles + 1) * sizeof(uint32_t));
    L->tile_local = take((ntiles + 1) * sizeof(uint32_t));
    L->group_total = take((ngroups + 1) * sizeof(uint64_t));
    L->group_off = take((ngroups + 1) * sizeof(uint64_t));
    L->unres = take((size_t)nruns_max * 65536 * sizeof(uint2));
    L->unres_count = take((size_t)nruns_max * sizeof(uint32_t));
    L->final_tab = take((size_t)nruns_max * 65536 * sizeof(uint32_t));
    L->carry = take((size_t)nruns_max * 65536 * sizeof(uint32_t));
    L->total = off;
    return off;
}

static cudaError_t set_smem_attrs_once() {
    static bool done = false;
    static cudaError_t err = cudaSuccess;
    if (!done) {
        err = cudaFuncSetAttribute(cham_flag_pass6, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Flag6Smem));
        if (err == cudaSuccess)
            err = cudaFuncSetAttribute(cham_protected_pass, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ProtSmem));
        done = true;
    }
    return err;
}

static cudaError_t prot_iterate_coop(int ctas, cudaStream_t stream, const uint32_t* sigw, uint64_t nbytes, uint64_t nblocks, uint32_t nseg, Status* st, int it,
                                     uint8_t* inc, uint8_t* cm_old, uint8_t* cm_new, uint32_t* in_state, uint32_t* out_state, uint16_t* ptab) {
    void* args[] = {&sigw, &nbytes, &nblocks, &nseg, &st, &it, &inc, &cm_old, &cm_new, &in_state, &out_state, &ptab};
    return cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(prot_iterate), dim3((unsigned)ctas), dim3(PI_THREADS), args, 0, stream);
}

cudaError_t prot_debug_read(unsigned long long* out32) { return cudaMemcpyFromSymbol(out32, g_prot_dbg, sizeof(unsigned long long) * 32); }

size_t prot_state_bytes(uint64_t nseg_max) { return (2 * (nseg_max + 2) + 64) * sizeof(uint32_t) + prot_table_elems(nseg_max) * sizeof(uint16_t); }

uint32_t cham_pick_runs(size_t nbytes, int num_sms) {
    const uint64_t nblocks = (nbytes + 255) / 256;
    const uint64_t ntiles = (nblocks + 63) / 64;
    // at least 16 tiles (256 KiB) per run so that first-touch traffic stays small
    uint64_t r = ntiles / 16;
    if (r < 1) r = 1;
    if (r > (uint64_t)num_sms) r = num_sms;
    return (uint32_t)r;
}

// One encode call's view of its workspace: the geometry of its `nbytes` and typed pointers to the arrays of ChamLayout. The segment
// states and candidate tables of the copy-map iteration sit in the seg_state region, in prot_iterate's layout: in_state [nseg + 1],
// out_state [nseg + 1] (unused by the sharded iteration), then ptab: gin [ngrp + 2] (as u32), T [nseg][PC_NC], GT [ngrp][PC_NC] (u16).
struct ChamBufs {
    size_t nbytes; uint64_t nquads, nblocks; uint32_t ntiles, ngroups, nseg, ngrp;
    Status* st; uint32_t* sigw; uint8_t *copymap, *copymap2, *incb; uint32_t *seg_state, *tile_bytes, *tile_local; uint64_t *group_total, *group_off;
    uint2* unres; uint32_t *unres_count, *final_tab, *carry;
    uint32_t *in_state, *out_state, *gin; uint16_t *ptab, *T, *GT;
    template <class X> static X* at(uint8_t* ws, size_t off) { return reinterpret_cast<X*>(ws + off); }
    ChamBufs(uint8_t* ws, const ChamLayout& L, size_t n) {
        nbytes = n; nquads = n / 4; nblocks = (n + 255) / 256;
        ntiles = (uint32_t)((nblocks + 63) / 64); ngroups = (ntiles + SCAN_G - 1) / SCAN_G;
        nseg = (uint32_t)((nblocks + PSEG - 1) / PSEG); ngrp = (nseg + PC_GROUP - 1) / PC_GROUP;
        st = at<Status>(ws, L.status); sigw = at<uint32_t>(ws, L.sigw);
        copymap = ws + L.copymap; copymap2 = ws + L.copymap2; incb = ws + L.incb;
        seg_state = at<uint32_t>(ws, L.seg_state);
        tile_bytes = at<uint32_t>(ws, L.tile_bytes); tile_local = at<uint32_t>(ws, L.tile_local);
        group_total = at<uint64_t>(ws, L.group_total); group_off = at<uint64_t>(ws, L.group_off);
        unres = at<uint2>(ws, L.unres); unres_count = at<uint32_t>(ws, L.unres_count);
        final_tab = at<uint32_t>(ws, L.final_tab); carry = at<uint32_t>(ws, L.carry);
        in_state = seg_state; out_state = seg_state + (nseg + 1);
        ptab = reinterpret_cast<uint16_t*>(seg_state + 2 * (nseg + 1));
        gin = reinterpret_cast<uint32_t*>(ptab); T = ptab + 2 * (ngrp + 2); GT = T + (size_t)nseg * PC_NC;
    }
};

// ---- the launches that more than one path makes. `gate` (may be nullptr = always): the kernels return at once unless the quiet check
// failed and the copy map has not settled yet.
// flags of every run, with the blocks of `copymap` (may be nullptr) hidden from the dictionary
static void launch_flag_pass(const ChamBufs& B, const uint8_t* d_in, uint32_t nruns, const uint8_t* copymap, const Status* gate, cudaStream_t stream,
                             uint64_t* launches) {
    cham_flag_pass6<<<nruns, F6_THREADS, sizeof(Flag6Smem), stream>>>(reinterpret_cast<const uint32_t*>(d_in), B.nquads, B.ntiles, nruns, B.sigw, B.unres,
                                                                      B.unres_count, B.final_tab, copymap, gate);
    ++*launches;
}
// the table carried into every run (d_carry_in before the first; nullptr = stream start), then the first-touch flags resolved against it
static void launch_carry_resolve(const ChamBufs& B, uint32_t nruns, const uint32_t* d_carry_in, const Status* gate, cudaStream_t stream,
                                 uint64_t* launches) {
    cham_carry_scan<<<65536 / 256, 256, 0, stream>>>(B.final_tab, d_carry_in, 0, nruns, B.carry, nullptr, gate);
    cham_resolve<<<dim3(32, nruns), 256, 0, stream>>>(B.unres, B.unres_count, B.carry, B.ntiles, nruns, B.sigw, gate);
    *launches += 2;
}
// export: the fold of the runs' last-writer tables with "nothing touched" as the initial state
static void launch_export_fold(const ChamBufs& B, uint32_t nruns, uint32_t* d_table_out, const Status* gate, cudaStream_t stream, uint64_t* launches) {
    cham_carry_scan<<<65536 / 256, 256, 0, stream>>>(B.final_tab, nullptr, 1, nruns, nullptr, d_table_out, gate);
    ++*launches;
}
// Sizes under `copymap` (nullptr: the sizes of cham_phase2_begin stand, and no block is copied), scan, emit. use_copymap_if_nonquiet:
// the map counts only if the quiet check failed (the in-order encode passes 0: its map always counts). The emit kernel that loads 16
// bytes at a time runs when `al16_ok` and the input is so aligned; the in-order encode has always taken the other one.
static cudaError_t sizes_scan_emit(const ChamBufs& B, const uint8_t* d_in, const uint8_t* copymap, int use_copymap_if_nonquiet, bool al16_ok,
                                   uint8_t* d_out, size_t cap, uint64_t* d_out_size, cudaStream_t stream, uint64_t* launches, cudaEvent_t* ev) {
    if (copymap) {
        cham_tile_sizes<<<(B.ntiles + 7) / 8, 256, 0, stream>>>(B.sigw, copymap, B.nbytes, B.nblocks, B.ntiles, use_copymap_if_nonquiet, 0, 0, B.st, B.tile_bytes);
        ++*launches;
    }
    cudaError_t e = scan_tiles_launch(B.tile_bytes, B.ntiles, B.tile_local, B.group_total, B.group_off, B.ngroups, B.st, (uint64_t)cap, d_out_size, stream);
    if (e != cudaSuccess) return e;
    *launches += 2;
    if (ev) cudaEventRecord(ev[2], stream);
    const uint32_t* in32 = reinterpret_cast<const uint32_t*>(d_in);
    if (al16_ok && (reinterpret_cast<uintptr_t>(d_in) & 15u) == 0)
        cham_emit<true><<<B.ntiles, EM_THREADS, 0, stream>>>(in32, B.nbytes, B.nblocks, B.sigw, copymap, use_copymap_if_nonquiet, B.st, B.tile_local, B.group_off, d_out);
    else
        cham_emit<false><<<B.ntiles, EM_THREADS, 0, stream>>>(in32, B.nbytes, B.nblocks, B.sigw, copymap, use_copymap_if_nonquiet, B.st, B.tile_local, B.group_off, d_out);
    ++*launches;
    if (ev) cudaEventRecord(ev[3], stream);
    return cudaGetLastError();
}

// Phase 1 of the encode: flag pass over all runs + fold of the last-writer tables.
cudaError_t cham_encode_phase1(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, uint32_t nruns,
                               uint32_t* d_table_out, cudaStream_t stream, uint64_t* launches, cudaEvent_t* ev) {
    cudaError_t e = set_smem_attrs_once();
    if (e != cudaSuccess) return e;
    const ChamBufs B(ws, L, nbytes);
    e = cudaMemsetAsync(B.st, 0, sizeof(Status), stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(&B.st->first_nonquiet_block, 0xFF, sizeof(unsigned long long), stream);   // it starts at ~0
    if (e != cudaSuccess) return e;
    if (B.nblocks == 0) return cudaSuccess;
    if (ev) cudaEventRecord(ev[0], stream);
    launch_flag_pass(B, d_in, nruns, nullptr, nullptr, stream, launches);
    if (ev) cudaEventRecord(ev[1], stream);
    if (d_table_out) launch_export_fold(B, nruns, d_table_out, nullptr, stream, launches);   // a shard's table
    return cudaGetLastError();
}

// Phase 2: carry-in tables, resolve, sizes, scan, (protected fallback), emit.
// Phase 2 in three parts, so that a caller that may synchronise with the host (the reference-facing entry points do anyway) can run
// further rounds of the copy-map iteration instead of dropping to the in-order walk when PROT_ITERS rounds were not enough
// (chains of copy-mode episodes that feed each other through the dictionary, e.g. the same incompressible blob several times).
//   begin : carry-in tables, first-touch flags, block sizes + quiet check
//   rounds: fixed-point rounds it_first .. it_last of the copy map (every kernel exits at once unless the quiet check failed and the
//           map has not settled yet); prot_iterate owns 8 grid-barrier slots, so a batch is at most 8 rounds and `reset_barriers`
//           clears them first
//   finish: the exact in-order walk if the map still has not settled (optional), sizes under the copy map, scan, emit
static cudaError_t cham_phase2_begin(const ChamBufs& B, uint32_t nruns, const uint32_t* d_carry_in, bool assume_prev_inc, cudaStream_t stream,
                                     uint64_t* launches) {
    launch_carry_resolve(B, nruns, d_carry_in, nullptr, stream, launches);
    cham_tile_sizes<<<(B.ntiles + 7) / 8, 256, 0, stream>>>(B.sigw, nullptr, B.nbytes, B.nblocks, B.ntiles, 0, 1, assume_prev_inc ? 1 : 0, B.st, B.tile_bytes);
    ++*launches;
    return cudaGetLastError();
}

static cudaError_t cham_phase2_rounds(const ChamBufs& B, const uint8_t* d_in, uint32_t nruns, const uint32_t* d_carry_in, int it_first, int it_last,
                                      bool reset_barriers, int num_sms, cudaStream_t stream, uint64_t* launches) {
    const int num_ctas = num_sms > 0 ? num_sms : 1;   // one CTA per SM
    if (it_last - it_first >= 8) return cudaErrorInvalidValue;
    if (reset_barriers) {
        cudaError_t e = cudaMemsetAsync(B.st->barrier, 0, sizeof(B.st->barrier), stream);
        if (e != cudaSuccess) return e;
    }
    for (int it = it_first; it <= it_last; ++it) {
        if (it > 0) {   // flags under the current copy map (copy-mode blocks hidden from the dictionary)
            launch_flag_pass(B, d_in, nruns, B.copymap, B.st, stream, launches);
            launch_carry_resolve(B, nruns, d_carry_in, B.st, stream, launches);
        }
        // cooperative launch: the software grid barriers need every CTA resident (the runtime checks it instead of a hang)
        cudaError_t le = prot_iterate_coop(num_ctas, stream, B.sigw, B.nbytes, B.nblocks, B.nseg, B.st, it, B.incb, B.copymap, B.copymap2, B.in_state,
                                           B.out_state, B.ptab);
        if (le != cudaSuccess) return le;
        ++*launches;
    }
    return cudaGetLastError();
}

static cudaError_t cham_phase2_finish(const ChamBufs& B, const uint8_t* d_in, uint8_t* d_out, size_t cap, uint64_t* d_out_size, bool with_copy_map,
                                      bool inorder_fallback, cudaStream_t stream, uint64_t* launches, cudaEvent_t* ev) {
    if (with_copy_map && inorder_fallback) {   // the exact in-order walk if the iteration did not settle
        cham_protected_pass<<<1, 1024, sizeof(ProtSmem), stream>>>(reinterpret_cast<const uint32_t*>(d_in), B.nbytes, B.st, 1, B.sigw, B.copymap);
        ++*launches;
    }
    return sizes_scan_emit(B, d_in, with_copy_map ? B.copymap : nullptr, 1, true, d_out, cap, d_out_size, stream, launches, ev);
}

// host-visible verdict of the iteration so far (synchronises the stream): 0 quiet or settled, 1 more rounds needed
static cudaError_t cham_phase2_needs_more(const ChamBufs& B, cudaStream_t stream, bool* more) {
    Status h;
    cudaError_t e = cudaMemcpyAsync(&h, B.st, sizeof h, cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return e;
    *more = h.nonquiet && !h.converged && !h.error;
    return cudaSuccess;
}

constexpr int PROT_ITERS = 4;   // rounds 0..4 are always enqueued (they cost ~3 us each when the input is quiet)

// What the callers of phase 2 choose.
struct Phase2Opts {
    const uint32_t* d_carry_in = nullptr;   // the dictionary carried in (nullptr = stream start)
    bool assume_prev_inc = false;           // count the block before the first as incompressible
    bool iterate = true;                    // run the copy-map iteration; false: no copy map, the sizes of `begin` stand
    int max_batches = 0;                    // after the standard rounds the host looks at the verdict (synchronising) and keeps iterating in
                                            // up to this many batches of rounds 8..15
    bool inorder_walk = true;               // the in-order walk settles a map that the rounds did not
    bool* give_up = nullptr;                // set: a map still unsettled after the batches means no emit and *give_up = true
    uint32_t* d_table_out = nullptr;        // set: export the last-writer table under the final copy map
    cudaEvent_t* ev = nullptr;              // stage events 2 and 3
};

static cudaError_t cham_phase2(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, uint32_t nruns, uint8_t* d_out, size_t cap,
                               uint64_t* d_out_size, const Phase2Opts& o, int num_sms, cudaStream_t stream, uint64_t* launches) {
    if (nbytes == 0) return cudaMemsetAsync(d_out_size, 0, sizeof(uint64_t), stream);
    const ChamBufs B(ws, L, nbytes);
    cudaError_t e = cham_phase2_begin(B, nruns, o.d_carry_in, o.assume_prev_inc, stream, launches);
    if (e == cudaSuccess && o.iterate) e = cham_phase2_rounds(B, d_in, nruns, o.d_carry_in, 0, PROT_ITERS, false, num_sms, stream, launches);
    // A caller that leaves the rest to the in-order walk does not look at the verdict after its last batch; one that gives up looks once
    // more, so that `more` is the verdict of the last batch.
    bool more = false;
    const int looks = o.max_batches + (o.give_up ? 1 : 0);
    for (int batch = 0; e == cudaSuccess && batch < looks; ++batch) {
        e = cham_phase2_needs_more(B, stream, &more);
        if (e != cudaSuccess || !more || batch >= o.max_batches) break;
        e = cham_phase2_rounds(B, d_in, nruns, o.d_carry_in, 8, 15, true, num_sms, stream, launches);
    }
    if (e != cudaSuccess) return e;
    if (o.give_up && more) { *o.give_up = true; return cudaSuccess; }
    e = cham_phase2_finish(B, d_in, d_out, cap, d_out_size, o.iterate, o.inorder_walk, stream, launches, o.ev);
    if (e == cudaSuccess && o.d_table_out) {
        launch_export_fold(B, nruns, o.d_table_out, nullptr, stream, launches);
        e = cudaGetLastError();
    }
    return e;
}

// Everything enqueued, no host synchronisation: rounds 0..PROT_ITERS, then the in-order walk if they were not enough.
cudaError_t cham_encode_phase2(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, uint32_t nruns,
                               const uint32_t* d_carry_in, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                               bool allow_protected_fallback, bool assume_prev_inc, int num_sms, cudaStream_t stream, uint64_t* launches,
                               cudaEvent_t* ev) {
    Phase2Opts o;
    o.d_carry_in = d_carry_in; o.assume_prev_inc = assume_prev_inc; o.iterate = allow_protected_fallback; o.ev = ev;
    return cham_phase2(d_in, nbytes, ws, L, nruns, d_out, cap, d_out_size, o, num_sms, stream, launches);
}

// Same result, for callers that may block: after the standard rounds the host looks at the verdict and keeps iterating in batches of 8
// rounds (up to `max_batches`) before the in-order walk is allowed to take over.
cudaError_t cham_encode_phase2_blocking(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, uint32_t nruns, uint8_t* d_out,
                                        size_t cap, uint64_t* d_out_size, int max_batches, int num_sms, cudaStream_t stream, uint64_t* launches) {
    Phase2Opts o;
    o.max_batches = max_batches;
    return cham_phase2(d_in, nbytes, ws, L, nruns, d_out, cap, d_out_size, o, num_sms, stream, launches);
}

// Phase 2 for a reused Codec instance: dictionary carried in, copy map by host-resumed iteration; when it does not settle nothing is
// emitted and *ok = false (the caller runs the in-order kernel on the instance's state instead). On success d_table_out = this call's
// last-writer table under the final copy map (copy-mode blocks never reach the dictionary, codec.rs:35-37).
cudaError_t cham_encode_phase2_stream(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, uint32_t nruns, const uint32_t* d_carry_in,
                                      uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint32_t* d_table_out, int max_batches, int num_sms,
                                      cudaStream_t stream, uint64_t* launches, bool* ok) {
    bool gave_up = false;
    Phase2Opts o;
    o.d_carry_in = d_carry_in; o.max_batches = max_batches; o.inorder_walk = false; o.give_up = &gave_up; o.d_table_out = d_table_out;
    const cudaError_t e = cham_phase2(d_in, nbytes, ws, L, nruns, d_out, cap, d_out_size, o, num_sms, stream, launches);
    *ok = !gave_up;
    return e;
}
cudaError_t cham_quads_to_table(const uint32_t* d_quads, uint32_t* d_table, cudaStream_t stream, uint64_t* launches) {
    cham_quads_to_table_k<<<65536 / 256, 256, 0, stream>>>(d_quads, d_table);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t cham_table_into_quads(const uint32_t* d_table, uint32_t* d_quads, cudaStream_t stream, uint64_t* launches) {
    cham_table_into_quads_k<<<65536 / 256, 256, 0, stream>>>(d_table, d_quads);
    ++*launches;
    return cudaGetLastError();
}

cudaError_t cham_status_accumulate(const uint8_t* ws, const ChamLayout& L, uint32_t* d_flag, cudaStream_t stream, uint64_t* launches) {
    cham_status_accumulate_k<<<1, 1, 0, stream>>>(reinterpret_cast<const Status*>(ws + L.status), d_flag);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t prot_iterate_launch(const uint32_t* sigw_or_null, uint64_t nbytes, uint64_t nblocks, uint32_t nseg, Status* st, int it, uint8_t* inc,
                                uint8_t* cm_old, uint8_t* cm_new, uint32_t* in_state, uint32_t* out_state, int num_sms, cudaStream_t stream) {
    int ctas = num_sms > 0 ? num_sms : 1;
    if ((uint32_t)ctas > nseg) ctas = nseg ? (int)nseg : 1;       // small inputs: cheaper grid barriers
    // the caller's state region is sized by prot_state_bytes(): the candidate tables live behind the 2 (nseg + 1) state words
    return prot_iterate_coop(ctas, stream, sigw_or_null, nbytes, nblocks, nseg, st, it, inc, cm_old, cm_new, in_state, out_state,
                             reinterpret_cast<uint16_t*>(out_state + (nseg + 1)));
}
cudaError_t scan_tiles_launch(const uint32_t* tile_bytes, uint32_t ntiles, uint32_t* tile_local, uint64_t* group_total, uint64_t* group_off,
                              uint32_t ngroups, Status* st, uint64_t cap, uint64_t* d_out_size, cudaStream_t stream) {
    scan_groups_local<<<ngroups, SCAN_T, 0, stream>>>(tile_bytes, ntiles, tile_local, group_total);
    scan_group_totals<<<1, SCAN_T, 0, stream>>>(group_total, ngroups, group_off, st, cap, d_out_size);
    return cudaGetLastError();
}
cudaError_t cham_rank_fold(const uint32_t* d_tables, uint32_t rank, uint32_t* d_carry, cudaStream_t stream, uint64_t* launches) {
    cham_rank_fold_k<<<65536 / 256, 256, 0, stream>>>(d_tables, rank, d_carry);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t cham_seam_words(const uint8_t* ws, const ChamLayout& L, size_t nbytes, const uint64_t* d_out_size, uint32_t* d_words, cudaStream_t stream, uint64_t* launches) {
    cham_seam_words_k<<<1, 1, 0, stream>>>(reinterpret_cast<const uint32_t*>(ws + L.sigw), nbytes, (nbytes + 255) / 256,
                                           reinterpret_cast<const Status*>(ws + L.status), d_out_size, d_words);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t cham_seam_verdict(const uint32_t* d_all_words, uint32_t world, uint32_t rank, uint32_t* d_flags, uint64_t* d_total, uint64_t* d_offsets,
                              cudaStream_t stream, uint64_t* launches) {
    cham_seam_verdict_k<<<1, 1, 0, stream>>>(d_all_words, world, rank, d_flags, d_total, d_offsets);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t cham_table_init(uint32_t* d_table, cudaStream_t stream, uint64_t* launches) {
    cham_table_init_k<<<65536 / 256, 256, 0, stream>>>(d_table);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t cham_table_fold(uint32_t* d_acc, const uint32_t* d_next, cudaStream_t stream, uint64_t* launches) {
    cham_table_fold_k<<<65536 / 256, 256, 0, stream>>>(d_acc, d_next);
    ++*launches;
    return cudaGetLastError();
}

// Exact sequential encode only (checker / forced fallback).
cudaError_t cham_encode_protected_only(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, uint8_t* d_out,
                                       size_t cap, uint64_t* d_out_size, cudaStream_t stream, uint64_t* launches) {
    cudaError_t e = set_smem_attrs_once();
    if (e != cudaSuccess) return e;
    const ChamBufs B(ws, L, nbytes);
    e = cudaMemsetAsync(B.st, 0, sizeof(Status), stream);
    if (e != cudaSuccess) return e;
    if (B.nblocks == 0) return cudaMemsetAsync(d_out_size, 0, sizeof(uint64_t), stream);
    cham_protected_pass<<<1, 1024, sizeof(ProtSmem), stream>>>(reinterpret_cast<const uint32_t*>(d_in), nbytes, B.st, 0, B.sigw, B.copymap);
    ++*launches;
    return sizes_scan_emit(B, d_in, B.copymap, 0, false, d_out, cap, d_out_size, stream, launches, nullptr);
}

// ---- sharded copy-map iteration (see cham_prot_start_k): the launches every codec shares, then Chameleon's phases -----------------------
ProtSegs prot_segs(Status* st, uint64_t nbytes, uint64_t nblocks, uint8_t* inc, uint8_t* cm, uint8_t* cm2, uint32_t* seg_state) {
    ProtSegs P;
    P.st = st; P.nbytes = nbytes; P.nblocks = nblocks; P.inc = inc; P.cm = cm; P.cm2 = cm2;
    P.nseg = (uint32_t)((nblocks + PSEG - 1) / PSEG); P.ngrp = (P.nseg + PC_GROUP - 1) / PC_GROUP;
    P.in_state = seg_state;
    uint16_t* ptab = reinterpret_cast<uint16_t*>(seg_state + 2 * (P.nseg + 1));
    P.gin = reinterpret_cast<uint32_t*>(ptab); P.T = ptab + 2 * (P.ngrp + 2); P.GT = P.T + (size_t)P.nseg * PC_NC;
    return P;
}
cudaError_t prot_start(const ProtSegs& P, ProtShard* ps, uint64_t first_block, const uint64_t* d_lengths, uint32_t rank, uint32_t block_bytes,
                       cudaStream_t stream, uint64_t* launches) {
    cham_prot_start_k<<<1, 32, 0, stream>>>(P.st, ps, first_block, d_lengths, rank, block_bytes);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t prot_transfer(const ProtSegs& P, const uint32_t* sigw, const ProtShard* ps, int it, uint32_t* d_transfer_out, cudaStream_t stream,
                          uint64_t* launches) {
    if (P.nblocks) {
        cham_prot_seg_k<<<P.nseg < 2048u ? P.nseg : 2048u, PSEG, 0, stream>>>(sigw, P.nbytes, P.nblocks, P.nseg, P.st, it, P.inc, P.cm, ps, P.T);
        cham_prot_groups_k<<<(P.ngrp * PC_NC + 255) / 256, 256, 0, stream>>>(P.nseg, P.st, P.T, P.GT);
        *launches += 2;
    }
    cham_prot_transfer_k<<<1, 256, 0, stream>>>(P.nseg, P.st, P.GT, d_transfer_out);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t prot_settle(const ProtSegs& P, ProtShard* ps, int it, int warm, const uint32_t* d_all_transfers, uint32_t rank, uint32_t* d_words,
                        cudaStream_t stream, uint64_t* launches) {
    cham_prot_enter_k<<<1, 32, 0, stream>>>(d_all_transfers, rank, P.nseg, P.st, P.GT, P.gin, ps, d_words);
    ++*launches;
    if (P.nseg) {
        cham_prot_seams_k<<<(P.ngrp + 127) / 128, 128, 0, stream>>>(P.nseg, P.st, P.T, P.gin, P.in_state);
        cham_prot_walk_k<<<(P.nseg + 127) / 128, 128, 0, stream>>>(P.nblocks, P.nseg, P.st, it, warm, P.inc, P.cm, P.cm2, P.in_state, P.gin, ps, d_words);
        *launches += 2;
    }
    return cudaGetLastError();
}
cudaError_t prot_commit(const ProtSegs& P, ProtShard* ps, int it, const uint32_t* d_all_words, uint32_t world, uint32_t stride, cudaStream_t stream,
                        uint64_t* launches) {
    if (P.nblocks) {
        cham_prot_commit_k<<<(uint32_t)((P.nblocks + 1023) / 1024 < 1024 ? (P.nblocks + 1023) / 1024 : 1024), 256, 0, stream>>>(
            d_all_words, world, stride, P.nblocks, P.st, it, P.cm, P.cm2);
        ++*launches;
    }
    cham_prot_verdict_k<<<1, 32, 0, stream>>>(d_all_words, world, stride, P.st, it, ps);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t prot_refuse_unsettled(Status* st, const ProtShard* ps, cudaStream_t stream, uint64_t* launches) {
    cham_prot_finish_k<<<1, 32, 0, stream>>>(st, ps);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t prot_seam_words(uint64_t nblocks, Status* st, uint64_t* d_out_size, uint32_t* d_seam8, cudaStream_t stream, uint64_t* launches) {
    cham_prot_seam_words_k<<<1, 32, 0, stream>>>(nblocks, st, d_out_size, d_seam8);
    ++*launches;
    return cudaGetLastError();
}

static ProtSegs cham_prot_segs(const ChamBufs& B) { return prot_segs(B.st, B.nbytes, B.nblocks, B.incb, B.copymap, B.copymap2, B.seg_state); }

cudaError_t cham_prot_start(uint8_t* ws, const ChamLayout& L, ProtShard* ps, uint64_t first_block, const uint64_t* d_lengths, uint32_t rank,
                            cudaStream_t stream, uint64_t* launches) {
    cham_prot_start_k<<<1, 32, 0, stream>>>(reinterpret_cast<Status*>(ws + L.status), ps, first_block, d_lengths, rank, 256u);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t cham_put_u64(uint64_t* d, uint64_t v, cudaStream_t stream, uint64_t* launches) {
    cham_put_u64_k<<<1, 32, 0, stream>>>(d, v);
    ++*launches;
    return cudaGetLastError();
}

cudaError_t cham_prot_transfer(size_t nbytes, uint8_t* ws, const ChamLayout& L, uint32_t nruns, const uint32_t* d_carry_in, const ProtShard* ps,
                               int it, uint32_t* d_transfer_out, cudaStream_t stream, uint64_t* launches) {
    const ChamBufs B(ws, L, nbytes);
    if (B.nblocks) launch_carry_resolve(B, nruns, d_carry_in, B.st, stream, launches);
    return prot_transfer(cham_prot_segs(B), B.sigw, ps, it, d_transfer_out, stream, launches);
}

cudaError_t cham_prot_settle(size_t nbytes, uint8_t* ws, const ChamLayout& L, ProtShard* ps, int it, const uint32_t* d_all_transfers, uint32_t rank,
                             uint32_t* d_words, cudaStream_t stream, uint64_t* launches) {
    const ChamBufs B(ws, L, nbytes);
    return prot_settle(cham_prot_segs(B), ps, it, 0, d_all_transfers, rank, d_words, stream, launches);
}

cudaError_t cham_prot_next(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, uint32_t nruns, ProtShard* ps, int it,
                           const uint32_t* d_all_words, uint32_t world, uint32_t* d_table_out, cudaStream_t stream, uint64_t* launches) {
    const ChamBufs B(ws, L, nbytes);
    cudaError_t e = prot_commit(cham_prot_segs(B), ps, it, d_all_words, world, PROT_ROUND_WORDS, stream, launches);
    if (e != cudaSuccess) return e;
    if (d_table_out) {
        if (B.nblocks) {   // round it + 1: flags under the new map (copy-mode blocks hidden from the dictionary) and the shard's table
            e = set_smem_attrs_once();
            if (e != cudaSuccess) return e;
            launch_flag_pass(B, d_in, nruns, B.copymap, B.st, stream, launches);
            launch_export_fold(B, nruns, d_table_out, B.st, stream, launches);
        } else {
            e = cudaMemsetAsync(d_table_out, 0, 65536 * sizeof(uint32_t), stream);   // nothing touched
            if (e != cudaSuccess) return e;
        }
    }
    return cudaGetLastError();
}

cudaError_t cham_prot_finish(const uint8_t* d_in, size_t nbytes, uint8_t* ws, const ChamLayout& L, const ProtShard* ps, uint8_t* d_out, size_t cap,
                             uint64_t* d_out_size, uint32_t* d_seam8, cudaStream_t stream, uint64_t* launches, cudaEvent_t* ev) {
    const ChamBufs B(ws, L, nbytes);
    cudaError_t e = prot_refuse_unsettled(B.st, ps, stream, launches);
    if (e == cudaSuccess && B.nblocks) e = cham_phase2_finish(B, d_in, d_out, cap, d_out_size, true, false, stream, launches, ev);
    if (e != cudaSuccess) return e;
    return prot_seam_words(B.nblocks, B.st, d_out_size, d_seam8, stream, launches);
}

}  // namespace dns
