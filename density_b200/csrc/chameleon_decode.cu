// chameleon_decode.cu — parallel Chameleon decode for sm_90a.
//
// Replaces /root/reference/src/algorithms/chameleon/chameleon.rs:55-68,103-135 (decode_plain / decode_map / decode_unit /
// decode_partial_unit) driven by /root/reference/src/codec/codec.rs:82-126 (Codec::decode), bit-exactly.
//
// The reference decoder has three serial chains (SURVEY §7.3 H4): block boundaries (block b+1 starts where block b's
// payload ends; nothing in the stream says where), the protection automaton, and the dictionary (a MAP quad reads the most
// recent PLAIN quad with that hash). This file breaks them as follows.
//
//  1. Boundaries.  A full encoded block is 8 + 256 - 2*popc(sig) bytes. The stream is cut into 16 KiB chunks; for each
//     chunk and each of the 132 possible (even) entry offsets in its first 264 bytes, `dec_chunk_walk` walks the chunk in
//     shared memory and records where that walk leaves the chunk and how many blocks it saw. Composing these 132-entry maps
//     (per group of 64 chunks, then over the groups, then back down) yields every chunk's true entry point and block
//     index; `dec_block_offsets` re-walks each chunk from its true entry and writes one offset per block.
//  2. Protection.  `dec_quiet_check`: if no two consecutive blocks are incompressible (>= 256 bytes consumed, codec.rs:98)
//     the automaton never leaves its initial state and no block is in copy mode (same argument as the encoder). Otherwise
//     the candidate walks are void (a copy-mode block has no signature) and `dec_seq_walk` redoes the boundaries in order
//     with the exact automaton: chunks in which the automaton provably stays in encoded mode are jumped in O(1) from the
//     candidate table, the others are walked block by block from shared memory and their copy-mode blocks marked; the
//     dictionary passes below then run unchanged (a copy-mode block is 64 raw quads that neither read nor write the
//     dictionary, codec.rs:89-92).
//  3. Dictionary.  `cham_decode_pass7`: one persistent CTA per contiguous run of blocks, the run's dictionary in shared
//     memory as 16-bit fingerprints (common.cuh). PLAIN quads (~7 %) are the writers, MAP quads the readers. A first launch, the
//     writer pass, looks at the writers only and leaves each run's last-writer table; `dec_carry_scan` folds those tables into the
//     dictionary each run starts from; a second launch decodes every run from it. Inside a run, tiles of 4096 quads go through a
//     write / verify / mailbox protocol (see the section comment above the kernel).
//  4. Tail.  The last < 264 bytes of the stream (codec.rs:102-123: per-unit bounds checks, partial units, 1-3 raw bytes) are
//     decoded by one thread with the reference's literal control flow, starting from the folded dictionary.
//  5. Sharded decode (DESIGN §5).  One piece of a sharded stream in two phases: phase 1 (boundaries, writer pass) needs no carry-in
//     and exports the piece's last-writer table, tail included; phase 2 folds the carry-in from the pieces before it into every
//     run's dictionary, decodes, and writes the piece's seam words for the cross-piece quiet check.
#include "common.cuh"
#include "encode_internal.cuh"
#include "decode_bounds.cuh"

namespace dns {
namespace chamdec {

using bounds::DecStatus;
using bounds::BLK_COPY;
using bounds::ldu16;
using T = bounds::ChamT;     // boundaries: decode_bounds.cuh (shared with the Cheetah decoder)

// ---- 3. decode pass ---------------------------------------------------------------------------------------------------------
constexpr int TILE_Q = 4096;   // quads per tile = 64 blocks

__device__ __forceinline__ bool bit_test(const uint32_t* bm, uint32_t i) { return (bm[i >> 5] >> (i & 31)) & 1u; }

// ------------------------------------------------------------------------------------------------------------------------------
// Decode pass: the structure of the encoder's flag pass (chameleon_encode.cu cham_flag_pass6): nothing but loads, compares and ballots
// on the per-quad path; atomics and searches only on the few "dirty" quads, one record per lane.
// One persistent CTA per run: run r owns tiles [r * ntiles / nruns, (r + 1) * ntiles / nruns) of the st->main_blocks blocks (blk_off:
// each block's stream offset and copy-mode bit) and keeps the run's dictionary in shared memory as 16-bit fingerprints. Nothing runs
// when st reports a non-quiet stream or an error. Both instances leave the run's last-writer table in final_tab (65536 x
// touched << 16 | fp per run).
// WONLY = true: "writer pass" — only the PLAIN quads are looked at; produces each run's last-writer table so that the carry-in
// dictionary of every run is known before the real decode pass starts (a MAP quad cannot tell what its bucket held at the start of
// the run). WONLY = false: the decode pass proper, dictionary preloaded from `carry`, every quad of the run written to `out`.
// 512 threads, 8 quads per thread, tile = 4096 quads = 64 blocks:
//   A  readers (MAP quads) read the pre-tile dictionary; writers (PLAIN quads, ~7 %) compute hash and fingerprint.        (barrier)
//   B  writers store their fingerprint (racy on purpose) and raise the bucket's byte in a hashed per-tile mark map.        (barrier)
//   C  raw and PLAIN quads go out as they are; a reader whose mark byte is clear saw no writer of its bucket in this tile: the
//      pre-tile value is its value (coalesced store). Writers and the remaining readers (suspects) are compacted in stream order into
//      the warp's record region; writers drop their record index into the mailbox of their bucket (4096 slots x 4 + overflow).  (barrier)
//   D  one record per lane: a suspect takes the fingerprint of the writer with the largest smaller index in its bucket, or its own
//      pre-tile value; the writer without a successor leaves the bucket's final fingerprint and clears the mark.            (barrier)
// The writer pass needs A, the deposit and D.
// A mailbox overflow (more than ~20 PLAIN quads of one bucket in one tile) sends the tile to d7_replay (one warp, in order).
// ------------------------------------------------------------------------------------------------------------------------------
constexpr int D7_THREADS = 512, D7_QPT = 8, D7_NW = D7_THREADS / 32, D7_WQ = 32 * D7_QPT;
static_assert(D7_THREADS * D7_QPT == TILE_Q, "tile geometry");
constexpr int D7_MB_SLOTS = 4096, D7_MB_CAP = 4, D7_SEC_SLOTS = 64, D7_SEC_CAP = 16, D7_MARK_N = 8192;
constexpr uint32_t D7_TOUCHED = 1u << 12, D7_WRITER = 1u << 13;   // record.y: pos (12) | touched | writer | pre-tile fingerprint << 16

struct Dec7Smem {
    uint16_t tab[65536];
    uint32_t vbit[2048];
    uint2 rec[TILE_Q];            // warp w: records [256 w, 256 w + cnt[w]) in stream order. x = hash | fp << 16 (fp: writers), y see above
    union {
        uint16_t mb[D7_MB_SLOTS][D7_MB_CAP];     // writers only: (hash >> 12) << 12 | record index
        uint32_t wseen[2048];                    // fallback only: bucket written so far in this tile
    };
    uint32_t mbcnt[2][D7_MB_SLOTS / 4];
    __align__(16) uint32_t sec[D7_SEC_SLOTS][D7_SEC_CAP];
    uint32_t seccnt[2][D7_SEC_SLOTS];
    uint8_t wmark[D7_MARK_N];     // per tile: some writer's bucket hashes here
    unsigned long long boff[2][64];
    uint32_t bsig[2][128];
    uint32_t bcopy[2][2];
    uint32_t cnt[32];
    uint32_t overflow;
};
static_assert(sizeof(Dec7Smem) <= 227 * 1024, "decode pass shared memory");

// Staging of a tile's block offsets and signatures, three tiles deep in registers of threads 0..63 so that neither of the two
// dependent global loads (offset -> signature) is waited for: at the top of tile t the values of tile t+1 (loads issued during tile
// t-1) go to shared memory, the signature loads of tile t+2 are issued from its offsets (loaded during tile t-1) and the offset loads
// of tile t+3 are issued.
struct Stage7 {
    unsigned long long o_sig;    // tile t+1 (then t+2): payload offset / copy flag as loaded
    uint32_t lo, hi;             // its signature halves (in flight)
    unsigned long long o_next;   // tile t+2 (then t+3): raw blk_off entry (in flight)
};
__device__ __forceinline__ unsigned long long stage7_load_off(const uint64_t* __restrict__ blk_off, uint64_t b, uint64_t nblocks) {
    return b < nblocks ? __ldg(reinterpret_cast<const unsigned long long*>(blk_off) + b) : ~0ull;     // ~0: no such block
}
__device__ __forceinline__ void stage7_load_sig(const uint8_t* __restrict__ in, unsigned long long o, uint32_t& lo, uint32_t& hi) {
    lo = 0; hi = 0;
    if (o != ~0ull && !(o & BLK_COPY)) {
        const uint8_t* p = in + o;
        lo = ldu16(p) | (ldu16(p + 2) << 16); hi = ldu16(p + 4) | (ldu16(p + 6) << 16);
    }
}
__device__ __forceinline__ void stage7_commit(Dec7Smem& S, int buf, unsigned long long o, uint32_t lo, uint32_t hi) {
    const uint32_t tid = threadIdx.x;     // < 64: warps 0 and 1, whole warps
    const bool none = o == ~0ull;
    const bool copied = !none && (o & BLK_COPY) != 0;
    unsigned long long off = none ? 0ull : (o & ~BLK_COPY);
    if (!none && !copied) off += 8;       // payload starts behind the signature; a copy-mode block is 64 raw quads at the block start
    S.boff[buf][tid] = off; S.bsig[buf][2 * tid] = lo; S.bsig[buf][2 * tid + 1] = hi;
    const uint32_t cmask = __ballot_sync(0xFFFFFFFFu, copied);
    if ((tid & 31) == 0) S.bcopy[buf][tid >> 5] = cmask;
}
// predicated 16-bit load without a branch: the loads of all sub-rows leave back to back (a branch per sub-row would make every
// sub-row wait for its own load: 8 exposed HBM latencies per tile)
__device__ __forceinline__ uint32_t ldu16_if(const uint8_t* p, bool pred) {
    uint32_t v;
    asm volatile("{ .reg .pred q; setp.ne.u32 q, %2, 0; mov.u32 %0, 0; @q ld.global.nc.u16 %0, [%1]; }" : "=r"(v) : "l"(p), "r"((uint32_t)pred));
    return v;
}
template <bool WONLY>
__device__ __forceinline__ void fetch_payload7(const Dec7Smem& S, int buf, const uint8_t* __restrict__ in, uint32_t nb_tile, uint32_t (&v)[D7_QPT]) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t a[D7_QPT], b[D7_QPT];
#pragma unroll
    for (int j = 0; j < D7_QPT; ++j) {
        const uint32_t bl = warp * (D7_WQ / 64) + (j >> 1);
        const uint32_t k = (j & 1) * 32 + lane;
        const bool in_tile = bl < nb_tile;
        const uint32_t blc = in_tile ? bl : 0u;
        const uint32_t lo = S.bsig[buf][2 * blc], hi = S.bsig[buf][2 * blc + 1];
        const uint32_t flag = (((j & 1) ? hi : lo) >> lane) & 1u;
        const uint32_t before = (j & 1) ? (__popc(lo) + __popc(hi & lanemask_lt())) : __popc(lo & lanemask_lt());
        const uint8_t* p = in + S.boff[buf][blc] + 4 * k - 2 * before;
        a[j] = ldu16_if(p, in_tile && !(WONLY && flag));        // MAP: the 16-bit hash (chameleon.rs:64); PLAIN: low half of the quad (:56)
        b[j] = ldu16_if(p + 2, in_tile && !flag);               // PLAIN: high half
    }
#pragma unroll
    for (int j = 0; j < D7_QPT; ++j) v[j] = a[j] | (b[j] << 16);
}

// Fallback: the tile's writers and suspects in stream order by one warp.
template <bool WONLY>
__device__ __noinline__ void d7_replay(Dec7Smem& S, uint32_t* __restrict__ out, uint64_t q0) {
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t i = lane; i < 2048; i += 32) S.wseen[i] = 0;
    const uint32_t c = lane < (uint32_t)D7_NW ? S.cnt[lane] : 0u;
    uint32_t incl = c;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d); if ((int)lane >= d) incl += t; }
    const uint32_t excl = incl - c;
    const uint32_t n = __shfl_sync(0xFFFFFFFFu, incl, 31);
    __syncwarp();
    #pragma unroll 1
    for (uint32_t i0 = 0; i0 < n; i0 += 32) {
        const uint32_t i = i0 + lane;
        const bool valid = i < n;
        uint32_t w = 0;
#pragma unroll
        for (int b = 16; b >= 1; b >>= 1) { const uint32_t t = __shfl_sync(0xFFFFFFFFu, incl, (w + b - 1) & 31); if (t <= i) w += b; }
        const uint32_t e = __shfl_sync(0xFFFFFFFFu, excl, w & 31);
        uint2 r = make_uint2(0, 0);
        if (valid) r = S.rec[w * D7_WQ + (i - e)];
        const uint32_t hh = r.x & 0xFFFFu, ff = r.x >> 16, pos = r.y & 0xFFFu;
        const bool writer = valid && (r.y & D7_WRITER);
        const uint32_t grp = __match_any_sync(0xFFFFFFFFu, valid ? hh : 0x10000u + lane);
        const uint32_t wm = __ballot_sync(0xFFFFFFFFu, writer);
        const uint32_t lw = grp & wm & lanemask_lt();              // earlier writers of my bucket inside the step
        const uint32_t fprev = __shfl_sync(0xFFFFFFFFu, ff, lw ? 31 - __clz(lw) : 0);
        if (valid && !writer && !WONLY) {
            uint32_t fv = r.y >> 16; bool have = (r.y & D7_TOUCHED) != 0;
            if (lw) { fv = fprev; have = true; }
            else if ((S.wseen[hh >> 5] >> (hh & 31)) & 1u) { fv = S.tab[hh]; have = true; }
            out[q0 + pos] = have ? quad_from_hf(hh, fv) : 0u;
        }
        __syncwarp();
        if (writer && (grp & wm & lanemask_gt()) == 0) {           // last writer of the bucket inside the step
            S.tab[hh] = (uint16_t)ff;
            if (ff == 0) atomicOr(&S.vbit[hh >> 5], 1u << (hh & 31));
            atomicOr(&S.wseen[hh >> 5], 1u << (hh & 31));
            S.wmark[hh & (D7_MARK_N - 1)] = 0;
        }
        __syncwarp();
    }
}

template <bool WONLY>
__global__ void __launch_bounds__(D7_THREADS, 1)
cham_decode_pass7(const uint8_t* __restrict__ in, const uint64_t* __restrict__ blk_off, DecStatus* st,
                  uint32_t nruns, uint32_t* __restrict__ out /* quads */, const uint32_t* __restrict__ carry,
                  uint32_t* __restrict__ final_tab) {
    if (st->nonquiet || st->error) return;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Dec7Smem& S = *reinterpret_cast<Dec7Smem*>(smem_raw);
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t run = blockIdx.x;
    const uint64_t nblocks = st->main_blocks;
    const uint64_t ntiles = (nblocks + 63) / 64;
    const uint64_t t_begin = (uint64_t)run * ntiles / nruns, t_end = (uint64_t)(run + 1) * ntiles / nruns;
    {
        const uint4 z = make_uint4(0, 0, 0, 0);
        uint4* t4 = reinterpret_cast<uint4*>(S.tab);
        for (uint32_t i = tid; i < 65536 * 2 / 16; i += D7_THREADS) t4[i] = z;
        for (uint32_t i = tid; i < 2048; i += D7_THREADS) S.vbit[i] = 0;
        for (uint32_t i = tid; i < D7_MB_SLOTS / 4; i += D7_THREADS) { S.mbcnt[0][i] = 0; S.mbcnt[1][i] = 0; }
        for (uint32_t i = tid; i < D7_MARK_N / 4; i += D7_THREADS) reinterpret_cast<uint32_t*>(S.wmark)[i] = 0;
        if (tid < D7_SEC_SLOTS) { S.seccnt[0][tid] = 0; S.seccnt[1][tid] = 0; }
        if (tid == 0) S.overflow = 0;
        if (!WONLY) {
            __syncthreads();
            const uint32_t* __restrict__ cr = carry + (size_t)run * 65536;   // dictionary before this run
            for (uint32_t i = tid; i < 65536; i += D7_THREADS) {
                const uint32_t c = cr[i];
                if (c & 0x10000u) {
                    S.tab[i] = (uint16_t)c;
                    if ((c & 0xFFFFu) == 0) atomicOr(&S.vbit[i >> 5], 1u << (i & 31));
                }
            }
        }
    }
    __syncthreads();
    uint32_t nval[D7_QPT];
    Stage7 sg; sg.o_sig = ~0ull; sg.lo = 0; sg.hi = 0; sg.o_next = ~0ull;
    if (t_begin < t_end && tid < 64) {
        const unsigned long long o0 = stage7_load_off(blk_off, t_begin * 64 + tid, nblocks);
        uint32_t lo0, hi0;
        stage7_load_sig(in, o0, lo0, hi0);
        stage7_commit(S, 0, o0, lo0, hi0);
        if (t_begin + 1 < t_end) { sg.o_sig = stage7_load_off(blk_off, (t_begin + 1) * 64 + tid, nblocks); stage7_load_sig(in, sg.o_sig, sg.lo, sg.hi); }
        if (t_begin + 2 < t_end) sg.o_next = stage7_load_off(blk_off, (t_begin + 2) * 64 + tid, nblocks);
    }
    __syncthreads();
    if (t_begin < t_end) fetch_payload7<WONLY>(S, 0, in, (uint32_t)((nblocks - t_begin * 64 < 64) ? (nblocks - t_begin * 64) : 64), nval);

    for (uint64_t t = t_begin; t < t_end; ++t) {
        const uint64_t b0 = t * 64;
        const uint32_t nb_tile = (uint32_t)((nblocks - b0 < 64) ? (nblocks - b0) : 64);
        const int cur = (int)((t - t_begin) & 1);
        const uint32_t buf = (uint32_t)cur;
        if (tid < 64) {
            if (t + 1 < t_end) stage7_commit(S, cur ^ 1, sg.o_sig, sg.lo, sg.hi);          // tile t+1: loaded during tile t-1
            sg.o_sig = sg.o_next;                                                           // tile t+2: its signatures leave now
            sg.lo = 0; sg.hi = 0;
            if (t + 2 < t_end) stage7_load_sig(in, sg.o_sig, sg.lo, sg.hi);
            sg.o_next = (t + 3 < t_end) ? stage7_load_off(blk_off, (t + 3) * 64 + tid, nblocks) : ~0ull;   // tile t+3: its offsets leave now
        }
#pragma unroll
        for (int k = 0; k < D7_MB_SLOTS / 4 / D7_THREADS; ++k) S.mbcnt[buf ^ 1u][tid + k * D7_THREADS] = 0;
        if (tid < D7_SEC_SLOTS) S.seccnt[buf ^ 1u][tid] = 0;

        // ---- A
        uint32_t val[D7_QPT], hk[D7_QPT], fa[D7_QPT];   // val: the quad (PLAIN / raw) or the hash (MAP); hk: hash; fa: readers pre-tile fp, writers own fp
        uint32_t act = 0, wr = 0, raw = 0, tch = 0;     // bit j
#pragma unroll
        for (int j = 0; j < D7_QPT; ++j) {
            const uint32_t bl = warp * (D7_WQ / 64) + (j >> 1);
            val[j] = nval[j]; hk[j] = 0; fa[j] = 0;
            if (bl < nb_tile) {
                act |= 1u << j;
                const uint32_t flag = (S.bsig[cur][2 * bl + (j & 1)] >> lane) & 1u;
                if ((S.bcopy[cur][bl >> 5] >> (bl & 31)) & 1u) raw |= 1u << j;
                else if (flag) {
                    if (!WONLY) {
                        hk[j] = val[j];
                        fa[j] = S.tab[hk[j]];
                        if (fa[j] != 0 || bit_test(S.vbit, hk[j])) tch |= 1u << j;
                    }
                } else {
                    wr |= 1u << j;
                    const uint32_t p = hash_prod(val[j]);
                    hk[j] = prod_hash(p); fa[j] = prod_fp(p, val[j]);
                }
            }
        }
        __syncthreads();  // S1: readers have read the pre-tile dictionary; next tile's signatures staged
        if (t + 1 < t_end)   // payload of the next tile: in flight during the rest of this tile
            fetch_payload7<WONLY>(S, cur ^ 1, in, (uint32_t)((nblocks - (b0 + 64) < 64) ? (nblocks - (b0 + 64)) : 64), nval);
        if (!WONLY) {
            // ---- B
#pragma unroll
            for (int j = 0; j < D7_QPT; ++j)
                if ((wr >> j) & 1u) { S.tab[hk[j]] = (uint16_t)fa[j]; S.wmark[hk[j] & (D7_MARK_N - 1)] = 1; }
            __syncthreads();  // S2
        }
        // ---- C
        const uint64_t q0 = b0 * 64;   // first output quad of the tile
        uint32_t base = 0;
        uint2* __restrict__ myrec = S.rec + warp * D7_WQ;
#pragma unroll
        for (int j = 0; j < D7_QPT; ++j) {
            const uint32_t pos = warp * D7_WQ + j * 32 + lane;
            const bool active = (act >> j) & 1u, writer = (wr >> j) & 1u;
            bool dirty = writer;
            if (!WONLY && active) {
                if (writer || ((raw >> j) & 1u)) out[q0 + pos] = val[j];
                else if (S.wmark[hk[j] & (D7_MARK_N - 1)] == 0)
                    out[q0 + pos] = ((tch >> j) & 1u) ? quad_from_hf(hk[j], fa[j]) : 0u;      // empty bucket -> 0 (chameleon.rs:41)
                else dirty = true;
            }
            const uint32_t db = __ballot_sync(0xFFFFFFFFu, dirty);
            if (dirty) myrec[base + __popc(db & lanemask_lt())] =
                make_uint2(hk[j] | (writer ? fa[j] << 16 : 0u), pos | (((tch >> j) & 1u) ? D7_TOUCHED : 0u) | (writer ? D7_WRITER : 0u) | (writer ? 0u : fa[j] << 16));
            base += __popc(db);
        }
        if (lane == 0) S.cnt[warp] = base;
        __syncwarp();
        // deposit (writers only)
        uint2 r0 = make_uint2(0, 0);
        #pragma unroll 1
        for (uint32_t i = lane; i < base; i += 32) {
            const uint2 r = myrec[i];
            if (i < 32) r0 = r;
            if (r.y & D7_WRITER) {
                const uint32_t hh = r.x & 0xFFFFu, slot = hh & (D7_MB_SLOTS - 1), sh = (slot & 3u) * 8u;
                const uint32_t k = (atomicAdd(&S.mbcnt[buf][slot >> 2], 1u << sh) >> sh) & 0xFFu;
                if (k < (uint32_t)D7_MB_CAP) S.mb[slot][k] = (uint16_t)(((hh >> 12) << 12) | (warp * D7_WQ + i));
                else {
                    const uint32_t s2 = slot & (D7_SEC_SLOTS - 1);
                    const uint32_t k2 = atomicAdd(&S.seccnt[buf][s2], 1u);
                    if (k2 < (uint32_t)D7_SEC_CAP) S.sec[s2][k2] = (hh << 12) | (warp * D7_WQ + i);
                    else S.overflow = 1;
                }
            }
        }
        __syncthreads();  // S3
        if (S.overflow) {
            if (warp == 0) d7_replay<WONLY>(S, out, q0);
        } else {
            // ---- D
            #pragma unroll 1
            for (uint32_t i0 = 0; i0 < base; i0 += 32) {
                const uint32_t i = i0 + lane;
                const bool valid = i < base;
                uint2 r = r0;
                if (i0) r = valid ? myrec[i] : make_uint2(0, 0);
                if (valid) {
                    const uint32_t hh = r.x & 0xFFFFu, slot = hh & (D7_MB_SLOTS - 1), myidx = warp * D7_WQ + i;
                    const uint32_t n = (S.mbcnt[buf][slot >> 2] >> ((slot & 3u) * 8u)) & 0xFFu;
                    const uint2 e2 = *reinterpret_cast<const uint2*>(&S.mb[slot][0]);
                    const uint32_t me = ((hh >> 12) << 12) | myidx;
                    int best = -1; bool later = false;
#pragma unroll
                    for (int tt = 0; tt < D7_MB_CAP; ++tt) {
                        const uint32_t e = ((tt & 2) ? e2.y : e2.x) >> ((tt & 1) * 16) & 0xFFFFu;
                        if ((uint32_t)tt < n && ((e ^ me) >> 12) == 0) {
                            if (e < me) best = max(best, (int)(e & 0xFFFu));
                            later |= e > me;
                        }
                    }
                    if (n > (uint32_t)D7_MB_CAP) {
                        const uint32_t s2 = slot & (D7_SEC_SLOTS - 1);
                        const uint32_t n2 = S.seccnt[buf][s2];
                        const uint32_t mine = (hh << 12) | myidx;
                        #pragma unroll 1
                        for (uint32_t t4 = 0; t4 < n2; t4 += 4) {
                            const uint4 e4 = *reinterpret_cast<const uint4*>(&S.sec[s2][t4]);
                            const uint32_t ev[4] = {e4.x, e4.y, e4.z, e4.w};
#pragma unroll
                            for (int tt = 0; tt < 4; ++tt) {
                                const uint32_t e = ev[tt];
                                if (t4 + tt < n2 && ((e ^ mine) & 0xFFFFF000u) == 0) {
                                    if (e < mine) best = max(best, (int)(e & 0xFFFu));
                                    later |= e > mine;
                                }
                            }
                        }
                    }
                    if (r.y & D7_WRITER) {
                        if (!later) {      // chameleon.rs:59: the last PLAIN quad of the bucket leaves its value
                            S.tab[hh] = (uint16_t)(r.x >> 16);
                            if ((r.x >> 16) == 0) atomicOr(&S.vbit[hh >> 5], 1u << (hh & 31));
                            S.wmark[hh & (D7_MARK_N - 1)] = 0;
                        }
                    } else if (!WONLY) {
                        uint32_t fv = r.y >> 16; bool have = (r.y & D7_TOUCHED) != 0;
                        if (best >= 0) { fv = S.rec[best].x >> 16; have = true; }
                        out[q0 + (r.y & 0xFFFu)] = have ? quad_from_hf(hh, fv) : 0u;
                    }
                }
            }
        }
        __syncthreads();  // S4
        if (tid == 0) S.overflow = 0;
    }
    for (uint32_t i = tid; i < 65536; i += D7_THREADS) {
        const uint32_t v = S.tab[i];
        const uint32_t tchd = (v != 0 || bit_test(S.vbit, i)) ? 0x10000u : 0u;
        final_tab[(size_t)run * 65536 + i] = v | tchd;
    }
}

// carry-in fold for decode, starting from `carry_in` (the dictionary before this piece of a sharded stream, shard format) or, when it
// is null, from the stream start: all zero values (chameleon.rs:41), nothing touched. The encoder's stream-start table (bucket 0
// touched with fingerprint 0) is the same dictionary: quad_from_hf(0, 0) == 0.
__global__ void dec_carry_scan(const uint32_t* __restrict__ final_tab, uint32_t nruns, uint32_t* __restrict__ carry, uint32_t* __restrict__ dict_out,
                               const uint32_t* __restrict__ carry_in) {
    uint32_t hb = blockIdx.x * blockDim.x + threadIdx.x;
    if (hb >= 65536) return;
    uint32_t c = carry_in ? carry_in[hb] : 0u;
    for (uint32_t r = 0; r < nruns; ++r) {
        carry[(size_t)r * 65536 + hb] = c;
        uint32_t v = final_tab[(size_t)r * 65536 + hb];
        if (v & 0x10000u) c = v;
    }
    dict_out[hb] = (c & 0x10000u) ? quad_from_hf(hb, c & 0xFFFFu) : 0u;   // full-width dictionary for the tail loop
}

// ---- 4. tail loop (codec.rs:102-123), one thread, literal control flow ---------------------------------------------------
__global__ void dec_tail(const uint8_t* __restrict__ in, uint64_t n, uint8_t* __restrict__ out, uint64_t cap, uint32_t* __restrict__ dict,
                         DecStatus* __restrict__ st, uint64_t* __restrict__ d_out_size) {
    if (threadIdx.x || blockIdx.x) return;
    if (st->nonquiet) { if (d_out_size) *d_out_size = 0; return; }   // gave up: the caller's in-order fallback (queued behind) produces the result
    if (st->error) { st->out_bytes = 0; if (d_out_size) *d_out_size = 0; return; }
    uint64_t idx = st->tail_off, oidx = st->main_blocks * 256;
    Protection ps = bounds::main_end_state(st);
    bool bad = false, overflow = false;
    auto emit = [&](uint32_t q) {
        if (oidx + 4 > cap) { overflow = true; return; }
        out[oidx] = (uint8_t)q; out[oidx + 1] = (uint8_t)(q >> 8); out[oidx + 2] = (uint8_t)(q >> 16); out[oidx + 3] = (uint8_t)(q >> 24);
        oidx += 4;
    };
    while (!bad && !overflow && n - idx > 0) {
        if (ps.revert_to_copy()) {
            const uint64_t rem = n - idx;
            const uint64_t len = rem > 256 ? 256 : rem;
            if (oidx + len > cap) { overflow = true; break; }
            for (uint64_t i = 0; i < len; ++i) out[oidx + i] = in[idx + i];
            oidx += len; idx += len;
            if (rem <= 256) break;
            ps.decay();
        } else {
            const uint64_t mark = idx;
            if (n - idx < 8) { bad = true; break; }
            uint64_t sig = 0;
            for (int i = 0; i < 8; ++i) sig |= (uint64_t)in[idx + i] << (8 * i);
            idx += 8;
            bool end = false;
            for (int u = 0; u < 32 && !end && !bad && !overflow; ++u) {        // 32 units of 2 quads (chameleon.rs:143)
                const bool checked = (n - idx) < 8;
                for (int k = 0; k < 2 && !end; ++k) {
                    const uint32_t fl = (uint32_t)(sig & 1); sig >>= 1;
                    if (checked && fl == 0) {                                    // decode_partial_unit, chameleon.rs:119-129
                        const uint64_t rem = n - idx;
                        if (rem == 0) { end = true; break; }
                        if (rem < 4) {
                            if (oidx + rem > cap) { overflow = true; end = true; break; }
                            for (uint64_t i = 0; i < rem; ++i) out[oidx++] = in[idx++];
                            end = true; break;
                        }
                    }
                    uint32_t q;
                    if (fl) {
                        if (n - idx < 2) { bad = true; break; }
                        q = dict[in[idx] | (in[idx + 1] << 8)]; idx += 2;
                    } else {
                        if (n - idx < 4) { bad = true; break; }
                        q = in[idx] | (in[idx + 1] << 8) | (in[idx + 2] << 16) | ((uint32_t)in[idx + 3] << 24); idx += 4;
                        dict[prod_hash(hash_prod(q))] = q;
                    }
                    emit(q);
                }
            }
            if (end) break;
            ps.update(idx - mark >= 256);
        }
    }
    uint64_t res = oidx;
    if (bad) { st->error = 3; res = 0; }
    else if (overflow) { st->error = 2; res = 0; }
    st->out_bytes = res;
    if (d_out_size) *d_out_size = res;
}

// ---- 5. sharded decode: a piece's exported table and its seam words ----------------------------------------------------------
// The tail's control flow: bounds::tail_walk (decode_bounds.cuh).
using bounds::TailWalk;
using bounds::tail_walk;

// The piece's exported table: the left fold of its run tables (writer pass) ...
__global__ void dec_export_fold(const uint32_t* __restrict__ final_tab, uint32_t nruns, uint32_t* __restrict__ table_out) {
    const uint32_t hb = blockIdx.x * blockDim.x + threadIdx.x;
    if (hb >= 65536) return;
    uint32_t c = 0;
    for (uint32_t r = 0; r < nruns; ++r) { const uint32_t v = final_tab[(size_t)r * 65536 + hb]; if (v & 0x10000u) c = v; }
    table_out[hb] = c;
}
// ... then the PLAIN quads of the tail on top: in a non-final piece the tail is usually its last block, and a MAP quad of the next
// piece may read what it wrote
__global__ void dec_export_tail(const uint8_t* __restrict__ in, uint64_t n, const DecStatus* __restrict__ st, uint32_t* __restrict__ table_out) {
    if (threadIdx.x || blockIdx.x) return;
    if (st->nonquiet || st->error) return;     // dec_tail will not run; the piece is refused
    tail_walk(in, n, st, [&](uint32_t q) { const uint32_t p = hash_prod(q); table_out[prod_hash(p)] = 0x10000u | prod_fp(p, q); });
}

// What a decoded piece tells the others, in the layout of cham_seam_words_k: {first block incompressible, last block incompressible,
// not quiet or error, has blocks, decoded size lo, hi, 0, 0}. Runs after dec_tail. Not quiet: copy-mode blocks in the main loop
// (dec_seq_walk ran) or in the tail, two incompressible blocks at the end (the next piece's first block would be copied: penalty > 0),
// an error (malformed, output beyond cap), or a non-final piece that does not decode to whole 256-byte blocks.
__global__ void dec_seam_words_k(const uint8_t* __restrict__ in, uint64_t n, const DecStatus* __restrict__ st, int is_last,
                                 const uint64_t* __restrict__ d_out_size, uint32_t* __restrict__ words) {
    if (threadIdx.x || blockIdx.x) return;
    const uint64_t sz = *d_out_size;
    uint32_t first = 0, last = 0, bad = (st->nonquiet || st->error || st->seq) ? 1u : 0u;
    if (!bad) {
        const TailWalk w = tail_walk(in, n, st, [](uint32_t) {});
        first = st->main_blocks ? (T::consumed(bounds::ldsig(in)) >= 256u ? 1u : 0u) : w.first_inc;
        last = w.ps.previous_incompressible;
        if (w.bad || w.copied || w.ps.copy_penalty) bad = 1;
    }
    if (!is_last && (sz % 256)) bad = 1;
    words[0] = first; words[1] = last; words[2] = bad; words[3] = 1;
    words[4] = (uint32_t)sz; words[5] = (uint32_t)(sz >> 32); words[6] = 0; words[7] = 0;
}

// ---- 6. sharded decode of a stream with copy-mode blocks (density_b200_decode_shard_prot_*, DESIGN §5) ----------------------------------
// The incoming state of a piece comes from bounds::dec_prot_enter_k (decode_bounds.cuh).
// The seam words of such a piece, in the layout of dec_seam_words_k. Copy-mode blocks, a pending penalty and incompressible blocks meet
// at the cuts legally here (the transfers carry the automaton across), so words 0 and 1 stay 0. Word 2: the transfers composed to no
// state, an error (malformed, output beyond cap), or a non-final piece that does not decode to whole 256-byte blocks. st == nullptr:
// an empty piece (no blocks, size 0), refused only by its seed.
__global__ void dec_prot_seam_words_k(const DecStatus* __restrict__ st, const uint32_t* __restrict__ seed, int is_last,
                                      uint64_t* __restrict__ d_out_size, uint32_t* __restrict__ words) {
    if (threadIdx.x || blockIdx.x) return;
    uint64_t sz = 0;
    uint32_t bad = seed[4];
    if (st) {
        sz = *d_out_size;
        if (st->nonquiet || st->error || (!is_last && (sz % 256))) bad = 1;
    } else *d_out_size = 0;
    words[0] = 0; words[1] = 0; words[2] = bad; words[3] = st ? 1u : 0u;
    words[4] = (uint32_t)sz; words[5] = (uint32_t)(sz >> 32); words[6] = 0; words[7] = 0;
}

}  // namespace chamdec

using namespace chamdec;

struct ChamDecLayout { bounds::BoundsLayout B; size_t final_tab, carry, dict, total; };

static size_t dec_layout(size_t nbytes, size_t cap, int nruns_max, ChamDecLayout* L) {
    size_t off = bounds::bounds_layout<T>(nbytes, cap, &L->B);
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
    L->final_tab = take((size_t)nruns_max * 65536 * sizeof(uint32_t));
    L->carry = take((size_t)nruns_max * 65536 * sizeof(uint32_t));
    L->dict = take(65536 * sizeof(uint32_t));
    L->total = off;
    return off;
}

size_t cham_decode_workspace_bytes(size_t nbytes, size_t cap, int nruns_max) { ChamDecLayout L; return dec_layout(nbytes, cap, nruns_max, &L); }

// run count from an upper bound of the block count (the kernels read the real one from the status block)
static uint32_t dec_pick_runs(const ChamDecLayout& L, int num_sms) {
    const uint64_t tiles_ub = (L.B.maxblocks + 63) / 64;
    uint32_t nruns = (uint32_t)(tiles_ub / 16); if (nruns < 1) nruns = 1; if (nruns > (uint32_t)num_sms) nruns = num_sms;
    return nruns;
}

// Phase 1 of the parallel decode, which needs no carry-in: boundaries, then the writer pass (each run's last-writer table). With
// d_table_out it also exports the piece's table (shard format) for the pieces after it.
cudaError_t cham_decode_phase1(const uint8_t* d_in, size_t nbytes, size_t cap, uint8_t* ws, int num_sms, uint32_t* d_table_out,
                               cudaStream_t stream, uint64_t* launches, const uint32_t* d_seed, bool rows_ready) {
    static bool attr_done = false;
    if (!attr_done) {
        cudaError_t e0 = cudaFuncSetAttribute(cham_decode_pass7<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Dec7Smem));
        if (e0 == cudaSuccess) e0 = cudaFuncSetAttribute(cham_decode_pass7<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Dec7Smem));
        if (e0 != cudaSuccess) return e0;
        attr_done = true;
    }
    ChamDecLayout L; dec_layout(nbytes, cap, num_sms, &L);
    DecStatus* st = reinterpret_cast<DecStatus*>(ws + L.B.status);
    uint64_t* blk_off = reinterpret_cast<uint64_t*>(ws + L.B.blk_off);
    cudaError_t e = bounds::bounds_launch<T>(d_in, nbytes, cap, ws, L.B, stream, launches, d_seed, rows_ready);
    if (e != cudaSuccess) return e;
    const uint32_t nruns = dec_pick_runs(L, num_sms);
    uint32_t* final_tab = reinterpret_cast<uint32_t*>(ws + L.final_tab);
    cham_decode_pass7<true><<<nruns, D7_THREADS, sizeof(Dec7Smem), stream>>>(d_in, blk_off, st, nruns, nullptr, nullptr, final_tab);
    ++*launches;
    if (d_table_out) {
        dec_export_fold<<<65536 / 256, 256, 0, stream>>>(final_tab, nruns, d_table_out);
        dec_export_tail<<<1, 32, 0, stream>>>(d_in, nbytes, st, d_table_out);
        *launches += 2;
    }
    return cudaGetLastError();
}

// Phase 2: the carry-in of every run folded from d_carry_in (NULL: stream start), the decode pass and the tail. The workspace is the one
// phase 1 filled for the same (d_in, nbytes, cap, num_sms).
cudaError_t cham_decode_phase2(const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws, int num_sms, const uint32_t* d_carry_in,
                               uint64_t* d_out_size, cudaStream_t stream, uint64_t* launches) {
    ChamDecLayout L; dec_layout(nbytes, cap, num_sms, &L);
    DecStatus* st = reinterpret_cast<DecStatus*>(ws + L.B.status);
    uint64_t* blk_off = reinterpret_cast<uint64_t*>(ws + L.B.blk_off);
    const uint32_t nruns = dec_pick_runs(L, num_sms);
    uint32_t* final_tab = reinterpret_cast<uint32_t*>(ws + L.final_tab);
    uint32_t* carry = reinterpret_cast<uint32_t*>(ws + L.carry);
    dec_carry_scan<<<65536 / 256, 256, 0, stream>>>(final_tab, nruns, carry, reinterpret_cast<uint32_t*>(ws + L.dict), d_carry_in); ++*launches;
    cham_decode_pass7<false><<<nruns, D7_THREADS, sizeof(Dec7Smem), stream>>>(d_in, blk_off, st, nruns, reinterpret_cast<uint32_t*>(d_out), carry, final_tab);
    ++*launches;
    dec_tail<<<1, 32, 0, stream>>>(d_in, nbytes, d_out, cap, reinterpret_cast<uint32_t*>(ws + L.dict), st, d_out_size); ++*launches;
    return cudaGetLastError();
}

// The 8 seam words of a decoded piece (after phase 2; d_out_size as phase 2 wrote it).
cudaError_t cham_decode_seam_words(const uint8_t* d_in, size_t nbytes, size_t cap, uint8_t* ws, int num_sms, int is_last, const uint64_t* d_out_size,
                                   uint32_t* d_words, cudaStream_t stream, uint64_t* launches) {
    ChamDecLayout L; dec_layout(nbytes, cap, num_sms, &L);
    dec_seam_words_k<<<1, 32, 0, stream>>>(d_in, nbytes, reinterpret_cast<const DecStatus*>(ws + L.B.status), is_last, d_out_size, d_words);
    ++*launches;
    return cudaGetLastError();
}

// The protection transfer of a piece (PT_NCAND words to d_transfer): the candidate rows of the boundary walk, then the head walk over them.
// The rows stay in the workspace for cham_decode_phase1 with a seed.
cudaError_t cham_decode_prot_transfer(const uint8_t* d_in, size_t nbytes, uint8_t* ws, int is_last, uint32_t* d_transfer, cudaStream_t stream,
                                      uint64_t* launches) {
    return bounds::prot_transfer_launch<T>(d_in, nbytes, is_last, ws, d_transfer, stream, launches);
}
cudaError_t cham_decode_prot_enter(const uint32_t* d_all_transfers, uint32_t rank, uint32_t x0, uint32_t* d_seed, cudaStream_t stream,
                                   uint64_t* launches) {
    bounds::dec_prot_enter_k<<<1, 32, 0, stream>>>(d_all_transfers, rank, x0, d_seed);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t cham_decode_prot_seam_words(size_t nbytes, size_t cap, uint8_t* ws, int num_sms, int is_last, const uint32_t* d_seed, uint64_t* d_out_size,
                                        uint32_t* d_words, cudaStream_t stream, uint64_t* launches) {
    const DecStatus* st = nullptr;
    if (nbytes) { ChamDecLayout L; dec_layout(nbytes, cap, num_sms, &L); st = reinterpret_cast<const DecStatus*>(ws + L.B.status); }
    dec_prot_seam_words_k<<<1, 32, 0, stream>>>(st, d_seed, is_last, d_out_size, d_words);
    ++*launches;
    return cudaGetLastError();
}

// The range map of d_in[0 .. n_range + n_halo) (sharded decode of a stream without known cuts): the candidate walks over the range's
// chunks, with the halo visible to the walks of its last chunk, their composition per group, then over the whole range. The scratch is
// the res / gres arrays of the boundary layout of n_range + n_halo bytes, where phase 1 puts them too.
size_t cham_locate_workspace_bytes(size_t nbytes) { bounds::BoundsLayout B; return bounds::bounds_layout<T>(nbytes, 0, &B); }

cudaError_t cham_decode_locate(const uint8_t* d_in, size_t n_range, size_t n_halo, uint8_t* ws, uint64_t* d_map, cudaStream_t stream,
                               uint64_t* launches) {
    bounds::range_map_launch<T>(d_in, n_range, n_halo, ws, reinterpret_cast<unsigned long long*>(d_map), stream, launches);
    return cudaGetLastError();
}

// The protected range map of d_in[0 .. n_range + n_halo) (DENSITY_B200_PROT_LOCATE_MAP_WORDS u32 to d_map); the scratch is
// cham_locate_workspace_bytes(n_range + n_halo).
cudaError_t cham_decode_prot_locate(const uint8_t* d_in, size_t n_range, size_t n_halo, uint8_t* ws, uint32_t* d_map, cudaStream_t stream,
                                    uint64_t* launches) {
    return bounds::prot_locate_launch<T>(d_in, n_range, n_halo, ws, d_map, stream, launches);
}

// Enqueues the parallel decode. On return (after the stream drains) *d_nonquiet != 0 means the caller must run the exact
// in-order kernel instead (copy-mode blocks present, or a pathological tile); d_out_size is only written when it is 0.
cudaError_t cham_decode_parallel(const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws, int num_sms,
                                 uint64_t* d_out_size, uint32_t* d_nonquiet, cudaStream_t stream, uint64_t* launches) {
    cudaError_t e = cham_decode_phase1(d_in, nbytes, cap, ws, num_sms, nullptr, stream, launches, nullptr);
    if (e == cudaSuccess) e = cham_decode_phase2(d_in, nbytes, d_out, cap, ws, num_sms, nullptr, d_out_size, stream, launches);
    if (e != cudaSuccess) return e;
    ChamDecLayout L; dec_layout(nbytes, cap, num_sms, &L);
    e = cudaMemcpyAsync(d_nonquiet, &reinterpret_cast<DecStatus*>(ws + L.B.status)->nonquiet, sizeof(uint32_t), cudaMemcpyDeviceToDevice, stream);
    if (e != cudaSuccess) return e;
    return cudaGetLastError();
}

}  // namespace dns
