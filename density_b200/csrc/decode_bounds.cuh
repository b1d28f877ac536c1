// decode_bounds.cuh — block boundaries of a density stream, in parallel, for all three algorithms (sm_90a).
//
// Replaces the cursor of /root/reference/src/codec/codec.rs:88-100 (the main decode loop): nothing in the stream says where block
// b + 1 starts; an encoded block is `SIG + payload(signature)` bytes, a copy-mode block (protection_state.rs) BS raw bytes.
//
//  1. The stream is cut into chunks of T::CH bytes; for each chunk and each of the T::NCAND possible (even) entry offsets in its
//     first T::MAXBLK bytes, `dec_chunk_walk` walks the chunk in shared memory and records where that walk leaves the chunk and how
//     many blocks it saw. Composing these maps (per group of GROUP chunks, then over the groups, then back down) yields every chunk's
//     true entry point and block index; `dec_block_offsets` re-walks each chunk from its true entry and writes one offset per block.
//  2. `dec_quiet_check`: if no two consecutive blocks are incompressible (consumed >= BS, codec.rs:98) the automaton never leaves its
//     initial state and no block is in copy mode. Otherwise the candidate walks are void (a copy-mode block has no signature) and
//     `dec_seq_walk` redoes the boundaries in order with the exact automaton: chunks (and whole groups) in which the automaton
//     provably stays in encoded mode are jumped in O(1) from the candidate table, the others are walked block by block from shared
//     memory and their copy-mode blocks marked.
//
// Traits (one per algorithm): BS block bytes, SIG signature bytes, MAXBLK = SIG + BS, NCAND = MAXBLK / 2, CH chunk bytes,
// NBB = bits of the per-chunk block count in a table row, consumed(sig) = bytes of an encoded block with that signature.
#pragma once
#include "common.cuh"
#include "cl_core.cuh"

namespace dns {
namespace bounds {

struct ChamT {   // chameleon.rs:138-147: 64 one-bit flags, hit -> 2 bytes, miss -> 4 bytes
    static constexpr uint32_t BS = 256, SIG = 8, MAXBLK = 264, NCAND = 132, CH = 16384, NBB = 8;
    static __device__ __forceinline__ uint32_t consumed(uint64_t sig) { return 264u - 2u * (uint32_t)__popcll(sig); }
};
struct CheeT {   // cheetah.rs:188-197
    static constexpr uint32_t BS = 128, SIG = 8, MAXBLK = 136, NCAND = 68, CH = 4096, NBB = 12;
    static __device__ __forceinline__ uint32_t consumed(uint64_t sig) { return cld::cheetah_block_bytes(sig); }
};
struct LionT {   // lion.rs:317-351: 6-byte signature
    static constexpr uint32_t BS = 64, SIG = 6, MAXBLK = 70, NCAND = 35, CH = 4096, NBB = 12;
    static __device__ __forceinline__ uint32_t consumed(uint64_t sig) { return cld::lion_block_bytes(sig & 0x0000FFFFFFFFFFFFull); }
};

constexpr int GROUP = 64;            // chunks per composition group
constexpr uint32_t TERM = 0xFFu;     // exit code: the walk reached the tail region / end of stream
constexpr uint32_t G_SKIP = 0xFEu;   // g_entry: dec_seq_walk handled this group chunk by chunk (c_entry already written)
constexpr unsigned long long BLK_COPY = 1ull << 63;   // blk_off flag: copy-mode block (raw BS bytes, no signature)

struct DecStatus {
    unsigned long long out_bytes;
    unsigned long long main_blocks;      // blocks decoded by the parallel main loop (codec.rs:88-100)
    unsigned long long tail_off;         // stream offset where the tail loop starts
    unsigned int nonquiet, error;        // nonquiet bit 0: copy-mode blocks present (cleared again by dec_seq_walk)
    unsigned int last_main_inc, seq;     // seq: the boundaries come from dec_seq_walk, automaton state below is valid
    unsigned int ps_penalty, ps_start, ps_prev, pad;   // protection state after the main loop (protection_state.rs:9-16)
    // the state the piece of a sharded stream is entered in (seeded = 1; dec_quiet_check copies it from the seed): the main loop and the
    // tail start from it instead of protection_state.rs:9-16. in_refused: the transfers composed to no state (the piece is refused)
    unsigned int seeded, in_penalty, in_start, in_prev, in_phase, in_refused;
};
// the incoming state of a seeded boundary walk, as density_b200_decode_shard_prot_phase1 composes it: {penalty, start,
// previous_incompressible, counter mod 16, refused}
constexpr uint32_t SEED_WORDS = 5;

__device__ __forceinline__ uint32_t ldu16(const uint8_t* p) { return *reinterpret_cast<const uint16_t*>(p); }
__device__ __forceinline__ uint64_t ldsig(const uint8_t* p) {   // 8 bytes at a 2-byte aligned address
    return (uint64_t)(ldu16(p) | (ldu16(p + 2) << 16)) | ((uint64_t)(ldu16(p + 4) | (ldu16(p + 6) << 16)) << 32);
}

// table row entry: exit_idx (8) | nblocks (NBB) | x, where x = term_rel when exit_idx == TERM (the walk ended inside this chunk at
// relative offset term_rel because fewer than MAXBLK bytes remain: that is where codec.rs's tail loop takes over), else the flags
// {bit 0: two consecutive incompressible blocks inside, bit 1: first block incompressible, bit 2: last block incompressible}.
template <class T> __device__ __forceinline__ uint32_t row_pack(uint32_t exitc, uint32_t nb, uint32_t x) { return exitc | (nb << 8) | (x << (8 + T::NBB)); }
template <class T> __device__ __forceinline__ uint32_t row_nb(uint32_t r) { return (r >> 8) & ((1u << T::NBB) - 1u); }
template <class T> __device__ __forceinline__ uint32_t row_x(uint32_t r) { return r >> (8 + T::NBB); }

// ---- 1a. candidate walks -----------------------------------------------------------------------------------------------
template <class T>
__global__ void __launch_bounds__(160) dec_chunk_walk(const uint8_t* __restrict__ in, uint64_t n, uint32_t nchunks, uint32_t* __restrict__ res) {
    constexpr uint32_t SM = T::CH + T::MAXBLK + 24;
    __shared__ __align__(16) uint8_t s[SM];
    const uint32_t c = blockIdx.x;
    const uint64_t base = (uint64_t)c * T::CH;
    for (uint32_t i = threadIdx.x * 2; i < SM; i += blockDim.x * 2) {
        const uint64_t g = base + i;
        *reinterpret_cast<uint16_t*>(s + i) = (g + 2 <= n) ? *reinterpret_cast<const uint16_t*>(in + g) : (uint16_t)((g < n) ? in[g] : 0);
    }
    __syncthreads();
    const uint32_t cand = threadIdx.x;
    if (cand >= T::NCAND) return;
    uint32_t off = cand * 2, nb = 0, exitc = TERM, term = 0;
    uint32_t pair = 0, first = 0, prev = 0;
    while (true) {
        if (off >= T::CH) { exitc = (off - T::CH) >> 1; break; }
        if (base + off + T::MAXBLK > n) { term = off; break; }
        const uint32_t consumed = T::consumed(ldsig(s + off));
        const uint32_t inc = consumed >= T::BS ? 1u : 0u;           // codec.rs:98
        if (nb == 0) first = inc;
        pair |= inc & prev;
        prev = inc;
        off += consumed;
        ++nb;
    }
    res[(size_t)c * T::NCAND + cand] = row_pack<T>(exitc, nb, exitc == TERM ? term : (pair | (first << 1) | (prev << 2)));
    (void)nchunks;
}

// ---- 1b. compose the maps of GROUP consecutive chunks ----------------------------------------------------------------------
// gres[g][cand] = {exit_idx (or TERM), blocks, term_chunk, term_rel}; exit_idx != TERM: z = the chunk flags composed along the path
// (bit 0: two consecutive incompressible blocks anywhere inside the group, bit 1: first block, bit 2: last block incompressible,
//  bit 3: short last group, which dec_seq_walk never jumps)
template <class T>
__global__ void dec_group_compose(const uint32_t* __restrict__ res, uint32_t nchunks, uint4* __restrict__ gres) {
    const uint32_t g = blockIdx.x, cand = threadIdx.x;
    if (cand >= T::NCAND) return;
    uint32_t idx = cand, blocks = 0, tchunk = 0, trel = 0;
    uint32_t pair = 0, first = 0, last = 0, have = 0;
    const uint32_t c0 = g * GROUP, c1 = min(nchunks, c0 + GROUP);
    for (uint32_t c = c0; c < c1; ++c) {
        const uint32_t r = res[(size_t)c * T::NCAND + idx];
        const uint32_t nb = row_nb<T>(r);
        blocks += nb;
        idx = r & 0xFFu;
        if (idx == TERM) { tchunk = c; trel = row_x<T>(r); break; }
        if (nb) {
            const uint32_t fl = row_x<T>(r);
            if (!have) { first = (fl >> 1) & 1u; have = 1; } else pair |= last & (fl >> 1) & 1u;
            pair |= fl & 1u;
            last = (fl >> 2) & 1u;
        }
    }
    if (idx != TERM) tchunk = pair | (first << 1) | (last << 2) | ((c1 - c0 < (uint32_t)GROUP) ? 8u : 0u);
    gres[(size_t)g * T::NCAND + cand] = make_uint4(idx, blocks, tchunk, trel);
}

// ---- 1c. walk the groups from the stream start ---------------------------------------------------------------------------
template <class T>
__global__ void dec_top_walk(const uint4* __restrict__ gres, uint32_t ngroups, uint64_t n, uint32_t* __restrict__ g_entry,
                             uint64_t* __restrict__ g_blockbase, DecStatus* __restrict__ st) {
    if (threadIdx.x || blockIdx.x) return;
    uint32_t idx = 0; uint64_t blocks = 0;
    bool done = false;
    for (uint32_t g = 0; g < ngroups; ++g) {
        g_entry[g] = done ? TERM : idx;
        g_blockbase[g] = blocks;
        if (done) continue;
        const uint4 r = gres[(size_t)g * T::NCAND + idx];
        blocks += r.y;
        idx = r.x;
        if (idx == TERM) { done = true; st->tail_off = (unsigned long long)r.z * T::CH + r.w; }
    }
    if (!done) st->tail_off = n;  // cannot happen for n > 0 (the last chunk always terminates); keeps the tail kernel safe
    st->main_blocks = blocks;
}

// ---- 1d. per chunk: true entry + block index -----------------------------------------------------------------------------
template <class T>
__global__ void dec_chunk_entries(const uint32_t* __restrict__ res, uint32_t nchunks, const uint32_t* __restrict__ g_entry,
                                  const uint64_t* __restrict__ g_blockbase, uint32_t ngroups, uint32_t* __restrict__ c_entry,
                                  uint64_t* __restrict__ c_blockbase, const DecStatus* __restrict__ only_if_seq) {
    if (only_if_seq && !only_if_seq->seq) return;
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= ngroups) return;
    uint32_t idx = g_entry[g]; uint64_t blocks = g_blockbase[g];
    if (idx == G_SKIP) return;
    const uint32_t c0 = g * GROUP, c1 = min(nchunks, c0 + GROUP);
    for (uint32_t c = c0; c < c1; ++c) {
        c_entry[c] = idx; c_blockbase[c] = blocks;
        if (idx == TERM) continue;
        const uint32_t r = res[(size_t)c * T::NCAND + idx];
        blocks += row_nb<T>(r);
        idx = r & 0xFFu;
    }
}

// ---- 1e. one offset per block ------------------------------------------------------------------------------------------------
template <class T>
__global__ void dec_block_offsets(const uint8_t* __restrict__ in, uint64_t n, uint32_t nchunks, const uint32_t* __restrict__ c_entry,
                                  const uint64_t* __restrict__ c_blockbase, uint64_t* __restrict__ blk_off, uint64_t maxblocks,
                                  const DecStatus* __restrict__ only_if_seq) {
    if (only_if_seq && !only_if_seq->seq) return;
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    const uint32_t e = c_entry[c];
    if (e == TERM) return;
    const uint64_t base = (uint64_t)c * T::CH;
    uint64_t b = c_blockbase[c];
    uint32_t off = e * 2;
    while (off < T::CH && base + off + T::MAXBLK <= n) {
        if (b < maxblocks) blk_off[b] = base + off;
        ++b;
        off += T::consumed(ldsig(in + base + off));
    }
}

// ---- 2. quiet check + capacity check -------------------------------------------------------------------------------------------
// seed (may be null): the incoming state of a piece (SEED_WORDS); the quiet path also needs penalty 0 on entry and no incompressible pair
// across the entry seam.
template <class T>
__global__ void dec_quiet_check(const uint8_t* __restrict__ in, const uint64_t* __restrict__ blk_off, uint64_t maxblocks, DecStatus* __restrict__ st, uint64_t cap,
                                const uint32_t* __restrict__ seed) {
    const uint64_t nb = st->main_blocks;
    const uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (seed && b == 0) {
        st->seeded = 1; st->in_penalty = seed[0]; st->in_start = seed[1]; st->in_prev = seed[2]; st->in_phase = seed[3]; st->in_refused = seed[4];
        if (seed[0] || (seed[2] && nb && T::consumed(ldsig(in)) >= T::BS)) atomicOr(&st->nonquiet, 1u);
    }
    // DENSITY_B200_ECAPACITY — unless the count is void because copy-mode blocks were misread as signatures: every block in front of the
    // first copy-mode block is read correctly, and that includes the incompressible pair that started the episode, so the blocks that
    // fit (blk_off holds no more) are enough to find it; dec_seq_walk then recounts and judges the capacity again
    if (b == 0 && nb * T::BS > cap) st->error = 2;
    if (b >= nb || b >= maxblocks) return;
    const bool inc = T::consumed(ldsig(in + blk_off[b])) >= T::BS;  // codec.rs:98
    if (b == nb - 1) st->last_main_inc = inc ? 1u : 0u;
    if (inc && b > 0) {
        if (T::consumed(ldsig(in + blk_off[b - 1])) >= T::BS) atomicOr(&st->nonquiet, 1u);
    }
}

// ---- 2b. in-order boundary walk for streams with copy-mode blocks (codec.rs:88-100 with protection_state.rs) ---------------------
// One CTA; thread 0 carries (stream offset, block count, protection state) through the stream chunk by chunk.
//  * A chunk is JUMPED in O(1) from dec_chunk_walk's table when the automaton provably stays in encoded mode inside it (penalty 0
//    on entry, no two consecutive incompressible blocks inside, none across the entry seam): all its blocks are encoded blocks, the
//    table row gives the exit offset and block count, and dec_block_offsets fills in the per-block offsets afterwards in parallel.
//  * Any other chunk is WALKED block by block from a shared-memory copy (the whole CTA stages it), marking copy-mode blocks.
constexpr int SW_THREADS = 256;
constexpr int SW_BATCH = 24;                 // table rows staged at a time
enum : uint32_t { SW_ROWS = 0, SW_DIRTY = 1, SW_DONE = 2 };
__device__ __forceinline__ uint4 sw_load16(const uint8_t* __restrict__ in, uint64_t g, uint64_t n, bool al16) {
    uint4 v = make_uint4(0, 0, 0, 0);
    if (al16 && g + 16 <= n) return *reinterpret_cast<const uint4*>(in + g);
    uint8_t* vb = reinterpret_cast<uint8_t*>(&v);
    for (int k = 0; k < 16; ++k) if (g + k < n) vb[k] = in[g + k];
    return v;
}
// Jump over nb blocks that never enter copy mode (protection_state.rs:18-24,37-47): the penalty start halves on every 16th block.
__device__ __forceinline__ void sw_jump(Protection& ps, uint32_t nb, uint32_t last_inc) {
    const uint64_t k = (ps.counter + nb + 15) / 16 - (ps.counter + 15) / 16;
    if (ps.copy_penalty_start > 1) { const uint32_t sh = k > 8 ? 8u : (uint32_t)k; const uint32_t v = ps.copy_penalty_start >> sh; ps.copy_penalty_start = v ? v : 1u; }
    ps.counter += nb;
    ps.previous_incompressible = last_inc;
}
// The stop-and-report mode (STOP = true, the range decode, DESIGN §4g): for the two block indices in `block`, where that block starts
// and the automaton state in front of it, to out[STOP_WORDS * i ..] = {1, stream offset, penalty | start << 8 | previous_incompressible
// << 16} when the main loop reaches it (block main_blocks included: the tail loop's start). In this mode the walk jumps no group and no
// chunk that holds a stop strictly inside, so it meets every stop on a block boundary.
constexpr uint32_t STOP_WORDS = 4;
struct WalkStops { uint64_t block[2]; unsigned long long* out; };
__device__ __forceinline__ unsigned long long stop_state(const Protection& ps) {
    return ps.copy_penalty | (ps.copy_penalty_start << 8) | ((unsigned long long)ps.previous_incompressible << 16);
}
// STOP: the state in front of block b at stream offset i; whether a stop lies strictly inside the nb blocks from block b
template <bool STOP>
__device__ __forceinline__ void stop_at(const WalkStops& w, uint64_t b, uint64_t i, const Protection& ps) {
    if constexpr (STOP)
        for (int k = 0; k < 2; ++k)
            if (b == w.block[k]) { unsigned long long* o = w.out + STOP_WORDS * k; o[0] = 1; o[1] = i; o[2] = stop_state(ps); }
}
template <bool STOP>
__device__ __forceinline__ bool stop_inside(const WalkStops& w, uint64_t b, uint32_t nb) {
    if constexpr (!STOP) return false;
    const uint64_t e = b + nb;
    return (w.block[0] > b && w.block[0] < e) || (w.block[1] > b && w.block[1] < e);
}
template <bool STOP>
struct PairStops {      // the walk's view of WalkStops
    WalkStops w;
    __device__ __forceinline__ void at(uint64_t b, uint64_t i, const Protection& ps) const { stop_at<STOP>(w, b, i, ps); }
    __device__ __forceinline__ bool inside(uint64_t b, uint32_t nb) const { return stop_inside<STOP>(w, b, nb); }
};
// The stride mode (the Chameleon seek index, DESIGN §4h): in front of every block b = j * every, 1 <= j <= max, out[STRIDE_WORDS (j - 1)
// ..] = {stream offset, the state as stop_state} when the main loop reaches it (block main_blocks included). As in the stop-and-report
// mode, the walk jumps no group and no chunk that holds such a block strictly inside.
constexpr uint32_t STRIDE_WORDS = 2;
struct StrideStops {
    uint64_t every, max; unsigned long long* out;
    __device__ __forceinline__ void at(uint64_t b, uint64_t i, const Protection& ps) const {
        const uint64_t j = b / every;
        if (b && j <= max && j * every == b) { unsigned long long* o = out + STRIDE_WORDS * (j - 1); o[0] = i; o[1] = stop_state(ps); }
    }
    __device__ __forceinline__ bool inside(uint64_t b, uint32_t nb) const { return nb > 1 && (b + nb - 1) / every > b / every; }
};
// The walk of both kernels below. Its pointers carry no __restrict__: the kernels' parameters state it, and restating it here gives the
// inlined body other alias scopes and dec_seq_walk<T, true> other code.
template <class T, class Stops>
__device__ __forceinline__ void seq_walk(const uint8_t* in, uint64_t n, uint64_t cap, uint32_t nchunks,
                                         const uint32_t* res, const uint4* gres, uint32_t ngroups,
                                         uint32_t* g_entry, uint64_t* g_blockbase,
                                         uint32_t* c_entry, uint64_t* c_blockbase,
                                         uint64_t* blk_off, uint64_t maxblocks, DecStatus* st, Stops stops) {
    if (!(st->nonquiet & 1u)) return;
    constexpr uint32_t SW_LOAD = T::CH + 16;            // + the signature bytes of a block starting at the chunk's last bytes, rounded up to 16
    __shared__ __align__(16) uint8_t win[2][SW_LOAD];   // the chunk being walked + the next one, prefetched during the walk
    __shared__ uint32_t rows[SW_BATCH * T::NCAND];
    __shared__ uint32_t s_cmd, s_chunk;
    const uint32_t tid = threadIdx.x;
    const bool al16 = (reinterpret_cast<uintptr_t>(in) & 15u) == 0;
    Protection ps; ps.init();
    if (st->seeded) { ps.copy_penalty = st->in_penalty; ps.copy_penalty_start = st->in_start; ps.previous_incompressible = st->in_prev; ps.counter = st->in_phase; }
    uint64_t idx = 0, b = 0;        // meaningful in thread 0 only
    uint32_t g_next = 0;            // first group not entered yet (thread 0)
    uint32_t cb = 0, cb_valid = 0;  // staged rows: chunks [cb, cb + cb_valid)
    uint32_t wchunk0 = 0xFFFFFFFFu, wchunk1 = 0xFFFFFFFFu;   // which chunk each window buffer holds (uniform over the CTA)
    while (true) {
        if (tid == 0) {
            uint32_t cmd = SW_DONE, c = 0;
            while (n - idx >= T::MAXBLK) {
                stops.at(b, idx, ps);
                c = (uint32_t)(idx / T::CH);
                const uint32_t e = (uint32_t)(idx - (uint64_t)c * T::CH) >> 1;          // < NCAND: a block is at most MAXBLK bytes
                if (c / GROUP == g_next) {
                    // entering a group of 64 chunks: jump over all of it if the automaton provably stays in encoded mode inside
                    const uint32_t g = g_next++;
                    const uint4 gr = gres[(size_t)g * T::NCAND + e];
                    if (ps.copy_penalty == 0 && gr.x != TERM && !(gr.z & 9u) && !(ps.previous_incompressible && (gr.z & 2u)) && !stops.inside(b, gr.y)) {
                        g_entry[g] = e; g_blockbase[g] = b;
                        sw_jump(ps, gr.y, (gr.z >> 2) & 1u);
                        b += gr.y;
                        idx = (uint64_t)(g + 1) * GROUP * T::CH + 2 * gr.x;
                        continue;
                    }
                    g_entry[g] = G_SKIP;                                             // chunk by chunk below
                }
                if (c < cb || c >= cb + cb_valid) { cmd = SW_ROWS; break; }
                const uint32_t r = rows[(c - cb) * T::NCAND + e];
                const uint32_t ex = r & 0xFFu, fl = row_x<T>(r);
                if (ps.copy_penalty == 0 && ex != TERM && !(fl & 1u) && !(ps.previous_incompressible && (fl & 2u)) && !stops.inside(b, row_nb<T>(r))) {
                    const uint32_t nb = row_nb<T>(r);
                    c_entry[c] = e; c_blockbase[c] = b;
                    sw_jump(ps, nb, (fl >> 2) & 1u);
                    b += nb;
                    idx = (uint64_t)(c + 1) * T::CH + 2 * ex;
                } else { cmd = SW_DIRTY; break; }
            }
            s_cmd = cmd; s_chunk = c;
        }
        __syncthreads();
        const uint32_t cmd = s_cmd, c = s_chunk;
        if (cmd == SW_DONE) break;
        if (cmd == SW_ROWS) {
            cb = c; cb_valid = (nchunks - c < (uint32_t)SW_BATCH) ? nchunks - c : (uint32_t)SW_BATCH;
            for (uint32_t i = tid; i < cb_valid * T::NCAND; i += SW_THREADS) rows[i] = res[(size_t)cb * T::NCAND + i];
        } else {
            const uint64_t wbase = (uint64_t)c * T::CH;
            int cur = (wchunk0 == c) ? 0 : (wchunk1 == c) ? 1 : -1;
            if (cur < 0) {                                                   // not prefetched: the whole CTA stages it now
                cur = 0; wchunk0 = c;
                for (uint32_t i = tid * 16; i < SW_LOAD; i += SW_THREADS * 16) *reinterpret_cast<uint4*>(win[0] + i) = sw_load16(in, wbase + i, n, al16);
                __syncthreads();
            }
            if (tid >= 32 && c + 1 < nchunks) {                              // the others fetch the next chunk while thread 0 walks this one
                constexpr int PER = (SW_LOAD / 16 + (SW_THREADS - 32) - 1) / (SW_THREADS - 32);
                uint4 v[PER];
#pragma unroll
                for (int t = 0; t < PER; ++t) {
                    const uint32_t i = ((tid - 32) + t * (SW_THREADS - 32)) * 16;
                    v[t] = (i < SW_LOAD) ? sw_load16(in, wbase + T::CH + i, n, al16) : make_uint4(0, 0, 0, 0);
                }
#pragma unroll
                for (int t = 0; t < PER; ++t) {
                    const uint32_t i = ((tid - 32) + t * (SW_THREADS - 32)) * 16;
                    if (i < SW_LOAD) *reinterpret_cast<uint4*>(win[cur ^ 1] + i) = v[t];
                }
            }
            if (c + 1 < nchunks) { if (cur) wchunk0 = c + 1; else wchunk1 = c + 1; }
            if (tid == 0) {
                const uint32_t* w32 = reinterpret_cast<const uint32_t*>(win[cur]);
                const uint64_t wend = wbase + T::CH;
                c_entry[c] = TERM;                                           // dec_block_offsets leaves this chunk alone
                while (idx < wend && n - idx >= T::MAXBLK) {
                    stops.at(b, idx, ps);
                    if (ps.revert_to_copy()) {                               // codec.rs:89-92
                        if (b < maxblocks) blk_off[b] = idx | BLK_COPY;
                        ++b; idx += T::BS; ps.decay();
                    } else {
                        const uint32_t o = (uint32_t)(idx - wbase), sh = (o & 2u) * 8;
                        const uint32_t w0 = w32[o >> 2], w1 = w32[(o >> 2) + 1], w2 = w32[(o >> 2) + 2];
                        const uint64_t sig = (uint64_t)__funnelshift_r(w0, w1, sh) | ((uint64_t)__funnelshift_r(w1, w2, sh) << 32);
                        const uint32_t consumed = T::consumed(sig);
                        if (b < maxblocks) blk_off[b] = idx;
                        ++b; idx += consumed; ps.update(consumed >= T::BS);   // codec.rs:94-98
                    }
                }
            }
        }
        __syncthreads();
    }
    // the chunk in which the main loop ended (if it was not walked it has no block either) and everything behind it carry no blocks
    {
        __shared__ uint32_t s_first_free, s_gnext;
        if (tid == 0) { s_first_free = (uint32_t)(idx / T::CH); s_gnext = g_next; }
        __syncthreads();
        for (uint32_t c = s_first_free + tid; c < nchunks; c += SW_THREADS) c_entry[c] = TERM;
        for (uint32_t g = s_gnext + tid; g < ngroups; g += SW_THREADS) g_entry[g] = G_SKIP;
    }
    if (tid == 0) {
        stops.at(b, idx, ps);
        st->main_blocks = b; st->tail_off = idx;
        st->ps_penalty = ps.copy_penalty; st->ps_start = ps.copy_penalty_start; st->ps_prev = ps.previous_incompressible;
        st->seq = 1;
        st->error = (b * T::BS > cap) ? 2u : 0u;     // the candidate walk's block count was void
        st->nonquiet &= ~1u;
    }
}
template <class T, bool STOP = false>
__global__ void __launch_bounds__(SW_THREADS) dec_seq_walk(const uint8_t* __restrict__ in, uint64_t n, uint64_t cap, uint32_t nchunks,
                                                           const uint32_t* __restrict__ res, const uint4* __restrict__ gres, uint32_t ngroups,
                                                           uint32_t* __restrict__ g_entry, uint64_t* __restrict__ g_blockbase,
                                                           uint32_t* __restrict__ c_entry, uint64_t* __restrict__ c_blockbase,
                                                           uint64_t* __restrict__ blk_off, uint64_t maxblocks, DecStatus* __restrict__ st,
                                                           WalkStops stops = WalkStops{}) {
    seq_walk<T>(in, n, cap, nchunks, res, gres, ngroups, g_entry, g_blockbase, c_entry, c_blockbase, blk_off, maxblocks, st, PairStops<STOP>{stops});
}
template <class T>
__global__ void __launch_bounds__(SW_THREADS) dec_seq_walk_stride(const uint8_t* __restrict__ in, uint64_t n, uint64_t cap, uint32_t nchunks,
                                                                  const uint32_t* __restrict__ res, const uint4* __restrict__ gres, uint32_t ngroups,
                                                                  uint32_t* __restrict__ g_entry, uint64_t* __restrict__ g_blockbase,
                                                                  uint32_t* __restrict__ c_entry, uint64_t* __restrict__ c_blockbase,
                                                                  DecStatus* __restrict__ st, StrideStops stops) {
    seq_walk<T>(in, n, cap, nchunks, res, gres, ngroups, g_entry, g_blockbase, c_entry, c_blockbase, nullptr, 0, st, stops);
}

// ---- 3. the map of a whole byte range (sharded decode of a stream whose cuts are not known) ----------------------------------------
// Folds the group rows of dec_group_compose over all `ngroups` groups of a range, for every candidate entry at once, and writes the
// range map (DENSITY_B200_LOCATE_MAP_WORDS u64): {n_range, n_halo}, then per candidate {exit index into the next range or ~0 (the walk
// reached the stream end), blocks}. With no groups (an empty range) every row is the identity. Each thread follows one candidate's
// chain of dependent rows; the whole CTA stages RC_BATCH groups of rows in shared memory at a time, so a link costs a shared load.
constexpr int RC_BATCH = 32;
constexpr int RC_THREADS = 256;
template <class T>
__global__ void __launch_bounds__(RC_THREADS) dec_range_compose(const uint4* __restrict__ gres, uint32_t ngroups, uint64_t n_range,
                                                                uint64_t n_halo, unsigned long long* __restrict__ map) {
    __shared__ uint2 rows[RC_BATCH * T::NCAND];     // {exit, blocks} of the staged groups
    const uint32_t tid = threadIdx.x;
    uint32_t idx = tid;
    unsigned long long blocks = 0;
    for (uint32_t g0 = 0; g0 < ngroups; g0 += RC_BATCH) {
        const uint32_t nb = min(ngroups - g0, (uint32_t)RC_BATCH);
        __syncthreads();
        for (uint32_t i = tid; i < nb * T::NCAND; i += RC_THREADS) {
            const uint4 r = gres[(size_t)g0 * T::NCAND + i];
            rows[i] = make_uint2(r.x, r.y);
        }
        __syncthreads();
        if (tid < T::NCAND && idx != TERM) {
            for (uint32_t g = 0; g < nb; ++g) {
                const uint2 r = rows[g * T::NCAND + idx];
                blocks += r.y;
                idx = r.x;
                if (idx == TERM) break;
            }
        }
    }
    if (tid < T::NCAND) {
        map[2 + 2 * tid] = idx == TERM ? ~0ull : (unsigned long long)idx;
        map[3 + 2 * tid] = blocks;
    }
    if (tid == 0) { map[0] = n_range; map[1] = n_halo; }
}

// ---- 3b. the start row of the range that holds the stream start (sharded Cheetah decode without known cuts) -------------------------
// The stream start's copy-mode blocks void the candidate walks of its range, so that range's exit comes from the exact boundary walk
// (bounds_launch over range + halo from the fresh automaton, copy-mode blocks included): the first block start >= n_range, found in
// blk_off, or the tail offset when the main loop ended behind n_range without another block start; ~0 when it ended (fewer than MAXBLK
// bytes left) in front of n_range, i.e. the stream ends inside this range or its halo. The exit is an index into the next range as in a
// candidate row, the block count includes the copy-mode blocks. Writes {range_offset, has_start_row, exit, blocks} to out4; st ==
// nullptr (a range without the stream start): {range_offset, 0, 0, 0}.
template <class T>
__global__ void dec_start_row(const DecStatus* __restrict__ st, const uint64_t* __restrict__ blk_off, uint64_t n_range, uint64_t range_offset,
                              unsigned long long* __restrict__ out4) {
    if (threadIdx.x || blockIdx.x) return;
    unsigned long long ex = 0, nb = 0;
    if (st) {
        const uint64_t mb = st->main_blocks;       // every block has its offset: the workspace holds one per T::SIG bytes
        uint64_t lo = 0, hi = mb;
        while (lo < hi) {
            const uint64_t mid = (lo + hi) >> 1;
            if ((blk_off[mid] & ~BLK_COPY) < n_range) lo = mid + 1; else hi = mid;
        }
        nb = lo;
        if (lo < mb) ex = ((blk_off[lo] & ~BLK_COPY) - n_range) >> 1;
        else if (st->tail_off >= n_range) ex = (st->tail_off - n_range) >> 1;
        else ex = ~0ull;
    }
    out4[0] = range_offset; out4[1] = st ? 1ull : 0ull; out4[2] = ex; out4[3] = nb;
}

// ---- 4. the protection transfer of a piece of a sharded stream (DESIGN §5) ----------------------------------------------------------
// A piece starts at a block boundary, in an automaton state and counter phase (revert_to_copy halves the start on every 16th block of
// the STREAM) that its decoder does not know. A decode candidate is (penalty 0..9, start 1..10, previous_incompressible, counter mod
// 16): PT_NCAND of them, candidate 0 the stream start. dec_prot_transfer walks codec.rs:88-100, copy-mode blocks included, from every
// candidate at once and writes one word per candidate where the walk leaves the piece at its CUT:
//  * known cuts (LOCATE false, cut == n, one CTA): the candidate at the piece end when the walk ends exactly on the cut, PT_ESC when
//    that state is not a candidate, PT_NOEND when it overshoots the cut, stops short of it or reads a malformed block;
//  * the protected range map (LOCATE true, DESIGN §5): in[0 .. n) is a range of `cut` bytes and its halo, and CTA e starts the walks
//    at the entry offset 2e. Its row of candidate c: the exit index x (the first block start at or after the cut is cut + 2x) and the
//    candidate there, packed by pt_row; PT_TERM when the main loop ends (fewer than MAXBLK bytes left) in front of the cut; PT_ESC when
//    the state at the exit is not a candidate; PT_NOEND for a head dropped at the cap. The range map is PT_MAP_HDR header words
//    {n_range lo, hi, n_halo lo, hi}, then the NCAND x PT_NCAND rows, entry-major.
// The walk follows HEADS keyed by (offset, state, phase), not candidates; heads that reach the same key merge for good, each candidate
// keeps the index of its head. All heads advance chunk by chunk: a head with penalty 0 jumps its group or its chunk in O(1) from the
// candidate rows (dec_seq_walk's rule), any other head walks the chunk block by block from shared memory, one thread per head. After a
// chunk step the heads are merged in a shared hash table; at most PT_CAP stay live, the candidates of the others get PT_NOEND (their
// piece is refused, never decoded wrong). tests/prot_decode_model.py and tests/prot_locate_model.py are the CPU twins.
constexpr uint32_t PT_NCAND = 3200, PT_ESC = 0xFFFFu, PT_NOEND = 0xFFFEu, PT_CAP = 256, PT_HT = 8192, PT_THREADS = 1024;
constexpr uint32_t PT_LIVE = 0xFFFFFFFFu, PT_DEAD = 0xFFFFu;
constexpr uint32_t PT_TERM = TERM, PT_MAP_HDR = 4;   // a range-map row whose walk reached the stream end; the map's header words
// a range-map row: exit index (bits 0-7, < NCAND) | exit candidate (bits 8-23). No row equals PT_ESC or PT_NOEND: their low byte
// would be TERM or 0xFE, and a PT_TERM row is TERM alone.
__host__ __device__ __forceinline__ uint32_t pt_row(uint32_t exit_idx, uint32_t cand) { return exit_idx | (cand << 8); }
__host__ __device__ __forceinline__ uint32_t pt_pack(uint32_t pen, uint32_t start, uint32_t prev, uint32_t phase) {
    return pen | (start << 8) | (prev << 16) | (phase << 17);
}
__host__ __device__ __forceinline__ uint32_t pt_cand(uint32_t s) {     // packed state -> candidate, PT_ESC outside the set
    const uint32_t pen = s & 0xFFu, start = (s >> 8) & 0xFFu, prev = (s >> 16) & 1u, phase = s >> 17;
    if (pen >= 10u || start < 1u || start > 10u) return PT_ESC;
    return phase * 200u + (prev * 10u + (start - 1u)) * 10u + pen;
}
__host__ __device__ __forceinline__ uint32_t pt_state(uint32_t c) {    // candidate -> packed state
    const uint32_t pc = c % 200u;
    return pt_pack(pc % 10u, (pc / 10u) % 10u + 1u, pc / 100u, c / 200u);
}
// nb encoded blocks with penalty 0 (sw_jump on a packed state)
__device__ __forceinline__ uint32_t pt_jump(uint32_t s, uint32_t nb, uint32_t last_inc) {
    uint32_t start = (s >> 8) & 0xFFu;
    const uint32_t ph = s >> 17;
    const uint32_t k = (ph + nb + 15) / 16 - (ph + 15) / 16;
    if (start > 1) { start >>= (k > 8 ? 8u : k); if (!start) start = 1; }
    return pt_pack(0, start, last_inc, (ph + nb) & 15u);
}
// the word of a head that reached off >= cut in state s (see dec_prot_transfer)
__device__ __forceinline__ uint32_t pt_exit(uint64_t off, uint32_t s, uint64_t cut, int locate) {
    const uint32_t c = pt_cand(s);
    if (!locate) return off == cut ? c : PT_NOEND;
    return c == PT_ESC ? PT_ESC : pt_row((uint32_t)((off - cut) >> 1), c);
}
struct PtSmem {
    unsigned long long off[2][PT_NCAND];    // head offsets in the piece, double-buffered across a merge
    uint32_t st[2][PT_NCAND];               // packed head states
    uint32_t end[PT_NCAND];                 // PT_LIVE, PT_LIVE - 1 (walks this chunk block by block), or the head's result
    uint16_t newid[PT_NCAND];               // merge: the hash slot, then the head's index after the merge (PT_DEAD: dropped)
    uint16_t cand_head[PT_NCAND];
    unsigned long long ht_key[PT_HT];
    uint16_t ht_val[PT_HT];
    uint32_t nh, nnew, need_win, min_chunk;
};
template <class T, bool LOCATE>
__global__ void __launch_bounds__(PT_THREADS, 1)
dec_prot_transfer(const uint8_t* __restrict__ in, uint64_t n, uint64_t cut, int is_last, const uint32_t* __restrict__ res,
                  const uint4* __restrict__ gres, uint32_t* __restrict__ out) {
    constexpr int locate = LOCATE ? 1 : 0;
    constexpr uint32_t SW_LOAD = T::CH + 16;
    extern __shared__ __align__(16) unsigned char pt_raw[];
    uint8_t* win = pt_raw;
    PtSmem& S = *reinterpret_cast<PtSmem*>(pt_raw + SW_LOAD);
    const uint32_t tid = threadIdx.x;
    const uint64_t entry = 2ull * blockIdx.x;
    if (locate) {
        if (blockIdx.x == 0 && tid < PT_MAP_HDR) out[tid] = (uint32_t)((tid < 2 ? cut : n - cut) >> (32 * (tid & 1)));
        out += PT_MAP_HDR + (size_t)blockIdx.x * PT_NCAND;
    }
    if (is_last || cut == 0) {        // the last piece's transfer is never composed; an empty piece or range is the identity
        for (uint32_t c = tid; c < PT_NCAND; c += PT_THREADS) out[c] = is_last ? PT_NOEND : pt_exit(entry, pt_state(c), 0, locate);
        return;
    }
    const bool al16 = (reinterpret_cast<uintptr_t>(in) & 15u) == 0;
    const uint32_t nchunks = (uint32_t)((cut + T::CH - 1) / T::CH);
    for (uint32_t c = tid; c < PT_NCAND; c += PT_THREADS) { S.off[0][c] = entry; S.st[0][c] = pt_state(c); S.cand_head[c] = (uint16_t)c; }
    if (tid == 0) S.nh = PT_NCAND;
    uint32_t cur = 0;
    __syncthreads();
    for (uint32_t c = 0; c < nchunks;) {
        const uint32_t nh = S.nh;
        const uint64_t cbase = (uint64_t)c * T::CH, cend = cbase + T::CH;
        if (tid == 0) { S.need_win = 0; S.nnew = 0; S.min_chunk = 0xFFFFFFFFu; }
        for (uint32_t i = tid; i < PT_HT; i += PT_THREADS) S.ht_key[i] = 0;
        __syncthreads();
        // 1. jumps from the group and chunk rows
        for (uint32_t h = tid; h < nh; h += PT_THREADS) {
            uint64_t off = S.off[cur][h];
            uint32_t s = S.st[cur][h], e = PT_LIVE;
            if (off < cend) {                                  // otherwise a group jump took it past this chunk
                const uint32_t ent = (uint32_t)(off - cbase) >> 1, prev = (s >> 16) & 1u;
                bool jumped = false;
                if ((s & 0xFFu) == 0 && c % GROUP == 0) {
                    const uint4 gr = gres[(size_t)(c / GROUP) * T::NCAND + ent];
                    if (gr.x != TERM && !(gr.z & 9u) && !(prev && (gr.z & 2u))) {
                        s = pt_jump(s, gr.y, (gr.z >> 2) & 1u); off = cbase + (uint64_t)GROUP * T::CH + 2 * gr.x; jumped = true;
                    }
                }
                if (!jumped && (s & 0xFFu) == 0) {
                    const uint32_t r = res[(size_t)c * T::NCAND + ent];
                    const uint32_t ex = r & 0xFFu, fl = row_x<T>(r);
                    if (ex != TERM && !(fl & 1u) && !(prev && (fl & 2u))) {
                        s = pt_jump(s, row_nb<T>(r), (fl >> 2) & 1u); off = cend + 2 * ex; jumped = true;
                    }
                }
                if (!jumped) { e = PT_LIVE - 1; S.need_win = 1; }
                else if (off >= cut) e = pt_exit(off, s, cut, locate);
            }
            S.off[cur][h] = off; S.st[cur][h] = s; S.end[h] = e;
        }
        __syncthreads();
        // 2. the heads that could not jump walk the chunk block by block
        if (S.need_win) {
            for (uint32_t i = tid * 16; i < SW_LOAD; i += PT_THREADS * 16) *reinterpret_cast<uint4*>(win + i) = sw_load16(in, cbase + i, n, al16);
            __syncthreads();
            for (uint32_t h = tid; h < nh; h += PT_THREADS) {
                if (S.end[h] != PT_LIVE - 1) continue;
                uint64_t off = S.off[cur][h];
                uint32_t s = S.st[cur][h], e = PT_LIVE;
                uint32_t pen = s & 0xFFu, start = (s >> 8) & 0xFFu, prev = (s >> 16) & 1u, ph = s >> 17;
                const uint64_t stop = cend < cut ? cend : cut;
                while (off < stop) {                           // codec.rs:88-98; every block of a non-final piece is a main-loop block
                    if (locate && off + T::MAXBLK > n) { e = PT_TERM; break; }   // the main loop ends in front of the cut
                    if (ph == 0 && start > 1) start >>= 1;
                    ph = (ph + 1) & 15u;
                    if (pen) {
                        pen = (pen - 1) & 0xFFu;
                        if (!pen) start = (start + 1) & 0xFFu;
                        off += T::BS;
                    } else {
                        if (off + T::SIG > n) { e = PT_NOEND; break; }
                        const uint8_t* p = win + (uint32_t)(off - cbase);
                        const uint32_t con = T::consumed(ldsig(p));
                        if (con >= T::BS) { if (prev) pen = start; prev = 1; } else prev = 0;
                        off += con;
                    }
                    if (off > n) { e = PT_NOEND; break; }
                }
                s = pt_pack(pen, start, prev, ph);
                if (e == PT_LIVE && off >= cut) e = pt_exit(off, s, cut, locate);
                S.off[cur][h] = off; S.st[cur][h] = s; S.end[h] = e;
            }
        }
        __syncthreads();
        // 3. merge: one head per key (offset, state, phase); the winners take the next indices, up to PT_CAP
        for (uint32_t h = tid; h < nh; h += PT_THREADS) {
            if (S.end[h] != PT_LIVE) continue;
            const uint64_t off = S.off[cur][h];
            const unsigned long long key = (((unsigned long long)(off - cend) << 21) | S.st[cur][h]) + 1ull;
            uint32_t slot = (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> 51) & (PT_HT - 1);
            while (true) {
                const unsigned long long was = atomicCAS(&S.ht_key[slot], 0ull, key);
                if (was == 0ull) { S.ht_val[slot] = (uint16_t)atomicAdd(&S.nnew, 1u); atomicMin(&S.min_chunk, (uint32_t)(off / T::CH)); break; }
                if (was == key) break;
                slot = (slot + 1) & (PT_HT - 1);
            }
            S.newid[h] = (uint16_t)slot;
        }
        __syncthreads();
        for (uint32_t h = tid; h < nh; h += PT_THREADS) {
            if (S.end[h] != PT_LIVE) continue;
            const uint32_t id = S.ht_val[S.newid[h]];
            S.newid[h] = id < PT_CAP ? (uint16_t)id : (uint16_t)PT_DEAD;
        }
        __syncthreads();
        // the winners move to the next buffer; every candidate follows its head, or takes its result
        for (uint32_t h = tid; h < nh; h += PT_THREADS) {
            if (S.end[h] != PT_LIVE) continue;
            const uint32_t id = S.newid[h];
            if (id != PT_DEAD) { S.off[cur ^ 1][id] = S.off[cur][h]; S.st[cur ^ 1][id] = S.st[cur][h]; }
        }
        for (uint32_t k = tid; k < PT_NCAND; k += PT_THREADS) {
            const uint32_t h = S.cand_head[k];
            if (h == PT_DEAD) continue;
            const uint32_t e = S.end[h];
            uint32_t nid = PT_DEAD;
            if (e != PT_LIVE) out[k] = e;
            else if ((nid = S.newid[h]) == PT_DEAD) out[k] = PT_NOEND;
            S.cand_head[k] = (uint16_t)nid;
        }
        __syncthreads();
        if (tid == 0) S.nh = S.nnew < PT_CAP ? S.nnew : PT_CAP;
        cur ^= 1;
        const uint32_t next = S.min_chunk;
        __syncthreads();
        if (S.nh == 0) break;
        c = next > c + 1 ? next : c + 1;
    }
    for (uint32_t k = tid; k < PT_NCAND; k += PT_THREADS) if (S.cand_head[k] != PT_DEAD) out[k] = PT_NOEND;   // cannot happen: the piece ends
}
template <class T> constexpr size_t prot_transfer_smem() { return T::CH + 16 + sizeof(PtSmem); }

// The incoming state of piece `rank` (SEED_WORDS): the transfers of the pieces before it (dec_prot_transfer, [rank][PT_NCAND]) composed
// from candidate x0 (0, the stream start, for known cuts; a located piece's entry candidate with rank 0). A path that meets PT_ESC or
// PT_NOEND refuses the piece; the kernels then run from the stream-start state, harmlessly. Static: every decoder's translation unit
// launches its own copy.
static __global__ void dec_prot_enter_k(const uint32_t* __restrict__ all_transfers, uint32_t rank, uint32_t x0, uint32_t* __restrict__ seed) {
    if (threadIdx.x || blockIdx.x) return;
    uint32_t x = x0;
    for (uint32_t r = 0; r < rank && x < PT_NCAND; ++r) x = all_transfers[(size_t)r * PT_NCAND + x];
    const uint32_t refused = x < PT_NCAND ? 0u : 1u;
    const uint32_t s = pt_state(refused ? 0u : x);
    seed[0] = s & 0xFFu; seed[1] = (s >> 8) & 0xFFu; seed[2] = (s >> 16) & 1u; seed[3] = s >> 17; seed[4] = refused;
}

// ---- 5. the located piece of a stream without known cuts, from the protected range maps of all ranks (DESIGN §5) --------------------
// Shared by density_b200_prot_locate_piece (host) and dec_prot_compose_k (device). maps: `world` range maps of PT_MAP_HDR + NC x
// PT_NCAND u32 (dec_prot_transfer<T, true>) in rank order. Checks the layout (non-last ranges multiples of PL_RANGE_UNIT, each
// halo min(PL_HALO, the bytes of the later ranges), no overflow) and every row on the path, then walks from (entry 0, candidate 0) of the
// first non-empty range; an empty range passes the entry on. The walk covers every range, not only those before `rank`, so that a
// refusal anywhere (a PT_ESC or PT_NOEND row on the path) is known on every rank alike. out6 = {start, end, is_final, is_first, entry
// candidate, refused}: this rank's piece is d_in[start .. end) entered in that candidate; a refused path zeroes the others.
enum : int { PL_OK = 0, PL_ERR_MULTIPLE, PL_ERR_HALO, PL_ERR_OVERFLOW, PL_ERR_ROW };
constexpr uint64_t PL_RANGE_UNIT = 16384, PL_HALO = 264;
template <uint32_t NC>
__host__ __device__ inline int prot_locate_walk(const uint32_t* maps, int world, int rank, uint64_t out6[6]) {
    constexpr uint64_t MW = PT_MAP_HDR + (uint64_t)NC * PT_NCAND;
    auto hdr = [&](int r, int k) { const uint32_t* m = maps + (size_t)r * MW; return (uint64_t)m[2 * k] | ((uint64_t)m[2 * k + 1] << 32); };
    uint64_t later = 0;                 // stream bytes behind range r
    for (int r = world - 1; r >= 0; --r) {
        const uint64_t nr = hdr(r, 0), nh = hdr(r, 1);
        if (r < world - 1 && nr % PL_RANGE_UNIT) return PL_ERR_MULTIPLE;
        if (nh != (later < PL_HALO ? later : PL_HALO)) return PL_ERR_HALO;
        if (nr > ~later) return PL_ERR_OVERFLOW;
        later += nr;
    }
    for (int k = 0; k < 6; ++k) out6[k] = 0;
    uint32_t idx = 0, cand = 0;
    bool started = false, ended = false;     // a non-empty range was passed; a walk reached the stream end
    for (int r = 0; r < world; ++r) {
        const uint64_t nr = hdr(r, 0), nh = hdr(r, 1);
        if (ended || nr == 0) {              // a piece behind the stream end, or an empty range: empty, the entry passes on
            if (r == rank) out6[2] = ended || nh == 0;
            continue;
        }
        const uint32_t row = maps[(size_t)r * MW + PT_MAP_HDR + (size_t)idx * PT_NCAND + cand];
        if (row == PT_ESC || row == PT_NOEND) { for (int k = 0; k < 5; ++k) out6[k] = 0; out6[5] = 1; return PL_OK; }
        const uint32_t x = row & 0xFFu;
        uint64_t end;
        if (x == PT_TERM) {
            if (row != PT_TERM) return PL_ERR_ROW;
            end = nr + nh; ended = true;
        } else {
            if (x >= NC || (row >> 8) >= PT_NCAND) return PL_ERR_ROW;
            end = nr + 2 * x;
        }
        if (2ull * idx > end || end > nr + nh) return PL_ERR_ROW;
        if (r == rank) { out6[0] = 2ull * idx; out6[1] = end; out6[2] = end == nr + nh; out6[3] = !started; out6[4] = cand; }
        if (!ended) { idx = x; cand = row >> 8; }
        started = true;
    }
    return PL_OK;
}
// the device twin for the NCCL drivers: out8 = {out6, rc, 0}, so that one small copy brings the piece to the host
template <uint32_t NC>
__global__ void dec_prot_compose_k(const uint32_t* __restrict__ maps, int world, int rank, unsigned long long* __restrict__ out8) {
    if (threadIdx.x || blockIdx.x) return;
    uint64_t o[6];
    const int rc = prot_locate_walk<NC>(maps, world, rank, o);
    for (int k = 0; k < 6; ++k) out8[k] = o[k];
    out8[6] = (unsigned long long)rc; out8[7] = 0;
}

// The automaton state behind the main loop: dec_seq_walk's, or (quiet: penalty 0 throughout) the entry state jumped over the main
// blocks. Entry state: protection_state.rs:9-16, or the seed of a piece of a sharded stream. Unseeded, this is counter = main_blocks,
// start 1 and the last main block's incompressible bit (or dec_seq_walk's state).
__device__ __forceinline__ Protection main_end_state(const DecStatus* __restrict__ st) {
    Protection ps; ps.init();
    if (st->seeded) { ps.copy_penalty = st->in_penalty; ps.copy_penalty_start = st->in_start; ps.previous_incompressible = st->in_prev; ps.counter = st->in_phase; }
    if (st->seq) {
        ps.copy_penalty = st->ps_penalty; ps.copy_penalty_start = st->ps_start; ps.previous_incompressible = st->ps_prev;
        ps.counter += st->main_blocks;
    } else if (st->main_blocks) {
        const uint64_t k = (ps.counter + st->main_blocks + 15) / 16 - (ps.counter + 15) / 16;
        if (ps.copy_penalty_start > 1) { const uint32_t sh = k > 8 ? 8u : (uint32_t)k; const uint32_t v = ps.copy_penalty_start >> sh; ps.copy_penalty_start = v ? v : 1u; }
        ps.counter += st->main_blocks;
        ps.previous_incompressible = st->last_main_inc;
    }
    return ps;
}

// Chameleon's tail loop (codec.rs:102-123, chameleon_decode.cu dec_tail) as it goes through the tail's blocks, without output: plain(q)
// sees every PLAIN quad in stream order, `out` counts the bytes dec_tail writes. The control flow does not depend on the dictionary, so
// this runs before the carry-in is known (sharded decode) or without any dictionary at all (the decoded-size query).
struct TailWalk {
    uint64_t blocks;        // blocks the tail loop entered (copy-mode, encoded, partial)
    uint64_t out;           // bytes the tail decodes to (meaningless when bad)
    uint32_t first_inc;     // the first tail block is a complete incompressible block
    uint32_t copied, bad;   // a copy-mode block; a malformed block
    Protection ps;          // protection state when the tail loop stops
};
// at_block(j, offset, state) sees the tail's block j before the tail loop enters it (the range decode's stops behind the main loop)
struct NoBlockHook { __device__ void operator()(uint64_t, uint64_t, const Protection&) const {} };
template <class F, class G = NoBlockHook>
__device__ TailWalk tail_walk(const uint8_t* __restrict__ in, uint64_t n, const DecStatus* __restrict__ st, F plain, G at_block = G()) {
    TailWalk w; w.blocks = 0; w.out = 0; w.first_inc = 0; w.copied = 0; w.bad = 0;
    Protection& ps = w.ps;
    ps = main_end_state(st);
    uint64_t idx = st->tail_off;
    while (n - idx > 0) {
        at_block(w.blocks, idx, ps);
        ++w.blocks;
        if (ps.revert_to_copy()) {
            w.copied = 1;
            const uint64_t rem = n - idx, len = rem > 256 ? 256 : rem;
            idx += len; w.out += len;
            if (rem <= 256) break;
            ps.decay();
            continue;
        }
        const uint64_t mark = idx;
        if (n - idx < 8) { w.bad = 1; break; }
        uint64_t sig = 0;
        for (int i = 0; i < 8; ++i) sig |= (uint64_t)in[idx + i] << (8 * i);
        idx += 8;
        bool end = false;
        for (int u = 0; u < 32 && !end && !w.bad; ++u) {
            const bool checked = (n - idx) < 8;
            for (int k = 0; k < 2 && !end; ++k) {
                const uint32_t fl = (uint32_t)(sig & 1); sig >>= 1;
                if (checked && fl == 0) {
                    const uint64_t rem = n - idx;
                    if (rem == 0) { end = true; break; }
                    if (rem < 4) { idx = n; w.out += rem; end = true; break; }
                }
                if (fl) {
                    if (n - idx < 2) { w.bad = 1; break; }
                    idx += 2;
                } else {
                    if (n - idx < 4) { w.bad = 1; break; }
                    plain(in[idx] | (in[idx + 1] << 8) | (in[idx + 2] << 16) | ((uint32_t)in[idx + 3] << 24));
                    idx += 4;
                }
                w.out += 4;
            }
        }
        if (end || w.bad) break;
        const bool inc = idx - mark >= 256;
        if (w.blocks == 1) w.first_inc = inc ? 1u : 0u;
        ps.update(inc);
    }
    return w;
}

// ---- host side: workspace layout + launch sequence ---------------------------------------------------------------------------------
struct BoundsLayout { size_t status, res, gres, g_entry, g_blockbase, c_entry, c_blockbase, blk_off, total; uint64_t maxblocks; };

template <class T>
inline size_t bounds_layout(size_t nbytes, size_t cap, BoundsLayout* L) {
    const uint64_t nchunks = (nbytes + T::CH - 1) / T::CH;
    const uint64_t ngroups = (nchunks + GROUP - 1) / GROUP;
    const uint64_t minblk = T::SIG + (T::BS == 256 ? 128 : 0);     // smallest encoded block: Chameleon 8 + 64 * 2, Cheetah 8, Lion 6
    L->maxblocks = nbytes / minblk + 2;                            // what the stream can hold ...
    if (L->maxblocks > cap / T::BS + 2) L->maxblocks = cap / T::BS + 2;   // ... and what the output can take (more is a capacity error)
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
    L->status = take(sizeof(DecStatus));
    L->res = take(nchunks * T::NCAND * sizeof(uint32_t));
    L->gres = take(ngroups * T::NCAND * sizeof(uint4));
    L->g_entry = take(ngroups * sizeof(uint32_t));
    L->g_blockbase = take(ngroups * sizeof(uint64_t));
    L->c_entry = take(nchunks * sizeof(uint32_t));
    L->c_blockbase = take(nchunks * sizeof(uint64_t));
    L->blk_off = take(L->maxblocks * sizeof(uint64_t));
    L->total = off;
    return off;
}

// Enqueues the candidate rows of the chunks of d_in[0 .. n_walk) into the res / gres arrays of L: dec_chunk_walk, whose walks see
// n_visible >= n_walk bytes (a range map's halo is visible to the walks of the range's last chunk), then dec_group_compose. Nothing for
// an empty walk. Returns the number of groups.
template <class T>
inline uint32_t rows_launch(const uint8_t* d_in, size_t n_walk, size_t n_visible, uint8_t* ws, const BoundsLayout& L, cudaStream_t stream,
                            uint64_t* launches) {
    const uint32_t nchunks = (uint32_t)((n_walk + T::CH - 1) / T::CH);
    const uint32_t ngroups = (nchunks + GROUP - 1) / GROUP;
    if (!nchunks) return 0;
    uint32_t* res = reinterpret_cast<uint32_t*>(ws + L.res);
    dec_chunk_walk<T><<<nchunks, 160, 0, stream>>>(d_in, n_visible, nchunks, res);
    dec_group_compose<T><<<ngroups, 160, 0, stream>>>(res, nchunks, reinterpret_cast<uint4*>(ws + L.gres));
    *launches += 2;
    return ngroups;
}

// Enqueues the exact in-order main loop of the whole stream d_in[0 .. n), n > 0, with no block offsets stored and no capacity (the
// decoded-size query and the range decode's locate step): a fresh status with nonquiet bit 0 set, which is dec_seq_walk's gate (the
// little-endian low byte of the word), the candidate rows, then dec_seq_walk, in stop-and-report mode when STOP. Afterwards (on the
// stream) st->main_blocks / tail_off and the automaton state behind the main loop. 3 kernels; the scratch is bounds_layout<T>(n, 0).
// STRIDE: dec_seq_walk_stride with the stops `stride` instead (the seek index's build).
template <class T, bool STOP = false, bool STRIDE = false>
inline cudaError_t forced_walk_launch(const uint8_t* d_in, size_t n, uint8_t* ws, const BoundsLayout& L, cudaStream_t stream, uint64_t* launches,
                                      WalkStops stops = WalkStops{}, StrideStops stride = StrideStops{}) {
    DecStatus* st = reinterpret_cast<DecStatus*>(ws + L.status);
    cudaError_t e = cudaMemsetAsync(st, 0, sizeof(DecStatus), stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(&st->nonquiet, 1, 1, stream);
    if (e != cudaSuccess) return e;
    const uint32_t nchunks = (uint32_t)((n + T::CH - 1) / T::CH);
    const uint32_t ngroups = rows_launch<T>(d_in, n, n, ws, L, stream, launches);
    const uint32_t* res = reinterpret_cast<const uint32_t*>(ws + L.res);
    const uint4* gres = reinterpret_cast<const uint4*>(ws + L.gres);
    uint32_t* g_entry = reinterpret_cast<uint32_t*>(ws + L.g_entry);
    uint64_t* g_blockbase = reinterpret_cast<uint64_t*>(ws + L.g_blockbase);
    uint32_t* c_entry = reinterpret_cast<uint32_t*>(ws + L.c_entry);
    uint64_t* c_blockbase = reinterpret_cast<uint64_t*>(ws + L.c_blockbase);
    if constexpr (STRIDE)
        dec_seq_walk_stride<T><<<1, SW_THREADS, 0, stream>>>(d_in, n, ~0ull, nchunks, res, gres, ngroups, g_entry, g_blockbase, c_entry, c_blockbase,
                                                             st, stride);
    else
        dec_seq_walk<T, STOP><<<1, SW_THREADS, 0, stream>>>(d_in, n, ~0ull, nchunks, res, gres, ngroups, g_entry, g_blockbase, c_entry, c_blockbase,
                                                            nullptr, 0, st, stops);
    ++*launches;
    return cudaGetLastError();
}

// Enqueues the boundary kernels. Afterwards (on the stream): st->main_blocks / tail_off / protection state, blk_off[0 .. main_blocks).
// d_seed (may be null): the incoming state of a piece of a sharded stream (SEED_WORDS, read on the device); rows_ready: dec_chunk_walk and
// dec_group_compose already filled res / gres for this input (dec_prot_transfer needed them first).
template <class T>
inline cudaError_t bounds_launch(const uint8_t* d_in, size_t nbytes, size_t cap, uint8_t* ws, const BoundsLayout& L, cudaStream_t stream, uint64_t* launches,
                                 const uint32_t* d_seed = nullptr, bool rows_ready = false) {
    DecStatus* st = reinterpret_cast<DecStatus*>(ws + L.status);
    cudaError_t e = cudaMemsetAsync(st, 0, sizeof(DecStatus), stream);
    if (e != cudaSuccess) return e;
    const uint32_t nchunks = (uint32_t)((nbytes + T::CH - 1) / T::CH);
    const uint32_t ngroups = (nchunks + GROUP - 1) / GROUP;
    uint32_t* res = reinterpret_cast<uint32_t*>(ws + L.res);
    uint4* gres = reinterpret_cast<uint4*>(ws + L.gres);
    uint32_t* g_entry = reinterpret_cast<uint32_t*>(ws + L.g_entry);
    uint64_t* g_bb = reinterpret_cast<uint64_t*>(ws + L.g_blockbase);
    uint32_t* c_entry = reinterpret_cast<uint32_t*>(ws + L.c_entry);
    uint64_t* c_bb = reinterpret_cast<uint64_t*>(ws + L.c_blockbase);
    uint64_t* blk_off = reinterpret_cast<uint64_t*>(ws + L.blk_off);
    if (!rows_ready) rows_launch<T>(d_in, nbytes, nbytes, ws, L, stream, launches);
    dec_top_walk<T><<<1, 32, 0, stream>>>(gres, ngroups, nbytes, g_entry, g_bb, st);
    dec_chunk_entries<T><<<(ngroups + 127) / 128, 128, 0, stream>>>(res, nchunks, g_entry, g_bb, ngroups, c_entry, c_bb, nullptr);
    dec_block_offsets<T><<<(nchunks + 127) / 128, 128, 0, stream>>>(d_in, nbytes, nchunks, c_entry, c_bb, blk_off, L.maxblocks, nullptr);
    dec_quiet_check<T><<<(unsigned)((L.maxblocks + 255) / 256), 256, 0, stream>>>(d_in, blk_off, L.maxblocks, st, cap, d_seed);
    // streams with copy-mode blocks only (the three kernels return at once otherwise): in-order walk, then the entries of the chunks of
    // jumped groups and the offsets of the blocks of jumped chunks
    dec_seq_walk<T><<<1, SW_THREADS, 0, stream>>>(d_in, nbytes, cap, nchunks, res, gres, ngroups, g_entry, g_bb, c_entry, c_bb, blk_off, L.maxblocks, st);
    dec_chunk_entries<T><<<(ngroups + 127) / 128, 128, 0, stream>>>(res, nchunks, g_entry, g_bb, ngroups, c_entry, c_bb, st);
    dec_block_offsets<T><<<(nchunks + 127) / 128, 128, 0, stream>>>(d_in, nbytes, nchunks, c_entry, c_bb, blk_off, L.maxblocks, st);
    *launches += 7;
    return cudaGetLastError();
}

// Enqueues the range map of d_in[0 .. n_range + n_halo) into map (DENSITY_B200_LOCATE_MAP_WORDS u64 for ChamT): the candidate rows of the
// range's chunks, then their composition over the whole range. The scratch is the res / gres arrays of bounds_layout<T>(n_range + n_halo).
template <class T>
inline void range_map_launch(const uint8_t* d_in, size_t n_range, size_t n_halo, uint8_t* ws, unsigned long long* map, cudaStream_t stream,
                             uint64_t* launches) {
    BoundsLayout B; bounds_layout<T>(n_range + n_halo, 0, &B);
    const uint32_t ngroups = rows_launch<T>(d_in, n_range, n_range + n_halo, ws, B, stream, launches);
    dec_range_compose<T><<<1, RC_THREADS, 0, stream>>>(reinterpret_cast<const uint4*>(ws + B.gres), ngroups, n_range, n_halo, map);
    ++*launches;
}

// The dynamic shared memory of dec_prot_transfer<T, LOCATE>, allowed once per process. Static, as are the two launchers that call it: the
// build has no relocatable device code, so every translation unit that launches dec_prot_transfer has its own copy of the kernel, whose
// attribute it must set itself.
template <class T, bool LOCATE>
static cudaError_t prot_transfer_attr() {
    static_assert(prot_transfer_smem<T>() <= 227u * 1024u, "the head walk's shared memory must fit in one SM");
    static bool attr_done = false;
    if (!attr_done) {
        const cudaError_t e = cudaFuncSetAttribute(dec_prot_transfer<T, LOCATE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   (int)prot_transfer_smem<T>());
        if (e != cudaSuccess) return e;
        attr_done = true;
    }
    return cudaSuccess;
}

// Enqueues the protection transfer of the piece d_in[0 .. n) (PT_NCAND words to d_transfer): the candidate rows of its chunks, which
// stay in the res / gres arrays of bounds_layout<T>(n) for the seeded bounds_launch (rows_ready), then the head walk over them. An empty
// piece reads nothing.
template <class T>
static cudaError_t prot_transfer_launch(const uint8_t* d_in, size_t n, int is_last, uint8_t* ws, uint32_t* d_transfer, cudaStream_t stream,
                                        uint64_t* launches) {
    const cudaError_t e = prot_transfer_attr<T, false>();
    if (e != cudaSuccess) return e;
    uint32_t* res = nullptr;
    uint4* gres = nullptr;
    if (n) {
        BoundsLayout B; bounds_layout<T>(n, 0, &B);
        res = reinterpret_cast<uint32_t*>(ws + B.res);
        gres = reinterpret_cast<uint4*>(ws + B.gres);
        rows_launch<T>(d_in, n, n, ws, B, stream, launches);
    }
    dec_prot_transfer<T, false><<<1, PT_THREADS, prot_transfer_smem<T>(), stream>>>(d_in, n, n, is_last, res, gres, d_transfer);
    ++*launches;
    return cudaGetLastError();
}

// Enqueues the protected range map of d_in[0 .. n_range + n_halo) into d_map (PT_MAP_HDR + T::NCAND x PT_NCAND u32): the candidate rows
// of the range's chunks, as range_map_launch computes them, then one head walk per entry offset. The scratch is the res / gres arrays of
// bounds_layout<T>(n_range + n_halo).
template <class T>
static cudaError_t prot_locate_launch(const uint8_t* d_in, size_t n_range, size_t n_halo, uint8_t* ws, uint32_t* d_map, cudaStream_t stream,
                                      uint64_t* launches) {
    const cudaError_t e = prot_transfer_attr<T, true>();
    if (e != cudaSuccess) return e;
    BoundsLayout B; bounds_layout<T>(n_range + n_halo, 0, &B);
    rows_launch<T>(d_in, n_range, n_range + n_halo, ws, B, stream, launches);
    dec_prot_transfer<T, true><<<T::NCAND, PT_THREADS, prot_transfer_smem<T>(), stream>>>(d_in, n_range + n_halo, n_range, 0,
                                                                                          reinterpret_cast<uint32_t*>(ws + B.res),
                                                                                          reinterpret_cast<uint4*>(ws + B.gres), d_map);
    ++*launches;
    return cudaGetLastError();
}

}  // namespace bounds
}  // namespace dns
