// cl_decode.cu — run-parallel Cheetah decode for sm_90a.
//
// Replaces /root/reference/src/algorithms/cheetah/cheetah.rs:67-103,152-185 (decode_plain / decode_map_a / decode_map_b /
// decode_predicted, decode_unit / decode_partial_unit) driven by /root/reference/src/codec/codec.rs:82-126, bit-exactly.
// The scheme (every stage with the table logic of cl_core.cuh) is checked on the CPU by tests/cl_model.cpp + tests/test_cl_model_cpu.py.
//
//  0. Boundaries        decode_bounds.cuh with 2-bit flags (an encoded block is 8 + 4*plain + 2*map bytes, a copy-mode block 128 raw bytes).
//  1. Unpack            one warp per block: flag planes, the 16-bit hash of every NOT-predicted quad (explicit for MAP_A / MAP_B,
//                       hash of the literal for PLAIN), literals and copy-mode blocks straight to the output.
//  2. Chunk-map values  (cheetah.rs:72-73,80,89-93) A decoder never compares values, so the MRU-2 state of a bucket can be run
//                       SYMBOLICALLY: one warp per run executes PLAIN = push literal / MAP_A = read slot 0 / MAP_B = read slot 1 + swap
//                       on lists whose slots are literals or "slot j of the list carried into the run"; a fold over the runs (one
//                       thread per bucket) makes every run's carried-in list concrete; reads that hit a carried-in slot are patched.
//  3. Predicted values  (cheetah.rs:98-103) pred[ctx] is written by every not-predicted quad at ctx = hash of the previous quad and
//                       read by predicted quads. The hash of a predicted quad comes out of the table, so the context of the quad
//                       after it is not known up front: ROUNDS. In a round every run walks its blocks in order from the context
//                       and the table snapshot the previous round's fold left for it (round 0: snapshot unknown -> a read of an
//                       entry the run has not written yet is UNKNOWN, and so is the context of the next quad, whose write is
//                       skipped), then the fold (one thread per context) recomputes the snapshots and a sweep the run-entry
//                       contexts. When nothing changed and nothing was unknown the round's values are the reference's (induction
//                       over the runs). Text settles in 5-8 rounds for any run count (tests/test_cl_model_cpu.py).
//  4. Tail              (codec.rs:102-123) the last < 136 stream bytes in order by one thread from the folded tables (scalar_codec.cu).
//  5. Sharded decode    one piece of a longer stream is more runs of the same scheme (DESIGN.md section 5): the blocks a non-final piece
//                       leaves to the tail are appended to its block list (cd_piece_end), its chunk-map lists compose into one transfer
//                       (cd_cmap_export) that the later pieces fold into their cd_cmap_fold, and every prediction round exchanges each
//                       piece's table transfer (cd_pred_export, into cd_pred_fold) and exit context (cd_round_words, into
//                       cd_shard_round_end); the rounds stop for all pieces at once when none of them walked a run.
//
// Lion runs stages 0-2 on its own geometry (64-byte blocks, two per row of 32 quads) and the tail, but not the rounds: its 5-deep
// move-to-front lists make them advance one run per round (a misplaced operation desynchronises a whole list; measured in
// tests/cl_model.cpp). Stage 3 is instead one walk in stream order, 32 quads per step (ld_walk, lion_walk.cuh), which never gives up.
#include <stdlib.h>
#include "common.cuh"
#include "encode_internal.cuh"
#include "decode_bounds.cuh"
#include "cl_core.cuh"
#include "lion_walk.cuh"

namespace dns {
namespace cheedec {

using bounds::DecStatus;
using bounds::BLK_COPY;
using bounds::ldu16;
using T = bounds::CheeT;
using namespace cld;

constexpr uint32_t CTX_PASS = 0xFFFFFFFEu;        // ctx_out of a run without encoded quads
constexpr int RP_WARPS = 4;                       // warps (runs) per CTA of the walk kernels
constexpr int MAX_ROUNDS = 40;

struct ClStatus {
    unsigned int changed, unknown, done, rounds;
    unsigned int final_ctx, gave_up, pad0, pad1;
};

__device__ __forceinline__ uint64_t run_step_begin(uint32_t r, uint32_t nruns, uint64_t nsteps) { return (uint64_t)r * nsteps / nruns; }

// ---- 1. unpack ------------------------------------------------------------------------------------------------------------------
// One warp per row of 32 quads (128 output bytes): one Cheetah block, or two Lion blocks (lanes 0-15 and 16-31), as the Lion encoder
// lays them out. flags[s] = {predicted, MAP_A, MAP_B, encoded} bit per lane (LSB-first signature, read_signature.rs:11-16); K = the
// 16-bit hash of a not-predicted quad, the depth (flag - 1, lion.rs:123-186) of a predicted one (0 for Cheetah).
template <class G> __device__ __forceinline__ uint64_t cd_steps(const DecStatus* st) { return (st->main_blocks * (G::BS / 4) + 31) / 32; }

template <class G>
__global__ void cd_unpack(const uint8_t* __restrict__ in, const uint64_t* __restrict__ blk_off, const DecStatus* __restrict__ st,
                          uint4* __restrict__ flags, uint16_t* __restrict__ K, uint32_t* __restrict__ out) {
    if (st->error) return;
    constexpr bool LION = G::BS == 64;
    constexpr uint32_t QPB = G::BS / 4, FB = LION ? 3 : 2;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t mine = QPB == 32 ? 0xFFFFFFFFu : (lane < 16 ? 0x0000FFFFu : 0xFFFF0000u);   // the lanes of my block
    const uint64_t nb = st->main_blocks, ns = cd_steps<G>(st);
    for (uint64_t s = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < ns; s += (uint64_t)gridDim.x * (blockDim.x >> 5)) {
        const uint64_t b = s * (32 / QPB) + lane / QPB;
        const uint32_t q = lane % QPB;
        const unsigned long long o = b < nb ? blk_off[b] : BLK_COPY;
        const bool enc = b < nb && !(o & BLK_COPY);
        const uint8_t* p = in + (o & ~BLK_COPY);
        if (b < nb && !enc)                                        // codec.rs:89-92: BS raw bytes
            out[s * 32 + lane] = ldu16(p + 4 * q) | (ldu16(p + 4 * q + 2) << 16);
        uint32_t flag = 0, kind = K_PRED;
        if (enc) {
            const uint64_t sig = LION ? ((uint64_t)(ldu16(p) | (ldu16(p + 2) << 16)) | ((uint64_t)ldu16(p + 4) << 32)) : bounds::ldsig(p);
            flag = (uint32_t)(sig >> (FB * q)) & ((1u << FB) - 1u);
            kind = LION ? lion_kind(flag) : cheetah_kind(flag);
        }
        const uint32_t act = __ballot_sync(0xFFFFFFFFu, enc);
        const uint32_t plain = __ballot_sync(0xFFFFFFFFu, enc && kind == K_PLAIN);
        const uint32_t ma = __ballot_sync(0xFFFFFFFFu, enc && kind == K_MAP_A), mb = __ballot_sync(0xFFFFFFFFu, enc && kind == K_MAP_B);
        const uint32_t lt = lanemask_lt() & mine;
        const uint8_t* d = p + G::SIG + 4 * __popc(plain & lt) + 2 * __popc((ma | mb) & lt);
        uint32_t k = 0;
        if (enc && kind == K_PLAIN) { const uint32_t v = ldu16(d) | (ldu16(d + 2) << 16); out[s * 32 + lane] = v; k = hash16(v); }   // cheetah.rs:68-70, lion.rs:86-87
        else if (enc && kind != K_PRED) k = ldu16(d);                                                                                 // cheetah.rs:78,88, lion.rs:100,112
        else if (LION && enc) k = lion_depth(flag);
        K[s * 32 + lane] = (uint16_t)k;
        if (lane == 0) flags[s] = make_uint4(act & ~(plain | ma | mb), ma, mb, act);
    }
}

// ---- 2. chunk-map values ------------------------------------------------------------------------------------------------------------
// entry per (run, bucket): {a, b, meta, 0}; meta = epoch << 20 | tags (cl_core.cuh). The tables are zeroed per call: epoch 1 = touched.
template <class G>
__global__ void __launch_bounds__(RP_WARPS * 32)
cd_cmap_walk(const DecStatus* __restrict__ st, uint32_t nruns, const uint4* __restrict__ flags, const uint16_t* __restrict__ K,
             uint4* __restrict__ entC_all, uint32_t* __restrict__ out, uint2* __restrict__ usym /* per block: reads of carried-in slot 0 / slot 1 */) {
    if (st->error) return;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t r = blockIdx.x * RP_WARPS + (threadIdx.x >> 5);
    if (r >= nruns) return;
    const uint64_t nsteps = cd_steps<G>(st);
    const uint64_t s0 = run_step_begin(r, nruns, nsteps), s1 = run_step_begin(r + 1, nruns, nsteps);
    uint4* __restrict__ entC = entC_all + (size_t)r * 65536;
    for (uint64_t s = s0; s < s1; ++s) {
        const uint4 fl = flags[s];
        const uint32_t member_mask = fl.w & ~fl.x;                 // encoded and not predicted
        if (member_mask == 0) { if (lane == 0) usym[s] = make_uint2(0, 0); continue; }
        const bool member = (member_mask >> lane) & 1u;
        const uint32_t kind = ((fl.y >> lane) & 1u) ? K_MAP_A : ((fl.z >> lane) & 1u) ? K_MAP_B : K_PLAIN;
        const uint32_t h = K[s * 32 + lane];
        uint32_t val = 0;
        uint4 e = make_uint4(0, 0, 0, 0);
        if (member) { e = __ldcg(&entC[h]); if (kind == K_PLAIN) val = out[s * 32 + lane]; }
        const uint32_t key = member ? h : 0x10000u + lane;
        const uint32_t grp = __match_any_sync(0xFFFFFFFFu, key);
        const uint32_t lower = grp & lanemask_lt();
        const uint32_t rank = __popc(lower);
        const int src = lower ? 31 - __clz(lower) : (int)lane;
        const uint32_t maxrank = __reduce_max_sync(0xFFFFFFFFu, member ? rank : 0u);
        List<2> L;
        if (meta_epoch(e.z) == 1u) { L.v[0] = e.x; L.v[1] = e.y; list_from_meta<2>(L, e.z); } else list_init<2>(L, nullptr);
        L.unk = 0;
        uint32_t sym = 0;                                          // 0: value known; j + 1: value = slot j of the carried-in list
        for (uint32_t rk = 0; rk <= maxrank; ++rk) {
            if (member && rank == rk) {
                if (kind == K_PLAIN) list_push<2>(L, val);                                   // cheetah.rs:72-73
                else {
                    const int sl = kind == K_MAP_A ? 0 : 1;
                    const uint32_t t = L.slot_tag(sl);
                    if (t == TAG_LIT) val = L.v[sl]; else sym = t;                               // cheetah.rs:80 / :90
                    if (sl == 1) list_mtf<2>(L, 1);                                              // cheetah.rs:92-93
                }
            }
            const uint32_t r0 = __shfl_sync(0xFFFFFFFFu, L.v[0], src), r1 = __shfl_sync(0xFFFFFFFFu, L.v[1], src), rt = __shfl_sync(0xFFFFFFFFu, L.tag, src);
            if (member && rank == rk + 1) { L.v[0] = r0; L.v[1] = r1; L.tag = rt; }
        }
        if (member && (grp & lanemask_gt()) == 0) entC[h] = make_uint4(L.v[0], L.v[1], list_meta<2>(L, 1u), 0u);
        if (member && kind != K_PLAIN && sym == 0) out[s * 32 + lane] = val;
        const uint32_t u0 = __ballot_sync(0xFFFFFFFFu, sym == 1), u1 = __ballot_sync(0xFFFFFFFFu, sym == 2);
        if (lane == 0) usym[s] = make_uint2(u0, u1);
        __syncwarp();
    }
}

// one thread per bucket: the list carried into every run, and the chunk map after the main loop (for the tail).
// carry (sharded decode, nullptr otherwise): the chunk map in front of this piece, concrete planes {tags 0, a, b} (cd_cmap_export).
__global__ void cd_cmap_fold(const DecStatus* __restrict__ st, uint32_t nruns, const uint4* __restrict__ entC_all, uint2* __restrict__ cin,
                             uint32_t* __restrict__ chunk_a, uint32_t* __restrict__ chunk_b, const uint32_t* __restrict__ carry) {
    if (st->error) return;
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= 65536) return;
    uint32_t c[2] = {0u, 0u};                                      // chunk map starts as (0, 0) (cheetah.rs:52)
    if (carry) { c[0] = carry[65536 + h]; c[1] = carry[2 * 65536 + h]; }
    for (uint32_t r0 = 0; r0 < nruns; r0 += 8) {
        uint4 e[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) e[k] = (r0 + k < nruns) ? entC_all[(size_t)(r0 + k) * 65536 + h] : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            if (r0 + k >= nruns) break;
            cin[(size_t)(r0 + k) * 65536 + h] = make_uint2(c[0], c[1]);
            if (meta_epoch(e[k].z) == 1u) { List<2> L; L.v[0] = e[k].x; L.v[1] = e[k].y; list_from_meta<2>(L, e[k].z); list_carry<2>(c, L); }
        }
    }
    chunk_a[h] = c[0]; chunk_b[h] = c[1];
}

__device__ __forceinline__ uint32_t run_of_step(uint64_t s, uint32_t nruns, uint64_t nsteps) {
    uint32_t r = (uint32_t)((s * nruns) / nsteps);
    if (r >= nruns) r = nruns - 1;
    while (r + 1 < nruns && run_step_begin(r + 1, nruns, nsteps) <= s) ++r;
    while (r > 0 && run_step_begin(r, nruns, nsteps) > s) --r;
    return r;
}

// reads that hit a carried-in slot
template <class G>
__global__ void cd_cmap_resolve(const DecStatus* __restrict__ st, uint32_t nruns, const uint2* __restrict__ usym, const uint16_t* __restrict__ K,
                                const uint2* __restrict__ cin, uint32_t* __restrict__ out) {
    if (st->error) return;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t nsteps = cd_steps<G>(st);
    for (uint64_t s = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < nsteps; s += (uint64_t)gridDim.x * (blockDim.x >> 5)) {
        const uint2 u = usym[s];
        if ((u.x | u.y) == 0) continue;
        const uint32_t r = run_of_step(s, nruns, nsteps);
        if (((u.x | u.y) >> lane) & 1u) {
            const uint2 c = cin[(size_t)r * 65536 + K[s * 32 + lane]];
            out[s * 32 + lane] = ((u.x >> lane) & 1u) ? c.x : c.y;
        }
    }
}

// ---- 3. predicted values --------------------------------------------------------------------------------------------------------------
// context of the first encoded quad of every run when the stream says it: the nearest earlier encoded block ends with a quad that is
// not predicted (its hash is in K); otherwise unknown until a round has produced it. last_hash starts as 0 (cheetah.rs:54).
__global__ void cd_ctx_init(const DecStatus* __restrict__ st, uint32_t nruns, const uint4* __restrict__ flags, const uint16_t* __restrict__ K,
                            uint32_t* __restrict__ ctx_in, uint32_t* __restrict__ dirty_cur, uint32_t* __restrict__ dirty_next, uint32_t* __restrict__ run_epoch,
                            ClStatus* __restrict__ cs) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r == 0) { cs->changed = 0; cs->unknown = 0; cs->done = st->error ? 1u : 0u; cs->rounds = 0; cs->final_ctx = 0; cs->gave_up = 0; cs->pad0 = 0; }
    if (r >= nruns || st->error) return;
    dirty_cur[r] = 1; dirty_next[r] = 0; run_epoch[r] = 0;      // round 0 walks every run
    uint64_t s = run_step_begin(r, nruns, st->main_blocks);
    uint32_t c = 0;
    while (s > 0) {
        --s;
        const uint4 fl = flags[s];
        if (fl.w == 0) continue;                                   // copy-mode block: touches nothing (codec.rs:89-92)
        c = (fl.x >> 31) ? H_UNKNOWN : (uint32_t)K[s * 32 + 31];
        break;
    }
    ctx_in[r] = c;
}

// entry per (run, context): {value, epoch << 20}. Only not-predicted quads write (a predicted quad would store back what it read,
// cheetah.rs:98-103), so an entry of the current epoch always holds a literal.
__global__ void __launch_bounds__(RP_WARPS * 32)
cd_pred_walk(const DecStatus* __restrict__ st, ClStatus* __restrict__ cs, uint32_t nruns, uint32_t round, const uint4* __restrict__ flags,
             const uint16_t* __restrict__ K, uint2* __restrict__ entP_all, const uint32_t* __restrict__ snap_all, const uint32_t* __restrict__ ctx_in,
             uint32_t* __restrict__ ctx_out, const uint32_t* __restrict__ dirty_cur, uint32_t* __restrict__ dirty_next, uint32_t* __restrict__ run_epoch,
             uint32_t* __restrict__ rbits_all, uint32_t* __restrict__ out, uint32_t run0_snap) {
    if (cs->done) return;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t r = blockIdx.x * RP_WARPS + (threadIdx.x >> 5);
    if (r >= nruns) return;
    // A run is walked again only if something it depends on changed: its entry context, or a snapshot entry it read (cd_pred_fold
    // compares against the run's read set), or it met an unknown last time. Otherwise its values, its table entries (validated by
    // run_epoch) and its exit context stand.
    if (!dirty_cur[r]) return;
    uint32_t* __restrict__ rbits = rbits_all + (size_t)r * 2048;
    for (uint32_t i = lane; i < 2048; i += 32) rbits[i] = 0;
    __syncwarp();
    const uint32_t epoch = round + 1;
    const bool has_snap = round > 0 || (r == 0 && run0_snap);     // run0_snap: run 0 starts at the stream start (its snapshot is the zero table)
    const uint64_t nsteps = st->main_blocks;
    const uint64_t s0 = run_step_begin(r, nruns, nsteps), s1 = run_step_begin(r + 1, nruns, nsteps);
    uint2* __restrict__ entP = entP_all + (size_t)r * 65536;
    const uint32_t* __restrict__ snap = snap_all + (size_t)r * 65536;
    uint32_t carry = ctx_in[r];
    bool any_active = false, unknown_seen = false;
    // software pipeline: the streaming loads of the next step are issued before this step's table work
    uint4 fl_n = make_uint4(0, 0, 0, 0); uint32_t k_n = 0, v_n = 0;
    if (s0 < s1) { fl_n = flags[s0]; k_n = K[s0 * 32 + lane]; v_n = out[s0 * 32 + lane]; }
    for (uint64_t s = s0; s < s1; ++s) {
        const uint4 fl = fl_n; const uint32_t kh = k_n; uint32_t v = v_n;
        if (s + 1 < s1) { fl_n = flags[s + 1]; k_n = K[(s + 1) * 32 + lane]; v_n = out[(s + 1) * 32 + lane]; }
        if (fl.w == 0) continue;                                   // copy-mode block
        any_active = true;
        const uint32_t P = fl.x;
        const bool pred = (P >> lane) & 1u;
        // my context: the hash of the previous quad. Known at once unless that quad is predicted.
        const uint32_t kprev = __shfl_up_sync(0xFFFFFFFFu, kh, 1);
        uint32_t ctx = lane == 0 ? carry : (((P >> (lane - 1)) & 1u) ? H_UNKNOWN : kprev);
        bool ctx_ready = lane == 0 || !((P >> (lane - 1)) & 1u);
        // predicted lanes whose context is known up front fetch their entry now (all in flight together)
        uint2 e = make_uint2(0, 0); uint32_t sv = 0;
        const bool pre = pred && ctx_ready && ctx != H_UNKNOWN;
        if (pre) { e = __ldcg(&entP[ctx]); if (has_snap) sv = __ldcg(&snap[ctx]); }
        uint32_t h = pred ? H_UNKNOWN : kh;                        // my own hash
        uint32_t todo = P;
        while (todo) {
            const int p = __ffs(todo) - 1;
            todo &= todo - 1;
            const uint32_t c = __shfl_sync(0xFFFFFFFFu, ctx, p);    // lane p's context is final by now
            uint32_t val = 0; bool unk = false;
            if (c == H_UNKNOWN) unk = true;
            else {
                // the latest earlier writer of this step with the same context (all earlier contexts are final)
                const uint32_t w = __ballot_sync(0xFFFFFFFFu, !pred && (int)lane < p && ctx == c);
                if (w) val = __shfl_sync(0xFFFFFFFFu, v, 31 - __clz(w));
                else {
                    uint2 ee = e; uint32_t ss = sv;
                    const bool had = __shfl_sync(0xFFFFFFFFu, (int)pre, p) != 0;
                    if (!had && (int)lane == p) { ee = __ldcg(&entP[c]); if (has_snap) ss = __ldcg(&snap[c]); }
                    uint32_t mv = ee.x, me = meta_epoch(ee.y), ms = ss;
                    mv = __shfl_sync(0xFFFFFFFFu, mv, p); me = __shfl_sync(0xFFFFFFFFu, me, p); ms = __shfl_sync(0xFFFFFFFFu, ms, p);
                    if (me == epoch) val = mv;                      // written earlier in this run
                    else if (has_snap) {                            // carried in (as of the previous round's fold): remember that I depend on it
                        val = ms;
                        if ((int)lane == p) atomicOr(&rbits[c >> 5], 1u << (c & 31));
                    } else unk = true;                              // round 0: nothing is known about what earlier runs left here
                }
            }
            const uint32_t hp = unk ? H_UNKNOWN : hash16(val);      // cheetah.rs:101
            unknown_seen |= unk;
            // a stretch of predicted quads right behind p reads the same entry as long as the hash maps the context onto itself
            uint32_t span = 1;
            if (!unk && hp == c) {
                const uint32_t rest = p == 31 ? 0u : ~(P >> (p + 1));
                const uint32_t follow = rest ? (uint32_t)(__ffs(rest) - 1) : (uint32_t)(31 - p);
                span += follow;
            }
            if ((int)lane >= p && (uint32_t)lane < (uint32_t)p + span) { v = val; h = hp; if ((int)lane > p) { ctx = c; ctx_ready = true; } }
            if (span > 1) { const uint32_t clr = ((span >= 32 ? 0xFFFFFFFFu : ((1u << span) - 1u)) << p); todo &= ~clr; }
            if ((uint32_t)lane == (uint32_t)p + span) { ctx = hp; ctx_ready = true; }
        }
        carry = __shfl_sync(0xFFFFFFFFu, h, 31);                    // cheetah.rs:102 (last_hash)
        // writers: pred[ctx] <- value (cheetah.rs:74,82,94); the last writer of a context inside the step leaves its value
        const bool writer = !pred && ctx != H_UNKNOWN;
        const uint32_t grp = __match_any_sync(0xFFFFFFFFu, writer ? ctx : 0x10000u + lane);
        if (writer && (grp & lanemask_gt()) == 0) entP[ctx] = make_uint2(v, epoch << META_EPOCH_SHIFT);
        if (pred && h != H_UNKNOWN) out[s * 32 + lane] = v;
        __syncwarp();
    }
    if (lane == 0) {
        ctx_out[r] = any_active ? carry : CTX_PASS;
        run_epoch[r] = epoch;
        if (unknown_seen) dirty_next[r] = 1;
    }
}

// one thread per context: snapshot of the table in front of every run (in place), and the table after the main loop (for the tail).
// A run whose snapshot changed at a context it read has to be walked again.
// carry (sharded decode, nullptr otherwise): the table in front of this piece as of this round, planes {touched, value} (cl_rank_fold P).
__global__ void cd_pred_fold(const DecStatus* __restrict__ st, ClStatus* __restrict__ cs, uint32_t nruns, uint32_t round, const uint2* __restrict__ entP_all,
                             uint32_t* __restrict__ snap, const uint32_t* __restrict__ run_epoch, const uint32_t* __restrict__ rbits_all,
                             uint32_t* __restrict__ dirty_next, uint32_t* __restrict__ pred_final, const uint32_t* __restrict__ carry) {
    if (cs->done) return;
    const uint32_t ctx = blockIdx.x * blockDim.x + threadIdx.x;
    if (ctx >= 65536) return;
    uint32_t c = carry ? carry[65536 + ctx] : 0u;                  // prediction table starts as 0 everywhere (cheetah.rs:53)
    for (uint32_t r0 = 0; r0 < nruns; r0 += 8) {
        uint2 e[8]; uint32_t so[8], ep[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const bool ok = r0 + k < nruns;
            e[k] = ok ? entP_all[(size_t)(r0 + k) * 65536 + ctx] : make_uint2(0, 0);
            so[k] = ok ? snap[(size_t)(r0 + k) * 65536 + ctx] : 0u;
            ep[k] = ok ? run_epoch[r0 + k] : 0u;
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            if (r0 + k >= nruns) break;
            if (so[k] != c) {
                snap[(size_t)(r0 + k) * 65536 + ctx] = c;
                if (round > 0 && ((rbits_all[(size_t)(r0 + k) * 2048 + (ctx >> 5)] >> (ctx & 31)) & 1u)) dirty_next[r0 + k] = 1;
            }
            if (meta_epoch(e[k].y) == ep[k] && ep[k] != 0) c = e[k].x;
        }
    }
    pred_final[ctx] = c;
    (void)st;
}

// context sweep + verdict of the round (one thread)
__global__ void cd_round_end(ClStatus* __restrict__ cs, uint32_t nruns, uint32_t round, uint32_t* __restrict__ ctx_in, const uint32_t* __restrict__ ctx_out,
                             uint32_t* __restrict__ dirty_cur, uint32_t* __restrict__ dirty_next) {
    if (threadIdx.x || blockIdx.x || cs->done) return;
    uint32_t c = 0, ndirty = 0;
    for (uint32_t r = 0; r < nruns; ++r) {
        uint32_t d = dirty_next[r];
        if (round == 0 && r > 0) d = 1;                            // runs > 0 had no snapshot in round 0
        if (ctx_in[r] != c) { d = 1; ctx_in[r] = c; }
        dirty_cur[r] = d; dirty_next[r] = 0;
        ndirty += d;
        const uint32_t o = ctx_out[r];
        if (o != CTX_PASS) c = o;
    }
    cs->final_ctx = c;
    cs->rounds = round + 1;
    cs->pad0 += ndirty;                                            // diagnostic: run walks queued after round 0
    if (ndirty == 0) cs->done = 1;
}

// verdict for the caller: *d_fallback != 0 -> the in-order kernel (queued behind, gated on it) has to produce the result
__global__ void cd_finish(const DecStatus* __restrict__ st, ClStatus* __restrict__ cs, uint32_t* __restrict__ d_fallback, uint64_t* __restrict__ d_out_size) {
    const bool ok = cs->done && !st->error;
    if (!ok && !st->error) cs->gave_up = 1;
    *d_fallback = ok ? 0u : 1u;
    if (!ok && d_out_size) *d_out_size = 0;
}

// ---- 3'. Lion: the prediction walk ---------------------------------------------------------------------------------------------------
// lion.rs:50-57,125-186 over every encoded quad in stream order (lion_walk.cuh): one warp, one row of 32 quads per step, the next row's
// stream data loaded during this row and later rows pulled into L2. The walk never gives up. The table (5 x u32 per context, zeroed per
// call, lion.rs:70) is the tail's, in the workspace, where the tail continues on it. A CTA whose producer warps fill a shared-memory
// ring ahead of the walker, and that ring with the table in an 8-CTA cluster's distributed shared memory, measured slower on text and
// synth_mixed (DESIGN.md section 8).
// status: a ClStatus prefix (final_ctx for the tail, done for cd_finish) followed by the walk's counts (density_b200_lion_decode_stats).
// ctx_in (a piece of a sharded stream after the first, nullptr otherwise): the context of the piece's first quad, last_hash behind the
// pieces before it; ctx_out (a piece of a sharded stream, nullptr otherwise) receives the context behind the piece. They may alias.
struct LionStatus { ClStatus c; unsigned long long quads, pred, dep, rows; };
constexpr uint32_t LW_PREFETCH = 16;                       // rows ahead whose stream data is pulled into L2 while the walk works

__global__ void __launch_bounds__(32) ld_walk(const DecStatus* __restrict__ st, const uint4* __restrict__ flags, const uint16_t* __restrict__ K,
                                              uint32_t* __restrict__ out, uint32_t* __restrict__ T, LionStatus* __restrict__ ls,
                                              const uint32_t* ctx_in, uint32_t* ctx_out) {
#if defined(__CUDA_ARCH__)                                   // lwalk::Warp / LV are the device lanes only in the device pass
    if (st->error) return;
    using namespace lwalk;
    Warp w{(int)(threadIdx.x & 31)};
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t ns = cd_steps<bounds::LionT>(st);
    // quads of the main loop: with an odd block count the last row has one block, and lanes 16-31 of it would read past the main loop's
    // output (past cap when the tail is shorter than a block); they are inactive, so they load 0. K holds whole rows (cd_unpack writes
    // all 32 lanes), so its guard only keeps the two loads alike.
    const uint64_t nq = st->main_blocks * 16;
    const FlatTable tab{T};
    WalkCounts cnt{0, 0, 0, 0};
    uint32_t carry = ctx_in ? *ctx_in : 0u;                // lion.rs:67
    uint4 fl_n = make_uint4(0, 0, 0, 0); uint32_t k_n = 0, v_n = 0;
    if (ns) { fl_n = flags[0]; if (lane < nq) { k_n = K[lane]; v_n = out[lane]; } }
    for (uint64_t s = 0; s < ns; ++s) {
        const uint4 fl = fl_n;
        LV<uint32_t> kh{k_n}, v{v_n};
        if (s + 1 < ns) {
            const uint64_t i = (s + 1) * 32 + lane;
            fl_n = flags[s + 1]; k_n = i < nq ? K[i] : 0u; v_n = i < nq ? out[i] : 0u;
        }
        if (s + LW_PREFETCH < ns) {
            const uint64_t f = s + LW_PREFETCH;
            if (lane == 0) asm volatile("prefetch.global.L2 [%0];" :: "l"(flags + f));
            if (lane == 1) asm volatile("prefetch.global.L2 [%0];" :: "l"(K + f * 32));
            if (lane == 2) asm volatile("prefetch.global.L2 [%0];" :: "l"(out + f * 32));
        }
        walk_row(w, fl.x, fl.w, kh, v, tab, carry, cnt);
        if ((fl.x >> lane) & 1u) out[s * 32 + lane] = v.x;
    }
    if (lane == 0) {
        ls->c.final_ctx = carry; ls->c.done = 1; ls->c.rounds = 1;
        ls->quads = cnt.quads; ls->pred = cnt.pred; ls->dep = cnt.dep; ls->rows = cnt.rows;
        if (ctx_out) *ctx_out = carry;
    }
#endif
}

// ---- 5. sharded decode: one piece of a longer stream --------------------------------------------------------------------------------
// A piece is more runs of the same scheme: the chunk-map lists and the prediction table come in from the pieces before it as transfers,
// the context of its first quad from their exit contexts (DESIGN.md section 5).
constexpr uint32_t PL = 65536;
constexpr uint32_t CM_IDENTITY = 1u | (2u << 3);          // chunk-map transfer tags: slot j = carried-in slot j

struct PieceStatus { unsigned int refuse, first_inc, last_inc, tail_blocks, pad[4]; };

// The end of the piece, right after the boundary walk. A non-final piece is followed by more stream bytes, so the reference decodes all of
// its blocks in the main loop (codec.rs:88-100); the blocks the boundary walk left to the tail (those starting in the last G::MAXBLK bytes)
// are appended to the block list. Their control flow does not depend on the tables. The final piece keeps its in-order tail; its control
// flow is walked here for the seam words. The automaton starts from the state behind the main loop (bounds::main_end_state: the piece's
// seed carried over its main blocks). Refused (pst->refuse): a non-final piece whose blocks do not end exactly at its last byte or that
// reads a malformed block; and, unless `prot`, a piece > 0 that is not quiet (copy mode, two consecutive incompressible blocks) or a
// non-final piece that meets copy mode at its end, ends with a copy penalty pending or inside a copy run. prot: a piece of the protected
// path (density_b200_cheetah_decode_shard_prot_*, density_b200_lion_decode_shard_prot_*), whose seed carries the automaton across the
// cuts, so the blocks at its end may be copy-mode blocks (appended with BLK_COPY) and it may end in any automaton state. G: the block
// geometry (bounds::CheeT: 128-byte blocks, 8-byte signatures of 2-bit flags; bounds::LionT: 64-byte blocks, 6-byte signatures of 3-bit
// flags).
template <class G>
__global__ void cd_piece_end(const uint8_t* __restrict__ in, uint64_t n, uint64_t cap, int first, int last, int prot, DecStatus* __restrict__ st,
                             uint64_t* __restrict__ blk_off, uint64_t maxblocks, PieceStatus* __restrict__ pst) {
    if (threadIdx.x || blockIdx.x) return;
    constexpr bool LION = G::BS == 64;
    constexpr uint32_t FB = LION ? 3 : 2;                          // flag bits per quad
    auto sig_at = [&](uint64_t o) { uint64_t s = 0; for (uint32_t i = 0; i < G::SIG; ++i) s |= (uint64_t)in[o + i] << (8 * i); return s; };
    if (st->error) { pst->refuse = 1; pst->first_inc = 0; pst->last_inc = 0; pst->tail_blocks = 0; return; }
    uint32_t refuse = (!prot && !first && st->seq) ? 1u : 0u;    // dec_seq_walk ran: two consecutive incompressible blocks in the main loop
    Protection ps = bounds::main_end_state(st);
    uint64_t idx = st->tail_off, b = st->main_blocks;
    uint32_t tail_first = 0, tail_blocks = 0;
    if (!last) {
        bool bad = false, ends_copy = b > 0 && (blk_off[b - 1] & BLK_COPY);
        while (idx < n) {
            if (ps.revert_to_copy()) {                             // codec.rs:89-92
                if (!prot || n - idx < G::BS) { bad = true; break; }   // quiet path: copy mode at the end of a non-final piece
                if (b < maxblocks) blk_off[b] = idx | BLK_COPY; else st->error = 2;
                ++b; ++tail_blocks; idx += G::BS; ends_copy = true;
                ps.decay();
                continue;
            }
            if (n - idx < G::SIG) { bad = true; break; }
            const uint32_t consumed = G::consumed(sig_at(idx));
            if (consumed > n - idx) { bad = true; break; }         // the block runs past the piece
            if (b < maxblocks) blk_off[b] = idx; else st->error = 2;
            ++b; ++tail_blocks; idx += consumed; ends_copy = false;
            ps.update(consumed >= G::BS);                          // codec.rs:94-98
        }
        if (bad || (!prot && (ends_copy || ps.copy_penalty))) refuse = 1;
        if (!bad) {
            st->main_blocks = b; st->tail_off = idx; st->last_main_inc = ps.previous_incompressible;
            if (prot) st->seq = 1;                                 // main_end_state reads the state below from now on
            if (st->seq) { st->ps_penalty = ps.copy_penalty; st->ps_start = ps.copy_penalty_start; st->ps_prev = ps.previous_incompressible; }
        }
        if (b * G::BS > cap) st->error = 2;
    } else {
        // the tail loop's control flow (codec.rs:102-123, scalar_codec.cu decode_loops): copy mode or a new incompressible pair there
        // is refused in a piece > 0; malformed input is left to the tail kernel, which reports it
        uint32_t copied = 0, pair = 0;
        while (n - idx > 0) {
            ++tail_blocks;
            if (ps.revert_to_copy()) {
                copied = 1;
                if (n - idx > G::BS) { idx += G::BS; ps.decay(); continue; }
                break;
            }
            const uint64_t mark = idx;
            if (n - idx < G::SIG) break;
            uint64_t sig = sig_at(idx);
            idx += G::SIG;
            bool end = false;
            for (uint32_t u = 0; u < G::BS / 4 && !end; ++u) {
                const uint32_t fl = (uint32_t)(sig & ((1u << FB) - 1u)); sig >>= FB;
                const uint32_t kind = LION ? lion_kind(fl) : cheetah_kind(fl);
                const uint64_t rem = n - idx;
                if (kind == K_PLAIN && rem < 4) end = true;        // decode_partial_unit: the stream ends inside this quad
                else if (kind == K_PLAIN) idx += 4;
                else if (kind != K_PRED) { if (rem < 2) end = true; else idx += 2; }
            }
            if (end) break;
            const uint32_t inc = idx - mark >= G::BS ? 1u : 0u;
            if (tail_blocks == 1) tail_first = inc;
            pair |= inc & ps.previous_incompressible;
            ps.update(inc);
        }
        if (!prot && !first && (copied || pair)) refuse = 1;
    }
    const uint64_t b0 = blk_off[0];
    pst->first_inc = st->main_blocks ? ((!(b0 & BLK_COPY) && G::consumed(sig_at(b0)) >= G::BS) ? 1u : 0u) : tail_first;
    pst->last_inc = ps.previous_incompressible;
    pst->refuse = refuse;
    pst->tail_blocks = tail_blocks;
}

// chunk-map transfer of a piece, planes {tags, a, b} per bucket: slot s of the list the piece leaves is the literal v[s] (tag 0) or
// slot t - 1 of the list carried into the piece (tag t, 3 bits per slot as in List<2>). "x, then y" applies y's tags to x's slots.
__device__ __forceinline__ void cm_compose(uint32_t (&v)[2], uint32_t& tag, const uint32_t (&yv)[2], uint32_t ytag) {
    uint32_t nv[2], nt = 0;
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        const uint32_t t = (ytag >> (3 * s)) & 7u;
        if (t == TAG_LIT || t > 2) nv[s] = yv[s];
        else { nv[s] = v[t - 1]; nt |= ((tag >> (3 * (t - 1))) & 7u) << (3 * s); }
    }
    v[0] = nv[0]; v[1] = nv[1]; tag = nt;
}
// the composition over the piece's runs (nruns 0 or st == nullptr: the identity, an empty piece)
__global__ void cd_cmap_export(const DecStatus* __restrict__ st, uint32_t nruns, const uint4* __restrict__ entC_all, uint32_t* __restrict__ out) {
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= PL) return;
    uint32_t v[2] = {0u, 0u}, tag = CM_IDENTITY;
    if (st && !st->error) {
        for (uint32_t r = 0; r < nruns; ++r) {
            const uint4 e = entC_all[(size_t)r * PL + h];
            if (meta_epoch(e.z) != 1u) continue;
            const uint32_t yv[2] = {e.x, e.y};
            cm_compose(v, tag, yv, e.z & 0x3Fu);
        }
    }
    out[h] = tag; out[PL + h] = v[0]; out[2 * PL + h] = v[1];
}
// the stream-start chunk map (0, 0) in every bucket (cheetah.rs:52); acc <- acc, then next; the carry-in of piece `rank`
__global__ void cd_cmap_init_k(uint32_t* __restrict__ t) {
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h < PL) { t[h] = 0; t[PL + h] = 0; t[2 * PL + h] = 0; }
}
__global__ void cd_cmap_fold_k(uint32_t* __restrict__ acc, const uint32_t* __restrict__ next) {
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= PL) return;
    uint32_t v[2] = {acc[PL + h], acc[2 * PL + h]}, tag = acc[h];
    const uint32_t yv[2] = {next[PL + h], next[2 * PL + h]};
    cm_compose(v, tag, yv, next[h]);
    acc[h] = tag; acc[PL + h] = v[0]; acc[2 * PL + h] = v[1];
}
__global__ void cd_cmap_rank_fold_k(const uint32_t* __restrict__ tables, uint32_t rank, uint32_t* __restrict__ carry) {
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= PL) return;
    uint32_t v[2] = {0u, 0u}, tag = 0;
    for (uint32_t r = 0; r < rank; ++r) {
        const uint32_t* t = tables + (size_t)r * 3 * PL;
        const uint32_t yv[2] = {t[PL + h], t[2 * PL + h]};
        cm_compose(v, tag, yv, t[h]);
    }
    carry[h] = tag; carry[PL + h] = v[0]; carry[2 * PL + h] = v[1];
}

// prediction transfer of this round, planes {touched, last value} per context: the entries cd_pred_fold counts (the epoch of their run's
// last walk), in run order. The format of the Cheetah encoder's P table, so cl_rank_fold / cl_table_fold compose it.
__global__ void cd_pred_export(const ClStatus* __restrict__ cs, uint32_t nruns, const uint2* __restrict__ entP_all, const uint32_t* __restrict__ run_epoch,
                               uint32_t* __restrict__ out) {
    if (cs->done) return;
    const uint32_t ctx = blockIdx.x * blockDim.x + threadIdx.x;
    if (ctx >= PL) return;
    uint32_t touched = 0, v = 0;
    for (uint32_t r = 0; r < nruns; ++r) {
        const uint32_t ep = run_epoch[r];
        const uint2 e = entP_all[(size_t)r * PL + ctx];
        if (ep != 0 && meta_epoch(e.y) == ep) { touched = 1; v = e.x; }
    }
    out[ctx] = touched; out[PL + ctx] = v;
}
// the piece's 4 round words after its walk: {has an exit context, exit context (the last run's with encoded quads; may be H_UNKNOWN),
// runs walked in this round, a run met an unknown}. A settled or failed piece walks nothing.
__global__ void cd_round_words(const DecStatus* __restrict__ st, const ClStatus* __restrict__ cs, uint32_t nruns, const uint32_t* __restrict__ ctx_out,
                               const uint32_t* __restrict__ dirty_cur, const uint32_t* __restrict__ dirty_next, uint32_t* __restrict__ words) {
    __shared__ int s_last;
    __shared__ uint32_t s_walked, s_unknown;
    if (threadIdx.x == 0) { s_last = -1; s_walked = 0; s_unknown = 0; }
    __syncthreads();
    const bool live = !st->error;
    const bool walking = live && !cs->done;
    int last = -1; uint32_t walked = 0, unknown = 0;
    for (uint32_t r = threadIdx.x; live && r < nruns; r += blockDim.x) {
        if (ctx_out[r] != CTX_PASS) last = (int)r;
        if (walking) { walked += dirty_cur[r]; unknown |= dirty_next[r]; }
    }
    if (last >= 0) atomicMax(&s_last, last);
    if (walked) atomicAdd(&s_walked, walked);
    if (unknown) atomicOr(&s_unknown, 1u);
    __syncthreads();
    if (threadIdx.x == 0) {
        words[0] = s_last >= 0 ? 1u : 0u; words[1] = s_last >= 0 ? ctx_out[s_last] : 0u;
        words[2] = s_walked; words[3] = s_unknown;
    }
}
// context sweep of a piece: run 0's entry context is the exit context of the nearest earlier piece that has one (0 if none,
// cheetah.rs:54). Round 0: only the run at the stream start had a snapshot. The rounds have settled when no piece walked a run in this
// round, which every piece reads off the same gathered words, so all pieces stop together.
__global__ void cd_shard_round_end(ClStatus* __restrict__ cs, uint32_t nruns, uint32_t round, uint32_t first, uint32_t rank, uint32_t world,
                                   const uint32_t* __restrict__ all_words, uint32_t* __restrict__ ctx_in, const uint32_t* __restrict__ ctx_out,
                                   uint32_t* __restrict__ dirty_cur, uint32_t* __restrict__ dirty_next) {
    if (threadIdx.x || blockIdx.x || cs->done) return;
    uint32_t c = 0, walked = 0, ndirty = 0;
    for (uint32_t q = 0; q < world; ++q) {
        const uint32_t* w = all_words + 4 * q;
        if (q < rank && w[0]) c = w[1];
        walked += w[2];
    }
    for (uint32_t r = 0; r < nruns; ++r) {
        uint32_t d = dirty_next[r];
        if (round == 0 && (r > 0 || !first)) d = 1;
        if (ctx_in[r] != c) { d = 1; ctx_in[r] = c; }
        dirty_cur[r] = d; dirty_next[r] = 0;
        ndirty += d;
        const uint32_t o = ctx_out[r];
        if (o != CTX_PASS) c = o;
    }
    cs->final_ctx = c;
    cs->rounds = round + 1;
    cs->pad0 += ndirty;
    if (walked == 0) cs->done = 1;
}
// the piece's 8 seam words in the layout of the Chameleon decoder's (after the tail): {first block incompressible, previous_incompressible
// at the end, refused, has blocks, decoded size lo, hi, 0, 0}. seed (the protected path, nullptr otherwise): the piece's incoming state
// (bounds::dec_prot_enter_k); words 0 and 1 are then 0, since incompressible blocks may meet at a cut when the transfers carry the
// automaton across it, and the piece is also refused when the transfers composed to no state. pst == nullptr: an empty piece of the
// protected path (no blocks, size 0), refused only by its seed. BS: the block size, of which a non-final piece decodes a whole number.
template <uint32_t BS>
__global__ void cd_seam_words(const PieceStatus* __restrict__ pst, const uint32_t* __restrict__ fallback, const Status* __restrict__ tail_status,
                              int is_last, const uint32_t* __restrict__ seed, uint64_t* __restrict__ d_out_size, uint32_t* __restrict__ words) {
    if (threadIdx.x || blockIdx.x) return;
    uint64_t sz = 0;
    uint32_t bad = seed ? seed[4] : 0u;
    if (pst) {
        sz = *d_out_size;
        if (pst->refuse || *fallback || tail_status->error) bad = 1;
        if (!is_last && (sz % BS)) bad = 1;
    } else *d_out_size = 0;
    words[0] = pst && !seed ? pst->first_inc : 0u; words[1] = pst && !seed ? pst->last_inc : 0u; words[2] = bad; words[3] = pst ? 1u : 0u;
    words[4] = (uint32_t)sz; words[5] = (uint32_t)(sz >> 32); words[6] = 0; words[7] = 0;
}

}  // namespace cheedec

using namespace cheedec;

struct CheeDecLayout { bounds::BoundsLayout B; size_t cs, flags, K, usym, ctx_in, ctx_out, dirty, run_epoch, rbits, cin, snap0, total; };

static uint32_t cd_pick_runs(size_t nbytes, int num_sms) {
    // a run should decode to >= 64 KiB (512 blocks); the stream is at most 8.5 bytes per block... use the stream size as a proxy
    uint64_t r = nbytes / (48u << 10);
    static const int per_sm = [] { const char* v = getenv("DENSITY_B200_DEC_RUNS_PER_SM"); const int k = v ? atoi(v) : 0; return (k >= 1 && k <= 32) ? k : 8; }();
    const uint64_t cap = (uint64_t)num_sms * per_sm;   // warps (runs) per SM: tuning knob, the result does not depend on it
    if (r > cap) r = cap;
    if (r < 1) r = 1;
    return (uint32_t)r;
}

// lion: the Lion geometry (two blocks per row) and no prediction-round arrays (the walk replaces the rounds)
static size_t cd_layout(size_t nbytes, size_t cap, uint32_t nruns, CheeDecLayout* L, bool lion = false) {
    size_t off = lion ? bounds::bounds_layout<bounds::LionT>(nbytes, cap, &L->B) : bounds::bounds_layout<bounds::CheeT>(nbytes, cap, &L->B);
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
    const uint64_t ms = lion ? (L->B.maxblocks + 1) / 2 : L->B.maxblocks;   // rows of 32 quads
    const size_t rr = lion ? 0 : nruns;                                       // runs with prediction-round arrays
    L->cs = take(lion ? sizeof(LionStatus) : sizeof(ClStatus));
    L->flags = take(ms * sizeof(uint4));
    L->K = take(ms * 32 * sizeof(uint16_t));
    L->usym = take(ms * sizeof(uint2));
    L->ctx_in = take(rr * 4 + 64);
    L->ctx_out = take(rr * 4 + 64);
    L->dirty = take(rr * 8 + 64);
    L->run_epoch = take(rr * 4 + 64);
    L->rbits = take(rr * 2048 * sizeof(uint32_t));
    L->cin = take((size_t)nruns * 65536 * sizeof(uint2));
    L->snap0 = take(rr * 65536 * sizeof(uint32_t));
    L->total = off;
    return off;
}

size_t chee_decode_workspace_bytes(size_t nbytes, size_t cap, int num_sms) { CheeDecLayout L; return cd_layout(nbytes, cap, cd_pick_runs(nbytes, num_sms), &L); }
// the per-run tables (zeroed at the start of every call): chunk map 16 B, prediction 8 B per run and key (Lion: the chunk map only)
size_t chee_decode_tables_bytes(size_t nbytes, int num_sms, bool lion) {
    return (size_t)cd_pick_runs(nbytes, num_sms) * 65536 * (sizeof(uint4) + (lion ? 0 : sizeof(uint2)));
}
size_t lion_decode_workspace_bytes(size_t nbytes, size_t cap, int num_sms) { CheeDecLayout L; return cd_layout(nbytes, cap, cd_pick_runs(nbytes, num_sms), &L, true); }

// The decoder's view of one call: the run geometry, the boundary layout and typed pointers into the workspace (cd_layout), the per-run
// tables and the tail's tables (the scalar_codec.cu workspace: Status (256 B) + chunk_a + chunk_b + pred), which receive the folded
// tables for the tail loop. A piece of a sharded stream keeps more behind the layout in its own workspace: the fallback word and the
// PieceStatus (256 B), then its tail tables, taken when `tail_ws` is null. `tables` may be null for a caller that only wants addresses
// inside the workspace.
struct CheeDecPtrs {
    uint32_t nruns, run_ctas; int wide; bounds::BoundsLayout B;
    DecStatus* st; ClStatus* cs; uint64_t* blk_off; uint4* flags; uint16_t* K; uint2* usym;
    uint32_t *ctx_in, *ctx_out, *dirty_cur, *dirty_next, *run_epoch, *rbits, *snap, *fallback, *chunk_a, *chunk_b, *pred_final;
    uint2* cin; uint8_t* tables; size_t tables_bytes; uint4* entC; uint2* entP; PieceStatus* pst; uint8_t* tail_ws;
    CheeDecPtrs(size_t n, size_t cap, int num_sms, uint8_t* ws, uint8_t* tables_, uint8_t* tail_ws_, bool lion = false) {
        nruns = cd_pick_runs(n, num_sms);
        run_ctas = (nruns + RP_WARPS - 1) / RP_WARPS;
        wide = num_sms * 8;
        CheeDecLayout L; cd_layout(n, cap, nruns, &L, lion);
        B = L.B;
        const size_t off = (L.total + 255) & ~(size_t)255;
        st = reinterpret_cast<DecStatus*>(ws + L.B.status);
        cs = reinterpret_cast<ClStatus*>(ws + L.cs);
        blk_off = reinterpret_cast<uint64_t*>(ws + L.B.blk_off);
        flags = reinterpret_cast<uint4*>(ws + L.flags);
        K = reinterpret_cast<uint16_t*>(ws + L.K);
        usym = reinterpret_cast<uint2*>(ws + L.usym);
        ctx_in = reinterpret_cast<uint32_t*>(ws + L.ctx_in);
        ctx_out = reinterpret_cast<uint32_t*>(ws + L.ctx_out);
        dirty_cur = reinterpret_cast<uint32_t*>(ws + L.dirty);
        dirty_next = dirty_cur + nruns;
        run_epoch = reinterpret_cast<uint32_t*>(ws + L.run_epoch);
        rbits = reinterpret_cast<uint32_t*>(ws + L.rbits);
        cin = reinterpret_cast<uint2*>(ws + L.cin);
        snap = reinterpret_cast<uint32_t*>(ws + L.snap0);
        fallback = reinterpret_cast<uint32_t*>(ws + off);
        pst = reinterpret_cast<PieceStatus*>(ws + off + 128);
        tail_ws = tail_ws_ ? tail_ws_ : ws + off + 256;
        chunk_a = reinterpret_cast<uint32_t*>(tail_ws + 256);
        chunk_b = chunk_a + PL;
        pred_final = chunk_a + 2 * PL;
        tables = tables_; tables_bytes = chee_decode_tables_bytes(n, num_sms, lion);
        entC = reinterpret_cast<uint4*>(tables);
        entP = tables && !lion ? reinterpret_cast<uint2*>(tables + (size_t)nruns * PL * sizeof(uint4)) : nullptr;
    }
};

// ---- the launch sequences that the one-shot decode and the phases of a piece share ------------------------------------------------------
// the per-run tables and run 0's snapshot (the zero table) start every call as zeros
static cudaError_t cd_clear_tables(const CheeDecPtrs& p, cudaStream_t stream) {
    cudaError_t e = cudaMemsetAsync(p.tables, 0, p.tables_bytes, stream);
    if (e == cudaSuccess && p.entP) e = cudaMemsetAsync(p.snap, 0, (size_t)p.nruns * PL * sizeof(uint32_t), stream);
    return e;
}
// unpack (literals and copy-mode blocks go straight to the output) and the symbolic chunk-map walk
template <class G = bounds::CheeT>
static void cd_launch_unpack_walk(const CheeDecPtrs& p, const uint8_t* d_in, uint32_t* out32, cudaStream_t stream, uint64_t* launches) {
    cd_unpack<G><<<p.wide, 256, 0, stream>>>(d_in, p.blk_off, p.st, p.flags, p.K, out32);
    cd_cmap_walk<G><<<p.run_ctas, RP_WARPS * 32, 0, stream>>>(p.st, p.nruns, p.flags, p.K, p.entC, out32, p.usym);
    *launches += 2;
}
// the chunk map carried in (d_cmap_carry: nullptr = the stream start), the reads of carried-in slots, the context init (Cheetah)
template <class G = bounds::CheeT>
static void cd_launch_cmap_resolve(const CheeDecPtrs& p, uint32_t* out32, const uint32_t* d_cmap_carry, cudaStream_t stream, uint64_t* launches) {
    cd_cmap_fold<<<PL / 128, 128, 0, stream>>>(p.st, p.nruns, p.entC, p.cin, p.chunk_a, p.chunk_b, d_cmap_carry);
    cd_cmap_resolve<G><<<p.wide, 256, 0, stream>>>(p.st, p.nruns, p.usym, p.K, p.cin, out32);
    *launches += 2;
    if (G::BS == 128) {
        cd_ctx_init<<<(p.nruns + 127) / 128, 128, 0, stream>>>(p.st, p.nruns, p.flags, p.K, p.ctx_in, p.dirty_cur, p.dirty_next, p.run_epoch, p.cs);
        ++*launches;
    }
}
// a prediction round: walk the dirty runs (run0_snap: run 0 starts from the stream start's zero table) ...
static void cd_launch_pred_walk(const CheeDecPtrs& p, uint32_t round, uint32_t* out32, uint32_t run0_snap, cudaStream_t stream, uint64_t* launches) {
    cd_pred_walk<<<p.run_ctas, RP_WARPS * 32, 0, stream>>>(p.st, p.cs, p.nruns, round, p.flags, p.K, p.entP, p.snap, p.ctx_in, p.ctx_out, p.dirty_cur,
                                                           p.dirty_next, p.run_epoch, p.rbits, out32, run0_snap);
    ++*launches;
}
// ... and the snapshots from the table carried into this round (d_pred_carry: nullptr = the stream start's zeros)
static void cd_launch_pred_fold(const CheeDecPtrs& p, uint32_t round, const uint32_t* d_pred_carry, cudaStream_t stream, uint64_t* launches) {
    cd_pred_fold<<<PL / 128, 128, 0, stream>>>(p.st, p.cs, p.nruns, round, p.entP, p.snap, p.run_epoch, p.rbits, p.dirty_next, p.pred_final, d_pred_carry);
    ++*launches;
}
// the verdict of the rounds: *d_fallback != 0 afterwards means the in-order kernel must run instead
static void cd_launch_finish(const CheeDecPtrs& p, uint32_t* d_fallback, uint64_t* d_out_size, cudaStream_t stream, uint64_t* launches) {
    cd_finish<<<1, 1, 0, stream>>>(p.st, p.cs, d_fallback, d_out_size);
    ++*launches;
}

// Enqueues the parallel Cheetah decode. The block count of the main loop is only known on the device; the output needs
// cap >= main_blocks * 128 (checked on the device). *d_fallback != 0 afterwards: the caller's in-order kernel must run instead.
// `tail_ws` = the scalar workspace (scalar_codec.cu layout): receives the folded tables for the tail loop.
cudaError_t chee_decode_parallel(const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws, uint8_t* tables, uint8_t* tail_ws,
                                 int num_sms, uint64_t* d_out_size, uint32_t* d_fallback, cudaStream_t stream, uint64_t* launches) {
    const CheeDecPtrs p(nbytes, cap, num_sms, ws, tables, tail_ws);
    cudaError_t e = bounds::bounds_launch<bounds::CheeT>(d_in, nbytes, cap, ws, p.B, stream, launches);
    if (e == cudaSuccess) e = cd_clear_tables(p, stream);
    if (e != cudaSuccess) return e;
    uint32_t* out32 = reinterpret_cast<uint32_t*>(d_out);
    cd_launch_unpack_walk(p, d_in, out32, stream, launches);
    cd_launch_cmap_resolve(p, out32, nullptr, stream, launches);
    for (uint32_t round = 0; round < (uint32_t)MAX_ROUNDS; ++round) {
        cd_launch_pred_walk(p, round, out32, 1u, stream, launches);
        cd_launch_pred_fold(p, round, nullptr, stream, launches);
        cd_round_end<<<1, 32, 0, stream>>>(p.cs, p.nruns, round, p.ctx_in, p.ctx_out, p.dirty_cur, p.dirty_next);
        ++*launches;
    }
    cd_launch_finish(p, d_fallback, d_out_size, stream, launches);
    return cudaGetLastError();
}

// device addresses the tail kernel needs (scalar_codec.cu): boundary status + iteration status
const void* chee_decode_status_ptr(uint8_t* ws, size_t nbytes, size_t cap, int num_sms, const void** cl_status) {
    const CheeDecPtrs p(nbytes, cap, num_sms, ws, nullptr, nullptr);
    if (cl_status) *cl_status = p.cs;
    return p.st;
}

// Enqueues the parallel Lion decode: boundaries, unpack, the chunk-map passes (the Cheetah decoder's kernels on the Lion geometry), the
// prediction walk on the tail's table, the verdict. *d_fallback != 0 afterwards (a boundary error: malformed stream or capacity): the
// caller's in-order kernel must run instead. `tail_ws` = the scalar workspace: receives the chunk map and the walked table for the tail.
cudaError_t lion_decode_parallel(const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws, uint8_t* tables, uint8_t* tail_ws,
                                 int num_sms, uint64_t* d_out_size, uint32_t* d_fallback, cudaStream_t stream, uint64_t* launches) {
    const CheeDecPtrs p(nbytes, cap, num_sms, ws, tables, tail_ws, true);
    LionStatus* ls = reinterpret_cast<LionStatus*>(p.cs);
    cudaError_t e = bounds::bounds_launch<bounds::LionT>(d_in, nbytes, cap, ws, p.B, stream, launches);
    if (e == cudaSuccess) e = cd_clear_tables(p, stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(ls, 0, sizeof(LionStatus), stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(p.pred_final, 0, (size_t)5 * PL * sizeof(uint32_t), stream);   // lion.rs:70
    if (e != cudaSuccess) return e;
    uint32_t* out32 = reinterpret_cast<uint32_t*>(d_out);
    cd_launch_unpack_walk<bounds::LionT>(p, d_in, out32, stream, launches);
    cd_launch_cmap_resolve<bounds::LionT>(p, out32, nullptr, stream, launches);
    ld_walk<<<1, 32, 0, stream>>>(p.st, p.flags, p.K, out32, p.pred_final, ls, nullptr, nullptr);
    ++*launches;
    cd_launch_finish(p, d_fallback, d_out_size, stream, launches);
    return cudaGetLastError();
}

// device addresses the tail kernel needs: boundary status + walk status (its ClStatus prefix; the counts follow it)
const void* lion_decode_status_ptr(uint8_t* ws, size_t nbytes, size_t cap, int num_sms, const void** walk_status) {
    const CheeDecPtrs p(nbytes, cap, num_sms, ws, nullptr, nullptr, true);
    if (walk_status) *walk_status = p.cs;
    return p.st;
}

// ---- sharded decode: one piece, in phases around the exchanges (include/density_b200.h, DESIGN.md section 5) --------------------------
// One piece protocol for both run-parallel decoders: a.lion picks the geometry (bounds::CheeT or bounds::LionT) of every step below.
// Between phase 2 and phase 3 Cheetah runs the prediction rounds (chee_shard_round_walk / _fold), Lion the walk on the state the pieces
// before it left (lion_shard_walk).
static CheeDecPtrs chee_shard_ptrs(const CheeShardArgs& a) { return CheeDecPtrs(a.n, a.cap, a.num_sms, a.ws, a.tables, nullptr, a.lion); }

size_t chee_shard_workspace_bytes(size_t n, size_t cap, int num_sms, bool lion) {
    CheeDecLayout L;
    const size_t off = (cd_layout(n, cap, cd_pick_runs(n, num_sms), &L, lion) + 255) & ~(size_t)255;
    return off + 256 + scalar_workspace_bytes(lion ? ALG_LION : ALG_CHEETAH);
}

// Phase 1: boundaries (piece 0 may use copy mode: dec_seq_walk from the fresh automaton), the end of the piece, unpack (literals and
// copy-mode blocks go straight to d_out), the symbolic chunk-map walk and the piece's chunk-map transfer (d_cmap_out, may be null).
// d_seed (the protected path, nullptr otherwise): the piece's incoming state; rows_ready: chee_shard_prot_transfer filled the candidate rows.
template <class G>
static cudaError_t shard_phase1(const CheeShardArgs& a, uint32_t* d_cmap_out, cudaStream_t stream, uint64_t* launches, const uint32_t* d_seed,
                                bool rows_ready) {
    const CheeDecPtrs p = chee_shard_ptrs(a);
    cudaError_t e = bounds::bounds_launch<G>(a.d_in, a.n, a.cap, a.ws, p.B, stream, launches, d_seed, rows_ready);
    if (e == cudaSuccess) e = cd_clear_tables(p, stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(p.tail_ws, 0, 256, stream);
    if (e == cudaSuccess && a.lion) e = cudaMemsetAsync(p.cs, 0, sizeof(LionStatus), stream);
    if (e != cudaSuccess) return e;
    cd_piece_end<G><<<1, 32, 0, stream>>>(a.d_in, a.n, a.cap, a.first ? 1 : 0, a.last ? 1 : 0, d_seed ? 1 : 0, p.st, p.blk_off, p.B.maxblocks, p.pst);
    ++*launches;
    cd_launch_unpack_walk<G>(p, a.d_in, reinterpret_cast<uint32_t*>(a.d_out), stream, launches);
    if (d_cmap_out) { cd_cmap_export<<<PL / 256, 256, 0, stream>>>(p.st, p.nruns, p.entC, d_cmap_out); ++*launches; }
    return cudaGetLastError();
}
cudaError_t chee_shard_phase1(const CheeShardArgs& a, uint32_t* d_cmap_out, cudaStream_t stream, uint64_t* launches, const uint32_t* d_seed,
                              bool rows_ready) {
    return a.lion ? shard_phase1<bounds::LionT>(a, d_cmap_out, stream, launches, d_seed, rows_ready)
                  : shard_phase1<T>(a, d_cmap_out, stream, launches, d_seed, rows_ready);
}

// Phase 2: the chunk map carried in (d_cmap_carry: concrete, the left fold of the earlier pieces' transfers over cd_cmap_init_k's state;
// nullptr = the stream start), the reads of carried-in slots, the context init (Cheetah).
cudaError_t chee_shard_phase2(const CheeShardArgs& a, const uint32_t* d_cmap_carry, cudaStream_t stream, uint64_t* launches) {
    const CheeDecPtrs p = chee_shard_ptrs(a);
    uint32_t* out32 = reinterpret_cast<uint32_t*>(a.d_out);
    if (a.lion) cd_launch_cmap_resolve<bounds::LionT>(p, out32, d_cmap_carry, stream, launches);
    else cd_launch_cmap_resolve<T>(p, out32, d_cmap_carry, stream, launches);
    return cudaGetLastError();
}

// A prediction round, first half: walk the dirty runs, export this round's transfer (d_pred_out, may be null) and the 4 round words.
cudaError_t chee_shard_round_walk(const CheeShardArgs& a, uint32_t round, uint32_t* d_pred_out, uint32_t* d_words, cudaStream_t stream, uint64_t* launches) {
    const CheeDecPtrs p = chee_shard_ptrs(a);
    cd_launch_pred_walk(p, round, reinterpret_cast<uint32_t*>(a.d_out), a.first ? 1u : 0u, stream, launches);
    if (d_pred_out) { cd_pred_export<<<PL / 128, 128, 0, stream>>>(p.cs, p.nruns, p.entP, p.run_epoch, d_pred_out); ++*launches; }
    cd_round_words<<<1, 256, 0, stream>>>(p.st, p.cs, p.nruns, p.ctx_out, p.dirty_cur, p.dirty_next, d_words);
    ++*launches;
    return cudaGetLastError();
}

// Second half: the snapshots from the carried-in table of this round (d_pred_carry, nullptr = the stream start's zeros) and the
// context sweep from the gathered round words of all `world` pieces.
cudaError_t chee_shard_round_fold(const CheeShardArgs& a, uint32_t round, const uint32_t* d_pred_carry, const uint32_t* d_all_words, uint32_t world,
                                  uint32_t rank, cudaStream_t stream, uint64_t* launches) {
    const CheeDecPtrs p = chee_shard_ptrs(a);
    cd_launch_pred_fold(p, round, d_pred_carry, stream, launches);
    cd_shard_round_end<<<1, 32, 0, stream>>>(p.cs, p.nruns, round, a.first ? 1u : 0u, rank, world, d_all_words, p.ctx_in, p.ctx_out, p.dirty_cur, p.dirty_next);
    ++*launches;
    return cudaGetLastError();
}

// The walk from the relayed state d_state (LION_STATE_WORDS: the 65536 lists, then last_hash): the lists into the tail's table (the first
// piece starts from the zero table and context 0, lion.rs:67,70), ld_walk, then the table and the context behind the piece back to d_state.
cudaError_t lion_shard_walk(const CheeShardArgs& a, uint32_t* d_state, cudaStream_t stream, uint64_t* launches) {
    const CheeDecPtrs p = chee_shard_ptrs(a);
    const size_t tb = (size_t)5 * PL * sizeof(uint32_t);
    uint32_t* ctx = d_state + 5 * PL;
    cudaError_t e = a.first ? cudaMemsetAsync(p.pred_final, 0, tb, stream) : cudaMemcpyAsync(p.pred_final, d_state, tb, cudaMemcpyDeviceToDevice, stream);
    if (e != cudaSuccess) return e;
    ld_walk<<<1, 32, 0, stream>>>(p.st, p.flags, p.K, reinterpret_cast<uint32_t*>(a.d_out), p.pred_final, reinterpret_cast<LionStatus*>(p.cs),
                                  a.first ? nullptr : ctx, ctx);
    ++*launches;
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_state, p.pred_final, tb, cudaMemcpyDeviceToDevice, stream);
    return e;
}

// the stream-start state of the relay: zero lists, context 0
cudaError_t lion_state_init(uint32_t* d_state, cudaStream_t stream) {
    return cudaMemsetAsync(d_state, 0, (size_t)LION_STATE_WORDS * sizeof(uint32_t), stream);
}

// Phase 3: the verdict of the rounds (Lion: of the walk), the final piece's tail from the folded (walked) tables (the tail of a non-final
// piece is empty), the size and the seam words (d_seed: the protected path's, see cd_seam_words). An empty piece of the protected path has
// its seam words only.
template <class G>
static cudaError_t shard_phase3(const CheeShardArgs& a, uint64_t* d_out_size, uint32_t* d_seam8, cudaStream_t stream, uint64_t* launches,
                                const uint32_t* d_seed) {
    if (!a.n) {
        cd_seam_words<G::BS><<<1, 1, 0, stream>>>(nullptr, nullptr, nullptr, a.last ? 1 : 0, d_seed, d_out_size, d_seam8);
        ++*launches;
        return cudaGetLastError();
    }
    const CheeDecPtrs p = chee_shard_ptrs(a);
    cd_launch_finish(p, p.fallback, d_out_size, stream, launches);
    cudaError_t e = scalar_decode_tail(a.lion ? ALG_LION : ALG_CHEETAH, a.d_in, a.n, a.d_out, a.cap, p.tail_ws, p.st, p.cs, d_out_size, stream,
                                       launches, p.fallback);
    if (e != cudaSuccess) return e;
    cd_seam_words<G::BS><<<1, 1, 0, stream>>>(p.pst, p.fallback, reinterpret_cast<const Status*>(p.tail_ws), a.last ? 1 : 0, d_seed, d_out_size, d_seam8);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t chee_shard_phase3(const CheeShardArgs& a, uint64_t* d_out_size, uint32_t* d_seam8, cudaStream_t stream, uint64_t* launches,
                              const uint32_t* d_seed) {
    return a.lion ? shard_phase3<bounds::LionT>(a, d_out_size, d_seam8, stream, launches, d_seed)
                  : shard_phase3<T>(a, d_out_size, d_seam8, stream, launches, d_seed);
}

// The protected path's first step on a piece (DESIGN.md section 5): the candidate rows of the boundary walk (they stay in the workspace
// for the phase 1 with a seed), then the head walk over them, PT_NCAND words to d_transfer. An empty piece reads nothing.
cudaError_t chee_shard_prot_transfer(const CheeShardArgs& a, uint32_t* d_transfer, cudaStream_t stream, uint64_t* launches) {
    return a.lion ? bounds::prot_transfer_launch<bounds::LionT>(a.d_in, a.n, a.last ? 1 : 0, a.ws, d_transfer, stream, launches)
                  : bounds::prot_transfer_launch<T>(a.d_in, a.n, a.last ? 1 : 0, a.ws, d_transfer, stream, launches);
}
// The incoming state of piece `rank` composed from candidate x0 and the transfers of the pieces before it (DECODE_PROT_SEED_WORDS to d_seed).
cudaError_t chee_shard_prot_enter(const uint32_t* d_all_transfers, uint32_t rank, uint32_t x0, uint32_t* d_seed, cudaStream_t stream,
                                  uint64_t* launches) {
    bounds::dec_prot_enter_k<<<1, 32, 0, stream>>>(d_all_transfers, rank, x0, d_seed);
    ++*launches;
    return cudaGetLastError();
}

// the diagnostic words of the piece's iteration (ClStatus, 8 x u32; Lion: the walk's LionStatus, a ClStatus prefix, then the 4 u64 counts)
const void* chee_shard_status_ptr(const CheeShardArgs& a) { return chee_shard_ptrs(a).cs; }

cudaError_t chee_cmap_identity(uint32_t* d_table, cudaStream_t stream, uint64_t* launches) {
    cd_cmap_export<<<PL / 256, 256, 0, stream>>>(nullptr, 0, nullptr, d_table); ++*launches; return cudaGetLastError();
}
cudaError_t chee_cmap_init(uint32_t* d_table, cudaStream_t stream, uint64_t* launches) {
    cd_cmap_init_k<<<PL / 256, 256, 0, stream>>>(d_table); ++*launches; return cudaGetLastError();
}
cudaError_t chee_cmap_fold(uint32_t* d_acc, const uint32_t* d_next, cudaStream_t stream, uint64_t* launches) {
    cd_cmap_fold_k<<<PL / 256, 256, 0, stream>>>(d_acc, d_next); ++*launches; return cudaGetLastError();
}
cudaError_t chee_cmap_rank_fold(const uint32_t* d_tables, uint32_t rank, uint32_t* d_carry, cudaStream_t stream, uint64_t* launches) {
    cd_cmap_rank_fold_k<<<PL / 128, 128, 0, stream>>>(d_tables, rank, d_carry); ++*launches; return cudaGetLastError();
}
uint32_t chee_shard_max_rounds() { return MAX_ROUNDS; }

// ---- the range map of a piece of a Cheetah stream without known cuts (DENSITY_B200_CHEETAH_LOCATE_MAP_WORDS u64) ---------------------
// Any range: the candidate walks over its chunks (the halo visible to its last chunk's walks), their composition per group and over the
// whole range, as cham_decode_locate does, then {range_offset, 0, 0, 0}. The range that holds the stream start (range_offset 0, n_range
// > 0) instead runs the exact boundary walk over range + halo and reads its start row off it (dec_start_row); its candidate rows are the
// identity. Its scratch is the whole boundary layout with one offset per possible block.
static bool chee_locate_has_start(size_t n_range, uint64_t range_offset) { return range_offset == 0 && n_range > 0; }

size_t chee_locate_workspace_bytes(size_t n_range, size_t n_halo, uint64_t range_offset) {
    bounds::BoundsLayout B;
    return bounds::bounds_layout<T>(n_range + n_halo, chee_locate_has_start(n_range, range_offset) ? ~(size_t)0 : 0, &B);
}

cudaError_t chee_decode_locate(const uint8_t* d_in, size_t n_range, size_t n_halo, uint64_t range_offset, uint8_t* ws, uint64_t* d_map,
                               cudaStream_t stream, uint64_t* launches) {
    const bool start = chee_locate_has_start(n_range, range_offset);
    bounds::BoundsLayout B; bounds::bounds_layout<T>(n_range + n_halo, start ? ~(size_t)0 : 0, &B);
    unsigned long long* map = reinterpret_cast<unsigned long long*>(d_map);
    if (start) {
        const cudaError_t e = bounds::bounds_launch<T>(d_in, n_range + n_halo, ~(size_t)0, ws, B, stream, launches);
        if (e != cudaSuccess) return e;
        // no group folded: the identity rows
        bounds::dec_range_compose<T><<<1, bounds::RC_THREADS, 0, stream>>>(reinterpret_cast<const uint4*>(ws + B.gres), 0, n_range, n_halo, map);
        ++*launches;
    } else {
        bounds::range_map_launch<T>(d_in, n_range, n_halo, ws, map, stream, launches);
    }
    bounds::dec_start_row<T><<<1, 32, 0, stream>>>(start ? reinterpret_cast<const DecStatus*>(ws + B.status) : nullptr,
                                                   reinterpret_cast<const uint64_t*>(ws + B.blk_off), n_range, range_offset,
                                                   map + 2 + 2 * T::NCAND);
    ++*launches;
    return cudaGetLastError();
}

// ---- the protected range map of a piece of a Cheetah stream without known cuts (DENSITY_B200_CHEETAH_PROT_LOCATE_MAP_WORDS u32) --------
// Every range alike, the one with the stream start included: its row (0, 0) is the exact walk from the fresh automaton.
size_t chee_prot_locate_workspace_bytes(size_t nbytes) { bounds::BoundsLayout B; return bounds::bounds_layout<T>(nbytes, 0, &B); }

cudaError_t chee_decode_prot_locate(const uint8_t* d_in, size_t n_range, size_t n_halo, uint8_t* ws, uint32_t* d_map, cudaStream_t stream,
                                    uint64_t* launches) {
    return bounds::prot_locate_launch<T>(d_in, n_range, n_halo, ws, d_map, stream, launches);
}

}  // namespace dns
