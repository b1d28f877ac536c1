// cheetah_encode.cu — run-parallel Cheetah and Lion encode for sm_90a (the Lion kernels start at "Lion (lion.rs:209-271)").
//
// Replaces cheetah.rs:121-150 and lion.rs:209-271 (encode_quad) driven by codec.rs:34-80, bit-exactly. Cheetah's decomposition (validated against the oracle by
// tools/proto_cheetah_runs.py; Lion's differs in step 1 only, see below and tools/proto_lion_runs.py):
//
//  1. PREDICTED_i <=> quad_i == the quad that followed the previous occurrence of the same CONTEXT, where the context is the
//     hash of the previous *encoded* quad (0 at the stream start) and the prediction table starts as "0 everywhere"
//     (cheetah.rs:53,125,144,148: pred[ctx] always ends up holding the last quad seen in that context).
//  2. On the subsequence of NON-predicted quads each hash bucket keeps an MRU-2 of values (a, b) (cheetah.rs:127-143):
//        v == a -> MAP_A, nothing changes;  v == b -> MAP_B, (a, b) <- (v, a);  else PLAIN, (a, b) <- (v, a).
//     Values are compared as the 16-bit in-bucket fingerprints of common.cuh.
//  3. Copy-mode blocks (codec/protection_state.rs) touch neither table nor the context chain; the copy map is the fixed point
//     of  M -> automaton(incompressible bits under M)  (prot_iterate, shared with the Chameleon encoder). Cheetah needs the
//     iteration on every input: a cold dictionary makes the first blocks incompressible (11 copied blocks on dickens).
//
// Parallelisation: the stream is cut into R contiguous runs (up to 8 per SM), ONE WARP PER RUN walks its run 32 quads at a time
// (one Cheetah block = one quad per lane), with the run's tables in global memory (768 KiB do not fit an SM) as epoch-tagged
// 16-byte entries: an entry whose tag is not the current round's counts as untouched, so the tables are never cleared. In-warp predecessors come from __match_any_sync; what a run cannot know — the tables carried in from earlier runs —
// is left "unresolved": per run and context at most one PREDICTED decision, per run and bucket at most two map decisions (the
// first touch, and the first access that differs from it). One fold kernel per table then walks the runs in order per
// context / bucket, resolves those accesses and carries the state on. Pass P (predictions) must be completely resolved before
// pass C (chunk map) starts, because only non-predicted quads take part in it.
#include <stdlib.h>
#include "common.cuh"
#include "encode_internal.cuh"

namespace dns {
namespace chee {

constexpr int TILE_B = 128;                 // blocks per tile (4096 quads = 16 KiB), the unit of run geometry and of the emit grid
constexpr uint32_t FP_INVALID = 0x10000u;   // a fingerprint value that matches nothing (bucket h != 0 initially "holds quad 0")

__device__ __forceinline__ uint64_t run_block_begin(uint32_t r, uint32_t nruns, uint64_t ntiles) { return ((uint64_t)r * ntiles / nruns) * TILE_B; }

// context of the first encoded quad of every run: hash of the last quad of the last encoded block before the run (0 if none; a
// shard of a longer stream passes the last quad of the shard before it in `prev_quad`). ctx0 opens every round that runs, so
// `epoch_out` (may be nullptr) ends up holding the epoch of the last one: the settled round once the copy map has converged.
__global__ void chee_ctx0(const uint32_t* __restrict__ in, uint64_t nquads, const uint8_t* __restrict__ copymap, uint32_t nruns, uint64_t ntiles,
                          const Status* __restrict__ gate, const uint32_t* __restrict__ prev_quad, uint32_t epoch, uint32_t* __restrict__ epoch_out,
                          uint32_t* __restrict__ ctx0) {
    if (gate && !(gate->nonquiet && !gate->converged)) return;
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (epoch_out && r == 0) *epoch_out = epoch;
    if (r >= nruns) return;
    uint64_t b = run_block_begin(r, nruns, ntiles);
    uint32_t c = prev_quad ? prod_hash(hash_prod(*prev_quad)) : 0u;
    while (b > 0) {
        --b;
        if (copymap && copymap[b]) continue;
        const uint64_t qi = b * 32 + 31;          // blocks before a run start are full blocks
        if (qi < nquads) c = prod_hash(hash_prod(in[qi]));
        break;
    }
    ctx0[r] = c;
}

constexpr int RP_WARPS = 4;   // warps (runs) per CTA

// ---- pass P: PREDICTED flags ----------------------------------------------------------------------------------------------
// Table entry per (run, context): {last quad seen, epoch, 1 + index of the run's first (unresolved) access, 0}. An entry whose epoch
// differs from the current round's is "untouched": no memset between rounds / calls (the workspace is zeroed once, epochs start at 1).
__global__ void __launch_bounds__(RP_WARPS * 32)
chee_pass_p(const uint32_t* __restrict__ in, uint64_t nquads, uint64_t nblocks, const uint8_t* __restrict__ copymap, uint32_t nruns, uint64_t ntiles,
            const Status* __restrict__ gate, const uint32_t* __restrict__ ctx0, uint4* __restrict__ entP_all, uint32_t epoch,
            uint32_t* __restrict__ Pbits) {
    if (gate && !(gate->nonquiet && !gate->converged)) return;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t r = blockIdx.x * RP_WARPS + (threadIdx.x >> 5);
    if (r >= nruns) return;
    uint4* __restrict__ entP = entP_all + (size_t)r * 65536;
    const uint64_t b0 = run_block_begin(r, nruns, ntiles);
    uint64_t b1 = run_block_begin(r + 1, nruns, ntiles);
    if (b1 > nblocks) b1 = nblocks;
    uint32_t last_h = ctx0[r];
    uint32_t qn = (b0 < b1 && b0 * 32 + lane < nquads) ? ld_stream_u32(in + b0 * 32 + lane) : 0u;   // software prefetch, one block ahead
    for (uint64_t b = b0; b < b1; ++b) {
        const uint32_t q = qn;
        if (b + 1 < b1) qn = ((b + 1) * 32 + lane < nquads) ? ld_stream_u32(in + (b + 1) * 32 + lane) : 0u;
        if (copymap && copymap[b]) { if (lane == 0) Pbits[b] = 0; continue; }
        const uint64_t q0 = b * 32;
        const uint32_t nq = (q0 >= nquads) ? 0u : (uint32_t)((nquads - q0 < 32) ? (nquads - q0) : 32);
        if (nq == 0) { if (lane == 0) Pbits[b] = 0; continue; }
        const bool active = lane < nq;
        const uint32_t h = prod_hash(hash_prod(q));
        const uint32_t hp = __shfl_up_sync(0xFFFFFFFFu, h, 1);
        const uint32_t ctx = lane ? hp : last_h;
        last_h = __shfl_sync(0xFFFFFFFFu, h, nq - 1);
        uint4 e = make_uint4(0, 0, 0, 0);
        if (active) e = __ldcg(&entP[ctx]);                           // issued for every lane up front: one 16-byte access
        const uint32_t key = active ? ctx : 0x10000u + lane;
        const uint32_t grp = __match_any_sync(0xFFFFFFFFu, key);
        const uint32_t lower = grp & lanemask_lt();
        const int src = lower ? 31 - __clz(lower) : 0;
        const uint32_t qprev = __shfl_sync(0xFFFFFFFFu, q, src);
        const bool touched = e.y == epoch;
        const bool known = lower != 0 || touched;
        const uint32_t pv = lower ? qprev : e.x;
        const bool P = active && known && pv == q;
        // the group's first lane owns the "first access" slot, its last lane leaves the value (cheetah.rs:144; :148 is implied)
        uint32_t u1 = touched ? e.z : 0u;
        if (active && !lower && !touched) u1 = (uint32_t)(q0 + lane) + 1u;
        const uint32_t u1g = __shfl_sync(0xFFFFFFFFu, u1, __ffs(grp) - 1);
        if (active && (grp & lanemask_gt()) == 0) entP[ctx] = make_uint4(q, epoch, u1g, 0u);
        const uint32_t pm = __ballot_sync(0xFFFFFFFFu, P);
        if (lane == 0) Pbits[b] = pm;
        __syncwarp();
    }
}

// walk the runs in order per context: resolve each run's first access from the carried-in value, carry the run's last value on.
// `carry` (nullptr: the stream start) = the value per context before the first run, for a shard of a longer stream.
__global__ void chee_fold_p(const uint32_t* __restrict__ in, uint32_t nruns, const Status* __restrict__ gate, const uint4* __restrict__ entP_all,
                            uint32_t epoch, const uint32_t* __restrict__ carry, uint32_t* __restrict__ Pbits) {
    if (gate && !(gate->nonquiet && !gate->converged)) return;
    const uint32_t ctx = blockIdx.x * blockDim.x + threadIdx.x;
    if (ctx >= 65536) return;
    uint32_t c = carry ? carry[ctx] : 0u;                             // prediction table starts as 0 everywhere (cheetah.rs:53)
    for (uint32_t r0 = 0; r0 < nruns; r0 += 8) {
        uint4 e[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) e[k] = (r0 + k < nruns) ? entP_all[(size_t)(r0 + k) * 65536 + ctx] : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            if (e[k].y != epoch) continue;
            const uint32_t i = e[k].z - 1;
            if (in[i] == c) atomicOr(&Pbits[i >> 5], 1u << (i & 31));
            c = e[k].x;
        }
    }
}

// ---- pass C: chunk map (MRU-2) on the non-predicted quads -----------------------------------------------------------------
// Table entry per (run, bucket): {a | b << 16, epoch << 2 | T, 1 + index of the first access, 1 + index of the first access that differs}
// T: 0 untouched, 1 a known, 2 a and b known.
// BPS = blocks per 32-quad step: Cheetah 1 (128-byte blocks), Lion 2 (64-byte blocks, lanes 0-15 / 16-31).
template <int BPS>
__device__ __forceinline__ uint32_t step_active_lanes(const uint8_t* __restrict__ copymap, uint64_t s, uint64_t nblocks_alg) {
    if (!copymap) return 0xFFFFFFFFu;
    if (BPS == 1) return copymap[s] ? 0u : 0xFFFFFFFFu;
    uint32_t m = 0;
    if (2 * s < nblocks_alg && !copymap[2 * s]) m |= 0x0000FFFFu;
    if (2 * s + 1 < nblocks_alg && !copymap[2 * s + 1]) m |= 0xFFFF0000u;
    return m;
}

template <int BPS>
__global__ void __launch_bounds__(RP_WARPS * 32)
chee_pass_c(const uint32_t* __restrict__ in, uint64_t nquads, uint64_t nblocks, uint64_t nblocks_alg, const uint8_t* __restrict__ copymap, uint32_t nruns,
            uint64_t ntiles, const Status* __restrict__ gate, const uint32_t* __restrict__ Pbits, uint4* __restrict__ entC_all, uint32_t epoch,
            uint32_t* __restrict__ Abits, uint32_t* __restrict__ Bbits) {
    if (gate && !(gate->nonquiet && !gate->converged)) return;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t r = blockIdx.x * RP_WARPS + (threadIdx.x >> 5);
    if (r >= nruns) return;
    uint4* __restrict__ entC = entC_all + (size_t)r * 65536;
    const uint64_t b0 = run_block_begin(r, nruns, ntiles);
    uint64_t b1 = run_block_begin(r + 1, nruns, ntiles);
    if (b1 > nblocks) b1 = nblocks;
    uint32_t qn = (b0 < b1 && b0 * 32 + lane < nquads) ? ld_stream_u32(in + b0 * 32 + lane) : 0u;
    uint32_t pmn = (b0 < b1) ? __ldcg(&Pbits[b0]) : 0u;
    for (uint64_t b = b0; b < b1; ++b) {
        const uint32_t q = qn, pm = pmn;
        if (b + 1 < b1) { qn = ((b + 1) * 32 + lane < nquads) ? ld_stream_u32(in + (b + 1) * 32 + lane) : 0u; pmn = __ldcg(&Pbits[b + 1]); }
        const uint32_t act = step_active_lanes<BPS>(copymap, b, nblocks_alg);
        if (act == 0) { if (lane == 0) { Abits[b] = 0; Bbits[b] = 0; } continue; }
        const uint64_t q0 = b * 32;
        const uint32_t nq = (q0 >= nquads) ? 0u : (uint32_t)((nquads - q0 < 32) ? (nquads - q0) : 32);
        if (nq == 0) { if (lane == 0) { Abits[b] = 0; Bbits[b] = 0; } continue; }
        const bool member = lane < nq && ((act >> lane) & 1u) && !((pm >> lane) & 1u);
        const uint32_t p = hash_prod(q);
        const uint32_t h = prod_hash(p), v = prod_fp(p, q);
        uint4 e = make_uint4(0, 0, 0, 0);
        if (member) e = __ldcg(&entC[h]);
        const uint32_t key = member ? h : 0x10000u + lane;
        const uint32_t grp = __match_any_sync(0xFFFFFFFFu, key);
        const uint32_t lower = grp & lanemask_lt();
        const uint32_t rank = __popc(lower);
        const int src = lower ? 31 - __clz(lower) : (int)lane;
        const uint32_t maxrank = __reduce_max_sync(0xFFFFFFFFu, member ? rank : 0u);
        // state before my access: the first lane of a group takes it from the table, the others from their in-warp predecessor
        const bool fresh = (e.y >> 2) == epoch;
        uint32_t a = fresh ? (e.x & 0xFFFFu) : 0u, bb = fresh ? (e.x >> 16) : 0u, T = fresh ? (e.y & 3u) : 0u;
        uint32_t u1 = fresh ? e.z : 0u, u2 = fresh ? e.w : 0u;
        uint32_t code = 0;          // 0 plain (or not yet decidable), 1 MAP_A, 2 MAP_B
        uint32_t na = 0, nb = 0, nT = 0, nu1 = 0, nu2 = 0;
        for (uint32_t rk = 0; rk <= maxrank; ++rk) {
            if (member && rank == rk) {
                nu1 = u1; nu2 = u2;
                if (T == 0) {                       // first touch of the bucket in this run: decided later from the carry-in
                    nu1 = (uint32_t)(q0 + lane) + 1u; na = v; nb = 0; nT = 1;
                } else if (T == 1) {
                    if (v == a) { code = 1; na = a; nb = 0; nT = 1; }
                    else { nu2 = (uint32_t)(q0 + lane) + 1u; na = v; nb = a; nT = 2; }        // MAP_B iff v == (unknown) b: decided later
                } else {
                    if (v == a) { code = 1; na = a; nb = bb; }
                    else { code = (v == bb) ? 2u : 0u; na = v; nb = a; }                       // cheetah.rs:137-142
                    nT = 2;
                }
            }
            const uint32_t ra = __shfl_sync(0xFFFFFFFFu, na, src), rb = __shfl_sync(0xFFFFFFFFu, nb, src), rT = __shfl_sync(0xFFFFFFFFu, nT, src);
            const uint32_t r1 = __shfl_sync(0xFFFFFFFFu, nu1, src), r2 = __shfl_sync(0xFFFFFFFFu, nu2, src);
            if (member && rank == rk + 1) { a = ra; bb = rb; T = rT; u1 = r1; u2 = r2; }
        }
        if (member && (grp & lanemask_gt()) == 0) entC[h] = make_uint4(na | (nb << 16), (epoch << 2) | nT, nu1, nu2);
        const uint32_t am = __ballot_sync(0xFFFFFFFFu, code == 1), bm = __ballot_sync(0xFFFFFFFFu, code == 2);
        if (lane == 0) { Abits[b] = am; Bbits[b] = bm; }
        __syncwarp();
    }
}

// walk the runs in order per bucket: resolve the (at most two) undecided accesses of each run, carry (a, b) on.
// `carry` (nullptr: the stream start) = planes a, b (65536 words apart) before the first run, for a shard of a longer stream.
__global__ void chee_fold_c(const uint32_t* __restrict__ in, uint32_t nruns, const Status* __restrict__ gate, const uint4* __restrict__ entC_all,
                            uint32_t epoch, const uint32_t* __restrict__ carry, uint32_t* __restrict__ Abits, uint32_t* __restrict__ Bbits) {
    if (gate && !(gate->nonquiet && !gate->converged)) return;
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= 65536) return;
    // chunk map starts as (quad 0, quad 0) (cheetah.rs:52): only bucket 0 can ever match that
    uint32_t a0 = h ? FP_INVALID : 0u, b0 = a0;
    if (carry) { a0 = carry[h]; b0 = carry[65536 + h]; }
    for (uint32_t r0 = 0; r0 < nruns; r0 += 8) {
        uint4 e[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) e[k] = (r0 + k < nruns) ? entC_all[(size_t)(r0 + k) * 65536 + h] : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            if ((e[k].y >> 2) != epoch) continue;
            const uint32_t T = e[k].y & 3u;
            const uint32_t i1 = e[k].z - 1;
            const uint32_t q1 = in[i1];
            const uint32_t v1 = prod_fp(hash_prod(q1), q1);
            uint32_t bafter;
            if (v1 == a0) { atomicOr(&Abits[i1 >> 5], 1u << (i1 & 31)); bafter = b0; }
            else { if (v1 == b0) atomicOr(&Bbits[i1 >> 5], 1u << (i1 & 31)); bafter = a0; }
            if (T == 2) {
                const uint32_t i2 = e[k].w - 1;
                const uint32_t q2 = in[i2];
                const uint32_t v2 = prod_fp(hash_prod(q2), q2);
                if (v2 == bafter) atomicOr(&Bbits[i2 >> 5], 1u << (i2 & 31));
                a0 = e[k].x & 0xFFFFu; b0 = e[k].x >> 16;
            } else if (v1 != a0) {                  // the run accessed the bucket with one value only
                b0 = a0; a0 = v1;
            }
        }
    }
}

// ---- sizes + incompressible bits ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t chee_block_bytes(uint64_t b, uint64_t nbytes, uint32_t pm, uint32_t am, uint32_t bm, bool copied) {
    const uint64_t boff = b * 128;
    const uint32_t blen = (uint32_t)((nbytes - boff < 128) ? (nbytes - boff) : 128);
    if (copied) return blen;
    const uint32_t nq = blen >> 2;
    const uint32_t act = nq >= 32 ? 0xFFFFFFFFu : ((1u << nq) - 1u);
    const uint32_t maps = (am | bm) & act;
    const uint32_t plain = act & ~(pm | am | bm);
    return 8 + 4 * __popc(plain) + 2 * __popc(maps) + (blen & 3u);
}

// one warp per tile of 128 blocks (4 per lane): tile byte counts; refreshes the incompressible bits of the encoded blocks
__global__ void chee_tile_sizes(const uint32_t* __restrict__ Pbits, const uint32_t* __restrict__ Abits, const uint32_t* __restrict__ Bbits,
                                const uint8_t* __restrict__ copymap, uint64_t nbytes, uint64_t nblocks, uint32_t ntiles, int final_pass,
                                const Status* __restrict__ st, uint8_t* __restrict__ inc, uint32_t* __restrict__ tile_bytes) {
    if (!final_pass && !(st->nonquiet && !st->converged)) return;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t tile = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (tile >= ntiles) return;
    uint32_t sum = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint64_t b = (uint64_t)tile * TILE_B + k * 32 + lane;
        if (b < nblocks) {
            const bool copied = copymap && copymap[b];
            const uint32_t sz = chee_block_bytes(b, nbytes, Pbits[b], Abits[b], Bbits[b], copied);
            sum += sz;
            if (!final_pass && !copied) inc[b] = (nbytes - b * 128 >= 128) && sz >= 128;     // codec.rs:68
        }
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, d);
    if (lane == 0) tile_bytes[tile] = sum;
}

// ---- emit: one CTA (256 threads) per tile of 128 blocks, warp w handles blocks w, w+8, ... ----------------------------------------
__device__ __forceinline__ uint32_t part1by1(uint32_t x) {   // spread the low 16 bits to the even bit positions
    x &= 0xFFFFu; x = (x | (x << 8)) & 0x00FF00FFu; x = (x | (x << 4)) & 0x0F0F0F0Fu; x = (x | (x << 2)) & 0x33333333u; x = (x | (x << 1)) & 0x55555555u;
    return x;
}
__global__ void __launch_bounds__(256)
chee_emit(const uint32_t* __restrict__ in, uint64_t nbytes, uint64_t nblocks, const uint32_t* __restrict__ Pbits, const uint32_t* __restrict__ Abits,
          const uint32_t* __restrict__ Bbits, const uint8_t* __restrict__ copymap, const Status* __restrict__ status,
          const uint32_t* __restrict__ tile_local, const uint64_t* __restrict__ group_off, uint32_t scan_group, uint8_t* __restrict__ out) {
    if (status->error || !status->converged) return;
    __shared__ uint32_t s_off[TILE_B + 1];
    __shared__ uint32_t s_wsum[4];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tile = blockIdx.x;
    const uint64_t tile_off = group_off[tile / scan_group] + tile_local[tile];
    const uint64_t nquads = nbytes / 4;
    if (tid < TILE_B) {
        const uint64_t b = (uint64_t)tile * TILE_B + tid;
        uint32_t sz = 0;
        if (b < nblocks) sz = chee_block_bytes(b, nbytes, Pbits[b], Abits[b], Bbits[b], copymap && copymap[b]);
        uint32_t incl = sz;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= (uint32_t)d) incl += u; }
        if (lane == 31) s_wsum[warp] = incl;
        s_off[tid + 1] = incl;
    }
    __syncthreads();
    if (tid < TILE_B && warp > 0) { uint32_t add = 0; for (uint32_t w = 0; w < warp; ++w) add += s_wsum[w]; s_off[tid + 1] += add; }
    if (tid == 0) s_off[0] = 0;
    __syncthreads();
    const uint8_t* in_b = reinterpret_cast<const uint8_t*>(in);
    for (uint32_t bl = warp; bl < TILE_B; bl += 8) {
        const uint64_t b = (uint64_t)tile * TILE_B + bl;
        if (b >= nblocks) break;
        const uint64_t boff = b * 128;
        const uint32_t blen = (uint32_t)((nbytes - boff < 128) ? (nbytes - boff) : 128);
        const uint32_t nq = blen >> 2;
        uint8_t* const bout = out + tile_off + s_off[bl];
        const uint32_t q = (lane < nq && boff / 4 + lane < nquads) ? in[boff / 4 + lane] : 0u;
        if (copymap && copymap[b]) {                        // copy-mode block: raw bytes (codec.rs:36)
            if (lane < nq) { st_u16(bout + 4 * lane, q & 0xFFFFu); st_u16(bout + 4 * lane + 2, q >> 16); }
            if (lane < (blen & 3u)) bout[(blen & ~3u) + lane] = in_b[boff + (blen & ~3u) + lane];
            continue;
        }
        const uint32_t act = nq >= 32 ? 0xFFFFFFFFu : ((1u << nq) - 1u);
        const uint32_t pm = Pbits[b] & act, am = Abits[b] & act, bm = Bbits[b] & act;
        const uint32_t maps = am | bm, plain = act & ~(pm | maps);
        if (lane < 4) {
            // signature: 2 bits per quad, MAP_A=1 MAP_B=2 PREDICTED=3 (cheetah.rs:18-21), LSB first (write_signature.rs:13-16)
            const uint32_t lowbits = am | pm, highbits = bm | pm;
            const uint32_t lo = part1by1(lowbits) | (part1by1(highbits) << 1);
            const uint32_t hi = part1by1(lowbits >> 16) | (part1by1(highbits >> 16) << 1);
            st_u16(bout + 2 * lane, ((lane < 2 ? lo : hi) >> (16 * (lane & 1))) & 0xFFFFu);
        }
        if (lane < nq) {
            uint8_t* p = bout + 8 + 4 * __popc(plain & lanemask_lt()) + 2 * __popc(maps & lanemask_lt());
            if ((plain >> lane) & 1u) { st_u16(p, q & 0xFFFFu); st_u16(p + 2, q >> 16); }       // cheetah.rs:131-132
            else if ((maps >> lane) & 1u) st_u16(p, prod_hash(hash_prod(q)));                     // cheetah.rs:134-135,140-141
        }
        if (lane < (blen & 3u)) {                           // 1..3 raw tail bytes of the last block (codec.rs:58-61)
            uint8_t* p = bout + 8 + 4 * __popc(plain) + 2 * __popc(maps);
            p[lane] = in_b[boff + (blen & ~3u) + lane];
        }
    }
}

// =====================================================================================================================================
// Lion (lion.rs:209-271): 64-byte blocks (16 quads), 3-bit flags, per CONTEXT a 5-deep move-to-front list of quads (lion.rs:43-57).
// Decomposition validated by tools/proto_lion_runs.py. A warp still walks 32 quads (= two Lion blocks) per step.
//
// Inside a run the values the run itself has put into a context's list sit at its FRONT in recency order, ahead of what is left
// of the carried-in list. An access is therefore decidable locally unless the quad is not in the run-local list while that list
// has m < 5 entries: at most 5 undecided accesses per run and context, the k-th one made with k local entries in front. The fold
// walks the runs in order per context, replays them against the carried-in remainder (found at position j -> depth k + j, the entry
// leaves the remainder; not found -> the visible remainder shrinks by one) and carries  local list + remainder  (5 entries) on.
// The chunk map on the not-predicted quads is Cheetah's (chee_pass_c<2>, chee_fold_c).
//
// Tables per (run, context): hot 32 B {p0..p4, epoch << 3 | m, -, -}; cold 32 B {1 + quad index of the k-th undecided access, k < 5}.
// =====================================================================================================================================
__global__ void lion_ctx0(const uint32_t* __restrict__ in, uint64_t nquads, const uint8_t* __restrict__ copymap, uint32_t nruns, uint64_t ntiles,
                          const Status* __restrict__ gate, const uint32_t* __restrict__ prev_quad, uint32_t epoch, uint32_t* __restrict__ epoch_out,
                          uint32_t* __restrict__ ctx0) {
    if (gate && !(gate->nonquiet && !gate->converged)) return;
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (epoch_out && r == 0) *epoch_out = epoch;
    if (r >= nruns) return;
    uint64_t b = run_block_begin(r, nruns, ntiles) * 2;       // in 64-byte blocks
    uint32_t c = prev_quad ? prod_hash(hash_prod(*prev_quad)) : 0u;
    while (b > 0) {
        --b;
        if (copymap && copymap[b]) continue;
        const uint64_t qi = b * 16 + 15;                      // blocks before a run start are full blocks
        if (qi < nquads) c = prod_hash(hash_prod(in[qi]));
        break;
    }
    ctx0[r] = c;
}

__global__ void __launch_bounds__(RP_WARPS * 32)
lion_pass_p(const uint32_t* __restrict__ in, uint64_t nquads, uint64_t nsteps, uint64_t nblocks_alg, const uint8_t* __restrict__ copymap, uint32_t nruns,
            uint64_t ntiles, const Status* __restrict__ gate, const uint32_t* __restrict__ ctx0, uint4* __restrict__ hot_all, uint32_t* __restrict__ cold_all,
            uint32_t epoch, uint32_t* __restrict__ F0, uint32_t* __restrict__ F1, uint32_t* __restrict__ F2, uint32_t* __restrict__ Pany) {
    if (gate && !(gate->nonquiet && !gate->converged)) return;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t r = blockIdx.x * RP_WARPS + (threadIdx.x >> 5);
    if (r >= nruns) return;
    uint4* __restrict__ hot = hot_all + (size_t)r * 65536 * 2;
    uint32_t* __restrict__ cold = cold_all + (size_t)r * 65536 * 8;
    const uint64_t s0 = run_block_begin(r, nruns, ntiles);
    uint64_t s1 = run_block_begin(r + 1, nruns, ntiles);
    if (s1 > nsteps) s1 = nsteps;
    uint32_t last_h = ctx0[r];
    uint32_t qn = (s0 < s1 && s0 * 32 + lane < nquads) ? ld_stream_u32(in + s0 * 32 + lane) : 0u;
    for (uint64_t s = s0; s < s1; ++s) {
        const uint32_t q = qn;
        if (s + 1 < s1) qn = ((s + 1) * 32 + lane < nquads) ? ld_stream_u32(in + (s + 1) * 32 + lane) : 0u;
        const uint64_t q0 = s * 32;
        const uint32_t nq = (q0 >= nquads) ? 0u : (uint32_t)((nquads - q0 < 32) ? (nquads - q0) : 32);
        const uint32_t act = step_active_lanes<2>(copymap, s, nblocks_alg) & (nq >= 32 ? 0xFFFFFFFFu : ((1u << nq) - 1u));
        if (act == 0) { if (lane == 0) { F0[s] = 0; F1[s] = 0; F2[s] = 0; Pany[s] = 0; } continue; }
        const bool active = (act >> lane) & 1u;
        const uint32_t h = prod_hash(hash_prod(q));
        // context = hash of the previous ENCODED quad: the nearest active lane below me, else what the warp carries along
        const uint32_t below = act & lanemask_lt();
        const uint32_t hsrc = __shfl_sync(0xFFFFFFFFu, h, below ? 31 - __clz(below) : 0);
        const uint32_t ctx = below ? hsrc : last_h;
        last_h = __shfl_sync(0xFFFFFFFFu, h, 31 - __clz(act));
        uint4 e0 = make_uint4(0, 0, 0, 0), e1 = make_uint4(0, 0, 0, 0);
        if (active) { e0 = __ldcg(&hot[2 * ctx]); e1 = __ldcg(&hot[2 * ctx + 1]); }
        const uint32_t key = active ? ctx : 0x10000u + lane;
        const uint32_t grp = __match_any_sync(0xFFFFFFFFu, key);
        const uint32_t lower = grp & lanemask_lt();
        const uint32_t rank = __popc(lower);
        const int src = lower ? 31 - __clz(lower) : (int)lane;
        const uint32_t maxrank = __reduce_max_sync(0xFFFFFFFFu, active ? rank : 0u);
        const bool fresh = (e1.y >> 3) == epoch;
        uint32_t p0 = fresh ? e0.x : 0u, p1 = fresh ? e0.y : 0u, p2 = fresh ? e0.z : 0u, p3 = fresh ? e0.w : 0u, p4 = fresh ? e1.x : 0u;
        uint32_t m = fresh ? (e1.y & 7u) : 0u;
        uint32_t n0 = 0, n1 = 0, n2 = 0, n3 = 0, n4 = 0, nm = 0, pcode = 0;
        for (uint32_t rk = 0; rk <= maxrank; ++rk) {
            if (active && rank == rk) {
                uint32_t k = 5;                                               // first (lowest) local depth holding q (lion.rs:214-262)
                if (m > 4 && p4 == q) k = 4;
                if (m > 3 && p3 == q) k = 3;
                if (m > 2 && p2 == q) k = 2;
                if (m > 1 && p1 == q) k = 1;
                if (m > 0 && p0 == q) k = 0;
                nm = m;
                if (k < 5) pcode = k + 1;
                else if (m < 5) { cold[(size_t)ctx * 8 + m] = (uint32_t)(q0 + lane) + 1u; nm = m + 1; }   // undecided: depends on the carry-in
                // entries [0..k] rotate (hit) / everything shifts (miss): n_j = j <= k ? p_(j-1) : p_j
                n0 = q; n1 = (k >= 1) ? p0 : p1; n2 = (k >= 2) ? p1 : p2; n3 = (k >= 3) ? p2 : p3; n4 = (k >= 4) ? p3 : p4;
            }
            const uint32_t r0 = __shfl_sync(0xFFFFFFFFu, n0, src), r1 = __shfl_sync(0xFFFFFFFFu, n1, src), r2 = __shfl_sync(0xFFFFFFFFu, n2, src);
            const uint32_t r3 = __shfl_sync(0xFFFFFFFFu, n3, src), r4 = __shfl_sync(0xFFFFFFFFu, n4, src), rm = __shfl_sync(0xFFFFFFFFu, nm, src);
            if (active && rank == rk + 1) { p0 = r0; p1 = r1; p2 = r2; p3 = r3; p4 = r4; m = rm; }
        }
        if (active && (grp & lanemask_gt()) == 0) {
            hot[2 * ctx] = make_uint4(n0, n1, n2, n3);
            hot[2 * ctx + 1] = make_uint4(n4, (epoch << 3) | nm, 0u, 0u);
        }
        const uint32_t f0 = __ballot_sync(0xFFFFFFFFu, pcode & 1u), f1 = __ballot_sync(0xFFFFFFFFu, pcode & 2u), f2 = __ballot_sync(0xFFFFFFFFu, pcode & 4u);
        if (lane == 0) { F0[s] = f0; F1[s] = f1; F2[s] = f2; Pany[s] = f0 | f1 | f2; }
        __syncwarp();
    }
}

// `carry` (nullptr: the stream start) = the five list planes (65536 words apart) before the first run, for a shard of a longer stream
__global__ void lion_fold_p(const uint32_t* __restrict__ in, uint32_t nruns, const Status* __restrict__ gate, const uint4* __restrict__ hot_all,
                            const uint32_t* __restrict__ cold_all, uint32_t epoch, const uint32_t* __restrict__ carry, uint32_t* __restrict__ F0,
                            uint32_t* __restrict__ F1, uint32_t* __restrict__ F2, uint32_t* __restrict__ Pany) {
    if (gate && !(gate->nonquiet && !gate->converged)) return;
    const uint32_t ctx = blockIdx.x * blockDim.x + threadIdx.x;
    if (ctx >= 65536) return;
    uint32_t c0 = 0, c1 = 0, c2 = 0, c3 = 0, c4 = 0;                 // the carried list: five zeros at the stream start (lion.rs:64-72)
    if (carry) { c0 = carry[ctx]; c1 = carry[65536 + ctx]; c2 = carry[2 * 65536 + ctx]; c3 = carry[3 * 65536 + ctx]; c4 = carry[4 * 65536 + ctx]; }
    for (uint32_t r0 = 0; r0 < nruns; r0 += 4) {
        uint4 ea[4], eb[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const bool ok = r0 + t < nruns;
            ea[t] = ok ? hot_all[((size_t)(r0 + t) * 65536 + ctx) * 2] : make_uint4(0, 0, 0, 0);
            eb[t] = ok ? hot_all[((size_t)(r0 + t) * 65536 + ctx) * 2 + 1] : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            if ((eb[t].y >> 3) != epoch) continue;
            const uint32_t mf = eb[t].y & 7u;
            const uint4* cold = reinterpret_cast<const uint4*>(cold_all + ((size_t)(r0 + t) * 65536 + ctx) * 8);
            const uint4 ua = cold[0];
            const uint32_t u4 = mf > 4 ? cold_all[((size_t)(r0 + t) * 65536 + ctx) * 8 + 4] : 0u;
            uint32_t v[5];
            v[0] = mf > 0 ? in[ua.x - 1] : 0u; v[1] = mf > 1 ? in[ua.y - 1] : 0u; v[2] = mf > 2 ? in[ua.z - 1] : 0u;
            v[3] = mf > 3 ? in[ua.w - 1] : 0u; v[4] = mf > 4 ? in[u4 - 1] : 0u;
            const uint32_t ui[5] = {ua.x, ua.y, ua.z, ua.w, u4};
#pragma unroll
            for (int k = 0; k < 5; ++k) {
                if ((uint32_t)k >= mf) break;
                const uint32_t len = 5 - k;                               // visible part of the remainder
                uint32_t j = 5;
                if (len > 4 && c4 == v[k]) j = 4;
                if (len > 3 && c3 == v[k]) j = 3;
                if (len > 2 && c2 == v[k]) j = 2;
                if (len > 1 && c1 == v[k]) j = 1;
                if (c0 == v[k]) j = 0;
                if (j < 5) {
                    const uint32_t code = k + j + 1, i = ui[k] - 1, bit = 1u << (i & 31);
                    if (code & 1u) atomicOr(&F0[i >> 5], bit);
                    if (code & 2u) atomicOr(&F1[i >> 5], bit);
                    if (code & 4u) atomicOr(&F2[i >> 5], bit);
                    atomicOr(&Pany[i >> 5], bit);
                    // the entry leaves the remainder
                    if (j <= 0) c0 = c1;
                    if (j <= 1) c1 = c2;
                    if (j <= 2) c2 = c3;
                    if (j <= 3) c3 = c4;
                }
            }
            // carry on: the run's local list (mf entries) followed by the remainder
            const uint32_t l0 = ea[t].x, l1 = ea[t].y, l2 = ea[t].z, l3 = ea[t].w, l4 = eb[t].x;
            uint32_t d0, d1, d2, d3, d4;
            switch (mf) {
                case 0: d0 = c0; d1 = c1; d2 = c2; d3 = c3; d4 = c4; break;
                case 1: d0 = l0; d1 = c0; d2 = c1; d3 = c2; d4 = c3; break;
                case 2: d0 = l0; d1 = l1; d2 = c0; d3 = c1; d4 = c2; break;
                case 3: d0 = l0; d1 = l1; d2 = l2; d3 = c0; d4 = c1; break;
                case 4: d0 = l0; d1 = l1; d2 = l2; d3 = l3; d4 = c0; break;
                default: d0 = l0; d1 = l1; d2 = l2; d3 = l3; d4 = l4; break;
            }
            c0 = d0; c1 = d1; c2 = d2; c3 = d3; c4 = d4;
        }
    }
}

// ---- Lion sizes / emit ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t lion_block_bytes(uint64_t b, uint64_t nbytes, uint32_t pany, uint32_t am, uint32_t bm, bool copied) {
    const uint64_t boff = b * 64;
    const uint32_t blen = (uint32_t)((nbytes - boff < 64) ? (nbytes - boff) : 64);
    if (copied) return blen;
    const uint32_t sh = (uint32_t)(b & 1) * 16;
    const uint32_t nq = blen >> 2;
    const uint32_t act = (1u << nq) - 1u;
    const uint32_t maps = ((am | bm) >> sh) & act;
    const uint32_t plain = act & ~((pany | am | bm) >> sh);
    return 6 + 4 * __popc(plain) + 2 * __popc(maps) + (blen & 3u);      // lion.rs:333-336: 6-byte signature
}

// one warp per tile of 256 blocks (8 per lane)
__global__ void lion_tile_sizes(const uint32_t* __restrict__ Pany, const uint32_t* __restrict__ Abits, const uint32_t* __restrict__ Bbits,
                                const uint8_t* __restrict__ copymap, uint64_t nbytes, uint64_t nblocks, uint32_t ntiles, int final_pass,
                                const Status* __restrict__ st, uint8_t* __restrict__ inc, uint32_t* __restrict__ tile_bytes) {
    if (!final_pass && !(st->nonquiet && !st->converged)) return;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t tile = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (tile >= ntiles) return;
    uint32_t sum = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint64_t b = (uint64_t)tile * (2 * TILE_B) + k * 32 + lane;
        if (b < nblocks) {
            const bool copied = copymap && copymap[b];
            const uint32_t sz = lion_block_bytes(b, nbytes, Pany[b >> 1], Abits[b >> 1], Bbits[b >> 1], copied);
            sum += sz;
            if (!final_pass && !copied) inc[b] = (nbytes - b * 64 >= 64) && sz >= 64;     // codec.rs:68
        }
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, d);
    if (lane == 0) tile_bytes[tile] = sum;
}

// one CTA (256 threads) per tile of 256 blocks; warp w handles steps w, w+8, ... (a step = two blocks, one per half warp)
__global__ void __launch_bounds__(256)
lion_emit(const uint32_t* __restrict__ in, uint64_t nbytes, uint64_t nblocks, const uint32_t* __restrict__ F0, const uint32_t* __restrict__ F1,
          const uint32_t* __restrict__ F2, const uint32_t* __restrict__ Pany, const uint32_t* __restrict__ Abits, const uint32_t* __restrict__ Bbits,
          const uint8_t* __restrict__ copymap, const Status* __restrict__ status, const uint32_t* __restrict__ tile_local,
          const uint64_t* __restrict__ group_off, uint32_t scan_group, uint8_t* __restrict__ out) {
    if (status->error || !status->converged) return;
    __shared__ uint32_t s_off[2 * TILE_B + 1];
    __shared__ uint32_t s_wsum[8];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tile = blockIdx.x;
    const uint64_t tile_off = group_off[tile / scan_group] + tile_local[tile];
    const uint64_t nquads = nbytes / 4;
    {
        const uint64_t b = (uint64_t)tile * (2 * TILE_B) + tid;
        uint32_t sz = 0;
        if (b < nblocks) sz = lion_block_bytes(b, nbytes, Pany[b >> 1], Abits[b >> 1], Bbits[b >> 1], copymap && copymap[b]);
        uint32_t incl = sz;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= (uint32_t)d) incl += u; }
        if (lane == 31) s_wsum[warp] = incl;
        s_off[tid + 1] = incl;
    }
    __syncthreads();
    if (warp > 0) { uint32_t add = 0; for (uint32_t w = 0; w < warp; ++w) add += s_wsum[w]; s_off[tid + 1] += add; }
    if (tid == 0) s_off[0] = 0;
    __syncthreads();
    const uint8_t* in_b = reinterpret_cast<const uint8_t*>(in);
    const uint32_t half = lane >> 4, hl = lane & 15;
    for (uint32_t sl = warp; sl < TILE_B; sl += 8) {
        const uint64_t s = (uint64_t)tile * TILE_B + sl;
        const uint64_t b = 2 * s + half;
        if (2 * s >= nblocks) break;
        const bool have = b < nblocks;
        const uint64_t boff = b * 64;
        const uint32_t blen = have ? (uint32_t)((nbytes - boff < 64) ? (nbytes - boff) : 64) : 0u;
        const uint32_t nq = blen >> 2;
        uint8_t* const bout = out + tile_off + s_off[have ? 2 * sl + half : 0];
        const uint32_t q = (hl < nq && boff / 4 + hl < nquads) ? in[boff / 4 + hl] : 0u;
        const bool copied = have && copymap && copymap[b];
        const uint32_t sh = half * 16;
        const uint32_t act = have && !copied ? ((1u << nq) - 1u) : 0u;
        const uint32_t f0 = (F0[s] >> sh) & act, f1 = (F1[s] >> sh) & act, f2 = (F2[s] >> sh) & act;
        const uint32_t maps = ((Abits[s] | Bbits[s]) >> sh) & act, bmask = (Bbits[s] >> sh) & act;
        const uint32_t plain = act & ~(f0 | f1 | f2 | maps);
        // my 3-bit flag: PREDICTED_A..E 1..5 from the planes, MAP_A 6, MAP_B 7 (lion.rs:18-25)
        uint32_t flag = ((f0 >> hl) & 1u) | (((f1 >> hl) & 1u) << 1) | (((f2 >> hl) & 1u) << 2);
        if ((maps >> hl) & 1u) flag = 6u | ((bmask >> hl) & 1u);
        // 48-bit signature of the block, LSB first (write_signature.rs:13-16), OR-reduced over the half warp
        unsigned long long sig = (hl < nq && !copied) ? ((unsigned long long)flag << (3 * hl)) : 0ull;
        uint32_t slo = (uint32_t)sig, shi = (uint32_t)(sig >> 32);
#pragma unroll
        for (int d = 8; d; d >>= 1) { slo |= __shfl_xor_sync(0xFFFFFFFFu, slo, d); shi |= __shfl_xor_sync(0xFFFFFFFFu, shi, d); }
        if (!have) continue;
        if (copied) {                                       // copy-mode block: raw bytes (codec.rs:36)
            if (hl < nq) { st_u16(bout + 4 * hl, q & 0xFFFFu); st_u16(bout + 4 * hl + 2, q >> 16); }
            if (hl < (blen & 3u)) bout[(blen & ~3u) + hl] = in_b[boff + (blen & ~3u) + hl];
            continue;
        }
        if (hl < 3) st_u16(bout + 2 * hl, (hl == 0 ? slo : hl == 1 ? (slo >> 16) : shi) & 0xFFFFu);
        if (hl < nq) {
            const uint32_t lt = (1u << hl) - 1u;
            uint8_t* p = bout + 6 + 4 * __popc(plain & lt) + 2 * __popc(maps & lt);
            if ((plain >> hl) & 1u) { st_u16(p, q & 0xFFFFu); st_u16(p + 2, q >> 16); }            // lion.rs:251-252
            else if ((maps >> hl) & 1u) st_u16(p, prod_hash(hash_prod(q)));                          // lion.rs:254-260
        }
        if (hl < (blen & 3u)) {                             // 1..3 raw tail bytes of the last block (codec.rs:58-61)
            uint8_t* p = bout + 6 + 4 * __popc(plain) + 2 * __popc(maps);
            p[hl] = in_b[boff + (blen & ~3u) + hl];
        }
    }
}

// hand the verdict to the caller; an unsettled copy map reports size 0 (the in-order kernel queued behind overwrites it on path 0)
__global__ void chee_finish(const Status* __restrict__ st, uint32_t* __restrict__ d_converged, uint64_t* __restrict__ d_out_size) {
    *d_converged = st->converged;
    if (!st->converged && d_out_size) *d_out_size = 0;
}
// open the gate of a stage of up to 8 rounds; a continuation stage inherits "already settled" from the stage before it
__global__ void chee_chain_gate(Status* __restrict__ st, const Status* __restrict__ prev) { st->nonquiet = 1; st->converged = prev ? prev->converged : 0u; }   // Cheetah always runs the copy-map iteration


// =====================================================================================================================================
// Sharded encode (one stream cut across GPUs / calls): what a shard tells the shards after it, as TRANSFERS per context / bucket.
// Every table is a stack of u32 planes of 65536 entries (word w of key i at [w * 65536 + i]); all-zero = the identity transfer.
//   P, Cheetah (2 planes)  {touched, last quad}: pred[ctx] always ends as the last quad seen in the context, so the fold overwrites.
//   P, Lion (12 planes)    {m, nu, l0..l4, v0..v4}: the shard leaves its m local values l in front of what is left of the carried-in
//                          list; its nu undecided accesses (values v, the k-th made with k local entries in front) each remove one
//                          matching carried entry, as lion_fold_p replays them. A concrete list is {5, 0, list, -}.
//   C, both (3 planes)     {T, a, b}: T0 untouched, T1 v = the bucket was accessed with one value v, T2 = it ends as (a, b).
// compose(x, y) = "x, then y" keeps each form closed; the stream-start states (cl_table_init) are concrete, and a left fold of shard
// transfers over them gives the concrete state the in-order encoder has at the cut.
// =====================================================================================================================================
constexpr uint32_t PL = 65536;

struct LionT { uint32_t m, nu, l[5], v[5]; };
__device__ __forceinline__ void lion_t_load(const uint32_t* __restrict__ t, uint32_t i, LionT& x) {
    x.m = t[i]; x.nu = t[PL + i];
#pragma unroll
    for (int s = 0; s < 5; ++s) { x.l[s] = t[(2 + s) * PL + i]; x.v[s] = t[(7 + s) * PL + i]; }
}
__device__ __forceinline__ void lion_t_store(uint32_t* __restrict__ t, uint32_t i, const LionT& x) {
    t[i] = x.m; t[PL + i] = x.nu;
#pragma unroll
    for (int s = 0; s < 5; ++s) { t[(2 + s) * PL + i] = x.l[s]; t[(7 + s) * PL + i] = x.v[s]; }
}
// x <- x then y. y's k-th undecided access sees the first 5 - k entries of what x leaves: x's literals first (a match there decides it
// and removes the literal), then x's unknown carried-in remainder (no literal match while that remainder is visible: the access stays
// undecided in the composition)
__device__ __forceinline__ void lion_t_compose(LionT& x, const LionT& y) {
    uint32_t lit[5], nl = x.m, nu = x.nu;
#pragma unroll
    for (int s = 0; s < 5; ++s) lit[s] = x.l[s];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        if ((uint32_t)k >= y.nu) break;
        const uint32_t vis = 5 - k, lim = nl < vis ? nl : vis;
        uint32_t j = 5;
#pragma unroll
        for (int s = 4; s >= 0; --s) if ((uint32_t)s < lim && lit[s] == y.v[k]) j = s;
        if (j < 5) {
#pragma unroll
            for (int s = 0; s < 4; ++s) if ((uint32_t)s >= j) lit[s] = lit[s + 1];
            --nl;
        } else if (nl < vis && nu < 5) {
#pragma unroll
            for (int s = 0; s < 5; ++s) if ((uint32_t)s == nu) x.v[s] = y.v[k];
            ++nu;
        }
    }
    const uint32_t keep = nl < 5 - y.m ? nl : 5 - y.m;
#pragma unroll
    for (int s = 0; s < 5; ++s) {
        uint32_t w = 0;
#pragma unroll
        for (int t = 0; t < 5; ++t) if ((uint32_t)s >= y.m && (uint32_t)(s - t) == y.m && (uint32_t)t < keep) w = lit[t];
        x.l[s] = (uint32_t)s < y.m ? y.l[s] : w;
    }
    x.m = y.m + keep; x.nu = nu;
}
__device__ __forceinline__ void chunk_t_compose(uint32_t& T, uint32_t& a, uint32_t& b, uint32_t T2, uint32_t a2, uint32_t b2) {
    if (T2 == 0) return;
    if (T2 == 2) { T = 2; a = a2; b = b2; return; }
    if (T == 0) { T = 1; a = a2; }                                     // T1 v after nothing
    else if (a2 != a) { b = a; a = a2; T = 2; }                        // T1 v after T1 w (v != w) or over (a, b) (v != a): (v, a)
}

// the shard's transfer, composed over its runs in order (the run tables of the round whose tag is *epoch_p). `gate` (may be nullptr =
// always): the copy-map rounds of density_b200_cl_shard_prot_* skip the exports once the map has settled, nobody reads them then.
__global__ void cl_export_p_chee(const uint4* __restrict__ entP_all, uint32_t nruns, const Status* __restrict__ gate, const uint32_t* __restrict__ epoch_p,
                                 uint32_t* __restrict__ out) {
    if (gate && !(gate->nonquiet && !gate->converged)) return;
    const uint32_t ctx = blockIdx.x * blockDim.x + threadIdx.x;
    if (ctx >= PL) return;
    const uint32_t epoch = *epoch_p;
    uint32_t touched = 0, q = 0;
    for (uint32_t r = 0; r < nruns; ++r) {
        const uint4 e = entP_all[(size_t)r * PL + ctx];
        if (e.y == epoch) { touched = 1; q = e.x; }
    }
    out[ctx] = touched; out[PL + ctx] = q;
}
__global__ void cl_export_p_lion(const uint32_t* __restrict__ in, const uint4* __restrict__ hot_all, const uint32_t* __restrict__ cold_all,
                                 uint32_t nruns, const Status* __restrict__ gate, const uint32_t* __restrict__ epoch_p, uint32_t* __restrict__ out) {
    if (gate && !(gate->nonquiet && !gate->converged)) return;
    const uint32_t ctx = blockIdx.x * blockDim.x + threadIdx.x;
    if (ctx >= PL) return;
    const uint32_t epoch = *epoch_p;
    LionT x = {};
    for (uint32_t r = 0; r < nruns; ++r) {
        const size_t i = (size_t)r * PL + ctx;
        const uint4 e1 = hot_all[2 * i + 1];
        if ((e1.y >> 3) != epoch) continue;
        const uint4 e0 = hot_all[2 * i];
        LionT y;
        y.m = y.nu = e1.y & 7u;
        y.l[0] = e0.x; y.l[1] = e0.y; y.l[2] = e0.z; y.l[3] = e0.w; y.l[4] = e1.x;
#pragma unroll
        for (int k = 0; k < 5; ++k) y.v[k] = (uint32_t)k < y.nu ? in[cold_all[i * 8 + k] - 1] : 0u;
        lion_t_compose(x, y);
    }
    lion_t_store(out, ctx, x);
}
__global__ void cl_export_c(const uint4* __restrict__ entC_all, uint32_t nruns, const Status* __restrict__ gate, const uint32_t* __restrict__ epoch_p,
                            uint32_t* __restrict__ out) {
    if (gate && !(gate->nonquiet && !gate->converged)) return;
    const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= PL) return;
    const uint32_t epoch = *epoch_p;
    uint32_t T = 0, a = 0, b = 0;
    for (uint32_t r = 0; r < nruns; ++r) {
        const uint4 e = entC_all[(size_t)r * PL + h];
        if ((e.y >> 2) == epoch) chunk_t_compose(T, a, b, e.y & 3u, e.x & 0xFFFFu, e.x >> 16);
    }
    out[h] = T; out[PL + h] = a; out[2 * PL + h] = b;
}

// kind 0 = P, 1 = C. The stream-start states: pred 0 everywhere; Lion lists of five zeros; chunk map (0, 0) in bucket 0, else nothing.
__device__ __forceinline__ void cl_t_init(int alg, int kind, uint32_t* __restrict__ t, uint32_t i) {
    if (kind == 1) { t[i] = 2; t[PL + i] = i ? FP_INVALID : 0u; t[2 * PL + i] = i ? FP_INVALID : 0u; }
    else if (alg == ALG_LION) { LionT x = {}; x.m = 5; lion_t_store(t, i, x); }
    else { t[i] = 1; t[PL + i] = 0; }
}
// acc[i] <- acc[i] then next[i]
__device__ __forceinline__ void cl_t_fold(int alg, int kind, uint32_t* __restrict__ acc, const uint32_t* __restrict__ next, uint32_t i) {
    if (kind == 1) {
        uint32_t T = acc[i], a = acc[PL + i], b = acc[2 * PL + i];
        chunk_t_compose(T, a, b, next[i], next[PL + i], next[2 * PL + i]);
        acc[i] = T; acc[PL + i] = a; acc[2 * PL + i] = b;
    } else if (alg == ALG_LION) {
        LionT x, y; lion_t_load(acc, i, x); lion_t_load(next, i, y);
        lion_t_compose(x, y);
        lion_t_store(acc, i, x);
    } else if (next[i]) {
        acc[i] = 1; acc[PL + i] = next[PL + i];
    }
}
__global__ void cl_table_init_k(int alg, int kind, uint32_t* __restrict__ t) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < PL) cl_t_init(alg, kind, t, i);
}
__global__ void cl_table_fold_k(int alg, int kind, uint32_t* __restrict__ acc, const uint32_t* __restrict__ next) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < PL) cl_t_fold(alg, kind, acc, next, i);
}
// carry-in of shard `rank` = the stream-start state, then the transfers of shards 0 .. rank - 1 (`tables` = [world][planes][65536])
__global__ void cl_rank_fold_k(int alg, int kind, const uint32_t* __restrict__ tables, uint32_t planes, uint32_t rank, uint32_t* __restrict__ carry) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= PL) return;
    cl_t_init(alg, kind, carry, i);
    for (uint32_t r = 0; r < rank; ++r) cl_t_fold(alg, kind, carry, tables + (size_t)r * planes * PL, i);
}
// the context of a shard's first quad comes from the last quad of the nearest earlier shard that has one (words: [world][stride], {has,
// quad} at the front of every row)
__global__ void cl_prev_quad_k(const uint32_t* __restrict__ words, uint32_t stride, uint32_t rank, uint32_t* __restrict__ out) {
    uint32_t q = 0;
    for (uint32_t r = 0; r < rank; ++r) if (words[stride * r]) q = words[stride * r + 1];
    *out = q;
}
__global__ void cl_last_quad_k(const uint32_t* __restrict__ in, uint64_t nquads, uint32_t* __restrict__ out) {
    out[0] = nquads ? 1u : 0u; out[1] = nquads ? in[nquads - 1] : 0u;
}

// shard gates: the passes of a later shard run under `gate` (open); emit runs under `emit`, settled when the copy-map iteration of the
// first shard settled (later shards have no copy map). A later shard's round uses `own_epoch`; the first shard's iteration has left
// the epoch of its settled round in *epoch_word already.
__global__ void cl_shard_gates(Status* __restrict__ gate, Status* __restrict__ emit, const Status* __restrict__ iter, uint32_t* __restrict__ pair_flag,
                               uint32_t* __restrict__ epoch_word, uint32_t own_epoch) {
    gate->nonquiet = 1; gate->converged = 0; gate->error = 0;
    if (!iter) *epoch_word = own_epoch;
    emit->nonquiet = 0; emit->error = 0; emit->out_bytes = 0; emit->converged = iter ? iter->converged : 1u;
    *pair_flag = 0;
}
// later shards: two consecutive incompressible blocks would start copy mode (protection_state.rs:38-43)
__global__ void cl_inc_pairs(const uint8_t* __restrict__ inc, uint64_t nblocks, uint32_t* __restrict__ flag) {
    for (uint64_t b = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; b + 1 < nblocks; b += (uint64_t)gridDim.x * blockDim.x)
        if (inc[b] && inc[b + 1]) *flag = 1;
}
// the shard's 8 seam words in the layout of the Chameleon encoder's: {first block incompressible, previous_incompressible at the end,
// refused, has blocks, size lo, size hi, 0, 0}. The first shard of a longer stream is refused when it ends inside a copy run or with a
// copy penalty pending (its last block incompressible after an incompressible or copied block)
__global__ void cl_seam_words_k(const uint8_t* __restrict__ inc, const uint8_t* __restrict__ copymap, uint64_t nblocks, int first, int is_last,
                                const Status* __restrict__ emit, const uint32_t* __restrict__ pair_flag, const uint64_t* __restrict__ d_out_size,
                                uint32_t* __restrict__ words) {
    const uint64_t lb = nblocks - 1;
    auto cp = [&](uint64_t b) { return copymap && copymap[b]; };
    uint32_t bad = (emit->error || !emit->converged || (pair_flag && *pair_flag)) ? 1u : 0u;
    if (first && !is_last && (cp(lb) || (inc[lb] && lb > 0 && (cp(lb - 1) || inc[lb - 1])))) bad = 1;
    words[0] = (!cp(0) && inc[0]) ? 1u : 0u;
    words[1] = (cp(lb) || inc[lb]) ? 1u : 0u;
    words[2] = bad; words[3] = 1;
    const uint64_t sz = *d_out_size;
    words[4] = (uint32_t)sz; words[5] = (uint32_t)(sz >> 32); words[6] = 0; words[7] = 0;
}

// ---- copy mode on every shard (density_b200_cl_shard_prot_*) ---------------------------------------------------------------------------
// words 4-7 of a shard's round words: {has an encoded quad, the last one, 0, 0} under `cm` (the map the next round uses). With `gate`
// closed the map has settled, and the record keeps what the round that settled it found. One CTA of 256 threads walks back from the last
// block; the automaton encodes a block at least every 256 blocks, so it stops within the first chunks.
__global__ void __launch_bounds__(256)
cl_prot_quad_k(const uint32_t* __restrict__ in, uint64_t nquads, uint64_t nblocks, uint32_t block_quads, const uint8_t* __restrict__ cm,
               const Status* __restrict__ gate, ProtShard* __restrict__ ps, uint32_t* __restrict__ words) {
    __shared__ unsigned long long s_best;               // 1 + the last encoded block that has a quad
    if (!gate || (gate->nonquiet && !gate->converged)) {
        if (threadIdx.x == 0) s_best = 0;
        __syncthreads();
        for (uint64_t base = 0; base < nblocks; base += blockDim.x) {
            bool found = false;
            if (base + threadIdx.x < nblocks) {
                const uint64_t b = nblocks - 1 - base - threadIdx.x;
                found = !cm[b] && b * block_quads < nquads;
                if (found) atomicMax(&s_best, (unsigned long long)b + 1);
            }
            if (__syncthreads_or(found)) break;
        }
        if (threadIdx.x == 0) {
            const uint64_t b = s_best;
            uint64_t qi = b ? b * block_quads - 1 : 0;       // the block's last quad (the stream's last, in a short last block)
            if (qi >= nquads) qi = nquads - 1;
            ps->has_quad = b ? 1u : 0u;
            ps->last_quad = b ? in[qi] : 0u;
        }
    }
    if (threadIdx.x == 0) { words[4] = ps->has_quad; words[5] = ps->last_quad; words[6] = 0; words[7] = 0; }
}
// phase 1 of the shard at the stream start: its staged iteration settled or not
__global__ void cl_prot_stage_k(const Status* __restrict__ iter, ProtShard* __restrict__ ps) { ps->stage_ok = iter->converged ? 1u : 0u; }

}  // namespace chee

using namespace chee;

int g_chee_stage_rounds = 7;   // rounds per stage of the copy-map iteration (7 = all; tests lower it, see density_b200_test_set_stage_rounds)

struct CheeLayout {
    size_t status, Pbits, Abits, Bbits, F0, F1, F2, copymap, copymap2, incb, seg_state, ctx0, tile_bytes, tile_local, group_total, group_off, total;
};

constexpr uint32_t PREFIX_TILES = 64;           // stage A settles the copy map of the first MiB on its own (cold-dictionary blocks)

static uint32_t chee_pick_runs(size_t nbytes, int num_sms) {
    const uint64_t nsteps = (nbytes + 127) / 128;
    const uint64_t ntiles = (nsteps + TILE_B - 1) / TILE_B;
    uint64_t r = ntiles / 2;                    // >= 32 KiB per run
    static const int per_sm = [] { const char* v = getenv("DENSITY_B200_RUNS_PER_SM"); int k = v ? atoi(v) : 0; return (k >= 1 && k <= 64) ? k : 8; }();
    const uint64_t cap = (uint64_t)num_sms * per_sm; // warps (runs) per SM: 8 by default (tuning knob; the result does not depend on it)
    if (r > cap) r = cap;
    if (r < PREFIX_TILES && ntiles >= PREFIX_TILES) r = PREFIX_TILES;
    if (r < 1) r = 1;
    return (uint32_t)r;
}

static size_t chee_layout(size_t nbytes, uint32_t nruns, CheeLayout* L) {
    const uint64_t nsteps = (nbytes + 127) / 128;
    const uint64_t ntiles = (nsteps + TILE_B - 1) / TILE_B;
    const uint64_t ngroups = (ntiles + 4095) / 4096;
    const uint64_t maxblocks = ntiles * TILE_B * 2;          // Lion: two 64-byte blocks per step
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
    L->status = take(4 * sizeof(Status));          // one per stage of the copy-map iteration (8 rounds each)
    L->Pbits = take((ntiles * TILE_B + 32) * 4);
    L->Abits = take((ntiles * TILE_B + 32) * 4);
    L->Bbits = take((ntiles * TILE_B + 32) * 4);
    L->F0 = take((ntiles * TILE_B + 32) * 4);
    L->F1 = take((ntiles * TILE_B + 32) * 4);
    L->F2 = take((ntiles * TILE_B + 32) * 4);
    L->copymap = take(maxblocks + 64);
    L->copymap2 = take(maxblocks + 64);
    L->incb = take(maxblocks + 64);
    L->seg_state = take(prot_state_bytes(maxblocks / 256 + 2));
    L->ctx0 = take((size_t)nruns * 4 + 64);
    L->tile_bytes = take((ntiles + 1) * 4);
    L->tile_local = take((ntiles + 1) * 4);
    L->group_total = take((ngroups + 1) * 8);
    L->group_off = take((ngroups + 1) * 8);
    L->total = off;
    return off;
}

size_t chee_workspace_bytes(size_t nbytes, int num_sms) {
    CheeLayout L;
    return chee_layout(nbytes, chee_pick_runs(nbytes, num_sms), &L);
}
// The per-run tables live in a buffer of their own: it must be zero when allocated and only ever be written by these kernels
// (entries are validated by epoch tags instead of being cleared). Cheetah: 16 + 16 B per run and context/bucket; Lion: 32 + 32 + 16 B.
// Three separately allocated regions, each with ONE entry format for its whole life, so that a stale word can never alias a tag:
// 0 = pass-P entries, 1 = Lion's undecided-access indices (untagged), 2 = pass-C entries.
size_t chee_tables_bytes(int alg, int region, size_t nbytes, int num_sms) {
    const size_t per = region == 0 ? (alg == ALG_LION ? 32 : 16) : region == 1 ? (alg == ALG_LION ? 32 : 0) : 16;
    return (size_t)chee_pick_runs(nbytes, num_sms) * 65536 * per;
}

// One encode over `n` bytes cut into `nruns` runs, as every launch below sees it: the geometry, and typed pointers into the workspace
// (chee_layout) and the three run-table regions. The last four pointers exist only behind a shard's workspace
// (cl_shard_workspace_bytes): its gate, its emit gate, its pair flag, the epoch of the round it exports and the quad before it.
struct CheeView {
    bool lion; const uint32_t* in32; size_t n; uint32_t bbytes, nruns, ntiles, ngroups, run_ctas, nseg; uint64_t nq, nstep, nblk;
    Status* stages; size_t stages_bytes; uint32_t *Pb, *Ab, *Bb, *F0, *F1, *F2; uint8_t *cm, *cm2, *incb; uint32_t *seg, *ctx0, *tile_bytes, *tile_local;
    uint64_t *group_total, *group_off; uint4* entP; uint32_t* coldP; uint4* entC;
    Status *gate, *emit; uint32_t *pair_flag, *epoch_word, *prev_quad;
    CheeView(int alg, const uint8_t* d_in, size_t nbytes, int num_sms, uint8_t* ws, uint8_t* const tables[3]) {
        lion = alg == ALG_LION; bbytes = lion ? 64 : 128; in32 = reinterpret_cast<const uint32_t*>(d_in);
        cut(nbytes, chee_pick_runs(nbytes, num_sms));
        CheeLayout L; chee_layout(nbytes, nruns, &L);
        stages = reinterpret_cast<Status*>(ws + L.status); stages_bytes = L.Pbits - L.status;
        Pb = reinterpret_cast<uint32_t*>(ws + L.Pbits); Ab = reinterpret_cast<uint32_t*>(ws + L.Abits); Bb = reinterpret_cast<uint32_t*>(ws + L.Bbits);
        F0 = reinterpret_cast<uint32_t*>(ws + L.F0); F1 = reinterpret_cast<uint32_t*>(ws + L.F1); F2 = reinterpret_cast<uint32_t*>(ws + L.F2);
        cm = ws + L.copymap; cm2 = ws + L.copymap2; incb = ws + L.incb;
        seg = reinterpret_cast<uint32_t*>(ws + L.seg_state);
        ctx0 = reinterpret_cast<uint32_t*>(ws + L.ctx0);
        tile_bytes = reinterpret_cast<uint32_t*>(ws + L.tile_bytes); tile_local = reinterpret_cast<uint32_t*>(ws + L.tile_local);
        group_total = reinterpret_cast<uint64_t*>(ws + L.group_total); group_off = reinterpret_cast<uint64_t*>(ws + L.group_off);
        entP = reinterpret_cast<uint4*>(tables[0]); coldP = reinterpret_cast<uint32_t*>(tables[1]); entC = reinterpret_cast<uint4*>(tables[2]);
        gate = reinterpret_cast<Status*>(ws + ((L.total + 255) & ~(size_t)255)); emit = gate + 1; pair_flag = reinterpret_cast<uint32_t*>(emit + 1);
        epoch_word = pair_flag + 1; prev_quad = epoch_word + 1;
    }
    // the same buffers for the first `nbytes` of the input cut into `runs` runs (the prefix stages of chee_iterate)
    CheeView prefix(size_t nbytes, uint32_t runs) const { CheeView v = *this; v.cut(nbytes, runs); return v; }
private:
    void cut(size_t nbytes, uint32_t runs) {
        n = nbytes; nruns = runs; nq = n / 4; nstep = (n + 127) / 128; nblk = (n + bbytes - 1) / bbytes;
        ntiles = (uint32_t)((nstep + TILE_B - 1) / TILE_B); ngroups = (ntiles + 4095) / 4096; run_ctas = (nruns + RP_WARPS - 1) / RP_WARPS;
        nseg = (uint32_t)((nblk + 255) / 256);
    }
};

// ---- the steps of one round, each the only place where Cheetah and Lion part for that step. `mask`: the copy map in force (nullptr =
// none), `gate`: the Status block the kernels run under; the carried-in tables are stacks of planes as cl_table_init / cl_rank_fold
// leave them (nullptr = stream start), of which the fold kernels take the state planes.
static void launch_ctx0_pass_p(const CheeView& V, const uint8_t* mask, Status* gate, const uint32_t* d_prev_quad, uint32_t epoch, uint32_t* d_epoch_out,
                               cudaStream_t stream, uint64_t* launches) {
    if (V.lion) {
        lion_ctx0<<<(V.nruns + 127) / 128, 128, 0, stream>>>(V.in32, V.nq, mask, V.nruns, V.ntiles, gate, d_prev_quad, epoch, d_epoch_out, V.ctx0);
        lion_pass_p<<<V.run_ctas, RP_WARPS * 32, 0, stream>>>(V.in32, V.nq, V.nstep, V.nblk, mask, V.nruns, V.ntiles, gate, V.ctx0, V.entP, V.coldP, epoch,
                                                              V.F0, V.F1, V.F2, V.Pb);
    } else {
        chee_ctx0<<<(V.nruns + 127) / 128, 128, 0, stream>>>(V.in32, V.nq, mask, V.nruns, V.ntiles, gate, d_prev_quad, epoch, d_epoch_out, V.ctx0);
        chee_pass_p<<<V.run_ctas, RP_WARPS * 32, 0, stream>>>(V.in32, V.nq, V.nstep, mask, V.nruns, V.ntiles, gate, V.ctx0, V.entP, epoch, V.Pb);
    }
    *launches += 2;
}
static void launch_fold_p_pass_c(const CheeView& V, const uint8_t* mask, Status* gate, uint32_t epoch, const uint32_t* d_carry_p, cudaStream_t stream,
                                 uint64_t* launches) {
    if (V.lion) {
        lion_fold_p<<<PL / 128, 128, 0, stream>>>(V.in32, V.nruns, gate, V.entP, V.coldP, epoch, d_carry_p ? d_carry_p + 2 * PL : nullptr, V.F0, V.F1, V.F2, V.Pb);
        chee_pass_c<2><<<V.run_ctas, RP_WARPS * 32, 0, stream>>>(V.in32, V.nq, V.nstep, V.nblk, mask, V.nruns, V.ntiles, gate, V.Pb, V.entC, epoch, V.Ab, V.Bb);
    } else {
        chee_fold_p<<<PL / 128, 128, 0, stream>>>(V.in32, V.nruns, gate, V.entP, epoch, d_carry_p ? d_carry_p + PL : nullptr, V.Pb);
        chee_pass_c<1><<<V.run_ctas, RP_WARPS * 32, 0, stream>>>(V.in32, V.nq, V.nstep, V.nblk, mask, V.nruns, V.ntiles, gate, V.Pb, V.entC, epoch, V.Ab, V.Bb);
    }
    *launches += 2;
}
static void launch_fold_c(const CheeView& V, Status* gate, uint32_t epoch, const uint32_t* d_carry_c, cudaStream_t stream, uint64_t* launches) {
    chee_fold_c<<<PL / 128, 128, 0, stream>>>(V.in32, V.nruns, gate, V.entC, epoch, d_carry_c ? d_carry_c + PL : nullptr, V.Ab, V.Bb);
    ++*launches;
}
// tile sizes and incompressible bits; final_pass: the sizes under a committed map, valid only if `gate` has converged
static void launch_tile_sizes(const CheeView& V, const uint8_t* mask, int final_pass, Status* gate, cudaStream_t stream, uint64_t* launches) {
    if (V.lion) lion_tile_sizes<<<(V.ntiles + 7) / 8, 256, 0, stream>>>(V.Pb, V.Ab, V.Bb, mask, V.n, V.nblk, V.ntiles, final_pass, gate, V.incb, V.tile_bytes);
    else chee_tile_sizes<<<(V.ntiles + 7) / 8, 256, 0, stream>>>(V.Pb, V.Ab, V.Bb, mask, V.n, V.nblk, V.ntiles, final_pass, gate, V.incb, V.tile_bytes);
    ++*launches;
}
// tile offsets from the tile sizes (and the stream's size, checked against `cap`), then emit; ev_emit (may be nullptr) is recorded between
static cudaError_t launch_scan_emit(const CheeView& V, const uint8_t* mask, Status* gate, size_t cap, uint64_t* d_out_size, uint8_t* d_out,
                                    cudaStream_t stream, uint64_t* launches, cudaEvent_t ev_emit = nullptr) {
    cudaError_t e = scan_tiles_launch(V.tile_bytes, V.ntiles, V.tile_local, V.group_total, V.group_off, V.ngroups, gate, cap, d_out_size, stream);
    if (e == cudaSuccess && ev_emit) e = cudaEventRecord(ev_emit, stream);
    if (e != cudaSuccess) return e;
    if (V.lion) lion_emit<<<V.ntiles, 256, 0, stream>>>(V.in32, V.n, V.nblk, V.F0, V.F1, V.F2, V.Pb, V.Ab, V.Bb, mask, gate, V.tile_local, V.group_off, 4096, d_out);
    else chee_emit<<<V.ntiles, 256, 0, stream>>>(V.in32, V.n, V.nblk, V.Pb, V.Ab, V.Bb, mask, gate, V.tile_local, V.group_off, 4096, d_out);
    *launches += 3;
    return cudaSuccess;
}

// The staged copy-map iteration (epochs epoch_base .. epoch_base + 31). *st_out = the Status block of the last stage: converged != 0
// means the committed copy map (cm) and the flags and run tables of the last round that ran are final; *d_epoch_out (device, may be
// nullptr) receives that round's epoch.
static cudaError_t chee_iterate(const CheeView& V, uint32_t epoch_base, int num_sms, bool resume, uint32_t* d_epoch_out, cudaStream_t stream,
                                uint64_t* launches, Status** st_out) {
    cudaError_t e = cudaMemsetAsync(V.stages, 0, V.stages_bytes, stream);     // every stage's status block
    if (e != cudaSuccess) return e;

    // one fixed-point round over R (the input or a prefix of it): flags under the current map, incompressible bits, automaton
    auto round = [&](const CheeView& R, Status* st, int it, uint32_t epoch) -> cudaError_t {
        const uint8_t* mask = it ? R.cm : nullptr;
        launch_ctx0_pass_p(R, mask, st, nullptr, epoch, d_epoch_out, stream, launches);
        launch_fold_p_pass_c(R, mask, st, epoch, nullptr, stream, launches);
        launch_fold_c(R, st, epoch, nullptr, stream, launches);
        launch_tile_sizes(R, mask, 0, st, stream, launches);
        ++*launches;
        return prot_iterate_launch(nullptr, R.n, R.nblk, R.nseg, st, it, R.incb, R.cm, R.cm2, R.seg, R.seg + (R.nseg + 1), num_sms, stream);
    };

    // A stage = up to 8 rounds on one Status block (prot_iterate owns 8 grid-barrier slots per block).
    // test hook (density_b200_test_set_stage_rounds): cut every stage to rounds first..k so that the resume path can be exercised
    const int last_it = g_chee_stage_rounds;
    auto stage = [&](const CheeView& R, Status* st, const Status* inherit, int first_it, uint32_t ep0) -> cudaError_t {
        chee_chain_gate<<<1, 1, 0, stream>>>(st, inherit); ++*launches;
        for (int it = first_it; it <= last_it; ++it) {
            cudaError_t err = round(R, st, it, ep0 + (uint32_t)it);
            if (err != cudaSuccess) return err;
        }
        return cudaSuccess;
    };
    Status* const stages = V.stages;
    Status* st;
    if (V.ntiles > 2 * PREFIX_TILES) {
        // Stages A1, A2: a cold dictionary makes the first blocks incompressible on every input, and settling that takes 4-10 rounds
        // (copied blocks perturb the sizes of their near-threshold neighbours): run them on the first MiB alone (the copy map of a
        // prefix does not depend on what follows). Stages B1, B2 then start from that map and normally confirm it in one round
        // over the whole input.
        const CheeView A = V.prefix((size_t)PREFIX_TILES * TILE_B * 128, PREFIX_TILES);
        if (!resume) {
            e = cudaMemsetAsync(V.cm, 0, (size_t)V.ntiles * TILE_B * 2, stream);
            if (e != cudaSuccess) return e;
            e = stage(A, &stages[0], nullptr, 0, epoch_base);
            if (e == cudaSuccess) e = stage(A, &stages[1], &stages[0], 1, epoch_base + 8);
        }
        if (e == cudaSuccess) e = stage(V, &stages[2], nullptr, 1, epoch_base + 16);
        if (e == cudaSuccess) e = stage(V, &stages[3], &stages[2], 1, epoch_base + 24);
        st = &stages[3];
    } else {
        e = stage(V, &stages[0], nullptr, resume ? 1 : 0, epoch_base);
        if (e == cudaSuccess) e = stage(V, &stages[1], &stages[0], 1, epoch_base + 8);
        st = &stages[1];
    }
    *st_out = st;
    return e;
}

// Enqueue the parallel Cheetah / Lion encode. *d_converged (device u32) != 0 afterwards means d_out / d_out_size hold the result;
// otherwise the caller's in-order kernel (queued behind, gated on that flag) produces it. `epoch_base`: the caller hands out 32 fresh
// epochs (values in 1 .. 2^28) per call and clears `tables` if it ever has to reuse one.
// `resume`: continue an iteration that a previous call on the same input and workspace left unsettled (callers that may block read
// *d_converged and call again): the stages on the prefix are skipped and the whole-input stages start from the last committed map.
cudaError_t chee_encode_parallel(int alg, const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws, uint8_t* const tables[3],
                                 uint32_t epoch_base, int num_sms, uint64_t* d_out_size, uint32_t* d_converged, bool resume,
                                 cudaStream_t stream, uint64_t* launches) {
    const CheeView V(alg, d_in, nbytes, num_sms, ws, tables);
    Status* st = nullptr;
    cudaError_t e = chee_iterate(V, epoch_base, num_sms, resume, nullptr, stream, launches, &st);
    if (e != cudaSuccess) return e;
    // final sizes under the committed copy map (valid only if converged), scan, emit
    launch_tile_sizes(V, V.cm, 1, st, stream, launches);
    e = launch_scan_emit(V, V.cm, st, cap, d_out_size, d_out, stream, launches);
    if (e != cudaSuccess) return e;
    chee_finish<<<1, 1, 0, stream>>>(st, d_converged, d_out_size);
    ++*launches;
    return cudaGetLastError();
}

// ---- sharded encode: one shard of a longer stream, in three phases around the two table exchanges ----------------------------------
// The shard's workspace = chee_layout of its length, then the shard's own status area (gate, emit gate, pair flag, the epoch of the
// round the shard exports). Every call takes CL_SHARD_EPOCHS fresh epochs: the first 32 for the copy-map iteration of the first shard,
// epoch_base + 32 for the one round of a later shard, which all three phases share.
//
// The first shard has no carry-in: when its iteration has settled, the flags and run tables of its settled round are final, so it
// only exports them (the epoch comes from ctx0, on the device) and, in phase 3, sizes, scans and emits under the committed map as
// chee_encode_parallel does. A later shard runs ctx0 and pass P, fold P and pass C, fold C, without a copy map.
constexpr uint32_t CL_SHARD_EPOCHS = 40;
uint32_t cl_shard_epochs() { return CL_SHARD_EPOCHS; }
uint32_t cl_table_planes(int alg, int kind) { return kind == 1 ? 3u : alg == ALG_LION ? 12u : 2u; }
size_t cl_shard_workspace_bytes(size_t nbytes, int num_sms) { return ((chee_workspace_bytes(nbytes, num_sms) + 255) & ~(size_t)255) + 1024; }

// Phase 1: the first shard (a.first) runs the copy-map iteration to the end; a later shard runs ctx0 and pass P. Both
// export their P transfer.
cudaError_t cl_shard_phase1(const ClShardArgs& a, const uint32_t* d_prev_quad, uint32_t* d_tab_p, cudaStream_t stream, uint64_t* launches) {
    const CheeView V(a.alg, a.d_in, a.n, a.num_sms, a.ws, a.tables);
    const uint32_t ep = a.epoch_base + 32;
    Status* iter = nullptr;
    cudaError_t e = cudaSuccess;
    if (a.first) e = chee_iterate(V, a.epoch_base, a.num_sms, false, V.epoch_word, stream, launches, &iter);
    if (e != cudaSuccess) return e;
    cl_shard_gates<<<1, 1, 0, stream>>>(V.gate, V.emit, iter, V.pair_flag, V.epoch_word, ep);
    ++*launches;
    if (!a.first) launch_ctx0_pass_p(V, nullptr, V.gate, d_prev_quad, ep, nullptr, stream, launches);
    if (V.lion) cl_export_p_lion<<<PL / 128, 128, 0, stream>>>(V.in32, V.entP, V.coldP, V.nruns, nullptr, V.epoch_word, d_tab_p);
    else cl_export_p_chee<<<PL / 128, 128, 0, stream>>>(V.entP, V.nruns, nullptr, V.epoch_word, d_tab_p);
    ++*launches;
    return cudaGetLastError();
}

// Phase 2: a later shard makes its predictions final from the carried-in P state (planes as cl_table_init / cl_rank_fold leave them;
// nullptr = stream start) and runs pass C; every shard exports its C transfer. The first shard ignores d_carry_p (its state is the
// stream start, and its flags are final already).
cudaError_t cl_shard_phase2(const ClShardArgs& a, const uint32_t* d_carry_p, uint32_t* d_tab_c, cudaStream_t stream, uint64_t* launches) {
    const CheeView V(a.alg, a.d_in, a.n, a.num_sms, a.ws, a.tables);
    if (!a.first) launch_fold_p_pass_c(V, nullptr, V.gate, a.epoch_base + 32, d_carry_p, stream, launches);
    cl_export_c<<<PL / 128, 128, 0, stream>>>(V.entC, V.nruns, nullptr, V.epoch_word, d_tab_c);
    ++*launches;
    return cudaGetLastError();
}

// Phase 3: a later shard makes its chunk-map flags final from the carried-in C state (the first shard ignores d_carry_c); then sizes
// and incompressible bits, scan, emit, the shard's 8 seam words.
cudaError_t cl_shard_phase3(const ClShardArgs& a, const uint32_t* d_carry_c, uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint32_t* d_seam8,
                            cudaStream_t stream, uint64_t* launches) {
    const CheeView V(a.alg, a.d_in, a.n, a.num_sms, a.ws, a.tables);
    const bool first = a.first;
    const uint8_t* mask = first ? V.cm : nullptr;
    if (!first) launch_fold_c(V, V.gate, a.epoch_base + 32, d_carry_c, stream, launches);
    launch_tile_sizes(V, mask, 0, V.gate, stream, launches);
    if (!first) {
        const uint64_t want = (V.nblk + 255) / 256;
        const uint32_t grid = (uint32_t)(want < (uint64_t)a.num_sms * 8 ? (want ? want : 1) : (uint64_t)a.num_sms * 8);
        cl_inc_pairs<<<grid, 256, 0, stream>>>(V.incb, V.nblk, V.pair_flag);
        ++*launches;
    }
    cudaError_t e = launch_scan_emit(V, mask, V.emit, cap, d_out_size, d_out, stream, launches);
    if (e != cudaSuccess) return e;
    cl_seam_words_k<<<1, 1, 0, stream>>>(V.incb, mask, V.nblk, first, a.last, V.emit, first ? nullptr : V.pair_flag, d_out_size, d_seam8);
    ++*launches;
    return cudaGetLastError();
}

cudaError_t cl_table_init(int alg, int kind, uint32_t* d_table, cudaStream_t stream, uint64_t* launches) {
    cl_table_init_k<<<PL / 256, 256, 0, stream>>>(alg, kind, d_table);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t cl_table_fold(int alg, int kind, uint32_t* d_acc, const uint32_t* d_next, cudaStream_t stream, uint64_t* launches) {
    cl_table_fold_k<<<PL / 256, 256, 0, stream>>>(alg, kind, d_acc, d_next);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t cl_rank_fold(int alg, int kind, const uint32_t* d_tables, uint32_t rank, uint32_t* d_carry, cudaStream_t stream, uint64_t* launches) {
    cl_rank_fold_k<<<PL / 128, 128, 0, stream>>>(alg, kind, d_tables, cl_table_planes(alg, kind), rank, d_carry);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t cl_last_quad(const uint8_t* d_in, size_t n, uint32_t* d_out2, cudaStream_t stream, uint64_t* launches) {
    cl_last_quad_k<<<1, 1, 0, stream>>>(reinterpret_cast<const uint32_t*>(d_in), n / 4, d_out2);
    ++*launches;
    return cudaGetLastError();
}
cudaError_t cl_prev_quad(const uint32_t* d_words, uint32_t rank, uint32_t* d_out, cudaStream_t stream, uint64_t* launches) {
    cl_prev_quad_k<<<1, 1, 0, stream>>>(d_words, 2, rank, d_out);
    ++*launches;
    return cudaGetLastError();
}

// ---- sharded encode with copy mode on every shard (density_b200_cl_shard_prot_*, DESIGN.md section 5) ---------------------------------
// Round k of the copy-map iteration runs on every shard at once: the context from the quad words of the round before, ctx0 and pass P
// under the map M_k, fold P and pass C, fold C, sizes and incompressible bits, then the automaton half shared with Chameleon (transfer,
// settle, commit: prot_*). The shard at the stream start (a.first) runs the staged iteration to the end in phase 1: the map of a prefix
// does not depend on what follows it, so its map, flags and run tables are final. In the rounds it only re-exports them and walks its
// blocks again (which changes nothing). A later shard starts from the empty map. Whatever the map the rounds start from, round k leaves a
// map that agrees with the single call's on one block more than M_k did, and a map that the round leaves unchanged is the single call's.
// Epochs: epoch_base .. + 31 for the staged iteration, epoch_base + 32 + k for round k; the exports read the epoch of the last round that
// ran from the ctx0 epoch word. Under the gate of the rounds (V.gate, opened by prot_start) every kernel returns once the map settled.
constexpr uint32_t CL_PROT_EPOCHS = 32 + PROT_MAX_ROUNDS + 1;
uint32_t cl_prot_epochs() { return CL_PROT_EPOCHS; }

static ProtSegs cl_prot_segs(const CheeView& V) { return prot_segs(V.gate, V.n, V.nblk, V.incb, V.cm, V.cm2, V.seg); }
static void launch_prot_quad(const CheeView& V, const uint8_t* cm, const Status* gate, ProtShard* ps, uint32_t* d_words8, cudaStream_t stream,
                             uint64_t* launches) {
    cl_prot_quad_k<<<1, 256, 0, stream>>>(V.in32, V.nq, V.nblk, V.bbytes / 4, cm, gate, ps, d_words8);
    ++*launches;
}

cudaError_t cl_prot_phase1(const ClShardArgs& a, uint32_t* d_words8, cudaStream_t stream, uint64_t* launches) {
    const CheeView V(a.alg, a.d_in, a.n, a.num_sms, a.ws, a.tables);
    Status* iter = nullptr;
    cudaError_t e = cudaSuccess;
    if (a.first) e = chee_iterate(V, a.epoch_base, a.num_sms, false, V.epoch_word, stream, launches, &iter);
    else if (V.nblk) e = cudaMemsetAsync(V.cm, 0, V.nblk, stream);                 // M_0: nothing copied
    if (e == cudaSuccess) e = cudaMemsetAsync(V.gate, 0, sizeof(Status), stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_words8, 0, CL_PROT_ROUND_WORDS * sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    e = prot_start(cl_prot_segs(V), a.ps, a.offset / V.bbytes, nullptr, 0, V.bbytes, stream, launches);
    if (e != cudaSuccess) return e;
    if (iter) { cl_prot_stage_k<<<1, 1, 0, stream>>>(iter, a.ps); ++*launches; }
    launch_prot_quad(V, V.cm, nullptr, a.ps, d_words8, stream, launches);
    return cudaGetLastError();
}

cudaError_t cl_prot_p(const ClShardArgs& a, int it, const uint32_t* d_all_words, uint32_t rank, uint32_t* d_tab_p, cudaStream_t stream,
                      uint64_t* launches) {
    const CheeView V(a.alg, a.d_in, a.n, a.num_sms, a.ws, a.tables);
    if (!V.nblk) return cudaMemsetAsync(d_tab_p, 0, (size_t)cl_table_planes(a.alg, 0) * PL * sizeof(uint32_t), stream);   // identity
    if (!a.first) {
        cl_prev_quad_k<<<1, 1, 0, stream>>>(d_all_words + 4, CL_PROT_ROUND_WORDS, rank, V.prev_quad);
        ++*launches;
        launch_ctx0_pass_p(V, V.cm, V.gate, V.prev_quad, a.epoch_base + 32 + (uint32_t)it, V.epoch_word, stream, launches);
    }
    if (V.lion) cl_export_p_lion<<<PL / 128, 128, 0, stream>>>(V.in32, V.entP, V.coldP, V.nruns, V.gate, V.epoch_word, d_tab_p);
    else cl_export_p_chee<<<PL / 128, 128, 0, stream>>>(V.entP, V.nruns, V.gate, V.epoch_word, d_tab_p);
    ++*launches;
    return cudaGetLastError();
}

cudaError_t cl_prot_c(const ClShardArgs& a, int it, const uint32_t* d_carry_p, uint32_t* d_tab_c, cudaStream_t stream, uint64_t* launches) {
    const CheeView V(a.alg, a.d_in, a.n, a.num_sms, a.ws, a.tables);
    if (!V.nblk) return cudaMemsetAsync(d_tab_c, 0, (size_t)cl_table_planes(a.alg, 1) * PL * sizeof(uint32_t), stream);
    if (!a.first) launch_fold_p_pass_c(V, V.cm, V.gate, a.epoch_base + 32 + (uint32_t)it, d_carry_p, stream, launches);
    cl_export_c<<<PL / 128, 128, 0, stream>>>(V.entC, V.nruns, V.gate, V.epoch_word, d_tab_c);
    ++*launches;
    return cudaGetLastError();
}

cudaError_t cl_prot_transfer(const ClShardArgs& a, int it, const uint32_t* d_carry_c, uint32_t* d_transfer, cudaStream_t stream, uint64_t* launches) {
    const CheeView V(a.alg, a.d_in, a.n, a.num_sms, a.ws, a.tables);
    if (!a.first && V.nblk) {          // the incompressible bits of the blocks M_k encodes; copied blocks keep those of the round before
        launch_fold_c(V, V.gate, a.epoch_base + 32 + (uint32_t)it, d_carry_c, stream, launches);
        launch_tile_sizes(V, V.cm, 0, V.gate, stream, launches);
    }
    return prot_transfer(cl_prot_segs(V), nullptr, a.ps, it, d_transfer, stream, launches);
}

cudaError_t cl_prot_settle(const ClShardArgs& a, int it, const uint32_t* d_all_transfers, uint32_t rank, uint32_t* d_words8, cudaStream_t stream,
                           uint64_t* launches) {
    const CheeView V(a.alg, a.d_in, a.n, a.num_sms, a.ws, a.tables);
    cudaError_t e = prot_settle(cl_prot_segs(V), a.ps, it, 1, d_all_transfers, rank, d_words8, stream, launches);
    if (e != cudaSuccess) return e;
    launch_prot_quad(V, V.cm2, V.gate, a.ps, d_words8, stream, launches);
    return cudaGetLastError();
}

cudaError_t cl_prot_next(const ClShardArgs& a, int it, const uint32_t* d_all_words, uint32_t world, cudaStream_t stream, uint64_t* launches) {
    const CheeView V(a.alg, a.d_in, a.n, a.num_sms, a.ws, a.tables);
    return prot_commit(cl_prot_segs(V), a.ps, it, d_all_words, world, CL_PROT_ROUND_WORDS, stream, launches);
}

// sizes under the committed map, scan, emit under the gate of the rounds (it has converged when the map settled; the error of an unsettled
// shard closes it), the seam words
cudaError_t cl_prot_finish(const ClShardArgs& a, uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint32_t* d_seam8, cudaStream_t stream,
                           uint64_t* launches, cudaEvent_t ev_emit) {
    const CheeView V(a.alg, a.d_in, a.n, a.num_sms, a.ws, a.tables);
    cudaError_t e = prot_refuse_unsettled(V.gate, a.ps, stream, launches);
    if (e == cudaSuccess && V.nblk) {
        launch_tile_sizes(V, V.cm, 1, V.gate, stream, launches);
        e = launch_scan_emit(V, V.cm, V.gate, cap, d_out_size, d_out, stream, launches, ev_emit);
    } else if (ev_emit) {
        e = cudaEventRecord(ev_emit, stream);
    }
    if (e != cudaSuccess) return e;
    return prot_seam_words(V.nblk, V.gate, d_out_size, d_seam8, stream, launches);
}

}  // namespace dns
