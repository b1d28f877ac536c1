// decode_range.cu — bytes [first, first + len) of what a Chameleon stream decodes to, without decoding the bytes in front of them
// (density_b200_chameleon_decode_range_device, DESIGN §4g).
//
// Chameleon's state at a block boundary does not depend on any decoded value: the dictionary in front of block k holds, per bucket, the
// last PLAIN quad before k that hashes there (MAP quads and copy-mode blocks never write it, chameleon.rs:55-68, codec.rs:89-92), and
// the protection automaton depends on the signatures alone. So the window is decoded as a piece of a sharded stream, from its own block
// k0 = first / 256, with the state in front of k0 carried in, by the sharded decode's phase functions:
//  1. locate: the exact in-order main loop of the whole stream in stop-and-report mode (forced_walk_launch<ChamT, true>), then
//     dec_range_report, the tail loop of the whole stream (tail_walk), which stops at the window's blocks behind the main loop too. It
//     gives the decoded size S and the verdict of the whole stream (what density_b200_decoded_size gives), writes {w, S, verdict} to
//     d_result and leaves the report: the offsets of blocks k0 and k1 + 1, the decode candidate in front of k0, main_blocks;
//  2. prefix dictionary: phase 1 of the piece [0, off(k0)) from the stream start (boundaries, writer pass, exported last-writer table);
//  3. window: the piece [off(k0), off(k1 + 1)), or [off(k0), n) as the final piece when the window reaches the main loop's end or S,
//     entered in the located candidate (cham_decode_prot_enter), phase 1 and phase 2 with the prefix table carried in, decoded whole
//     blocks into staging; the caller copies the w window bytes out of it.
// The host reads the report between steps 1 and 2: the pieces' lengths size their grids and their workspace.
#include "../../include/density_b200.h"
#include "common.cuh"
#include "encode_internal.cuh"
#include "decode_bounds.cuh"

namespace dns {
namespace drange {

using bounds::DecStatus;
using T = bounds::ChamT;

// the report (RANGE_REPORT_WORDS u64 at the workspace's start, encode_internal.cuh)
enum : uint32_t { R_W, R_SIZE, R_VERDICT, R_MAIN_BLOCKS, R_OFF0, R_CAND0, R_OFF1, R_FOUND };

// One thread, behind the stop-and-report walk: the tail loop of the whole stream from its start, the stops the main loop did not reach
// found among the tail's blocks, then d_result = {w, S, verdict} and the report. stops: the walk's (bounds::STOP_WORDS per stop).
__global__ void dec_range_report(const uint8_t* __restrict__ in, uint64_t n, const DecStatus* __restrict__ st, uint64_t first, uint64_t len,
                                 uint64_t stop0, uint64_t stop1, const unsigned long long* __restrict__ stops,
                                 unsigned long long* __restrict__ d_result, unsigned long long* __restrict__ report) {
    if (threadIdx.x || blockIdx.x) return;
    const uint64_t mb = st->main_blocks, blk[2] = {stop0, stop1};
    unsigned long long found[2], off[2], state[2];
    for (int k = 0; k < 2; ++k) { found[k] = stops[bounds::STOP_WORDS * k]; off[k] = stops[bounds::STOP_WORDS * k + 1]; state[k] = stops[bounds::STOP_WORDS * k + 2]; }
    const bounds::TailWalk w = bounds::tail_walk(in, n, st, [](uint32_t) {}, [&](uint64_t j, uint64_t i, const Protection& ps) {
        for (int k = 0; k < 2; ++k)
            if (!found[k] && mb + j == blk[k]) { found[k] = 1; off[k] = i; state[k] = bounds::stop_state(ps); }
    });
    const uint64_t size = w.bad ? 0 : mb * T::BS + w.out;
    const uint64_t wlen = (w.bad || first >= size) ? 0 : (len < size - first ? len : size - first);
    const unsigned long long verdict = w.bad ? (unsigned long long)DENSITY_B200_EMALFORMED : 0ull;
    const uint32_t s0 = (uint32_t)state[0];
    d_result[0] = wlen; d_result[1] = size; d_result[2] = verdict;
    report[R_W] = wlen; report[R_SIZE] = size; report[R_VERDICT] = verdict; report[R_MAIN_BLOCKS] = mb;
    report[R_OFF0] = off[0];
    report[R_CAND0] = bounds::pt_cand(bounds::pt_pack(s0 & 0xFFu, (s0 >> 8) & 0xFFu, (s0 >> 16) & 1u, (uint32_t)(stop0 & 15u)));
    report[R_OFF1] = off[1];
    report[R_FOUND] = found[0] | (found[1] << 1);
}

// workspace: the report and the stops, the seed, the window's decoded size, the prefix table, then the body
constexpr size_t H_REPORT = 0, H_STOPS = 256, H_SEED = 512, H_SIZE = 768, H_TABLE = 1024, H_BODY = H_TABLE + 65536 * sizeof(uint32_t);
static size_t up256(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace drange

using namespace drange;

size_t range_locate_workspace_bytes(size_t nbytes) { bounds::BoundsLayout L; return H_BODY + bounds::bounds_layout<T>(nbytes, 0, &L); }

cudaError_t range_locate_launch(const uint8_t* d_in, size_t nbytes, uint64_t first, uint64_t len, uint8_t* ws, uint64_t* d_result,
                                cudaStream_t stream, uint64_t* launches) {
    uint8_t* body = ws + H_BODY;
    bounds::BoundsLayout L; bounds::bounds_layout<T>(nbytes, 0, &L);
    unsigned long long* stops = reinterpret_cast<unsigned long long*>(ws + H_STOPS);
    // the stops: block k0 and the block behind the window's last byte if the window ends in front of S (any larger index is never met)
    const uint64_t end = len > ~first ? ~0ull : first + len;
    const uint64_t stop0 = first / T::BS, stop1 = (end - 1) / T::BS + 1;
    cudaError_t e = cudaMemsetAsync(stops, 0, 2 * bounds::STOP_WORDS * sizeof(uint64_t), stream);
    if (e == cudaSuccess) e = bounds::forced_walk_launch<T, true>(d_in, nbytes, body, L, stream, launches, bounds::WalkStops{{stop0, stop1}, stops});
    if (e != cudaSuccess) return e;
    dec_range_report<<<1, 32, 0, stream>>>(d_in, nbytes, reinterpret_cast<const DecStatus*>(body + L.status), first, len, stop0, stop1, stops,
                                           reinterpret_cast<unsigned long long*>(d_result), reinterpret_cast<unsigned long long*>(ws + H_REPORT));
    ++*launches;
    return cudaGetLastError();
}

bool range_plan(const uint64_t* report, size_t nbytes, uint64_t first, int num_sms, RangePlan* p) {
    *p = RangePlan{};
    p->w = report[R_W];
    if (report[R_VERDICT] || p->w == 0) return true;                   // nothing to decode
    const uint64_t k0 = first / T::BS, k1 = (first + p->w - 1) / T::BS, mb = report[R_MAIN_BLOCKS];
    p->final_piece = first + p->w == report[R_SIZE] || k1 >= mb;
    if (!(report[R_FOUND] & 1u) || (!p->final_piece && !(report[R_FOUND] & 2u)) || report[R_CAND0] >= DECODE_PROT_TRANSFER_WORDS) return false;
    p->k0 = k0; p->skip = first - k0 * T::BS; p->cand0 = (uint32_t)report[R_CAND0];
    p->off0 = report[R_OFF0];
    const uint64_t end = p->final_piece ? nbytes : report[R_OFF1];
    if (p->off0 > end || end > nbytes || (k0 && p->off0 == 0)) return false;
    p->piece_n = end - p->off0;
    p->stage_cap = p->final_piece ? report[R_SIZE] - k0 * T::BS : (k1 - k0 + 1) * T::BS;
    p->window_ws = up256(cham_decode_workspace_bytes(p->piece_n, p->stage_cap, num_sms));
    const size_t prefix = k0 ? cham_decode_workspace_bytes(p->off0, k0 * T::BS, num_sms) : 0;
    const size_t window = p->window_ws + up256(p->stage_cap);
    p->ws_bytes = H_BODY + (prefix > window ? prefix : window);
    return true;
}

cudaError_t range_decode_launch(const uint8_t* d_in, const RangePlan& p, uint8_t* ws, int num_sms, cudaStream_t stream, uint64_t* launches,
                                const uint8_t** d_window) {
    uint8_t* body = ws + H_BODY;
    uint32_t* table = reinterpret_cast<uint32_t*>(ws + H_TABLE);
    uint32_t* seed = reinterpret_cast<uint32_t*>(ws + H_SEED);
    uint8_t* stage = body + p.window_ws;
    cudaError_t e = cudaSuccess;
    // the prefix's last-writer table (block k0 = 0: the stream start, no prefix, no seed). It is the window's carry-in as it stands:
    // folding it over density_b200_table_init's state would only mark bucket 0 touched with fingerprint 0, which decodes to the 0 quad
    // an untouched bucket gives (chameleon.rs:41)
    if (p.k0) {
        e = cham_decode_phase1(d_in, p.off0, p.k0 * T::BS, body, num_sms, table, stream, launches);
        if (e == cudaSuccess) e = cham_decode_prot_enter(nullptr, 0, p.cand0, seed, stream, launches);
    }
    if (e == cudaSuccess)
        e = cham_decode_phase1(d_in + p.off0, p.piece_n, p.stage_cap, body, num_sms, nullptr, stream, launches, p.k0 ? seed : nullptr);
    if (e == cudaSuccess)
        e = cham_decode_phase2(d_in + p.off0, p.piece_n, stage, p.stage_cap, body, num_sms, p.k0 ? table : nullptr,
                               reinterpret_cast<uint64_t*>(ws + H_SIZE), stream, launches);
    *d_window = stage + p.skip;
    return e;
}

}  // namespace dns
