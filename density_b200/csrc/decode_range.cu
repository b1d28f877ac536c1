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
//
// The seek index (density_b200_chameleon_index_build / _decode_range_indexed, DESIGN §4h) records steps 1 and 2 once per stream at
// fixed checkpoints: a range read then runs step 3 alone on the piece between two checkpoints, with the checkpoint's snapshot as the
// carry-in, and a checked copy-out.
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

// workspace: the report and the stops, the seed, the window's decoded size, the prefix table (the indexed decode: a snapshot staged from
// host memory; the index build: a piece's table), then the body
constexpr size_t H_REPORT = 0, H_STOPS = 256, H_SEED = 512, H_SIZE = 768, H_TABLE = 1024, H_BODY = H_TABLE + 65536 * sizeof(uint32_t);
static size_t up256(size_t b) { return (b + 255) & ~(size_t)255; }

// ---- the seek index (DESIGN §4h; the format: include/density_b200.h and encode_internal.cuh) ----------------------------------------
// The build's locate step leaves at the body's start: the report {index bytes, S, verdict, 0 ..} (8 u64), then the index's header and
// directory as they go to d_index, then the stride stops (bounds::STRIDE_WORDS u64 per checkpoint), then the boundary walk's scratch.
constexpr size_t X_REPORT_BYTES = 64;
static uint64_t max_blocks(size_t nbytes) { bounds::BoundsLayout L; bounds::bounds_layout<T>(nbytes, ~(size_t)0, &L); return L.maxblocks; }

// One thread, behind the stride walk: the tail loop of the whole stream (S and the verdict, as dec_size_tail), then the report, the
// header and the directory: checkpoint j = 1 .. C at block j * every, C = (main_blocks - 1) / every, its offset and its decode candidate.
__global__ void dec_index_report(const uint8_t* __restrict__ in, uint64_t n, const DecStatus* __restrict__ st, uint64_t interval, uint64_t cmax,
                                 const unsigned long long* __restrict__ stops, unsigned long long* __restrict__ d_result,
                                 unsigned long long* __restrict__ rep) {
    if (threadIdx.x || blockIdx.x) return;
    const uint64_t mb = st->main_blocks, every = interval / T::BS;
    const bounds::TailWalk w = bounds::tail_walk(in, n, st, [](uint32_t) {});
    const uint64_t size = w.bad ? 0 : mb * T::BS + w.out;
    uint64_t count = mb ? (mb - 1) / every : 0;
    if (count > cmax) count = cmax;                  // cannot happen: main_blocks <= the bound cmax is taken from
    const unsigned long long verdict = w.bad ? (unsigned long long)DENSITY_B200_EMALFORMED : 0ull;
    const uint64_t bytes = w.bad ? 0 : cidx_bytes(count);
    d_result[0] = bytes; d_result[1] = size; d_result[2] = verdict;
    rep[0] = bytes; rep[1] = size; rep[2] = verdict;
    for (int k = 3; k < 8; ++k) rep[k] = 0;
    unsigned long long* hdr = rep + 8;
    hdr[CIDX_MAGIC_W] = CIDX_MAGIC; hdr[CIDX_VERSION_W] = CIDX_VERSION; hdr[CIDX_N_W] = n; hdr[CIDX_SIZE_W] = size;
    hdr[CIDX_MAIN_BLOCKS_W] = mb; hdr[CIDX_INTERVAL_W] = interval; hdr[CIDX_COUNT_W] = count; hdr[CIDX_BYTES_W] = bytes;
    for (uint64_t j = 1; j <= count; ++j) {
        const unsigned long long* o = stops + bounds::STRIDE_WORDS * (j - 1);
        const uint32_t s = (uint32_t)o[1];
        const uint32_t cand = bounds::pt_cand(bounds::pt_pack(s & 0xFFu, (s >> 8) & 0xFFu, (s >> 16) & 1u, (uint32_t)((j * every) & 15u)));
        hdr[8 + 2 * (j - 1)] = o[0];
        hdr[8 + 2 * (j - 1) + 1] = cand;             // {u32 candidate, u32 0}, little-endian
    }
    for (uint64_t k = 8 + 2 * count; k < cidx_snapshots_at(count) / 8; ++k) hdr[k] = 0;   // the directory's padding
}

// The checked copy-out of the indexed decode: the w window bytes from the staging to out (any alignment; NULL: the caller copies them)
// and {w, S, 0} to d_result, only when phase 2 decoded the size the index promises for the piece (got == NULL: no piece, w = 0); else
// {0, S, DENSITY_B200_EMALFORMED} and nothing to out.
__global__ void dec_index_copy_out(const uint8_t* __restrict__ win, uint8_t* __restrict__ out, uint64_t w, uint64_t size, uint64_t expect,
                                   const unsigned long long* __restrict__ got, unsigned long long* __restrict__ d_result) {
    const bool ok = !got || *got == expect;
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t == 0) { d_result[0] = ok ? w : 0; d_result[1] = size; d_result[2] = ok ? 0ull : (unsigned long long)DENSITY_B200_EMALFORMED; }
    if (!ok || !out) return;
    for (uint64_t i = t; i < w; i += (uint64_t)gridDim.x * blockDim.x) out[i] = win[i];
}

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
    // an untouched bucket gives (chameleon.rs:41). An indexed piece has its carry-in already (p.carry_in) and is always entered in its
    // checkpoint's candidate, the stream start's (0) included, so that its launch count does not depend on where the window is.
    const bool enter = p.k0 || p.indexed;
    if (p.k0 && !p.indexed) e = cham_decode_phase1(d_in, p.off0, p.k0 * T::BS, body, num_sms, table, stream, launches);
    if (e == cudaSuccess && enter) e = cham_decode_prot_enter(nullptr, 0, p.cand0, seed, stream, launches);
    if (e == cudaSuccess)
        e = cham_decode_phase1(d_in + p.off0, p.piece_n, p.stage_cap, body, num_sms, nullptr, stream, launches, enter ? seed : nullptr);
    if (e == cudaSuccess)
        e = cham_decode_phase2(d_in + p.off0, p.piece_n, stage, p.stage_cap, body, num_sms, p.indexed ? p.carry_in : p.k0 ? table : nullptr,
                               reinterpret_cast<uint64_t*>(ws + H_SIZE), stream, launches);
    *d_window = stage + p.skip;
    return e;
}

// ---- the seek index ------------------------------------------------------------------------------------------------------------
uint64_t index_max_count(size_t nbytes, uint64_t interval) {
    if (interval < T::BS || interval % T::BS) return 0;
    return (max_blocks(nbytes) - 1) / (interval / T::BS);
}

size_t index_report_bytes(uint64_t cmax) { return X_REPORT_BYTES + cidx_snapshots_at(cmax); }

size_t index_locate_workspace_bytes(size_t nbytes, uint64_t interval) {
    const uint64_t cmax = index_max_count(nbytes, interval);
    bounds::BoundsLayout L;
    return H_BODY + up256(index_report_bytes(cmax)) + up256(cmax * bounds::STRIDE_WORDS * sizeof(uint64_t)) + bounds::bounds_layout<T>(nbytes, 0, &L);
}

cudaError_t index_locate_launch(const uint8_t* d_in, size_t nbytes, uint64_t interval, uint8_t* ws, uint64_t* d_result, uint64_t* h_report,
                                cudaStream_t stream, uint64_t* launches) {
    const uint64_t cmax = index_max_count(nbytes, interval);
    unsigned long long* rep = reinterpret_cast<unsigned long long*>(ws + H_BODY);
    unsigned long long* stops = reinterpret_cast<unsigned long long*>(ws + H_BODY + up256(index_report_bytes(cmax)));
    uint8_t* walk = reinterpret_cast<uint8_t*>(stops) + up256(cmax * bounds::STRIDE_WORDS * sizeof(uint64_t));
    bounds::BoundsLayout L; bounds::bounds_layout<T>(nbytes, 0, &L);
    const cudaError_t e = bounds::forced_walk_launch<T, false, true>(d_in, nbytes, walk, L, stream, launches, bounds::WalkStops{},
                                                                     bounds::StrideStops{interval / T::BS, cmax, stops});
    if (e != cudaSuccess) return e;
    dec_index_report<<<1, 32, 0, stream>>>(d_in, nbytes, reinterpret_cast<const DecStatus*>(walk + L.status), interval, cmax, stops,
                                           reinterpret_cast<unsigned long long*>(d_result), rep);
    ++*launches;
    const cudaError_t e2 = cudaGetLastError();
    return e2 == cudaSuccess ? cudaMemcpyAsync(h_report, rep, index_report_bytes(cmax), cudaMemcpyDeviceToHost, stream) : e2;
}

// the piece in front of checkpoint j + 1 (j = 0 .. C - 1), from the header and directory at hdr
static void index_piece(const uint64_t* hdr, uint64_t j, uint64_t* off, uint64_t* len) {
    const uint64_t* dir = hdr + CIDX_HEADER_WORDS;
    *off = j ? dir[2 * (j - 1)] : 0;
    *len = dir[2 * j] - *off;
}

bool index_build_plan(const uint64_t* rep, size_t nbytes, int num_sms, size_t* ws_bytes) {
    const uint64_t* hdr = rep + X_REPORT_BYTES / 8;
    const uint64_t count = hdr[CIDX_COUNT_W], cap = hdr[CIDX_INTERVAL_W];
    size_t most = 0;
    for (uint64_t j = 0; j < count; ++j) {
        uint64_t off, len;
        index_piece(hdr, j, &off, &len);
        if (hdr[CIDX_HEADER_WORDS + 2 * j] > nbytes || off >= hdr[CIDX_HEADER_WORDS + 2 * j] || hdr[CIDX_HEADER_WORDS + 2 * j + 1] >= DECODE_PROT_TRANSFER_WORDS)
            return false;
        const size_t need = cham_decode_workspace_bytes(len, cap, num_sms);
        if (need > most) most = need;
    }
    *ws_bytes = H_BODY + most;
    return true;
}

cudaError_t index_build_launch(const uint8_t* d_in, const uint64_t* rep, uint8_t* ws, uint8_t* d_index, int num_sms, cudaStream_t stream,
                               uint64_t* launches) {
    const uint64_t* hdr = rep + X_REPORT_BYTES / 8;
    const uint64_t count = hdr[CIDX_COUNT_W], cap = hdr[CIDX_INTERVAL_W];
    uint8_t* body = ws + H_BODY;
    uint32_t* table = reinterpret_cast<uint32_t*>(ws + H_TABLE);
    uint32_t* seed = reinterpret_cast<uint32_t*>(ws + H_SEED);
    auto snapshot = [&](uint64_t j) { return reinterpret_cast<uint32_t*>(d_index + cidx_snapshots_at(count) + (j - 1) * CIDX_SNAPSHOT_BYTES); };
    cudaError_t e = cudaMemcpyAsync(d_index, hdr, cidx_snapshots_at(count), cudaMemcpyHostToDevice, stream);
    // snapshot j + 1 = snapshot j (density_b200_table_init's state for j = 0) folded with piece j's last-writer table
    if (e == cudaSuccess && count) e = cham_table_init(snapshot(1), stream, launches);
    for (uint64_t j = 0; j < count && e == cudaSuccess; ++j) {
        uint64_t off, len;
        index_piece(hdr, j, &off, &len);
        if (j) {
            e = cudaMemcpyAsync(snapshot(j + 1), snapshot(j), CIDX_SNAPSHOT_BYTES, cudaMemcpyDeviceToDevice, stream);
            if (e == cudaSuccess) e = cham_decode_prot_enter(nullptr, 0, (uint32_t)hdr[CIDX_HEADER_WORDS + 2 * (j - 1) + 1], seed, stream, launches);
        }
        if (e == cudaSuccess) e = cham_decode_phase1(d_in + off, len, cap, body, num_sms, table, stream, launches, j ? seed : nullptr);
        if (e == cudaSuccess) e = cham_table_fold(snapshot(j + 1), table, stream, launches);
    }
    return e;
}

uint64_t index_count_for_bytes(uint64_t index_len) {
    for (uint64_t c = index_len / (CIDX_SNAPSHOT_BYTES + 16); c <= index_len / CIDX_SNAPSHOT_BYTES; ++c)
        if (cidx_bytes(c) == index_len) return c;
    return ~0ull;
}

const char* index_check(const uint64_t* hdr, size_t nbytes, uint64_t index_len, uint64_t count) {
    const uint64_t* dir = hdr + CIDX_HEADER_WORDS;
    const uint64_t interval = hdr[CIDX_INTERVAL_W], mb = hdr[CIDX_MAIN_BLOCKS_W], size = hdr[CIDX_SIZE_W];
    if (hdr[CIDX_MAGIC_W] != CIDX_MAGIC || hdr[CIDX_VERSION_W] != CIDX_VERSION) return "not a version 1 Chameleon index";
    if (hdr[CIDX_N_W] != nbytes) return "the index was built for a stream of another length";
    if (hdr[CIDX_COUNT_W] != count || hdr[CIDX_BYTES_W] != index_len) return "index_len does not match the index's checkpoint count";
    if (interval < T::BS || interval % T::BS) return "the index's interval is not a positive multiple of 256";
    // main_blocks within what n bytes can hold, S within the 2 x 264 bytes a tail loop can add to the main loop's blocks
    if (mb > max_blocks(nbytes) || size < mb * T::BS || size - mb * T::BS > 2 * T::MAXBLK) return "the index's sizes are inconsistent";
    if (count && (mb == 0 || count > (mb - 1) / (interval / T::BS))) return "a checkpoint lies behind the main loop";
    for (uint64_t j = 0; j < count; ++j) {
        if (dir[2 * j] >= nbytes || (j && dir[2 * j] <= dir[2 * (j - 1)]) || (j == 0 && dir[0] == 0)) return "the directory's offsets are not increasing";
        if (dir[2 * j] & 1) return "a directory offset is odd";   // every block of a Chameleon stream starts at an even offset
        if (dir[2 * j + 1] >= DECODE_PROT_TRANSFER_WORDS) return "a directory candidate is out of range";
    }
    return nullptr;
}

bool index_plan(const uint64_t* hdr, size_t nbytes, uint64_t first, uint64_t len, int num_sms, RangePlan* p, uint64_t* snapshot) {
    *p = RangePlan{};
    *snapshot = 0;
    const uint64_t* dir = hdr + CIDX_HEADER_WORDS;
    const uint64_t size = hdr[CIDX_SIZE_W], mb = hdr[CIDX_MAIN_BLOCKS_W], every = hdr[CIDX_INTERVAL_W] / T::BS, count = hdr[CIDX_COUNT_W];
    if (first >= size) return false;                                  // nothing to decode
    p->w = len < size - first ? len : size - first;
    const uint64_t k0 = first / T::BS, k1 = (first + p->w - 1) / T::BS;
    const uint64_t a = k0 / every < count ? k0 / every : count, b = k1 / every + 1;
    p->final_piece = b > count || k1 >= mb || first + p->w == size;
    p->indexed = true;
    p->off0 = 0;                                                      // the caller passes the piece, d_in + piece_off
    p->piece_off = a ? dir[2 * (a - 1)] : 0;
    p->cand0 = a ? (uint32_t)dir[2 * (a - 1) + 1] : 0;                // 0: the stream start's state
    p->piece_n = (p->final_piece ? nbytes : dir[2 * (b - 1)]) - p->piece_off;
    p->skip = first - a * every * T::BS;
    p->stage_cap = p->final_piece ? size - a * every * T::BS : (b - a) * every * T::BS;
    p->window_ws = up256(cham_decode_workspace_bytes(p->piece_n, p->stage_cap, num_sms));
    p->ws_bytes = H_BODY + p->window_ws + up256(p->stage_cap);
    *snapshot = a;
    return true;
}

uint32_t* range_table_slot(uint8_t* ws) { return reinterpret_cast<uint32_t*>(ws + H_TABLE); }

cudaError_t index_copy_out_launch(const RangePlan& p, const uint8_t* d_window, uint64_t size, uint8_t* d_out, uint8_t* ws, uint64_t* d_result,
                                  int num_sms, cudaStream_t stream, uint64_t* launches) {
    const uint64_t blocks = (p.w + 256 * 16 - 1) / (256 * 16);
    const uint32_t grid = blocks < 1 ? 1u : blocks > (uint64_t)num_sms * 8 ? (uint32_t)num_sms * 8 : (uint32_t)blocks;
    dec_index_copy_out<<<grid, 256, 0, stream>>>(d_window, d_out, p.w, size, p.stage_cap,
                                                 p.w ? reinterpret_cast<const unsigned long long*>(ws + H_SIZE) : nullptr,
                                                 reinterpret_cast<unsigned long long*>(d_result));
    ++*launches;
    return cudaGetLastError();
}

}  // namespace dns
