// decoded_size.cu — the length a stream decodes to, without decoding it (density_b200_decoded_size_device, DESIGN §4f).
//
// What Codec::decode writes (codec.rs:82-126) depends only on the signatures and on the protection automaton, never on the dictionary
// contents: every flag yields one 4-byte quad, a copy-mode block its raw bytes, a partial unit at the end the 0-3 bytes that are left.
// So the size is main_blocks x BS plus what the tail loop writes, and the boundary machinery of decode_bounds.cuh already finds the
// first two:
//  1. the candidate rows of the whole stream (rows_launch: dec_chunk_walk, dec_group_compose);
//  2. dec_seq_walk, forced to run, storing no block offset (maxblocks 0) and with no capacity: the exact in-order main loop, which jumps
//     every group and chunk in which the automaton stays in encoded mode and walks the others block by block; it leaves main_blocks,
//     tail_off and the automaton state behind the main loop;
//  3. dec_size_tail: the tail loop's control flow from there (codec.rs:102-123), counting output bytes and reads past the stream end.
// Workspace: bounds_layout<T>(n, 0): the rows and the per-chunk and per-group entries, independent of the decoded size.
#include "../../include/density_b200.h"
#include "common.cuh"
#include "encode_internal.cuh"
#include "decode_bounds.cuh"

namespace dns {
namespace dsize {

using bounds::DecStatus;

// Cheetah / Lion tail loop (scalar_codec.cu decode_loops with a 4-byte unit): the bytes it writes; *bad when it reads past the end.
template <class T>
__device__ uint64_t cl_tail_bytes(const uint8_t* __restrict__ in, uint64_t n, const DecStatus* __restrict__ st, bool* bad) {
    constexpr bool LION = T::BS == 64;
    constexpr uint32_t FB = LION ? 3 : 2;                          // flag bits per quad
    Protection ps = bounds::main_end_state(st);
    uint64_t idx = st->tail_off, out = 0;
    while (n - idx > 0) {
        if (ps.revert_to_copy()) {                                 // codec.rs:104-110: at most BS raw bytes, the last copy stops
            const uint64_t rem = n - idx;
            if (rem <= T::BS) { out += rem; break; }
            idx += T::BS; out += T::BS;
            ps.decay();
            continue;
        }
        const uint64_t mark = idx;
        if (n - idx < T::SIG) { *bad = true; return 0; }
        uint64_t sig = 0;
        for (uint32_t i = 0; i < T::SIG; ++i) sig |= (uint64_t)in[idx + i] << (8 * i);
        idx += T::SIG;
        bool end = false;
        for (uint32_t u = 0; u < T::BS / 4 && !end; ++u) {
            const uint32_t fl = (uint32_t)(sig & ((1u << FB) - 1u)); sig >>= FB;
            const uint32_t kind = LION ? cld::lion_kind(fl) : cld::cheetah_kind(fl);
            const uint64_t rem = n - idx;
            if (kind == cld::K_PLAIN) {
                if (rem < 4) { out += rem; end = true; }           // decode_partial_unit: the last 0-3 bytes, raw, and the stream ends
                else { idx += 4; out += 4; }
            } else if (kind == cld::K_PRED) {
                out += 4;                                          // reads nothing, also behind the stream end
            } else {
                if (rem < 2) { *bad = true; return 0; }
                idx += 2; out += 4;
            }
        }
        if (end) break;
        ps.update(idx - mark >= T::BS);                            // codec.rs:121
    }
    return out;
}

// One thread: d_result = {decoded size, 0} or {0, DENSITY_B200_EMALFORMED}.
template <class T>
__global__ void dec_size_tail(const uint8_t* __restrict__ in, uint64_t n, const DecStatus* __restrict__ st, unsigned long long* __restrict__ d_result) {
    if (threadIdx.x || blockIdx.x) return;
    bool bad = false;
    uint64_t tail;
    if constexpr (T::BS == 256) {
        const bounds::TailWalk w = bounds::tail_walk(in, n, st, [](uint32_t) {});
        bad = w.bad != 0; tail = w.out;
    } else {
        tail = cl_tail_bytes<T>(in, n, st, &bad);
    }
    d_result[0] = bad ? 0ull : (unsigned long long)(st->main_blocks * T::BS + tail);
    d_result[1] = bad ? (unsigned long long)DENSITY_B200_EMALFORMED : 0ull;
}

template <class T>
static cudaError_t launch(const uint8_t* d_in, size_t n, uint8_t* ws, uint64_t* d_result, cudaStream_t stream, uint64_t* launches) {
    bounds::BoundsLayout L; bounds::bounds_layout<T>(n, 0, &L);
    const cudaError_t e = bounds::forced_walk_launch<T>(d_in, n, ws, L, stream, launches);
    if (e != cudaSuccess) return e;
    dec_size_tail<T><<<1, 32, 0, stream>>>(d_in, n, reinterpret_cast<const DecStatus*>(ws + L.status), reinterpret_cast<unsigned long long*>(d_result));
    ++*launches;
    return cudaGetLastError();
}

}  // namespace dsize

size_t decoded_size_workspace_bytes(int alg, size_t nbytes) {
    bounds::BoundsLayout L;
    return alg == ALG_CHAMELEON ? bounds::bounds_layout<bounds::ChamT>(nbytes, 0, &L)
         : alg == ALG_CHEETAH   ? bounds::bounds_layout<bounds::CheeT>(nbytes, 0, &L)
                                : bounds::bounds_layout<bounds::LionT>(nbytes, 0, &L);
}

cudaError_t decoded_size_launch(int alg, const uint8_t* d_in, size_t nbytes, uint8_t* ws, uint64_t* d_result, cudaStream_t stream,
                                uint64_t* launches) {
    switch (alg) {
    case ALG_CHAMELEON: return dsize::launch<bounds::ChamT>(d_in, nbytes, ws, d_result, stream, launches);
    case ALG_CHEETAH:   return dsize::launch<bounds::CheeT>(d_in, nbytes, ws, d_result, stream, launches);
    default:            return dsize::launch<bounds::LionT>(d_in, nbytes, ws, d_result, stream, launches);
    }
}

}  // namespace dns
