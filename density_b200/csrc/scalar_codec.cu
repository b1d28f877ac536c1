// scalar_codec.cu — exact in-order device codec for all three algorithms (one thread walks the stream).
//
// This is the always-correct GPU path: it executes the reference's sequential semantics literally, with the
// dictionaries in global memory (L1/L2-resident). It is used for
//   * Cheetah and Lion encode/decode (cheetah.rs:121-185, lion.rs:209-314) until their segment-parallel
//     kernels land, and
//   * Chameleon decode (chameleon.rs:103-135) and as a device-side cross-check of the parallel Chameleon encoder.
// Stream/driver semantics follow codec/codec.rs:34-126 and codec/protection_state.rs:9-47.
#include "common.cuh"
#include "encode_internal.cuh"
#include "decode_bounds.cuh"

namespace dns {
namespace scalar {

struct Tables {
    uint32_t* chunk_a;  // chameleon chunk_map / cheetah+lion chunk_a   (65536)
    uint32_t* chunk_b;  // cheetah+lion chunk_b                          (65536)
    uint32_t* pred;     // cheetah: 65536, lion: 5 x 65536
};

__device__ __forceinline__ uint32_t ldq(const uint8_t* p) {  // 2-byte aligned little-endian u32
    const uint16_t* s = reinterpret_cast<const uint16_t*>(p);
    return (uint32_t)s[0] | ((uint32_t)s[1] << 16);
}
__device__ __forceinline__ uint32_t ldq_any(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }
__device__ __forceinline__ void stq(uint8_t* p, uint32_t v) { st_u16(p, v & 0xFFFFu); st_u16(p + 2, v >> 16); }

template <int ALG>
struct Enc {
    Tables T;
    uint32_t last_hash = 0;
    uint8_t* out; uint64_t cap; uint64_t idx = 0; bool overflow = false;
    uint64_t sig = 0; uint32_t shift = 0;

    __device__ __forceinline__ bool room(uint32_t n) { if (idx + n > cap) { overflow = true; return false; } return true; }
    __device__ __forceinline__ void push32(uint32_t v) { if (room(4)) { stq(out + idx, v); idx += 4; } }
    __device__ __forceinline__ void push16(uint32_t v) { if (room(2)) { st_u16(out + idx, v); idx += 2; } }
    __device__ __forceinline__ void flag(uint64_t v) { sig |= v << shift; shift += (ALG == ALG_CHAMELEON ? 1 : ALG == ALG_CHEETAH ? 2 : 3); }

    __device__ __forceinline__ void quad(uint32_t q) {
        const uint32_t h = prod_hash(hash_prod(q));
        if (ALG == ALG_CHAMELEON) {  // chameleon.rs:86-101
            if (T.chunk_a[h] != q) { flag(0); push32(q); T.chunk_a[h] = q; }
            else { flag(1); push16(h); }
        } else if (ALG == ALG_CHEETAH) {  // cheetah.rs:121-150
            uint32_t* pr = &T.pred[last_hash];
            if (*pr != q) {
                const uint32_t a = T.chunk_a[h];
                if (a != q) {
                    if (T.chunk_b[h] != q) { flag(0); push32(q); } else { flag(2); push16(h); }
                    T.chunk_b[h] = a; T.chunk_a[h] = q;
                } else { flag(1); push16(h); }
                *pr = q;
            } else flag(3);
            last_hash = h;
        } else {  // lion.rs:209-271
            uint32_t* p = &T.pred[(size_t)last_hash * 5];
            uint32_t v0 = p[0], v1 = p[1], v2 = p[2], v3 = p[3], v4 = p[4];
            if (v0 == q) { flag(1); }
            else if (v1 == q) { flag(2); p[1] = v0; p[0] = q; }
            else if (v2 == q) { flag(3); p[2] = v1; p[1] = v0; p[0] = q; }
            else if (v3 == q) { flag(4); p[3] = v2; p[2] = v1; p[1] = v0; p[0] = q; }
            else {
                if (v4 == q) { flag(5); }
                else {
                    const uint32_t a = T.chunk_a[h];
                    if (a != q) {
                        if (T.chunk_b[h] != q) { flag(0); push32(q); } else { flag(7); push16(h); }
                        T.chunk_b[h] = a; T.chunk_a[h] = q;
                    } else { flag(6); push16(h); }
                }
                p[4] = v3; p[3] = v2; p[2] = v1; p[1] = v0; p[0] = q;  // shift_predictions, lion.rs:50-57
            }
            last_hash = h;
        }
    }
};

template <int ALG>
__global__ void encode_kernel(const uint8_t* __restrict__ in, uint64_t n, uint8_t* __restrict__ out, uint64_t cap, Tables T,
                              Status* __restrict__ status, uint64_t* __restrict__ d_out_size, const uint32_t* __restrict__ run_if_zero,
                              uint32_t* __restrict__ last_hash_io) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (run_if_zero && *run_if_zero != 0) return;   // the parallel encoder already produced the result
    constexpr uint32_t B = ALG == ALG_CHAMELEON ? 256 : ALG == ALG_CHEETAH ? 128 : 64;
    constexpr uint32_t SB = ALG == ALG_LION ? 6 : 8;
    Enc<ALG> E; E.T = T; E.out = out; E.cap = cap;
    if (last_hash_io) E.last_hash = *last_hash_io;      // a reused Codec instance keeps last_hash (cheetah.rs:26, lion.rs:30)
    Protection ps; ps.init();
    const bool aligned4 = (reinterpret_cast<uintptr_t>(in) & 3) == 0;
    for (uint64_t off = 0; off < n && !E.overflow; off += B) {  // codec.rs:76
        const uint32_t blen = (uint32_t)((n - off < B) ? (n - off) : B);
        const uint8_t* blk = in + off;
        if (ps.revert_to_copy()) {  // codec.rs:35-37
            if (E.room(blen)) { for (uint32_t i = 0; i < blen; ++i) out[E.idx + i] = blk[i]; E.idx += blen; }
            ps.decay();
        } else {
            const uint64_t mark = E.idx;
            E.sig = 0; E.shift = 0;
            if (!E.room(SB)) break;
            E.idx += SB;
            uint32_t k = 0;
            if (aligned4) { const uint32_t* b4 = reinterpret_cast<const uint32_t*>(blk); for (; k + 4 <= blen; k += 4) E.quad(b4[k >> 2]); }
            else for (; k + 4 <= blen; k += 4) E.quad(ldq_any(blk + k));
            if (k < blen && E.room(blen - k)) { for (; k < blen; ++k) out[E.idx++] = blk[k]; }  // codec.rs:58-61
            if (E.overflow) break;
            for (uint32_t i = 0; i < SB; ++i) out[mark + i] = (uint8_t)(E.sig >> (8 * i));  // codec.rs:67 / lion.rs:333-336
            ps.update(E.idx - mark >= B);  // codec.rs:68
        }
    }
    if (E.overflow) { status->error = 2; E.idx = 0; }
    status->out_bytes = E.idx;
    if (d_out_size) *d_out_size = E.idx;
    if (last_hash_io) *last_hash_io = E.last_hash;
}

template <int ALG>
struct Dec {
    Tables T;
    uint32_t last_hash = 0;
    const uint8_t* in; uint64_t n; uint64_t idx = 0; bool bad = false;
    uint8_t* out; uint64_t cap; uint64_t oidx = 0; bool overflow = false;

    __device__ __forceinline__ uint64_t remaining() const { return n - idx; }
    __device__ __forceinline__ uint32_t rd32() { if (remaining() < 4) { bad = true; return 0; } uint32_t v = ldq_any(in + idx); idx += 4; return v; }
    __device__ __forceinline__ uint32_t rd16() { if (remaining() < 2) { bad = true; return 0; } uint32_t v = in[idx] | (in[idx + 1] << 8); idx += 2; return v; }
    __device__ __forceinline__ void emit(uint32_t q) {
        if (oidx + 4 > cap) { overflow = true; return; }
        out[oidx] = (uint8_t)q; out[oidx + 1] = (uint8_t)(q >> 8); out[oidx + 2] = (uint8_t)(q >> 16); out[oidx + 3] = (uint8_t)(q >> 24);
        oidx += 4;
    }
    __device__ __forceinline__ void note_pred(uint32_t q) {
        if (ALG == ALG_CHEETAH) T.pred[last_hash] = q;
        else { uint32_t* p = &T.pred[(size_t)last_hash * 5]; p[4] = p[3]; p[3] = p[2]; p[2] = p[1]; p[1] = p[0]; p[0] = q; }
    }
    // returns true when the stream ended inside a partial unit (decode_partial_unit semantics)
    __device__ __forceinline__ bool one(uint64_t& sig, bool checked) {
        constexpr uint32_t FB = ALG == ALG_CHAMELEON ? 1 : ALG == ALG_CHEETAH ? 2 : 3;
        const uint32_t fl = (uint32_t)(sig & ((1u << FB) - 1));
        sig >>= FB;
        if (checked && fl == 0) {  // chameleon.rs:119-129, cheetah.rs:168-176, lion.rs:294-302
            const uint64_t rem = remaining();
            if (rem == 0) return true;
            if (rem < 4) {
                if (oidx + rem > cap) { overflow = true; return true; }
                for (uint64_t i = 0; i < rem; ++i) out[oidx++] = in[idx++];
                return true;
            }
        }
        uint32_t q, h = 0;
        if (ALG == ALG_CHAMELEON) {
            if (fl) q = T.chunk_a[rd16() & 0xFFFFu];                                   // decode_map, chameleon.rs:63-68
            else { q = rd32(); T.chunk_a[prod_hash(hash_prod(q))] = q; }               // decode_plain, :55-61
        } else {
            const bool is_plain = fl == 0;
            const bool is_map_a = (ALG == ALG_CHEETAH) ? fl == 1 : fl == 6;
            const bool is_map_b = (ALG == ALG_CHEETAH) ? fl == 2 : fl == 7;
            if (is_plain) {            // cheetah.rs:67-76, lion.rs:84-96
                q = rd32(); h = prod_hash(hash_prod(q));
                T.chunk_b[h] = T.chunk_a[h]; T.chunk_a[h] = q; note_pred(q);
            } else if (is_map_a) {     // cheetah.rs:78-85, lion.rs:98-107
                h = rd16() & 0xFFFFu; q = T.chunk_a[h]; note_pred(q);
            } else if (is_map_b) {     // cheetah.rs:87-96, lion.rs:109-121
                h = rd16() & 0xFFFFu; q = T.chunk_b[h]; T.chunk_b[h] = T.chunk_a[h]; T.chunk_a[h] = q; note_pred(q);
            } else if (ALG == ALG_CHEETAH) {  // predicted, cheetah.rs:98-103
                q = T.pred[last_hash]; h = prod_hash(hash_prod(q));
            } else {                   // predicted a..e, lion.rs:123-186
                uint32_t* p = &T.pred[(size_t)last_hash * 5];
                const int k = (int)fl - 1;
                q = p[k];
                for (int j = k; j > 0; --j) p[j] = p[j - 1];
                p[0] = q;
                h = prod_hash(hash_prod(q));
            }
            last_hash = h;
        }
        emit(q);
        return false;
    }
};

// main loop (codec.rs:88-100) and tail loop (codec.rs:102-123) of Codec::decode
template <int ALG>
__device__ __forceinline__ void decode_loops(Dec<ALG>& D, Protection& ps, bool with_main) {
    constexpr uint32_t B = ALG == ALG_CHAMELEON ? 256 : ALG == ALG_CHEETAH ? 128 : 64;
    constexpr uint32_t SB = ALG == ALG_LION ? 6 : 8;
    constexpr uint32_t UNIT = ALG == ALG_CHAMELEON ? 8 : 4;
    const uint8_t* in = D.in; uint8_t* out = D.out; const uint64_t cap = D.cap;
    auto read_sig = [&]() -> uint64_t {  // codec.rs:29-31, lion.rs:338-351
        uint64_t v = 0;
        if (D.remaining() < SB) { D.bad = true; return 0; }
        for (uint32_t i = 0; i < SB; ++i) v |= (uint64_t)in[D.idx + i] << (8 * i);
        D.idx += SB;
        return v;
    };
    auto copy_raw = [&](uint64_t len) {
        if (D.oidx + len > cap) { D.overflow = true; return; }
        for (uint64_t i = 0; i < len; ++i) out[D.oidx + i] = in[D.idx + i];
        D.oidx += len; D.idx += len;
    };
    // main loop, codec.rs:88-100
    while (with_main && !D.bad && !D.overflow && D.remaining() >= SB + B) {
        if (ps.revert_to_copy()) { copy_raw(B); ps.decay(); }
        else {
            const uint64_t mark = D.idx;
            uint64_t sig = read_sig();
            for (uint32_t i = 0; i < B / 4; ++i) D.one(sig, false);
            ps.update(D.idx - mark >= B);
        }
    }
    // tail loop, codec.rs:102-123
    while (!D.bad && !D.overflow && D.remaining() > 0) {
        if (ps.revert_to_copy()) {
            if (D.remaining() > B) copy_raw(B);
            else { copy_raw(D.remaining()); break; }
            ps.decay();
        } else {
            const uint64_t mark = D.idx;
            uint64_t sig = read_sig();
            bool end = false;
            for (uint32_t u = 0; u < B / UNIT && !end && !D.bad && !D.overflow; ++u) {
                if (D.remaining() >= UNIT) { for (uint32_t k = 0; k < UNIT / 4; ++k) D.one(sig, false); }
                else { for (uint32_t k = 0; k < UNIT / 4 && !end; ++k) end = D.one(sig, true); }
            }
            if (end) break;
            ps.update(D.idx - mark >= B);
        }
    }
}

template <int ALG>
__global__ void decode_kernel(const uint8_t* __restrict__ in, uint64_t n, uint8_t* __restrict__ out, uint64_t cap, Tables T,
                              Status* __restrict__ status, uint64_t* __restrict__ d_out_size, const uint32_t* __restrict__ run_if,
                              uint32_t* __restrict__ last_hash_io) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (run_if && *run_if == 0) return;   // the parallel decoder already produced the result
    Dec<ALG> D; D.T = T; D.in = in; D.n = n; D.out = out; D.cap = cap;
    if (last_hash_io) D.last_hash = *last_hash_io;
    Protection ps; ps.init();
    decode_loops<ALG>(D, ps, true);
    uint64_t res = D.oidx;
    if (D.bad) { status->error = 3; res = 0; }
    else if (D.overflow) { status->error = 2; res = 0; }
    status->out_bytes = res;
    if (d_out_size) *d_out_size = res;
    if (last_hash_io) *last_hash_io = D.last_hash;
}

// the iteration status of cl_decode.cu, as far as the tail needs it
struct TailIter { unsigned int changed, unknown, done, rounds, final_ctx, gave_up, pad0, pad1; };

// Tail loop only, continuing where the parallel main loop stopped (tables = what the folds left in the workspace).
template <int ALG>
__global__ void decode_tail_kernel(const uint8_t* __restrict__ in, uint64_t n, uint8_t* __restrict__ out, uint64_t cap, Tables T,
                                   Status* __restrict__ status, const bounds::DecStatus* __restrict__ tb, const TailIter* __restrict__ ti,
                                   uint64_t* __restrict__ d_out_size, const uint32_t* __restrict__ skip_if) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (skip_if && *skip_if != 0) return;   // the parallel decoder gave up: the in-order kernel (queued behind) does everything
    constexpr uint32_t B = ALG == ALG_CHAMELEON ? 256 : ALG == ALG_CHEETAH ? 128 : 64;
    Dec<ALG> D; D.T = T; D.in = in; D.n = n; D.out = out; D.cap = cap;
    D.idx = tb->tail_off; D.oidx = tb->main_blocks * B; D.last_hash = ti->final_ctx;
    Protection ps = bounds::main_end_state(tb);   // the entry state of a piece of a sharded stream, carried over the main loop
    decode_loops<ALG>(D, ps, false);
    uint64_t res = D.oidx;
    if (D.bad) { status->error = 3; res = 0; }
    else if (D.overflow) { status->error = 2; res = 0; }
    status->out_bytes = res;
    if (d_out_size) *d_out_size = res;
}

}  // namespace scalar

// workspace: Status (256 B) + chunk_a + chunk_b + pred
size_t scalar_workspace_bytes(int alg) {
    size_t t = 256 + 65536 * 4;
    if (alg != ALG_CHAMELEON) t += 65536 * 4 + (size_t)(alg == ALG_LION ? 5 : 1) * 65536 * 4;
    return t;
}

static scalar::Tables carve(int alg, uint8_t* ws) {
    scalar::Tables T;
    T.chunk_a = reinterpret_cast<uint32_t*>(ws + 256);
    T.chunk_b = (alg != ALG_CHAMELEON) ? T.chunk_a + 65536 : nullptr;
    T.pred = (alg != ALG_CHAMELEON) ? T.chunk_a + 2 * 65536 : nullptr;
    return T;
}

// keep_state: `ws` is the state of a reused Codec instance (tables + last_hash at byte 192): nothing is cleared except the status words
cudaError_t scalar_encode(int alg, const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws,
                          uint64_t* d_out_size, cudaStream_t stream, uint64_t* launches, const uint32_t* d_run_if_zero, bool keep_state) {
    cudaError_t e = cudaMemsetAsync(ws, 0, keep_state ? 128 : scalar_workspace_bytes(alg), stream);  // X::new(): zeroed tables
    if (e != cudaSuccess) return e;
    scalar::Tables T = carve(alg, ws);
    Status* st = reinterpret_cast<Status*>(ws);
    uint32_t* lh = keep_state ? reinterpret_cast<uint32_t*>(ws + 192) : nullptr;
    switch (alg) {
    case ALG_CHAMELEON: scalar::encode_kernel<ALG_CHAMELEON><<<1, 32, 0, stream>>>(d_in, nbytes, d_out, cap, T, st, d_out_size, d_run_if_zero, lh); break;
    case ALG_CHEETAH:   scalar::encode_kernel<ALG_CHEETAH><<<1, 32, 0, stream>>>(d_in, nbytes, d_out, cap, T, st, d_out_size, d_run_if_zero, lh); break;
    default:            scalar::encode_kernel<ALG_LION><<<1, 32, 0, stream>>>(d_in, nbytes, d_out, cap, T, st, d_out_size, d_run_if_zero, lh); break;
    }
    ++*launches;
    return cudaGetLastError();
}

cudaError_t scalar_decode(int alg, const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws,
                          uint64_t* d_out_size, cudaStream_t stream, uint64_t* launches, const uint32_t* d_run_if, bool keep_state) {
    cudaError_t e = cudaMemsetAsync(ws, 0, keep_state ? 128 : scalar_workspace_bytes(alg), stream);
    if (e != cudaSuccess) return e;
    scalar::Tables T = carve(alg, ws);
    Status* st = reinterpret_cast<Status*>(ws);
    uint32_t* lh = keep_state ? reinterpret_cast<uint32_t*>(ws + 192) : nullptr;
    switch (alg) {
    case ALG_CHAMELEON: scalar::decode_kernel<ALG_CHAMELEON><<<1, 32, 0, stream>>>(d_in, nbytes, d_out, cap, T, st, d_out_size, d_run_if, lh); break;
    case ALG_CHEETAH:   scalar::decode_kernel<ALG_CHEETAH><<<1, 32, 0, stream>>>(d_in, nbytes, d_out, cap, T, st, d_out_size, d_run_if, lh); break;
    default:            scalar::decode_kernel<ALG_LION><<<1, 32, 0, stream>>>(d_in, nbytes, d_out, cap, T, st, d_out_size, d_run_if, lh); break;
    }
    ++*launches;
    return cudaGetLastError();
}

cudaError_t scalar_decode_tail(int alg, const uint8_t* d_in, size_t nbytes, uint8_t* d_out, size_t cap, uint8_t* ws, const void* d_bounds_status,
                               const void* d_cl_status, uint64_t* d_out_size, cudaStream_t stream, uint64_t* launches, const uint32_t* d_skip_if) {
    if (alg != ALG_CHEETAH && alg != ALG_LION) return cudaErrorInvalidValue;
    scalar::Tables T = carve(alg, ws);   // cl_decode.cu has filled chunk_a / chunk_b (the fold) and pred (the Cheetah fold / the Lion walk)
    Status* st = reinterpret_cast<Status*>(ws);
    const bounds::DecStatus* tb = reinterpret_cast<const bounds::DecStatus*>(d_bounds_status);
    const scalar::TailIter* ti = reinterpret_cast<const scalar::TailIter*>(d_cl_status);
    if (alg == ALG_CHEETAH) scalar::decode_tail_kernel<ALG_CHEETAH><<<1, 32, 0, stream>>>(d_in, nbytes, d_out, cap, T, st, tb, ti, d_out_size, d_skip_if);
    else scalar::decode_tail_kernel<ALG_LION><<<1, 32, 0, stream>>>(d_in, nbytes, d_out, cap, T, st, tb, ti, d_out_size, d_skip_if);
    ++*launches;
    return cudaGetLastError();
}

}  // namespace dns
