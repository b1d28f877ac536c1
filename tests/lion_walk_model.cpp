// lion_walk_model.cpp — host-side model of the parallel Lion decoder of density_b200/csrc/cl_decode.cu.
// TEST INFRASTRUCTURE (built by tests/test_lion_walk_model_cpu.py with g++, loaded with ctypes): boundaries and unpack as the kernels
// produce them (rows of 32 quads, two 64-byte blocks per row), the chunk-map values in stream order (the run-parallel chunk-map passes
// are the Cheetah decoder's, checked by tests/cl_model.cpp), then the prediction walk with the row algorithm of
// density_b200/csrc/lion_walk.cuh on 32 emulated lanes, then the in-order tail (codec.rs:102-123) from the walked table.
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <vector>

#include "../density_b200/csrc/lion_walk.cuh"

using namespace dns::cld;
using namespace dns::lwalk;

namespace {

struct Prot {   // codec/protection_state.rs:9-47
    uint32_t pen = 0, start = 1, prev = 0; uint64_t counter = 0;
    bool revert() { if ((counter & 15) == 0 && start > 1) start >>= 1; ++counter; return pen > 0; }
    void decay() { pen = (pen - 1) & 0xff; if (pen == 0) start = (start + 1) & 0xff; }
    void update(bool inc) { if (inc) { if (prev) pen = start; prev = 1; } else prev = 0; }
};

inline uint32_t rd16(const uint8_t* p) { return p[0] | (p[1] << 8); }
inline uint32_t rd32(const uint8_t* p) { return rd16(p) | (rd16(p + 2) << 16); }

}  // namespace

// Decodes a Lion stream; returns the decoded size (0: malformed or over capacity). counts4 = {encoded quads walked, predicted quads,
// table reads that waited on a predicted quad, rows walked}.
extern "C" size_t lion_walk_model_decode(const uint8_t* in, size_t n, uint8_t* out, size_t cap, uint64_t* counts4) {
    constexpr uint32_t BS = 64, SB = 6, QPB = 16;
    auto read_sig = [&](uint64_t o) { uint64_t s = 0; for (uint32_t i = 0; i < SB; ++i) s |= (uint64_t)in[o + i] << (8 * i); return s; };
    // ---- 0. boundaries (codec.rs:88-100) ------------------------------------------------------------------------------------------
    struct Blk { uint64_t off; bool copy; };
    std::vector<Blk> blocks;
    Prot ps; uint64_t idx = 0;
    while (n - idx >= SB + BS) {
        if (ps.revert()) { blocks.push_back({idx, true}); idx += BS; ps.decay(); }
        else { const uint32_t sz = lion_block_bytes(read_sig(idx)); blocks.push_back({idx, false}); idx += sz; ps.update(sz >= BS); }
    }
    const uint64_t nb = blocks.size();
    if (nb * BS > cap) return 0;
    // ---- 1. unpack: flag planes per row, K = hash (not predicted) or depth (predicted), values of literals and copy-mode blocks --------
    const uint64_t nrows = (nb + 1) / 2;
    std::vector<uint32_t> P(nrows, 0), A(nrows, 0), kind(nrows * 32, 0), K(nrows * 32, 0), val(nrows * 32, 0);
    for (uint64_t b = 0; b < nb; ++b) {
        const uint8_t* p = in + blocks[b].off;
        if (blocks[b].copy) { for (uint32_t k = 0; k < QPB; ++k) val[b * QPB + k] = rd32(p + 4 * k); continue; }
        uint64_t sig = read_sig(blocks[b].off); p += SB;
        for (uint32_t k = 0; k < QPB; ++k) {
            const uint32_t fl = (uint32_t)(sig & 7u); sig >>= 3;
            const uint64_t i = b * QPB + k;
            const uint32_t lane = (uint32_t)(i & 31);
            A[i / 32] |= 1u << lane;
            kind[i] = lion_kind(fl);
            if (kind[i] == K_PLAIN) { val[i] = rd32(p); p += 4; K[i] = hash16(val[i]); }
            else if (kind[i] != K_PRED) { K[i] = rd16(p); p += 2; }
            else { K[i] = lion_depth(fl); P[i / 32] |= 1u << lane; }
        }
    }
    // ---- 2. chunk-map values (lion.rs:84-123), in stream order --------------------------------------------------------------------
    std::vector<uint32_t> cm(2 * 65536, 0);
    for (uint64_t i = 0; i < nrows * 32; ++i) {
        if (!((A[i / 32] >> (i & 31)) & 1u) || kind[i] == K_PRED) continue;
        uint32_t* e = &cm[2 * K[i]];
        if (kind[i] == K_PLAIN) { e[1] = e[0]; e[0] = val[i]; }
        else if (kind[i] == K_MAP_A) val[i] = e[0];
        else { val[i] = e[1]; e[1] = e[0]; e[0] = val[i]; }
    }
    // ---- 3. the prediction walk --------------------------------------------------------------------------------------------------
    std::vector<uint32_t> T(65536 * 5, 0);
    Warp w;
    WalkCounts cnt{0, 0, 0, 0};
    uint32_t carry = 0;
    for (uint64_t s = 0; s < nrows; ++s) {
        LV<uint32_t> kh, v;
        for (int l = 0; l < 32; ++l) { kh[l] = K[s * 32 + l]; v[l] = val[s * 32 + l]; }
        walk_row(w, P[s], A[s], kh, v, FlatTable{T.data()}, carry, cnt);
        for (int l = 0; l < 32; ++l) val[s * 32 + l] = v[l];
    }
    if (counts4) { counts4[0] = cnt.quads; counts4[1] = cnt.pred; counts4[2] = cnt.dep; counts4[3] = cnt.rows; }
    for (uint64_t i = 0; i < nb * QPB; ++i) { const uint32_t q = val[i]; memcpy(out + 4 * i, &q, 4); }
    // ---- 4. tail (codec.rs:102-123, lion.rs:291-314), in order from the walked table ------------------------------------------------
    uint64_t oidx = nb * BS;
    uint32_t last_hash = carry;
    auto emit = [&](uint32_t q) { if (oidx + 4 > cap) return false; memcpy(out + oidx, &q, 4); oidx += 4; return true; };
    while (n - idx > 0) {
        if (ps.revert()) {
            const uint64_t rem = n - idx, len = rem > BS ? BS : rem;
            if (oidx + len > cap) return 0;
            memcpy(out + oidx, in + idx, len); oidx += len; idx += len;
            if (rem <= BS) break;
            ps.decay();
        } else {
            const uint64_t mark = idx;
            if (n - idx < SB) return 0;
            uint64_t sig = read_sig(idx); idx += SB;
            bool end = false;
            for (uint32_t u = 0; u < QPB && !end; ++u) {
                const uint32_t fl = (uint32_t)(sig & 7u); sig >>= 3;
                if (fl == 0 && n - idx < 4) {                      // decode_partial_unit, lion.rs:293-302
                    const uint64_t rem = n - idx;
                    if (oidx + rem > cap) return 0;
                    memcpy(out + oidx, in + idx, rem); oidx += rem; idx += rem; end = true; break;
                }
                const uint32_t kd = lion_kind(fl);
                L5 L = l5_load(T.data(), last_hash);
                uint32_t q, h;
                if (kd == K_PRED) { q = l5_get(L, lion_depth(fl)); L = l5_mtf(L, lion_depth(fl)); h = hash16(q); }
                else {
                    if (kd == K_PLAIN) { if (n - idx < 4) return 0; q = rd32(in + idx); idx += 4; h = hash16(q); cm[2 * h + 1] = cm[2 * h]; cm[2 * h] = q; }
                    else {
                        if (n - idx < 2) return 0;
                        h = rd16(in + idx); idx += 2;
                        if (kd == K_MAP_A) q = cm[2 * h]; else { q = cm[2 * h + 1]; cm[2 * h + 1] = cm[2 * h]; cm[2 * h] = q; }
                    }
                    L = l5_push(L, q);
                }
                l5_store(T.data(), last_hash, L);
                last_hash = h;
                if (!emit(q)) return 0;
            }
            if (end) break;
            ps.update(idx - mark >= BS);
        }
    }
    return oidx;
}
