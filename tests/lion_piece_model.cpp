// lion_piece_model.cpp — host-side model of the walk of a sharded Lion decode (density_b200_lion_decode_shard_walk).
// TEST INFRASTRUCTURE (built by tests/test_sharded_lion_decode_cpu.py with g++, loaded with ctypes). The main-loop blocks of a Lion stream
// are unpacked and their chunk-map values resolved in stream order (as tests/lion_walk_model.cpp does), then walked twice with the row
// algorithm of density_b200/csrc/lion_walk.cuh:
//   whole   one walk over all blocks, two blocks per row, from the stream-start state (zero lists, context 0; lion.rs:67,70);
//   pieces  the blocks cut at the given block indices; every piece lays out its own rows from its first block, as the piece kernels do,
//           and walks them from the state the piece before it left (the lists and last_hash); an empty piece leaves the state as it is.
// Both must give the same values, the same lists and last_hash at the end, and the same encoded and predicted quad counts.
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

constexpr uint32_t QPB = 16;

// per block: copy-mode or not, and per quad its kind, K (hash or depth) and value (not-predicted quads)
struct Blocks { std::vector<uint8_t> copy; std::vector<uint32_t> kind, K, val; uint64_t nb = 0; };

// walks blocks [b0, b1) laid out in rows of their own from state (T, carry); writes the values of the predicted quads into val
void walk_blocks(const Blocks& B, uint64_t b0, uint64_t b1, std::vector<uint32_t>& val, std::vector<uint32_t>& T, uint32_t& carry,
                 WalkCounts& cnt) {
    Warp w;
    for (uint64_t rb = b0; rb < b1; rb += 2) {                     // a row: blocks rb and rb + 1 (if it is in the piece)
        LV<uint32_t> kh, v;
        uint32_t P = 0, A = 0;
        for (int l = 0; l < 32; ++l) {
            const uint64_t b = rb + (uint64_t)l / QPB, i = b * QPB + (uint64_t)l % QPB;
            kh[l] = 0; v[l] = 0;
            if (b >= b1) continue;
            v[l] = val[i];
            if (B.copy[b]) continue;
            A |= 1u << l;
            kh[l] = B.K[i];
            if (B.kind[i] == K_PRED) P |= 1u << l;
        }
        walk_row(w, P, A, kh, v, FlatTable{T.data()}, carry, cnt);
        for (int l = 0; l < 32; ++l) {
            const uint64_t b = rb + (uint64_t)l / QPB;
            if (b < b1) val[b * QPB + (uint64_t)l % QPB] = v[l];
        }
    }
}

}  // namespace

// in[0 .. n): a Lion stream; cuts[0 .. ncuts): block indices 0 = c_0 <= c_1 <= ... <= c_k = main blocks (clamped to them). Returns the
// number of main-loop blocks, or -1 when a value, a list, last_hash or a count differs between the whole walk and the piece walks.
// counts8 = {whole: quads, pred, dep, rows; pieces: the same summed}.
extern "C" long lion_piece_model_check(const uint8_t* in, size_t n, const uint64_t* cuts, int ncuts, uint64_t* counts8) {
    constexpr uint32_t BS = 64, SB = 6;
    auto read_sig = [&](uint64_t o) { uint64_t s = 0; for (uint32_t i = 0; i < SB; ++i) s |= (uint64_t)in[o + i] << (8 * i); return s; };
    std::vector<uint64_t> off;
    Blocks B;
    Prot ps; uint64_t idx = 0;
    while (n - idx >= SB + BS) {                                   // codec.rs:88-100
        if (ps.revert()) { off.push_back(idx); B.copy.push_back(1); idx += BS; ps.decay(); }
        else { const uint32_t sz = lion_block_bytes(read_sig(idx)); off.push_back(idx); B.copy.push_back(0); idx += sz; ps.update(sz >= BS); }
    }
    B.nb = off.size();
    B.kind.assign(B.nb * QPB, K_PRED); B.K.assign(B.nb * QPB, 0); B.val.assign(B.nb * QPB, 0);
    std::vector<uint32_t> cm(2 * 65536, 0);
    for (uint64_t b = 0; b < B.nb; ++b) {
        const uint8_t* p = in + off[b];
        if (B.copy[b]) { for (uint32_t k = 0; k < QPB; ++k) B.val[b * QPB + k] = rd32(p + 4 * k); continue; }
        uint64_t sig = read_sig(off[b]); p += SB;
        for (uint32_t k = 0; k < QPB; ++k) {
            const uint32_t fl = (uint32_t)(sig & 7u); sig >>= 3;
            const uint64_t i = b * QPB + k;
            B.kind[i] = lion_kind(fl);
            if (B.kind[i] == K_PLAIN) { B.val[i] = rd32(p); p += 4; B.K[i] = hash16(B.val[i]); }
            else if (B.kind[i] != K_PRED) { B.K[i] = rd16(p); p += 2; }
            else { B.K[i] = lion_depth(fl); continue; }
            uint32_t* e = &cm[2 * B.K[i]];                         // lion.rs:84-123, in stream order
            if (B.kind[i] == K_PLAIN) { e[1] = e[0]; e[0] = B.val[i]; }
            else if (B.kind[i] == K_MAP_A) B.val[i] = e[0];
            else { B.val[i] = e[1]; e[1] = e[0]; e[0] = B.val[i]; }
        }
    }
    std::vector<uint32_t> vw = B.val, vp = B.val, Tw(65536 * 5, 0), Tp(65536 * 5, 0);
    uint32_t cw = 0, cp = 0;
    WalkCounts kw{0, 0, 0, 0}, kp{0, 0, 0, 0};
    walk_blocks(B, 0, B.nb, vw, Tw, cw, kw);
    for (int k = 0; k + 1 < ncuts; ++k) {
        const uint64_t a = cuts[k] < B.nb ? cuts[k] : B.nb, b = cuts[k + 1] < B.nb ? cuts[k + 1] : B.nb;
        if (a < b) walk_blocks(B, a, b, vp, Tp, cp, kp);           // an empty piece: the state passes on unchanged
    }
    if (counts8) {
        counts8[0] = kw.quads; counts8[1] = kw.pred; counts8[2] = kw.dep; counts8[3] = kw.rows;
        counts8[4] = kp.quads; counts8[5] = kp.pred; counts8[6] = kp.dep; counts8[7] = kp.rows;
    }
    if (vw != vp || Tw != Tp || cw != cp || kw.quads != kp.quads || kw.pred != kp.pred) return -1;
    return (long)B.nb;
}
