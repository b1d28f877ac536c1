// cl_piece_model.cpp — host-side model of the SHARDED Cheetah decode of density_b200/csrc/cl_decode.cu (DESIGN.md section 5).
// TEST INFRASTRUCTURE (built by tests/test_sharded_cheetah_decode_cpu.py with g++, loaded with ctypes). One Cheetah stream is cut into
// pieces; every piece runs the stages of the kernels on its own runs, with the table logic of density_b200/csrc/cl_core.cuh:
//   boundaries (piece 0 from the fresh protection automaton, copy mode allowed; later pieces must be quiet), the end of a non-final piece
//   (its last blocks appended to the block list), unpack, the symbolic chunk-map pass, the piece's chunk-map transfer, the carry-in as
//   the fold of the earlier pieces' transfers, then prediction rounds in which every piece walks, exports {touched, last value} per
//   context and 4 round words, and folds the earlier pieces' exports into its snapshots; the rounds stop for all pieces at once when no
//   piece walked a run. An in-order decode of the whole stream records the chunk map, the prediction table and the last hash at every
//   cut, and the carries are compared with them.
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <vector>

#include "../density_b200/csrc/cl_core.cuh"

using namespace dns::cld;

namespace {

constexpr uint32_t BS = 128, SB = 8, QPB = 32, PASS = 0xFFFFFFFEu;

struct Prot {   // codec/protection_state.rs:9-47
    uint32_t pen = 0, start = 1, prev = 0; uint64_t counter = 0;
    bool revert() { if ((counter & 15) == 0 && start > 1) start >>= 1; ++counter; return pen > 0; }
    void decay() { pen = (pen - 1) & 0xff; if (pen == 0) start = (start + 1) & 0xff; }
    void update(bool inc) { if (inc) { if (prev) pen = start; prev = 1; } else prev = 0; }
};

inline uint32_t rd16(const uint8_t* p) { return p[0] | (p[1] << 8); }
inline uint32_t rd32(const uint8_t* p) { return rd16(p) | (rd16(p + 2) << 16); }
inline uint64_t rdsig(const uint8_t* p) { uint64_t s = 0; for (uint32_t i = 0; i < SB; ++i) s |= (uint64_t)p[i] << (8 * i); return s; }

struct Snapshot { std::vector<uint32_t> a, b, pred; uint32_t last_hash = 0; };

// in-order decode (codec.rs:82-126, cheetah.rs:67-103) of the whole stream; the state in front of the block that starts at each cut
void in_order(const uint8_t* in, size_t n, const std::vector<uint64_t>& cuts, std::vector<Snapshot>& snaps) {
    std::vector<uint32_t> A(65536, 0), B(65536, 0), P(65536, 0);
    uint32_t lh = 0;
    size_t q = 1;
    auto snap_at = [&](uint64_t idx) {
        while (q < cuts.size() && cuts[q] <= idx) {
            if (cuts[q] == idx) { snaps[q].a = A; snaps[q].b = B; snaps[q].pred = P; snaps[q].last_hash = lh; }
            ++q;
        }
    };
    Prot ps; uint64_t idx = 0;
    while (idx < n) {
        snap_at(idx);
        const bool main = n - idx >= SB + BS;
        if (ps.revert()) {                             // copy mode: BS raw bytes, or the rest of the stream in the tail loop
            if (n - idx > BS) { idx += BS; ps.decay(); continue; }
            idx = n; break;
        }
        if (n - idx < SB) return;
        const uint64_t mark = idx;
        uint64_t sig = rdsig(in + idx); idx += SB;
        bool end = false;
        for (uint32_t u = 0; u < QPB && !end; ++u) {
            const uint32_t fl = (uint32_t)(sig & 3u); sig >>= 2;
            if (!main && n - idx < 4 && fl == 0) { idx = n; end = true; break; }
            uint32_t v, h;
            if (fl == K_PLAIN) { v = rd32(in + idx); idx += 4; h = hash16(v); B[h] = A[h]; A[h] = v; P[lh] = v; }
            else if (fl == K_MAP_A) { if (n - idx < 2) return; h = rd16(in + idx); idx += 2; v = A[h]; P[lh] = v; }
            else if (fl == K_MAP_B) { if (n - idx < 2) return; h = rd16(in + idx); idx += 2; v = B[h]; B[h] = A[h]; A[h] = v; P[lh] = v; }
            else { v = P[lh]; h = hash16(v); }
            lh = h;
        }
        if (end) break;
        ps.update(idx - mark >= BS);
    }
    snap_at(n);
}

struct Piece {
    const uint8_t* in = nullptr; uint64_t n = 0; bool first = false, last = false;
    std::vector<uint64_t> off; std::vector<uint8_t> copy;
    uint64_t tail_off = 0;
    bool refuse = false; uint32_t first_inc = 0, last_inc = 0;
    uint32_t nruns = 1; uint64_t nsteps = 0;
    std::vector<uint8_t> kind, active; std::vector<uint16_t> K; std::vector<uint32_t> val; std::vector<uint8_t> usym;
    std::vector<std::vector<uint32_t>> cmv, cmt;     // per run: chunk-map lists {v0, v1} and meta (epoch 1 | tags) per bucket
    std::vector<uint32_t> cin;                        // per run and bucket: the concrete list carried in
    std::vector<uint32_t> cm_final;
    std::vector<std::vector<uint32_t>> ptv, pte;      // per run: prediction value and epoch per context
    std::vector<uint32_t> snap, final_pred;
    std::vector<uint32_t> ctx_in, ctx_out, run_epoch; std::vector<uint8_t> dirty, dirty_next;
    std::vector<std::vector<uint8_t>> rset;
    uint32_t final_ctx = 0; bool done = false;
    uint64_t run_begin(uint32_t r) const { return (uint64_t)r * nsteps / nruns; }
};

void piece_front(Piece& P) {
    const uint8_t* in = P.in; const uint64_t n = P.n;
    Prot ps; uint64_t idx = 0; bool pair = false, copied = false;
    while (n - idx >= SB + BS) {                       // the main loop's blocks (codec.rs:88-100)
        if (ps.revert()) { P.off.push_back(idx); P.copy.push_back(1); idx += BS; ps.decay(); copied = true; }
        else {
            const uint32_t sz = cheetah_block_bytes(rdsig(in + idx));
            P.off.push_back(idx); P.copy.push_back(0); idx += sz;
            pair |= (sz >= BS) && ps.prev; ps.update(sz >= BS);
        }
    }
    if (!P.first && (pair || copied)) P.refuse = true;
    uint32_t tail_first = 0; uint64_t tail_blocks = 0;
    if (!P.last) {                                     // more stream bytes follow: every block of the piece is a main-loop block
        bool bad = false, ends_copy = !P.copy.empty() && P.copy.back();
        while (idx < n) {
            if (ps.revert() || n - idx < SB) { bad = true; break; }
            const uint32_t sz = cheetah_block_bytes(rdsig(in + idx));
            if (sz > n - idx) { bad = true; break; }
            P.off.push_back(idx); P.copy.push_back(0); idx += sz; ends_copy = false;
            ps.update(sz >= BS);
        }
        if (bad || ends_copy || ps.pen) P.refuse = true;
    } else {                                           // the tail loop's control flow (codec.rs:102-123)
        uint64_t t = idx; bool tcopied = false, tpair = false;
        while (n - t > 0) {
            ++tail_blocks;
            if (ps.revert()) { tcopied = true; if (n - t > BS) { t += BS; ps.decay(); continue; } break; }
            const uint64_t mark = t;
            if (n - t < SB) break;
            uint64_t sig = rdsig(in + t); t += SB;
            bool end = false;
            for (uint32_t u = 0; u < QPB && !end; ++u) {
                const uint32_t fl = (uint32_t)(sig & 3u); sig >>= 2;
                const uint64_t rem = n - t;
                if (fl == 0 && rem < 4) end = true; else if (fl == 0) t += 4; else if (fl != 3) { if (rem < 2) end = true; else t += 2; }
            }
            if (end) break;
            const bool inc = t - mark >= BS;
            if (tail_blocks == 1) tail_first = inc;
            tpair |= inc && ps.prev; ps.update(inc);
        }
        if (!P.first && (tcopied || tpair)) P.refuse = true;
    }
    P.tail_off = P.last ? idx : n;
    P.first_inc = !P.off.empty() ? (!P.copy[0] && cheetah_block_bytes(rdsig(in + P.off[0])) >= BS) : tail_first;
    P.last_inc = ps.prev;
}

void piece_unpack(Piece& P) {
    const uint64_t nb = P.off.size();
    P.nsteps = nb;
    P.kind.assign(nb * 32, 0); P.active.assign(nb * 32, 0); P.K.assign(nb * 32, 0); P.val.assign(nb * 32, 0); P.usym.assign(nb * 32, 0);
    for (uint64_t b = 0; b < nb; ++b) {
        const uint8_t* p = P.in + P.off[b];
        if (P.copy[b]) { for (uint32_t k = 0; k < QPB; ++k) P.val[b * 32 + k] = rd32(p + 4 * k); continue; }
        uint64_t sig = rdsig(p); p += SB;
        for (uint32_t k = 0; k < QPB; ++k) {
            const uint32_t fl = (uint32_t)(sig & 3u); sig >>= 2;
            const uint64_t i = b * 32 + k;
            P.active[i] = 1; P.kind[i] = (uint8_t)cheetah_kind(fl);
            if (fl == K_PLAIN) { P.val[i] = rd32(p); p += 4; P.K[i] = (uint16_t)hash16(P.val[i]); }
            else if (fl != K_PRED) { P.K[i] = (uint16_t)rd16(p); p += 2; }
        }
    }
}

// symbolic chunk-map pass per run; returns the piece's transfer {tags, a, b} per bucket (the composition over its runs)
void piece_cmap(Piece& P, std::vector<uint32_t>& xfer) {
    P.cmv.assign(P.nruns, std::vector<uint32_t>(65536 * 2, 0)); P.cmt.assign(P.nruns, std::vector<uint32_t>(65536, 0));
    for (uint32_t r = 0; r < P.nruns; ++r)
        for (uint64_t i = P.run_begin(r) * 32; i < P.run_begin(r + 1) * 32; ++i) {
            if (!P.active[i] || P.kind[i] == K_PRED) continue;
            List<2> L; const uint32_t h = P.K[i];
            if (P.cmt[r][h]) { L.v[0] = P.cmv[r][2 * h]; L.v[1] = P.cmv[r][2 * h + 1]; L.tag = P.cmt[r][h] & 0x3Fu; L.unk = 0; }
            else { list_init<2>(L, nullptr); L.unk = 0; }
            if (P.kind[i] == K_PLAIN) list_push<2>(L, P.val[i]);
            else {
                const int s = P.kind[i] == K_MAP_A ? 0 : 1;
                const uint32_t t = L.slot_tag(s);
                if (t == TAG_LIT) P.val[i] = L.v[s]; else P.usym[i] = (uint8_t)t;
                if (s == 1) list_mtf<2>(L, 1);
            }
            P.cmv[r][2 * h] = L.v[0]; P.cmv[r][2 * h + 1] = L.v[1]; P.cmt[r][h] = 0x100u | L.tag;
        }
    xfer.assign(3 * 65536, 0);
    for (uint32_t h = 0; h < 65536; ++h) {
        uint32_t v[2] = {0, 0}, tag = 1u | (2u << 3);   // identity
        for (uint32_t r = 0; r < P.nruns; ++r) {
            if (!P.cmt[r][h]) continue;
            const uint32_t yt = P.cmt[r][h] & 0x3Fu; uint32_t nv[2], nt = 0;
            for (int s = 0; s < 2; ++s) {
                const uint32_t t = (yt >> (3 * s)) & 7u;
                if (t == TAG_LIT) nv[s] = P.cmv[r][2 * h + s]; else { nv[s] = v[t - 1]; nt |= ((tag >> (3 * (t - 1))) & 7u) << (3 * s); }
            }
            v[0] = nv[0]; v[1] = nv[1]; tag = nt;
        }
        xfer[h] = tag; xfer[65536 + h] = v[0]; xfer[2 * 65536 + h] = v[1];
    }
}

// acc <- acc, then next (chunk-map transfers)
void cmap_fold(std::vector<uint32_t>& acc, const std::vector<uint32_t>& next) {
    for (uint32_t h = 0; h < 65536; ++h) {
        uint32_t v[2] = {acc[65536 + h], acc[2 * 65536 + h]}, tag = acc[h], nv[2], nt = 0;
        for (int s = 0; s < 2; ++s) {
            const uint32_t t = (next[h] >> (3 * s)) & 7u;
            if (t == TAG_LIT) nv[s] = next[(1 + s) * 65536 + h]; else { nv[s] = v[t - 1]; nt |= ((tag >> (3 * (t - 1))) & 7u) << (3 * s); }
        }
        acc[h] = nt; acc[65536 + h] = nv[0]; acc[2 * 65536 + h] = nv[1];
    }
}

void piece_cmap_resolve(Piece& P, const std::vector<uint32_t>& carry) {
    P.cin.assign((size_t)P.nruns * 65536 * 2, 0); P.cm_final.assign(65536 * 2, 0);
    for (uint32_t h = 0; h < 65536; ++h) {
        uint32_t c[2] = {carry[65536 + h], carry[2 * 65536 + h]};
        for (uint32_t r = 0; r < P.nruns; ++r) {
            P.cin[((size_t)r * 65536 + h) * 2] = c[0]; P.cin[((size_t)r * 65536 + h) * 2 + 1] = c[1];
            if (P.cmt[r][h]) { List<2> L; L.v[0] = P.cmv[r][2 * h]; L.v[1] = P.cmv[r][2 * h + 1]; L.tag = P.cmt[r][h] & 0x3Fu; L.unk = 0; list_carry<2>(c, L); }
        }
        P.cm_final[2 * h] = c[0]; P.cm_final[2 * h + 1] = c[1];
    }
    for (uint32_t r = 0; r < P.nruns; ++r)
        for (uint64_t i = P.run_begin(r) * 32; i < P.run_begin(r + 1) * 32; ++i)
            if (P.usym[i]) P.val[i] = P.cin[((size_t)r * 65536 + P.K[i]) * 2 + (P.usym[i] - 1)];
}

void piece_rounds_init(Piece& P) {
    P.ptv.assign(P.nruns, std::vector<uint32_t>(65536, 0)); P.pte.assign(P.nruns, std::vector<uint32_t>(65536, 0));
    P.snap.assign((size_t)P.nruns * 65536, 0); P.final_pred.assign(65536, 0);
    P.ctx_in.assign(P.nruns, 0); P.ctx_out.assign(P.nruns, PASS); P.run_epoch.assign(P.nruns, 0);
    P.dirty.assign(P.nruns, 1); P.dirty_next.assign(P.nruns, 0);
    P.rset.assign(P.nruns, std::vector<uint8_t>(65536, 0));
    for (uint32_t r = 0; r < P.nruns; ++r) {      // cd_ctx_init: the stream says it when the nearest earlier active quad is not predicted
        uint64_t i = P.run_begin(r) * 32; uint32_t c = 0;
        while (i > 0) { --i; if (P.active[i]) { c = P.kind[i] != K_PRED ? P.K[i] : H_UNKNOWN; break; } }
        P.ctx_in[r] = c;
    }
}

// one round's walk of the dirty runs; the 4 round words and the prediction transfer {touched, value}
uint64_t piece_walk(Piece& P, uint32_t round, uint32_t words[4], std::vector<uint32_t>& xfer) {
    uint64_t walks = 0; uint32_t unknown = 0;
    const uint32_t epoch = round + 1;
    for (uint32_t r = 0; r < P.nruns && !P.done; ++r) {
        if (!P.dirty[r]) continue;
        ++walks;
        std::fill(P.rset[r].begin(), P.rset[r].end(), 0);
        const bool has_snap = round > 0 || (r == 0 && P.first);
        uint32_t ctx = P.ctx_in[r];
        bool any = false, unk_seen = false;
        for (uint64_t i = P.run_begin(r) * 32; i < P.run_begin(r + 1) * 32; ++i) {
            if (!P.active[i]) continue;
            any = true;
            uint32_t H;
            if (ctx == H_UNKNOWN) { if (P.kind[i] == K_PRED) { H = H_UNKNOWN; unk_seen = true; } else H = P.K[i]; ctx = H; continue; }
            if (P.kind[i] == K_PRED) {
                bool unk = false;
                if (P.pte[r][ctx] == epoch) P.val[i] = P.ptv[r][ctx];
                else if (has_snap) { P.val[i] = P.snap[(size_t)r * 65536 + ctx]; P.rset[r][ctx] = 1; }
                else unk = true;
                H = unk ? H_UNKNOWN : hash16(P.val[i]);
                unk_seen |= unk;
            } else { P.ptv[r][ctx] = P.val[i]; P.pte[r][ctx] = epoch; H = P.K[i]; }
            ctx = H;
        }
        P.ctx_out[r] = any ? ctx : PASS;
        P.run_epoch[r] = epoch;
        if (unk_seen) { P.dirty_next[r] = 1; unknown = 1; }
    }
    int last = -1;
    for (uint32_t r = 0; r < P.nruns; ++r) if (P.ctx_out[r] != PASS) last = (int)r;
    words[0] = last >= 0; words[1] = last >= 0 ? P.ctx_out[last] : 0; words[2] = (uint32_t)walks; words[3] = unknown;
    if (!P.done) {
        xfer.assign(2 * 65536, 0);
        for (uint32_t r = 0; r < P.nruns; ++r)
            for (uint32_t c = 0; c < 65536; ++c)
                if (P.run_epoch[r] && P.pte[r][c] == P.run_epoch[r]) { xfer[c] = 1; xfer[65536 + c] = P.ptv[r][c]; }
    }
    return walks;
}

void piece_fold(Piece& P, uint32_t round, const std::vector<uint32_t>& carry_pred, const std::vector<uint32_t>& all_words, uint32_t rank) {
    if (P.done) return;
    for (uint32_t c = 0; c < 65536; ++c) {
        uint32_t v = carry_pred[c];
        for (uint32_t r = 0; r < P.nruns; ++r) {
            uint32_t& sn = P.snap[(size_t)r * 65536 + c];
            if (sn != v) { sn = v; if (round > 0 && P.rset[r][c]) P.dirty_next[r] = 1; }
            if (P.run_epoch[r] && P.pte[r][c] == P.run_epoch[r]) v = P.ptv[r][c];
        }
        P.final_pred[c] = v;
    }
    uint32_t c = 0, walked = 0;
    for (size_t q = 0; q < all_words.size() / 4; ++q) { if (q < rank && all_words[4 * q]) c = all_words[4 * q + 1]; walked += all_words[4 * q + 2]; }
    for (uint32_t r = 0; r < P.nruns; ++r) {
        uint8_t d = P.dirty_next[r];
        if (round == 0 && (r > 0 || !P.first)) d = 1;
        if (P.ctx_in[r] != c) { d = 1; P.ctx_in[r] = c; }
        P.dirty[r] = d; P.dirty_next[r] = 0;
        if (P.ctx_out[r] != PASS) c = P.ctx_out[r];
    }
    P.final_ctx = c;
    if (walked == 0) P.done = true;
}

// the final piece's tail (codec.rs:102-123) from the folded tables; false: malformed or beyond cap
bool piece_tail(Piece& P, uint8_t* out, uint64_t cap, uint64_t& oidx) {
    Prot ps;                                           // the protection state in front of the tail: the main loop's automaton, replayed
    for (uint64_t b = 0; b < P.off.size(); ++b) { ps.revert(); if (P.copy[b]) ps.decay(); else ps.update(cheetah_block_bytes(rdsig(P.in + P.off[b])) >= BS); }
    uint64_t idx = P.tail_off; const uint64_t n = P.n; uint32_t lh = P.final_ctx;
    auto emit = [&](uint32_t q) { if (oidx + 4 > cap) return false; memcpy(out + oidx, &q, 4); oidx += 4; return true; };
    while (n - idx > 0) {
        if (ps.revert()) {
            const uint64_t rem = n - idx, len = rem > BS ? BS : rem;
            if (oidx + len > cap) return false;
            memcpy(out + oidx, P.in + idx, len); oidx += len; idx += len;
            if (rem <= BS) break;
            ps.decay();
            continue;
        }
        const uint64_t mark = idx;
        if (n - idx < SB) return false;
        uint64_t sig = rdsig(P.in + idx); idx += SB;
        bool end = false;
        for (uint32_t u = 0; u < QPB && !end; ++u) {
            const uint32_t fl = (uint32_t)(sig & 3u); sig >>= 2;
            if (n - idx < 4 && fl == 0) {
                const uint64_t rem = n - idx;
                if (oidx + rem > cap) return false;
                memcpy(out + oidx, P.in + idx, rem); oidx += rem; idx += rem; end = true; break;
            }
            uint32_t q, h;
            if (fl == K_PRED) { q = P.final_pred[lh]; h = hash16(q); }
            else {
                if (fl == K_PLAIN) { q = rd32(P.in + idx); idx += 4; h = hash16(q); P.cm_final[2 * h + 1] = P.cm_final[2 * h]; P.cm_final[2 * h] = q; }
                else {
                    if (n - idx < 2) return false;
                    h = rd16(P.in + idx); idx += 2;
                    if (fl == K_MAP_A) q = P.cm_final[2 * h]; else { q = P.cm_final[2 * h + 1]; P.cm_final[2 * h + 1] = P.cm_final[2 * h]; P.cm_final[2 * h] = q; }
                }
                P.final_pred[lh] = q;
            }
            lh = h;
            if (!emit(q)) return false;
        }
        if (end) break;
        ps.update(idx - mark >= BS);
    }
    return true;
}

}  // namespace

// stats (8): {rounds until settled, settled, verdict, refused pieces (bit mask), chunk-map carries that differ from the in-order chunk
// map at their cut (buckets), prediction carries that differ (contexts), entry contexts that differ, run walks}
extern "C" size_t cl_piece_model_decode(const uint8_t* in, size_t n, const uint64_t* cuts_in, uint32_t npieces, const uint32_t* nruns,
                                        uint32_t max_rounds, uint8_t* out, size_t cap, uint32_t* stats) {
    std::vector<uint64_t> cuts(cuts_in, cuts_in + npieces + 1);
    std::vector<Piece> P(npieces);
    for (uint32_t p = 0; p < npieces; ++p) {
        P[p].in = in + cuts[p]; P[p].n = cuts[p + 1] - cuts[p]; P[p].first = p == 0; P[p].last = p == npieces - 1; P[p].nruns = nruns[p] ? nruns[p] : 1;
        if (P[p].n) { piece_front(P[p]); piece_unpack(P[p]); }
    }
    // chunk map: transfers, the carries (stream start: (0, 0), tags 0), resolve
    std::vector<std::vector<uint32_t>> xc(npieces), carry_c(npieces);
    for (uint32_t p = 0; p < npieces; ++p) {
        if (P[p].n) piece_cmap(P[p], xc[p]);
        else { xc[p].assign(3 * 65536, 0); for (uint32_t h = 0; h < 65536; ++h) xc[p][h] = 1u | (2u << 3); }
    }
    std::vector<uint32_t> acc(3 * 65536, 0);
    for (uint32_t p = 0; p < npieces; ++p) {
        carry_c[p] = acc;
        if (P[p].n) { piece_cmap_resolve(P[p], acc); piece_rounds_init(P[p]); }
        else P[p].done = true;
        cmap_fold(acc, xc[p]);
    }
    // rounds: every piece walks, exports, folds the earlier pieces' exports of the same round
    std::vector<std::vector<uint32_t>> xp(npieces, std::vector<uint32_t>(2 * 65536, 0)), carry_p(npieces);
    std::vector<uint32_t> words(4 * npieces, 0);
    uint32_t rounds = 0; uint64_t walks = 0; bool settled = false;
    for (uint32_t round = 0; round < max_rounds && !settled; ++round) {
        for (uint32_t p = 0; p < npieces; ++p) {
            if (P[p].n) walks += piece_walk(P[p], round, &words[4 * p], xp[p]);
            else { for (int k = 0; k < 4; ++k) words[4 * p + k] = 0; }
        }
        std::vector<uint32_t> pacc(65536, 0);
        for (uint32_t p = 0; p < npieces; ++p) {
            carry_p[p] = pacc;
            if (P[p].n) piece_fold(P[p], round, pacc, words, p);
            if (P[p].n) for (uint32_t c = 0; c < 65536; ++c) if (xp[p][c]) pacc[c] = xp[p][65536 + c];
        }
        rounds = round + 1;
        settled = true;
        for (uint32_t p = 0; p < npieces; ++p) if (P[p].n && !P[p].done) settled = false;
    }
    // in-order check of the carries at every cut
    std::vector<Snapshot> snaps(npieces + 1);
    in_order(in, n, cuts, snaps);
    uint32_t bad_c = 0, bad_p = 0, bad_x = 0;
    for (uint32_t p = 1; p < npieces; ++p) {
        if (snaps[p].a.empty()) { ++bad_x; continue; }
        for (uint32_t h = 0; h < 65536; ++h) {
            bad_c += carry_c[p][65536 + h] != snaps[p].a[h] || carry_c[p][2 * 65536 + h] != snaps[p].b[h];
            bad_p += carry_p[p][h] != snaps[p].pred[h];
        }
        uint32_t c = 0;
        for (uint32_t q = 0; q < p; ++q) if (words[4 * q]) c = words[4 * q + 1];
        bad_x += c != snaps[p].last_hash;
    }
    // output and the verdict (seam words: first block incompressible, last incompressible, refused, has blocks)
    uint32_t refused = 0, verdict = settled ? 0u : 1u; uint32_t prev_inc = 0;
    uint64_t oidx = 0;
    for (uint32_t p = 0; p < npieces; ++p) {
        Piece& Q = P[p];
        if (!Q.n) continue;
        const uint64_t base = oidx;
        const uint64_t nq = Q.off.size() * 32;
        if (oidx + nq * 4 > cap) return 0;
        for (uint64_t i = 0; i < nq; ++i) { memcpy(out + oidx, &Q.val[i], 4); oidx += 4; }
        if (Q.last && !piece_tail(Q, out, cap, oidx)) Q.refuse = true;
        if (!Q.last && (oidx - base) % BS) Q.refuse = true;
        if (Q.refuse) { refused |= 1u << p; verdict = 1; }
        if (prev_inc && Q.first_inc) verdict = 1;
        prev_inc = Q.last_inc;
    }
    if (stats) { stats[0] = rounds; stats[1] = settled; stats[2] = verdict; stats[3] = refused; stats[4] = bad_c; stats[5] = bad_p; stats[6] = bad_x; stats[7] = (uint32_t)walks; }
    return verdict ? 0 : oidx;
}
