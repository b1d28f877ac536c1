// cl_model.cpp — host-side model of the run-parallel Cheetah / Lion decoder scheme of density_b200/csrc/cl_decode.cu.
// TEST INFRASTRUCTURE (built by tests/test_cl_model_cpu.py with g++, loaded with ctypes): it executes the same stages as the CUDA
// kernels — boundaries, unpack, symbolic chunk-map pass + fold + resolve, iterated prediction rounds with snapshots / tags /
// unknown propagation + fold + context sweep, in-order tail — with the table logic of density_b200/csrc/cl_core.cuh (shared with the
// kernels), one run after the other instead of one warp per run. Its output is compared with the oracle-encoded inputs.
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <vector>
#include <stdio.h>
#include <stdlib.h>

#include "../density_b200/csrc/cl_core.cuh"

using namespace dns::cld;

namespace {

struct Prot {   // codec/protection_state.rs:9-47
    uint32_t pen = 0, start = 1, prev = 0; uint64_t counter = 0;
    bool revert() { if ((counter & 15) == 0 && start > 1) start >>= 1; ++counter; return pen > 0; }
    void decay() { pen = (pen - 1) & 0xff; if (pen == 0) start = (start + 1) & 0xff; }
    void update(bool inc) { if (inc) { if (prev) pen = start; prev = 1; } else prev = 0; }
};

template <int N> struct Entry { List<N> L; uint32_t epoch = 0; };

inline uint32_t rd16(const uint8_t* p) { return p[0] | (p[1] << 8); }
inline uint32_t rd32(const uint8_t* p) { return rd16(p) | (rd16(p + 2) << 16); }

template <int NP /* prediction slots: 1 cheetah, 5 lion */>
size_t decode_impl(const uint8_t* in, size_t n, uint8_t* out, size_t cap, uint32_t nruns, uint32_t max_rounds, uint32_t* stats, uint32_t nstats = 4) {
    constexpr bool LION = NP == 5;
    constexpr uint32_t BS = LION ? 64 : 128, SB = LION ? 6 : 8, QPB = BS / 4, FB = LION ? 3 : 2;
    // ---- 0. boundaries (codec.rs:88-100) ------------------------------------------------------------------------------
    struct Blk { uint64_t off; bool copy; };
    std::vector<Blk> blocks;
    Prot ps; uint64_t idx = 0;
    auto read_sig = [&](uint64_t o) { uint64_t s = 0; for (uint32_t i = 0; i < SB; ++i) s |= (uint64_t)in[o + i] << (8 * i); return s; };
    while (n - idx >= SB + BS) {
        if (ps.revert()) { blocks.push_back({idx, true}); idx += BS; ps.decay(); }
        else {
            const uint64_t sig = read_sig(idx);
            const uint32_t sz = LION ? lion_block_bytes(sig) : cheetah_block_bytes(sig);
            blocks.push_back({idx, false}); idx += sz; ps.update(sz >= BS);
        }
    }
    const uint64_t tail_off = idx;
    const uint64_t nb = blocks.size();
    if (nb * BS > cap) return 0;
    // ---- 1. unpack ---------------------------------------------------------------------------------------------------------
    const uint64_t nq = nb * QPB;
    const uint64_t nsteps = (nq + 31) / 32;
    std::vector<uint8_t> kind(nsteps * 32, 0), depth(nsteps * 32, 0), active(nsteps * 32, 0);
    std::vector<uint16_t> K(nsteps * 32, 0);
    std::vector<uint32_t> val(nsteps * 32, 0);
    for (uint64_t b = 0; b < nb; ++b) {
        const uint8_t* p = in + blocks[b].off;
        if (blocks[b].copy) { for (uint32_t k = 0; k < QPB; ++k) val[b * QPB + k] = rd32(p + 4 * k); continue; }
        uint64_t sig = read_sig(blocks[b].off); p += SB;
        for (uint32_t k = 0; k < QPB; ++k) {
            const uint32_t fl = (uint32_t)(sig & ((1u << FB) - 1)); sig >>= FB;
            const uint64_t i = b * QPB + k;
            active[i] = 1;
            kind[i] = (uint8_t)(LION ? lion_kind(fl) : cheetah_kind(fl));
            if (kind[i] == K_PLAIN) { val[i] = rd32(p); p += 4; K[i] = (uint16_t)hash16(val[i]); }
            else if (kind[i] != K_PRED) { K[i] = (uint16_t)rd16(p); p += 2; }
            else depth[i] = (uint8_t)(LION ? lion_depth(fl) : 0);
        }
    }
    if (nruns < 1) nruns = 1;
    if (nruns > nsteps && nsteps) nruns = (uint32_t)nsteps;
    auto run_begin = [&](uint32_t r) { return (uint64_t)r * nsteps / nruns * 32; };   // in quads
    // ---- 2. chunk-map values: symbolic pass per run, fold, resolve --------------------------------------------------------------------
    std::vector<std::vector<Entry<2>>> cm(nruns, std::vector<Entry<2>>(65536));
    std::vector<uint8_t> usym(nsteps * 32, 0);            // 0 resolved, j + 1: value = slot j of the list carried into the run
    for (uint32_t r = 0; r < nruns; ++r) {
        for (uint64_t i = run_begin(r); i < run_begin(r + 1); ++i) {
            if (!active[i] || kind[i] == K_PRED) continue;
            Entry<2>& e = cm[r][K[i]];
            if (e.epoch != 1) { list_init<2>(e.L, nullptr); e.epoch = 1; }
            if (kind[i] == K_PLAIN) list_push<2>(e.L, val[i]);
            else {
                const int s = kind[i] == K_MAP_A ? 0 : 1;
                const uint32_t t = e.L.slot_tag(s);
                if (t == TAG_LIT) val[i] = e.L.v[s]; else usym[i] = (uint8_t)t;
                if (s == 1) list_mtf<2>(e.L, 1);
            }
        }
    }
    std::vector<uint32_t> cin((size_t)nruns * 65536 * 2);
    std::vector<uint32_t> cm_final(65536 * 2);
    for (uint32_t h = 0; h < 65536; ++h) {
        uint32_t c[2] = {0, 0};                            // chunk map starts as (0, 0) (cheetah.rs:52)
        for (uint32_t r = 0; r < nruns; ++r) {
            cin[((size_t)r * 65536 + h) * 2] = c[0]; cin[((size_t)r * 65536 + h) * 2 + 1] = c[1];
            if (cm[r][h].epoch == 1) list_carry<2>(c, cm[r][h].L);
        }
        cm_final[2 * h] = c[0]; cm_final[2 * h + 1] = c[1];
    }
    for (uint32_t r = 0; r < nruns; ++r)
        for (uint64_t i = run_begin(r); i < run_begin(r + 1); ++i)
            if (usym[i]) val[i] = cin[((size_t)r * 65536 + K[i]) * 2 + (usym[i] - 1)];
    // ---- 3. predicted values: rounds --------------------------------------------------------------------------------------------------
    std::vector<std::vector<Entry<NP>>> pt(nruns, std::vector<Entry<NP>>(65536));
    std::vector<uint32_t> snap((size_t)nruns * 65536 * NP, 0), snap_new((size_t)nruns * 65536 * NP, 0);
    std::vector<uint32_t> ctx_in(nruns, H_UNKNOWN), ctx_out(nruns, 0);
    // context of the first active quad of each run when it can be read off the stream: the nearest earlier active quad is not predicted
    for (uint32_t r = 0; r < nruns; ++r) {
        uint64_t i = run_begin(r); uint32_t c = r == 0 ? 0u : H_UNKNOWN; bool found = false;
        while (i > 0) { --i; if (active[i]) { found = true; c = kind[i] != K_PRED ? K[i] : H_UNKNOWN; break; } }
        if (!found) c = 0;                                 // last_hash starts as 0 (cheetah.rs:54)
        ctx_in[r] = c;
    }
    uint32_t rounds = 0; bool converged = false;
    std::vector<uint32_t> final_list(65536 * NP, 0);
    uint32_t final_ctx = 0;
    // A run is walked again only if something it depends on changed (its entry context, a snapshot entry it read, an unknown it met):
    // per-run read sets, per-run epochs (an entry is part of the run's transfer function iff it carries the epoch of the run's LAST walk)
    std::vector<uint8_t> dirty(nruns, 1), dirty_next(nruns, 0);
    std::vector<uint32_t> run_epoch(nruns, 0);
    std::vector<std::vector<uint8_t>> rset(nruns, std::vector<uint8_t>(65536, 0));
    uint64_t walks = 0, queued = 0;                        // queued: run walks the context sweeps ask for (cd_round_end's counter)
    uint32_t last_queued = 0;
    for (uint32_t round = 0; round < max_rounds && !converged; ++round) {
        ++rounds;
        const uint32_t epoch = round + 1;
        for (uint32_t r = 0; r < nruns; ++r) {
            if (!dirty[r]) continue;
            ++walks;
            std::fill(rset[r].begin(), rset[r].end(), 0);
            const bool has_snap = round > 0 || r == 0;
            uint32_t ctx = ctx_in[r];
            bool any_active = false, unknown_seen = false;
            for (uint64_t i = run_begin(r); i < run_begin(r + 1); ++i) {
                if (!active[i]) continue;
                any_active = true;
                uint32_t H;
                if (ctx == H_UNKNOWN) {
                    if (kind[i] == K_PRED) { H = H_UNKNOWN; unknown_seen = true; } else H = K[i];
                    ctx = H; continue;
                }
                Entry<NP>& e = pt[r][ctx];
                if (e.epoch != epoch) {
                    list_init<NP>(e.L, has_snap ? &snap[((size_t)r * 65536 + ctx) * NP] : nullptr); e.epoch = epoch;
                    if (NP > 1 || kind[i] == K_PRED) rset[r][ctx] = 1;      // the carried-in list matters (Cheetah: only to a reader)
                }
                if (kind[i] == K_PRED) {
                    const int k = depth[i];
                    const bool unk = (e.L.unk >> k) & 1u;
                    val[i] = e.L.v[k];
                    H = unk ? H_UNKNOWN : hash16(val[i]);
                    if (unk) unknown_seen = true;
                    if (NP == 1 && e.L.slot_tag(0) != TAG_LIT) rset[r][ctx] = 1;
                    if (k) list_mtf<NP>(e.L, k);
                } else {
                    list_push<NP>(e.L, val[i]);
                    H = K[i];
                }
                ctx = H;
            }
            ctx_out[r] = any_active ? ctx : 0xFFFFFFFEu;   // PASS: the run has no encoded quad
            run_epoch[r] = epoch;
            if (unknown_seen) dirty_next[r] = 1;
        }
        // fold: snapshots in place; a run whose snapshot changed at a key it read is dirty
        for (uint32_t key = 0; key < 65536; ++key) {
            uint32_t c[NP]; for (int s = 0; s < NP; ++s) c[s] = 0;          // prediction tables start as zeros (cheetah.rs:53, lion.rs:70)
            for (uint32_t r = 0; r < nruns; ++r) {
                uint32_t* sn = &snap[((size_t)r * 65536 + key) * NP];
                bool ch = false;
                for (int s = 0; s < NP; ++s) { if (sn[s] != c[s]) { sn[s] = c[s]; ch = true; } }
                if (ch && round > 0 && rset[r][key]) dirty_next[r] = 1;
                if (pt[r][key].epoch == run_epoch[r] && run_epoch[r] != 0) list_carry<NP>(c, pt[r][key].L);
            }
            for (int s = 0; s < NP; ++s) final_list[key * NP + s] = c[s];
        }
        // context sweep + verdict
        uint32_t c = 0, ndirty = 0;
        for (uint32_t r = 0; r < nruns; ++r) {
            uint8_t d = dirty_next[r];
            // runs > 0 had no snapshot in round 0. This changes no value: such a run that read carried-in state met an unknown and is
            // dirty anyway (list_init without a snapshot); one that did not is walked again when its entry context changes, and was exact
            // otherwise. The rule only adds walks, as in cd_round_end, whose walk counts the GPU tests compare with these.
            if (round == 0 && r > 0) d = 1;
            if (ctx_in[r] != c) { d = 1; ctx_in[r] = c; }
            dirty[r] = d; dirty_next[r] = 0; ndirty += d;
            if (ctx_out[r] != 0xFFFFFFFEu) c = ctx_out[r];
        }
        final_ctx = c;
        converged = ndirty == 0;
        queued += ndirty; last_queued = ndirty;
        if (getenv("CL_MODEL_TRUTH")) fprintf(stderr, "round %u: dirty runs for the next round %u\n", round, ndirty);
    }
    if (stats) stats[3] = (uint32_t)walks;
    if (stats) { stats[0] = rounds; stats[1] = converged; stats[2] = (uint32_t)nb; }
    if (stats && nstats >= 7) { stats[4] = (uint32_t)queued; stats[5] = last_queued; stats[6] = nruns; }
    if (!converged) return 0;
    // ---- write the main part --------------------------------------------------------------------------------------------------------
    for (uint64_t i = 0; i < nq; ++i) { out[4 * i] = (uint8_t)val[i]; out[4 * i + 1] = (uint8_t)(val[i] >> 8); out[4 * i + 2] = (uint8_t)(val[i] >> 16); out[4 * i + 3] = (uint8_t)(val[i] >> 24); }
    // ---- 4. tail (codec.rs:102-123), in order from the folded tables ------------------------------------------------------------------
    uint64_t oidx = nq * 4; idx = tail_off;
    uint32_t last_hash = final_ctx;
    auto emit = [&](uint32_t q) { if (oidx + 4 > cap) return false; out[oidx] = (uint8_t)q; out[oidx + 1] = (uint8_t)(q >> 8); out[oidx + 2] = (uint8_t)(q >> 16); out[oidx + 3] = (uint8_t)(q >> 24); oidx += 4; return true; };
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
                const uint32_t fl = (uint32_t)(sig & ((1u << FB) - 1)); sig >>= FB;
                const bool checked = (n - idx) < 4;
                if (checked && fl == 0) {
                    const uint64_t rem = n - idx;
                    if (rem == 0) { end = true; break; }
                    if (oidx + rem > cap) return 0;
                    memcpy(out + oidx, in + idx, rem); oidx += rem; idx += rem; end = true; break;
                }
                const uint32_t kd = LION ? lion_kind(fl) : cheetah_kind(fl);
                uint32_t q, h;
                uint32_t* pl = &final_list[(size_t)last_hash * NP];
                if (kd == K_PRED) {
                    const int k = LION ? (int)lion_depth(fl) : 0;
                    q = pl[k]; for (int j = k; j > 0; --j) pl[j] = pl[j - 1]; pl[0] = q; h = hash16(q);
                } else {
                    if (kd == K_PLAIN) { if (n - idx < 4) return 0; q = rd32(in + idx); idx += 4; h = hash16(q); cm_final[2 * h + 1] = cm_final[2 * h]; cm_final[2 * h] = q; }
                    else { if (n - idx < 2) return 0; h = rd16(in + idx); idx += 2;
                        if (kd == K_MAP_A) q = cm_final[2 * h]; else { q = cm_final[2 * h + 1]; cm_final[2 * h + 1] = cm_final[2 * h]; cm_final[2 * h] = q; } }
                    for (int j = NP - 1; j > 0; --j) pl[j] = pl[j - 1]; pl[0] = q;
                }
                last_hash = h;
                if (!emit(q)) return 0;
            }
            if (end) break;
            ps.update(idx - mark >= BS);
        }
    }
    return oidx;
}

}  // namespace

extern "C" size_t cl_model_decode(int alg, const uint8_t* in, size_t n, uint8_t* out, size_t cap, uint32_t nruns, uint32_t max_rounds, uint32_t* stats) {
    if (alg == 1) return decode_impl<1>(in, n, out, cap, nruns, max_rounds, stats);
    if (alg == 2) return decode_impl<5>(in, n, out, cap, nruns, max_rounds, stats);
    return 0;
}

// Cheetah only, stats7 = {rounds, settled, main blocks, run walks, run walks queued by the context sweeps of all rounds (the GPU's counter:
// the walks after round 0, plus those the last round queued when it did not settle), walks queued by the last round, run count used}
extern "C" size_t cl_model_decode_stats(const uint8_t* in, size_t n, uint8_t* out, size_t cap, uint32_t nruns, uint32_t max_rounds, uint32_t* stats7) {
    return decode_impl<1>(in, n, out, cap, nruns, max_rounds, stats7, 7);
}
