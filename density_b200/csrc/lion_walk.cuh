// lion_walk.cuh — the prediction walk of the parallel Lion decoder (cl_decode.cu, stage 3), written once for device and host.
//
// Reference semantics: /root/reference/src/algorithms/lion/lion.rs:50-57 (shift_predictions), :84-186 (decode_plain / decode_map_a /
// decode_map_b / decode_predicted_a..e), driven by codec/codec.rs:82-126. Every encoded quad works on the 5-slot list of its context,
// the hash of the quad before it (last_hash starts as 0, lion.rs:67):
//     not predicted (value v from the stream or the chunk map):  push v in front, the last slot falls out
//     predicted at depth k (flag k + 1):                         read slot k, move it to the front
// The values of the not-predicted quads and their hashes are known before the walk (stages 1 and 2). Only the quad behind a predicted
// quad has to wait for a table read to learn its context, so one warp walks the stream in order, 32 quads (one row) per step:
//   1. every lane whose context is known at the row start (the quad before it is not predicted, or lies in an earlier row) reads its
//      context's list, all in one round;
//   2. the predicted lanes, in order: the list in front of lane p is the list the latest earlier predicted lane at the same context
//      left, or that context's row-start list (a lane that read it, else a read now: the only read that waits on a predicted quad),
//      followed by the pushes of the not-predicted lanes at that context after it (only the last 5 matter). Predicted-A lanes right
//      behind p that map the context onto itself (zero fill) read the same slot and change nothing;
//   3. write-back: the last lane of every context group builds the group's final list the same way and stores it;
//   4. the row's last encoded quad gives the next row's context.
// The lanes of a copy-mode block are inactive: they leave the context and the table untouched (codec.rs:89-92).
//
// The code is written against a small lane interface: on the device a Warp is the 32 threads of the walking warp and LV<T> one value
// per thread; on the host (tests/lion_walk_model.cpp, built with g++) a Warp runs the 32 lanes one after the other and LV<T> holds all
// 32 values. Every cross-lane step goes through the interface, so the model executes the kernel's row algorithm step for step.
#pragma once
#include "cl_core.cuh"

namespace dns {
namespace lwalk {

// a prediction list (lion.rs:41-48: next_a .. next_e); named slots keep it in registers on the device
struct L5 { uint32_t a, b, c, d, e; };

CLD_HD uint32_t l5_get(const L5& L, uint32_t k) { return k == 0 ? L.a : k == 1 ? L.b : k == 2 ? L.c : k == 3 ? L.d : L.e; }
CLD_HD L5 l5_push(const L5& L, uint32_t v) { return L5{v, L.a, L.b, L.c, L.d}; }                 // shift_predictions, lion.rs:50-57
CLD_HD L5 l5_mtf(const L5& L, uint32_t k) {                                                       // decode_predicted_a..e, lion.rs:125-186
    return L5{l5_get(L, k), k >= 1 ? L.a : L.b, k >= 2 ? L.b : L.c, k >= 3 ? L.c : L.d, k >= 4 ? L.d : L.e};
}
// 5 consecutive u32 per context: the layout of the in-order kernel's table (scalar_codec.cu), so the tail continues on it
CLD_HD L5 l5_load(const uint32_t* T, uint32_t ctx) { const uint32_t* p = T + (size_t)ctx * 5; return L5{p[0], p[1], p[2], p[3], p[4]}; }
CLD_HD void l5_store(uint32_t* T, uint32_t ctx, const L5& L) { uint32_t* p = T + (size_t)ctx * 5; p[0] = L.a; p[1] = L.b; p[2] = L.c; p[3] = L.d; p[4] = L.e; }
// The walk reaches the table through load / store / row_end (after a row's write-back, before the next row's reads). A flat table is
// one array of 65536 lists; the walk kernel may place the lists elsewhere (cl_decode.cu).
struct FlatTable {
    uint32_t* T;
    CLD_HD L5 load(uint32_t ctx) const { return l5_load(T, ctx); }
    CLD_HD void store(uint32_t ctx, const L5& L) const { l5_store(T, ctx, L); }
    CLD_HD void row_end() const {}
};

CLD_HD int lw_ffs(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __ffs(x);
#else
    return __builtin_ffs((int)x);
#endif
}
CLD_HD int lw_popc(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __popc(x);
#else
    return __builtin_popcount(x);
#endif
}
CLD_HD int lw_top(uint32_t x) {   // highest set bit of x != 0
#if defined(__CUDA_ARCH__)
    return 31 - __clz(x);
#else
    return 31 - __builtin_clz(x);
#endif
}

#if defined(__CUDA_ARCH__)
template <class T> struct LV {
    T x;
    __device__ __forceinline__ T& operator[](int) { return x; }
    __device__ __forceinline__ const T& operator[](int) const { return x; }
};
struct Warp {
    int lane;
    static constexpr uint32_t FULL = 0xFFFFFFFFu;
    template <class F> __device__ __forceinline__ void each(F f) { f(lane); }
    template <class F> __device__ __forceinline__ uint32_t ballot(F f) { return __ballot_sync(FULL, f(lane)); }
    __device__ __forceinline__ uint32_t shfl(const LV<uint32_t>& v, int src) { return __shfl_sync(FULL, v.x, src); }
    __device__ __forceinline__ LV<uint32_t> shfl_up1(const LV<uint32_t>& v) { return LV<uint32_t>{__shfl_up_sync(FULL, v.x, 1)}; }
    __device__ __forceinline__ LV<uint32_t> gather(const LV<uint32_t>& v, const LV<int>& src) { return LV<uint32_t>{__shfl_sync(FULL, v.x, src.x)}; }
    __device__ __forceinline__ LV<L5> gather(const LV<L5>& v, const LV<int>& src) {
        const int s = src.x;
        return LV<L5>{L5{__shfl_sync(FULL, v.x.a, s), __shfl_sync(FULL, v.x.b, s), __shfl_sync(FULL, v.x.c, s), __shfl_sync(FULL, v.x.d, s),
                         __shfl_sync(FULL, v.x.e, s)}};
    }
    __device__ __forceinline__ LV<uint32_t> match_any(const LV<uint32_t>& k) { return LV<uint32_t>{__match_any_sync(FULL, k.x)}; }
    __device__ __forceinline__ void sync() { __syncwarp(); }   // the next row reads what this row's write-back stored
};
#else
template <class T> struct LV {
    T x[32];
    T& operator[](int l) { return x[l]; }
    const T& operator[](int l) const { return x[l]; }
};
struct Warp {
    template <class F> void each(F f) { for (int l = 0; l < 32; ++l) f(l); }
    template <class F> uint32_t ballot(F f) { uint32_t m = 0; for (int l = 0; l < 32; ++l) if (f(l)) m |= 1u << l; return m; }
    uint32_t shfl(const LV<uint32_t>& v, int src) { return v[src]; }
    LV<uint32_t> shfl_up1(const LV<uint32_t>& v) { LV<uint32_t> r; for (int l = 0; l < 32; ++l) r[l] = v[l > 0 ? l - 1 : 0]; return r; }
    template <class T> LV<T> gather(const LV<T>& v, const LV<int>& src) { LV<T> r; for (int l = 0; l < 32; ++l) r[l] = v[src[l]]; return r; }
    LV<uint32_t> match_any(const LV<uint32_t>& k) {
        LV<uint32_t> r;
        for (int l = 0; l < 32; ++l) { r[l] = 0; for (int m = 0; m < 32; ++m) if (k[m] == k[l]) r[l] |= 1u << m; }
        return r;
    }
    void sync() {}
};
#endif

// what the walk did: encoded quads, predicted quads, table reads that waited on a predicted quad, rows
struct WalkCounts { unsigned long long quads, pred, dep, rows; };

// The list of context c[l] in front of an operation, for every lane l in `need`. ops[l]: the lanes at c[l] whose operations come
// first; all[l]: every lane at c[l]; done: the predicted lanes resolved so far; ldm: lanes whose rs holds their context's row-start list.
template <class W, class Tab>
CLD_HD LV<L5> list_before(W& w, uint32_t need, uint32_t P, uint32_t done, uint32_t& ldm, const LV<uint32_t>& c, const LV<uint32_t>& ops,
                          const LV<uint32_t>& all, const LV<uint32_t>& v, LV<L5>& rs, const LV<L5>& la, const Tab& T, WalkCounts& cnt) {
    LV<int> src; LV<uint32_t> pushes, from_la, read;
    w.each([&](int l) {
        src[l] = l; pushes[l] = 0; from_la[l] = 0; read[l] = 0;
        if (!((need >> l) & 1u)) return;
        const uint32_t pd = ops[l] & done;
        uint32_t pu = ops[l] & ~P;
        if (pd) {                                                   // the list the latest earlier predicted lane left
            const int lp = lw_top(pd);
            src[l] = lp; from_la[l] = 1;
            pu &= lp == 31 ? 0u : ~((2u << lp) - 1u);
        }
        while (lw_popc(pu) > 5) pu &= pu - 1u;                       // five pushes replace the whole list
        pushes[l] = pu;
        if (!pd && lw_popc(pu) < 5) {                               // the row-start list
            const uint32_t holders = ldm & all[l];
            if (holders) src[l] = lw_ffs(holders) - 1;
            else { rs[l] = T.load(c[l]); read[l] = 1; }
        }
    });
    const uint32_t reads = w.ballot([&](int l) { return read[l] != 0; });
    cnt.dep += (unsigned)lw_popc(reads);
    ldm |= reads;
    LV<L5> L = w.gather(rs, src);
    const LV<L5> Lp = w.gather(la, src);
    w.each([&](int l) { if (from_la[l]) L[l] = Lp[l]; });
    while (w.ballot([&](int l) { return pushes[l] != 0; })) {       // the pushes in stream order
        LV<int> q; LV<uint32_t> has;
        w.each([&](int l) { has[l] = pushes[l] != 0; q[l] = has[l] ? lw_ffs(pushes[l]) - 1 : l; pushes[l] &= pushes[l] - 1u; });
        const LV<uint32_t> pv = w.gather(v, q);
        w.each([&](int l) { if (has[l]) L[l] = l5_push(L[l], pv[l]); });
    }
    return L;
}

// One row. P: predicted lanes, A: encoded lanes. kh: the hash of a not-predicted quad (explicit for MAP_A / MAP_B, of the literal for
// PLAIN), the depth (flag - 1) of a predicted one. v: the value of every not-predicted lane; on return also of every predicted lane.
// carry: the context of the row's first quad, on return of the next row's. T: the table (FlatTable or a placement of the kernel's),
// updated in place.
template <class W, class Tab>
CLD_HD void walk_row(W& w, uint32_t P, const uint32_t A, const LV<uint32_t>& kh, LV<uint32_t>& v, const Tab& T, uint32_t& carry, WalkCounts& cnt) {
    ++cnt.rows;
    P &= A;
    if (!A) return;                                                 // two copy-mode blocks
    cnt.quads += (unsigned)lw_popc(A);
    cnt.pred += (unsigned)lw_popc(P);
    const uint32_t inrow = A & (A << 1);                            // the quad before the lane is the lane before it; else it is `carry`
    const uint32_t known = A & ~(inrow & (P << 1));                 // context known before any table read
    const uint32_t pa0 = P & w.ballot([&](int l) { return kh[l] == 0; });   // predicted-A lanes
    const LV<uint32_t> kprev = w.shfl_up1(kh);
    LV<uint32_t> ctx, h;
    LV<L5> rs, la;
    const uint32_t c0 = carry;
    w.each([&](int l) {                                             // 1. contexts and row-start lists
        const uint32_t bit = 1u << l;
        ctx[l] = (known & bit) ? ((inrow & bit) ? kprev[l] : c0) : cld::H_UNKNOWN;
        h[l] = (P & bit) ? cld::H_UNKNOWN : kh[l];
        la[l] = L5{0, 0, 0, 0, 0};
        rs[l] = (known & bit) ? T.load(ctx[l]) : L5{0, 0, 0, 0, 0};
    });
    uint32_t ldm = known, done = 0, todo = P;
    while (todo) {                                                  // 2. predicted lanes in order
        const int p = lw_ffs(todo) - 1;
        const uint32_t c = w.shfl(ctx, p);                          // final: the lanes before p are resolved
        const uint32_t at_c = w.ballot([&](int l) { return ctx[l] == c; });
        const uint32_t k = w.shfl(kh, p);
        LV<uint32_t> cc, ops, all;
        w.each([&](int l) { cc[l] = c; ops[l] = at_c & A & ((1u << p) - 1u); all[l] = at_c; });
        const LV<L5> Lb = list_before(w, 1u << p, P, done, ldm, cc, ops, all, v, rs, la, T, cnt);
        w.each([&](int l) { if (l == p) { v[l] = l5_get(Lb[l], k); la[l] = l5_mtf(Lb[l], k); } });
        const uint32_t val = w.shfl(v, p);
        const uint32_t hp = cld::hash16(val);
        uint32_t span = 0;
        if (hp == c && p < 31) { const uint32_t r = pa0 >> (p + 1); span = (uint32_t)(lw_ffs(~r) - 1); }
        const uint32_t S = span ? (((1u << span) - 1u) << (p + 1)) : 0u;
        const int next = p + 1 + (int)span;
        w.each([&](int l) {
            const uint32_t bit = 1u << l;
            if (l == p || (S & bit)) { v[l] = val; h[l] = hp; ctx[l] = l == p ? ctx[l] : c; }
            if (l == next && (inrow & bit)) ctx[l] = hp;
        });
        done |= 1u << p;
        todo &= ~((1u << p) | S);
    }
    LV<uint32_t> key;                                               // 3. write-back by the last lane of every context group
    w.each([&](int l) { key[l] = ((A >> l) & 1u) ? ctx[l] : 0x10000u + (uint32_t)l; });
    const LV<uint32_t> grp = w.match_any(key);
    const uint32_t leaders = A & w.ballot([&](int l) { return ((grp[l] >> l) >> 1) == 0; });
    const LV<L5> Lf = list_before(w, leaders, P, done, ldm, ctx, grp, grp, v, rs, la, T, cnt);
    w.each([&](int l) { if ((leaders >> l) & 1u) T.store(ctx[l], Lf[l]); });
    T.row_end();
    carry = w.shfl(h, lw_top(A));                                   // 4. lion.rs:286 (last_hash)
    w.sync();
}

}  // namespace lwalk
}  // namespace dns
