// api.cu — the C ABI of libdensity_b200.so (see include/density_b200.h).
//
// Entry points mirror the reference's extern "C" exports
//   /root/reference/src/algorithms/chameleon/chameleon.rs:70-83
//   /root/reference/src/algorithms/cheetah/cheetah.rs:105-118
//   /root/reference/src/algorithms/lion/lion.rs:193-206
// and add stream-ordered device-pointer variants. There is no CPU fallback anywhere in this file: if CUDA is
// unavailable every call fails with DENSITY_B200_ECUDA / returns 0.
#include "../../include/density_b200.h"
#include "common.cuh"
#include "encode_internal.cuh"
#include "decode_bounds.cuh"

#include <dlfcn.h>

#include <atomic>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <deque>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

namespace dns {

static thread_local std::string g_last_error;
static std::atomic<uint64_t> g_launches{0};

static void set_error(const char* what, cudaError_t e) {
    char buf[512];
    snprintf(buf, sizeof buf, "%s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
    g_last_error = buf;
}
static void set_error(const char* what) { g_last_error = what; }
// the end of an enqueued step: its kernel launches are counted, and a CUDA error becomes DENSITY_B200_ECUDA with `what` as the message
static int step_result(cudaError_t e, uint64_t launches, const char* what) {
    g_launches += launches;
    if (e != cudaSuccess) { set_error(what, e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}
// the outputs of an empty piece of a sharded stream: size 0, and seam words that say it has no blocks
static cudaError_t empty_piece_outputs(uint64_t* d_out_size, uint32_t* d_seam8, cudaStream_t st) {
    const cudaError_t e = cudaMemsetAsync(d_out_size, 0, sizeof(uint64_t), st);
    return e == cudaSuccess ? cudaMemsetAsync(d_seam8, 0, 8 * sizeof(uint32_t), st) : e;
}

// grow-only device buffer
struct DevBuf {
    uint8_t* p = nullptr; size_t bytes = 0;
    // `stream`: the stream that next touches the buffer. The zero fill (the Cheetah / Lion encoder tables rely on starting out
    // zeroed) is ordered on it; cudaFree of the old buffer synchronises the device, so nothing can still be using it. There is no
    // default: the library's streams do not order against the legacy default stream, so a fill there could land after the next write.
    cudaError_t ensure(size_t need, cudaStream_t stream) {
        if (need <= bytes) return cudaSuccess;
        if (p) { cudaFree(p); p = nullptr; bytes = 0; }
        size_t want = need + need / 8 + 4096;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { cudaGetLastError(); e = cudaMalloc(&p, need); want = need; }
        if (e == cudaSuccess) { bytes = want; e = cudaMemsetAsync(p, 0, want, stream); }
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
};

// ---- pageable host buffers ------------------------------------------------------------------------------------------------------
// A Rust Vec<u8> (what the reference's callers pass) is pageable memory: cudaMemcpy from / to it goes through the driver's own bounce
// buffer with one host thread (~8-12 GB/s). The synchronous entry points therefore stage pageable buffers through a pinned ring of
// two slots per direction with a multi-threaded memcpy, so that the host copy of piece k + 1 overlaps the DMA of piece k.
class CopyPool {
public:
    static CopyPool& get() { static CopyPool p; return p; }
    // blocking parallel memcpy
    void copy(void* dst, const void* src, size_t n) {
        const size_t nparts = (n >= (8u << 20) && !th_.empty()) ? th_.size() : 1;
        if (nparts == 1) { memcpy(dst, src, n); return; }
        Job job; job.left = (int)nparts;
        const size_t per = ((n + nparts - 1) / nparts + 4095) & ~(size_t)4095;
        {
            std::lock_guard<std::mutex> lk(m_);
            for (size_t k = 0; k < nparts; ++k) {
                const size_t off = k * per;
                const size_t len = off >= n ? 0 : (n - off < per ? n - off : per);
                q_.push_back(Task{static_cast<uint8_t*>(dst) + off, static_cast<const uint8_t*>(src) + off, len, &job});
            }
        }
        cv_.notify_all();
        std::unique_lock<std::mutex> lk(m_);
        done_.wait(lk, [&] { return job.left == 0; });
    }
private:
    struct Job { int left; };
    struct Task { uint8_t* d; const uint8_t* s; size_t n; Job* job; };
    CopyPool() {
        unsigned hw = std::thread::hardware_concurrency();
        unsigned nt = hw >= 128 ? 32 : (hw >= 32 ? 16 : (hw >= 8 ? hw / 2 : 0));
        for (unsigned i = 0; i < nt; ++i) th_.emplace_back([this] { run(); });
    }
    ~CopyPool() {
        { std::lock_guard<std::mutex> lk(m_); stop_ = true; }
        cv_.notify_all();
        for (auto& t : th_) t.join();
    }
    void run() {
        for (;;) {
            Task t;
            {
                std::unique_lock<std::mutex> lk(m_);
                cv_.wait(lk, [&] { return stop_ || !q_.empty(); });
                if (stop_ && q_.empty()) return;
                t = q_.front(); q_.pop_front();
            }
            if (t.n) memcpy(t.d, t.s, t.n);
            {
                std::lock_guard<std::mutex> lk(m_);
                if (--t.job->left == 0) done_.notify_all();
            }
        }
    }
    std::vector<std::thread> th_;
    std::mutex m_;
    std::condition_variable cv_, done_;
    std::deque<Task> q_;
    bool stop_ = false;
};

constexpr size_t PIN_SLOT = 64u << 20;      // bytes per ring slot (= one chunk of the pipelined encode)
struct PinRing {
    uint8_t* slot[2] = {nullptr, nullptr};
    cudaEvent_t ev[2] = {nullptr, nullptr};  // DMA that last used the slot
    bool used[2] = {false, false};
    unsigned next = 0;
    cudaError_t ensure() {
        for (int k = 0; k < 2; ++k) {
            if (!slot[k]) { cudaError_t e = cudaHostAlloc(reinterpret_cast<void**>(&slot[k]), PIN_SLOT, cudaHostAllocDefault); if (e != cudaSuccess) return e; }
            if (!ev[k]) { cudaError_t e = cudaEventCreateWithFlags(&ev[k], cudaEventDisableTiming); if (e != cudaSuccess) return e; }
        }
        return cudaSuccess;
    }
    void release() {
        for (int k = 0; k < 2; ++k) { if (slot[k]) cudaFreeHost(slot[k]); if (ev[k]) cudaEventDestroy(ev[k]); slot[k] = nullptr; ev[k] = nullptr; used[k] = false; }
    }
};

static bool is_pageable_host(const void* p) {
    cudaPointerAttributes a;
    cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) { cudaGetLastError(); return true; }
    return a.type == cudaMemoryTypeUnregistered;
}
// host -> device, asynchronous on `s` for pinned sources; for pageable sources the host copies are done when it returns, the DMA is not
static cudaError_t h2d_any(PinRing& ring, uint8_t* dst_dev, const uint8_t* src, size_t n, cudaStream_t s, bool pageable) {
    if (!pageable) return cudaMemcpyAsync(dst_dev, src, n, cudaMemcpyHostToDevice, s);
    cudaError_t e = ring.ensure();
    for (size_t off = 0; off < n && e == cudaSuccess; off += PIN_SLOT) {
        const size_t len = n - off < PIN_SLOT ? n - off : PIN_SLOT;
        const unsigned k = ring.next++ & 1u;
        if (ring.used[k]) e = cudaEventSynchronize(ring.ev[k]);
        if (e != cudaSuccess) break;
        CopyPool::get().copy(ring.slot[k], src + off, len);
        e = cudaMemcpyAsync(dst_dev + off, ring.slot[k], len, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = cudaEventRecord(ring.ev[k], s);
        ring.used[k] = true;
    }
    return e;
}
// device -> host; synchronous for pageable destinations (returns when the bytes are in `dst`), asynchronous on `s` otherwise
static cudaError_t d2h_any(PinRing& ring, uint8_t* dst, const uint8_t* src_dev, size_t n, cudaStream_t s, bool pageable) {
    if (!pageable) return cudaMemcpyAsync(dst, src_dev, n, cudaMemcpyDeviceToHost, s);
    cudaError_t e = ring.ensure();
    size_t pend_off = 0, pend_len = 0; unsigned pend_k = 0; bool pending = false;
    for (size_t off = 0; off < n && e == cudaSuccess; off += PIN_SLOT) {
        const size_t len = n - off < PIN_SLOT ? n - off : PIN_SLOT;
        const unsigned k = ring.next++ & 1u;
        if (ring.used[k] && !(pending && pend_k == k)) e = cudaEventSynchronize(ring.ev[k]);
        if (e != cudaSuccess) break;
        e = cudaMemcpyAsync(ring.slot[k], src_dev + off, len, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaEventRecord(ring.ev[k], s);
        ring.used[k] = true;
        if (pending && e == cudaSuccess) {       // drain the previous piece while this one is in flight
            e = cudaEventSynchronize(ring.ev[pend_k]);
            if (e == cudaSuccess) CopyPool::get().copy(dst + pend_off, ring.slot[pend_k], pend_len);
        }
        pend_off = off; pend_len = len; pend_k = k; pending = true;
    }
    if (pending && e == cudaSuccess) {
        e = cudaEventSynchronize(ring.ev[pend_k]);
        if (e == cudaSuccess) CopyPool::get().copy(dst + pend_off, ring.slot[pend_k], pend_len);
    }
    return e;
}

struct DeviceCtx {
    int dev = -1;
    int num_sms = 0;
    bool ready = false;
    cudaStream_t stream = nullptr;     // for the synchronous host-pointer entry points (compute)
    cudaStream_t h2d_stream = nullptr, d2h_stream = nullptr;   // copy engines of the pipelined host path
    DevBuf ws, stage_in, stage_out, pipe_tables, dec_tables;
    DevBuf chee_tables[2][3];          // epoch-tagged run tables of the Cheetah / Lion encoders (zero at allocation, one entry format each)
    uint32_t chee_epoch = 0;
    uint64_t* h_sizes = nullptr;       // pinned, PIPE_MAX_CHUNKS entries
    cudaEvent_t ev_h2d[2] = {nullptr, nullptr};
    PinRing ring_in, ring_out;         // pinned staging of pageable host buffers
    uint64_t* d_size = nullptr;        // 8 B device
    uint64_t* h_size = nullptr;        // 8 B pinned
    ChamLayout layout{};
    int last_was_chameleon_fastpath_capable = 0;
    bool profile = false;              // record per-stage events (density_b200_profile_*)
    static constexpr int PROF_RING = 64;
    cudaEvent_t ev[PROF_RING][4] = {};
    uint64_t prof_count = 0;           // encodes recorded since profile_enable(1)
    // the diagnostics of the last run-parallel decodes, copied out of the workspace (which later calls reuse and may reallocate) behind
    // the decode: bytes 0-31 the 8 status words of the last run-parallel Cheetah decode, bytes 32-63 the 4 walk counts of the last Lion
    // decode. lion_stats_valid is cleared when a Lion decode runs on the in-order kernel
    DevBuf diag; bool chee_rounds_valid = false, lion_stats_valid = false;
    // One workspace per device: a call may only start using it when the previous call (on whatever stream) has finished with it (WsLease).
    cudaEvent_t ws_free = nullptr;
    bool ws_free_recorded = false;
    std::mutex mu;

    // frees everything the context owns and resets every flag, so that the next current_ctx() sets it up afresh (device dev is current)
    void release() {
        for (DevBuf* b : {&ws, &stage_in, &stage_out, &pipe_tables, &dec_tables, &diag}) b->release();
        for (auto& tables : chee_tables) for (DevBuf& b : tables) b.release();
        ring_in.release(); ring_out.release();
        for (cudaStream_t* s : {&stream, &h2d_stream, &d2h_stream}) { if (*s) cudaStreamDestroy(*s); *s = nullptr; }
        for (cudaEvent_t* e : {&ev_h2d[0], &ev_h2d[1], &ws_free}) { if (*e) cudaEventDestroy(*e); *e = nullptr; }
        for (auto& set : ev) for (cudaEvent_t& e : set) { if (e) cudaEventDestroy(e); e = nullptr; }
        if (d_size) cudaFree(d_size);
        for (void* p : {(void*)h_size, (void*)h_sizes}) if (p) cudaFreeHost(p);
        d_size = h_size = h_sizes = nullptr;
        chee_epoch = 0; layout = ChamLayout{}; last_was_chameleon_fastpath_capable = 0;
        profile = false; prof_count = 0;
        chee_rounds_valid = lion_stats_valid = ws_free_recorded = ready = false;
    }
};

constexpr int MAX_DEVICES = 64;
static DeviceCtx g_ctx[MAX_DEVICES];
static std::mutex g_ctx_mu;

static DeviceCtx* current_ctx() {
    int dev = -1;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) { set_error("cudaGetDevice", e); return nullptr; }
    if (dev < 0 || dev >= MAX_DEVICES) { set_error("device index out of range"); return nullptr; }
    DeviceCtx* c = &g_ctx[dev];
    std::lock_guard<std::mutex> lk(g_ctx_mu);
    if (!c->ready) {
        cudaDeviceProp prop;
        e = cudaGetDeviceProperties(&prop, dev);
        if (e != cudaSuccess) { set_error("cudaGetDeviceProperties", e); return nullptr; }
        if (prop.major != 9 || prop.minor != 0) { set_error("density_b200 is built for sm_90a and requires a compute capability 9.0 device (H100)"); return nullptr; }
        c->dev = dev;
        c->num_sms = prop.multiProcessorCount;
        e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->h2d_stream, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&c->d2h_stream, cudaStreamNonBlocking);
        if (e != cudaSuccess) { set_error("cudaStreamCreate", e); return nullptr; }
        e = cudaMalloc(&c->d_size, 64);
        if (e != cudaSuccess) { set_error("cudaMalloc", e); return nullptr; }
        e = cudaMallocHost(&c->h_size, 64);
        if (e == cudaSuccess) e = cudaMallocHost(&c->h_sizes, sizeof(uint64_t) * 4096);
        if (e != cudaSuccess) { set_error("cudaMallocHost", e); return nullptr; }
        e = cudaEventCreateWithFlags(&c->ws_free, cudaEventDisableTiming);
        if (e != cudaSuccess) { set_error("cudaEventCreate", e); return nullptr; }
        c->ready = true;
    }
    return c;
}

static size_t safe_size(int alg, size_t size) {  // codec/codec.rs:18-21
    const size_t B = alg_block_bytes(alg), S = alg_sig_bytes(alg);
    return size + (size / B) * S + ((size % B) ? S : 0);
}

static bool is_device_pointer(const void* p) {
    cudaPointerAttributes a;
    cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// The device's workspace, held by a call on `stream` for the lease's lifetime: the constructor makes the stream wait until the previous
// holder's work (on whatever stream) is done with it, the destructor records ws_free on the stream. ok is false, with the error set,
// when the wait could not be enqueued; then nothing is recorded.
struct WsLease {
    DeviceCtx* c; cudaStream_t stream; bool ok = true;
    WsLease(DeviceCtx* c_, cudaStream_t s) : c(c_), stream(s) {
        if (!c->ws_free_recorded) return;
        const cudaError_t e = cudaStreamWaitEvent(stream, c->ws_free, 0);
        if (e != cudaSuccess) { set_error("cudaStreamWaitEvent", e); ok = false; }
    }
    ~WsLease() { if (ok && cudaEventRecord(c->ws_free, stream) == cudaSuccess) c->ws_free_recorded = true; }
    WsLease(const WsLease&) = delete;
    WsLease& operator=(const WsLease&) = delete;
};

// path: 0 auto (fast path with exact fallback), 1 fast only (no fallback), 2 protected walk only, 3 scalar kernel
// path 4 (internal): Chameleon auto path for callers that may block on the stream (the synchronous reference-facing entry points): the
// copy-map iteration gets up to 12 more batches of 8 rounds before the in-order walk may take over
static int encode_device_locked(DeviceCtx* c, int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                uint64_t* d_out_size, cudaStream_t stream, int path) {
    const WsLease lease(c, stream);
    if (!lease.ok) return DENSITY_B200_ECUDA;
    uint64_t launches = 0;
    cudaError_t e;
    const bool aligned = !(reinterpret_cast<uintptr_t>(d_in) & 3) && !(reinterpret_cast<uintptr_t>(d_out) & 1);
    if (alg == ALG_CHAMELEON && path != 3 && aligned) {
        ChamLayout L;
        size_t need = cham_workspace_bytes(n, c->num_sms, &L);
        e = c->ws.ensure(need, stream);
        if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
        c->layout = L;
        if (path == 2) {
            e = cham_encode_protected_only(d_in, n, c->ws.p, L, d_out, cap, d_out_size, stream, &launches);
        } else {
            const uint32_t nruns = cham_pick_runs(n, c->num_sms);
            cudaEvent_t* ev = nullptr;
            if (c->profile) {
                ev = c->ev[c->prof_count % DeviceCtx::PROF_RING];
                for (int i = 0; i < 4; ++i) if (!ev[i]) cudaEventCreate(&ev[i]);
            }
            e = cham_encode_phase1(d_in, n, c->ws.p, L, nruns, nullptr, stream, &launches, ev);
            if (e == cudaSuccess && path == 4)
                e = cham_encode_phase2_blocking(d_in, n, c->ws.p, L, nruns, d_out, cap, d_out_size, 12, c->num_sms, stream, &launches);
            else if (e == cudaSuccess)
                e = cham_encode_phase2(d_in, n, c->ws.p, L, nruns, nullptr, d_out, cap, d_out_size, path == 0, false, c->num_sms, stream, &launches, ev);
            if (ev != nullptr && e == cudaSuccess) c->prof_count++;
        }
        c->last_was_chameleon_fastpath_capable = (path != 2);
    } else if ((alg == ALG_CHEETAH || alg == ALG_LION) && path != 3 && !(reinterpret_cast<uintptr_t>(d_in) & 3) && !(reinterpret_cast<uintptr_t>(d_out) & 1)) {
        // run-parallel Cheetah / Lion encoder; the exact in-order kernel is queued behind it and only runs if the copy map did not settle
        const size_t pw = (chee_workspace_bytes(n, c->num_sms) + 255) & ~(size_t)255;
        e = c->ws.ensure(pw + 256 + scalar_workspace_bytes(alg), stream);
        if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
        DevBuf* tb = c->chee_tables[alg == ALG_LION];
        for (int rg = 0; rg < 3 && e == cudaSuccess; ++rg) e = tb[rg].ensure(chee_tables_bytes(alg, rg, n, c->num_sms) + 256, stream);
        if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
        if (c->chee_epoch > 0x0FFFFF00u) {                 // epochs exhausted (2^23 calls): start over on cleared tables
            for (int a2 = 0; a2 < 2; ++a2) for (int rg = 0; rg < 3; ++rg)
                if (c->chee_tables[a2][rg].p) { e = cudaMemsetAsync(c->chee_tables[a2][rg].p, 0, c->chee_tables[a2][rg].bytes, stream); if (e != cudaSuccess) break; }
            if (e != cudaSuccess) { set_error("cudaMemsetAsync", e); return DENSITY_B200_ECUDA; }
            c->chee_epoch = 0;
        }
        uint32_t* d_conv = reinterpret_cast<uint32_t*>(c->ws.p + pw);
        uint8_t* const tabs[3] = {tb[0].p, tb[1].p, tb[2].p};
        // path 4 (callers that may block): read the verdict and resume the iteration up to 12 times before the in-order kernel takes over
        for (int attempt = 0; attempt <= (path == 4 ? 12 : 0); ++attempt) {
            if (attempt > 0) {
                uint32_t conv = 0;
                e = cudaMemcpyAsync(&conv, d_conv, sizeof conv, cudaMemcpyDeviceToHost, stream);
                if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
                if (e != cudaSuccess || conv) break;
            }
            const uint32_t epoch_base = c->chee_epoch + 1;
            c->chee_epoch += 32;
            e = chee_encode_parallel(alg, d_in, n, d_out, cap, c->ws.p, tabs, epoch_base, c->num_sms, d_out_size, d_conv, attempt > 0, stream, &launches);
            if (e != cudaSuccess) break;
        }
        if (e == cudaSuccess && path != 1)
            e = scalar_encode(alg, d_in, n, d_out, cap, c->ws.p + pw + 256, d_out_size, stream, &launches, d_conv);
        c->last_was_chameleon_fastpath_capable = 0;
    } else {
        if (reinterpret_cast<uintptr_t>(d_out) & 1) { set_error("encode_device: d_out must be 2-byte aligned"); return DENSITY_B200_EARG; }
        e = c->ws.ensure(scalar_workspace_bytes(alg), stream);
        if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
        e = scalar_encode(alg, d_in, n, d_out, cap, c->ws.p, d_out_size, stream, &launches);
        c->last_was_chameleon_fastpath_capable = 0;
    }
    return step_result(e, launches, "encode launch");
}

// path: 0 auto (parallel decoder with exact in-order fallback), 1 parallel only, 3 in-order kernel only
static int decode_device_locked(DeviceCtx* c, int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                uint64_t* d_out_size, cudaStream_t stream, int path) {
    const WsLease lease(c, stream);
    if (!lease.ok) return DENSITY_B200_ECUDA;
    uint64_t launches = 0;
    cudaError_t e;
    const bool parallel_ok = alg == ALG_CHAMELEON && path != 3 && !(reinterpret_cast<uintptr_t>(d_in) & 1) && !(reinterpret_cast<uintptr_t>(d_out) & 3);
    if (parallel_ok) {
        // parallel decoder; the exact in-order kernel is queued behind it and only runs when the stream has copy-mode blocks
        const size_t pw = (cham_decode_workspace_bytes(n, cap, c->num_sms) + 255) & ~(size_t)255;
        e = c->ws.ensure(pw + 256 + scalar_workspace_bytes(alg), stream);
        if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
        uint32_t* d_nonquiet = reinterpret_cast<uint32_t*>(c->ws.p + pw);
        e = cham_decode_parallel(d_in, n, d_out, cap, c->ws.p, c->num_sms, d_out_size, d_nonquiet, stream, &launches);
        if (e == cudaSuccess && path != 1)
            e = scalar_decode(alg, d_in, n, d_out, cap, c->ws.p + pw + 256, d_out_size, stream, &launches, d_nonquiet);
        return step_result(e, launches, "decode launch");
    }
    if ((alg == ALG_CHEETAH || alg == ALG_LION) && path != 3 && !(reinterpret_cast<uintptr_t>(d_in) & 1) && !(reinterpret_cast<uintptr_t>(d_out) & 3)) {
        // run-parallel Cheetah decoder / parallel Lion decoder (cl_decode.cu) + in-order tail; the exact in-order kernel is queued behind
        // it and only runs on a boundary error or (Cheetah) if the context iteration did not settle within its round budget
        const bool lion = alg == ALG_LION;
        const size_t pw = ((lion ? lion_decode_workspace_bytes(n, cap, c->num_sms) : chee_decode_workspace_bytes(n, cap, c->num_sms)) + 255) & ~(size_t)255;
        e = c->ws.ensure(pw + 256 + 2 * ((scalar_workspace_bytes(alg) + 255) & ~(size_t)255), stream);
        if (e == cudaSuccess) e = c->dec_tables.ensure(chee_decode_tables_bytes(n, c->num_sms, lion) + 256, stream);
        if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
        uint32_t* d_fallback = reinterpret_cast<uint32_t*>(c->ws.p + pw);
        uint8_t* tail_ws = c->ws.p + pw + 256;
        uint8_t* scalar_ws = tail_ws + ((scalar_workspace_bytes(alg) + 255) & ~(size_t)255);
        e = cudaMemsetAsync(tail_ws, 0, 256, stream);
        if (e == cudaSuccess)
            e = (lion ? lion_decode_parallel : chee_decode_parallel)(d_in, n, d_out, cap, c->ws.p, c->dec_tables.p, tail_ws, c->num_sms, d_out_size, d_fallback,
                                                                     stream, &launches);
        if (e == cudaSuccess) {
            const void* cl_st = nullptr;
            const void* b_st = (lion ? lion_decode_status_ptr : chee_decode_status_ptr)(c->ws.p, n, cap, c->num_sms, &cl_st);
            e = scalar_decode_tail(alg, d_in, n, d_out, cap, tail_ws, b_st, cl_st, d_out_size, stream, &launches, d_fallback);
            const size_t at = lion ? 32 : 0;   // Cheetah: the 8 status words at the block's start; Lion: the 4 walk counts at byte 32
            if (e == cudaSuccess) e = c->diag.ensure(64, stream);
            if (e == cudaSuccess) e = cudaMemcpyAsync(c->diag.p + at, static_cast<const uint8_t*>(cl_st) + at, 32, cudaMemcpyDeviceToDevice, stream);
            (lion ? c->lion_stats_valid : c->chee_rounds_valid) = e == cudaSuccess;
        }
        if (e == cudaSuccess && path != 1)
            e = scalar_decode(alg, d_in, n, d_out, cap, scalar_ws, d_out_size, stream, &launches, d_fallback);
        return step_result(e, launches, "decode launch");
    }
    if (alg == ALG_LION) c->lion_stats_valid = false;
    e = c->ws.ensure(scalar_workspace_bytes(alg), stream);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    e = scalar_decode(alg, d_in, n, d_out, cap, c->ws.p, d_out_size, stream, &launches);
    return step_result(e, launches, "decode launch");
}

// Host-pointer Chameleon encode, pipelined over PCIe: the input is cut into chunks that are treated as shards of one
// bit-exact stream (same mechanism as the multi-GPU path): while chunk i+1 is still crossing PCIe, chunk i runs
// phase 1 (flags) + phase 2 (carry-in from the chunks before it, scan, emit) and chunk i-1's output travels back.
// Returns bytes written, 0 on error, or (size_t)-1 when the stream turned out not to be "quiet" (caller falls back
// to the whole-buffer path with the protection-aware walk; the input is already resident in stage_in).
constexpr size_t PIPE_CHUNK = 64u << 20;
constexpr size_t PIPE_MIN_BYTES = 96u << 20;

// The pipeline runs on the device's one workspace like every other call: it waits on c->stream for the calls enqueued before it (on
// whatever stream) and releases the workspace on every exit, the "not quiet" one included (the fallback then acquires it again).
static size_t chameleon_encode_host_pipelined(DeviceCtx* c, const uint8_t* in, size_t n, uint8_t* out, size_t out_cap) {
    const WsLease lease(c, c->stream);
    if (!lease.ok) return 0;
    const size_t nchunks = (n + PIPE_CHUNK - 1) / PIPE_CHUNK;
    if (nchunks > 4096) return (size_t)-1;
    cudaError_t e = c->stage_in.ensure(n + 16, c->h2d_stream);
    if (e == cudaSuccess) e = c->stage_out.ensure(safe_size(ALG_CHAMELEON, n) + 16, c->stream);
    if (e == cudaSuccess) e = c->pipe_tables.ensure(2 * 65536 * sizeof(uint32_t) + (nchunks + 1) * sizeof(uint64_t) + 256, c->stream);
    ChamLayout L;
    if (e == cudaSuccess) e = c->ws.ensure(cham_workspace_bytes(PIPE_CHUNK, c->num_sms, &L), c->stream);
    if (e != cudaSuccess) { set_error("pipeline cudaMalloc", e); return 0; }
    c->layout = L;
    uint32_t* d_acc = reinterpret_cast<uint32_t*>(c->pipe_tables.p);            // dictionary before the current chunk
    uint32_t* d_tab = d_acc + 65536;                                              // last-writer table of the current chunk
    uint64_t* d_sizes = reinterpret_cast<uint64_t*>(c->pipe_tables.p + 2 * 65536 * sizeof(uint32_t));
    uint32_t* d_flag = reinterpret_cast<uint32_t*>(d_sizes + nchunks);
    for (int k = 0; k < 2; ++k) if (!c->ev_h2d[k]) cudaEventCreateWithFlags(&c->ev_h2d[k], cudaEventDisableTiming);
    uint64_t launches = 0;
    // pinned input: all H2D copies are queued up front on the copy stream, one event per chunk. Pageable input: chunk 0 is staged
    // now, chunk i + 1 while the GPU works on chunk i (the host copy into the pinned ring is the slow part)
    const bool pg_in = is_pageable_host(in), pg_out = is_pageable_host(out);
    std::vector<cudaEvent_t> evs(nchunks, nullptr);
    bool ok = true;
    auto stage_chunk = [&](size_t i) {
        const size_t off = i * PIPE_CHUNK, len = (n - off < PIPE_CHUNK) ? (n - off) : PIPE_CHUNK;
        ok = h2d_any(c->ring_in, c->stage_in.p + off, in + off, len, c->h2d_stream, pg_in) == cudaSuccess;
        if (ok) ok = cudaEventCreateWithFlags(&evs[i], cudaEventDisableTiming) == cudaSuccess;
        if (ok) ok = cudaEventRecord(evs[i], c->h2d_stream) == cudaSuccess;
    };
    size_t staged = 0;
    for (; staged < (pg_in ? (size_t)1 : nchunks) && ok; ++staged) stage_chunk(staged);
    size_t out_off = 0;
    bool nonquiet = false;
    e = cudaMemsetAsync(d_flag, 0, sizeof(uint32_t), c->stream);
    if (ok && e == cudaSuccess) e = cham_table_init(d_acc, c->stream, &launches);
    for (size_t i = 0; i < nchunks && ok && e == cudaSuccess; ++i) {
        const size_t off = i * PIPE_CHUNK, len = (n - off < PIPE_CHUNK) ? (n - off) : PIPE_CHUNK;
        const uint32_t nruns = cham_pick_runs(len, c->num_sms);
        e = cudaStreamWaitEvent(c->stream, evs[i], 0);
        if (e == cudaSuccess) e = cham_encode_phase1(c->stage_in.p + off, len, c->ws.p, L, nruns, d_tab, c->stream, &launches);
        if (e == cudaSuccess) e = cham_encode_phase2(c->stage_in.p + off, len, c->ws.p, L, nruns, i ? d_acc : nullptr, c->stage_out.p + out_off,
                                                     c->stage_out.bytes - out_off, d_sizes + i, false, i != 0, c->num_sms, c->stream, &launches);
        if (e == cudaSuccess) e = cham_status_accumulate(c->ws.p, L, d_flag, c->stream, &launches);
        if (e == cudaSuccess) e = cham_table_fold(d_acc, d_tab, c->stream, &launches);
        if (e == cudaSuccess) e = cudaMemcpyAsync(c->h_sizes + i, d_sizes + i, sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(c->h_size, d_flag, sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream);
        if (e == cudaSuccess && pg_in && staged < nchunks) { stage_chunk(staged); ++staged; }
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);   // chunk i done; later H2D copies keep flowing meanwhile
        if (e != cudaSuccess) break;
        if (*reinterpret_cast<uint32_t*>(c->h_size) != 0) { nonquiet = true; break; }
        const uint64_t sz = c->h_sizes[i];
        if (sz == 0) { ok = false; set_error("pipelined encode: device reported an error"); break; }
        if (out_off + sz > out_cap) { ok = false; set_error("output buffer too small"); break; }
        e = d2h_any(c->ring_out, out + out_off, c->stage_out.p + out_off, sz, c->d2h_stream, pg_out);
        out_off += sz;
    }
    g_launches += launches;
    if (nonquiet) for (; staged < nchunks && ok; ++staged) stage_chunk(staged);   // the fallback wants the whole input in stage_in
    cudaError_t e2 = cudaStreamSynchronize(c->h2d_stream);
    cudaError_t e3 = cudaStreamSynchronize(c->d2h_stream);
    for (auto ev : evs) if (ev) cudaEventDestroy(ev);
    if (e != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess) { set_error("pipelined encode", e != cudaSuccess ? e : (e2 != cudaSuccess ? e2 : e3)); return 0; }
    if (!ok) return 0;
    if (nonquiet) return (size_t)-1;
    c->last_was_chameleon_fastpath_capable = 2;   // pipelined: quiet by construction
    return out_off;
}

constexpr size_t OWN_OUTPUT = ~(size_t)0;   // SyncCall::run's stage_cap: the entry writes the caller's output itself

// The frame of the synchronous host-or-device entries (the nine symbols, codec instances, decoded size, range decode). Constructing it
// takes the context and its lock, and synchronises the device when a buffer is on it: the call cannot know which stream produced or
// reads a device buffer. c is NULL, with the error set, when either fails.
struct SyncCall {
    DeviceCtx* c = current_ctx();
    std::unique_lock<std::mutex> lk;
    bool in_dev = false, out_dev = false;
    const uint8_t* staged_in = nullptr;    // the input, when the entry has already put it in stage_in
    SyncCall(const void* in, const void* out) {
        if (!c) return;
        lk = std::unique_lock<std::mutex>(c->mu);
        in_dev = is_device_pointer(in);
        out_dev = is_device_pointer(out);
        const cudaError_t e = in_dev || out_dev ? cudaDeviceSynchronize() : cudaSuccess;
        if (e != cudaSuccess) { set_error("cudaDeviceSynchronize", e); c = nullptr; }
    }
    // Stages the input: a host input through the pinned ring, and with stage_odd a device input at an odd address copied into stage_in
    // (otherwise the kernels read a device input where it is). A host output is staged in stage_out, stage_cap bytes, unless stage_cap is
    // OWN_OUTPUT. Then enqueue(d_in, d_out, d_cap) on c->stream, and the k result words at c->d_size are read back into c->h_size. A
    // staged output gets c->h_size[0] bytes when that is in (0, out_cap]. Returns DENSITY_B200_OK, or an error code with the error set.
    template <class F>
    int run(const uint8_t* in, size_t n, bool stage_odd, uint8_t* out, size_t out_cap, size_t stage_cap, int k, F enqueue) {
        cudaError_t e = cudaSuccess;
        const uint8_t* d_in = staged_in ? staged_in : in;
        if (!staged_in && (!in_dev || (stage_odd && (reinterpret_cast<uintptr_t>(in) & 1)))) {
            e = c->stage_in.ensure(n + 16, c->stream);
            if (e != cudaSuccess) { set_error("staging cudaMalloc", e); return DENSITY_B200_ECUDA; }
            e = in_dev ? cudaMemcpyAsync(c->stage_in.p, in, n, cudaMemcpyDeviceToDevice, c->stream)
                       : h2d_any(c->ring_in, c->stage_in.p, in, n, c->stream, is_pageable_host(in));
            if (e != cudaSuccess) { set_error("input copy", e); return DENSITY_B200_ECUDA; }
            d_in = c->stage_in.p;
        }
        const bool stage_out = !out_dev && stage_cap != OWN_OUTPUT;
        if (stage_out) {
            e = c->stage_out.ensure(stage_cap + 16, c->stream);
            if (e != cudaSuccess) { set_error("staging cudaMalloc", e); return DENSITY_B200_ECUDA; }
        }
        const int rc = stage_out ? enqueue(d_in, c->stage_out.p, stage_cap) : enqueue(d_in, out, out_cap);
        if (rc != DENSITY_B200_OK) { cudaStreamSynchronize(c->stream); return rc; }
        e = cudaMemcpyAsync(c->h_size, c->d_size, k * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        if (e != cudaSuccess) { set_error("stream sync", e); return DENSITY_B200_ECUDA; }
        const uint64_t produced = c->h_size[0];
        if (!stage_out || produced == 0 || produced > out_cap) return DENSITY_B200_OK;
        e = d2h_any(c->ring_out, out, c->stage_out.p, produced, c->stream, is_pageable_host(out));
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        if (e != cudaSuccess) { set_error("D2H copy", e); return DENSITY_B200_ECUDA; }
        return DENSITY_B200_OK;
    }
};

// what a synchronous encode or decode returns: the bytes it wrote (the result word), or 0 with the error set
static size_t sync_bytes(int rc, const DeviceCtx* c, bool encode, size_t out_cap) {
    if (rc != DENSITY_B200_OK) return 0;
    const uint64_t produced = c->h_size[0];
    if (produced == 0) { set_error(encode ? "encode failed on device (output capacity?)" : "decode failed on device (malformed stream or output capacity)"); return 0; }
    if (produced > out_cap) { set_error("output buffer too small"); return 0; }
    return (size_t)produced;
}

// Synchronous entry point shared by the nine reference-shaped symbols.
static size_t run_sync(bool encode, int alg, const uint8_t* in, size_t n, uint8_t* out, size_t out_cap) {
    g_last_error.clear();
    if ((!in && n) || (!out && out_cap)) { set_error("null pointer"); return 0; }
    if (n == 0) return 0;  // Codec::encode/decode of an empty slice writes nothing (codec.rs:76,102)
    SyncCall f(in, out);
    if (!f.c) return 0;
    if (encode && alg == ALG_CHAMELEON && !f.in_dev && !f.out_dev && n >= PIPE_MIN_BYTES) {
        const size_t r = chameleon_encode_host_pipelined(f.c, in, n, out, out_cap);
        if (r != (size_t)-1) return r;
        f.staged_in = f.c->stage_in.p;   // not quiet: the whole input is already in stage_in; redo with the protection-aware fallback
    }
    // encode: stage into a full safe-size buffer and check the real size against the caller's capacity afterwards
    // (the reference only fails when the bytes actually written exceed the slice, write_buffer.rs:19)
    const int rc = f.run(in, n, false, out, out_cap, encode ? safe_size(alg, n) : out_cap, 1, [&](const uint8_t* d_in, uint8_t* d_out, size_t d_cap) {
        return encode ? encode_device_locked(f.c, alg, d_in, n, d_out, d_cap, f.c->d_size, f.c->stream, 4)
                      : decode_device_locked(f.c, alg, d_in, n, d_out, d_cap, f.c->d_size, f.c->stream, 0);
    });
    return sync_bytes(rc, f.c, encode, out_cap);
}

// The prologue of the stream-ordered entries (encode / decode, decoded size, range decode): the error cleared and the arguments checked
// (d_in and d_out NULL only when their lengths are 0, d_in in_align-byte aligned, the k result words at d_result not NULL and 8-byte
// aligned), then the context taken and locked. An empty call zeroes the result words with a memset and launches nothing; otherwise
// enqueue(c, stream) enqueues the call.
template <class F>
static int stream_entry(const uint8_t* d_in, size_t n, const uint8_t* d_out, size_t cap, uint64_t* d_result, int k, uintptr_t in_align,
                        bool empty, void* stream, F enqueue) {
    g_last_error.clear();
    if (!d_result || (!d_in && n) || (!d_out && cap)) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if ((reinterpret_cast<uintptr_t>(d_in) & (in_align - 1)) || (reinterpret_cast<uintptr_t>(d_result) & 7)) {
        set_error("misaligned pointer: d_out_size / d_result must be 8-byte aligned, and d_in 2-byte for decoded size and range decode");
        return DENSITY_B200_EARG;
    }
    DeviceCtx* c = current_ctx();
    if (!c) return DENSITY_B200_ECUDA;
    std::lock_guard<std::mutex> lk(c->mu);
    const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (!empty) return enqueue(c, s);
    const cudaError_t e = cudaMemsetAsync(d_result, 0, k * sizeof(uint64_t), s);
    if (e != cudaSuccess) { set_error("memset", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}

}  // namespace dns

using namespace dns;

extern "C" {

/* diagnostic: the device-side status block of the last parallel Chameleon decode on the current device (synchronises) */
int density_b200_decode_status(uint64_t* out10) {
    DeviceCtx* c = current_ctx();
    if (!c || !c->ws.p) return DENSITY_B200_EARG;
    std::lock_guard<std::mutex> lk(c->mu);
    unsigned char raw[64] = {0};
    if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpy(raw, c->ws.p, sizeof(raw), cudaMemcpyDeviceToHost) != cudaSuccess) return DENSITY_B200_ECUDA;
    const unsigned long long* q = reinterpret_cast<const unsigned long long*>(raw);
    const unsigned int* w = reinterpret_cast<const unsigned int*>(raw + 24);
    out10[0] = q[0]; out10[1] = q[1]; out10[2] = q[2];               // out_bytes, main_blocks, tail_off
    for (int k = 0; k < 7; ++k) out10[3 + k] = w[k];                 // nonquiet, error, last_main_inc, seq, ps_penalty, ps_start, ps_prev
    return DENSITY_B200_OK;
}

size_t chameleon_encode(const uint8_t* i, size_t n, uint8_t* o, size_t c) { return run_sync(true, ALG_CHAMELEON, i, n, o, c); }
size_t chameleon_decode(const uint8_t* i, size_t n, uint8_t* o, size_t c) { return run_sync(false, ALG_CHAMELEON, i, n, o, c); }
size_t chameleon_safe_encode_buffer_size(size_t s) { return safe_size(ALG_CHAMELEON, s); }
size_t cheetah_encode(const uint8_t* i, size_t n, uint8_t* o, size_t c) { return run_sync(true, ALG_CHEETAH, i, n, o, c); }
size_t cheetah_decode(const uint8_t* i, size_t n, uint8_t* o, size_t c) { return run_sync(false, ALG_CHEETAH, i, n, o, c); }
size_t cheetah_safe_encode_buffer_size(size_t s) { return safe_size(ALG_CHEETAH, s); }
size_t lion_encode(const uint8_t* i, size_t n, uint8_t* o, size_t c) { return run_sync(true, ALG_LION, i, n, o, c); }
size_t lion_decode(const uint8_t* i, size_t n, uint8_t* o, size_t c) { return run_sync(false, ALG_LION, i, n, o, c); }
size_t lion_safe_encode_buffer_size(size_t s) { return safe_size(ALG_LION, s); }

static int device_entry(bool encode, int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                        void* stream, int path) {
    if (alg < 0 || alg > 2) { set_error("bad algorithm id"); return DENSITY_B200_EARG; }
    return stream_entry(d_in, n, d_out, cap, d_out_size, 1, 1, n == 0, stream, [&](DeviceCtx* c, cudaStream_t s) {
        return encode ? encode_device_locked(c, alg, d_in, n, d_out, cap, d_out_size, s, path)
                      : decode_device_locked(c, alg, d_in, n, d_out, cap, d_out_size, s, path);
    });
}

int density_b200_encode_device(int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size, void* stream) {
    return device_entry(true, alg, d_in, n, d_out, cap, d_out_size, stream, 0);
}
int density_b200_decode_device(int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size, void* stream) {
    return device_entry(false, alg, d_in, n, d_out, cap, d_out_size, stream, 0);
}
int density_b200_encode_device_path(int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                    void* stream, int path) {
    if (path < 0 || path > 4) { set_error("bad path"); return DENSITY_B200_EARG; }
    return device_entry(true, alg, d_in, n, d_out, cap, d_out_size, stream, path);
}
int density_b200_decode_device_path(int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                    void* stream, int path) {
    if (path != 0 && path != 1 && path != 3) { set_error("bad path"); return DENSITY_B200_EARG; }
    return device_entry(false, alg, d_in, n, d_out, cap, d_out_size, stream, path);
}

// ---- decoded size (decoded_size.cu) -------------------------------------------------------------------------------------------
// n > 0, d_in 2-byte aligned; on the device's workspace like decode_device
static int decoded_size_locked(DeviceCtx* c, int alg, const uint8_t* d_in, size_t n, uint64_t* d_result, cudaStream_t stream) {
    const WsLease lease(c, stream);
    if (!lease.ok) return DENSITY_B200_ECUDA;
    uint64_t launches = 0;
    cudaError_t e = c->ws.ensure(decoded_size_workspace_bytes(alg, n), stream);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    e = decoded_size_launch(alg, d_in, n, c->ws.p, d_result, stream, &launches);
    return step_result(e, launches, "decoded size launch");
}

int density_b200_decoded_size_device(int alg, const uint8_t* d_in, size_t n, uint64_t* d_result, void* stream) {
    if (alg < 0 || alg > 2) { set_error("bad algorithm id"); return DENSITY_B200_EARG; }
    // n == 0: an empty stream decodes to nothing (codec.rs:102)
    return stream_entry(d_in, n, nullptr, 0, d_result, 2, 2, n == 0, stream, [&](DeviceCtx* c, cudaStream_t s) {
        return decoded_size_locked(c, alg, d_in, n, d_result, s);
    });
}

int density_b200_decoded_size(int alg, const uint8_t* input, size_t n, uint64_t* out_size) {
    g_last_error.clear();
    if (alg < 0 || alg > 2) { set_error("bad algorithm id"); return DENSITY_B200_EARG; }
    if (!out_size || (!input && n)) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (n == 0) { *out_size = 0; return DENSITY_B200_OK; }
    SyncCall f(input, nullptr);
    if (!f.c) return DENSITY_B200_ECUDA;
    const int rc = f.run(input, n, true, nullptr, 0, OWN_OUTPUT, 2, [&](const uint8_t* d_in, uint8_t*, size_t) {
        return decoded_size_locked(f.c, alg, d_in, n, f.c->d_size, f.c->stream);
    });
    if (rc != DENSITY_B200_OK) return rc;
    if (f.c->h_size[1] != 0) { set_error("malformed stream: the decoder would read past its end"); return DENSITY_B200_EMALFORMED; }
    *out_size = f.c->h_size[0];
    return DENSITY_B200_OK;
}

// ---- Chameleon range decode (decode_range.cu) --------------------------------------------------------------------------------------
// n > 0, len > 0, d_in 2-byte aligned; on the device's workspace like decode_device. The locate step runs first and the host waits for
// it on `stream` (the pieces' lengths size the rest); then the pieces are decoded and the w window bytes copied to out: device memory
// (d_out) or, out_host, host memory (the synchronous entry). d_result receives {w, S, verdict} in stream order.
static int range_locked(DeviceCtx* c, const uint8_t* d_in, size_t n, uint64_t first, uint64_t len, uint8_t* out, bool out_host,
                        uint64_t* d_result, cudaStream_t stream) {
    const WsLease lease(c, stream);
    if (!lease.ok) return DENSITY_B200_ECUDA;
    uint64_t launches = 0;
    const char* what = "range decode locate";
    cudaError_t e = c->ws.ensure(range_locate_workspace_bytes(n), stream);
    if (e == cudaSuccess) e = range_locate_launch(d_in, n, first, len, c->ws.p, d_result, stream, &launches);
    if (e == cudaSuccess) e = cudaMemcpyAsync(c->h_size, c->ws.p, RANGE_REPORT_WORDS * sizeof(uint64_t), cudaMemcpyDeviceToHost, stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    RangePlan p{};
    bool planned = false;
    if (e == cudaSuccess) planned = range_plan(c->h_size, n, first, c->num_sms, &p);
    if (e == cudaSuccess && planned && p.w) {
        const uint8_t* window = nullptr;
        what = "range decode workspace";
        e = c->ws.ensure(p.ws_bytes, stream);
        if (e == cudaSuccess) { what = "range decode launch"; e = range_decode_launch(d_in, p, c->ws.p, c->num_sms, stream, &launches, &window); }
        if (e == cudaSuccess) {
            what = "range decode window copy";
            e = out_host ? d2h_any(c->ring_out, out, window, p.w, stream, is_pageable_host(out))
                         : cudaMemcpyAsync(out, window, p.w, cudaMemcpyDeviceToDevice, stream);
        }
    }
    const int rc = step_result(e, launches, what);
    if (rc == DENSITY_B200_OK && !planned) { set_error("range decode: the locate step's report is inconsistent"); return DENSITY_B200_ECUDA; }
    return rc;
}

int density_b200_chameleon_decode_range_device(const uint8_t* d_in, size_t n, uint64_t first, uint64_t len, uint8_t* d_out, uint64_t* d_result,
                                               void* stream) {
    // n == 0 or len == 0: nothing to write (codec.rs:102 for an empty stream)
    return stream_entry(d_in, n, d_out, len, d_result, 3, 2, n == 0 || len == 0, stream, [&](DeviceCtx* c, cudaStream_t s) {
        return range_locked(c, d_in, n, first, len, d_out, false, d_result, s);
    });
}

int density_b200_chameleon_decode_range(const uint8_t* input, size_t n, uint64_t first, uint8_t* output, uint64_t len, uint64_t* written) {
    g_last_error.clear();
    if (!written || (!input && n) || (!output && len)) { set_error("null pointer"); return DENSITY_B200_EARG; }
    *written = 0;
    if (n == 0 || len == 0) return DENSITY_B200_OK;
    SyncCall f(input, output);
    if (!f.c) return DENSITY_B200_ECUDA;
    const int rc = f.run(input, n, true, output, len, OWN_OUTPUT, 3, [&](const uint8_t* d_in, uint8_t* out, size_t) {
        return range_locked(f.c, d_in, n, first, len, out, !f.out_dev, f.c->d_size, f.c->stream);
    });
    if (rc != DENSITY_B200_OK) return rc;
    if (f.c->h_size[2] != 0) { set_error("malformed stream: the decoder would read past its end"); return DENSITY_B200_EMALFORMED; }
    *written = f.c->h_size[0];
    return DENSITY_B200_OK;
}

// ---- Chameleon seek index (decode_range.cu) -----------------------------------------------------------------------------------------
// n > 0, d_in 2-byte aligned, a valid interval. The locate step runs first and the host waits for it (the pieces' lengths size the
// rest); then, on a well-formed stream, the index is written to `at` (device, 4-byte aligned) and, when out is set, copied from there to
// out: host memory (out_host) or device memory of any alignment. h3 = {index bytes, S, verdict}; d_result receives the same.
static int index_build_locked(DeviceCtx* c, const uint8_t* d_in, size_t n, uint64_t interval, uint8_t* at, uint8_t* out, bool out_host,
                              uint64_t* d_result, cudaStream_t stream, uint64_t h3[3]) {
    const WsLease lease(c, stream);
    if (!lease.ok) return DENSITY_B200_ECUDA;
    uint64_t launches = 0;
    const char* what = "index build locate";
    std::vector<uint64_t> rep(index_report_bytes(index_max_count(n, interval)) / sizeof(uint64_t));
    cudaError_t e = c->ws.ensure(index_locate_workspace_bytes(n, interval), stream);
    if (e == cudaSuccess) e = index_locate_launch(d_in, n, interval, c->ws.p, d_result, rep.data(), stream, &launches);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
    bool planned = false;
    if (e == cudaSuccess) {
        for (int k = 0; k < 3; ++k) h3[k] = rep[k];
        size_t ws_bytes = 0;
        planned = index_build_plan(rep.data(), n, c->num_sms, &ws_bytes);
        if (planned && !rep[2]) {
            what = "index build workspace";
            e = c->ws.ensure(ws_bytes, stream);
            if (e == cudaSuccess) { what = "index build launch"; e = index_build_launch(d_in, rep.data(), c->ws.p, at, c->num_sms, stream, &launches); }
            if (e == cudaSuccess && out) {
                what = "index copy";
                e = out_host ? d2h_any(c->ring_out, out, at, rep[0], stream, is_pageable_host(out))
                             : cudaMemcpyAsync(out, at, rep[0], cudaMemcpyDeviceToDevice, stream);
            }
        }
    }
    const int rc = step_result(e, launches, what);
    if (rc != DENSITY_B200_OK) return rc;
    if (rep[2]) { set_error("malformed stream: the decoder would read past its end"); return DENSITY_B200_EMALFORMED; }
    if (!planned) { set_error("index build: the locate step's report is inconsistent"); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}

// The header and the directory of an index of index_len bytes at `index` (host or device; a device index is read on `stream`, with one
// wait) into hdr, checked against the stream length. DENSITY_B200_EARG with the error set when they do not describe a valid index.
static int index_read(const uint8_t* index, bool index_dev, size_t index_len, size_t n, cudaStream_t stream, std::vector<uint64_t>* hdr) {
    const uint64_t count = index_count_for_bytes(index_len);
    if (count == ~0ull || count > index_max_count(n, 256)) { set_error("index_len is not the length of an index of this stream"); return DENSITY_B200_EARG; }
    hdr->assign(cidx_snapshots_at(count) / sizeof(uint64_t), 0);
    if (index_dev) {
        cudaError_t e = cudaMemcpyAsync(hdr->data(), index, cidx_snapshots_at(count), cudaMemcpyDeviceToHost, stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
        if (e != cudaSuccess) { set_error("index directory copy", e); return DENSITY_B200_ECUDA; }
    } else {
        memcpy(hdr->data(), index, cidx_snapshots_at(count));
    }
    if (const char* why = index_check(hdr->data(), n, index_len, count)) { set_error(why); return DENSITY_B200_EARG; }
    return DENSITY_B200_OK;
}

// The decode of an indexed piece (d_piece: the piece's first byte, 2-byte aligned) and the checked copy of the window to d_out (device,
// any alignment), on the device's workspace. snap: the carry-in snapshot, NULL at the stream start; snap_copy: it is in host memory or
// misaligned, and is staged in the workspace first. With p.w == 0 only the result words {0, S, 0} are written.
static int range_indexed_locked(DeviceCtx* c, const uint8_t* d_piece, RangePlan p, const uint8_t* snap, bool snap_copy, uint64_t size,
                                uint8_t* d_out, uint64_t* d_result, cudaStream_t stream) {
    const WsLease lease(c, stream);
    if (!lease.ok) return DENSITY_B200_ECUDA;
    uint64_t launches = 0;
    const uint8_t* window = nullptr;
    cudaError_t e = c->ws.ensure(p.ws_bytes, stream);
    if (e == cudaSuccess && p.w && snap) {
        p.carry_in = snap_copy ? range_table_slot(c->ws.p) : reinterpret_cast<const uint32_t*>(snap);
        if (snap_copy) e = cudaMemcpyAsync(range_table_slot(c->ws.p), snap, CIDX_SNAPSHOT_BYTES, cudaMemcpyDefault, stream);
    }
    if (e == cudaSuccess && p.w) e = range_decode_launch(d_piece, p, c->ws.p, c->num_sms, stream, &launches, &window);
    if (e == cudaSuccess) e = index_copy_out_launch(p, window, size, d_out, c->ws.p, d_result, c->num_sms, stream, &launches);
    return step_result(e, launches, "indexed range decode launch");
}

// the snapshot an indexed piece starts from (NULL: the stream start)
static const uint8_t* index_snapshot(const uint8_t* index, const std::vector<uint64_t>& hdr, uint64_t j) {
    return j ? index + cidx_snapshots_at(hdr[CIDX_COUNT_W]) + (j - 1) * CIDX_SNAPSHOT_BYTES : nullptr;
}

uint64_t density_b200_chameleon_index_bytes(size_t n, uint64_t interval) {
    return (interval < 256 || interval % 256) ? 0 : cidx_bytes(index_max_count(n, interval));
}

int density_b200_chameleon_index_build_device(const uint8_t* d_in, size_t n, uint64_t interval, uint8_t* d_index, size_t index_cap,
                                              uint64_t* d_result, void* stream) {
    g_last_error.clear();
    if (n == 0) { set_error("index build: an empty stream has nothing to index"); return DENSITY_B200_EARG; }
    if (!density_b200_chameleon_index_bytes(n, interval)) { set_error("index build: interval must be a positive multiple of 256"); return DENSITY_B200_EARG; }
    if (index_cap < density_b200_chameleon_index_bytes(n, interval)) { set_error("index build: index_cap < density_b200_chameleon_index_bytes(n, interval)"); return DENSITY_B200_EARG; }
    if (reinterpret_cast<uintptr_t>(d_index) & 3) { set_error("index build: d_index must be 4-byte aligned"); return DENSITY_B200_EARG; }
    return stream_entry(d_in, n, d_index, index_cap, d_result, 3, 2, false, stream, [&](DeviceCtx* c, cudaStream_t s) {
        uint64_t h3[3];
        return index_build_locked(c, d_in, n, interval, d_index, nullptr, false, d_result, s, h3);
    });
}

int density_b200_chameleon_index_build(const uint8_t* input, size_t n, uint64_t interval, uint8_t* index, size_t index_cap, uint64_t* index_len) {
    g_last_error.clear();
    if (!index_len || !input || !index) { set_error("null pointer"); return DENSITY_B200_EARG; }
    *index_len = 0;
    if (n == 0) { set_error("index build: an empty stream has nothing to index"); return DENSITY_B200_EARG; }
    const uint64_t bound = density_b200_chameleon_index_bytes(n, interval);
    if (!bound) { set_error("index build: interval must be a positive multiple of 256"); return DENSITY_B200_EARG; }
    if (index_cap < bound) { set_error("index build: index_cap < density_b200_chameleon_index_bytes(n, interval)"); return DENSITY_B200_EARG; }
    SyncCall f(input, index);
    if (!f.c) return DENSITY_B200_ECUDA;
    uint64_t h3[3] = {0, 0, 0};
    const int rc = f.run(input, n, true, index, index_cap, OWN_OUTPUT, 3, [&](const uint8_t* d_in, uint8_t* out, size_t) {
        // a device index that is 4-byte aligned is written in place; any other is built in stage_out and copied
        const bool direct = f.out_dev && !(reinterpret_cast<uintptr_t>(out) & 3);
        if (!direct) {
            const cudaError_t e = f.c->stage_out.ensure(bound, f.c->stream);
            if (e != cudaSuccess) { set_error("staging cudaMalloc", e); return DENSITY_B200_ECUDA; }
        }
        return index_build_locked(f.c, d_in, n, interval, direct ? out : f.c->stage_out.p, direct ? nullptr : out, !f.out_dev, f.c->d_size,
                                  f.c->stream, h3);
    });
    if (rc != DENSITY_B200_OK) return rc;
    *index_len = h3[0];
    return DENSITY_B200_OK;
}

int density_b200_chameleon_decode_range_indexed_device(const uint8_t* d_in, size_t n, const uint8_t* d_index, size_t index_len, uint64_t first,
                                                       uint64_t len, uint8_t* d_out, uint64_t* d_result, void* stream) {
    g_last_error.clear();
    if (!d_index || (reinterpret_cast<uintptr_t>(d_index) & 3)) { set_error("indexed range decode: d_index must be non-NULL and 4-byte aligned"); return DENSITY_B200_EARG; }
    // n == 0 or len == 0: nothing to write, as density_b200_chameleon_decode_range_device (the index is not read)
    return stream_entry(d_in, n, d_out, len, d_result, 3, 2, n == 0 || len == 0, stream, [&](DeviceCtx* c, cudaStream_t s) {
        std::vector<uint64_t> hdr;
        int rc = index_read(d_index, true, index_len, n, s, &hdr);
        if (rc != DENSITY_B200_OK) return rc;
        RangePlan p{};
        uint64_t j = 0;
        index_plan(hdr.data(), n, first, len, c->num_sms, &p, &j);
        return range_indexed_locked(c, d_in + p.piece_off, p, index_snapshot(d_index, hdr, j), false, hdr[CIDX_SIZE_W], d_out, d_result, s);
    });
}

int density_b200_chameleon_decode_range_indexed(const uint8_t* input, size_t n, const uint8_t* index, size_t index_len, uint64_t first,
                                                uint8_t* output, uint64_t len, uint64_t* written) {
    g_last_error.clear();
    if (!written || (!input && n) || (!output && len) || !index) { set_error("null pointer"); return DENSITY_B200_EARG; }
    *written = 0;
    if (n == 0 || len == 0) return DENSITY_B200_OK;
    SyncCall f(input, output);
    if (!f.c) return DENSITY_B200_ECUDA;
    const bool index_dev = is_device_pointer(index);
    if (index_dev && !f.in_dev && !f.out_dev) {      // the frame synchronises only for the stream and the output
        const cudaError_t e = cudaDeviceSynchronize();
        if (e != cudaSuccess) { set_error("cudaDeviceSynchronize", e); return DENSITY_B200_ECUDA; }
    }
    std::vector<uint64_t> hdr;
    int rc = index_read(index, index_dev, index_len, n, f.c->stream, &hdr);
    if (rc != DENSITY_B200_OK) return rc;
    RangePlan p{};
    uint64_t j = 0;
    if (!index_plan(hdr.data(), n, first, len, f.c->num_sms, &p, &j)) return DENSITY_B200_OK;     // first >= S
    // only the piece of the stream is staged (SyncCall stages what it is given), and only snapshot j of the index
    const uint8_t* snap = index_snapshot(index, hdr, j);
    const bool snap_copy = !index_dev || (reinterpret_cast<uintptr_t>(snap) & 3);
    rc = f.run(input + p.piece_off, p.piece_n, true, output, len, p.w, 3, [&](const uint8_t* d_piece, uint8_t* out, size_t) {
        return range_indexed_locked(f.c, d_piece, p, snap, snap_copy, hdr[CIDX_SIZE_W], out, f.c->d_size, f.c->stream);
    });
    if (rc != DENSITY_B200_OK) return rc;
    if (f.c->h_size[2] != 0) { set_error("indexed range decode: the stream does not decode to what its index describes"); return DENSITY_B200_EMALFORMED; }
    *written = f.c->h_size[0];
    return DENSITY_B200_OK;
}

// ---- the argument rule of the sharded entries (include/density_b200.h, "Sharded encode" and "Sharded decode"). Each helper returns
// DENSITY_B200_EARG with the error set, or DENSITY_B200_OK.
static bool al4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) == 0; }
static bool al8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }
// the input and the output of a shard or a piece; either may be null when its length is 0. Decode: d_in 2-byte, d_out 4-byte aligned.
// Encode: d_in 4-byte, d_out 2-byte aligned, and a shard that does not end the stream (!is_last) a multiple of 256 bytes.
static int in_args(bool encode, const uint8_t* d_in, size_t n, const uint8_t* d_out, size_t cap, bool is_last = true) {
    if ((!d_in && n) || (!d_out && cap)) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (encode && !is_last && (n % 256)) { set_error("non-final shards must be a multiple of 256 bytes"); return DENSITY_B200_EARG; }
    const uintptr_t in = reinterpret_cast<uintptr_t>(d_in), out = reinterpret_cast<uintptr_t>(d_out);
    if (encode && ((in & 3) || (out & 1))) { set_error("d_in must be 4-byte, d_out 2-byte aligned"); return DENSITY_B200_EARG; }
    if (!encode && ((in & 1) || (out & 3))) { set_error("d_in must be 2-byte, d_out 4-byte aligned"); return DENSITY_B200_EARG; }
    return DENSITY_B200_OK;
}
// tables, transfers, carries, words and flags, null where the entry allows it (the caller checks that)
static int table_args(std::initializer_list<const void*> tables) {
    for (const void* t : tables)
        if (!al4(t)) { set_error("tables, transfers, carries, words and flags must be 4-byte aligned"); return DENSITY_B200_EARG; }
    return DENSITY_B200_OK;
}
// the sizes an entry writes: d_out_size (not null) and d_total_size (null where the entry allows it), both 8-byte aligned
static int size_args(const uint64_t* d_out_size, const uint64_t* d_total_size = nullptr) {
    if (!d_out_size) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (!al8(d_out_size) || !al8(d_total_size)) { set_error("d_out_size and d_total_size must be 8-byte aligned"); return DENSITY_B200_EARG; }
    return DENSITY_B200_OK;
}
// the size and the seam words a shard or a piece writes
static int out_args(const uint64_t* d_out_size, const uint32_t* d_seam8) {
    if (!d_seam8) { set_error("null pointer"); return DENSITY_B200_EARG; }
    const int rc = size_args(d_out_size);
    return rc == DENSITY_B200_OK ? table_args({d_seam8}) : rc;
}
// the order rule of every sharded encode entry: s is not null, its stage is one of `stages` and it has committed at least min_round
// rounds; otherwise the error `what`
extern "C++" {
template <class S> static bool in_stage(const S* s, std::initializer_list<int> stages, const char* what, int min_round = 0) {
    if (s && s->round >= min_round)
        for (int k : stages) if (s->stage == k) return true;
    set_error(what);
    return false;
}
}
// after a commit (waits for the device): words 2 .. 19 of the status of a shard's copy-map iteration from its device record, which
// lands in *h for the caller's words 0 and 1
static int prot_status_read(const DevBuf& rec, uint32_t* out, ProtShard* h, const char* what) {
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(h, rec.p, sizeof *h, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { set_error(what, e); return DENSITY_B200_ECUDA; }
    out[3] = h->esc;
    const uint32_t c = h->in_state;   // pc_encode candidate -> penalty | start << 8 | previous_incompressible << 16
    out[2] = c >= PROT_TRANSFER_WORDS ? 0xFFFFFFFFu : (c % 10) | (((c / 10) % 10 + 1) << 8) | ((c / 100) << 16);
    for (int k = 0; k < 16; ++k) out[4 + k] = h->changed[k];
    return DENSITY_B200_OK;
}

// ---- sharded Chameleon encode ------------------------------------------------------------------------
struct density_b200_shard {
    // PHASE1: the quiet phase 1 done (phase 2 may follow, any number of times). The copy-map iteration of density_b200_shard_prot_*:
    // FLAGS after prot_phase1 or prot_next with a table, then TRANSFER, SETTLED, COMMITTED (prot_next without a table), FINISHED.
    enum { NONE, PHASE1, FLAGS, TRANSFER, SETTLED, COMMITTED, FINISHED };
    DevBuf ws;
    DevBuf prot;                    // the device record of the copy-map iteration (ProtShard)
    ChamLayout L{};
    const uint8_t* d_in = nullptr;
    size_t n = 0;
    uint32_t nruns = 0;
    int num_sms = 0;
    int stage = NONE;
    int round = 0;                  // the rounds of the copy-map iteration that went on to the next
    ~density_b200_shard() { ws.release(); prot.release(); }
};

// a phase object of the sharded API for the current device (NULL, with the error set, without one)
extern "C++" {
template <class S> static S* new_shard() {
    g_last_error.clear();
    DeviceCtx* c = current_ctx();
    if (!c) return nullptr;
    S* s = new S();
    s->num_sms = c->num_sms;
    return s;
}
}
density_b200_shard* density_b200_shard_create(void) { return new_shard<density_b200_shard>(); }
void density_b200_shard_destroy(density_b200_shard* s) { delete s; }

// the shard d_in[0 .. n) set up in s (phase 1 and prot_phase1): every step of the shard before it void, the workspace and with_prot the
// iteration's record ensured, the shard stored
static int cham_shard_setup(density_b200_shard* s, const uint8_t* d_in, size_t n, bool with_prot, cudaStream_t st) {
    s->stage = density_b200_shard::NONE;
    cudaError_t e = s->ws.ensure(cham_workspace_bytes(n, s->num_sms, &s->L), st);
    if (e == cudaSuccess && with_prot) e = s->prot.ensure(sizeof(ProtShard), st);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    s->d_in = d_in; s->n = n; s->nruns = cham_pick_runs(n, s->num_sms);
    return DENSITY_B200_OK;
}
int density_b200_shard_phase1(density_b200_shard* s, const uint8_t* d_in, size_t n, int is_last_shard, uint32_t* d_table_out, void* stream) {
    g_last_error.clear();
    if (!s || !d_table_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int rc = in_args(true, d_in, n, nullptr, 0, is_last_shard);
    if (rc == DENSITY_B200_OK) rc = table_args({d_table_out});
    if (rc == DENSITY_B200_OK) rc = cham_shard_setup(s, d_in, n, false, st);
    if (rc != DENSITY_B200_OK) return rc;
    uint64_t launches = 0;
    const cudaError_t e = n ? cham_encode_phase1(d_in, n, s->ws.p, s->L, s->nruns, d_table_out, st, &launches)
                            : cudaMemsetAsync(d_table_out, 0, 65536 * sizeof(uint32_t), st);  // nothing touched
    rc = step_result(e, launches, "shard phase1");
    if (rc == DENSITY_B200_OK) s->stage = density_b200_shard::PHASE1;
    return rc;
}
// phase 2 on the shard's workspace: carry-in, first-touch flags, sizes, scan, emit. assume_prev_inc: the block before the shard counts
// as incompressible; ev (may be NULL): the stage events of cham_encode_phase2.
static int shard_phase2_impl(density_b200_shard* s, const uint32_t* d_carry_in, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                             bool assume_prev_inc, cudaEvent_t* ev, cudaStream_t st) {
    uint64_t launches = 0;
    const cudaError_t e = cham_encode_phase2(s->d_in, s->n, s->ws.p, s->L, s->nruns, d_carry_in, d_out, cap, d_out_size, false,
                                             assume_prev_inc, s->num_sms, st, &launches, ev);
    return step_result(e, launches, "shard phase2");
}
int density_b200_shard_phase2(density_b200_shard* s, const uint32_t* d_carry_in, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                              uint32_t* d_flags, void* stream) {
    g_last_error.clear();
    if (!in_stage(s, {density_b200_shard::PHASE1}, "shard_phase2: null pointer / phase1 not done")) return DENSITY_B200_EARG;
    int rc = in_args(true, nullptr, 0, d_out, 0);       // d_out's alignment; phase 2 takes a NULL d_out at any capacity
    if (rc == DENSITY_B200_OK) rc = table_args({d_carry_in, d_flags});
    if (rc == DENSITY_B200_OK) rc = size_args(d_out_size);
    if (rc != DENSITY_B200_OK) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    rc = shard_phase2_impl(s, d_carry_in, d_out, cap, d_out_size, d_carry_in != nullptr, nullptr, st);
    if (rc != DENSITY_B200_OK || !d_flags) return rc;
    const cudaError_t e = s->n ? cudaMemcpyAsync(d_flags, s->ws.p + s->L.status + offsetof(Status, nonquiet), sizeof(uint32_t),
                                                 cudaMemcpyDeviceToDevice, st)
                               : cudaMemsetAsync(d_flags, 0, sizeof(uint32_t), st);
    return step_result(e, 0, "shard phase2");
}

// ---- sharded Chameleon encode with copy mode: the copy-map iteration carried over the cuts ---------------------------------------------
static int g_prot_rounds = (int)PROT_MAX_ROUNDS;   // round budget (density_b200_test_set_prot_rounds)
static ProtShard* prot_rec(density_b200_shard* s) { return reinterpret_cast<ProtShard*>(s->prot.p); }

int density_b200_prot_round_budget(void) { return g_prot_rounds; }
void density_b200_test_set_prot_rounds(int k) { g_prot_rounds = (k >= 1 && k <= (int)PROT_MAX_ROUNDS) ? k : (int)PROT_MAX_ROUNDS; }

// first_block = ~0: taken from d_lengths (the gathered shard lengths) on the device instead
static int prot_phase1_impl(density_b200_shard* s, const uint8_t* d_in, size_t n, uint64_t first_block, const uint64_t* d_lengths, int rank,
                            int is_last_shard, uint32_t* d_table_out, cudaStream_t st) {
    if (!s || !d_table_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    int rc = in_args(true, d_in, n, nullptr, 0, is_last_shard);
    if (rc == DENSITY_B200_OK) rc = table_args({d_table_out});
    if (rc == DENSITY_B200_OK) rc = cham_shard_setup(s, d_in, n, true, st);
    if (rc != DENSITY_B200_OK) return rc;
    s->round = 0;
    uint64_t launches = 0;
    cudaError_t e = cham_encode_phase1(d_in, n, s->ws.p, s->L, s->nruns, n ? d_table_out : nullptr, st, &launches);
    if (e == cudaSuccess && !n) e = cudaMemsetAsync(d_table_out, 0, 65536 * sizeof(uint32_t), st);   // nothing touched
    if (e == cudaSuccess) e = cham_prot_start(s->ws.p, s->L, prot_rec(s), d_lengths ? 0 : first_block, d_lengths, (uint32_t)rank, st, &launches);
    rc = step_result(e, launches, "shard prot phase1");
    if (rc == DENSITY_B200_OK) s->stage = density_b200_shard::FLAGS;
    return rc;
}
// ev (may be NULL): the stage events of cham_encode_phase2
static int prot_finish_impl(density_b200_shard* s, uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint32_t* d_seam8, cudaStream_t st,
                            cudaEvent_t* ev) {
    if (!in_stage(s, {density_b200_shard::COMMITTED}, "shard_prot_finish: call it after prot_next without a table")) return DENSITY_B200_EARG;
    int rc = in_args(true, nullptr, 0, d_out, cap);
    if (rc == DENSITY_B200_OK) rc = out_args(d_out_size, d_seam8);
    if (rc != DENSITY_B200_OK) return rc;
    uint64_t launches = 0;
    const cudaError_t e = cham_prot_finish(s->d_in, s->n, s->ws.p, s->L, prot_rec(s), d_out, cap, d_out_size, d_seam8, st, &launches, ev);
    rc = step_result(e, launches, "shard prot finish");
    if (rc == DENSITY_B200_OK) s->stage = density_b200_shard::FINISHED;
    return rc;
}

int density_b200_shard_prot_phase1(density_b200_shard* s, const uint8_t* d_in, size_t n, uint64_t first_block, int is_last_shard,
                                   uint32_t* d_table_out, void* stream) {
    g_last_error.clear();
    if (first_block == ~0ull) { set_error("bad first_block"); return DENSITY_B200_EARG; }
    return prot_phase1_impl(s, d_in, n, first_block, nullptr, 0, is_last_shard, d_table_out, reinterpret_cast<cudaStream_t>(stream));
}
int density_b200_shard_prot_transfer(density_b200_shard* s, const uint32_t* d_carry_in, uint32_t* d_transfer_out, void* stream) {
    g_last_error.clear();
    if (!in_stage(s, {density_b200_shard::FLAGS}, "shard_prot_transfer: call it after prot_phase1 or prot_next with a table")) return DENSITY_B200_EARG;
    if (!d_transfer_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (table_args({d_carry_in, d_transfer_out}) != DENSITY_B200_OK) return DENSITY_B200_EARG;
    uint64_t launches = 0;
    const cudaError_t e = cham_prot_transfer(s->n, s->ws.p, s->L, s->nruns, d_carry_in, prot_rec(s), s->round, d_transfer_out,
                                             reinterpret_cast<cudaStream_t>(stream), &launches);
    const int rc = step_result(e, launches, "shard prot transfer");
    if (rc == DENSITY_B200_OK) s->stage = density_b200_shard::TRANSFER;
    return rc;
}
int density_b200_shard_prot_settle(density_b200_shard* s, const uint32_t* d_all_transfers, int world, int rank, uint32_t* d_words_out, void* stream) {
    g_last_error.clear();
    if (!in_stage(s, {density_b200_shard::TRANSFER}, "shard_prot_settle: call it after prot_transfer")) return DENSITY_B200_EARG;
    if (!d_all_transfers || !d_words_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (world < 1 || rank < 0 || rank >= world) { set_error("bad rank / world"); return DENSITY_B200_EARG; }
    if (table_args({d_all_transfers, d_words_out}) != DENSITY_B200_OK) return DENSITY_B200_EARG;
    uint64_t launches = 0;
    const cudaError_t e = cham_prot_settle(s->n, s->ws.p, s->L, prot_rec(s), s->round, d_all_transfers, (uint32_t)rank, d_words_out,
                                           reinterpret_cast<cudaStream_t>(stream), &launches);
    const int rc = step_result(e, launches, "shard prot settle");
    if (rc == DENSITY_B200_OK) s->stage = density_b200_shard::SETTLED;
    return rc;
}
int density_b200_shard_prot_next(density_b200_shard* s, const uint32_t* d_all_words, int world, uint32_t* d_table_out, void* stream) {
    g_last_error.clear();
    if (!in_stage(s, {density_b200_shard::SETTLED}, "shard_prot_next: call it after prot_settle")) return DENSITY_B200_EARG;
    if (!d_all_words) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (world < 1) { set_error("bad world"); return DENSITY_B200_EARG; }
    if (table_args({d_all_words, d_table_out}) != DENSITY_B200_OK) return DENSITY_B200_EARG;
    if (d_table_out && s->round + 1 >= g_prot_rounds) { set_error("shard_prot_next: the round budget is used up"); return DENSITY_B200_EARG; }
    uint64_t launches = 0;
    const cudaError_t e = cham_prot_next(s->d_in, s->n, s->ws.p, s->L, s->nruns, prot_rec(s), s->round, d_all_words, (uint32_t)world,
                                         d_table_out, reinterpret_cast<cudaStream_t>(stream), &launches);
    const int rc = step_result(e, launches, "shard prot next");
    if (rc != DENSITY_B200_OK) return rc;
    if (d_table_out) { ++s->round; s->stage = density_b200_shard::FLAGS; }
    else s->stage = density_b200_shard::COMMITTED;
    return DENSITY_B200_OK;
}
int density_b200_shard_prot_finish(density_b200_shard* s, uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint32_t* d_seam8, void* stream) {
    g_last_error.clear();
    return prot_finish_impl(s, d_out, cap, d_out_size, d_seam8, reinterpret_cast<cudaStream_t>(stream), nullptr);
}
int density_b200_shard_prot_status(density_b200_shard* s, uint32_t* out) {
    g_last_error.clear();
    if (!out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (!in_stage(s, {density_b200_shard::COMMITTED, density_b200_shard::FINISHED}, "shard_prot_status: rounds not committed")) return DENSITY_B200_EARG;
    ProtShard h{};
    const int rc = prot_status_read(s->prot, out, &h, "shard_prot_status");
    if (rc == DENSITY_B200_OK) { out[0] = h.rounds; out[1] = h.settled; }
    return rc;
}

// ---- sharded Cheetah / Lion encode: one shard of a longer stream in three phases around two table exchanges ---------------------------
struct density_b200_cl_shard {
    // the quiet phases: PHASE1 -> PHASE2 -> PHASE3, once each. The copy-map iteration of density_b200_cl_shard_prot_*: READY after
    // prot_phase1 or a commit, then P, C, TRANSFER, SETTLED per round, FINISHED.
    enum { NONE, PHASE1, PHASE2, PHASE3, READY, P, C, TRANSFER, SETTLED, FINISHED };
    DevBuf ws, tables[3];           // workspace; the epoch-tagged run tables (zero at allocation, one entry format each)
    DevBuf prot;                    // the device record of the copy-map iteration (ProtShard)
    ClShardArgs a{};                // the current shard, as every phase takes it
    uint32_t epoch = 0;
    int num_sms = 0;
    int stage = NONE;
    int round = 0;                  // rounds committed
    ~density_b200_cl_shard() { ws.release(); for (auto& t : tables) t.release(); prot.release(); }
};

static bool cl_alg_ok(int alg) { return alg == ALG_CHEETAH || alg == ALG_LION; }

density_b200_cl_shard* density_b200_cl_shard_create(int alg) {
    if (!cl_alg_ok(alg)) { set_error("cl_shard_create: alg must be DENSITY_B200_CHEETAH or DENSITY_B200_LION"); return nullptr; }
    density_b200_cl_shard* s = new_shard<density_b200_cl_shard>();
    if (s) s->a.alg = alg;
    return s;
}
void density_b200_cl_shard_destroy(density_b200_cl_shard* s) { delete s; }
size_t density_b200_cl_table_words(int alg, int kind) {
    if (!cl_alg_ok(alg) || (kind != DENSITY_B200_CL_TABLE_P && kind != DENSITY_B200_CL_TABLE_C)) return 0;
    return (size_t)cl_table_planes(alg, kind) * 65536;
}

// the shard d_in[0 .. n) set up in s->a (phase 1 and prot_phase1): every step of the shard before it void, the workspace, the tables and
// with_prot the iteration's record ensured, the shard's epochs taken (cl_prot_epochs() with_prot, else cl_shard_epochs())
static int cl_shard_setup(density_b200_cl_shard* s, const uint8_t* d_in, size_t n, uint64_t offset, bool first, int is_last, bool with_prot,
                          cudaStream_t st) {
    s->stage = density_b200_cl_shard::NONE;
    ClShardArgs& a = s->a;
    cudaError_t e = s->ws.ensure(cl_shard_workspace_bytes(n, s->num_sms), st);
    for (int rg = 0; rg < 3 && e == cudaSuccess; ++rg) e = s->tables[rg].ensure(chee_tables_bytes(a.alg, rg, n, s->num_sms) + 256, st);
    if (e == cudaSuccess && with_prot) e = s->prot.ensure(sizeof(ProtShard), st);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    if (s->epoch > 0x0FFFFF00u) {                      // epochs exhausted: start over on cleared tables
        for (int rg = 0; rg < 3 && e == cudaSuccess; ++rg) e = cudaMemsetAsync(s->tables[rg].p, 0, s->tables[rg].bytes, st);
        if (e != cudaSuccess) { set_error("cudaMemsetAsync", e); return DENSITY_B200_ECUDA; }
        s->epoch = 0;
    }
    a.epoch_base = s->epoch + 1; s->epoch += with_prot ? cl_prot_epochs() : cl_shard_epochs();
    a.d_in = d_in; a.n = n; a.offset = offset; a.first = first; a.last = is_last != 0;
    a.ws = s->ws.p; for (int rg = 0; rg < 3; ++rg) a.tables[rg] = s->tables[rg].p;
    a.num_sms = s->num_sms; a.ps = reinterpret_cast<ProtShard*>(s->prot.p);
    return DENSITY_B200_OK;
}

int density_b200_cl_shard_phase1(density_b200_cl_shard* s, const uint8_t* d_in, size_t n, int is_last_shard, const uint32_t* d_prev_quad,
                                 uint32_t* d_table_p_out, void* stream) {
    g_last_error.clear();
    if (!s || !d_table_p_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int rc = in_args(true, d_in, n, nullptr, 0, is_last_shard);
    if (rc == DENSITY_B200_OK) rc = table_args({d_prev_quad, d_table_p_out});
    if (rc == DENSITY_B200_OK) rc = cl_shard_setup(s, d_in, n, 0, d_prev_quad == nullptr, is_last_shard, false, st);
    if (rc != DENSITY_B200_OK) return rc;
    uint64_t launches = 0;
    // an empty shard exports the identity
    const cudaError_t e = n ? cl_shard_phase1(s->a, d_prev_quad, d_table_p_out, st, &launches)
                            : cudaMemsetAsync(d_table_p_out, 0, density_b200_cl_table_words(s->a.alg, DENSITY_B200_CL_TABLE_P) * sizeof(uint32_t), st);
    rc = step_result(e, launches, "cl shard phase1");
    if (rc == DENSITY_B200_OK) s->stage = density_b200_cl_shard::PHASE1;
    return rc;
}
int density_b200_cl_shard_phase2(density_b200_cl_shard* s, const uint32_t* d_carry_p, uint32_t* d_table_c_out, void* stream) {
    g_last_error.clear();
    if (!in_stage(s, {density_b200_cl_shard::PHASE1}, "cl_shard_phase2: null pointer / phase 1 not done")) return DENSITY_B200_EARG;
    if (!d_table_c_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    int rc = table_args({d_carry_p, d_table_c_out});
    if (rc != DENSITY_B200_OK) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    uint64_t launches = 0;
    const cudaError_t e = s->a.n ? cl_shard_phase2(s->a, d_carry_p, d_table_c_out, st, &launches)
                                 : cudaMemsetAsync(d_table_c_out, 0, density_b200_cl_table_words(s->a.alg, DENSITY_B200_CL_TABLE_C) * sizeof(uint32_t), st);
    rc = step_result(e, launches, "cl shard phase2");
    if (rc == DENSITY_B200_OK) s->stage = density_b200_cl_shard::PHASE2;
    return rc;
}
int density_b200_cl_shard_phase3(density_b200_cl_shard* s, const uint32_t* d_carry_c, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                 uint32_t* d_seam8, void* stream) {
    g_last_error.clear();
    if (!in_stage(s, {density_b200_cl_shard::PHASE2}, "cl_shard_phase3: null pointer / phase 2 not done")) return DENSITY_B200_EARG;
    int rc = in_args(true, nullptr, 0, d_out, cap);
    if (rc == DENSITY_B200_OK) rc = table_args({d_carry_c});
    if (rc == DENSITY_B200_OK) rc = out_args(d_out_size, d_seam8);
    if (rc != DENSITY_B200_OK) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    uint64_t launches = 0;
    const cudaError_t e = s->a.n ? cl_shard_phase3(s->a, d_carry_c, d_out, cap, d_out_size, d_seam8, st, &launches)
                                 : empty_piece_outputs(d_out_size, d_seam8, st);
    rc = step_result(e, launches, "cl shard phase3");
    if (rc == DENSITY_B200_OK) s->stage = density_b200_cl_shard::PHASE3;
    return rc;
}
// ---- sharded Cheetah / Lion encode with copy mode: the copy-map iteration carried over the cuts ------------------------------------------
int density_b200_cl_shard_prot_phase1(density_b200_cl_shard* s, const uint8_t* d_in, size_t n, uint64_t offset, int is_last_shard,
                                      uint32_t* d_words_out, void* stream) {
    g_last_error.clear();
    if (!s || !d_words_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (offset % 256) { set_error("offset must be a multiple of 256 bytes"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int rc = in_args(true, d_in, n, nullptr, 0, is_last_shard);
    if (rc == DENSITY_B200_OK) rc = table_args({d_words_out});
    if (rc == DENSITY_B200_OK) rc = cl_shard_setup(s, d_in, n, offset, offset == 0 && n > 0, is_last_shard, true, st);
    if (rc != DENSITY_B200_OK) return rc;
    s->round = 0;
    uint64_t launches = 0;
    const cudaError_t e = cl_prot_phase1(s->a, d_words_out, st, &launches);
    rc = step_result(e, launches, "cl shard prot phase1");
    if (rc == DENSITY_B200_OK) s->stage = density_b200_cl_shard::READY;
    return rc;
}
int density_b200_cl_shard_prot_p(density_b200_cl_shard* s, const uint32_t* d_all_words, int world, int rank, uint32_t* d_table_p_out, void* stream) {
    g_last_error.clear();
    if (!d_all_words || !d_table_p_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (!in_stage(s, {density_b200_cl_shard::READY}, "cl_shard_prot_p: call it after prot_phase1 or prot_next")) return DENSITY_B200_EARG;
    if (s->round >= g_prot_rounds) { set_error("cl_shard_prot_p: the round budget is used up"); return DENSITY_B200_EARG; }
    if (world < 1 || rank < 0 || rank >= world) { set_error("bad rank / world"); return DENSITY_B200_EARG; }
    if (table_args({d_all_words, d_table_p_out}) != DENSITY_B200_OK) return DENSITY_B200_EARG;
    uint64_t launches = 0;
    const cudaError_t e = cl_prot_p(s->a, s->round, d_all_words, (uint32_t)rank, d_table_p_out, reinterpret_cast<cudaStream_t>(stream), &launches);
    const int rc = step_result(e, launches, "cl shard prot p");
    if (rc == DENSITY_B200_OK) s->stage = density_b200_cl_shard::P;
    return rc;
}
int density_b200_cl_shard_prot_c(density_b200_cl_shard* s, const uint32_t* d_carry_p, uint32_t* d_table_c_out, void* stream) {
    g_last_error.clear();
    if (!d_carry_p || !d_table_c_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (!in_stage(s, {density_b200_cl_shard::P}, "cl_shard_prot_c: call it after prot_p")) return DENSITY_B200_EARG;
    if (table_args({d_carry_p, d_table_c_out}) != DENSITY_B200_OK) return DENSITY_B200_EARG;
    uint64_t launches = 0;
    const cudaError_t e = cl_prot_c(s->a, s->round, d_carry_p, d_table_c_out, reinterpret_cast<cudaStream_t>(stream), &launches);
    const int rc = step_result(e, launches, "cl shard prot c");
    if (rc == DENSITY_B200_OK) s->stage = density_b200_cl_shard::C;
    return rc;
}
int density_b200_cl_shard_prot_transfer(density_b200_cl_shard* s, const uint32_t* d_carry_c, uint32_t* d_transfer_out, void* stream) {
    g_last_error.clear();
    if (!d_carry_c || !d_transfer_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (!in_stage(s, {density_b200_cl_shard::C}, "cl_shard_prot_transfer: call it after prot_c")) return DENSITY_B200_EARG;
    if (table_args({d_carry_c, d_transfer_out}) != DENSITY_B200_OK) return DENSITY_B200_EARG;
    uint64_t launches = 0;
    const cudaError_t e = cl_prot_transfer(s->a, s->round, d_carry_c, d_transfer_out, reinterpret_cast<cudaStream_t>(stream), &launches);
    const int rc = step_result(e, launches, "cl shard prot transfer");
    if (rc == DENSITY_B200_OK) s->stage = density_b200_cl_shard::TRANSFER;
    return rc;
}
int density_b200_cl_shard_prot_settle(density_b200_cl_shard* s, const uint32_t* d_all_transfers, int world, int rank, uint32_t* d_words_out,
                                      void* stream) {
    g_last_error.clear();
    if (!d_all_transfers || !d_words_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (!in_stage(s, {density_b200_cl_shard::TRANSFER}, "cl_shard_prot_settle: call it after prot_transfer")) return DENSITY_B200_EARG;
    if (world < 1 || rank < 0 || rank >= world) { set_error("bad rank / world"); return DENSITY_B200_EARG; }
    if (table_args({d_all_transfers, d_words_out}) != DENSITY_B200_OK) return DENSITY_B200_EARG;
    uint64_t launches = 0;
    const cudaError_t e = cl_prot_settle(s->a, s->round, d_all_transfers, (uint32_t)rank, d_words_out, reinterpret_cast<cudaStream_t>(stream), &launches);
    const int rc = step_result(e, launches, "cl shard prot settle");
    if (rc == DENSITY_B200_OK) s->stage = density_b200_cl_shard::SETTLED;
    return rc;
}
int density_b200_cl_shard_prot_next(density_b200_cl_shard* s, const uint32_t* d_all_words, int world, void* stream) {
    g_last_error.clear();
    if (!d_all_words) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (!in_stage(s, {density_b200_cl_shard::SETTLED}, "cl_shard_prot_next: call it after prot_settle")) return DENSITY_B200_EARG;
    if (world < 1) { set_error("bad world"); return DENSITY_B200_EARG; }
    if (table_args({d_all_words}) != DENSITY_B200_OK) return DENSITY_B200_EARG;
    uint64_t launches = 0;
    const cudaError_t e = cl_prot_next(s->a, s->round, d_all_words, (uint32_t)world, reinterpret_cast<cudaStream_t>(stream), &launches);
    const int rc = step_result(e, launches, "cl shard prot next");
    if (rc == DENSITY_B200_OK) { s->stage = density_b200_cl_shard::READY; ++s->round; }
    return rc;
}
// ev_emit (may be NULL): recorded between the scan and the emit
static int cl_prot_finish_impl(density_b200_cl_shard* s, uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint32_t* d_seam8, cudaStream_t st,
                               cudaEvent_t ev_emit) {
    int rc = in_args(true, nullptr, 0, d_out, cap);
    if (rc == DENSITY_B200_OK) rc = out_args(d_out_size, d_seam8);
    if (rc != DENSITY_B200_OK) return rc;
    if (!in_stage(s, {density_b200_cl_shard::READY}, "cl_shard_prot_finish: call it after prot_next", 1)) return DENSITY_B200_EARG;
    uint64_t launches = 0;
    const cudaError_t e = cl_prot_finish(s->a, d_out, cap, d_out_size, d_seam8, st, &launches, ev_emit);
    rc = step_result(e, launches, "cl shard prot finish");
    if (rc == DENSITY_B200_OK) s->stage = density_b200_cl_shard::FINISHED;
    return rc;
}
int density_b200_cl_shard_prot_finish(density_b200_cl_shard* s, uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint32_t* d_seam8, void* stream) {
    g_last_error.clear();
    return cl_prot_finish_impl(s, d_out, cap, d_out_size, d_seam8, reinterpret_cast<cudaStream_t>(stream), nullptr);
}
int density_b200_cl_shard_prot_status(density_b200_cl_shard* s, uint32_t* out) {
    g_last_error.clear();
    if (!out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    using S = density_b200_cl_shard;
    if (!in_stage(s, {S::READY, S::P, S::C, S::TRANSFER, S::SETTLED, S::FINISHED}, "cl_shard_prot_status: no round committed", 1)) return DENSITY_B200_EARG;
    ProtShard h{};
    const int rc = prot_status_read(s->prot, out, &h, "cl_shard_prot_status");
    if (rc == DENSITY_B200_OK) { out[0] = h.stage_ok; out[1] = h.rounds; }
    return rc;
}

int density_b200_cl_table_init(int alg, int kind, uint32_t* d_table, void* stream) {
    g_last_error.clear();
    if (!density_b200_cl_table_words(alg, kind) || !d_table) { set_error("cl_table_init: bad algorithm / kind or null pointer"); return DENSITY_B200_EARG; }
    if (table_args({d_table}) != DENSITY_B200_OK) return DENSITY_B200_EARG;
    uint64_t l = 0;
    const cudaError_t e = cl_table_init(alg, kind, d_table, reinterpret_cast<cudaStream_t>(stream), &l);
    return step_result(e, l, "cl_table_init");
}
int density_b200_cl_table_fold(int alg, int kind, uint32_t* d_acc, const uint32_t* d_next, void* stream) {
    g_last_error.clear();
    if (!density_b200_cl_table_words(alg, kind) || !d_acc || !d_next) { set_error("cl_table_fold: bad algorithm / kind or null pointer"); return DENSITY_B200_EARG; }
    if (table_args({d_acc, d_next}) != DENSITY_B200_OK) return DENSITY_B200_EARG;
    uint64_t l = 0;
    const cudaError_t e = cl_table_fold(alg, kind, d_acc, d_next, reinterpret_cast<cudaStream_t>(stream), &l);
    return step_result(e, l, "cl_table_fold");
}

// ---- sharded Chameleon decode: one piece of a sharded stream, decoded with the dictionary carried in from the pieces before it ------
struct density_b200_decode_shard {
    DevBuf ws;
    DevBuf seed;                    // the incoming automaton state of the prot_* phases (DECODE_PROT_SEED_WORDS)
    const uint8_t* d_in = nullptr;
    size_t n = 0, cap = 0;
    int is_last = 1;
    int num_sms = 0;
    bool phase1_done = false;
    int prot_stage = 0;             // prot_*: 1 after the transfer, 2 after phase 1
    void reset() { phase1_done = false; prot_stage = 0; }     // no step of any piece done
};

density_b200_decode_shard* density_b200_decode_shard_create(void) { return new_shard<density_b200_decode_shard>(); }
void density_b200_decode_shard_destroy(density_b200_decode_shard* s) {
    if (!s) return;
    s->ws.release();
    s->seed.release();
    delete s;
}
// the piece set up in s (phase 1, prot_transfer and prot_enter): every step of the piece before it void, the workspace and with_seed the
// seed ensured, the piece stored
static int decode_piece_setup(density_b200_decode_shard* s, const uint8_t* d_in, size_t n, size_t cap, int is_last, bool with_seed, cudaStream_t st) {
    s->reset();
    cudaError_t e = s->ws.ensure(cham_decode_workspace_bytes(n, cap, s->num_sms), st);
    if (e == cudaSuccess && with_seed) e = s->seed.ensure(DECODE_PROT_SEED_WORDS * sizeof(uint32_t), st);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    s->d_in = d_in; s->n = n; s->cap = cap; s->is_last = is_last;
    return DENSITY_B200_OK;
}
int density_b200_decode_shard_phase1(density_b200_decode_shard* s, const uint8_t* d_in, size_t n, size_t cap, int is_last_shard,
                                     uint32_t* d_table_out, void* stream) {
    g_last_error.clear();
    if (!s || !d_table_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int rc = in_args(false, d_in, n, nullptr, 0);
    if (rc == DENSITY_B200_OK) rc = table_args({d_table_out});
    if (rc == DENSITY_B200_OK) rc = decode_piece_setup(s, d_in, n, cap, is_last_shard, false, st);
    if (rc != DENSITY_B200_OK) return rc;
    uint64_t launches = 0;
    const cudaError_t e = n ? cham_decode_phase1(d_in, n, cap, s->ws.p, s->num_sms, d_table_out, st, &launches)
                            : cudaMemsetAsync(d_table_out, 0, 65536 * sizeof(uint32_t), st);  // nothing touched
    rc = step_result(e, launches, "decode shard phase1");
    if (rc == DENSITY_B200_OK) s->phase1_done = true;
    return rc;
}
// the arguments of both phase-2 entries
static int decode_phase2_args(const density_b200_decode_shard* s, const uint32_t* d_carry_in, const uint8_t* d_out, const uint64_t* d_out_size,
                              const uint32_t* d_seam8) {
    int rc = in_args(false, nullptr, 0, d_out, s->cap);
    if (rc == DENSITY_B200_OK) rc = table_args({d_carry_in});
    return rc == DENSITY_B200_OK ? out_args(d_out_size, d_seam8) : rc;
}
int density_b200_decode_shard_phase2(density_b200_decode_shard* s, const uint32_t* d_carry_in, uint8_t* d_out, uint64_t* d_out_size,
                                     uint32_t* d_seam8, void* stream) {
    g_last_error.clear();
    if (!s || !s->phase1_done) { set_error("decode_shard_phase2: phase1 not done"); return DENSITY_B200_EARG; }
    const int rc = decode_phase2_args(s, d_carry_in, d_out, d_out_size, d_seam8);
    if (rc != DENSITY_B200_OK) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    uint64_t launches = 0;
    cudaError_t e = s->n ? cham_decode_phase2(s->d_in, s->n, d_out, s->cap, s->ws.p, s->num_sms, d_carry_in, d_out_size, st, &launches)
                         : empty_piece_outputs(d_out_size, d_seam8, st);
    if (e == cudaSuccess && s->n) e = cham_decode_seam_words(s->d_in, s->n, s->cap, s->ws.p, s->num_sms, s->is_last, d_out_size, d_seam8, st, &launches);
    s->phase1_done = false;     // the decode pass overwrites the run tables: one phase 2 per phase 1
    return step_result(e, launches, "decode shard phase2");
}

// ---- the same for streams with copy-mode blocks: the piece's protection transfer first, then the two phases from the composed state -----
int density_b200_decode_shard_prot_transfer(density_b200_decode_shard* s, const uint8_t* d_in, size_t n, size_t cap, int is_last_shard,
                                            uint32_t* d_transfer_out, void* stream) {
    g_last_error.clear();
    if (!s || !d_transfer_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int rc = in_args(false, d_in, n, nullptr, 0);
    if (rc == DENSITY_B200_OK) rc = table_args({d_transfer_out});
    if (rc == DENSITY_B200_OK) rc = decode_piece_setup(s, d_in, n, cap, is_last_shard, true, st);
    if (rc != DENSITY_B200_OK) return rc;
    uint64_t launches = 0;
    const cudaError_t e = cham_decode_prot_transfer(d_in, n, s->ws.p, is_last_shard, d_transfer_out, st, &launches);
    rc = step_result(e, launches, "decode shard prot transfer");
    if (rc == DENSITY_B200_OK) s->prot_stage = 1;
    return rc;
}
// The protected phase 1 of the piece set up in s, from the seed composed from candidate x0 and the transfers of the pieces before `rank`
// (prot_phase1: x0 = 0, the rows of prot_transfer ready; prot_enter: a located piece's candidate, no transfers, the rows not computed yet).
static int decode_prot_phase1_body(density_b200_decode_shard* s, const uint32_t* d_all_transfers, int rank, uint32_t x0, bool rows_ready,
                                   uint32_t* d_table_out, cudaStream_t st, const char* what) {
    uint32_t* seed = reinterpret_cast<uint32_t*>(s->seed.p);
    uint64_t launches = 0;
    cudaError_t e = cham_decode_prot_enter(d_all_transfers, (uint32_t)rank, x0, seed, st, &launches);
    if (e == cudaSuccess) {
        if (s->n == 0) e = cudaMemsetAsync(d_table_out, 0, 65536 * sizeof(uint32_t), st);  // nothing touched
        else e = cham_decode_phase1(s->d_in, s->n, s->cap, s->ws.p, s->num_sms, d_table_out, st, &launches, seed, rows_ready);
    }
    const int rc = step_result(e, launches, what);
    s->prot_stage = rc == DENSITY_B200_OK ? 2 : 0;
    return rc;
}
int density_b200_decode_shard_prot_phase1(density_b200_decode_shard* s, const uint32_t* d_all_transfers, int world, int rank,
                                          uint32_t* d_table_out, void* stream) {
    g_last_error.clear();
    if (!s || s->prot_stage != 1) { set_error("decode_shard_prot_phase1: null pointer / transfer not done"); return DENSITY_B200_EARG; }
    if (world < 1 || rank < 0 || rank >= world || (rank > 0 && !d_all_transfers) || !d_table_out) { set_error("bad rank / world or null pointer"); return DENSITY_B200_EARG; }
    const int rc = table_args({d_all_transfers, d_table_out});
    if (rc != DENSITY_B200_OK) return rc;
    return decode_prot_phase1_body(s, d_all_transfers, rank, 0, true, d_table_out, reinterpret_cast<cudaStream_t>(stream), "decode shard prot phase1");
}
int density_b200_decode_shard_prot_enter(density_b200_decode_shard* s, const uint8_t* d_in, size_t n, size_t cap, int is_last_shard,
                                         uint32_t candidate, uint32_t* d_table_out, void* stream) {
    g_last_error.clear();
    if (!s || !d_table_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int rc = in_args(false, d_in, n, nullptr, 0);
    if (rc == DENSITY_B200_OK) rc = table_args({d_table_out});
    if (rc != DENSITY_B200_OK) return rc;
    if (candidate >= DECODE_PROT_TRANSFER_WORDS) { set_error("decode_shard_prot_enter: candidate >= 3200"); return DENSITY_B200_EARG; }
    if ((rc = decode_piece_setup(s, d_in, n, cap, is_last_shard, true, st)) != DENSITY_B200_OK) return rc;
    return decode_prot_phase1_body(s, nullptr, 0, candidate, false, d_table_out, st, "decode shard prot enter");
}
int density_b200_decode_shard_prot_phase2(density_b200_decode_shard* s, const uint32_t* d_carry_in, uint8_t* d_out, uint64_t* d_out_size,
                                          uint32_t* d_seam8, void* stream) {
    g_last_error.clear();
    if (!s || s->prot_stage != 2) { set_error("decode_shard_prot_phase2: null pointer / phase1 not done"); return DENSITY_B200_EARG; }
    const int rc = decode_phase2_args(s, d_carry_in, d_out, d_out_size, d_seam8);
    if (rc != DENSITY_B200_OK) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    uint64_t launches = 0;
    cudaError_t e = s->n ? cham_decode_phase2(s->d_in, s->n, d_out, s->cap, s->ws.p, s->num_sms, d_carry_in, d_out_size, st, &launches) : cudaSuccess;
    if (e == cudaSuccess)
        e = cham_decode_prot_seam_words(s->n, s->cap, s->ws.p, s->num_sms, s->is_last, reinterpret_cast<const uint32_t*>(s->seed.p), d_out_size, d_seam8,
                                        st, &launches);
    s->prot_stage = 0;          // one phase 2 per transfer
    return step_result(e, launches, "decode shard prot phase2");
}

// ---- sharded Cheetah and Lion decode: one piece, its chunk map carried in, then Cheetah's prediction rounds run over all pieces or Lion's
// prediction walk continued from the state the piece before it left ----------------------------------------------------------------------
static int g_chee_dec_rounds = 40;    // round budget of the sharded Cheetah decode (density_b200_test_set_decode_rounds)

// the phase object of one piece; a.lion: a Lion piece
struct ClDecodePiece {
    DevBuf ws, tables;
    DevBuf seed;                    // the incoming automaton state of the prot_* phases (DECODE_PROT_SEED_WORDS)
    CheeShardArgs a{};
    int num_sms = 0;
    // the last step done on the current piece: 0 none, 1 phase 1, 2 phase 2 or (Cheetah) a round's fold, 3 a round's walk (Cheetah) or
    // the walk (Lion), 4 phase 3
    int phase = 0;
    uint32_t round = 0;             // Cheetah: the rounds folded
    bool transfer_done = false;     // prot_transfer done, prot_phase1 not yet
    bool prot = false;              // the current piece went through prot_phase1 or prot_enter: phase 3 writes the protected seam words
    void reset() { phase = 0; round = 0; transfer_done = false; prot = false; }     // no step of any piece done
    ~ClDecodePiece() { ws.release(); tables.release(); seed.release(); }
};
struct density_b200_cheetah_decode_shard : ClDecodePiece {};
struct density_b200_lion_decode_shard : ClDecodePiece {};
static_assert(LION_STATE_WORDS == DENSITY_B200_LION_STATE_WORDS, "the relayed state of the header and of cl_decode.cu");

density_b200_cheetah_decode_shard* density_b200_cheetah_decode_shard_create(void) { return new_shard<density_b200_cheetah_decode_shard>(); }
density_b200_lion_decode_shard* density_b200_lion_decode_shard_create(void) { return new_shard<density_b200_lion_decode_shard>(); }
void density_b200_cheetah_decode_shard_destroy(density_b200_cheetah_decode_shard* s) { delete s; }
void density_b200_lion_decode_shard_destroy(density_b200_lion_decode_shard* s) { delete s; }
int density_b200_cheetah_decode_round_budget(void) { return g_chee_dec_rounds; }
size_t density_b200_cheetah_cmap_words(void) { return 3 * 65536; }

// the argument checks and the piece set up in s->a (phase 1, prot_transfer and prot_enter): the piece's state reset, its workspace and
// tables (with_seed: and the seed) ensured for its geometry. d_table: the chunk-map or protection transfer out (need_table: not null).
// DENSITY_B200_OK, or the error code with nothing enqueued.
static int cl_piece_setup(ClDecodePiece* s, bool lion, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, int is_first, int is_last,
                          const uint32_t* d_table, bool need_table, bool with_seed, cudaStream_t st) {
    if (!s || (need_table && !d_table)) { set_error("null pointer"); return DENSITY_B200_EARG; }
    int rc = in_args(false, d_in, n, d_out, cap);
    if (rc == DENSITY_B200_OK) rc = table_args({d_table});
    if (rc != DENSITY_B200_OK) return rc;
    s->reset();
    CheeShardArgs& a = s->a;
    a.d_in = d_in; a.n = n; a.d_out = d_out; a.cap = cap; a.first = is_first != 0; a.last = is_last != 0; a.lion = lion; a.num_sms = s->num_sms;
    cudaError_t e = with_seed ? s->seed.ensure(DECODE_PROT_SEED_WORDS * sizeof(uint32_t), st) : cudaSuccess;
    if (n) {
        if (e == cudaSuccess) e = s->ws.ensure(chee_shard_workspace_bytes(n, cap, s->num_sms, lion), st);
        if (e == cudaSuccess) e = s->tables.ensure(chee_decode_tables_bytes(n, s->num_sms, lion) + 256, st);
    }
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    a.ws = s->ws.p; a.tables = s->tables.p;
    return DENSITY_B200_OK;
}
// phase 1 of the piece set up in s->a (d_seed, rows_ready: chee_shard_phase1's); an empty piece passes the chunk map on unchanged
static cudaError_t cl_piece_phase1_launch(const ClDecodePiece* s, uint32_t* d_cmap_out, cudaStream_t st, uint64_t* launches,
                                          const uint32_t* d_seed = nullptr, bool rows_ready = false) {
    if (s->a.n) return chee_shard_phase1(s->a, d_cmap_out, st, launches, d_seed, rows_ready);
    return d_cmap_out ? chee_cmap_identity(d_cmap_out, st, launches) : cudaSuccess;
}
static int cl_piece_phase1(ClDecodePiece* s, bool lion, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, int is_first, int is_last,
                           uint32_t* d_cmap_out, void* stream) {
    g_last_error.clear();
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int rc = cl_piece_setup(s, lion, d_in, n, d_out, cap, is_first, is_last, d_cmap_out, false, false, st);
    if (rc != DENSITY_B200_OK) return rc;
    uint64_t launches = 0;
    const cudaError_t e = cl_piece_phase1_launch(s, d_cmap_out, st, &launches);
    rc = step_result(e, launches, "cl decode shard phase1");
    if (rc == DENSITY_B200_OK) s->phase = 1;
    return rc;
}
static int cl_piece_phase2(ClDecodePiece* s, const uint32_t* d_cmap_carry, void* stream) {
    g_last_error.clear();
    if (!s || s->phase != 1) { set_error("cl decode shard phase2: null pointer / phase 1 not done"); return DENSITY_B200_EARG; }
    int rc = table_args({d_cmap_carry});
    if (rc != DENSITY_B200_OK) return rc;
    uint64_t launches = 0;
    const cudaError_t e = s->a.n ? chee_shard_phase2(s->a, d_cmap_carry, reinterpret_cast<cudaStream_t>(stream), &launches) : cudaSuccess;
    rc = step_result(e, launches, "cl decode shard phase2");
    if (rc == DENSITY_B200_OK) s->phase = 2;
    return rc;
}
// ready: the step before phase 3 is done (the wrappers' rule)
static int cl_piece_phase3(ClDecodePiece* s, bool ready, uint64_t* d_out_size, uint32_t* d_seam8, void* stream) {
    g_last_error.clear();
    if (!s || !ready) { set_error("cl decode shard phase3: null pointer / the step before it not done"); return DENSITY_B200_EARG; }
    int rc = out_args(d_out_size, d_seam8);
    if (rc != DENSITY_B200_OK) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    uint64_t launches = 0;
    const uint32_t* seed = s->prot ? reinterpret_cast<const uint32_t*>(s->seed.p) : nullptr;
    const cudaError_t e = (s->a.n || seed) ? chee_shard_phase3(s->a, d_out_size, d_seam8, st, &launches, seed) : empty_piece_outputs(d_out_size, d_seam8, st);
    rc = step_result(e, launches, "cl decode shard phase3");
    if (rc == DENSITY_B200_OK) s->phase = 4;
    return rc;
}

// ---- the same for streams with copy-mode blocks: the piece's protection transfer, then phase 1 from the composed state -------------------
static int cl_piece_prot_transfer(ClDecodePiece* s, bool lion, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, int is_first, int is_last,
                                  uint32_t* d_transfer_out, void* stream) {
    g_last_error.clear();
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    int rc = cl_piece_setup(s, lion, d_in, n, d_out, cap, is_first, is_last, d_transfer_out, true, true, st);
    if (rc != DENSITY_B200_OK) return rc;
    uint64_t launches = 0;
    const cudaError_t e = chee_shard_prot_transfer(s->a, d_transfer_out, st, &launches);
    rc = step_result(e, launches, "cl decode shard prot transfer");
    if (rc == DENSITY_B200_OK) s->transfer_done = true;
    return rc;
}
// The protected phase 1 of the piece set up in s->a (see decode_prot_phase1_body)
static int cl_piece_prot_phase1_body(ClDecodePiece* s, const uint32_t* d_all_transfers, int rank, uint32_t x0, bool rows_ready,
                                     uint32_t* d_cmap_out, cudaStream_t st, const char* what) {
    uint32_t* seed = reinterpret_cast<uint32_t*>(s->seed.p);
    uint64_t launches = 0;
    s->transfer_done = false;   // one phase 1 per transfer
    cudaError_t e = chee_shard_prot_enter(d_all_transfers, (uint32_t)rank, x0, seed, st, &launches);
    if (e == cudaSuccess) e = cl_piece_phase1_launch(s, d_cmap_out, st, &launches, seed, rows_ready);
    const int rc = step_result(e, launches, what);
    if (rc == DENSITY_B200_OK) { s->phase = 1; s->prot = true; }
    return rc;
}
static int cl_piece_prot_phase1(ClDecodePiece* s, const uint32_t* d_all_transfers, int world, int rank, uint32_t* d_cmap_out, void* stream) {
    g_last_error.clear();
    if (!s || !s->transfer_done || s->phase != 0) { set_error("cl decode shard prot_phase1: null pointer / transfer not done"); return DENSITY_B200_EARG; }
    if (world < 1 || rank < 0 || rank >= world || (rank > 0 && !d_all_transfers)) { set_error("bad rank / world or null pointer"); return DENSITY_B200_EARG; }
    const int rc = table_args({d_all_transfers, d_cmap_out});
    if (rc != DENSITY_B200_OK) return rc;
    return cl_piece_prot_phase1_body(s, d_all_transfers, rank, 0, true, d_cmap_out, reinterpret_cast<cudaStream_t>(stream), "cl decode shard prot phase1");
}

// ---- the Cheetah piece: the phases above, the prediction rounds between phase 2 and phase 3, and the entry of a located piece ------------
int density_b200_cheetah_decode_shard_phase1(density_b200_cheetah_decode_shard* s, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                             int is_first, int is_last, uint32_t* d_cmap_out, void* stream) {
    return cl_piece_phase1(s, false, d_in, n, d_out, cap, is_first, is_last, d_cmap_out, stream);
}
int density_b200_cheetah_decode_shard_phase2(density_b200_cheetah_decode_shard* s, const uint32_t* d_cmap_carry, void* stream) {
    return cl_piece_phase2(s, d_cmap_carry, stream);
}
int density_b200_cheetah_decode_shard_round_walk(density_b200_cheetah_decode_shard* s, uint32_t* d_pred_out, uint32_t* d_words4, void* stream) {
    g_last_error.clear();
    if (!s || s->phase != 2) { set_error("cheetah_decode_shard_round_walk: null pointer / phase 2 or the previous round's fold not done"); return DENSITY_B200_EARG; }
    if (!d_words4) { set_error("null pointer"); return DENSITY_B200_EARG; }
    int rc = table_args({d_pred_out, d_words4});
    if (rc != DENSITY_B200_OK) return rc;
    if (s->round >= (uint32_t)g_chee_dec_rounds) { set_error("cheetah_decode_shard_round_walk: round budget used up"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    uint64_t launches = 0;
    cudaError_t e;
    if (s->a.n) e = chee_shard_round_walk(s->a, s->round, d_pred_out, d_words4, st, &launches);
    else {   // an empty piece: the identity transfer, no exit context, nothing walked
        e = cudaMemsetAsync(d_words4, 0, 4 * sizeof(uint32_t), st);
        if (e == cudaSuccess && d_pred_out) e = cudaMemsetAsync(d_pred_out, 0, 2 * 65536 * sizeof(uint32_t), st);
    }
    rc = step_result(e, launches, "cheetah decode shard round walk");
    if (rc == DENSITY_B200_OK) s->phase = 3;
    return rc;
}
int density_b200_cheetah_decode_shard_round_fold(density_b200_cheetah_decode_shard* s, const uint32_t* d_pred_carry, const uint32_t* d_all_words,
                                                 int world, int rank, void* stream) {
    g_last_error.clear();
    if (!s || s->phase != 3) { set_error("cheetah_decode_shard_round_fold: null pointer / the round's walk not done"); return DENSITY_B200_EARG; }
    if (!d_all_words || world < 1 || rank < 0 || rank >= world) { set_error("cheetah_decode_shard_round_fold: null pointer / bad rank or world"); return DENSITY_B200_EARG; }
    int rc = table_args({d_pred_carry, d_all_words});
    if (rc != DENSITY_B200_OK) return rc;
    uint64_t launches = 0;
    const cudaError_t e = s->a.n ? chee_shard_round_fold(s->a, s->round, d_pred_carry, d_all_words, (uint32_t)world, (uint32_t)rank,
                                                         reinterpret_cast<cudaStream_t>(stream), &launches)
                                 : cudaSuccess;
    rc = step_result(e, launches, "cheetah decode shard round fold");
    if (rc == DENSITY_B200_OK) { s->phase = 2; ++s->round; }
    return rc;
}
int density_b200_cheetah_decode_shard_phase3(density_b200_cheetah_decode_shard* s, uint64_t* d_out_size, uint32_t* d_seam8, void* stream) {
    return cl_piece_phase3(s, s && s->phase == 2, d_out_size, d_seam8, stream);     // after phase 2 or the last round's fold
}
int density_b200_cheetah_decode_shard_prot_transfer(density_b200_cheetah_decode_shard* s, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                                    int is_first, int is_last, uint32_t* d_transfer_out, void* stream) {
    return cl_piece_prot_transfer(s, false, d_in, n, d_out, cap, is_first, is_last, d_transfer_out, stream);
}
int density_b200_cheetah_decode_shard_prot_phase1(density_b200_cheetah_decode_shard* s, const uint32_t* d_all_transfers, int world, int rank,
                                                  uint32_t* d_cmap_out, void* stream) {
    return cl_piece_prot_phase1(s, d_all_transfers, world, rank, d_cmap_out, stream);
}
int density_b200_cheetah_decode_shard_prot_enter(density_b200_cheetah_decode_shard* s, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                                 int is_first, int is_last, uint32_t candidate, uint32_t* d_cmap_out, void* stream) {
    g_last_error.clear();
    if (candidate >= DECODE_PROT_TRANSFER_WORDS) { set_error("cheetah_decode_shard_prot_enter: candidate >= 3200"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int rc = cl_piece_setup(s, false, d_in, n, d_out, cap, is_first, is_last, d_cmap_out, false, true, st);
    if (rc != DENSITY_B200_OK) return rc;
    return cl_piece_prot_phase1_body(s, nullptr, 0, candidate, false, d_cmap_out, st, "cheetah decode shard prot enter");
}

int density_b200_cheetah_decode_shard_status(density_b200_cheetah_decode_shard* s, uint32_t* out4) {
    g_last_error.clear();
    if (!s || !out4 || s->phase != 4) { set_error("cheetah_decode_shard_status: null pointer / phase 3 not done"); return DENSITY_B200_EARG; }
    unsigned int raw[8] = {0};
    if (s->a.n) {
        cudaError_t e = cudaDeviceSynchronize();
        if (e == cudaSuccess) e = cudaMemcpy(raw, chee_shard_status_ptr(s->a), sizeof raw, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) { set_error("cheetah_decode_shard_status", e); return DENSITY_B200_ECUDA; }
    } else raw[2] = 1;
    out4[0] = raw[3]; out4[1] = raw[2] && !raw[5]; out4[2] = raw[6]; out4[3] = s->round;
    return DENSITY_B200_OK;
}
int density_b200_cheetah_cmap_init(uint32_t* d_table, void* stream) {
    g_last_error.clear();
    if (!d_table) { set_error("null pointer"); return DENSITY_B200_EARG; }
    uint64_t l = 0;
    const cudaError_t e = chee_cmap_init(d_table, reinterpret_cast<cudaStream_t>(stream), &l);
    return step_result(e, l, "cheetah_cmap_init");
}
int density_b200_cheetah_cmap_fold(uint32_t* d_acc, const uint32_t* d_next, void* stream) {
    g_last_error.clear();
    if (!d_acc || !d_next) { set_error("null pointer"); return DENSITY_B200_EARG; }
    uint64_t l = 0;
    const cudaError_t e = chee_cmap_fold(d_acc, d_next, reinterpret_cast<cudaStream_t>(stream), &l);
    return step_result(e, l, "cheetah_cmap_fold");
}

// ---- the Lion piece: the phases above and the prediction walk between phase 2 and phase 3 ----------------------------------------------
int density_b200_lion_decode_shard_phase1(density_b200_lion_decode_shard* s, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                          int is_first, int is_last, uint32_t* d_cmap_out, void* stream) {
    return cl_piece_phase1(s, true, d_in, n, d_out, cap, is_first, is_last, d_cmap_out, stream);
}
int density_b200_lion_decode_shard_phase2(density_b200_lion_decode_shard* s, const uint32_t* d_cmap_carry, void* stream) {
    return cl_piece_phase2(s, d_cmap_carry, stream);
}
int density_b200_lion_decode_shard_walk(density_b200_lion_decode_shard* s, uint32_t* d_state, void* stream) {
    g_last_error.clear();
    if (!s || s->phase != 2) { set_error("lion_decode_shard_walk: null pointer / phase 2 not done"); return DENSITY_B200_EARG; }
    if (!d_state || !al4(d_state)) { set_error("d_state must be a 4-byte aligned pointer"); return DENSITY_B200_EARG; }
    uint64_t launches = 0;
    const cudaError_t e = s->a.n ? lion_shard_walk(s->a, d_state, reinterpret_cast<cudaStream_t>(stream), &launches) : cudaSuccess;  // empty: unchanged
    const int rc = step_result(e, launches, "lion decode shard walk");
    if (rc == DENSITY_B200_OK) s->phase = 3;
    return rc;
}
int density_b200_lion_state_init(uint32_t* d_state, void* stream) {
    g_last_error.clear();
    if (!d_state || !al4(d_state)) { set_error("d_state must be a 4-byte aligned pointer"); return DENSITY_B200_EARG; }
    return step_result(lion_state_init(d_state, reinterpret_cast<cudaStream_t>(stream)), 0, "lion_state_init");
}
int density_b200_lion_decode_shard_phase3(density_b200_lion_decode_shard* s, uint64_t* d_out_size, uint32_t* d_seam8, void* stream) {
    return cl_piece_phase3(s, s && s->phase == 3, d_out_size, d_seam8, stream);     // after the walk
}
int density_b200_lion_decode_shard_prot_transfer(density_b200_lion_decode_shard* s, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                                 int is_first, int is_last, uint32_t* d_transfer_out, void* stream) {
    return cl_piece_prot_transfer(s, true, d_in, n, d_out, cap, is_first, is_last, d_transfer_out, stream);
}
int density_b200_lion_decode_shard_prot_phase1(density_b200_lion_decode_shard* s, const uint32_t* d_all_transfers, int world, int rank,
                                               uint32_t* d_cmap_out, void* stream) {
    return cl_piece_prot_phase1(s, d_all_transfers, world, rank, d_cmap_out, stream);
}
int density_b200_lion_decode_shard_stats(density_b200_lion_decode_shard* s, uint64_t* out4) {
    g_last_error.clear();
    if (!s || !out4 || s->phase != 4) { set_error("lion_decode_shard_stats: null pointer / phase 3 not done"); return DENSITY_B200_EARG; }
    for (int k = 0; k < 4; ++k) out4[k] = 0;
    if (!s->a.n) return DENSITY_B200_OK;    // an empty piece walks nothing
    cudaError_t e = cudaDeviceSynchronize();
    // the counts follow the ClStatus prefix of the walk's status (8 u32)
    if (e == cudaSuccess) e = cudaMemcpy(out4, static_cast<const uint8_t*>(chee_shard_status_ptr(s->a)) + 32, 4 * sizeof(uint64_t), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { set_error("lion_decode_shard_stats", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}

// ---- sharded Chameleon encode across the GPUs of one box (SURVEY §8e): one process per GPU, NCCL over NVLink ---------------------
// NCCL is resolved at run time from the library that is already in the process (torch loads its bundled libnccl.so.2), else the
// system one: no link-time dependency, one NCCL per process.
namespace {
typedef struct ncclComm* nccl_comm_t;
struct nccl_unique_id { char internal[128]; };
enum { NCCL_UINT8 = 1, NCCL_UINT32 = 3 };
struct NcclApi {
    int (*GetUniqueId)(nccl_unique_id*) = nullptr;
    int (*CommInitRank)(nccl_comm_t*, int, nccl_unique_id, int) = nullptr;
    int (*CommDestroy)(nccl_comm_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t) = nullptr;
    int (*Send)(const void*, size_t, int, int, nccl_comm_t, cudaStream_t) = nullptr;
    int (*Recv)(void*, size_t, int, int, nccl_comm_t, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool ok = false;
};
NcclApi g_nccl;                     // the resolved table
bool g_nccl_resolved = false;       // false: resolve libnccl.so.2 on the next use
std::mutex g_nccl_mu;
std::atomic<int> g_nccl_handles{0}; // live handles with world > 1: the table they use must not change under them
NcclApi nccl_resolve(void* h) {
    NcclApi api;
    auto sym = [&](const char* n) { return dlsym(h, n); };
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(sym("ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(sym("ncclCommInitRank"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(sym("ncclCommDestroy"));
    api.AllGather = reinterpret_cast<decltype(api.AllGather)>(sym("ncclAllGather"));
    api.Send = reinterpret_cast<decltype(api.Send)>(sym("ncclSend"));
    api.Recv = reinterpret_cast<decltype(api.Recv)>(sym("ncclRecv"));
    api.GroupStart = reinterpret_cast<decltype(api.GroupStart)>(sym("ncclGroupStart"));
    api.GroupEnd = reinterpret_cast<decltype(api.GroupEnd)>(sym("ncclGroupEnd"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(sym("ncclGetErrorString"));
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.Send && api.Recv && api.GroupStart && api.GroupEnd;
    return api;
}
NcclApi* nccl_api() {
    std::lock_guard<std::mutex> lk(g_nccl_mu);
    if (!g_nccl_resolved) {
        g_nccl_resolved = true;
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (h) g_nccl = nccl_resolve(h);
    }
    return g_nccl.ok ? &g_nccl : nullptr;
}
bool nccl_check(int rc, const char* what) {
    if (rc == 0) return true;
    NcclApi* a = nccl_api();
    std::string m = std::string(what) + ": " + ((a && a->GetErrorString) ? a->GetErrorString(rc) : "NCCL error");
    dns::set_error(m.c_str());
    return false;
}
}  // namespace

int density_b200_test_set_nccl_library(const char* path) {
    g_last_error.clear();
    std::lock_guard<std::mutex> lk(g_nccl_mu);
    if (g_nccl_handles.load()) { set_error("test_set_nccl_library: a sharded handle with world > 1 is alive"); return DENSITY_B200_EARG; }
    if (!path) { g_nccl = NcclApi(); g_nccl_resolved = false; return DENSITY_B200_OK; }
    void* h = dlopen(path, RTLD_NOW | RTLD_LOCAL);
    if (!h) { set_error(dlerror()); return DENSITY_B200_EARG; }
    const NcclApi api = nccl_resolve(h);
    if (!api.ok || !api.GetErrorString) {
        dlclose(h);
        set_error("test_set_nccl_library: the library lacks an NCCL symbol the sharded drivers use");
        return DENSITY_B200_EARG;
    }
    g_nccl = api; g_nccl_resolved = true;      // the library stays loaded: error strings of earlier calls may point into it
    return DENSITY_B200_OK;
}

struct density_b200_sharded {
    int rank = 0, world = 1, num_sms = 0;
    nccl_comm_t comm = nullptr;
    DevBuf aux;                     // the exchange buffers of the drivers (Exchange)
    // the phase state of each driver, apart from the others', so that the drivers may alternate on one handle
    density_b200_shard* enc = nullptr;                   // density_b200_encode_sharded
    density_b200_shard* prot = nullptr;                  // density_b200_encode_sharded_protected
    density_b200_cl_shard* cl[2] = {nullptr, nullptr};   // Cheetah / Lion of density_b200_encode_sharded_cl
    density_b200_cl_shard* clp[2] = {nullptr, nullptr};  // Cheetah / Lion of density_b200_encode_sharded_cl_protected
    density_b200_decode_shard* dec = nullptr;            // density_b200_decode_sharded[_stream]
    density_b200_decode_shard* pdec = nullptr;           // density_b200_decode_sharded_protected
    density_b200_cheetah_decode_shard* cdec = nullptr;   // density_b200_decode_sharded_cheetah[_stream]
    density_b200_lion_decode_shard* ldec = nullptr;      // density_b200_decode_sharded_lion
    density_b200_lion_decode_shard* lpdec = nullptr;     // density_b200_decode_sharded_lion_protected
    uint64_t* h_offsets = nullptr;  // pinned, world + 1
    uint64_t* h_maps = nullptr;     // pinned, world range maps (the stream decodes)
    cudaEvent_t ev[6] = {};         // stage timing of the last call: start, flag pass, exchange, phase 2 up to emit, emit, gather
    bool timed = false;
};

int density_b200_sharded_unique_id(uint8_t* out128) {
    g_last_error.clear();
    NcclApi* a = nccl_api();
    if (!a || !out128) { set_error("NCCL is not available in this process"); return DENSITY_B200_ECUDA; }
    nccl_unique_id id;
    if (!nccl_check(a->GetUniqueId(&id), "ncclGetUniqueId")) return DENSITY_B200_ECUDA;
    memcpy(out128, id.internal, 128);
    return DENSITY_B200_OK;
}

density_b200_sharded* density_b200_sharded_create(const uint8_t* nccl_unique_id_128, int rank, int world) {
    g_last_error.clear();
    if (world < 1 || rank < 0 || rank >= world) { set_error("bad rank / world"); return nullptr; }
    DeviceCtx* c = current_ctx();
    if (!c) return nullptr;
    density_b200_sharded* h = new density_b200_sharded();
    h->rank = rank; h->world = world; h->num_sms = c->num_sms;
    if (world > 1) {
        NcclApi* a = nccl_api();
        if (!a || !nccl_unique_id_128) { set_error("NCCL is not available / no unique id"); delete h; return nullptr; }
        nccl_unique_id id; memcpy(id.internal, nccl_unique_id_128, 128);
        if (!nccl_check(a->CommInitRank(&h->comm, world, id, rank), "ncclCommInitRank")) { delete h; return nullptr; }
        ++g_nccl_handles;
    }
    if (cudaMallocHost(&h->h_offsets, sizeof(uint64_t) * (world + 2)) != cudaSuccess ||
        cudaMallocHost(&h->h_maps, sizeof(uint64_t) * DENSITY_B200_LOCATE_MAP_WORDS * world) != cudaSuccess) {
        set_error("cudaMallocHost");
        density_b200_sharded_destroy(h);
        return nullptr;
    }
    h->enc = density_b200_shard_create(); h->prot = density_b200_shard_create();
    h->cl[0] = density_b200_cl_shard_create(ALG_CHEETAH); h->cl[1] = density_b200_cl_shard_create(ALG_LION);
    h->clp[0] = density_b200_cl_shard_create(ALG_CHEETAH); h->clp[1] = density_b200_cl_shard_create(ALG_LION);
    h->dec = density_b200_decode_shard_create(); h->pdec = density_b200_decode_shard_create(); h->cdec = density_b200_cheetah_decode_shard_create();
    h->ldec = density_b200_lion_decode_shard_create(); h->lpdec = density_b200_lion_decode_shard_create();
    for (auto& e : h->ev) cudaEventCreate(&e);
    return h;
}

void density_b200_sharded_destroy(density_b200_sharded* h) {
    if (!h) return;
    if (h->comm) { NcclApi* a = nccl_api(); if (a) a->CommDestroy(h->comm); --g_nccl_handles; }
    h->aux.release();
    density_b200_shard_destroy(h->enc);
    density_b200_shard_destroy(h->prot);
    for (auto* s : h->cl) density_b200_cl_shard_destroy(s);
    for (auto* s : h->clp) density_b200_cl_shard_destroy(s);
    density_b200_decode_shard_destroy(h->dec);
    density_b200_decode_shard_destroy(h->pdec);
    density_b200_cheetah_decode_shard_destroy(h->cdec);
    density_b200_lion_decode_shard_destroy(h->ldec);
    density_b200_lion_decode_shard_destroy(h->lpdec);
    if (h->h_offsets) cudaFreeHost(h->h_offsets);
    if (h->h_maps) cudaFreeHost(h->h_maps);
    for (auto& e : h->ev) if (e) cudaEventDestroy(e);
    delete h;
}

// The collectives of one driver call on the handle's communicator, enqueued on `st`, and the exchange buffers they share. Every rank
// issues the same collectives in the same order (include/density_b200.h lists them per driver); all of them are all-gathers but the
// grouped send / recv of gather_pieces.
struct Exchange {
    density_b200_sharded* h = nullptr;
    cudaStream_t st = nullptr;
    NcclApi* a = nullptr;               // NULL with world == 1
    uint32_t *tables = nullptr, *carry = nullptr, *words = nullptr;   // [world][65536] tables, [65536] carry-in, [world][8] seam words
    uint64_t *offsets = nullptr, *maps = nullptr;                     // [world + 2] piece offsets, [world][LOCATE_MAP_WORDS] range maps
    uint8_t* extra = nullptr;           // the driver's own exchange buffers

    // NCCL (world > 1) and the buffers, extra_bytes of them the driver's; DENSITY_B200_ECUDA with the error set when either is missing
    int open(density_b200_sharded* handle, void* stream, size_t extra_bytes = 0) {
        h = handle; st = reinterpret_cast<cudaStream_t>(stream);
        a = h->world > 1 ? nccl_api() : nullptr;
        if (h->world > 1 && !a) { set_error("NCCL is not available"); return DENSITY_B200_ECUDA; }
        const size_t W = (size_t)h->world;
        const size_t n_tables = W * 65536, n_carry = 65536, n_words = W * 8, n_offsets = W + 2;
        size_t bytes = (n_tables + n_carry + n_words) * sizeof(uint32_t) + (n_offsets + W * DENSITY_B200_LOCATE_MAP_WORDS) * sizeof(uint64_t);
        bytes = (bytes + 255) & ~(size_t)255;
        const cudaError_t e = h->aux.ensure(bytes + extra_bytes + 256, st);
        if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
        tables = reinterpret_cast<uint32_t*>(h->aux.p);
        carry = tables + n_tables;
        words = carry + n_carry;
        offsets = reinterpret_cast<uint64_t*>(words + n_words);
        maps = offsets + n_offsets;
        extra = h->aux.p + bytes;
        return DENSITY_B200_OK;
    }
    // this rank's slot of buf ([world][n] u32) to every rank
    bool gather(uint32_t* buf, size_t n, const char* what) const {
        return h->world == 1 || nccl_check(a->AllGather(buf + (size_t)h->rank * n, buf, n, NCCL_UINT32, h->comm, st), what);
    }
    uint32_t* my_words() const { return words + 8 * (size_t)h->rank; }
    // this rank's Chameleon table (its slot of `tables`) to every rank, then one fold kernel: `carry` = the dictionary before this rank
    int fold_tables(const char* what) const {
        if (!gather(tables, 65536, "ncclAllGather(tables)")) return DENSITY_B200_ECUDA;
        uint64_t launches = 0;
        const cudaError_t e = cham_rank_fold(tables, (uint32_t)h->rank, carry, st, &launches);
        return step_result(e, launches, what);
    }
    // this rank's Cheetah / Lion table of `kind` (its slot of tabs, [world][table words]) to every rank, then one fold kernel: *carry =
    // the state before this rank
    int fold_cl_tables(int alg, int kind, uint32_t* tabs, uint32_t* carry_out, const char* what) const {
        const bool p = kind == DENSITY_B200_CL_TABLE_P;
        if (!gather(tabs, density_b200_cl_table_words(alg, kind), p ? "ncclAllGather(P tables)" : "ncclAllGather(C tables)")) return DENSITY_B200_ECUDA;
        uint64_t launches = 0;
        const cudaError_t e = cl_rank_fold(alg, kind, tabs, (uint32_t)h->rank, carry_out, st, &launches);
        return step_result(e, launches, what);
    }
    // this rank's shard length n to every rank: lengths[world] u64
    int exchange_lengths(uint64_t* lengths, size_t n, const char* what) const {
        uint64_t launches = 0;
        const cudaError_t e = cham_put_u64(lengths + h->rank, (uint64_t)n, st, &launches);
        const int rc = step_result(e, launches, what);
        if (rc != DENSITY_B200_OK) return rc;
        return gather(reinterpret_cast<uint32_t*>(lengths), 2, "ncclAllGather(lengths)") ? DENSITY_B200_OK : DENSITY_B200_ECUDA;
    }
    // this rank's seam words (my_words) to every rank -> the verdict over all pieces; *d_out_offset (may be NULL) = where this rank's
    // output starts
    int verdict(uint32_t* d_flags, uint64_t* d_total_size, uint64_t* d_out_offset) const {
        if (!gather(words, 8, "ncclAllGather(seams)")) return DENSITY_B200_ECUDA;
        uint64_t launches = 0;
        cudaError_t e = cham_seam_verdict(words, (uint32_t)h->world, (uint32_t)h->rank, d_flags, d_total_size, offsets, st, &launches);
        if (e == cudaSuccess && d_out_offset) e = cudaMemcpyAsync(d_out_offset, offsets + h->rank, sizeof(uint64_t), cudaMemcpyDeviceToDevice, st);
        return step_result(e, launches, "seam verdict");
    }
    // this rank's range map (map_words u64 in its slot of `maps`) to every rank, then all of them to h->h_maps: the call's one host
    // synchronisation
    int maps_to_host(size_t map_words) const {
        if (!gather(reinterpret_cast<uint32_t*>(maps), 2 * map_words, "ncclAllGather(maps)")) return DENSITY_B200_ECUDA;
        cudaError_t e = cudaMemcpyAsync(h->h_maps, maps, (size_t)h->world * map_words * sizeof(uint64_t), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        return step_result(e, 0, "range maps to host");
    }
};

// variable-length gather of the pieces to `gather_root` at their stream offsets (d_offsets: world + 1 prefix sums, d_words: the gathered
// seam words, whose words 6-7 of the root's row hold its gather_cap; both on the device); blocks. The capacity check is collective:
// every rank reads the root's capacity, so when it is short all of them return DENSITY_B200_ECAPACITY and none posts a send that no
// receive would ever match.
static int gather_pieces(density_b200_sharded* h, NcclApi* a, const uint64_t* d_offsets, const uint32_t* d_words, const uint8_t* d_out,
                         int gather_root, uint8_t* d_gather, cudaStream_t st) {
    const size_t W = (size_t)h->world;
    cudaError_t e;
    // variable-length gather of the pieces at their stream offsets (SURVEY §8e step 5): sizes -> host -> grouped send / recv
    e = cudaMemcpyAsync(h->h_offsets, d_offsets, (W + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->h_offsets + W + 1, d_words + 8 * (size_t)gather_root + 6, sizeof(uint64_t), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("gather: sizes to host", e); return DENSITY_B200_ECUDA; }
    const uint64_t total = h->h_offsets[W], root_cap = h->h_offsets[W + 1];
    const uint64_t my_off = h->h_offsets[h->rank], my_size = h->h_offsets[h->rank + 1] - my_off;
    if (root_cap < total) { set_error("gather buffer too small"); return DENSITY_B200_ECAPACITY; }
    if (h->rank == gather_root) {
        if (my_size) e = cudaMemcpyAsync(d_gather + my_off, d_out, my_size, cudaMemcpyDeviceToDevice, st);
        if (e != cudaSuccess) { set_error("gather: local piece", e); return DENSITY_B200_ECUDA; }
    }
    if (h->world > 1) {
        if (!nccl_check(a->GroupStart(), "ncclGroupStart")) return DENSITY_B200_ECUDA;
        bool ok = true;
        if (h->rank == gather_root) {
            for (int r = 0; r < h->world && ok; ++r) {
                const uint64_t sz = h->h_offsets[r + 1] - h->h_offsets[r];
                if (r != h->rank && sz) ok = nccl_check(a->Recv(d_gather + h->h_offsets[r], sz, NCCL_UINT8, r, h->comm, st), "ncclRecv");
            }
        } else if (my_size) ok = nccl_check(a->Send(d_out, my_size, NCCL_UINT8, gather_root, h->comm, st), "ncclSend");
        if (!nccl_check(a->GroupEnd(), "ncclGroupEnd") || !ok) return DENSITY_B200_ECUDA;
    }
    return DENSITY_B200_OK;
}

// the argument checks of the sharded encoders, every one of them before the first collective: a rank that returned EARG half way
// through would leave the others waiting in an all-gather. cl: a Cheetah / Lion driver, whose alg must be one of those two.
static int encode_sharded_args(density_b200_sharded* h, bool cl, int alg, const uint8_t* d_in, size_t n, const uint8_t* d_out,
                               const uint64_t* d_out_size, const uint32_t* d_flags, const uint64_t* d_total_size, int gather_root,
                               const uint8_t* d_gather) {
    if (!h || !d_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (cl && !cl_alg_ok(alg)) { set_error("encode_sharded_cl: alg must be DENSITY_B200_CHEETAH or DENSITY_B200_LION"); return DENSITY_B200_EARG; }
    int rc = in_args(true, d_in, n, d_out, 0, h->rank == h->world - 1);
    if (rc == DENSITY_B200_OK) rc = size_args(d_out_size, d_total_size);
    if (rc == DENSITY_B200_OK) rc = table_args({d_flags});
    if (rc != DENSITY_B200_OK) return rc;
    if (gather_root >= h->world) { set_error("bad gather root"); return DENSITY_B200_EARG; }
    if (h->rank == gather_root && !d_gather) { set_error("null pointer: d_gather on the gather root"); return DENSITY_B200_EARG; }
    return DENSITY_B200_OK;
}

// the end of every sharded encode: the verdict, the optional gather of the pieces to gather_root, the last stage event. The root's
// gather_cap travels to every rank in words 6-7 of its seam words (zero otherwise), so that all ranks judge the capacity alike.
static int encode_sharded_end(const Exchange& x, const uint8_t* d_out, uint32_t* d_flags, uint64_t* d_total_size, int gather_root,
                              uint8_t* d_gather, size_t gather_cap) {
    if (x.h->rank == gather_root) {
        const uint64_t cap = gather_cap;        // pageable: consumed before cudaMemcpyAsync returns
        const cudaError_t e = cudaMemcpyAsync(x.my_words() + 6, &cap, sizeof cap, cudaMemcpyHostToDevice, x.st);
        if (e != cudaSuccess) { set_error("gather capacity to the seam words", e); return DENSITY_B200_ECUDA; }
    }
    int rc = x.verdict(d_flags, d_total_size, nullptr);
    if (rc == DENSITY_B200_OK && gather_root >= 0) rc = gather_pieces(x.h, x.a, x.offsets, x.words, d_out, gather_root, d_gather, x.st);
    if (rc != DENSITY_B200_OK) return rc;
    cudaEventRecord(x.h->ev[5], x.st);
    x.h->timed = true;
    return DENSITY_B200_OK;
}

// One bit-exact stream cut across `world` GPUs; this rank's shard is d_in[0 .. n) (n % 256 == 0 except on the last rank).
// All work is enqueued on `stream`. With gather_root >= 0 the call BLOCKS on the stream once (the piece sizes must reach the host before
// the variable-length ncclSend / ncclRecv can be posted) and the pieces land in d_gather on rank gather_root at their stream offsets.
int density_b200_encode_sharded(density_b200_sharded* h, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                uint32_t* d_flags, uint64_t* d_total_size, int gather_root, uint8_t* d_gather, size_t gather_cap, void* stream_v) {
    g_last_error.clear();
    int rc = encode_sharded_args(h, false, ALG_CHAMELEON, d_in, n, d_out, d_out_size, d_flags, d_total_size, gather_root, d_gather);
    Exchange x;
    if (rc != DENSITY_B200_OK || (rc = x.open(h, stream_v)) != DENSITY_B200_OK) return rc;
    density_b200_shard* s = h->enc;
    cudaEventRecord(h->ev[0], x.st);
    // phase 1: flags with unknown carry-in; my last-writer table lands in my slot of the gather buffer
    rc = density_b200_shard_phase1(s, d_in, n, h->rank == h->world - 1, x.tables + (size_t)h->rank * 65536, x.st);
    if (rc != DENSITY_B200_OK) return rc;
    cudaEventRecord(h->ev[1], x.st);
    // the one exchange step of the path: 256 KiB per rank over NVLink, then ONE fold kernel
    if ((rc = x.fold_tables("sharded fold")) != DENSITY_B200_OK) return rc;
    cudaEventRecord(h->ev[2], x.st);
    // phase 2: carry-in, first-touch flags, sizes, scan, emit (seams are judged below, exactly, once every shard knows its flags)
    cudaEvent_t pev[4] = {nullptr, nullptr, h->ev[3], h->ev[4]};
    if ((rc = shard_phase2_impl(s, x.carry, d_out, cap, d_out_size, false, n ? pev : nullptr, x.st)) != DENSITY_B200_OK) return rc;
    if (!n) { cudaEventRecord(h->ev[3], x.st); cudaEventRecord(h->ev[4], x.st); }
    uint64_t launches = 0;
    cudaError_t e;
    if (n) e = cham_seam_words(s->ws.p, s->L, n, d_out_size, x.my_words(), x.st, &launches);
    else e = cudaMemsetAsync(x.my_words(), 0, 8 * sizeof(uint32_t), x.st);
    if ((rc = step_result(e, launches, "sharded seam words")) != DENSITY_B200_OK) return rc;
    return encode_sharded_end(x, d_out, d_flags, d_total_size, gather_root, d_gather, gather_cap);
}

// The exchange buffers of the Cheetah / Lion encode drivers behind Exchange::extra (extra: nullptr for the size alone), in this order:
// prot: the shard lengths [world] u64; the gathered P tables [world][P words] and their carry, the gathered C tables [world][C words]
// and their carry; then quiet: the last quads [world][2] and the previous quad (one word of the 64 behind the buffers); prot: the
// transfers [world][PROT_TRANSFER_WORDS] and the round words [world][CL_PROT_ROUND_WORDS].
struct ClEncodeBufs {
    uint64_t* lengths;
    uint32_t *tab_p, *carry_p, *tab_c, *carry_c, *quads, *prev_quad, *transfers, *rwords;
    size_t bytes;
};
static ClEncodeBufs cl_encode_bufs(int alg, size_t world, bool prot, uint8_t* extra = nullptr) {
    ClEncodeBufs b{};
    size_t off = 0;    // u32 words
    auto take = [&](size_t words) { uint32_t* p = extra ? reinterpret_cast<uint32_t*>(extra) + off : nullptr; off += words; return p; };
    const size_t wp = density_b200_cl_table_words(alg, DENSITY_B200_CL_TABLE_P), wc = density_b200_cl_table_words(alg, DENSITY_B200_CL_TABLE_C);
    if (prot) b.lengths = reinterpret_cast<uint64_t*>(take(2 * world));
    b.tab_p = take(world * wp);
    b.carry_p = take(wp);
    b.tab_c = take(world * wc);
    b.carry_c = take(wc);
    if (prot) {
        b.transfers = take(world * PROT_TRANSFER_WORDS);
        b.rwords = take(world * CL_PROT_ROUND_WORDS);
    } else {
        b.quads = take(2 * world);
        b.prev_quad = take(0);
    }
    b.bytes = (off + 64) * sizeof(uint32_t);
    return b;
}

// Sharded Cheetah / Lion encode over the handle's communicator: last quads -> phase 1 -> P tables -> fold -> phase 2 -> C tables -> fold
// -> phase 3 -> seam words -> verdict -> optional gather, as density_b200_encode_sharded. The exchanges are ncclAllGathers on `stream`.
int density_b200_encode_sharded_cl(density_b200_sharded* h, int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                   uint32_t* d_flags, uint64_t* d_total_size, int gather_root, uint8_t* d_gather, size_t gather_cap, void* stream_v) {
    g_last_error.clear();
    int rc = encode_sharded_args(h, true, alg, d_in, n, d_out, d_out_size, d_flags, d_total_size, gather_root, d_gather);
    if (rc != DENSITY_B200_OK) return rc;
    density_b200_cl_shard* s = h->cl[alg - ALG_CHEETAH];
    const size_t W = (size_t)h->world, R = (size_t)h->rank;
    const size_t wp = density_b200_cl_table_words(alg, DENSITY_B200_CL_TABLE_P), wc = density_b200_cl_table_words(alg, DENSITY_B200_CL_TABLE_C);
    Exchange x;
    if ((rc = x.open(h, stream_v, cl_encode_bufs(alg, W, false).bytes)) != DENSITY_B200_OK) return rc;
    cudaStream_t st = x.st;
    const ClEncodeBufs b = cl_encode_bufs(alg, W, false, x.extra);
    uint64_t launches = 0;
    // 0. the context of my first quad: the last quad of the nearest earlier shard that has one
    cudaError_t e = cl_last_quad(d_in, n, b.quads + 2 * R, st, &launches);
    if (e == cudaSuccess && !x.gather(b.quads, 2, "ncclAllGather(last quads)")) return DENSITY_B200_ECUDA;
    if (e == cudaSuccess) e = cl_prev_quad(b.quads, (uint32_t)R, b.prev_quad, st, &launches);
    if ((rc = step_result(e, launches, "sharded cl: last quads")) != DENSITY_B200_OK) return rc;
    // 1-2. predictions, exchange, fold
    cudaEventRecord(h->ev[0], st);
    if ((rc = density_b200_cl_shard_phase1(s, d_in, n, R == W - 1, R ? b.prev_quad : nullptr, b.tab_p + R * wp, st)) != DENSITY_B200_OK) return rc;
    cudaEventRecord(h->ev[1], st);
    if ((rc = x.fold_cl_tables(alg, DENSITY_B200_CL_TABLE_P, b.tab_p, b.carry_p, "sharded cl: P fold")) != DENSITY_B200_OK) return rc;
    cudaEventRecord(h->ev[2], st);
    // 3-4. chunk map, exchange, fold
    if ((rc = density_b200_cl_shard_phase2(s, b.carry_p, b.tab_c + R * wc, st)) != DENSITY_B200_OK) return rc;
    if ((rc = x.fold_cl_tables(alg, DENSITY_B200_CL_TABLE_C, b.tab_c, b.carry_c, "sharded cl: C fold")) != DENSITY_B200_OK) return rc;
    cudaEventRecord(h->ev[3], st);
    // 5. emit and seam words, the verdict over all shards, the optional gather
    if ((rc = density_b200_cl_shard_phase3(s, b.carry_c, d_out, cap, d_out_size, x.my_words(), st)) != DENSITY_B200_OK) return rc;
    cudaEventRecord(h->ev[4], st);
    return encode_sharded_end(x, d_out, d_flags, d_total_size, gather_root, d_gather, gather_cap);
}

// Sharded Chameleon encode with copy mode over the handle's communicator: the shard lengths -> phase 1 -> the round budget of
// {tables -> fold -> transfer -> transfers -> settle -> round words -> commit (+ next round's flags)} -> finish -> seam words -> verdict
// -> optional gather. Every rank runs the same rounds, so the collectives match; the gates keep the settled rounds cheap.
int density_b200_encode_sharded_protected(density_b200_sharded* h, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                          uint32_t* d_flags, uint64_t* d_total_size, int gather_root, uint8_t* d_gather, size_t gather_cap,
                                          void* stream_v) {
    g_last_error.clear();
    int rc = encode_sharded_args(h, false, ALG_CHAMELEON, d_in, n, d_out, d_out_size, d_flags, d_total_size, gather_root, d_gather);
    if (rc != DENSITY_B200_OK) return rc;
    density_b200_shard* s = h->prot;
    const size_t W = (size_t)h->world, R = (size_t)h->rank;
    Exchange x;
    if ((rc = x.open(h, stream_v, W * (2 * sizeof(uint64_t) + (PROT_TRANSFER_WORDS + PROT_ROUND_WORDS) * sizeof(uint32_t)))) != DENSITY_B200_OK) return rc;
    cudaStream_t st = x.st;
    // the workspace and the record before the first collective (DevBuf::ensure may cudaFree, which waits for the device); phase 1 finds
    // them in place
    if ((rc = cham_shard_setup(s, d_in, n, true, st)) != DENSITY_B200_OK) return rc;
    uint64_t* lengths = reinterpret_cast<uint64_t*>(x.extra);                         // [world]
    uint32_t* transfers = reinterpret_cast<uint32_t*>(lengths + W);                   // [world][PROT_TRANSFER_WORDS]
    uint32_t* rwords = transfers + W * PROT_TRANSFER_WORDS;                          // [world][PROT_ROUND_WORDS]
    uint32_t* my_table = x.tables + R * 65536;
    cudaEventRecord(h->ev[0], st);
    if ((rc = x.exchange_lengths(lengths, n, "sharded protected: length")) != DENSITY_B200_OK) return rc;
    if ((rc = prot_phase1_impl(s, d_in, n, 0, lengths, (int)R, R == W - 1, my_table, st)) != DENSITY_B200_OK) return rc;
    cudaEventRecord(h->ev[1], st);
    for (int k = 0; k < g_prot_rounds; ++k) {
        if (k > 0 && (rc = density_b200_shard_prot_next(s, rwords, (int)W, my_table, st)) != DENSITY_B200_OK) return rc;
        if ((rc = x.fold_tables("sharded protected: fold")) != DENSITY_B200_OK) return rc;
        if (k == 0) cudaEventRecord(h->ev[2], st);
        if ((rc = density_b200_shard_prot_transfer(s, x.carry, transfers + R * PROT_TRANSFER_WORDS, st)) != DENSITY_B200_OK) return rc;
        if (!x.gather(transfers, PROT_TRANSFER_WORDS, "ncclAllGather(transfers)")) return DENSITY_B200_ECUDA;
        if ((rc = density_b200_shard_prot_settle(s, transfers, (int)W, (int)R, rwords + R * PROT_ROUND_WORDS, st)) != DENSITY_B200_OK) return rc;
        if (!x.gather(rwords, PROT_ROUND_WORDS, "ncclAllGather(round words)")) return DENSITY_B200_ECUDA;
    }
    if ((rc = density_b200_shard_prot_next(s, rwords, (int)W, nullptr, st)) != DENSITY_B200_OK) return rc;
    cudaEvent_t pev[4] = {nullptr, nullptr, h->ev[3], h->ev[4]};
    if ((rc = prot_finish_impl(s, d_out, cap, d_out_size, x.my_words(), st, n ? pev : nullptr)) != DENSITY_B200_OK) return rc;
    if (!n) { cudaEventRecord(h->ev[3], st); cudaEventRecord(h->ev[4], st); }
    return encode_sharded_end(x, d_out, d_flags, d_total_size, gather_root, d_gather, gather_cap);
}

// Sharded Cheetah / Lion encode with copy mode over the handle's communicator: the shard lengths (to the host: the shard at the stream start
// runs the staged iteration) -> phase 1 -> its round words -> the round budget of {P tables -> fold -> C tables -> fold -> transfers ->
// round words -> commit} -> finish -> seam words -> verdict -> optional gather. Every rank runs the same rounds, so the collectives match.
int density_b200_encode_sharded_cl_protected(density_b200_sharded* h, int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                             uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, int gather_root, uint8_t* d_gather,
                                             size_t gather_cap, void* stream_v) {
    g_last_error.clear();
    int rc = encode_sharded_args(h, true, alg, d_in, n, d_out, d_out_size, d_flags, d_total_size, gather_root, d_gather);
    if (rc != DENSITY_B200_OK) return rc;
    density_b200_cl_shard* s = h->clp[alg - ALG_CHEETAH];
    const size_t W = (size_t)h->world, R = (size_t)h->rank;
    const size_t wp = density_b200_cl_table_words(alg, DENSITY_B200_CL_TABLE_P), wc = density_b200_cl_table_words(alg, DENSITY_B200_CL_TABLE_C);
    const size_t rw = CL_PROT_ROUND_WORDS;
    Exchange x;
    if ((rc = x.open(h, stream_v, cl_encode_bufs(alg, W, true).bytes)) != DENSITY_B200_OK) return rc;
    cudaStream_t st = x.st;
    const ClEncodeBufs b = cl_encode_bufs(alg, W, true, x.extra);
    cudaEventRecord(h->ev[0], st);
    // the byte offset of my shard, on the host: whether this shard holds the stream start decides what phase 1 enqueues
    if ((rc = x.exchange_lengths(b.lengths, n, "sharded cl protected: length")) != DENSITY_B200_OK) return rc;
    cudaError_t e = cudaMemcpyAsync(h->h_offsets, b.lengths, W * sizeof(uint64_t), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if ((rc = step_result(e, 0, "sharded cl protected: lengths to host")) != DENSITY_B200_OK) return rc;
    uint64_t offset = 0;
    for (size_t r = 0; r < R; ++r) offset += h->h_offsets[r];
    if ((rc = density_b200_cl_shard_prot_phase1(s, d_in, n, offset, R == W - 1, b.rwords + R * rw, st)) != DENSITY_B200_OK) return rc;
    if (!x.gather(b.rwords, rw, "ncclAllGather(round words)")) return DENSITY_B200_ECUDA;
    cudaEventRecord(h->ev[1], st);
    for (int k = 0; k < g_prot_rounds; ++k) {
        if ((rc = density_b200_cl_shard_prot_p(s, b.rwords, (int)W, (int)R, b.tab_p + R * wp, st)) != DENSITY_B200_OK) return rc;
        if ((rc = x.fold_cl_tables(alg, DENSITY_B200_CL_TABLE_P, b.tab_p, b.carry_p, "sharded cl protected: P fold")) != DENSITY_B200_OK) return rc;
        if (k == 0) cudaEventRecord(h->ev[2], st);
        if ((rc = density_b200_cl_shard_prot_c(s, b.carry_p, b.tab_c + R * wc, st)) != DENSITY_B200_OK) return rc;
        if ((rc = x.fold_cl_tables(alg, DENSITY_B200_CL_TABLE_C, b.tab_c, b.carry_c, "sharded cl protected: C fold")) != DENSITY_B200_OK) return rc;
        if ((rc = density_b200_cl_shard_prot_transfer(s, b.carry_c, b.transfers + R * PROT_TRANSFER_WORDS, st)) != DENSITY_B200_OK) return rc;
        if (!x.gather(b.transfers, PROT_TRANSFER_WORDS, "ncclAllGather(transfers)")) return DENSITY_B200_ECUDA;
        if ((rc = density_b200_cl_shard_prot_settle(s, b.transfers, (int)W, (int)R, b.rwords + R * rw, st)) != DENSITY_B200_OK) return rc;
        if (!x.gather(b.rwords, rw, "ncclAllGather(round words)")) return DENSITY_B200_ECUDA;
        if ((rc = density_b200_cl_shard_prot_next(s, b.rwords, (int)W, st)) != DENSITY_B200_OK) return rc;
    }
    if ((rc = cl_prot_finish_impl(s, d_out, cap, d_out_size, x.my_words(), st, h->ev[3])) != DENSITY_B200_OK) return rc;
    cudaEventRecord(h->ev[4], st);
    return encode_sharded_end(x, d_out, d_flags, d_total_size, gather_root, d_gather, gather_cap);
}

// the argument checks of the sharded decoders; n: the bytes of d_in
static int decode_sharded_args(density_b200_sharded* h, const uint8_t* d_in, size_t n, const uint8_t* d_out, size_t cap, const uint64_t* d_out_size,
                               const uint32_t* d_flags) {
    if (!h || !d_out_size || !d_flags) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (!al8(d_out_size)) { set_error("d_out_size must be 8-byte aligned"); return DENSITY_B200_EARG; }
    return in_args(false, d_in, n, d_out, cap);
}

// The decode of this rank's piece d_in[0 .. n) with the dictionary carried in from the pieces before it:
//   head  [prot: prot_transfer -> ncclAllGather(transfers) -> prot_phase1 | cand >= 0: prot_enter from that candidate (a located piece of a
//         stream with copy-mode blocks, density_b200_decode_sharded_stream_protected) | phase 1]
//   tail  table exchange -> fold -> phase 2 (prot_phase2 after either protected head) -> seam words -> verdict
// The protected heads run on the handle's protected decode shard; prot: x is opened with [world][DECODE_PROT_TRANSFER_WORDS] u32 of extra
// bytes for the transfers. is_last: the piece ends the stream (a non-final piece must decode to whole 256-byte blocks). d_out_offset
// (may be NULL): where the piece's output starts, from the verdict's prefix offsets.
static int decode_sharded_piece(const Exchange& x, const uint8_t* d_in, size_t n, int is_last, uint8_t* d_out, size_t cap,
                                uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, uint64_t* d_out_offset, bool prot,
                                int64_t cand = -1) {
    const bool seeded = prot || cand >= 0;
    density_b200_decode_shard* s = seeded ? x.h->pdec : x.h->dec;
    const size_t R = (size_t)x.h->rank;
    uint32_t* my_table = x.tables + R * 65536;
    // phase 1: boundaries and writer pass need no carry-in; the piece's table (runs + tail) lands in my slot of the gather buffer
    int rc;
    if (prot) {
        uint32_t* transfers = reinterpret_cast<uint32_t*>(x.extra);
        rc = density_b200_decode_shard_prot_transfer(s, d_in, n, cap, is_last, transfers + R * DECODE_PROT_TRANSFER_WORDS, x.st);
        if (rc != DENSITY_B200_OK) return rc;
        if (!x.gather(transfers, DECODE_PROT_TRANSFER_WORDS, "ncclAllGather(transfers)")) return DENSITY_B200_ECUDA;
        rc = density_b200_decode_shard_prot_phase1(s, transfers, x.h->world, (int)R, my_table, x.st);
    } else if (cand >= 0) {
        rc = density_b200_decode_shard_prot_enter(s, d_in, n, cap, is_last, (uint32_t)cand, my_table, x.st);
    } else {
        rc = density_b200_decode_shard_phase1(s, d_in, n, cap, is_last, my_table, x.st);
    }
    if (rc != DENSITY_B200_OK) return rc;
    if ((rc = x.fold_tables("sharded decode fold")) != DENSITY_B200_OK) return rc;
    // phase 2: decode from the carried-in dictionary, then the seam words; the verdict reads them from every rank
    rc = seeded ? density_b200_decode_shard_prot_phase2(s, x.carry, d_out, d_out_size, x.my_words(), x.st)
                : density_b200_decode_shard_phase2(s, x.carry, d_out, d_out_size, x.my_words(), x.st);
    if (rc != DENSITY_B200_OK) return rc;
    return x.verdict(d_flags, d_total_size, d_out_offset);
}

// The inverse of density_b200_encode_sharded without a gather: this rank's piece d_in[0 .. n) decodes to the shard it was encoded from.
// Everything is enqueued on `stream`; nothing blocks.
int density_b200_decode_sharded(density_b200_sharded* h, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                uint32_t* d_flags, uint64_t* d_total_size, void* stream_v) {
    g_last_error.clear();
    int rc = decode_sharded_args(h, d_in, n, d_out, cap, d_out_size, d_flags);
    Exchange x;
    if (rc != DENSITY_B200_OK || (rc = x.open(h, stream_v)) != DENSITY_B200_OK) return rc;
    return decode_sharded_piece(x, d_in, n, h->rank == h->world - 1, d_out, cap, d_out_size, d_flags, d_total_size, nullptr, false);
}

// The inverse of density_b200_encode_sharded_protected (any stream): transfer -> transfers exchange -> phase 1 from the composed state ->
// table exchange -> fold -> phase 2 -> seam words -> verdict. Everything is enqueued on `stream`; nothing blocks.
int density_b200_decode_sharded_protected(density_b200_sharded* h, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                          uint32_t* d_flags, uint64_t* d_total_size, void* stream_v) {
    g_last_error.clear();
    int rc = decode_sharded_args(h, d_in, n, d_out, cap, d_out_size, d_flags);
    Exchange x;
    if (rc != DENSITY_B200_OK || (rc = x.open(h, stream_v, (size_t)h->world * DECODE_PROT_TRANSFER_WORDS * sizeof(uint32_t))) != DENSITY_B200_OK) return rc;
    return decode_sharded_piece(x, d_in, n, h->rank == h->world - 1, d_out, cap, d_out_size, d_flags, d_total_size, nullptr, true);
}

// The exchange buffers of decode_sharded_cl_piece behind Exchange::extra (extra: nullptr for the size alone), in this order: the gathered
// chunk-map transfers [world][cmap words] and the carry; Cheetah: the gathered prediction transfers [world][2 * 65536], their carry and
// the round words [world][4]; Lion: the walk state (DENSITY_B200_LION_STATE_WORDS); then with prot the gathered protection transfers
// [world][DECODE_PROT_TRANSFER_WORDS], with map_words the range maps [world][map_words] and the composition's 8 u64 words.
struct ClPieceBufs {
    uint32_t *tab_c, *carry_c, *tab_p, *carry_p, *rwords, *state, *transfers, *maps;
    size_t bytes;
};
static ClPieceBufs cl_piece_bufs(int alg, size_t world, bool prot, size_t map_words, uint8_t* extra = nullptr) {
    ClPieceBufs b{};
    size_t off = 0;    // u32 words
    auto take = [&](size_t words) { uint32_t* p = extra ? reinterpret_cast<uint32_t*>(extra) + off : nullptr; off += words; return p; };
    const size_t wc = density_b200_cheetah_cmap_words(), wp = 2 * 65536;
    b.tab_c = take(world * wc);
    b.carry_c = take(wc);
    if (alg == ALG_CHEETAH) {
        b.tab_p = take(world * wp);
        b.carry_p = take(wp);
        b.rwords = take(4 * world);
    } else {
        b.state = take(DENSITY_B200_LION_STATE_WORDS);
    }
    if (prot) b.transfers = take(world * DECODE_PROT_TRANSFER_WORDS);
    if (map_words) b.maps = take(world * map_words + 16);
    b.bytes = (off + 64) * sizeof(uint32_t);
    return b;
}

// Sharded Cheetah or Lion decode of this rank's piece d_in[0 .. n) over the handle's communicator; x is opened with
// cl_piece_bufs(alg, world, prot, ..).bytes.
//   head    [prot: prot_transfer -> ncclAllGather(transfers) -> prot_phase1 | cand >= 0: prot_enter from that candidate (a located piece of
//           a Cheetah stream with copy-mode blocks, density_b200_decode_sharded_cheetah_stream_protected) | phase 1] -> chunk-map transfers
//           -> fold -> phase 2
//   middle  Cheetah: every round of the budget (walk -> prediction transfers + round words -> fold); the rounds after the settled one are
//           gated off on the device, their all-gathers still run. Lion: the relay of the walk's state (receive from rank - 1, walk, send
//           to rank + 1).
//   tail    phase 3 -> seam words -> verdict
// Every rank issues the same collectives in the same order whatever its piece holds: an empty piece sends identity transfers and zero
// words and forwards the walk's state unchanged, a refused one keeps exchanging until the verdict. first: the piece holds the stream
// start; last: no stream byte follows it. d_out_offset (may be NULL): where the piece's output starts, from the verdict's prefix offsets.
static int decode_sharded_cl_piece(const Exchange& x, int alg, const uint8_t* d_in, size_t n, bool first, bool last, uint8_t* d_out, size_t cap,
                                   uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, uint64_t* d_out_offset, bool prot,
                                   int64_t cand = -1) {
    density_b200_sharded* h = x.h;
    cudaStream_t st = x.st;
    const bool lion = alg == ALG_LION;
    density_b200_lion_decode_shard* ls = prot ? h->lpdec : h->ldec;
    ClDecodePiece* s = lion ? static_cast<ClDecodePiece*>(ls) : h->cdec;
    const size_t W = (size_t)h->world, R = (size_t)h->rank;
    const size_t wc = density_b200_cheetah_cmap_words(), wp = 2 * 65536;
    const ClPieceBufs b = cl_piece_bufs(alg, W, prot, 0, x.extra);
    // the last piece's transfers are never read: it sends what its slot holds
    uint32_t* cmap_out = last ? nullptr : b.tab_c + R * wc;
    int rc;
    if (prot) {
        rc = cl_piece_prot_transfer(s, lion, d_in, n, d_out, cap, first, last, b.transfers + R * DECODE_PROT_TRANSFER_WORDS, st);
        if (rc != DENSITY_B200_OK) return rc;
        if (!x.gather(b.transfers, DECODE_PROT_TRANSFER_WORDS, "ncclAllGather(transfers)")) return DENSITY_B200_ECUDA;
        rc = cl_piece_prot_phase1(s, b.transfers, (int)W, (int)R, cmap_out, st);
    } else if (cand >= 0) {
        rc = density_b200_cheetah_decode_shard_prot_enter(h->cdec, d_in, n, d_out, cap, first, last, (uint32_t)cand, cmap_out, st);
    } else {
        rc = cl_piece_phase1(s, lion, d_in, n, d_out, cap, first, last, cmap_out, st);
    }
    if (rc != DENSITY_B200_OK) return rc;
    if (!x.gather(b.tab_c, wc, "ncclAllGather(chunk-map transfers)")) return DENSITY_B200_ECUDA;
    // the first piece has nothing to fold; Lion's relay starts from the stream-start state there
    uint64_t launches = 0;
    cudaError_t e = !first ? chee_cmap_rank_fold(b.tab_c, (uint32_t)R, b.carry_c, st, &launches) : lion ? lion_state_init(b.state, st) : cudaSuccess;
    if ((rc = step_result(e, launches, "sharded cl decode: chunk-map fold")) != DENSITY_B200_OK) return rc;
    if ((rc = cl_piece_phase2(s, first ? nullptr : b.carry_c, st)) != DENSITY_B200_OK) return rc;
    if (!lion) {
        for (int k = 0; k < g_chee_dec_rounds; ++k) {
            rc = density_b200_cheetah_decode_shard_round_walk(h->cdec, last ? nullptr : b.tab_p + R * wp, b.rwords + 4 * R, st);
            if (rc != DENSITY_B200_OK) return rc;
            if (!x.gather(b.tab_p, wp, "ncclAllGather(prediction transfers)") || !x.gather(b.rwords, 4, "ncclAllGather(round words)"))
                return DENSITY_B200_ECUDA;
            launches = 0;
            e = first ? cudaSuccess : cl_rank_fold(ALG_CHEETAH, DENSITY_B200_CL_TABLE_P, b.tab_p, (uint32_t)R, b.carry_p, st, &launches);
            if ((rc = step_result(e, launches, "sharded cheetah decode: prediction fold")) != DENSITY_B200_OK) return rc;
            rc = density_b200_cheetah_decode_shard_round_fold(h->cdec, first ? nullptr : b.carry_p, b.rwords, (int)W, (int)R, st);
            if (rc != DENSITY_B200_OK) return rc;
        }
    } else {
        // the receive and the send are separate groups, since one group would send the state from before the walk
        if (!first) {
            if (!nccl_check(x.a->GroupStart(), "ncclGroupStart")) return DENSITY_B200_ECUDA;
            const bool ok = nccl_check(x.a->Recv(b.state, DENSITY_B200_LION_STATE_WORDS, NCCL_UINT32, (int)R - 1, h->comm, st), "ncclRecv(walk state)");
            if (!nccl_check(x.a->GroupEnd(), "ncclGroupEnd") || !ok) return DENSITY_B200_ECUDA;
        }
        if ((rc = density_b200_lion_decode_shard_walk(ls, b.state, st)) != DENSITY_B200_OK) return rc;
        if (!last) {
            if (!nccl_check(x.a->GroupStart(), "ncclGroupStart")) return DENSITY_B200_ECUDA;
            const bool ok = nccl_check(x.a->Send(b.state, DENSITY_B200_LION_STATE_WORDS, NCCL_UINT32, (int)R + 1, h->comm, st), "ncclSend(walk state)");
            if (!nccl_check(x.a->GroupEnd(), "ncclGroupEnd") || !ok) return DENSITY_B200_ECUDA;
        }
    }
    rc = lion ? density_b200_lion_decode_shard_phase3(ls, d_out_size, x.my_words(), st)
              : density_b200_cheetah_decode_shard_phase3(h->cdec, d_out_size, x.my_words(), st);
    if (rc != DENSITY_B200_OK) return rc;
    return x.verdict(d_flags, d_total_size, d_out_offset);
}

// The pieces of a sharded Cheetah or Lion encode, rank 0 holding the stream start and the last rank its end. prot: the inverse of
// density_b200_encode_sharded_cl_protected for any stream, whose pieces exchange their protection transfers first.
static int decode_sharded_cl(density_b200_sharded* h, int alg, bool prot, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                             uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, void* stream_v) {
    g_last_error.clear();
    int rc = decode_sharded_args(h, d_in, n, d_out, cap, d_out_size, d_flags);
    Exchange x;
    if (rc != DENSITY_B200_OK || (rc = x.open(h, stream_v, cl_piece_bufs(alg, (size_t)h->world, prot, 0).bytes)) != DENSITY_B200_OK) return rc;
    return decode_sharded_cl_piece(x, alg, d_in, n, h->rank == 0, h->rank == h->world - 1, d_out, cap, d_out_size, d_flags, d_total_size, nullptr,
                                   prot);
}
int density_b200_decode_sharded_cheetah(density_b200_sharded* h, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                        uint32_t* d_flags, uint64_t* d_total_size, void* stream_v) {
    return decode_sharded_cl(h, ALG_CHEETAH, false, d_in, n, d_out, cap, d_out_size, d_flags, d_total_size, stream_v);
}
int density_b200_decode_sharded_cheetah_protected(density_b200_sharded* h, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                                  uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, void* stream_v) {
    return decode_sharded_cl(h, ALG_CHEETAH, true, d_in, n, d_out, cap, d_out_size, d_flags, d_total_size, stream_v);
}
int density_b200_decode_sharded_lion(density_b200_sharded* h, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                     uint32_t* d_flags, uint64_t* d_total_size, void* stream_v) {
    return decode_sharded_cl(h, ALG_LION, false, d_in, n, d_out, cap, d_out_size, d_flags, d_total_size, stream_v);
}
int density_b200_decode_sharded_lion_protected(density_b200_sharded* h, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                               uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, void* stream_v) {
    return decode_sharded_cl(h, ALG_LION, true, d_in, n, d_out, cap, d_out_size, d_flags, d_total_size, stream_v);
}

// The body of the four locate entries: the argument checks (d_map: the u64 range maps 8-byte, the u32 protected range maps 4-byte
// aligned), then every step of the piece s held void (the locate scratch is phase 1's), ws_bytes of workspace ensured, and
// launch(workspace, stream, &launches) enqueued.
extern "C++" {
template <class S, class M, class F>
static int locate_entry(S* s, const uint8_t* d_in, size_t n, const M* d_map, size_t ws_bytes, void* stream, const char* what, F launch) {
    g_last_error.clear();
    if (!s || !d_map) { set_error("null pointer"); return DENSITY_B200_EARG; }
    int rc = in_args(false, d_in, n, nullptr, 0);
    if (rc != DENSITY_B200_OK) return rc;
    if (sizeof(M) == 8 && !al8(d_map)) { set_error("d_map must be 8-byte aligned"); return DENSITY_B200_EARG; }
    if ((rc = table_args({d_map})) != DENSITY_B200_OK) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    s->reset();
    cudaError_t e = s->ws.ensure(ws_bytes, st);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    uint64_t launches = 0;
    e = launch(s->ws.p, st, &launches);
    return step_result(e, launches, what);
}
}

int density_b200_decode_locate(density_b200_decode_shard* s, const uint8_t* d_in, size_t n_range, size_t n_halo, uint64_t* d_map, void* stream) {
    return locate_entry(s, d_in, n_range + n_halo, d_map, cham_locate_workspace_bytes(n_range + n_halo), stream, "decode locate",
                        [&](uint8_t* ws, cudaStream_t st, uint64_t* l) { return cham_decode_locate(d_in, n_range, n_halo, ws, d_map, st, l); });
}

// The layout checks and the walk from the stream start shared by density_b200_locate_piece (Chameleon) and
// density_b200_cheetah_locate_piece. A map is {n_range, n_halo}, NCAND candidate rows {exit index or ~0, blocks}, and with START the
// four words {range_offset, has_start_row, start exit, start blocks}: the first non-empty range then takes its exit from its start row
// rather than from candidate 0. out5 = {start, end, blocks_before, is_final, is_first}.
extern "C++" { namespace {
template <uint64_t W, uint64_t NCAND, bool START>
int locate_piece_walk(const uint64_t* h_maps, int world, int rank, uint64_t out5[5]) {
    constexpr uint64_t TERM = ~0ull, CH = 16384, HALO = 264;
    if (!h_maps || world < 1 || rank < 0 || rank >= world) { set_error("locate_piece: null pointer / bad rank or world"); return DENSITY_B200_EARG; }
    uint64_t later = 0;                 // stream bytes behind range r
    for (int r = world - 1; r >= 0; --r) {
        const uint64_t* m = h_maps + (size_t)r * W;
        if (r < world - 1 && m[0] % CH) { set_error("locate_piece: a non-last range is not a multiple of 16384 bytes"); return DENSITY_B200_EARG; }
        if (m[1] != (later < HALO ? later : HALO)) { set_error("locate_piece: a halo is not min(264, the bytes of the later ranges)"); return DENSITY_B200_EARG; }
        for (uint64_t c = 0; c < NCAND + (START ? 1 : 0); ++c) {    // + the start row's exit
            const uint64_t x = c < NCAND ? m[2 + 2 * c] : m[4 + 2 * NCAND];
            if (x != TERM && x >= NCAND) { set_error("locate_piece: bad exit index in a range map"); return DENSITY_B200_EARG; }
        }
        if (m[0] > ~later) { set_error("locate_piece: ranges overflow"); return DENSITY_B200_EARG; }
        later += m[0];
    }
    if (START) {
        uint64_t off = 0;
        bool seen = false;              // a non-empty range before r
        for (int r = 0; r < world; ++r) {
            const uint64_t* m = h_maps + (size_t)r * W;
            const uint64_t* s = m + 2 + 2 * NCAND;
            if (s[0] != off) { set_error("locate_piece: a range offset is not the sum of the earlier ranges"); return DENSITY_B200_EARG; }
            const bool holds_start = !seen && m[0] > 0;
            if (s[1] != (holds_start ? 1u : 0u)) { set_error("locate_piece: the start row is not on exactly the first non-empty range"); return DENSITY_B200_EARG; }
            seen |= m[0] > 0;
            off += m[0];
        }
    }
    // walk from the stream start; an empty range passes the entry on unchanged
    uint64_t idx = 0, blocks = 0;
    bool started = !START;              // START: the first non-empty range has not been passed yet
    for (int r = 0; r < rank; ++r) {
        const uint64_t* m = h_maps + (size_t)r * W;
        if (m[0] == 0) continue;
        const uint64_t* row = started ? m + 2 + 2 * idx : m + 4 + 2 * NCAND;
        started = true;
        blocks += row[1];
        idx = row[0];
        if (idx == TERM) { out5[0] = 0; out5[1] = 0; out5[2] = blocks; out5[3] = 1; out5[4] = 0; return DENSITY_B200_OK; }   // behind the stream end
    }
    const uint64_t* m = h_maps + (size_t)rank * W;
    const uint64_t n_range = m[0], n_halo = m[1];
    if (n_range == 0) { out5[0] = 0; out5[1] = 0; out5[2] = blocks; out5[3] = n_halo == 0; out5[4] = 0; return DENSITY_B200_OK; }
    const uint64_t ex = started ? m[2 + 2 * idx] : m[4 + 2 * NCAND];
    const uint64_t start = 2 * idx, end = ex == TERM ? n_range + n_halo : n_range + 2 * ex;
    if (start > end || end > n_range + n_halo) { set_error("locate_piece: inconsistent range maps"); return DENSITY_B200_EARG; }
    out5[0] = start; out5[1] = end; out5[2] = blocks; out5[3] = end == n_range + n_halo; out5[4] = started ? 0 : 1;
    return DENSITY_B200_OK;
}
} }  // namespace, extern "C++"

int density_b200_locate_piece(const uint64_t* h_maps, int world, int rank, uint64_t out4[4]) {
    g_last_error.clear();
    if (!out4) { set_error("locate_piece: null pointer"); return DENSITY_B200_EARG; }
    uint64_t out5[5];
    const int rc = locate_piece_walk<DENSITY_B200_LOCATE_MAP_WORDS, 132, false>(h_maps, world, rank, out5);
    if (rc == DENSITY_B200_OK) memcpy(out4, out5, 4 * sizeof(uint64_t));
    return rc;
}

int density_b200_cheetah_locate_piece(const uint64_t* h_maps, int world, int rank, uint64_t out5[5]) {
    g_last_error.clear();
    if (!out5) { set_error("locate_piece: null pointer"); return DENSITY_B200_EARG; }
    return locate_piece_walk<DENSITY_B200_CHEETAH_LOCATE_MAP_WORDS, 68, true>(h_maps, world, rank, out5);
}

int density_b200_cheetah_decode_locate(density_b200_cheetah_decode_shard* s, const uint8_t* d_in, size_t n_range, size_t n_halo, uint64_t range_offset,
                                       uint64_t* d_map, void* stream) {
    return locate_entry(s, d_in, n_range + n_halo, d_map, chee_locate_workspace_bytes(n_range, n_halo, range_offset), stream, "cheetah decode locate",
                        [&](uint8_t* ws, cudaStream_t st, uint64_t* l) { return chee_decode_locate(d_in, n_range, n_halo, range_offset, ws, d_map, st, l); });
}

// Sharded decode of a stream without known cuts: this rank holds its range + halo (include/density_b200.h). Locates the piece (one
// host synchronisation), then decodes it as density_b200_decode_sharded does.
int density_b200_decode_sharded_stream(density_b200_sharded* h, const uint8_t* d_in, size_t n_range, size_t n_halo, uint8_t* d_out, size_t cap,
                                       uint64_t* d_out_size, uint64_t* d_out_offset, uint32_t* d_flags, uint64_t* d_total_size, void* stream_v) {
    g_last_error.clear();
    int rc = decode_sharded_args(h, d_in, n_range + n_halo, d_out, cap, d_out_size, d_flags);
    Exchange x;
    if (rc != DENSITY_B200_OK || (rc = x.open(h, stream_v)) != DENSITY_B200_OK) return rc;
    // sized for the whole range + halo: covers the locate scratch and the phases on any piece of it, so that phase 1 does not reallocate
    const cudaError_t e = h->dec->ws.ensure(cham_decode_workspace_bytes(n_range + n_halo, cap, h->num_sms), x.st);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    constexpr size_t MW = DENSITY_B200_LOCATE_MAP_WORDS;
    if ((rc = density_b200_decode_locate(h->dec, d_in, n_range, n_halo, x.maps + (size_t)h->rank * MW, x.st)) != DENSITY_B200_OK ||
        (rc = x.maps_to_host(MW)) != DENSITY_B200_OK)
        return rc;
    uint64_t piece[4];
    rc = density_b200_locate_piece(h->h_maps, h->world, h->rank, piece);
    if (rc != DENSITY_B200_OK) return rc;    // the same verdict on every rank: none enters the collectives below
    return decode_sharded_piece(x, d_in + piece[0], (size_t)(piece[1] - piece[0]), (int)piece[3], d_out, cap, d_out_size, d_flags,
                                d_total_size, d_out_offset, false);
}

// Sharded decode of a Cheetah stream without known cuts: this rank holds its range + halo at range_offset (include/density_b200.h).
// Locates the piece (one host synchronisation), then decodes it as density_b200_decode_sharded_cheetah does, with the piece's own
// "holds the stream start" and "ends the stream" rather than the rank's.
int density_b200_decode_sharded_cheetah_stream(density_b200_sharded* h, const uint8_t* d_in, size_t n_range, size_t n_halo, uint64_t range_offset,
                                               uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint64_t* d_out_offset, uint32_t* d_flags,
                                               uint64_t* d_total_size, void* stream_v) {
    g_last_error.clear();
    int rc = decode_sharded_args(h, d_in, n_range + n_halo, d_out, cap, d_out_size, d_flags);
    Exchange x;
    if (rc != DENSITY_B200_OK || (rc = x.open(h, stream_v, cl_piece_bufs(ALG_CHEETAH, (size_t)h->world, false, 0).bytes)) != DENSITY_B200_OK) return rc;
    // sized for the locate scratch and for the phases on any piece of range + halo, so that phase 1 does not reallocate
    const size_t locate_bytes = chee_locate_workspace_bytes(n_range, n_halo, range_offset);
    const size_t piece_bytes = chee_shard_workspace_bytes(n_range + n_halo, cap, h->num_sms, false);
    const cudaError_t e = h->cdec->ws.ensure(locate_bytes > piece_bytes ? locate_bytes : piece_bytes, x.st);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    constexpr size_t MW = DENSITY_B200_CHEETAH_LOCATE_MAP_WORDS;    // the map slots hold DENSITY_B200_LOCATE_MAP_WORDS >= MW words per rank
    if ((rc = density_b200_cheetah_decode_locate(h->cdec, d_in, n_range, n_halo, range_offset, x.maps + (size_t)h->rank * MW, x.st)) != DENSITY_B200_OK ||
        (rc = x.maps_to_host(MW)) != DENSITY_B200_OK)
        return rc;
    uint64_t piece[5];
    rc = density_b200_cheetah_locate_piece(h->h_maps, h->world, h->rank, piece);
    if (rc != DENSITY_B200_OK) return rc;    // the same verdict on every rank: none enters the collectives below
    return decode_sharded_cl_piece(x, ALG_CHEETAH, d_in + piece[0], (size_t)(piece[1] - piece[0]), piece[4] != 0, piece[3] != 0, d_out, cap,
                                   d_out_size, d_flags, d_total_size, d_out_offset, false);
}

// ---- sharded decode of a stream without known cuts, copy-mode blocks included (DESIGN.md section 5) ----------------------------------
int density_b200_decode_prot_locate(density_b200_decode_shard* s, const uint8_t* d_in, size_t n_range, size_t n_halo, uint32_t* d_map, void* stream) {
    return locate_entry(s, d_in, n_range + n_halo, d_map, cham_locate_workspace_bytes(n_range + n_halo), stream, "decode prot locate",
                        [&](uint8_t* ws, cudaStream_t st, uint64_t* l) { return cham_decode_prot_locate(d_in, n_range, n_halo, ws, d_map, st, l); });
}
int density_b200_cheetah_decode_prot_locate(density_b200_cheetah_decode_shard* s, const uint8_t* d_in, size_t n_range, size_t n_halo, uint32_t* d_map,
                                            void* stream) {
    return locate_entry(s, d_in, n_range + n_halo, d_map, chee_prot_locate_workspace_bytes(n_range + n_halo), stream, "cheetah decode prot locate",
                        [&](uint8_t* ws, cudaStream_t st, uint64_t* l) { return chee_decode_prot_locate(d_in, n_range, n_halo, ws, d_map, st, l); });
}

// the message of a prot_locate_walk error code
static const char* prot_locate_error(int rc) {
    switch (rc) {
        case bounds::PL_ERR_MULTIPLE: return "prot_locate_piece: a non-last range is not a multiple of 16384 bytes";
        case bounds::PL_ERR_HALO: return "prot_locate_piece: a halo is not min(264, the bytes of the later ranges)";
        case bounds::PL_ERR_OVERFLOW: return "prot_locate_piece: ranges overflow";
        default: return "prot_locate_piece: bad row in a range map";
    }
}

int density_b200_prot_locate_piece(int alg, const uint32_t* h_maps, int world, int rank, uint64_t out6[6]) {
    g_last_error.clear();
    if (alg != ALG_CHAMELEON && alg != ALG_CHEETAH) { set_error("prot_locate_piece: alg must be DENSITY_B200_CHAMELEON or DENSITY_B200_CHEETAH"); return DENSITY_B200_EARG; }
    if (!h_maps || !out6 || world < 1 || rank < 0 || rank >= world) { set_error("prot_locate_piece: null pointer / bad rank or world"); return DENSITY_B200_EARG; }
    const int rc = alg == ALG_CHAMELEON ? bounds::prot_locate_walk<bounds::ChamT::NCAND>(h_maps, world, rank, out6)
                                        : bounds::prot_locate_walk<bounds::CheeT::NCAND>(h_maps, world, rank, out6);
    if (rc != bounds::PL_OK) { set_error(prot_locate_error(rc)); return DENSITY_B200_EARG; }
    return DENSITY_B200_OK;
}

namespace {
// the refusal of a composition that met 0xFFFF / 0xFFFE: the outputs of a void verdict, without another collective
__global__ void prot_locate_refused_k(uint32_t* __restrict__ d_flags, uint64_t* __restrict__ d_out_size, uint64_t* __restrict__ d_out_offset,
                                      uint64_t* __restrict__ d_total_size) {
    if (threadIdx.x || blockIdx.x) return;
    *d_flags = 1; *d_out_size = 0;
    if (d_out_offset) *d_out_offset = 0;
    if (d_total_size) *d_total_size = 0;
}
}  // namespace

// The protected range maps (this rank's already in its slot of `maps`, [world][map words]) to every rank -> the compose kernel -> its 8
// words to the host: the call's one host synchronisation. piece = {start, end, is_final, is_first, entry candidate, refused}. The layout
// errors are the same on every rank (the same maps), so is the refusal: a refused rank writes its void outputs and no rank enters
// another collective.
static int prot_locate_exchange(const Exchange& x, int alg, uint32_t* maps, uint32_t* d_flags, uint64_t* d_out_size, uint64_t* d_out_offset,
                                uint64_t* d_total_size, uint64_t piece[6]) {
    density_b200_sharded* h = x.h;
    const size_t MW = alg == ALG_CHAMELEON ? DENSITY_B200_PROT_LOCATE_MAP_WORDS : DENSITY_B200_CHEETAH_PROT_LOCATE_MAP_WORDS;
    if (!x.gather(maps, MW, "ncclAllGather(maps)")) return DENSITY_B200_ECUDA;
    unsigned long long* d_out8 = reinterpret_cast<unsigned long long*>(maps + (size_t)h->world * MW);
    if (alg == ALG_CHAMELEON) bounds::dec_prot_compose_k<bounds::ChamT::NCAND><<<1, 32, 0, x.st>>>(maps, h->world, h->rank, d_out8);
    else bounds::dec_prot_compose_k<bounds::CheeT::NCAND><<<1, 32, 0, x.st>>>(maps, h->world, h->rank, d_out8);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(h->h_maps, d_out8, 8 * sizeof(uint64_t), cudaMemcpyDeviceToHost, x.st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(x.st);
    int rc = step_result(e, 1, "protected range maps: compose");
    if (rc != DENSITY_B200_OK) return rc;
    if (h->h_maps[6] != bounds::PL_OK) { set_error(prot_locate_error((int)h->h_maps[6])); return DENSITY_B200_EARG; }
    memcpy(piece, h->h_maps, 6 * sizeof(uint64_t));
    if (piece[5]) {
        prot_locate_refused_k<<<1, 32, 0, x.st>>>(d_flags, d_out_size, d_out_offset, d_total_size);
        rc = step_result(cudaGetLastError(), 1, "protected range maps: refusal");
    }
    return rc;
}

// Sharded decode of a stream without known cuts, copy-mode blocks included: protected range map -> ncclAllGather(maps) -> compose kernel ->
// one copy to the host and one host synchronisation -> prot_enter on the located piece -> the rest of density_b200_decode_sharded_protected.
int density_b200_decode_sharded_stream_protected(density_b200_sharded* h, const uint8_t* d_in, size_t n_range, size_t n_halo, uint8_t* d_out,
                                                 size_t cap, uint64_t* d_out_size, uint64_t* d_out_offset, uint32_t* d_flags,
                                                 uint64_t* d_total_size, void* stream_v) {
    g_last_error.clear();
    int rc = decode_sharded_args(h, d_in, n_range + n_halo, d_out, cap, d_out_size, d_flags);
    constexpr size_t MW = DENSITY_B200_PROT_LOCATE_MAP_WORDS;
    Exchange x;
    if (rc != DENSITY_B200_OK || (rc = x.open(h, stream_v, (size_t)h->world * MW * sizeof(uint32_t) + 64)) != DENSITY_B200_OK) return rc;
    // sized for the whole range + halo: covers the locate scratch and the phases on any piece of it, so that phase 1 does not reallocate
    const cudaError_t e = h->pdec->ws.ensure(cham_decode_workspace_bytes(n_range + n_halo, cap, h->num_sms), x.st);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    uint32_t* maps = reinterpret_cast<uint32_t*>(x.extra);           // [world][MW], then the 8 words of the composition
    uint64_t piece[6];
    if ((rc = density_b200_decode_prot_locate(h->pdec, d_in, n_range, n_halo, maps + (size_t)h->rank * MW, x.st)) != DENSITY_B200_OK ||
        (rc = prot_locate_exchange(x, ALG_CHAMELEON, maps, d_flags, d_out_size, d_out_offset, d_total_size, piece)) != DENSITY_B200_OK)
        return rc;
    if (piece[5]) return DENSITY_B200_OK;    // refused on every rank alike: none enters the collectives below
    return decode_sharded_piece(x, d_in + piece[0], (size_t)(piece[1] - piece[0]), (int)piece[2], d_out, cap, d_out_size, d_flags,
                                d_total_size, d_out_offset, false, (int64_t)piece[4]);
}

// The same for a Cheetah stream: no range offset is needed, the composition finds the range that holds the stream start.
int density_b200_decode_sharded_cheetah_stream_protected(density_b200_sharded* h, const uint8_t* d_in, size_t n_range, size_t n_halo, uint8_t* d_out,
                                                         size_t cap, uint64_t* d_out_size, uint64_t* d_out_offset, uint32_t* d_flags,
                                                         uint64_t* d_total_size, void* stream_v) {
    g_last_error.clear();
    int rc = decode_sharded_args(h, d_in, n_range + n_halo, d_out, cap, d_out_size, d_flags);
    constexpr size_t MW = DENSITY_B200_CHEETAH_PROT_LOCATE_MAP_WORDS;
    Exchange x;
    if (rc != DENSITY_B200_OK || (rc = x.open(h, stream_v, cl_piece_bufs(ALG_CHEETAH, (size_t)h->world, false, MW).bytes)) != DENSITY_B200_OK)
        return rc;
    // sized for the locate scratch and for the phases on any piece of range + halo, so that phase 1 does not reallocate
    const size_t locate_bytes = chee_prot_locate_workspace_bytes(n_range + n_halo);
    const size_t piece_bytes = chee_shard_workspace_bytes(n_range + n_halo, cap, h->num_sms, false);
    const cudaError_t e = h->cdec->ws.ensure(locate_bytes > piece_bytes ? locate_bytes : piece_bytes, x.st);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    uint32_t* maps = cl_piece_bufs(ALG_CHEETAH, (size_t)h->world, false, MW, x.extra).maps;
    uint64_t piece[6];
    if ((rc = density_b200_cheetah_decode_prot_locate(h->cdec, d_in, n_range, n_halo, maps + (size_t)h->rank * MW, x.st)) != DENSITY_B200_OK ||
        (rc = prot_locate_exchange(x, ALG_CHEETAH, maps, d_flags, d_out_size, d_out_offset, d_total_size, piece)) != DENSITY_B200_OK)
        return rc;
    if (piece[5]) return DENSITY_B200_OK;    // refused on every rank alike: none enters the collectives below
    return decode_sharded_cl_piece(x, ALG_CHEETAH, d_in + piece[0], (size_t)(piece[1] - piece[0]), piece[3] != 0, piece[2] != 0, d_out, cap,
                                   d_out_size, d_flags, d_total_size, d_out_offset, false, (int64_t)piece[4]);
}

/* stage times of the last density_b200_encode_sharded or density_b200_encode_sharded_cl call (waits for it). Chameleon: out_ms[0] flag
   pass, [1] table exchange + fold, [2] carry / resolve / sizes / scan, [3] emit, [4] seam exchange + gather. Cheetah / Lion: [0] phase 1
   (after the last-quad exchange), [1] P exchange + fold, [2] phase 2 + C exchange + fold, [3] phase 3, [4] seam exchange + gather. */
int density_b200_sharded_profile(density_b200_sharded* h, float* out_ms) {
    if (!h || !out_ms || !h->timed) return DENSITY_B200_EARG;
    cudaError_t e = cudaEventSynchronize(h->ev[5]);
    for (int k = 0; k < 5 && e == cudaSuccess; ++k) e = cudaEventElapsedTime(&out_ms[k], h->ev[k], h->ev[k + 1]);
    if (e != cudaSuccess) { set_error("sharded_profile", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}


// ---- a reused Codec instance (streaming continuation, SURVEY §8f.1) ---------------------------------------------------------------
// /root/reference/src/codec/codec.rs:16,72,82: `encode` / `decode` are methods of an instance whose dictionary survives from call to
// call until clear_state() (chameleon.rs:148-150, cheetah.rs:198-202, lion.rs:327-331); ProtectionState is created inside every call
// (codec.rs:75,85). The state is kept the way the reference keeps it (65536 quads per table + last_hash) in device memory.
struct density_b200_codec {
    int alg = 0;
    DevBuf state;       // scalar_codec.cu layout: status 256 B (last_hash at byte 192) + chunk_a + chunk_b + pred
    DevBuf tables;      // Chameleon: carried-in table + this call's last-writer table (touched | fingerprint form)
};

density_b200_codec* density_b200_codec_create(int alg) {
    g_last_error.clear();
    if (alg < 0 || alg > 2) { set_error("bad algorithm id"); return nullptr; }
    DeviceCtx* c = current_ctx();
    if (!c) return nullptr;
    density_b200_codec* h = new density_b200_codec();
    h->alg = alg;
    cudaError_t e = h->state.ensure(scalar_workspace_bytes(alg) + 256, c->stream);      // zeroed: X::new()
    if (e == cudaSuccess && alg == ALG_CHAMELEON) e = h->tables.ensure(2 * 65536 * sizeof(uint32_t), c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { set_error("codec_create", e); h->state.release(); h->tables.release(); delete h; return nullptr; }
    return h;
}
void density_b200_codec_destroy(density_b200_codec* h) {
    if (!h) return;
    h->state.release(); h->tables.release();
    delete h;
}
int density_b200_codec_clear_state(density_b200_codec* h) {
    g_last_error.clear();
    DeviceCtx* c = current_ctx();
    if (!h || !c) return DENSITY_B200_EARG;
    std::lock_guard<std::mutex> lk(c->mu);
    cudaError_t e = cudaMemsetAsync(h->state.p, 0, scalar_workspace_bytes(h->alg) + 256, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { set_error("clear_state", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}

// Codec::encode / Codec::decode on the instance: synchronous, host or device pointers, returns the bytes written (0 on error).
static size_t codec_run(density_b200_codec* h, bool encode, const uint8_t* in, size_t n, uint8_t* out, size_t out_cap) {
    g_last_error.clear();
    if (!h || (!in && n) || (!out && out_cap)) { set_error("null pointer"); return 0; }
    if (n == 0) return 0;
    SyncCall f(in, out);
    if (!f.c) return 0;
    DeviceCtx* c = f.c;
    const int alg = h->alg;
    const int rc = f.run(in, n, false, out, out_cap, encode ? safe_size(alg, n) : out_cap, 1, [&](const uint8_t* d_in, uint8_t* d_out, size_t d_cap) {
        // the encoders store 2-byte words (encode_device's rule)
        if (encode && (reinterpret_cast<uintptr_t>(d_out) & 1)) { set_error("codec encode: a device output must be 2-byte aligned"); return DENSITY_B200_EARG; }
        cudaStream_t st = c->stream;
        const WsLease lease(c, st);
        if (!lease.ok) return DENSITY_B200_ECUDA;
        cudaError_t e = cudaSuccess;
        uint64_t launches = 0;
        uint32_t* quads = reinterpret_cast<uint32_t*>(h->state.p + 256);      // chunk_a = Chameleon's chunk_map
        bool done = false;
        if (encode && alg == ALG_CHAMELEON && !(reinterpret_cast<uintptr_t>(d_in) & 3) && !(reinterpret_cast<uintptr_t>(d_out) & 1)) {
            // run-parallel encoder with the instance's dictionary carried in; the state is only written back when the call succeeded
            uint32_t* d_carry = reinterpret_cast<uint32_t*>(h->tables.p);
            uint32_t* d_tab = d_carry + 65536;
            ChamLayout L;
            e = c->ws.ensure(cham_workspace_bytes(n, c->num_sms, &L), st);
            c->layout = L;
            const uint32_t nruns = cham_pick_runs(n, c->num_sms);
            bool ok = false;
            if (e == cudaSuccess) e = cham_quads_to_table(quads, d_carry, st, &launches);
            if (e == cudaSuccess) e = cham_encode_phase1(d_in, n, c->ws.p, L, nruns, nullptr, st, &launches);
            if (e == cudaSuccess) e = cham_encode_phase2_stream(d_in, n, c->ws.p, L, nruns, d_carry, d_out, d_cap, c->d_size, d_tab, 12, c->num_sms, st, &launches, &ok);
            if (e == cudaSuccess && ok) { e = cham_table_into_quads(d_tab, quads, st, &launches); done = true; }
            c->last_was_chameleon_fastpath_capable = 0;
        }
        if (e == cudaSuccess && !done) {
            // exact in-order kernel on the instance's state (Cheetah / Lion; Chameleon decode; a Chameleon encode whose copy map did not settle)
            if (!encode && alg == ALG_LION) c->lion_stats_valid = false;
            e = encode ? scalar_encode(alg, d_in, n, d_out, d_cap, h->state.p, c->d_size, st, &launches, nullptr, true)
                       : scalar_decode(alg, d_in, n, d_out, d_cap, h->state.p, c->d_size, st, &launches, nullptr, true);
        }
        return step_result(e, launches, "codec call");
    });
    return sync_bytes(rc, c, encode, out_cap);
}
size_t density_b200_codec_encode(density_b200_codec* h, const uint8_t* in, size_t n, uint8_t* out, size_t cap) { return codec_run(h, true, in, n, out, cap); }
size_t density_b200_codec_decode(density_b200_codec* h, const uint8_t* in, size_t n, uint8_t* out, size_t cap) { return codec_run(h, false, in, n, out, cap); }

int density_b200_table_init(uint32_t* d_table, void* stream) {
    g_last_error.clear();
    if (!d_table) { set_error("table_init: null pointer"); return DENSITY_B200_EARG; }
    if (table_args({d_table}) != DENSITY_B200_OK) return DENSITY_B200_EARG;
    uint64_t l = 0;
    const cudaError_t e = cham_table_init(d_table, reinterpret_cast<cudaStream_t>(stream), &l);
    return step_result(e, l, "table_init");
}
int density_b200_table_fold(uint32_t* d_acc, const uint32_t* d_next, void* stream) {
    g_last_error.clear();
    if (!d_acc || !d_next) { set_error("table_fold: null pointer"); return DENSITY_B200_EARG; }
    if (table_args({d_acc, d_next}) != DENSITY_B200_OK) return DENSITY_B200_EARG;
    uint64_t l = 0;
    const cudaError_t e = cham_table_fold(d_acc, d_next, reinterpret_cast<cudaStream_t>(stream), &l);
    return step_result(e, l, "table_fold");
}

// ---- per-stage device timing of the last Chameleon encode (bench.py's roofline) -----------------------------
void density_b200_profile_enable(int enable) {
    DeviceCtx* c = current_ctx();
    if (!c) return;
    std::lock_guard<std::mutex> lk(c->mu);
    c->profile = enable != 0;
    c->prof_count = 0;
}
// out[0] = flag pass ms, out[1] = between (carry/resolve/sizes/scan) ms, out[2] = emit ms. Returns 0 on success.
int density_b200_profile_get(float* out_ms) {
    DeviceCtx* c = current_ctx();
    if (!c || !out_ms) return DENSITY_B200_EARG;
    std::lock_guard<std::mutex> lk(c->mu);
    if (c->prof_count == 0) return DENSITY_B200_EARG;
    const int nset = (int)(c->prof_count < (uint64_t)DeviceCtx::PROF_RING ? c->prof_count : DeviceCtx::PROF_RING);
    double acc[3] = {0, 0, 0};
    cudaError_t e = cudaSuccess;
    for (int s = 0; s < nset && e == cudaSuccess; ++s) {
        cudaEvent_t* ev = c->ev[s];
        float ms[3];
        e = cudaEventSynchronize(ev[3]);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&ms[0], ev[0], ev[1]);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&ms[1], ev[1], ev[2]);
        if (e == cudaSuccess) e = cudaEventElapsedTime(&ms[2], ev[2], ev[3]);
        for (int k = 0; k < 3; ++k) acc[k] += ms[k];
    }
    if (e != cudaSuccess) { set_error("profile_get", e); return DENSITY_B200_ECUDA; }
    for (int k = 0; k < 3; ++k) out_ms[k] = (float)(acc[k] / nset);
    return DENSITY_B200_OK;
}

// ---- housekeeping ----------------------------------------------------------------------------------------
const char* density_b200_last_error(void) { return g_last_error.c_str(); }
uint64_t density_b200_kernel_launches(void) { return g_launches.load(); }

int density_b200_last_encode_was_fast(void) {
    DeviceCtx* c = current_ctx();
    if (!c) return 0;
    std::lock_guard<std::mutex> lk(c->mu);
    if (c->last_was_chameleon_fastpath_capable == 2) return 1;
    if (!c->last_was_chameleon_fastpath_capable || !c->ws.p) return 0;
    Status st;
    if (cudaDeviceSynchronize() != cudaSuccess) return 0;
    if (cudaMemcpy(&st, c->ws.p + c->layout.status, sizeof st, cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
    return st.nonquiet ? 0 : 1;
}

/* diagnostic: status block of the last Chameleon encode on the current device (synchronises) */
int density_b200_encode_status(uint64_t* out6) {
    DeviceCtx* c = current_ctx();
    if (!c || !c->ws.p) return DENSITY_B200_EARG;
    std::lock_guard<std::mutex> lk(c->mu);
    Status st;
    if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpy(&st, c->ws.p + c->layout.status, sizeof st, cudaMemcpyDeviceToHost) != cudaSuccess) return DENSITY_B200_ECUDA;
    out6[0] = st.out_bytes; out6[1] = st.nonquiet; out6[2] = st.error; out6[3] = st.first_nonquiet_block; out6[4] = st.converged; out6[5] = st.iter_changed;
    return DENSITY_B200_OK;
}

void density_b200_shutdown(void) {
    std::lock_guard<std::mutex> lk(g_ctx_mu);
    int cur = -1;
    cudaGetDevice(&cur);
    for (int d = 0; d < MAX_DEVICES; ++d) {
        DeviceCtx& c = g_ctx[d];
        if (!c.ready) continue;
        cudaSetDevice(d);
        c.release();
    }
    if (cur >= 0) cudaSetDevice(cur);
}

/* diagnostic: the context iteration of the last parallel Cheetah decode on the current device (synchronises):
   out4 = {rounds used, settled (0 = the in-order kernel had to take over), run walks after round 0 (of rounds x runs), round budget} */
int density_b200_cheetah_decode_rounds(uint32_t* out4) {
    DeviceCtx* c = current_ctx();
    if (!c || !out4) return DENSITY_B200_EARG;
    std::lock_guard<std::mutex> lk(c->mu);
    if (!c->chee_rounds_valid) return DENSITY_B200_EARG;
    unsigned int raw[8] = {0};
    if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpy(raw, c->diag.p, sizeof raw, cudaMemcpyDeviceToHost) != cudaSuccess) return DENSITY_B200_ECUDA;
    out4[0] = raw[3]; out4[1] = raw[2] && !raw[5]; out4[2] = raw[6]; out4[3] = chee_shard_max_rounds();   // cl_decode.cu MAX_ROUNDS
    return DENSITY_B200_OK;
}

/* diagnostic: the prediction walk of the last Lion decode on the current device (synchronises; DENSITY_B200_EARG when that decode ran
   on the in-order kernel or there was none): out4 = {encoded quads walked, predicted quads, table reads that waited on a predicted quad,
   rows walked} */
int density_b200_lion_decode_stats(uint64_t* out4) {
    DeviceCtx* c = current_ctx();
    if (!c || !out4) return DENSITY_B200_EARG;
    std::lock_guard<std::mutex> lk(c->mu);
    if (cudaDeviceSynchronize() != cudaSuccess) return DENSITY_B200_ECUDA;
    if (!c->lion_stats_valid) return DENSITY_B200_EARG;
    return cudaMemcpy(out4, c->diag.p + 32, 4 * sizeof(uint64_t), cudaMemcpyDeviceToHost) == cudaSuccess ? DENSITY_B200_OK : DENSITY_B200_ECUDA;
}

/* test hook: rounds per stage of the Cheetah / Lion copy-map iteration (1..7; 7 = default) */
void density_b200_test_set_stage_rounds(int k) { g_chee_stage_rounds = (k >= 1 && k <= 7) ? k : 7; }
void density_b200_test_set_decode_rounds(int k) { g_chee_dec_rounds = (k >= 1 && k <= 40) ? k : 40; }

/* diagnostic: the last copy-map iteration on the current device, per fixed-point round {first block whose copy status changed (~0: none),
   number of such blocks}; 16 rounds x 2 values (synchronises) */
int density_b200_prot_debug(uint64_t* out32) {
    if (!out32) return DENSITY_B200_EARG;
    if (cudaDeviceSynchronize() != cudaSuccess) return DENSITY_B200_ECUDA;
    return prot_debug_read(reinterpret_cast<unsigned long long*>(out32)) == cudaSuccess ? DENSITY_B200_OK : DENSITY_B200_ECUDA;
}

const char* density_b200_version(void) { return "density_b200 0.1.0 (sm_90a)"; }

}  // extern "C"
