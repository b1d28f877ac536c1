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

// grow-only device buffer
struct DevBuf {
    uint8_t* p = nullptr; size_t bytes = 0;
    // `stream`: the stream the buffer is about to be used on. The zero fill (the Cheetah / Lion encoder tables rely on starting out
    // zeroed) is ordered on it; cudaFree of the old buffer synchronises the device, so nothing can still be using it.
    cudaError_t ensure(size_t need, cudaStream_t stream = nullptr) {
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
    // One workspace per device: a call may only start using it when the previous call (on whatever stream) has finished with it.
    // Every enqueue ends with cudaEventRecord(ws_free, its stream) and starts with cudaStreamWaitEvent(its stream, ws_free).
    const void* last_cl_status = nullptr;   // iteration status block of the last parallel Cheetah decode (diagnostics)
    cudaEvent_t ws_free = nullptr;
    bool ws_free_recorded = false;
    std::mutex mu;
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

// path: 0 auto (fast path with exact fallback), 1 fast only (no fallback), 2 protected walk only, 3 scalar kernel
// path 4 (internal): Chameleon auto path for callers that may block on the stream (the synchronous reference-facing entry points): the
// copy-map iteration gets up to 12 more batches of 8 rounds before the in-order walk may take over
static bool ws_acquire(DeviceCtx* c, cudaStream_t stream) {
    if (!c->ws_free_recorded) return true;
    cudaError_t e = cudaStreamWaitEvent(stream, c->ws_free, 0);
    if (e != cudaSuccess) { set_error("cudaStreamWaitEvent", e); return false; }
    return true;
}
static void ws_release(DeviceCtx* c, cudaStream_t stream) {
    if (cudaEventRecord(c->ws_free, stream) == cudaSuccess) c->ws_free_recorded = true;
}

static int encode_device_locked_impl(DeviceCtx* c, int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                     uint64_t* d_out_size, cudaStream_t stream, int path);
static int encode_device_locked(DeviceCtx* c, int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                uint64_t* d_out_size, cudaStream_t stream, int path) {
    if (!ws_acquire(c, stream)) return DENSITY_B200_ECUDA;
    const int rc = encode_device_locked_impl(c, alg, d_in, n, d_out, cap, d_out_size, stream, path);
    ws_release(c, stream);
    return rc;
}
static int encode_device_locked_impl(DeviceCtx* c, int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                     uint64_t* d_out_size, cudaStream_t stream, int path) {
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
                e = cham_encode_phase2_blocking(d_in, n, c->ws.p, L, nruns, d_out, cap, d_out_size, 12, stream, &launches);
            else if (e == cudaSuccess)
                e = cham_encode_phase2(d_in, n, c->ws.p, L, nruns, nullptr, d_out, cap, d_out_size, path == 0, false, stream, &launches, ev);
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
    g_launches += launches;
    if (e != cudaSuccess) { set_error("encode launch", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}

// path: 0 auto (parallel decoder with exact in-order fallback), 1 parallel only, 3 in-order kernel only
static int decode_device_locked_impl(DeviceCtx* c, int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                     uint64_t* d_out_size, cudaStream_t stream, int path);
static int decode_device_locked(DeviceCtx* c, int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                uint64_t* d_out_size, cudaStream_t stream, int path = 0) {
    if (!ws_acquire(c, stream)) return DENSITY_B200_ECUDA;
    const int rc = decode_device_locked_impl(c, alg, d_in, n, d_out, cap, d_out_size, stream, path);
    ws_release(c, stream);
    return rc;
}
static int decode_device_locked_impl(DeviceCtx* c, int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                     uint64_t* d_out_size, cudaStream_t stream, int path) {
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
        g_launches += launches;
        if (e != cudaSuccess) { set_error("decode launch", e); return DENSITY_B200_ECUDA; }
        return DENSITY_B200_OK;
    }
    if (alg == ALG_CHEETAH && path != 3 && !(reinterpret_cast<uintptr_t>(d_in) & 1) && !(reinterpret_cast<uintptr_t>(d_out) & 3)) {
        // run-parallel Cheetah decoder (cl_decode.cu) + in-order tail; the exact in-order kernel is queued behind it and only runs if
        // the context iteration did not settle within its round budget
        const size_t pw = (chee_decode_workspace_bytes(n, cap, c->num_sms) + 255) & ~(size_t)255;
        e = c->ws.ensure(pw + 256 + 2 * ((scalar_workspace_bytes(alg) + 255) & ~(size_t)255), stream);
        if (e == cudaSuccess) e = c->dec_tables.ensure(chee_decode_tables_bytes(n, c->num_sms) + 256, stream);
        if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
        uint32_t* d_fallback = reinterpret_cast<uint32_t*>(c->ws.p + pw);
        uint8_t* tail_ws = c->ws.p + pw + 256;
        uint8_t* scalar_ws = tail_ws + ((scalar_workspace_bytes(alg) + 255) & ~(size_t)255);
        e = cudaMemsetAsync(tail_ws, 0, 256, stream);
        if (e == cudaSuccess) e = chee_decode_parallel(d_in, n, d_out, cap, c->ws.p, c->dec_tables.p, tail_ws, c->num_sms, d_out_size, d_fallback, stream, &launches);
        if (e == cudaSuccess) {
            const void* cl_st = nullptr;
            const void* b_st = chee_decode_status_ptr(c->ws.p, n, cap, c->num_sms, &cl_st);
            c->last_cl_status = cl_st;
            e = scalar_decode_tail(alg, d_in, n, d_out, cap, tail_ws, b_st, cl_st, d_out_size, stream, &launches, d_fallback);
        }
        if (e == cudaSuccess && path != 1)
            e = scalar_decode(alg, d_in, n, d_out, cap, scalar_ws, d_out_size, stream, &launches, d_fallback);
        g_launches += launches;
        if (e != cudaSuccess) { set_error("decode launch", e); return DENSITY_B200_ECUDA; }
        return DENSITY_B200_OK;
    }
    e = c->ws.ensure(scalar_workspace_bytes(alg), stream);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    e = scalar_decode(alg, d_in, n, d_out, cap, c->ws.p, d_out_size, stream, &launches);
    g_launches += launches;
    if (e != cudaSuccess) { set_error("decode launch", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}

// Host-pointer Chameleon encode, pipelined over PCIe: the input is cut into chunks that are treated as shards of one
// bit-exact stream (same mechanism as the multi-GPU path): while chunk i+1 is still crossing PCIe, chunk i runs
// phase 1 (flags) + phase 2 (carry-in from the chunks before it, scan, emit) and chunk i-1's output travels back.
// Returns bytes written, 0 on error, or (size_t)-1 when the stream turned out not to be "quiet" (caller falls back
// to the whole-buffer path with the protection-aware walk; the input is already resident in stage_in).
constexpr size_t PIPE_CHUNK = 64u << 20;
constexpr size_t PIPE_MIN_BYTES = 96u << 20;

static size_t chameleon_encode_host_pipelined(DeviceCtx* c, const uint8_t* in, size_t n, uint8_t* out, size_t out_cap) {
    const size_t nchunks = (n + PIPE_CHUNK - 1) / PIPE_CHUNK;
    if (nchunks > 4096) return (size_t)-1;
    cudaError_t e = c->stage_in.ensure(n + 16);
    if (e == cudaSuccess) e = c->stage_out.ensure(safe_size(ALG_CHAMELEON, n) + 16);
    if (e == cudaSuccess) e = c->pipe_tables.ensure(2 * 65536 * sizeof(uint32_t) + (nchunks + 1) * sizeof(uint64_t) + 256);
    ChamLayout L;
    if (e == cudaSuccess) e = c->ws.ensure(cham_workspace_bytes(PIPE_CHUNK, c->num_sms, &L));
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
                                                     c->stage_out.bytes - out_off, d_sizes + i, false, i != 0, c->stream, &launches);
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

// Synchronous entry point shared by the nine reference-shaped symbols.
static size_t run_sync(bool encode, int alg, const uint8_t* in, size_t n, uint8_t* out, size_t out_cap) {
    g_last_error.clear();
    if ((!in && n) || (!out && out_cap)) { set_error("null pointer"); return 0; }
    if (n == 0) return 0;  // Codec::encode/decode of an empty slice writes nothing (codec.rs:76,102)
    DeviceCtx* c = current_ctx();
    if (!c) return 0;
    std::lock_guard<std::mutex> lk(c->mu);
    const bool in_dev = is_device_pointer(in), out_dev = is_device_pointer(out);
    cudaError_t e;
    if (in_dev || out_dev) {
        // the call is synchronous and cannot know which stream produced a device buffer: wait for all of them
        e = cudaDeviceSynchronize();
        if (e != cudaSuccess) { set_error("cudaDeviceSynchronize", e); return 0; }
    }
    const uint8_t* d_in = in;
    uint8_t* d_out = out;
    size_t d_cap = out_cap;
    bool input_staged = false;
    if (encode && alg == ALG_CHAMELEON && !in_dev && !out_dev && n >= PIPE_MIN_BYTES) {
        const size_t r = chameleon_encode_host_pipelined(c, in, n, out, out_cap);
        if (r != (size_t)-1) return r;
        input_staged = true;   // not quiet: the whole input is already in stage_in; redo with the protection-aware fallback
        d_in = c->stage_in.p;
    }
    if (!in_dev && !input_staged) {
        e = c->stage_in.ensure(n + 16);
        if (e != cudaSuccess) { set_error("staging cudaMalloc", e); return 0; }
        e = h2d_any(c->ring_in, c->stage_in.p, in, n, c->stream, is_pageable_host(in));
        if (e != cudaSuccess) { set_error("H2D copy", e); return 0; }
        d_in = c->stage_in.p;
    }
    if (!out_dev) {
        // encode: stage into a full safe-size buffer and check the real size against the caller's capacity afterwards
        // (the reference only fails when the bytes actually written exceed the slice, write_buffer.rs:19)
        d_cap = encode ? safe_size(alg, n) : out_cap;
        e = c->stage_out.ensure(d_cap + 16);
        if (e != cudaSuccess) { set_error("staging cudaMalloc", e); return 0; }
        d_out = c->stage_out.p;
    }
    int rc = encode ? encode_device_locked(c, alg, d_in, n, d_out, d_cap, c->d_size, c->stream, 4)
                    : decode_device_locked(c, alg, d_in, n, d_out, d_cap, c->d_size, c->stream);
    if (rc != DENSITY_B200_OK) { cudaStreamSynchronize(c->stream); return 0; }
    e = cudaMemcpyAsync(c->h_size, c->d_size, sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { set_error("stream sync", e); return 0; }
    const uint64_t produced = *c->h_size;
    if (produced == 0) { set_error(encode ? "encode failed on device (output capacity?)" : "decode failed on device (malformed stream or output capacity)"); return 0; }
    if (produced > out_cap) { set_error("output buffer too small"); return 0; }
    if (!out_dev) {
        e = d2h_any(c->ring_out, out, d_out, produced, c->stream, is_pageable_host(out));
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        if (e != cudaSuccess) { set_error("D2H copy", e); return 0; }
    }
    return (size_t)produced;
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
    g_last_error.clear();
    if (alg < 0 || alg > 2) { set_error("bad algorithm id"); return DENSITY_B200_EARG; }
    if (!d_out_size || (!d_in && n) || (!d_out && cap)) { set_error("null pointer"); return DENSITY_B200_EARG; }
    DeviceCtx* c = current_ctx();
    if (!c) return DENSITY_B200_ECUDA;
    std::lock_guard<std::mutex> lk(c->mu);
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (n == 0) {
        cudaError_t e = cudaMemsetAsync(d_out_size, 0, sizeof(uint64_t), s);
        if (e != cudaSuccess) { set_error("memset", e); return DENSITY_B200_ECUDA; }
        return DENSITY_B200_OK;
    }
    return encode ? encode_device_locked(c, alg, d_in, n, d_out, cap, d_out_size, s, path)
                  : decode_device_locked(c, alg, d_in, n, d_out, cap, d_out_size, s, path);
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

// ---- sharded Chameleon encode ------------------------------------------------------------------------
struct density_b200_shard {
    DevBuf ws;
    ChamLayout L{};
    const uint8_t* d_in = nullptr;
    size_t n = 0;
    uint32_t nruns = 0;
    int is_last = 1;
    int num_sms = 0;
    bool phase1_done = false;
};

density_b200_shard* density_b200_shard_create(void) {
    g_last_error.clear();
    DeviceCtx* c = current_ctx();
    if (!c) return nullptr;
    density_b200_shard* s = new density_b200_shard();
    s->num_sms = c->num_sms;
    return s;
}
void density_b200_shard_destroy(density_b200_shard* s) {
    if (!s) return;
    s->ws.release();
    delete s;
}
int density_b200_shard_phase1(density_b200_shard* s, const uint8_t* d_in, size_t n, int is_last_shard, uint32_t* d_table_out, void* stream) {
    g_last_error.clear();
    if (!s || (!d_in && n) || !d_table_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (!is_last_shard && (n % 256)) { set_error("non-final shards must be a multiple of 256 bytes"); return DENSITY_B200_EARG; }
    if (reinterpret_cast<uintptr_t>(d_in) & 3) { set_error("d_in must be 4-byte aligned"); return DENSITY_B200_EARG; }
    size_t need = cham_workspace_bytes(n, s->num_sms, &s->L);
    cudaError_t e = s->ws.ensure(need);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    s->d_in = d_in; s->n = n; s->is_last = is_last_shard; s->nruns = cham_pick_runs(n, s->num_sms);
    uint64_t launches = 0;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (n == 0) {
        e = cudaMemsetAsync(d_table_out, 0, 65536 * sizeof(uint32_t), st);  // nothing touched
    } else {
        e = cham_encode_phase1(d_in, n, s->ws.p, s->L, s->nruns, d_table_out, st, &launches);
    }
    g_launches += launches;
    if (e != cudaSuccess) { set_error("shard phase1", e); return DENSITY_B200_ECUDA; }
    s->phase1_done = true;
    return DENSITY_B200_OK;
}
int density_b200_shard_phase2(density_b200_shard* s, const uint32_t* d_carry_in, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                              uint32_t* d_flags, void* stream) {
    g_last_error.clear();
    if (!s || !s->phase1_done || !d_out_size) { set_error("shard_phase2: phase1 not done / null pointer"); return DENSITY_B200_EARG; }
    if (reinterpret_cast<uintptr_t>(d_out) & 1) { set_error("d_out must be 2-byte aligned"); return DENSITY_B200_EARG; }
    uint64_t launches = 0;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    cudaError_t e = cham_encode_phase2(s->d_in, s->n, s->ws.p, s->L, s->nruns, d_carry_in, d_out, cap, d_out_size, false,
                                       d_carry_in != nullptr, st, &launches, nullptr);
    if (e == cudaSuccess && d_flags) {
        if (s->n) e = cudaMemcpyAsync(d_flags, s->ws.p + s->L.status + offsetof(Status, nonquiet), sizeof(uint32_t), cudaMemcpyDeviceToDevice, st);
        else e = cudaMemsetAsync(d_flags, 0, sizeof(uint32_t), st);
    }
    g_launches += launches;
    if (e != cudaSuccess) { set_error("shard phase2", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}

// ---- sharded Cheetah / Lion encode: one shard of a longer stream in three phases around two table exchanges ---------------------------
struct density_b200_cl_shard {
    int alg = ALG_CHEETAH, num_sms = 0;
    DevBuf ws, tables[3];           // workspace; the epoch-tagged run tables (zero at allocation, one entry format each)
    uint32_t epoch = 0, epoch_base = 0;
    const uint8_t* d_in = nullptr;
    size_t n = 0;
    bool first = true, is_last = true;
    int phase = 0;                  // the last phase done on the current shard
};

static bool cl_alg_ok(int alg) { return alg == ALG_CHEETAH || alg == ALG_LION; }

density_b200_cl_shard* density_b200_cl_shard_create(int alg) {
    g_last_error.clear();
    if (!cl_alg_ok(alg)) { set_error("cl_shard_create: alg must be DENSITY_B200_CHEETAH or DENSITY_B200_LION"); return nullptr; }
    DeviceCtx* c = current_ctx();
    if (!c) return nullptr;
    density_b200_cl_shard* s = new density_b200_cl_shard();
    s->alg = alg; s->num_sms = c->num_sms;
    return s;
}
void density_b200_cl_shard_destroy(density_b200_cl_shard* s) {
    if (!s) return;
    s->ws.release(); for (auto& t : s->tables) t.release();
    delete s;
}
size_t density_b200_cl_table_words(int alg, int kind) {
    if (!cl_alg_ok(alg) || (kind != DENSITY_B200_CL_TABLE_P && kind != DENSITY_B200_CL_TABLE_C)) return 0;
    return (size_t)cl_table_planes(alg, kind) * 65536;
}

static int cl_phase1_impl(density_b200_cl_shard* s, const uint8_t* d_in, size_t n, int is_last, const uint32_t* d_prev_quad, uint32_t* d_tab_p,
                          cudaStream_t st) {
    if ((!d_in && n) || !d_tab_p) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (!is_last && (n % 256)) { set_error("non-final shards must be a multiple of 256 bytes"); return DENSITY_B200_EARG; }
    if ((reinterpret_cast<uintptr_t>(d_in) & 3) || (reinterpret_cast<uintptr_t>(d_prev_quad) & 3)) { set_error("d_in and d_prev_quad must be 4-byte aligned"); return DENSITY_B200_EARG; }
    s->phase = 0;
    cudaError_t e = s->ws.ensure(cl_shard_workspace_bytes(n, s->num_sms), st);
    for (int rg = 0; rg < 3 && e == cudaSuccess; ++rg) e = s->tables[rg].ensure(chee_tables_bytes(s->alg, rg, n, s->num_sms) + 256, st);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    if (s->epoch > 0x0FFFFF00u) {                      // epochs exhausted: start over on cleared tables
        for (int rg = 0; rg < 3 && e == cudaSuccess; ++rg) e = cudaMemsetAsync(s->tables[rg].p, 0, s->tables[rg].bytes, st);
        if (e != cudaSuccess) { set_error("cudaMemsetAsync", e); return DENSITY_B200_ECUDA; }
        s->epoch = 0;
    }
    s->epoch_base = s->epoch + 1; s->epoch += cl_shard_epochs();
    s->d_in = d_in; s->n = n; s->first = d_prev_quad == nullptr; s->is_last = is_last != 0;
    uint64_t launches = 0;
    uint8_t* const tabs[3] = {s->tables[0].p, s->tables[1].p, s->tables[2].p};
    if (n == 0) e = cudaMemsetAsync(d_tab_p, 0, density_b200_cl_table_words(s->alg, DENSITY_B200_CL_TABLE_P) * sizeof(uint32_t), st);   // identity
    else e = cl_shard_phase1(s->alg, d_in, n, d_prev_quad, s->ws.p, tabs, s->epoch_base, s->num_sms, d_tab_p, st, &launches);
    g_launches += launches;
    if (e != cudaSuccess) { set_error("cl shard phase1", e); return DENSITY_B200_ECUDA; }
    s->phase = 1;
    return DENSITY_B200_OK;
}
static int cl_phase2_impl(density_b200_cl_shard* s, const uint32_t* d_carry_p, uint32_t* d_tab_c, cudaStream_t st) {
    if (s->phase != 1) { set_error("cl_shard_phase2: phase 1 not done"); return DENSITY_B200_EARG; }
    if (!d_tab_c) { set_error("null pointer"); return DENSITY_B200_EARG; }
    uint64_t launches = 0;
    uint8_t* const tabs[3] = {s->tables[0].p, s->tables[1].p, s->tables[2].p};
    cudaError_t e;
    if (s->n == 0) e = cudaMemsetAsync(d_tab_c, 0, density_b200_cl_table_words(s->alg, DENSITY_B200_CL_TABLE_C) * sizeof(uint32_t), st);
    else e = cl_shard_phase2(s->alg, s->d_in, s->n, s->first, d_carry_p, s->ws.p, tabs, s->epoch_base, s->num_sms, d_tab_c, st, &launches);
    g_launches += launches;
    if (e != cudaSuccess) { set_error("cl shard phase2", e); return DENSITY_B200_ECUDA; }
    s->phase = 2;
    return DENSITY_B200_OK;
}
static int cl_phase3_impl(density_b200_cl_shard* s, const uint32_t* d_carry_c, uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint32_t* d_seam8,
                          cudaStream_t st) {
    if (s->phase != 2) { set_error("cl_shard_phase3: phase 2 not done"); return DENSITY_B200_EARG; }
    if ((!d_out && cap) || !d_out_size || !d_seam8) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (reinterpret_cast<uintptr_t>(d_out) & 1) { set_error("d_out must be 2-byte aligned"); return DENSITY_B200_EARG; }
    uint64_t launches = 0;
    uint8_t* const tabs[3] = {s->tables[0].p, s->tables[1].p, s->tables[2].p};
    cudaError_t e;
    if (s->n == 0) {
        e = cudaMemsetAsync(d_out_size, 0, sizeof(uint64_t), st);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_seam8, 0, 8 * sizeof(uint32_t), st);
    } else {
        e = cl_shard_phase3(s->alg, s->d_in, s->n, s->first, s->is_last, d_carry_c, s->ws.p, tabs, s->epoch_base, s->num_sms, d_out, cap, d_out_size,
                            d_seam8, st, &launches);
    }
    g_launches += launches;
    if (e != cudaSuccess) { set_error("cl shard phase3", e); return DENSITY_B200_ECUDA; }
    s->phase = 3;
    return DENSITY_B200_OK;
}
int density_b200_cl_shard_phase1(density_b200_cl_shard* s, const uint8_t* d_in, size_t n, int is_last_shard, const uint32_t* d_prev_quad,
                                 uint32_t* d_table_p_out, void* stream) {
    g_last_error.clear();
    if (!s) { set_error("null pointer"); return DENSITY_B200_EARG; }
    return cl_phase1_impl(s, d_in, n, is_last_shard, d_prev_quad, d_table_p_out, reinterpret_cast<cudaStream_t>(stream));
}
int density_b200_cl_shard_phase2(density_b200_cl_shard* s, const uint32_t* d_carry_p, uint32_t* d_table_c_out, void* stream) {
    g_last_error.clear();
    if (!s) { set_error("null pointer"); return DENSITY_B200_EARG; }
    return cl_phase2_impl(s, d_carry_p, d_table_c_out, reinterpret_cast<cudaStream_t>(stream));
}
int density_b200_cl_shard_phase3(density_b200_cl_shard* s, const uint32_t* d_carry_c, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                 uint32_t* d_seam8, void* stream) {
    g_last_error.clear();
    if (!s) { set_error("null pointer"); return DENSITY_B200_EARG; }
    return cl_phase3_impl(s, d_carry_c, d_out, cap, d_out_size, d_seam8, reinterpret_cast<cudaStream_t>(stream));
}
int density_b200_cl_table_init(int alg, int kind, uint32_t* d_table, void* stream) {
    g_last_error.clear();
    if (!density_b200_cl_table_words(alg, kind) || !d_table) { set_error("cl_table_init: bad algorithm / kind or null pointer"); return DENSITY_B200_EARG; }
    uint64_t l = 0;
    cudaError_t e = cl_table_init(alg, kind, d_table, reinterpret_cast<cudaStream_t>(stream), &l);
    g_launches += l;
    if (e != cudaSuccess) { set_error("cl_table_init", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}
int density_b200_cl_table_fold(int alg, int kind, uint32_t* d_acc, const uint32_t* d_next, void* stream) {
    g_last_error.clear();
    if (!density_b200_cl_table_words(alg, kind) || !d_acc || !d_next) { set_error("cl_table_fold: bad algorithm / kind or null pointer"); return DENSITY_B200_EARG; }
    uint64_t l = 0;
    cudaError_t e = cl_table_fold(alg, kind, d_acc, d_next, reinterpret_cast<cudaStream_t>(stream), &l);
    g_launches += l;
    if (e != cudaSuccess) { set_error("cl_table_fold", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}

// ---- sharded Chameleon decode: one piece of a sharded stream, decoded with the dictionary carried in from the pieces before it ------
struct density_b200_decode_shard {
    DevBuf ws;
    const uint8_t* d_in = nullptr;
    size_t n = 0, cap = 0;
    int is_last = 1;
    int num_sms = 0;
    bool phase1_done = false;
};

density_b200_decode_shard* density_b200_decode_shard_create(void) {
    g_last_error.clear();
    DeviceCtx* c = current_ctx();
    if (!c) return nullptr;
    density_b200_decode_shard* s = new density_b200_decode_shard();
    s->num_sms = c->num_sms;
    return s;
}
void density_b200_decode_shard_destroy(density_b200_decode_shard* s) {
    if (!s) return;
    s->ws.release();
    delete s;
}
int density_b200_decode_shard_phase1(density_b200_decode_shard* s, const uint8_t* d_in, size_t n, size_t cap, int is_last_shard,
                                     uint32_t* d_table_out, void* stream) {
    g_last_error.clear();
    if (!s || (!d_in && n) || !d_table_out) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (reinterpret_cast<uintptr_t>(d_in) & 1) { set_error("d_in must be 2-byte aligned"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    s->phase1_done = false;
    cudaError_t e = s->ws.ensure(cham_decode_workspace_bytes(n, cap, s->num_sms), st);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    s->d_in = d_in; s->n = n; s->cap = cap; s->is_last = is_last_shard;
    uint64_t launches = 0;
    if (n == 0) e = cudaMemsetAsync(d_table_out, 0, 65536 * sizeof(uint32_t), st);  // nothing touched
    else e = cham_decode_phase1(d_in, n, cap, s->ws.p, s->num_sms, d_table_out, st, &launches);
    g_launches += launches;
    if (e != cudaSuccess) { set_error("decode shard phase1", e); return DENSITY_B200_ECUDA; }
    s->phase1_done = true;
    return DENSITY_B200_OK;
}
int density_b200_decode_shard_phase2(density_b200_decode_shard* s, const uint32_t* d_carry_in, uint8_t* d_out, uint64_t* d_out_size,
                                     uint32_t* d_seam8, void* stream) {
    g_last_error.clear();
    if (!s || !s->phase1_done) { set_error("decode_shard_phase2: phase1 not done"); return DENSITY_B200_EARG; }
    if ((!d_out && s->cap) || !d_out_size || !d_seam8) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (reinterpret_cast<uintptr_t>(d_out) & 3) { set_error("d_out must be 4-byte aligned"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    uint64_t launches = 0;
    cudaError_t e;
    if (s->n == 0) {
        e = cudaMemsetAsync(d_out_size, 0, sizeof(uint64_t), st);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_seam8, 0, 8 * sizeof(uint32_t), st);
    } else {
        e = cham_decode_phase2(s->d_in, s->n, d_out, s->cap, s->ws.p, s->num_sms, d_carry_in, d_out_size, st, &launches);
        if (e == cudaSuccess) e = cham_decode_seam_words(s->d_in, s->n, s->cap, s->ws.p, s->num_sms, s->is_last, d_out_size, d_seam8, st, &launches);
    }
    g_launches += launches;
    s->phase1_done = false;     // the decode pass overwrites the run tables: one phase 2 per phase 1
    if (e != cudaSuccess) { set_error("decode shard phase2", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}

// ---- sharded Cheetah decode: one piece, its chunk map carried in and its prediction rounds run over all pieces ------------------------
static int g_chee_dec_rounds = 40;    // round budget of the sharded Cheetah decode (density_b200_test_set_decode_rounds)

struct density_b200_cheetah_decode_shard {
    DevBuf ws, tables;
    CheeShardArgs a{};
    int num_sms = 0;
    // the last step done on the current piece: 0 none, 1 phase 1, 2 phase 2 or a round's fold, 3 a round's walk, 4 phase 3
    int phase = 0;
    uint32_t round = 0;
};

density_b200_cheetah_decode_shard* density_b200_cheetah_decode_shard_create(void) {
    g_last_error.clear();
    DeviceCtx* c = current_ctx();
    if (!c) return nullptr;
    density_b200_cheetah_decode_shard* s = new density_b200_cheetah_decode_shard();
    s->num_sms = c->num_sms;
    return s;
}
void density_b200_cheetah_decode_shard_destroy(density_b200_cheetah_decode_shard* s) {
    if (!s) return;
    s->ws.release(); s->tables.release();
    delete s;
}
int density_b200_cheetah_decode_round_budget(void) { return g_chee_dec_rounds; }
size_t density_b200_cheetah_cmap_words(void) { return 3 * 65536; }

static int cd_phase1_impl(density_b200_cheetah_decode_shard* s, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, int is_first, int is_last,
                          uint32_t* d_cmap_out, cudaStream_t st) {
    if ((!d_in && n) || (!d_out && cap)) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if ((reinterpret_cast<uintptr_t>(d_in) & 1) || (reinterpret_cast<uintptr_t>(d_out) & 3)) { set_error("d_in must be 2-byte, d_out 4-byte aligned"); return DENSITY_B200_EARG; }
    s->phase = 0; s->round = 0;
    CheeShardArgs& a = s->a;
    a.d_in = d_in; a.n = n; a.d_out = d_out; a.cap = cap; a.first = is_first != 0; a.last = is_last != 0; a.num_sms = s->num_sms;
    cudaError_t e = cudaSuccess;
    if (n) {
        e = s->ws.ensure(chee_shard_workspace_bytes(n, cap, s->num_sms), st);
        if (e == cudaSuccess) e = s->tables.ensure(chee_decode_tables_bytes(n, s->num_sms) + 256, st);
        if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    }
    a.ws = s->ws.p; a.tables = s->tables.p;
    uint64_t launches = 0;
    if (n) e = chee_shard_phase1(a, d_cmap_out, st, &launches);
    else if (d_cmap_out) e = chee_cmap_identity(d_cmap_out, st, &launches);    // an empty piece passes the chunk map on unchanged
    g_launches += launches;
    if (e != cudaSuccess) { set_error("cheetah decode shard phase1", e); return DENSITY_B200_ECUDA; }
    s->phase = 1;
    return DENSITY_B200_OK;
}
static int cd_phase2_impl(density_b200_cheetah_decode_shard* s, const uint32_t* d_cmap_carry, cudaStream_t st) {
    if (s->phase != 1) { set_error("cheetah_decode_shard_phase2: phase 1 not done"); return DENSITY_B200_EARG; }
    uint64_t launches = 0;
    cudaError_t e = s->a.n ? chee_shard_phase2(s->a, d_cmap_carry, st, &launches) : cudaSuccess;
    g_launches += launches;
    if (e != cudaSuccess) { set_error("cheetah decode shard phase2", e); return DENSITY_B200_ECUDA; }
    s->phase = 2;
    return DENSITY_B200_OK;
}
static int cd_round_walk_impl(density_b200_cheetah_decode_shard* s, uint32_t* d_pred_out, uint32_t* d_words4, cudaStream_t st) {
    if (s->phase != 2) { set_error("cheetah_decode_shard_round_walk: phase 2 or the previous round's fold not done"); return DENSITY_B200_EARG; }
    if (!d_words4) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (s->round >= (uint32_t)g_chee_dec_rounds) { set_error("cheetah_decode_shard_round_walk: round budget used up"); return DENSITY_B200_EARG; }
    uint64_t launches = 0;
    cudaError_t e;
    if (s->a.n) e = chee_shard_round_walk(s->a, s->round, d_pred_out, d_words4, st, &launches);
    else {   // an empty piece: the identity transfer, no exit context, nothing walked
        e = cudaMemsetAsync(d_words4, 0, 4 * sizeof(uint32_t), st);
        if (e == cudaSuccess && d_pred_out) e = cudaMemsetAsync(d_pred_out, 0, 2 * 65536 * sizeof(uint32_t), st);
    }
    g_launches += launches;
    if (e != cudaSuccess) { set_error("cheetah decode shard round walk", e); return DENSITY_B200_ECUDA; }
    s->phase = 3;
    return DENSITY_B200_OK;
}
static int cd_round_fold_impl(density_b200_cheetah_decode_shard* s, const uint32_t* d_pred_carry, const uint32_t* d_all_words, int world, int rank,
                              cudaStream_t st) {
    if (s->phase != 3) { set_error("cheetah_decode_shard_round_fold: the round's walk not done"); return DENSITY_B200_EARG; }
    if (!d_all_words || world < 1 || rank < 0 || rank >= world) { set_error("cheetah_decode_shard_round_fold: null pointer / bad rank or world"); return DENSITY_B200_EARG; }
    uint64_t launches = 0;
    cudaError_t e = s->a.n ? chee_shard_round_fold(s->a, s->round, d_pred_carry, d_all_words, (uint32_t)world, (uint32_t)rank, st, &launches) : cudaSuccess;
    g_launches += launches;
    if (e != cudaSuccess) { set_error("cheetah decode shard round fold", e); return DENSITY_B200_ECUDA; }
    s->phase = 2; ++s->round;
    return DENSITY_B200_OK;
}
static int cd_phase3_impl(density_b200_cheetah_decode_shard* s, uint64_t* d_out_size, uint32_t* d_seam8, cudaStream_t st) {
    if (s->phase != 2) { set_error("cheetah_decode_shard_phase3: phase 2 or the last round's fold not done"); return DENSITY_B200_EARG; }
    if (!d_out_size || !d_seam8) { set_error("null pointer"); return DENSITY_B200_EARG; }
    uint64_t launches = 0;
    cudaError_t e;
    if (s->a.n) e = chee_shard_phase3(s->a, d_out_size, d_seam8, st, &launches);
    else {
        e = cudaMemsetAsync(d_out_size, 0, sizeof(uint64_t), st);
        if (e == cudaSuccess) e = cudaMemsetAsync(d_seam8, 0, 8 * sizeof(uint32_t), st);
    }
    g_launches += launches;
    if (e != cudaSuccess) { set_error("cheetah decode shard phase3", e); return DENSITY_B200_ECUDA; }
    s->phase = 4;
    return DENSITY_B200_OK;
}
int density_b200_cheetah_decode_shard_phase1(density_b200_cheetah_decode_shard* s, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap,
                                             int is_first, int is_last, uint32_t* d_cmap_out, void* stream) {
    g_last_error.clear();
    if (!s) { set_error("null pointer"); return DENSITY_B200_EARG; }
    return cd_phase1_impl(s, d_in, n, d_out, cap, is_first, is_last, d_cmap_out, reinterpret_cast<cudaStream_t>(stream));
}
int density_b200_cheetah_decode_shard_phase2(density_b200_cheetah_decode_shard* s, const uint32_t* d_cmap_carry, void* stream) {
    g_last_error.clear();
    if (!s) { set_error("null pointer"); return DENSITY_B200_EARG; }
    return cd_phase2_impl(s, d_cmap_carry, reinterpret_cast<cudaStream_t>(stream));
}
int density_b200_cheetah_decode_shard_round_walk(density_b200_cheetah_decode_shard* s, uint32_t* d_pred_out, uint32_t* d_words4, void* stream) {
    g_last_error.clear();
    if (!s) { set_error("null pointer"); return DENSITY_B200_EARG; }
    return cd_round_walk_impl(s, d_pred_out, d_words4, reinterpret_cast<cudaStream_t>(stream));
}
int density_b200_cheetah_decode_shard_round_fold(density_b200_cheetah_decode_shard* s, const uint32_t* d_pred_carry, const uint32_t* d_all_words,
                                                 int world, int rank, void* stream) {
    g_last_error.clear();
    if (!s) { set_error("null pointer"); return DENSITY_B200_EARG; }
    return cd_round_fold_impl(s, d_pred_carry, d_all_words, world, rank, reinterpret_cast<cudaStream_t>(stream));
}
int density_b200_cheetah_decode_shard_phase3(density_b200_cheetah_decode_shard* s, uint64_t* d_out_size, uint32_t* d_seam8, void* stream) {
    g_last_error.clear();
    if (!s) { set_error("null pointer"); return DENSITY_B200_EARG; }
    return cd_phase3_impl(s, d_out_size, d_seam8, reinterpret_cast<cudaStream_t>(stream));
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
    cudaError_t e = chee_cmap_init(d_table, reinterpret_cast<cudaStream_t>(stream), &l);
    g_launches += l;
    if (e != cudaSuccess) { set_error("cheetah_cmap_init", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}
int density_b200_cheetah_cmap_fold(uint32_t* d_acc, const uint32_t* d_next, void* stream) {
    g_last_error.clear();
    if (!d_acc || !d_next) { set_error("null pointer"); return DENSITY_B200_EARG; }
    uint64_t l = 0;
    cudaError_t e = chee_cmap_fold(d_acc, d_next, reinterpret_cast<cudaStream_t>(stream), &l);
    g_launches += l;
    if (e != cudaSuccess) { set_error("cheetah_cmap_fold", e); return DENSITY_B200_ECUDA; }
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
NcclApi* nccl_api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return;
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
    });
    return api.ok ? &api : nullptr;
}
bool nccl_check(int rc, const char* what) {
    if (rc == 0) return true;
    NcclApi* a = nccl_api();
    std::string m = std::string(what) + ": " + ((a && a->GetErrorString) ? a->GetErrorString(rc) : "NCCL error");
    dns::set_error(m.c_str());
    return false;
}
}  // namespace

struct density_b200_sharded {
    int rank = 0, world = 1, num_sms = 0;
    nccl_comm_t comm = nullptr;
    DevBuf ws, aux;                 // aux: gathered tables [world][65536] + carry [65536] + seam words [world][8] + offsets [world + 1] + size
    DevBuf dws;                     // decode workspace (density_b200_decode_sharded[_stream]), apart from the encoder's
    density_b200_cl_shard* cl[2] = {nullptr, nullptr};   // Cheetah / Lion shard state of density_b200_encode_sharded_cl
    DevBuf cl_aux;                  // its exchange buffers: gathered P and C tables, the carries, the last quads
    density_b200_cheetah_decode_shard* cdec = nullptr;   // piece state of density_b200_decode_sharded_cheetah
    DevBuf cd_aux;                  // its exchange buffers: gathered chunk-map and prediction transfers, the carries, the round words
    ChamLayout L{};
    uint64_t* h_offsets = nullptr;  // pinned, world + 1
    uint64_t* h_maps = nullptr;     // pinned, world range maps (density_b200_decode_sharded_stream)
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
    }
    if (cudaMallocHost(&h->h_offsets, sizeof(uint64_t) * (world + 2)) != cudaSuccess ||
        cudaMallocHost(&h->h_maps, sizeof(uint64_t) * DENSITY_B200_LOCATE_MAP_WORDS * world) != cudaSuccess) {
        set_error("cudaMallocHost");
        if (h->h_offsets) cudaFreeHost(h->h_offsets);
        if (h->comm) { NcclApi* a = nccl_api(); if (a) a->CommDestroy(h->comm); }
        delete h;
        return nullptr;
    }
    for (auto& e : h->ev) cudaEventCreate(&e);
    return h;
}

void density_b200_sharded_destroy(density_b200_sharded* h) {
    if (!h) return;
    if (h->comm) { NcclApi* a = nccl_api(); if (a) a->CommDestroy(h->comm); }
    h->ws.release(); h->aux.release(); h->dws.release(); h->cl_aux.release(); h->cd_aux.release();
    for (auto* s : h->cl) density_b200_cl_shard_destroy(s);
    density_b200_cheetah_decode_shard_destroy(h->cdec);
    if (h->h_offsets) cudaFreeHost(h->h_offsets);
    if (h->h_maps) cudaFreeHost(h->h_maps);
    for (auto& e : h->ev) if (e) cudaEventDestroy(e);
    delete h;
}

// the exchange buffers of a handle, shared by encode and decode
struct ShardedAux { uint32_t *tables, *carry, *words; uint64_t *offsets, *maps; };
static cudaError_t sharded_aux(density_b200_sharded* h, cudaStream_t st, ShardedAux* x) {
    const size_t W = (size_t)h->world;
    const size_t aux_tables = W * 65536 * sizeof(uint32_t), aux_carry = 65536 * sizeof(uint32_t), aux_words = W * 8 * sizeof(uint32_t);
    const size_t aux_offsets = (W + 2) * sizeof(uint64_t), aux_maps = W * DENSITY_B200_LOCATE_MAP_WORDS * sizeof(uint64_t);
    const cudaError_t e = h->aux.ensure(aux_tables + aux_carry + aux_words + aux_offsets + aux_maps + 256, st);
    x->tables = reinterpret_cast<uint32_t*>(h->aux.p);
    x->carry = reinterpret_cast<uint32_t*>(h->aux.p + aux_tables);
    x->words = reinterpret_cast<uint32_t*>(h->aux.p + aux_tables + aux_carry);
    x->offsets = reinterpret_cast<uint64_t*>(h->aux.p + aux_tables + aux_carry + aux_words);
    x->maps = reinterpret_cast<uint64_t*>(h->aux.p + aux_tables + aux_carry + aux_words + aux_offsets);
    return e;
}

// variable-length gather of the pieces to `gather_root` at their stream offsets (d_offsets: world + 1 prefix sums, on the device); blocks
static int gather_pieces(density_b200_sharded* h, NcclApi* a, const uint64_t* d_offsets, const uint8_t* d_out, int gather_root, uint8_t* d_gather,
                         size_t gather_cap, cudaStream_t st) {
    const size_t W = (size_t)h->world;
    cudaError_t e;
    // variable-length gather of the pieces at their stream offsets (SURVEY §8e step 5): sizes -> host -> grouped send / recv
    e = cudaMemcpyAsync(h->h_offsets, d_offsets, (W + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("gather: sizes to host", e); return DENSITY_B200_ECUDA; }
    const uint64_t total = h->h_offsets[W];
    const uint64_t my_off = h->h_offsets[h->rank], my_size = h->h_offsets[h->rank + 1] - my_off;
    if (h->rank == gather_root) {
        if (!d_gather || gather_cap < total) { set_error("gather buffer too small"); return DENSITY_B200_ECAPACITY; }
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

// One bit-exact stream cut across `world` GPUs; this rank's shard is d_in[0 .. n) (n % 256 == 0 except on the last rank).
// All work is enqueued on `stream`. With gather_root >= 0 the call BLOCKS on the stream once (the piece sizes must reach the host before
// the variable-length ncclSend / ncclRecv can be posted) and the pieces land in d_gather on rank gather_root at their stream offsets.
int density_b200_encode_sharded(density_b200_sharded* h, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                uint32_t* d_flags, uint64_t* d_total_size, int gather_root, uint8_t* d_gather, size_t gather_cap, void* stream_v) {
    g_last_error.clear();
    if (!h || (!d_in && n) || !d_out || !d_out_size) { set_error("null pointer"); return DENSITY_B200_EARG; }
    const bool last = h->rank == h->world - 1;
    if (!last && (n % 256)) { set_error("non-final shards must be a multiple of 256 bytes"); return DENSITY_B200_EARG; }
    if ((reinterpret_cast<uintptr_t>(d_in) & 3) || (reinterpret_cast<uintptr_t>(d_out) & 1)) { set_error("d_in must be 4-byte, d_out 2-byte aligned"); return DENSITY_B200_EARG; }
    if (gather_root >= h->world) { set_error("bad gather root"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
    NcclApi* a = h->world > 1 ? nccl_api() : nullptr;
    cudaError_t e = h->ws.ensure(cham_workspace_bytes(n, h->num_sms, &h->L), st);
    ShardedAux x;
    if (e == cudaSuccess) e = sharded_aux(h, st, &x);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    uint32_t* d_tables = x.tables;
    uint32_t* d_carry = x.carry;
    uint32_t* d_words = x.words;
    uint64_t* d_offsets = x.offsets;
    const uint32_t nruns = cham_pick_runs(n, h->num_sms);
    uint64_t launches = 0;
    cudaEventRecord(h->ev[0], st);
    // phase 1: flags with unknown carry-in; my last-writer table lands in my slot of the gather buffer
    cudaEvent_t pev[4] = {nullptr, nullptr, nullptr, nullptr};
    if (n) e = cham_encode_phase1(d_in, n, h->ws.p, h->L, nruns, d_tables + (size_t)h->rank * 65536, st, &launches);
    else e = cudaMemsetAsync(d_tables + (size_t)h->rank * 65536, 0, 65536 * sizeof(uint32_t), st);
    if (e != cudaSuccess) { set_error("sharded phase 1", e); return DENSITY_B200_ECUDA; }
    cudaEventRecord(h->ev[1], st);
    // the one exchange step of the path: 256 KiB per rank over NVLink, then ONE fold kernel
    if (h->world > 1) {
        if (!a) { set_error("NCCL is not available"); return DENSITY_B200_ECUDA; }
        if (!nccl_check(a->AllGather(d_tables + (size_t)h->rank * 65536, d_tables, 65536, NCCL_UINT32, h->comm, st), "ncclAllGather(tables)")) return DENSITY_B200_ECUDA;
    }
    e = cham_rank_fold(d_tables, (uint32_t)h->rank, d_carry, st, &launches);
    cudaEventRecord(h->ev[2], st);
    // phase 2: carry-in, first-touch flags, sizes, scan, emit (seams are judged below, exactly, once every shard knows its flags)
    pev[2] = h->ev[3]; pev[3] = h->ev[4];
    if (e == cudaSuccess) e = cham_encode_phase2(d_in, n, h->ws.p, h->L, nruns, d_carry, d_out, cap, d_out_size, false, false, st, &launches, n ? pev : nullptr);
    if (!n) { cudaEventRecord(h->ev[3], st); cudaEventRecord(h->ev[4], st); }
    if (e == cudaSuccess && n) e = cham_seam_words(h->ws.p, h->L, n, d_out_size, d_words + 8 * h->rank, st, &launches);
    else if (e == cudaSuccess) e = cudaMemsetAsync(d_words + 8 * h->rank, 0, 8 * sizeof(uint32_t), st);
    if (e != cudaSuccess) { set_error("sharded phase 2", e); return DENSITY_B200_ECUDA; }
    if (h->world > 1 && !nccl_check(a->AllGather(d_words + 8 * h->rank, d_words, 8, NCCL_UINT32, h->comm, st), "ncclAllGather(seams)")) return DENSITY_B200_ECUDA;
    e = cham_seam_verdict(d_words, (uint32_t)h->world, (uint32_t)h->rank, d_flags, d_total_size, d_offsets, st, &launches);
    if (e != cudaSuccess) { set_error("seam verdict", e); return DENSITY_B200_ECUDA; }
    if (gather_root >= 0) {
        const int rc = gather_pieces(h, a, d_offsets, d_out, gather_root, d_gather, gather_cap, st);
        if (rc != DENSITY_B200_OK) return rc;
    }
    cudaEventRecord(h->ev[5], st);
    h->timed = true;
    g_launches += launches;
    return DENSITY_B200_OK;
}

// Sharded Cheetah / Lion encode over the handle's communicator: last quads -> phase 1 -> P tables -> fold -> phase 2 -> C tables -> fold
// -> phase 3 -> seam words -> verdict -> optional gather, as density_b200_encode_sharded. The exchanges are ncclAllGathers on `stream`.
int density_b200_encode_sharded_cl(density_b200_sharded* h, int alg, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                   uint32_t* d_flags, uint64_t* d_total_size, int gather_root, uint8_t* d_gather, size_t gather_cap, void* stream_v) {
    g_last_error.clear();
    if (!h || (!d_in && n) || !d_out || !d_out_size) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if (!cl_alg_ok(alg)) { set_error("encode_sharded_cl: alg must be DENSITY_B200_CHEETAH or DENSITY_B200_LION"); return DENSITY_B200_EARG; }
    const bool last = h->rank == h->world - 1;
    if (!last && (n % 256)) { set_error("non-final shards must be a multiple of 256 bytes"); return DENSITY_B200_EARG; }
    if ((reinterpret_cast<uintptr_t>(d_in) & 3) || (reinterpret_cast<uintptr_t>(d_out) & 1)) { set_error("d_in must be 4-byte, d_out 2-byte aligned"); return DENSITY_B200_EARG; }
    if (gather_root >= h->world) { set_error("bad gather root"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
    NcclApi* a = h->world > 1 ? nccl_api() : nullptr;
    if (h->world > 1 && !a) { set_error("NCCL is not available"); return DENSITY_B200_ECUDA; }
    density_b200_cl_shard*& s = h->cl[alg - ALG_CHEETAH];
    if (!s) { s = new density_b200_cl_shard(); s->alg = alg; s->num_sms = h->num_sms; }
    const size_t W = (size_t)h->world, R = (size_t)h->rank;
    const size_t wp = density_b200_cl_table_words(alg, DENSITY_B200_CL_TABLE_P), wc = density_b200_cl_table_words(alg, DENSITY_B200_CL_TABLE_C);
    ShardedAux x;
    cudaError_t e = sharded_aux(h, st, &x);
    if (e == cudaSuccess) e = h->cl_aux.ensure(((W + 1) * (wp + wc) + 2 * W + 64) * sizeof(uint32_t), st);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    uint32_t* tab_p = reinterpret_cast<uint32_t*>(h->cl_aux.p);          // [world][wp]
    uint32_t* carry_p = tab_p + W * wp;
    uint32_t* tab_c = carry_p + wp;                                       // [world][wc]
    uint32_t* carry_c = tab_c + W * wc;
    uint32_t* quads = carry_c + wc;                                       // [world] {has a quad, last quad}
    uint32_t* prev_quad = quads + 2 * W;
    uint64_t launches = 0;
    auto gather = [&](uint32_t* buf, size_t words, const char* what) {
        return h->world == 1 || nccl_check(a->AllGather(buf + R * words, buf, words, NCCL_UINT32, h->comm, st), what);
    };
    // 0. the context of my first quad: the last quad of the nearest earlier shard that has one
    e = cl_last_quad(d_in, n, quads + 2 * R, st, &launches);
    if (e == cudaSuccess && !gather(quads, 2, "ncclAllGather(last quads)")) return DENSITY_B200_ECUDA;
    if (e == cudaSuccess) e = cl_prev_quad(quads, (uint32_t)R, prev_quad, st, &launches);
    g_launches += launches; launches = 0;
    if (e != cudaSuccess) { set_error("sharded cl: last quads", e); return DENSITY_B200_ECUDA; }
    // 1-2. predictions, exchange, fold
    cudaEventRecord(h->ev[0], st);
    int rc = cl_phase1_impl(s, d_in, n, last, R ? prev_quad : nullptr, tab_p + R * wp, st);
    if (rc != DENSITY_B200_OK) return rc;
    cudaEventRecord(h->ev[1], st);
    if (!gather(tab_p, wp, "ncclAllGather(P tables)")) return DENSITY_B200_ECUDA;
    e = cl_rank_fold(alg, DENSITY_B200_CL_TABLE_P, tab_p, (uint32_t)R, carry_p, st, &launches);
    g_launches += launches; launches = 0;
    if (e != cudaSuccess) { set_error("sharded cl: P fold", e); return DENSITY_B200_ECUDA; }
    cudaEventRecord(h->ev[2], st);
    // 3-4. chunk map, exchange, fold
    rc = cl_phase2_impl(s, carry_p, tab_c + R * wc, st);
    if (rc != DENSITY_B200_OK) return rc;
    if (!gather(tab_c, wc, "ncclAllGather(C tables)")) return DENSITY_B200_ECUDA;
    e = cl_rank_fold(alg, DENSITY_B200_CL_TABLE_C, tab_c, (uint32_t)R, carry_c, st, &launches);
    g_launches += launches; launches = 0;
    if (e != cudaSuccess) { set_error("sharded cl: C fold", e); return DENSITY_B200_ECUDA; }
    cudaEventRecord(h->ev[3], st);
    // 5. emit and seam words, the verdict over all shards, the optional gather
    rc = cl_phase3_impl(s, carry_c, d_out, cap, d_out_size, x.words + 8 * R, st);
    if (rc != DENSITY_B200_OK) return rc;
    cudaEventRecord(h->ev[4], st);
    if (!gather(x.words, 8, "ncclAllGather(seams)")) return DENSITY_B200_ECUDA;
    e = cham_seam_verdict(x.words, (uint32_t)h->world, (uint32_t)h->rank, d_flags, d_total_size, x.offsets, st, &launches);
    g_launches += launches;
    if (e != cudaSuccess) { set_error("seam verdict", e); return DENSITY_B200_ECUDA; }
    if (gather_root >= 0) {
        rc = gather_pieces(h, a, x.offsets, d_out, gather_root, d_gather, gather_cap, st);
        if (rc != DENSITY_B200_OK) return rc;
    }
    cudaEventRecord(h->ev[5], st);
    h->timed = true;
    return DENSITY_B200_OK;
}

// The decode of this rank's piece d_in[0 .. n) with the dictionary carried in from the pieces before it, over the handle's communicator:
// phase 1 -> table exchange -> fold -> phase 2 -> seam words -> verdict. is_last: the piece ends the stream (a non-final piece must decode
// to whole 256-byte blocks). d_out_offset (may be NULL): where the piece's output starts, from the verdict's prefix offsets.
static int decode_sharded_piece(density_b200_sharded* h, const uint8_t* d_in, size_t n, int is_last, uint8_t* d_out, size_t cap,
                                uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, uint64_t* d_out_offset, cudaStream_t st) {
    NcclApi* a = h->world > 1 ? nccl_api() : nullptr;
    if (h->world > 1 && !a) { set_error("NCCL is not available"); return DENSITY_B200_ECUDA; }
    ShardedAux x;
    cudaError_t e = h->dws.ensure(cham_decode_workspace_bytes(n, cap, h->num_sms), st);
    if (e == cudaSuccess) e = sharded_aux(h, st, &x);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    uint32_t* my_table = x.tables + (size_t)h->rank * 65536;
    uint32_t* my_words = x.words + 8 * h->rank;
    uint64_t launches = 0;
    // phase 1: boundaries and writer pass need no carry-in; the piece's table (runs + tail) lands in my slot of the gather buffer
    if (n) e = cham_decode_phase1(d_in, n, cap, h->dws.p, h->num_sms, my_table, st, &launches);
    else e = cudaMemsetAsync(my_table, 0, 65536 * sizeof(uint32_t), st);
    if (e != cudaSuccess) { set_error("sharded decode phase 1", e); return DENSITY_B200_ECUDA; }
    if (h->world > 1 && !nccl_check(a->AllGather(my_table, x.tables, 65536, NCCL_UINT32, h->comm, st), "ncclAllGather(tables)")) return DENSITY_B200_ECUDA;
    e = cham_rank_fold(x.tables, (uint32_t)h->rank, x.carry, st, &launches);
    // phase 2: decode from the carried-in dictionary, then the seam words; the verdict reads them from every rank
    if (e == cudaSuccess && n) e = cham_decode_phase2(d_in, n, d_out, cap, h->dws.p, h->num_sms, x.carry, d_out_size, st, &launches);
    if (e == cudaSuccess && n) e = cham_decode_seam_words(d_in, n, cap, h->dws.p, h->num_sms, is_last, d_out_size, my_words, st, &launches);
    if (e == cudaSuccess && !n) e = cudaMemsetAsync(d_out_size, 0, sizeof(uint64_t), st);
    if (e == cudaSuccess && !n) e = cudaMemsetAsync(my_words, 0, 8 * sizeof(uint32_t), st);
    if (e != cudaSuccess) { set_error("sharded decode phase 2", e); return DENSITY_B200_ECUDA; }
    if (h->world > 1 && !nccl_check(a->AllGather(my_words, x.words, 8, NCCL_UINT32, h->comm, st), "ncclAllGather(seams)")) return DENSITY_B200_ECUDA;
    e = cham_seam_verdict(x.words, (uint32_t)h->world, (uint32_t)h->rank, d_flags, d_total_size, x.offsets, st, &launches);
    g_launches += launches;
    if (e == cudaSuccess && d_out_offset) e = cudaMemcpyAsync(d_out_offset, x.offsets + h->rank, sizeof(uint64_t), cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) { set_error("seam verdict", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}

// The inverse of density_b200_encode_sharded without a gather: this rank's piece d_in[0 .. n) decodes to the shard it was encoded from.
// Everything is enqueued on `stream`; nothing blocks.
int density_b200_decode_sharded(density_b200_sharded* h, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                uint32_t* d_flags, uint64_t* d_total_size, void* stream_v) {
    g_last_error.clear();
    if (!h || (!d_in && n) || (!d_out && cap) || !d_out_size || !d_flags) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if ((reinterpret_cast<uintptr_t>(d_in) & 1) || (reinterpret_cast<uintptr_t>(d_out) & 3)) { set_error("d_in must be 2-byte, d_out 4-byte aligned"); return DENSITY_B200_EARG; }
    return decode_sharded_piece(h, d_in, n, h->rank == h->world - 1, d_out, cap, d_out_size, d_flags, d_total_size, nullptr,
                                reinterpret_cast<cudaStream_t>(stream_v));
}

static density_b200_cheetah_decode_shard* sharded_cdec(density_b200_sharded* h) {
    if (!h->cdec) { h->cdec = new density_b200_cheetah_decode_shard(); h->cdec->num_sms = h->num_sms; }
    return h->cdec;
}

// Sharded Cheetah decode of this rank's piece d_in[0 .. n) over the handle's communicator: phase 1 -> chunk-map transfers -> fold ->
// phase 2 -> every round of the budget (walk -> prediction transfers + round words -> fold) -> phase 3 -> seam words -> verdict. Every
// rank issues the same collectives in the same order whatever its piece holds: an empty piece sends identity transfers and zero words, a
// refused one keeps exchanging until the verdict. The rounds after the settled one are gated off on the device; their all-gathers still
// run. first: the piece holds the stream start; last: no stream byte follows it. d_out_offset (may be NULL): where the piece's output
// starts, from the verdict's prefix offsets.
static int decode_sharded_cheetah_piece(density_b200_sharded* h, const uint8_t* d_in, size_t n, bool first, bool last, uint8_t* d_out, size_t cap,
                                        uint64_t* d_out_size, uint32_t* d_flags, uint64_t* d_total_size, uint64_t* d_out_offset, cudaStream_t st) {
    NcclApi* a = h->world > 1 ? nccl_api() : nullptr;
    if (h->world > 1 && !a) { set_error("NCCL is not available"); return DENSITY_B200_ECUDA; }
    density_b200_cheetah_decode_shard* s = sharded_cdec(h);
    const size_t W = (size_t)h->world, R = (size_t)h->rank;
    const size_t wc = density_b200_cheetah_cmap_words(), wp = 2 * 65536;
    ShardedAux x;
    cudaError_t e = sharded_aux(h, st, &x);
    if (e == cudaSuccess) e = h->cd_aux.ensure(((W + 1) * (wc + wp) + 4 * W + 64) * sizeof(uint32_t), st);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    uint32_t* tab_c = reinterpret_cast<uint32_t*>(h->cd_aux.p);         // [world][wc]
    uint32_t* carry_c = tab_c + W * wc;
    uint32_t* tab_p = carry_c + wc;                                       // [world][wp]
    uint32_t* carry_p = tab_p + W * wp;
    uint32_t* rwords = carry_p + wp;                                      // [world][4]
    uint64_t launches = 0;
    auto gather = [&](uint32_t* buf, size_t words, const char* what) {
        return h->world == 1 || nccl_check(a->AllGather(buf + R * words, buf, words, NCCL_UINT32, h->comm, st), what);
    };
    // the last piece's transfers are never read: it sends what its slot holds
    int rc = cd_phase1_impl(s, d_in, n, d_out, cap, first, last, last ? nullptr : tab_c + R * wc, st);
    if (rc != DENSITY_B200_OK) return rc;
    if (!gather(tab_c, wc, "ncclAllGather(chunk-map transfers)")) return DENSITY_B200_ECUDA;
    if (!first) e = chee_cmap_rank_fold(tab_c, (uint32_t)R, carry_c, st, &launches);
    g_launches += launches; launches = 0;
    if (e != cudaSuccess) { set_error("sharded cheetah decode: chunk-map fold", e); return DENSITY_B200_ECUDA; }
    rc = cd_phase2_impl(s, first ? nullptr : carry_c, st);
    if (rc != DENSITY_B200_OK) return rc;
    for (int k = 0; k < g_chee_dec_rounds; ++k) {
        rc = cd_round_walk_impl(s, last ? nullptr : tab_p + R * wp, rwords + 4 * R, st);
        if (rc != DENSITY_B200_OK) return rc;
        if (!gather(tab_p, wp, "ncclAllGather(prediction transfers)") || !gather(rwords, 4, "ncclAllGather(round words)")) return DENSITY_B200_ECUDA;
        if (!first) e = cl_rank_fold(ALG_CHEETAH, DENSITY_B200_CL_TABLE_P, tab_p, (uint32_t)R, carry_p, st, &launches);
        g_launches += launches; launches = 0;
        if (e != cudaSuccess) { set_error("sharded cheetah decode: prediction fold", e); return DENSITY_B200_ECUDA; }
        rc = cd_round_fold_impl(s, first ? nullptr : carry_p, rwords, (int)W, (int)R, st);
        if (rc != DENSITY_B200_OK) return rc;
    }
    rc = cd_phase3_impl(s, d_out_size, x.words + 8 * R, st);
    if (rc != DENSITY_B200_OK) return rc;
    if (!gather(x.words, 8, "ncclAllGather(seams)")) return DENSITY_B200_ECUDA;
    e = cham_seam_verdict(x.words, (uint32_t)h->world, (uint32_t)h->rank, d_flags, d_total_size, x.offsets, st, &launches);
    g_launches += launches;
    if (e == cudaSuccess && d_out_offset) e = cudaMemcpyAsync(d_out_offset, x.offsets + h->rank, sizeof(uint64_t), cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) { set_error("seam verdict", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}

// The pieces of a sharded Cheetah encode: rank 0 holds the stream start, the last rank its end.
int density_b200_decode_sharded_cheetah(density_b200_sharded* h, const uint8_t* d_in, size_t n, uint8_t* d_out, size_t cap, uint64_t* d_out_size,
                                        uint32_t* d_flags, uint64_t* d_total_size, void* stream_v) {
    g_last_error.clear();
    if (!h || (!d_in && n) || (!d_out && cap) || !d_out_size || !d_flags) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if ((reinterpret_cast<uintptr_t>(d_in) & 1) || (reinterpret_cast<uintptr_t>(d_out) & 3)) { set_error("d_in must be 2-byte, d_out 4-byte aligned"); return DENSITY_B200_EARG; }
    return decode_sharded_cheetah_piece(h, d_in, n, h->rank == 0, h->rank == h->world - 1, d_out, cap, d_out_size, d_flags, d_total_size, nullptr,
                                        reinterpret_cast<cudaStream_t>(stream_v));
}

int density_b200_decode_locate(density_b200_decode_shard* s, const uint8_t* d_in, size_t n_range, size_t n_halo, uint64_t* d_map, void* stream) {
    g_last_error.clear();
    if (!s || (!d_in && n_range + n_halo) || !d_map) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if ((reinterpret_cast<uintptr_t>(d_in) & 1) || (reinterpret_cast<uintptr_t>(d_map) & 7)) { set_error("d_in must be 2-byte, d_map 8-byte aligned"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    s->phase1_done = false;     // the scratch is phase 1's
    cudaError_t e = s->ws.ensure(cham_locate_workspace_bytes(n_range + n_halo), st);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    uint64_t launches = 0;
    e = cham_decode_locate(d_in, n_range, n_halo, s->ws.p, d_map, st, &launches);
    g_launches += launches;
    if (e != cudaSuccess) { set_error("decode locate", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
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
    g_last_error.clear();
    if (!s || (!d_in && n_range + n_halo) || !d_map) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if ((reinterpret_cast<uintptr_t>(d_in) & 1) || (reinterpret_cast<uintptr_t>(d_map) & 7)) { set_error("d_in must be 2-byte, d_map 8-byte aligned"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    s->phase = 0;               // the scratch is phase 1's
    cudaError_t e = s->ws.ensure(chee_locate_workspace_bytes(n_range, n_halo, range_offset), st);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    uint64_t launches = 0;
    e = chee_decode_locate(d_in, n_range, n_halo, range_offset, s->ws.p, d_map, st, &launches);
    g_launches += launches;
    if (e != cudaSuccess) { set_error("cheetah decode locate", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}

// Sharded decode of a stream without known cuts: this rank holds its range + halo (include/density_b200.h). Locates the piece (one
// host synchronisation), then decodes it as density_b200_decode_sharded does.
int density_b200_decode_sharded_stream(density_b200_sharded* h, const uint8_t* d_in, size_t n_range, size_t n_halo, uint8_t* d_out, size_t cap,
                                       uint64_t* d_out_size, uint64_t* d_out_offset, uint32_t* d_flags, uint64_t* d_total_size, void* stream_v) {
    g_last_error.clear();
    if (!h || (!d_in && n_range + n_halo) || (!d_out && cap) || !d_out_size || !d_flags) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if ((reinterpret_cast<uintptr_t>(d_in) & 1) || (reinterpret_cast<uintptr_t>(d_out) & 3)) { set_error("d_in must be 2-byte, d_out 4-byte aligned"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
    NcclApi* a = h->world > 1 ? nccl_api() : nullptr;
    if (h->world > 1 && !a) { set_error("NCCL is not available"); return DENSITY_B200_ECUDA; }
    const size_t W = (size_t)h->world;
    ShardedAux x;
    // sized for the whole range + halo: covers the locate scratch and the phases on any piece of it
    cudaError_t e = h->dws.ensure(cham_decode_workspace_bytes(n_range + n_halo, cap, h->num_sms), st);
    if (e == cudaSuccess) e = sharded_aux(h, st, &x);
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    uint64_t* my_map = x.maps + (size_t)h->rank * DENSITY_B200_LOCATE_MAP_WORDS;
    uint64_t launches = 0;
    e = cham_decode_locate(d_in, n_range, n_halo, h->dws.p, my_map, st, &launches);
    g_launches += launches;
    if (e != cudaSuccess) { set_error("decode locate", e); return DENSITY_B200_ECUDA; }
    if (h->world > 1 && !nccl_check(a->AllGather(my_map, x.maps, DENSITY_B200_LOCATE_MAP_WORDS * 8, NCCL_UINT8, h->comm, st), "ncclAllGather(maps)"))
        return DENSITY_B200_ECUDA;
    e = cudaMemcpyAsync(h->h_maps, x.maps, W * DENSITY_B200_LOCATE_MAP_WORDS * sizeof(uint64_t), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("range maps to host", e); return DENSITY_B200_ECUDA; }
    uint64_t piece[4];
    const int rc = density_b200_locate_piece(h->h_maps, h->world, h->rank, piece);
    if (rc != DENSITY_B200_OK) return rc;    // the same verdict on every rank: none enters the collectives below
    return decode_sharded_piece(h, d_in + piece[0], (size_t)(piece[1] - piece[0]), (int)piece[3], d_out, cap, d_out_size, d_flags,
                                d_total_size, d_out_offset, st);
}

// Sharded decode of a Cheetah stream without known cuts: this rank holds its range + halo at range_offset (include/density_b200.h).
// Locates the piece (one host synchronisation), then decodes it as density_b200_decode_sharded_cheetah does, with the piece's own
// "holds the stream start" and "ends the stream" rather than the rank's.
int density_b200_decode_sharded_cheetah_stream(density_b200_sharded* h, const uint8_t* d_in, size_t n_range, size_t n_halo, uint64_t range_offset,
                                               uint8_t* d_out, size_t cap, uint64_t* d_out_size, uint64_t* d_out_offset, uint32_t* d_flags,
                                               uint64_t* d_total_size, void* stream_v) {
    g_last_error.clear();
    if (!h || (!d_in && n_range + n_halo) || (!d_out && cap) || !d_out_size || !d_flags) { set_error("null pointer"); return DENSITY_B200_EARG; }
    if ((reinterpret_cast<uintptr_t>(d_in) & 1) || (reinterpret_cast<uintptr_t>(d_out) & 3)) { set_error("d_in must be 2-byte, d_out 4-byte aligned"); return DENSITY_B200_EARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_v);
    NcclApi* a = h->world > 1 ? nccl_api() : nullptr;
    if (h->world > 1 && !a) { set_error("NCCL is not available"); return DENSITY_B200_ECUDA; }
    constexpr size_t MW = DENSITY_B200_CHEETAH_LOCATE_MAP_WORDS;
    density_b200_cheetah_decode_shard* s = sharded_cdec(h);
    ShardedAux x;
    // sized for the locate scratch and for the phases on any piece of range + halo, so that phase 1 does not reallocate
    const size_t locate_bytes = chee_locate_workspace_bytes(n_range, n_halo, range_offset);
    const size_t piece_bytes = chee_shard_workspace_bytes(n_range + n_halo, cap, h->num_sms);
    cudaError_t e = s->ws.ensure(locate_bytes > piece_bytes ? locate_bytes : piece_bytes, st);
    if (e == cudaSuccess) e = sharded_aux(h, st, &x);    // its map slots hold DENSITY_B200_LOCATE_MAP_WORDS >= MW words per rank
    if (e != cudaSuccess) { set_error("workspace cudaMalloc", e); return DENSITY_B200_ECUDA; }
    uint64_t* my_map = x.maps + (size_t)h->rank * MW;
    uint64_t launches = 0;
    e = chee_decode_locate(d_in, n_range, n_halo, range_offset, s->ws.p, my_map, st, &launches);
    g_launches += launches;
    if (e != cudaSuccess) { set_error("cheetah decode locate", e); return DENSITY_B200_ECUDA; }
    if (h->world > 1 && !nccl_check(a->AllGather(my_map, x.maps, MW * 8, NCCL_UINT8, h->comm, st), "ncclAllGather(maps)")) return DENSITY_B200_ECUDA;
    e = cudaMemcpyAsync(h->h_maps, x.maps, (size_t)h->world * MW * sizeof(uint64_t), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("range maps to host", e); return DENSITY_B200_ECUDA; }
    uint64_t piece[5];
    const int rc = density_b200_cheetah_locate_piece(h->h_maps, h->world, h->rank, piece);
    if (rc != DENSITY_B200_OK) return rc;    // the same verdict on every rank: none enters the collectives below
    return decode_sharded_cheetah_piece(h, d_in + piece[0], (size_t)(piece[1] - piece[0]), piece[4] != 0, piece[3] != 0, d_out, cap, d_out_size,
                                        d_flags, d_total_size, d_out_offset, st);
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
    DeviceCtx* c = current_ctx();
    if (!c) return 0;
    std::lock_guard<std::mutex> lk(c->mu);
    const int alg = h->alg;
    const bool in_dev = is_device_pointer(in), out_dev = is_device_pointer(out);
    cudaError_t e = cudaSuccess;
    if (in_dev || out_dev) { e = cudaDeviceSynchronize(); if (e != cudaSuccess) { set_error("cudaDeviceSynchronize", e); return 0; } }
    cudaStream_t st = c->stream;
    if (!ws_acquire(c, st)) return 0;
    const uint8_t* d_in = in; uint8_t* d_out = out; size_t d_cap = out_cap;
    if (!in_dev) {
        e = c->stage_in.ensure(n + 16, st);
        if (e == cudaSuccess) e = cudaMemcpyAsync(c->stage_in.p, in, n, cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) { set_error("H2D copy", e); return 0; }
        d_in = c->stage_in.p;
    }
    if (!out_dev) {
        d_cap = encode ? safe_size(alg, n) : out_cap;
        e = c->stage_out.ensure(d_cap + 16, st);
        if (e != cudaSuccess) { set_error("staging cudaMalloc", e); return 0; }
        d_out = c->stage_out.p;
    }
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
        if (e == cudaSuccess) e = cham_encode_phase2_stream(d_in, n, c->ws.p, L, nruns, d_carry, d_out, d_cap, c->d_size, d_tab, 12, st, &launches, &ok);
        if (e == cudaSuccess && ok) { e = cham_table_into_quads(d_tab, quads, st, &launches); done = true; }
        c->last_was_chameleon_fastpath_capable = 0;
    }
    if (e == cudaSuccess && !done) {
        // exact in-order kernel on the instance's state (Cheetah / Lion; Chameleon decode; a Chameleon encode whose copy map did not settle)
        e = encode ? scalar_encode(alg, d_in, n, d_out, d_cap, h->state.p, c->d_size, st, &launches, nullptr, true)
                   : scalar_decode(alg, d_in, n, d_out, d_cap, h->state.p, c->d_size, st, &launches, nullptr, true);
    }
    g_launches += launches;
    if (e == cudaSuccess) e = cudaMemcpyAsync(c->h_size, c->d_size, sizeof(uint64_t), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    ws_release(c, st);
    if (e != cudaSuccess) { set_error("codec call", e); return 0; }
    const uint64_t produced = *c->h_size;
    if (produced == 0) { set_error(encode ? "encode failed on device (output capacity?)" : "decode failed on device (malformed stream or output capacity)"); return 0; }
    if (produced > out_cap) { set_error("output buffer too small"); return 0; }
    if (!out_dev) {
        e = cudaMemcpyAsync(out, d_out, produced, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("D2H copy", e); return 0; }
    }
    return (size_t)produced;
}
size_t density_b200_codec_encode(density_b200_codec* h, const uint8_t* in, size_t n, uint8_t* out, size_t cap) { return codec_run(h, true, in, n, out, cap); }
size_t density_b200_codec_decode(density_b200_codec* h, const uint8_t* in, size_t n, uint8_t* out, size_t cap) { return codec_run(h, false, in, n, out, cap); }

int density_b200_table_init(uint32_t* d_table, void* stream) {
    uint64_t l = 0;
    cudaError_t e = cham_table_init(d_table, reinterpret_cast<cudaStream_t>(stream), &l);
    g_launches += l;
    if (e != cudaSuccess) { set_error("table_init", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
}
int density_b200_table_fold(uint32_t* d_acc, const uint32_t* d_next, void* stream) {
    uint64_t l = 0;
    cudaError_t e = cham_table_fold(d_acc, d_next, reinterpret_cast<cudaStream_t>(stream), &l);
    g_launches += l;
    if (e != cudaSuccess) { set_error("table_fold", e); return DENSITY_B200_ECUDA; }
    return DENSITY_B200_OK;
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
        c.ws.release(); c.stage_in.release(); c.stage_out.release(); c.dec_tables.release(); for (int a2 = 0; a2 < 2; ++a2) for (int rg = 0; rg < 3; ++rg) c.chee_tables[a2][rg].release();
        c.chee_epoch = 0;
        if (c.d_size) cudaFree(c.d_size);
        if (c.h_size) cudaFreeHost(c.h_size);
        if (c.stream) cudaStreamDestroy(c.stream);
        if (c.ws_free) { cudaEventDestroy(c.ws_free); c.ws_free = nullptr; c.ws_free_recorded = false; }
        if (c.h2d_stream) cudaStreamDestroy(c.h2d_stream);
        if (c.d2h_stream) cudaStreamDestroy(c.d2h_stream);
        if (c.h_sizes) cudaFreeHost(c.h_sizes);
        c.h2d_stream = c.d2h_stream = nullptr; c.h_sizes = nullptr; c.pipe_tables.release();
        c.ring_in.release(); c.ring_out.release();
        for (auto& set : c.ev) for (auto& e : set) if (e) { cudaEventDestroy(e); e = nullptr; }
        c.d_size = nullptr; c.h_size = nullptr; c.stream = nullptr; c.ready = false;
    }
    if (cur >= 0) cudaSetDevice(cur);
}

/* diagnostic: the context iteration of the last parallel Cheetah decode on the current device (synchronises):
   out4 = {rounds used, settled (0 = the in-order kernel had to take over), run walks after round 0 (of rounds x runs), round budget} */
int density_b200_cheetah_decode_rounds(uint32_t* out4) {
    DeviceCtx* c = current_ctx();
    if (!c || !c->last_cl_status || !out4) return DENSITY_B200_EARG;
    std::lock_guard<std::mutex> lk(c->mu);
    unsigned int raw[8] = {0};
    if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpy(raw, c->last_cl_status, sizeof raw, cudaMemcpyDeviceToHost) != cudaSuccess) return DENSITY_B200_ECUDA;
    out4[0] = raw[3]; out4[1] = raw[2] && !raw[5]; out4[2] = raw[6]; out4[3] = chee_shard_max_rounds();   // cl_decode.cu MAX_ROUNDS
    return DENSITY_B200_OK;
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
