// A loopback collective library for the tests: the nine NCCL entry points the sharded drivers of libdensity_b200.so resolve
// (api.cu, NcclApi), serving W ranks that live in ONE process on ONE device, one host thread per rank. Installed with
// density_b200_test_set_nccl_library, it lets every sharded driver run at W > 1 on a single GPU.
//
//   all-gather   a rendezvous of all ranks of the comm. The arriving rank first compares (op, count, datatype) with the ranks already
//                there; the last one to arrive enqueues every copy (each rank's send slot into every rank's receive buffer, in place or
//                not) on its own stream and then releases the others, so no rank can enqueue a write over its send slot before the
//                copies are queued.
//   send / recv  grouped between GroupStart and GroupEnd, matched per (src, dst) pair in FIFO order at GroupEnd. The receiver
//                enqueues the copy; the sender waits until all its sends have been taken.
//
// Copies are cuMemcpyDtoDAsync_v2 on the caller's stream, through dlopen("libcuda.so.1"): the file needs no CUDA headers and builds
// with g++ -shared -fPIC. Nothing on the device ever waits for the host, so a driver that issues its collectives in the wrong order can
// at worst make the host waits below time out. Every host wait is bounded (60 s, loopback_set_timeout_ms); a mismatch or a timeout
// poisons the comm, after which every rank's call returns the error at once, and ncclGetErrorString gives the message of the calling
// thread's last failure (the operation, the counts, the ranks that had arrived).
//
// Test-only exports: loopback_set_host_copy (plain memcpy: the CPU test needs no device), loopback_set_timeout_ms, and a per-rank call
// log {op, count, datatype, peer} (loopback_log_read / loopback_log_clear).
#include <dlfcn.h>

#include <chrono>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <deque>
#include <map>
#include <mutex>
#include <string>
#include <vector>

namespace {

enum { OK = 0, UNHANDLED_CUDA = 1, INTERNAL = 3, INVALID_ARGUMENT = 4, INVALID_USAGE = 5 };
enum { OP_ALLGATHER = 1, OP_SEND = 2, OP_RECV = 3 };
constexpr int MAX_RANKS = 64;

// bytes of one element of an ncclDataType_t; 0 for an unknown type
size_t elem_bytes(int t) {
    switch (t) {
        case 0: case 1: return 1;           // int8, uint8
        case 6: case 9: return 2;           // float16, bfloat16
        case 2: case 3: case 7: return 4;   // int32, uint32, float32
        case 4: case 5: case 8: return 8;   // int64, uint64, float64
        default: return 0;
    }
}

// ---- copies -----------------------------------------------------------------------------------------------------------------------
bool g_host_copy = false;
long g_timeout_ms = 60000;
typedef int (*memcpy_dtod_async_t)(unsigned long long, unsigned long long, size_t, void*);
memcpy_dtod_async_t dtod() {
    static memcpy_dtod_async_t f = [] {
        void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_LOCAL);
        return h ? reinterpret_cast<memcpy_dtod_async_t>(dlsym(h, "cuMemcpyDtoDAsync_v2")) : nullptr;
    }();
    return f;
}
// dst <- src, n bytes, on `stream`; false when the copy could not be enqueued
bool copy(void* dst, const void* src, size_t n, void* stream) {
    if (!n || dst == src) return true;
    if (g_host_copy) { memmove(dst, src, n); return true; }
    memcpy_dtod_async_t f = dtod();
    return f && f(reinterpret_cast<unsigned long long>(dst), reinterpret_cast<unsigned long long>(src), n, stream) == 0;
}

// ---- the per-rank call log and the calling thread's last error ----------------------------------------------------------------------
struct LogEntry { int64_t op, count, datatype, peer; };
std::mutex g_log_mu;
std::vector<LogEntry> g_log[MAX_RANKS];
void log_call(int rank, int op, size_t count, int datatype, int peer) {
    std::lock_guard<std::mutex> lk(g_log_mu);
    g_log[rank].push_back(LogEntry{op, (int64_t)count, datatype, peer});
}
thread_local std::string t_error;
int fail(int rc, const std::string& msg) { t_error = msg; return rc; }

// ---- communicators ------------------------------------------------------------------------------------------------------------------
struct Pending { const void* buf; size_t bytes; bool taken; bool ok; };
struct Comm {
    std::string key;
    int nranks = 0, joined = 0, alive = 0;
    std::mutex mu;
    std::condition_variable cv;
    int poisoned = OK;                       // the error every later call on the comm returns
    std::string poison_msg;
    // the all-gather in progress
    uint64_t gen = 0;
    int arrived = 0;
    size_t ag_count[MAX_RANKS] = {};
    int ag_type[MAX_RANKS] = {};
    const void* ag_send[MAX_RANKS] = {};
    void* ag_recv[MAX_RANKS] = {};
    bool ag_here[MAX_RANKS] = {};
    // grouped sends waiting for their receiver, per (src, dst)
    std::map<std::pair<int, int>, std::deque<Pending*>> sends;
};
struct RankComm { Comm* c; int rank; };

std::mutex g_comms_mu;
std::map<std::string, Comm*> g_comms;

std::chrono::steady_clock::time_point deadline() { return std::chrono::steady_clock::now() + std::chrono::milliseconds(g_timeout_ms); }

// the comm's error as this thread's error (c->mu held)
int poisoned_rc(Comm* c) { t_error = c->poison_msg; return c->poisoned; }
int poison(Comm* c, int rc, const std::string& msg) {       // c->mu held
    if (!c->poisoned) { c->poisoned = rc; c->poison_msg = msg; }
    c->cv.notify_all();
    return poisoned_rc(c);
}
std::string arrived_list(Comm* c) {
    std::string s;
    for (int r = 0; r < c->nranks; ++r) {
        if (!c->ag_here[r]) continue;
        char b[64];
        snprintf(b, sizeof b, "%s%d (count %zu, type %d)", s.empty() ? "" : ", ", r, c->ag_count[r], c->ag_type[r]);
        s += b;
    }
    return s.empty() ? "none" : s;
}

// ---- grouped send / recv of the calling thread --------------------------------------------------------------------------------------
struct P2p { int op; RankComm* rc; const void* sbuf; void* rbuf; size_t bytes; int peer; void* stream; };
thread_local int t_group_depth = 0;
thread_local std::vector<P2p> t_group;

// take this rank's sends that no receiver has taken out of the queues (c->mu held): they point into run_p2p's frame
void withdraw(Comm* c, const std::vector<Pending>& mine) {
    for (auto& kv : c->sends) {
        auto& q = kv.second;
        for (auto it = q.begin(); it != q.end();) {
            bool own = false;
            for (const Pending& p : mine) own |= *it == &p;
            it = own ? q.erase(it) : it + 1;
        }
    }
}

int run_p2p(const std::vector<P2p>& ops) {
    if (ops.empty()) return OK;
    Comm* c = ops[0].rc->c;
    const int me = ops[0].rc->rank;
    for (const P2p& p : ops) if (p.rc->c != c) return fail(INVALID_USAGE, "loopback: one group spans two communicators");
    std::unique_lock<std::mutex> lk(c->mu);
    if (c->poisoned) return poisoned_rc(c);
    // post the sends
    std::vector<Pending> mine(ops.size());
    size_t nsend = 0;
    for (size_t i = 0; i < ops.size(); ++i) {
        if (ops[i].op != OP_SEND) continue;
        mine[i] = Pending{ops[i].sbuf, ops[i].bytes, false, false};
        c->sends[{me, ops[i].peer}].push_back(&mine[i]);
        ++nsend;
    }
    c->cv.notify_all();
    // take the receives in posting order
    const auto until = deadline();
    for (const P2p& p : ops) {
        if (p.op != OP_RECV) continue;
        auto& q = c->sends[{p.peer, me}];
        if (!c->cv.wait_until(lk, until, [&] { return c->poisoned || !q.empty(); })) {
            char b[256];
            snprintf(b, sizeof b, "loopback: unmatched recv: rank %d waited %ld ms for a send of %zu bytes from rank %d", me, g_timeout_ms,
                     p.bytes, p.peer);
            return poison(c, INTERNAL, b);
        }
        if (c->poisoned) return poisoned_rc(c);
        Pending* s = q.front();
        q.pop_front();
        if (s->bytes != p.bytes) {
            char b[256];
            snprintf(b, sizeof b, "loopback: send / recv size mismatch: rank %d sends %zu bytes, rank %d receives %zu", p.peer, s->bytes, me, p.bytes);
            s->taken = true;
            return poison(c, INVALID_USAGE, b);
        }
        s->ok = copy(p.rbuf, s->buf, p.bytes, p.stream);
        s->taken = true;
        c->cv.notify_all();
        if (!s->ok) return poison(c, UNHANDLED_CUDA, "loopback: cuMemcpyDtoDAsync failed (recv)");
    }
    // wait until every send of this rank has been taken
    auto all_taken = [&] {
        for (size_t i = 0; i < ops.size(); ++i) if (ops[i].op == OP_SEND && !mine[i].taken) return false;
        return true;
    };
    if (nsend && !c->cv.wait_until(lk, until, [&] { return c->poisoned || all_taken(); })) {
        std::string m = "loopback: unmatched send: rank " + std::to_string(me) + " waited " + std::to_string(g_timeout_ms) + " ms for";
        for (size_t i = 0; i < ops.size(); ++i)
            if (ops[i].op == OP_SEND && !mine[i].taken) m += " rank " + std::to_string(ops[i].peer) + " (" + std::to_string(ops[i].bytes) + " bytes)";
        withdraw(c, mine);
        return poison(c, INTERNAL, m);
    }
    if (c->poisoned) { withdraw(c, mine); return poisoned_rc(c); }
    return OK;
}

}  // namespace

extern "C" {

struct ncclUniqueId { char internal[128]; };

int ncclGetUniqueId(ncclUniqueId* id) {
    static std::mutex mu;
    static uint64_t next = 0;
    if (!id) return fail(INVALID_ARGUMENT, "loopback: ncclGetUniqueId(NULL)");
    std::lock_guard<std::mutex> lk(mu);
    memset(id->internal, 0, sizeof id->internal);
    snprintf(id->internal, sizeof id->internal, "loopback-%llu", (unsigned long long)++next);
    return OK;
}

int ncclCommInitRank(void** comm, int nranks, ncclUniqueId id, int rank) {
    if (!comm || nranks < 1 || nranks > MAX_RANKS || rank < 0 || rank >= nranks)
        return fail(INVALID_ARGUMENT, "loopback: ncclCommInitRank: bad comm pointer, nranks or rank");
    const std::string key(id.internal, strnlen(id.internal, sizeof id.internal));
    Comm* c;
    {
        std::lock_guard<std::mutex> lk(g_comms_mu);
        auto it = g_comms.find(key);
        if (it == g_comms.end()) { c = new Comm(); c->key = key; c->nranks = nranks; g_comms[key] = c; }
        else c = it->second;
    }
    std::unique_lock<std::mutex> lk(c->mu);
    if (c->nranks != nranks) return poison(c, INVALID_USAGE, "loopback: ncclCommInitRank: ranks disagree on nranks");
    ++c->joined; ++c->alive;
    c->cv.notify_all();
    if (!c->cv.wait_until(lk, deadline(), [&] { return c->poisoned || c->joined >= c->nranks; })) {
        char b[160];
        snprintf(b, sizeof b, "loopback: ncclCommInitRank: %d of %d ranks joined within %ld ms", c->joined, c->nranks, g_timeout_ms);
        --c->alive;
        return poison(c, INTERNAL, b);
    }
    if (c->poisoned) { --c->alive; return poisoned_rc(c); }
    *comm = new RankComm{c, rank};
    return OK;
}

int ncclCommDestroy(void* comm) {
    if (!comm) return OK;
    RankComm* rc = static_cast<RankComm*>(comm);
    Comm* c = rc->c;
    bool last;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        last = --c->alive == 0;
    }
    delete rc;
    if (last) {
        std::lock_guard<std::mutex> lk(g_comms_mu);
        g_comms.erase(c->key);
        delete c;
    }
    return OK;
}

int ncclAllGather(const void* sendbuff, void* recvbuff, size_t count, int datatype, void* comm, void* stream) {
    if (!comm) return fail(INVALID_ARGUMENT, "loopback: ncclAllGather: NULL comm");
    RankComm* rc = static_cast<RankComm*>(comm);
    Comm* c = rc->c;
    const int me = rc->rank;
    log_call(me, OP_ALLGATHER, count, datatype, -1);
    std::unique_lock<std::mutex> lk(c->mu);
    if (c->poisoned) return poisoned_rc(c);
    // compare with the ranks already here
    for (int r = 0; r < c->nranks; ++r) {
        if (!c->ag_here[r] || (c->ag_count[r] == count && c->ag_type[r] == datatype)) continue;
        char b[160];
        snprintf(b, sizeof b, "loopback: ncclAllGather mismatch: rank %d arrives with count %zu, type %d; arrived: ", me, count, datatype);
        return poison(c, INVALID_USAGE, b + arrived_list(c));
    }
    c->ag_here[me] = true; c->ag_count[me] = count; c->ag_type[me] = datatype;
    c->ag_send[me] = sendbuff; c->ag_recv[me] = recvbuff;
    const uint64_t my_gen = c->gen;
    if (++c->arrived < c->nranks) {
        if (!c->cv.wait_until(lk, deadline(), [&] { return c->poisoned || c->gen != my_gen; })) {
            char b[200];
            snprintf(b, sizeof b, "loopback: ncclAllGather timed out after %ld ms at rank %d (count %zu, type %d); arrived: ", g_timeout_ms, me,
                     count, datatype);
            return poison(c, INTERNAL, b + arrived_list(c));
        }
        return c->poisoned ? poisoned_rc(c) : OK;
    }
    // the last rank: every send slot into every receive buffer, then release the others. In place, rank s's send slot is slot s of
    // its own receive buffer, which no copy writes (the copy onto itself is skipped), so the order of the copies does not matter.
    const size_t bytes = count * elem_bytes(datatype);
    bool ok = elem_bytes(datatype) != 0;
    for (int d = 0; d < c->nranks && ok; ++d)
        for (int s = 0; s < c->nranks && ok; ++s)
            ok = copy(static_cast<uint8_t*>(c->ag_recv[d]) + (size_t)s * bytes, c->ag_send[s], bytes, stream);
    for (int r = 0; r < c->nranks; ++r) c->ag_here[r] = false;
    c->arrived = 0;
    ++c->gen;
    if (!ok) return poison(c, UNHANDLED_CUDA, "loopback: ncclAllGather: a copy could not be enqueued (or an unknown datatype)");
    c->cv.notify_all();
    return OK;
}

int ncclSend(const void* sendbuff, size_t count, int datatype, int peer, void* comm, void* stream) {
    if (!comm) return fail(INVALID_ARGUMENT, "loopback: ncclSend: NULL comm");
    RankComm* rc = static_cast<RankComm*>(comm);
    if (peer < 0 || peer >= rc->c->nranks || !elem_bytes(datatype)) return fail(INVALID_ARGUMENT, "loopback: ncclSend: bad peer or datatype");
    log_call(rc->rank, OP_SEND, count, datatype, peer);
    P2p p{OP_SEND, rc, sendbuff, nullptr, count * elem_bytes(datatype), peer, stream};
    if (t_group_depth) { t_group.push_back(p); return OK; }
    return run_p2p({p});
}

int ncclRecv(void* recvbuff, size_t count, int datatype, int peer, void* comm, void* stream) {
    if (!comm) return fail(INVALID_ARGUMENT, "loopback: ncclRecv: NULL comm");
    RankComm* rc = static_cast<RankComm*>(comm);
    if (peer < 0 || peer >= rc->c->nranks || !elem_bytes(datatype)) return fail(INVALID_ARGUMENT, "loopback: ncclRecv: bad peer or datatype");
    log_call(rc->rank, OP_RECV, count, datatype, peer);
    P2p p{OP_RECV, rc, nullptr, recvbuff, count * elem_bytes(datatype), peer, stream};
    if (t_group_depth) { t_group.push_back(p); return OK; }
    return run_p2p({p});
}

int ncclGroupStart() { ++t_group_depth; return OK; }

int ncclGroupEnd() {
    if (t_group_depth == 0) return fail(INVALID_USAGE, "loopback: ncclGroupEnd without ncclGroupStart");
    if (--t_group_depth) return OK;
    std::vector<P2p> ops;
    ops.swap(t_group);
    return run_p2p(ops);
}

const char* ncclGetErrorString(int rc) {
    if (!t_error.empty()) return t_error.c_str();
    switch (rc) {
        case OK: return "no error";
        case INTERNAL: return "loopback: internal error";
        case INVALID_ARGUMENT: return "loopback: invalid argument";
        case INVALID_USAGE: return "loopback: invalid usage";
        default: return "loopback: error";
    }
}

// ---- test-only exports ----------------------------------------------------------------------------------------------------------------
void loopback_set_host_copy(int on) { g_host_copy = on != 0; }
void loopback_set_timeout_ms(long ms) { g_timeout_ms = ms > 0 ? ms : 60000; }
// the call log of `rank`: up to max_entries entries of 4 int64 {op (1 all-gather, 2 send, 3 recv), count, datatype, peer (-1)} to out;
// returns the number of entries logged
int loopback_log_read(int rank, int64_t* out, int max_entries) {
    if (rank < 0 || rank >= MAX_RANKS) return -1;
    std::lock_guard<std::mutex> lk(g_log_mu);
    const std::vector<LogEntry>& v = g_log[rank];
    for (int i = 0; i < (int)v.size() && i < max_entries; ++i) {
        out[4 * i] = v[i].op; out[4 * i + 1] = v[i].count; out[4 * i + 2] = v[i].datatype; out[4 * i + 3] = v[i].peer;
    }
    return (int)v.size();
}
void loopback_log_clear() {
    std::lock_guard<std::mutex> lk(g_log_mu);
    for (auto& v : g_log) v.clear();
}

}  // extern "C"
