// hb_dist.cu — one-process-per-GPU plumbing for the row-sharded local_laplacian.
//
// The reference has no distributed layer at all (SURVEY.md §2b "Collectives: none"); row-sharding is new work
// (SURVEY.md §8e).  Ranks are laid out top to bottom over the frame's rows.  A sharded call communicates twice
// (DESIGN.md §7): one exchange of input halo rows with the two row neighbours and one all-to-all gather of a coarse
// pyramid level — each ONE ncclGroup of ncclSend / ncclRecv on the compute stream (`exchange`).  The bands of all ranks
// are gathered once per geometry with `allgather_bytes`.
//
// NCCL is bound at run time (dlopen "libnccl.so.2") so the library has no link-time dependency and
// shares the NCCL instance torch already loaded when the host process is the Python bench/test.
// Bootstrap: rank 0 calls halide_b200_dist_unique_id, the 128-byte id travels over the host's own
// control plane (torch.distributed broadcast in halide_b200/dist.py), every rank calls
// halide_b200_dist_init.
//
// halide_b200_dist_init_loopback binds the calling host thread instead to one rank of an in-process group whose
// ranks are threads sharing one device: every line of the sharded path and its kernels then runs on a single GPU
// (tests/test_dist_loopback_gpu.py).  The binding is thread-local and checked before the NCCL communicator.
#include <dlfcn.h>
#include <nccl.h>
#include <string.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <vector>

#include "hb_common.h"
#include "hb_dist.h"

namespace {

struct NcclApi {
    void *handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
};
NcclApi g_nccl;
ncclComm_t g_comm = nullptr;
int g_rank = 0, g_size = 1;

int load_nccl() {
    if (g_nccl.handle) return 0;
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return hb::fail(halide_error_code_generic_error, "dist: cannot load libnccl.so.2: %s", dlerror());
#define HB_SYM(field, name)                                                                             \
    g_nccl.field = reinterpret_cast<decltype(g_nccl.field)>(dlsym(h, name));                            \
    if (!g_nccl.field) return hb::fail(halide_error_code_generic_error, "dist: libnccl lacks %s", name);
    HB_SYM(GetUniqueId, "ncclGetUniqueId")
    HB_SYM(CommInitRank, "ncclCommInitRank")
    HB_SYM(CommDestroy, "ncclCommDestroy")
    HB_SYM(Send, "ncclSend")
    HB_SYM(Recv, "ncclRecv")
    HB_SYM(AllGather, "ncclAllGather")
    HB_SYM(GroupStart, "ncclGroupStart")
    HB_SYM(GroupEnd, "ncclGroupEnd")
    HB_SYM(GetErrorString, "ncclGetErrorString")
#undef HB_SYM
    g_nccl.handle = h;
    return 0;
}

int check(ncclResult_t r, const char *what) {
    if (r == ncclSuccess) return 0;
    return hb::fail(halide_error_code_generic_error, "dist: %s failed: %s", what,
                    g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
}

// ---- in-process loopback group ---------------------------------------------------------------------------------
// A send records an event on the sender's stream and queues (pointer, bytes, event) for its (sender, receiver) pair; the
// receiver orders its stream after that event and copies.  The device only ever waits on events already recorded, so
// a rank that stops early can stall host threads (each host wait is bounded by kLoopbackWaitS) but never the GPU.
constexpr int kLoopbackWaitS = 20;

struct LoopbackSend {
    const void *ptr = nullptr;
    size_t bytes = 0;
    cudaEvent_t ready = nullptr, done = nullptr;  // recorded by the sender after its data / by the receiver after its copy
    bool copied = false;                          // done has been recorded
    ~LoopbackSend() {
        if (ready) cudaEventDestroy(ready);
        if (done) cudaEventDestroy(done);
    }
};

struct Loopback {
    std::mutex mu;
    std::condition_variable cv;
    int size = 0, members = 0;
    std::vector<char> joined;
    std::map<std::pair<int, int>, std::deque<std::shared_ptr<LoopbackSend>>> fifo;  // (sender, receiver)
    bool failed = false;  // a host wait expired: every later wait in the group fails at once
    // allgather_bytes: ranks deposit their blob, then all read; the next round starts once every rank has read
    std::vector<char> blobs, arrived;
    size_t blob_bytes = 0;
    int n_arrived = 0, n_read = 0;
    bool reading = false;

    void reset(int nranks) {
        size = nranks;
        joined.assign(nranks, 0);
        arrived.assign(nranks, 0);
        fifo.clear();
        blobs.clear();
        failed = reading = false;
        n_arrived = n_read = 0;
    }
};
Loopback &loopback() {
    static Loopback *g = new Loopback;  // intentionally leaked: queued sends destroy CUDA events
    return *g;
}
thread_local int t_lb_rank = -1;  // the calling thread's rank in the loopback group, -1: not bound
thread_local int t_lb_epoch = 0;
int g_epoch = 0;                   // NCCL communicator
std::atomic<int> g_epochs{0};

// Bounded wait for ready() under lk.  On expiry the group is marked failed (its other ranks stop waiting too) and the
// error names the waiting rank and the rank it waited for (peer < 0: the first rank missing from the all-gather).
// Errors are reported after lk is released.
template<typename Pred>
int loopback_wait(std::unique_lock<std::mutex> &lk, Pred ready, int peer, const char *what) {
    Loopback &g = loopback();
    const bool woke = g.cv.wait_for(lk, std::chrono::seconds(kLoopbackWaitS), [&] { return g.failed || ready(); });
    if (woke && ready()) return 0;
    const bool expired = !woke;
    if (peer < 0) {
        peer = 0;
        while (peer < g.size - 1 && g.arrived[peer]) peer++;
    }
    g.failed = true;
    g.cv.notify_all();
    lk.unlock();
    if (expired) {
        return hb::fail(halide_error_code_generic_error, "dist loopback: rank %d waited %d s for rank %d (%s)", t_lb_rank,
                        kLoopbackWaitS, peer, what);
    }
    return hb::fail(halide_error_code_generic_error, "dist loopback: rank %d stopped waiting for rank %d (%s): the group failed",
                    t_lb_rank, peer, what);
}

int loopback_exchange(const hbdist::Msg *msgs, int n, cudaStream_t s) {
    Loopback &g = loopback();
    const int me = t_lb_rank;
    std::vector<std::shared_ptr<LoopbackSend>> sent;
    for (int i = 0; i < n; i++) {  // sends first (NCCL posts a group's sends and receives together)
        const hbdist::Msg &m = msgs[i];
        if (m.bytes == 0 || !m.send) continue;
        auto e = std::make_shared<LoopbackSend>();
        e->ptr = m.ptr;
        e->bytes = m.bytes;
        if (cudaEventCreateWithFlags(&e->ready, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&e->done, cudaEventDisableTiming) != cudaSuccess || cudaEventRecord(e->ready, s) != cudaSuccess) {
            return hb::fail(halide_error_code_generic_error, "dist loopback: event set-up failed: %s", cudaGetErrorString(cudaGetLastError()));
        }
        std::lock_guard<std::mutex> lock(g.mu);
        g.fifo[{me, m.peer}].push_back(e);
        g.cv.notify_all();
        sent.push_back(e);
    }
    for (int i = 0; i < n; i++) {
        const hbdist::Msg &m = msgs[i];
        if (m.bytes == 0 || m.send) continue;
        std::shared_ptr<LoopbackSend> e;
        {
            std::unique_lock<std::mutex> lk(g.mu);
            auto &q = g.fifo[{m.peer, me}];
            int r = loopback_wait(lk, [&] { return !q.empty(); }, m.peer, "its send");
            if (r) return r;
            e = q.front();
            q.pop_front();
        }
        if (e->bytes != m.bytes) {
            {
                std::lock_guard<std::mutex> lock(g.mu);
                g.failed = true;
                g.cv.notify_all();
            }
            return hb::fail(halide_error_code_generic_error, "dist loopback: rank %d expects %zu bytes from rank %d, which sent %zu",
                            me, m.bytes, m.peer, e->bytes);
        }
        cudaStreamWaitEvent(s, e->ready, 0);
        cudaMemcpyAsync(m.ptr, e->ptr, m.bytes, cudaMemcpyDeviceToDevice, s);
        cudaEventRecord(e->done, s);
        std::lock_guard<std::mutex> lock(g.mu);
        e->copied = true;
        g.cv.notify_all();
    }
    // NCCL's group completion: the sender's later work on s (reuse of the sent buffer included) follows the peer's copy
    for (size_t i = 0, k = 0; i < (size_t)n && k < sent.size(); i++) {
        if (msgs[i].bytes == 0 || !msgs[i].send) continue;
        const std::shared_ptr<LoopbackSend> &e = sent[k++];
        {
            std::unique_lock<std::mutex> lk(g.mu);
            int r = loopback_wait(lk, [&] { return e->copied; }, msgs[i].peer, "its receive");
            if (r) return r;
        }
        cudaStreamWaitEvent(s, e->done, 0);
    }
    return 0;
}

int loopback_allgather(const void *send, void *recv_all, size_t bytes) {
    Loopback &g = loopback();
    const int me = t_lb_rank;
    std::unique_lock<std::mutex> lk(g.mu);
    int r = loopback_wait(lk, [&] { return !g.reading; }, me, "the previous all-gather to be read");
    if (r) return r;
    if (g.n_arrived == 0) {
        g.blob_bytes = bytes;
        g.blobs.assign(bytes * g.size, 0);
    } else if (bytes != g.blob_bytes) {
        g.failed = true;
        g.cv.notify_all();
        lk.unlock();
        return hb::fail(halide_error_code_generic_error, "dist loopback: rank %d all-gathers %zu bytes, other ranks %zu", me, bytes,
                        g.blob_bytes);
    }
    memcpy(&g.blobs[bytes * me], send, bytes);
    g.arrived[me] = 1;
    if (++g.n_arrived == g.size) {
        g.reading = true;
        g.cv.notify_all();
    } else {
        if ((r = loopback_wait(lk, [&] { return g.reading; }, -1, "the all-gather"))) return r;
    }
    memcpy(recv_all, g.blobs.data(), bytes * g.size);
    if (++g.n_read == g.size) {
        g.n_arrived = g.n_read = 0;
        g.arrived.assign(g.size, 0);
        g.reading = false;
        g.cv.notify_all();
    }
    return 0;
}

}  // namespace

namespace hbdist {

// a 1-rank communicator is legal (timing the sharded path without neighbours)
bool active() { return t_lb_rank >= 0 || g_comm != nullptr; }
int rank() { return t_lb_rank >= 0 ? t_lb_rank : g_rank; }
int size() { return t_lb_rank >= 0 ? loopback().size : g_size; }
int epoch() { return t_lb_rank >= 0 ? t_lb_epoch : g_epoch; }

int exchange(const Msg *msgs, int n, cudaStream_t s) {
    if (t_lb_rank >= 0) return loopback_exchange(msgs, n, s);
    if (!active()) return hb::fail(halide_error_code_generic_error, "dist: halo exchange without an initialised communicator");
    int r;
    if ((r = check(g_nccl.GroupStart(), "ncclGroupStart"))) return r;
    for (int i = 0; i < n; i++) {
        const Msg &m = msgs[i];
        if (m.bytes == 0) continue;
        if (m.send) r = check(g_nccl.Send(m.ptr, m.bytes, ncclInt8, m.peer, g_comm, s), "ncclSend");
        else r = check(g_nccl.Recv(m.ptr, m.bytes, ncclInt8, m.peer, g_comm, s), "ncclRecv");
        if (r) {
            g_nccl.GroupEnd();
            return r;
        }
    }
    return check(g_nccl.GroupEnd(), "ncclGroupEnd");
}

int allgather_bytes(const void *send, void *recv_all, size_t bytes) {
    if (t_lb_rank >= 0) return loopback_allgather(send, recv_all, bytes);
    if (!active()) return hb::fail(halide_error_code_generic_error, "dist: all-gather without an initialised communicator");
    void *dsend = nullptr, *drecv = nullptr;
    cudaStream_t s = hb::stream();
    if (cudaMalloc(&dsend, bytes) != cudaSuccess || cudaMalloc(&drecv, bytes * g_size) != cudaSuccess) {
        cudaGetLastError();
        return hb::fail(halide_error_code_device_malloc_failed, "dist: all-gather staging allocation failed");
    }
    cudaMemcpyAsync(dsend, send, bytes, cudaMemcpyHostToDevice, s);
    int r = check(g_nccl.AllGather(dsend, drecv, bytes, ncclInt8, g_comm, s), "ncclAllGather");
    if (!r) {
        cudaMemcpyAsync(recv_all, drecv, bytes * g_size, cudaMemcpyDeviceToHost, s);
        if (cudaStreamSynchronize(s) != cudaSuccess) r = hb::fail(halide_error_code_generic_error, "dist: all-gather failed");
    }
    cudaFree(dsend);
    cudaFree(drecv);
    return r;
}

}  // namespace hbdist

extern "C" {

int halide_b200_dist_unique_id(char *out128) {
    int r = load_nccl();
    if (r) return r;
    ncclUniqueId id;
    if ((r = check(g_nccl.GetUniqueId(&id), "ncclGetUniqueId"))) return r;
    memcpy(out128, id.internal, NCCL_UNIQUE_ID_BYTES);
    return 0;
}

int halide_b200_dist_init(int rank, int nranks, const char *id128) {
    int r = load_nccl();
    if (r) return r;
    if (g_comm) return hb::fail(halide_error_code_generic_error, "dist: already initialised");
    ncclUniqueId id;
    memcpy(id.internal, id128, NCCL_UNIQUE_ID_BYTES);
    if ((r = check(g_nccl.CommInitRank(&g_comm, nranks, id, rank), "ncclCommInitRank"))) return r;
    g_rank = rank;
    g_epoch = ++g_epochs;
    g_size = nranks;
    return 0;
}

int halide_b200_dist_init_loopback(int rank, int nranks) {
    if (nranks < 1 || rank < 0 || rank >= nranks) {
        return hb::fail(halide_error_code_generic_error, "dist loopback: rank %d of %d ranks", rank, nranks);
    }
    if (t_lb_rank >= 0) return hb::fail(halide_error_code_generic_error, "dist loopback: this thread is already rank %d", t_lb_rank);
    Loopback &g = loopback();
    int group_size;
    {
        std::lock_guard<std::mutex> lock(g.mu);
        if (g.members == 0) g.reset(nranks);
        if (g.size == nranks && !g.joined[rank]) {
            g.joined[rank] = 1;
            g.members++;
            t_lb_rank = rank;
            t_lb_epoch = ++g_epochs;
            return 0;
        }
        group_size = g.size;
    }
    return hb::fail(halide_error_code_generic_error, "dist loopback: cannot join as rank %d of %d (the group has %d ranks)", rank,
                    nranks, group_size);
}

int halide_b200_dist_shutdown(void) {
    if (t_lb_rank >= 0) {
        Loopback &g = loopback();
        std::lock_guard<std::mutex> lock(g.mu);
        g.joined[t_lb_rank] = 0;
        if (--g.members == 0) g.reset(0);
        t_lb_rank = -1;
        return 0;
    }
    if (g_comm) {
        cudaDeviceSynchronize();
        g_nccl.CommDestroy(g_comm);
        g_comm = nullptr;
    }
    g_rank = 0;
    g_size = 1;
    return 0;
}

int halide_b200_dist_rank(void) { return hbdist::rank(); }
int halide_b200_dist_size(void) { return hbdist::size(); }

}  // extern "C"
