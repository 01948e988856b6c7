// kb_core.cu -- context lifecycle, buffer pools, profiling hooks and the NCCL revision-cursor exchange of
// libkbb200.so (the snapshot itself is kb_store.cu).
#include <dlfcn.h>
#include <stdarg.h>

#include <algorithm>
#include <atomic>

#include "kb_internal.cuh"

// ------------------------------------------------------------------------------------------------
// errors / buffers
// ------------------------------------------------------------------------------------------------
// Every failure is recorded twice: in the context (the last failure of any thread) and in the failing thread's slot.
// kb_last_error answers from the thread's slot while no kb_last_error has returned that failure, so threads that share a
// context without a lock of their own each read their own message.  Once it has been returned, or when the thread has
// none, the answer is the context's last failure: a caller that holds its own lock across the call and the read (the Go
// binding, whose goroutine may read on another thread than the one that failed) reads the failure it just made.
namespace {
struct ThreadErr {
    uint64_t serial = 0, seq = 0;
    std::string msg;
};
thread_local ThreadErr t_err;
thread_local std::string t_err_out;  // what kb_last_error returned last on this thread
std::atomic<uint64_t> g_ctx_serial{0};
constexpr size_t KB_ERR_UNREAD_MAX = 256;  // past this many unread failures the oldest reads as the context's last
}  // namespace

int kb_fail(kb_ctx *ctx, int code, const char *fmt, ...)
{
    if (ctx) {
        char buf[512];
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(buf, sizeof(buf), fmt, ap);
        va_end(ap);
        std::lock_guard<std::mutex> g(ctx->err_mu);
        std::vector<uint64_t> &u = ctx->err_unread;
        if (t_err.serial == ctx->serial) u.erase(std::remove(u.begin(), u.end(), t_err.seq), u.end());  // overwritten
        if (u.size() >= KB_ERR_UNREAD_MAX) u.erase(u.begin());
        u.push_back(++ctx->err_seq);
        t_err.serial = ctx->serial;
        t_err.seq = ctx->err_seq;
        t_err.msg = buf;
        ctx->err = buf;
    }
    return code;
}

int kb_cuda_fail(kb_ctx *ctx, cudaError_t e, const char *what)
{
    return kb_fail(ctx, e == cudaErrorMemoryAllocation ? KB_ENOMEM : KB_ECUDA, "CUDA error %d (%s) at %s", (int)e,
                   cudaGetErrorString(e), what);
}

int dbuf_ensure(kb_ctx *ctx, DBuf &b, size_t bytes)
{
    if (bytes <= b.cap && b.p) return KB_OK;
    size_t want = std::max(bytes + bytes / 4, (size_t)4096);
    want = (want + 255) & ~(size_t)255;
    if (b.p) {
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->lane().stream));
        if (ctx->stream_g) KB_CUDA(ctx, cudaStreamSynchronize(ctx->stream_g));
        cudaFree(b.p);
        b.p = nullptr;
        b.cap = 0;
    }
    KB_CUDA(ctx, cudaMalloc(&b.p, want));
    b.cap = want;
    return KB_OK;
}

int hbuf_ensure(kb_ctx *ctx, HBuf &b, size_t bytes)
{
    if (bytes <= b.cap && b.p) return KB_OK;
    size_t want = std::max(bytes + bytes / 4, (size_t)4096);
    if (b.p) {
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->lane().stream));
        if (ctx->stream_g) KB_CUDA(ctx, cudaStreamSynchronize(ctx->stream_g));
        cudaFreeHost(b.p);
        b.p = nullptr;
        b.cap = 0;
    }
    KB_CUDA(ctx, cudaHostAlloc(&b.p, want, cudaHostAllocDefault));
    b.cap = want;
    return KB_OK;
}

int hostpub_ensure(kb_ctx *ctx, HostPub &pub, size_t bytes, cudaStream_t drain_stream)
{
    if (pub.p && pub.cap >= bytes) return KB_OK;
    if (pub.p) {
        KB_CUDA(ctx, cudaStreamSynchronize(drain_stream));
        hostpub_free(pub);
    }
    const size_t cap = bytes + bytes / 2;
    KB_CUDA(ctx, cudaHostAlloc((void **)&pub.p, cap, cudaHostAllocMapped));
    memset(pub.p, 0, cap);
    pub.cap = cap;
    pub.epoch = 0;
    return KB_OK;
}

int hostpub_wait(kb_ctx *ctx, const HostPub &pub, uint64_t epoch, cudaStream_t stream, const char *what, bool count_spins)
{
    volatile const uint64_t *flag = (volatile const uint64_t *)pub.p;
    for (uint64_t spins = 1;; spins++) {
        if (*flag == epoch) {
            if (count_spins && ctx->prof_on) ctx->prof[prof_index(ctx, "host:search_wait_spins")].launches += spins;
            return KB_OK;
        }
        kb_cpu_relax();
        if ((spins & 0xFFFF) == 0) {
            const cudaError_t q = cudaStreamQuery(stream);
            if (q == cudaSuccess) return *flag == epoch ? KB_OK : kb_fail(ctx, KB_ECUDA, "%s: results were not published", what);
            if (q != cudaErrorNotReady) return kb_cuda_fail(ctx, q, what);
        }
    }
}

void hostpub_free(HostPub &pub)
{
    if (pub.p) cudaFreeHost(pub.p);
    pub = HostPub();
}

template <typename B>
static bool pool_take(std::vector<B> &pool, size_t bytes, B *out)
{
    int best = -1;
    for (int i = 0; i < (int)pool.size(); i++)
        if (pool[i].cap >= bytes && (best < 0 || pool[i].cap < pool[best].cap)) best = i;
    if (best < 0) return false;
    *out = pool[best];
    pool.erase(pool.begin() + best);
    return true;
}

int pool_get_dev(kb_ctx *ctx, size_t bytes, DBuf *out)
{
    if (bytes == 0) bytes = 16;
    if (pool_take(ctx->free_dev, bytes, out)) return KB_OK;
    DBuf b;
    KB_TRY(dbuf_ensure(ctx, b, bytes));
    *out = b;
    return KB_OK;
}

int pool_get_host(kb_ctx *ctx, size_t bytes, HBuf *out)
{
    if (bytes == 0) bytes = 16;
    if (pool_take(ctx->free_host, bytes, out)) return KB_OK;
    HBuf b;
    KB_TRY(hbuf_ensure(ctx, b, bytes));
    *out = b;
    return KB_OK;
}

int pool_get_arena(kb_ctx *ctx, size_t bytes, DBuf *out, bool get)
{
    if (bytes == 0) bytes = 16;
    if (pool_take(get ? ctx->free_get_arena : ctx->free_arena, bytes, out)) return KB_OK;
    DBuf b;
    KB_TRY(dbuf_ensure(ctx, b, bytes));
    *out = b;
    return KB_OK;
}

void pool_put_arena(kb_ctx *ctx, DBuf b, bool get)
{
    if (!b.p) return;
    std::vector<DBuf> &pool = get ? ctx->free_get_arena : ctx->free_arena;
    if (pool.size() >= 8) {
        cudaFree(b.p);  // implicit device synchronisation: nothing can still be writing it
        return;
    }
    pool.push_back(b);
}

int ctx_quiesce(kb_ctx *ctx)
{
    // submitted range batches: their kernels are done once their rows are back; point-read batches publish after their copy
    KB_TRY(kb_pending_harvest_all(ctx));
    if (ctx->stream_g) KB_CUDA(ctx, cudaStreamSynchronize(ctx->stream_g));
    if (ctx->stream2) KB_CUDA(ctx, cudaStreamSynchronize(ctx->stream2));  // a prefetched bound search may still read the slabs
    return KB_OK;
}

void pool_put_dev(kb_ctx *ctx, DBuf b)
{
    if (!b.p) return;
    if (ctx->free_dev.size() >= 16) {
        cudaFree(b.p);
        return;
    }
    ctx->free_dev.push_back(b);
}

void pool_put_host(kb_ctx *ctx, HBuf b)
{
    if (!b.p) return;
    if (ctx->free_host.size() >= 16) {
        cudaFreeHost(b.p);
        return;
    }
    ctx->free_host.push_back(b);
}

// ------------------------------------------------------------------------------------------------
// profiling
// ------------------------------------------------------------------------------------------------
int prof_index(kb_ctx *ctx, const char *name)
{
    for (int i = 0; i < (int)ctx->prof.size(); i++)
        if (ctx->prof[i].name == name) return i;
    ProfEntry e;
    e.name = name;
    ctx->prof.push_back(e);
    return (int)ctx->prof.size() - 1;
}

int ev_take(kb_ctx *ctx, cudaEvent_t *ev)
{
    *ev = nullptr;
    if (!ctx->ev_pool.empty()) {
        *ev = ctx->ev_pool.back();
        ctx->ev_pool.pop_back();
        return KB_OK;
    }
    cudaEvent_t e;
    KB_CUDA(ctx, cudaEventCreate(&e));
    *ev = e;
    return KB_OK;
}

void prof_begin(kb_ctx *ctx, int idx, uint64_t alg_bytes, cudaStream_t strm)
{
    ProfPending p{idx, nullptr, nullptr};
    // without both events the launch is counted but not timed
    if (ev_take(ctx, &p.a) == KB_OK && ev_take(ctx, &p.b) == KB_OK) cudaEventRecord(p.a, strm);
    ctx->prof_pending.push_back(p);
    ctx->prof[idx].launches++;
    ctx->prof[idx].bytes += alg_bytes;
}

void prof_end(kb_ctx *ctx, cudaStream_t strm)
{
    if (cudaEvent_t b = ctx->prof_pending.back().b) cudaEventRecord(b, strm);
}

static void prof_resolve(kb_ctx *ctx)
{
    if (ctx->prof_pending.empty()) return;
    cudaStreamSynchronize(ctx->lane().stream);
    if (ctx->stream_g) cudaStreamSynchronize(ctx->stream_g);
    for (auto &p : ctx->prof_pending) {
        float ms = 0;
        if (p.b && cudaEventElapsedTime(&ms, p.a, p.b) == cudaSuccess) ctx->prof[p.idx].ms += ms;
        for (cudaEvent_t e : {p.a, p.b})
            if (e) ctx->ev_pool.push_back(e);
    }
    ctx->prof_pending.clear();
}

extern "C" int kb_prof_enable(kb_ctx *ctx, int on)
{
    if (!ctx) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!on) prof_resolve(ctx);
    ctx->prof_on = on;
    return KB_OK;
}

extern "C" int kb_prof_reset(kb_ctx *ctx)
{
    if (!ctx) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    prof_resolve(ctx);
    ctx->prof.clear();
    return KB_OK;
}

extern "C" int kb_prof_read(kb_ctx *ctx, kb_prof_entry *entries, int cap, int *n)
{
    if (!ctx || !n) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    prof_resolve(ctx);
    int k = 0;
    for (auto &e : ctx->prof) {
        if (k < cap && entries) {
            memset(&entries[k], 0, sizeof(kb_prof_entry));
            strncpy(entries[k].name, e.name.c_str(), sizeof(entries[k].name) - 1);
            entries[k].launches = e.launches;
            entries[k].total_ms = e.ms;
            entries[k].alg_bytes = e.bytes;
        }
        k++;
    }
    *n = k;
    return KB_OK;
}

extern "C" uint64_t kb_launch_count(kb_ctx *ctx)
{
    if (!ctx) return 0;
    std::lock_guard<std::mutex> g(ctx->mu);
    return ctx->launches;
}

// ------------------------------------------------------------------------------------------------
// lifecycle
// ------------------------------------------------------------------------------------------------
extern "C" int kb_abi_version(void) { return KB_ABI_VERSION; }

extern "C" int kb_open(int device_ordinal, const kb_config *cfg, kb_ctx **out)
{
    if (!out) return KB_EINVAL;
    const uint32_t flags = cfg && cfg->struct_size >= sizeof(kb_config) ? cfg->flags : 0u;
    const bool high = flags & KB_CFG_HIGH_PRIORITY;
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev <= 0 || device_ordinal < 0 || device_ordinal >= ndev) {
        // no CPU fallback: the product path refuses to run without a CUDA device
        return KB_ECUDA;
    }
    kb_ctx *ctx = new kb_ctx();
    ctx->serial = ++g_ctx_serial;
    ctx->device = device_ordinal;
    ctx->host_values = flags & KB_CFG_HOST_VALUES;
    int prio_lo = 0, prio_hi = 0, prio_lane = 0, sms = 0;
    if (cudaSetDevice(device_ordinal) != cudaSuccess ||
        cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi) != cudaSuccess)
        prio_lo = prio_hi = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device_ordinal) != cudaSuccess || sms < 1) {
        delete ctx;
        return KB_ECUDA;
    }
    ctx->n_sms = (uint32_t)sms;
    // three levels when the device has them (numerically lower = more urgent): bound search > lane streams (short kernels of a
    // batch) > bulk kernels (gather / wire copy, by their stream)
    static const bool split = !(getenv("KB_PRIO_SPLIT") && atoi(getenv("KB_PRIO_SPLIT")) == 0);
    prio_lane = (split && prio_lo - prio_hi >= 2) ? prio_lo - 1 : prio_lo;
    if (
        cudaStreamCreateWithPriority(&ctx->lanes[0].stream, cudaStreamNonBlocking, high ? prio_hi : prio_lane) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->lanes[0].ev_jobs, cudaEventDisableTiming) != cudaSuccess ||
        // the bound search is tiny and the host waits for it: always ahead of everything; the copy stream (gather / wire
        // copy) is throughput work that the next batch's short kernels should not queue behind: always behind
        cudaStreamCreateWithPriority(&ctx->stream2, cudaStreamNonBlocking, prio_hi) != cudaSuccess ||
        cudaStreamCreateWithPriority(&ctx->stream_g, cudaStreamNonBlocking, prio_lo) != cudaSuccess ||
        // the stream of the device -> host answer copies
        cudaStreamCreateWithPriority(&ctx->stream_h, cudaStreamNonBlocking, prio_lo) != cudaSuccess ||
        // work counters of every lane + the error flag: zeroed once, before any stream can touch them
        cudaMalloc(&ctx->d_ctrs.p, 1024) != cudaSuccess || cudaMemset(ctx->d_ctrs.p, 0, 1024) != cudaSuccess ||
        cudaDeviceSynchronize() != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->jobsets[0].ev_gather, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->jobsets[1].ev_gather, cudaEventDisableTiming) != cudaSuccess) {
        delete ctx;
        return KB_ECUDA;
    }
    ctx->d_ctrs.cap = 1024;
    // the done counters of the bound searches that publish: d_ctrs[16 + slot], prefetch slots 0 and 1, lane i at slot 2 + i
    for (int i = 0; i < 2; i++) ctx->prefetch[i].search.pub_ctr = 16 + i;
    for (int i = 0; i < KB_MAX_LANES; i++) ctx->lanes[i].search.pub_ctr = 18 + i;
    // lanes of range batches (kb_range_submit): KB_LANES batches in flight at most; the streams of lanes 1.. are created
    // when a submission first moves onto them
    ctx->n_lanes = getenv("KB_LANES") ? std::min(std::max(atoi(getenv("KB_LANES")), 1), KB_MAX_LANES) : 3;
    ctx->prio_lane = high ? prio_hi : prio_lane;
    *out = ctx;
    return KB_OK;
}

// move the context to the next lane, round robin (the enqueued work of the batches in flight holds raw pointers)
void lane_swap(kb_ctx *ctx)
{
    const int next = (ctx->cur_lane + 1) % ctx->n_lanes;
    ScanLane &a = ctx->lanes[next];
    if (!a.stream) {  // first use of this lane (a context that never submits ahead -- the watch context -- uses lane 0 only)
        if (cudaStreamCreateWithPriority(&a.stream, cudaStreamNonBlocking, ctx->prio_lane) != cudaSuccess ||
            cudaEventCreateWithFlags(&a.ev_jobs, cudaEventDisableTiming) != cudaSuccess) {
            if (a.stream) cudaStreamDestroy(a.stream);
            a.stream = nullptr;
            cudaGetLastError();
            return;  // stay on the current lane: the next submission first reads this lane's rows back
        }
    }
    ctx->cur_lane = next;
}

static void dfree(DBuf &b)
{
    if (b.p) cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
}

static void search_free(BoundSearch &s)
{
    dfree(s.d_bounds);
    dfree(s.d_bres);
    hostpub_free(s.pub);
}

// every buffer, the event and the stream of a lane whose work has finished
static void lane_free(ScanLane &L)
{
    for (DBuf *b : {&L.d_reqs, &L.d_meta, &L.d_tgt, &L.d_tcnt, &L.d_tscan, &L.d_reqout, &L.d_sel, &L.d_slot, &L.d_get}) dfree(*b);
    search_free(L.search);
    hostpub_free(L.rows);
    for (void *h : {L.h_stage.p, L.h_stage2.p})
        if (h) cudaFreeHost(h);
    if (L.ev_jobs) cudaEventDestroy(L.ev_jobs);
    if (L.stream) cudaStreamDestroy(L.stream);
}

extern "C" void kb_close(kb_ctx *ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    kb_pending_drop_all(ctx);
    for (ScanLane &L : ctx->lanes)
        if (L.stream) cudaStreamSynchronize(L.stream);
    if (ctx->stream_g) cudaStreamSynchronize(ctx->stream_g);
    if (ctx->stream2) cudaStreamSynchronize(ctx->stream2);
    if (ctx->stream_h) cudaStreamSynchronize(ctx->stream_h);
    kb_stream_drop_all(ctx);
    watch_tables_free(ctx);
    vheap_free(ctx, ctx->d_vslab);  // while the streams it synchronises still exist
    for (ScanLane &L : ctx->lanes) lane_free(L);
    if (ctx->stream_h) cudaStreamDestroy(ctx->stream_h);
    for (DBuf *b : {&ctx->d_kslab, &ctx->d_flags, &ctx->d_cursor, &ctx->d_ctrs}) dfree(*b);
    for (JobSet &j : ctx->jobsets) {
        dfree(j.jobs);
        dfree(j.gjobs);
        if (j.ev_gather) cudaEventDestroy(j.ev_gather);
    }
    for (DirSet *d : {&ctx->live, &ctx->spare}) d->each([](DBuf &b, size_t) { dfree(b); });
    for (auto &b : ctx->free_dev) cudaFree(b.p);
    for (auto &b : ctx->free_host) cudaFreeHost(b.p);
    for (auto &p : ctx->prof_pending) {
        cudaEventDestroy(p.a);
        cudaEventDestroy(p.b);
    }
    for (auto e : ctx->ev_pool) cudaEventDestroy(e);
    for (size_t r = 0; r < ctx->p2p_peer.size(); r++)
        if (ctx->p2p_peer[r] && ctx->p2p_peer[r] != ctx->p2p_mine) cudaIpcCloseMemHandle(ctx->p2p_peer[r]);
    if (ctx->p2p_mine) cudaFree(ctx->p2p_mine);
    if (ctx->d_p2p_ptrs.p) cudaFree(ctx->d_p2p_ptrs.p);
    if (ctx->h_p2p_out) cudaFreeHost(ctx->h_p2p_out);
    if (ctx->nccl_comm) {
        void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        if (h) {
            typedef int (*destroy_t)(void *);
            destroy_t f = (destroy_t)dlsym(h, "ncclCommDestroy");
            if (f) f(ctx->nccl_comm);
        }
    }
    hostpub_free(ctx->wpub);
    hostpub_free(ctx->ppub);
    for (auto &b : ctx->free_arena) cudaFree(b.p);
    for (auto &b : ctx->free_get_arena) cudaFree(b.p);
    for (auto &sl : ctx->prefetch) {
        if (sl.stage.p) cudaFreeHost(sl.stage.p);
        search_free(sl.search);
    }
    if (ctx->stream_g) cudaStreamDestroy(ctx->stream_g);
    if (ctx->stream2) cudaStreamDestroy(ctx->stream2);
    delete ctx;
}

extern "C" const char *kb_last_error(kb_ctx *ctx)
{
    if (!ctx) return "no context";
    std::lock_guard<std::mutex> g(ctx->err_mu);
    std::vector<uint64_t> &u = ctx->err_unread;
    auto it = t_err.serial == ctx->serial ? std::find(u.begin(), u.end(), t_err.seq) : u.end();
    if (it != u.end()) {
        t_err_out = t_err.msg;
    } else {
        t_err_out = ctx->err;
        it = std::find(u.begin(), u.end(), ctx->err_seq);
    }
    if (it != u.end()) u.erase(it);
    return t_err_out.c_str();
}

extern "C" void *kb_stream(kb_ctx *ctx)
{
    if (!ctx) return nullptr;
    std::lock_guard<std::mutex> g(ctx->mu);  // the current lane moves with every range submission
    return (void *)ctx->lane().stream;
}

extern "C" int kb_sync(kb_ctx *ctx)
{
    if (!ctx) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    for (ScanLane &L : ctx->lanes)
        if (L.stream) KB_CUDA(ctx, cudaStreamSynchronize(L.stream));
    if (ctx->stream_g) KB_CUDA(ctx, cudaStreamSynchronize(ctx->stream_g));
    if (ctx->stream_h) KB_CUDA(ctx, cudaStreamSynchronize(ctx->stream_h));
    if (ctx->stream2) KB_CUDA(ctx, cudaStreamSynchronize(ctx->stream2));  // the delivery lists of the last watch match
    return KB_OK;
}

// ------------------------------------------------------------------------------------------------
// NCCL revision cursor (one ncclAllGather of one uint64 per rank; min over ranks on the device)
// ------------------------------------------------------------------------------------------------
struct IdBlob {
    char internal[KB_NCCL_ID_BYTES];
};

namespace {
struct NcclApi {
    void *h = nullptr;
    int (*GetUniqueId)(void *) = nullptr;
    int (*CommInitRank)(void **, int, /* ncclUniqueId by value */ IdBlob, int) = nullptr;
    int (*AllGather)(const void *, void *, size_t, int, void *, cudaStream_t) = nullptr;
    int (*CommDestroy)(void *) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
};
}  // namespace

static NcclApi *nccl_api()
{
    static NcclApi api;
    static bool tried = false;
    if (tried) return api.h ? &api : nullptr;
    tried = true;
    // reuse the copy already mapped into the process (torch bundles one) before falling back to the system lib
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return nullptr;
    api.GetUniqueId = (int (*)(void *))dlsym(h, "ncclGetUniqueId");
    api.CommInitRank = (int (*)(void **, int, IdBlob, int))dlsym(h, "ncclCommInitRank");
    api.AllGather = (int (*)(const void *, void *, size_t, int, void *, cudaStream_t))dlsym(h, "ncclAllGather");
    api.CommDestroy = (int (*)(void *))dlsym(h, "ncclCommDestroy");
    api.GetErrorString = (const char *(*)(int))dlsym(h, "ncclGetErrorString");
    if (!api.GetUniqueId || !api.CommInitRank || !api.AllGather) return nullptr;
    api.h = h;
    return &api;
}

extern "C" int kb_nccl_unique_id(uint8_t id[KB_NCCL_ID_BYTES])
{
    NcclApi *a = nccl_api();
    if (!a) return KB_ENCCL;
    IdBlob b;
    memset(&b, 0, sizeof(b));
    if (a->GetUniqueId(&b) != 0) return KB_ENCCL;
    memcpy(id, &b, KB_NCCL_ID_BYTES);
    return KB_OK;
}

// ---- peer-memory cursor exchange ------------------------------------------------------------------------------
// The one collective of the path moves 8 bytes per rank; ncclAllGather spends tens of microseconds of launch and
// protocol latency on it.  Here every rank owns a small slot buffer that all peers map (cudaIpc over NVLink / NVSwitch): a rank stores
// its cursor and then an epoch flag straight into every peer's buffer and spins on its own buffer until all flags
// of the epoch have arrived.  Two slot sets alternate by epoch parity: a rank can be at most one exchange ahead of
// the slowest peer (it needs that peer's flag to finish), so it never overwrites a set that is still being read.
constexpr int KB_P2P_MAX_RANKS = 1024;

__global__ void __launch_bounds__(KB_P2P_MAX_RANKS)
k_cursor_p2p(uint64_t *const *__restrict__ peers, int me, int n, uint64_t epoch, uint64_t local, uint64_t *out)
{
    __shared__ unsigned long long smin;
    __shared__ int failed;
    const int r = threadIdx.x;
    if (r == 0) {
        smin = ~0ull;
        failed = 0;
    }
    __syncthreads();
    const size_t set = (size_t)(epoch & 1) * n * 2;
    if (r < n) {
        volatile uint64_t *p = peers[r] + set + (size_t)me * 2;
        p[0] = local;
        __threadfence_system();
        p[1] = epoch;
        volatile uint64_t *mine = peers[me] + set + (size_t)r * 2;
        const long long t0 = clock64();
        bool ok = true;
        while (mine[1] < epoch) {  // a peer that is AHEAD (this rank skipped an exchange) also releases the wait
            if (clock64() - t0 > 8000000000ll) {  // ~4 s: a peer never joined this exchange
                ok = false;
                break;
            }
        }
        __threadfence_system();
        const uint64_t v = mine[0];
        out[r] = v;
        if (ok) atomicMin(&smin, (unsigned long long)v);
        else atomicExch(&failed, 1);
    }
    __syncthreads();
    if (r < n) __threadfence_system();  // the gathered values reach the mapped host buffer before the status word
    __syncthreads();
    if (r == 0) {
        out[n] = smin;
        __threadfence_system();
        *(volatile uint64_t *)&out[n + 1] = failed ? 2 : 1;  // status: 1 done, 2 timed out
    }
}

static void p2p_setup(kb_ctx *ctx, NcclApi *a)
{
    const int n = ctx->nccl_nranks, me = ctx->nccl_rank;
    if (n > KB_P2P_MAX_RANKS) return;
    const size_t slot_bytes = (size_t)2 * n * 2 * 8;
    void *mine = nullptr, *d_handles = nullptr;
    std::vector<cudaIpcMemHandle_t> handles(n);
    std::vector<void *> peer(n, nullptr);
    bool ok = cudaMalloc(&mine, slot_bytes) == cudaSuccess && cudaMemset(mine, 0, slot_bytes) == cudaSuccess &&
              cudaMalloc(&d_handles, (size_t)(n + 1) * sizeof(cudaIpcMemHandle_t) + 64) == cudaSuccess;
    cudaIpcMemHandle_t my_h;
    memset(&my_h, 0, sizeof(my_h));
    // a rank that cannot export its buffer still takes part in the handle all-gather (it is collective) and sends zeros
    const bool exported = ok && cudaIpcGetMemHandle(&my_h, mine) == cudaSuccess;
    if (d_handles) {
        uint8_t *dh = (uint8_t *)d_handles;
        cudaMemcpyAsync(dh, &my_h, sizeof(my_h), cudaMemcpyHostToDevice, ctx->lane().stream);
        int rc = a->AllGather(dh, dh + sizeof(my_h), sizeof(my_h), /*ncclUint8*/ 1, ctx->nccl_comm, ctx->lane().stream);
        if (rc != 0) ok = false;
        cudaMemcpyAsync(handles.data(), dh + sizeof(my_h), (size_t)n * sizeof(my_h), cudaMemcpyDeviceToHost, ctx->lane().stream);
        if (cudaStreamSynchronize(ctx->lane().stream) != cudaSuccess) ok = false;
    }
    ok = ok && exported;
    static const cudaIpcMemHandle_t zero_h = {};
    for (int r = 0; ok && r < n; r++) {
        if (memcmp(&handles[r], &zero_h, sizeof(zero_h)) == 0) {
            ok = false;  // that peer could not export
        } else if (r == me) {
            peer[r] = mine;
        } else if (cudaIpcOpenMemHandle(&peer[r], handles[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
            peer[r] = nullptr;
            ok = false;
        }
    }
    if (ok) ok = dbuf_ensure(ctx, ctx->d_p2p_ptrs, (size_t)n * sizeof(void *)) == KB_OK &&
                 cudaMemcpy(ctx->d_p2p_ptrs.p, peer.data(), (size_t)n * sizeof(void *), cudaMemcpyHostToDevice) == cudaSuccess &&
                 cudaHostAlloc((void **)&ctx->h_p2p_out, (size_t)(n + 2) * 8, cudaHostAllocMapped) == cudaSuccess;
    // all ranks must take the same path: agree on the outcome (one more tiny all-gather, still collective on failure)
    if (d_handles) {
        uint8_t *dh = (uint8_t *)d_handles;
        const uint8_t mine_ok = ok ? 1 : 0;
        std::vector<uint8_t> all_ok(n, 0);
        cudaMemcpyAsync(dh, &mine_ok, 1, cudaMemcpyHostToDevice, ctx->lane().stream);
        int rc = a->AllGather(dh, dh + 16, 1, /*ncclUint8*/ 1, ctx->nccl_comm, ctx->lane().stream);
        cudaMemcpyAsync(all_ok.data(), dh + 16, (size_t)n, cudaMemcpyDeviceToHost, ctx->lane().stream);
        if (rc != 0 || cudaStreamSynchronize(ctx->lane().stream) != cudaSuccess) ok = false;
        for (int r = 0; r < n; r++) ok = ok && all_ok[r] == 1;
        cudaFree(d_handles);
    } else {
        ok = false;
    }
    cudaGetLastError();  // a failed IPC call must not poison later error checks
    if (!ok) {
        for (int r = 0; r < n; r++)
            if (peer[r] && peer[r] != mine) cudaIpcCloseMemHandle(peer[r]);
        if (mine) cudaFree(mine);
        return;
    }
    ctx->p2p_mine = mine;
    ctx->p2p_peer = peer;
    ctx->p2p_epoch = 0;
    ctx->p2p_ready = true;
}

extern "C" int kb_nccl_init(kb_ctx *ctx, const uint8_t id[KB_NCCL_ID_BYTES], int rank, int nranks)
{
    if (!ctx || !id || rank < 0 || rank >= nranks) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    NcclApi *a = nccl_api();
    if (!a) return kb_fail(ctx, KB_ENCCL, "libnccl.so.2 not loadable");
    cudaSetDevice(ctx->device);
    IdBlob b;
    memcpy(&b, id, KB_NCCL_ID_BYTES);
    int rc = a->CommInitRank(&ctx->nccl_comm, nranks, b, rank);
    if (rc != 0) return kb_fail(ctx, KB_ENCCL, "ncclCommInitRank: %s", a->GetErrorString ? a->GetErrorString(rc) : "?");
    ctx->nccl_rank = rank;
    ctx->nccl_nranks = nranks;
    if (nranks > 1) p2p_setup(ctx, a);  // best effort: without it the cursor exchange stays on ncclAllGather
    return KB_OK;
}

extern "C" int kb_cursor_transport(kb_ctx *ctx)
{
    if (!ctx) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->nccl_comm) return KB_CURSOR_NONE;
    if (ctx->nccl_nranks == 1) return KB_CURSOR_SINGLE;
    return ctx->p2p_ready && !ctx->cursor_force_nccl ? KB_CURSOR_P2P : KB_CURSOR_NCCL;
}

extern "C" int kb_cursor_force_nccl(kb_ctx *ctx, int on)
{
    if (!ctx) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    ctx->cursor_force_nccl = on != 0;
    return KB_OK;
}

__global__ void k_cursor_min(const uint64_t *all, int n, uint64_t *out)
{
    uint64_t m = ~0ull;
    for (int i = 0; i < n; i++) m = all[i] < m ? all[i] : m;
    *out = m;
}

extern "C" int kb_cursor_allgather(kb_ctx *ctx, uint64_t local_rev, uint64_t *all_revs, uint64_t *min_rev)
{
    if (!ctx) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->nccl_comm) return kb_fail(ctx, KB_ESTATE, "kb_nccl_init has not been called");
    NcclApi *a = nccl_api();
    cudaSetDevice(ctx->device);
    int n = ctx->nccl_nranks;
    if (n == 1) {
        // a single shard has nobody to exchange with: the readable revision is its own cursor
        if (all_revs) all_revs[0] = local_rev;
        if (min_rev) *min_rev = local_rev;
        return KB_OK;
    }
    if (ctx->p2p_ready && !ctx->cursor_force_nccl) {
        const uint64_t epoch = ++ctx->p2p_epoch;
        volatile uint64_t *out = ctx->h_p2p_out;
        out[n + 1] = 0;
        const int threads = ((n + 31) / 32) * 32;
        KB_LAUNCH(ctx, "k_cursor_p2p", (uint64_t)n * 16,
                  (k_cursor_p2p<<<1, threads, 0, ctx->lane().stream>>>((uint64_t *const *)ctx->d_p2p_ptrs.p, ctx->nccl_rank, n, epoch,
                                                              local_rev, ctx->h_p2p_out)));
        // the kernel's last store is the status word in mapped pinned memory: polling it is a few microseconds cheaper
        // than a stream synchronisation; a launch failure or a hung device still ends in the synchronise below
        const auto t0 = std::chrono::steady_clock::now();
        for (uint64_t spins = 1; out[n + 1] == 0; spins++) {
            kb_cpu_relax();
            if ((spins & 0xFFFF) == 0 && std::chrono::steady_clock::now() - t0 > std::chrono::seconds(6)) break;
        }
        if (out[n + 1] == 0) KB_CUDA(ctx, cudaStreamSynchronize(ctx->lane().stream));
        if (out[n + 1] != 1) {
            // A peer never joined.  This rank leaves the peer-memory path for good: the late peer still finds this rank's
            // flag for the epoch it missed, then times out on the next one and falls back too, so the ranks meet again in
            // ncclAllGather instead of waiting 4 s on every exchange from here on.
            ctx->p2p_ready = false;
            return kb_fail(ctx, KB_ENCCL, "cursor exchange: a peer did not join epoch %llu (falling back to ncclAllGather)",
                           (unsigned long long)epoch);
        }
        if (all_revs)
            for (int r = 0; r < n; r++) all_revs[r] = out[r];
        if (min_rev) *min_rev = out[n];
        return KB_OK;
    }
    KB_TRY(dbuf_ensure(ctx, ctx->d_cursor, (size_t)(n + 2) * 8));
    uint64_t *d = (uint64_t *)ctx->d_cursor.p;  // [0]=local, [1..n]=gathered, [n+1]=min
    KB_TRY(lane_take(ctx));  // the staging below may still hold a submitted range batch's request table
    ScanLane &L = ctx->lane();
    KB_TRY(hbuf_ensure(ctx, L.h_stage2, 64));
    *(uint64_t *)L.h_stage2.p = local_rev;
    KB_CUDA(ctx, cudaMemcpyAsync(d, L.h_stage2.p, 8, cudaMemcpyHostToDevice, L.stream));
    int rc = a->AllGather(d, d + 1, 1, /*ncclUint64*/ 5, ctx->nccl_comm, L.stream);
    if (rc != 0) return kb_fail(ctx, KB_ENCCL, "ncclAllGather: %s", a->GetErrorString ? a->GetErrorString(rc) : "?");
    KB_LAUNCH(ctx, "cursor_min", (uint64_t)n * 8, (k_cursor_min<<<1, 1, 0, L.stream>>>(d + 1, n, d + 1 + n)));
    std::vector<uint64_t> host(n + 1);
    KB_CUDA(ctx, cudaMemcpyAsync(host.data(), d + 1, (size_t)(n + 1) * 8, cudaMemcpyDeviceToHost, L.stream));
    KB_CUDA(ctx, cudaStreamSynchronize(L.stream));
    if (all_revs) memcpy(all_revs, host.data(), (size_t)n * 8);
    if (min_rev) *min_rev = host[n];
    return KB_OK;
}
