// kb_internal.cuh -- shared host/device plumbing of libkbb200.so (sm_90a only, no CPU fallback).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <chrono>
#include <initializer_list>
#include <map>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/kb_b200.h"

// ------------------------------------------------------------------------------------------------
// HBM layouts (DESIGN.md section 3)
// ------------------------------------------------------------------------------------------------
struct StoreDev {
    const uint4    *kslab;   // internal keys, every record starts on a 16-byte boundary, zero padded
    const uint32_t *koff16;  // n+1 offsets in 16-byte units
    const uint16_t *klen;    // n exact key lengths
    const uint4    *vslab;   // values, 16-byte aligned, zero padded
    const uint64_t *voff16;  // n+1 offsets in 16-byte units
    const uint32_t *vlen;    // n exact value lengths
    const uint64_t *srev;    // n scan-summary revisions (kb_store.cu summarize_record)
    const uint32_t *sword;   // n scan-summary words: LCP with record i - 1 | static flags (KB_M_DEC_OK, KB_M_REV0, KB_S_*)
    uint32_t        n;
};

// The bound slab: a batch of n keys laid out the way k_search finds their lower bounds in the directory (kb_search.cu),
// in pinned staging and then on the device -- [each key zero padded to 16 bytes, then KB_BOUND_READAHEAD16 zero chunks
// | off16 u32 x n | len u32 x n].  bounds_pack builds one, bound_search uploads and searches it, BoundsDev reads it.
constexpr uint64_t KB_BOUND_READAHEAD16 = 3;  // key_less loads a bound's first three chunks together, whatever its length
__host__ __device__ constexpr uint64_t bound_chunks(uint64_t len) { return (len + 15) / 16 + KB_BOUND_READAHEAD16; }

struct BoundsDev {  // no kernel writes a slab it reads: every read goes through the read-only data path (__ldg)
    const uint4 *keys;
    const uint32_t *off16, *lens;
    uint32_t n;
    __device__ __forceinline__ const uint4 *key(uint32_t w) const { return keys + __ldg(off16 + w); }
    __device__ __forceinline__ uint32_t len(uint32_t w) const { return __ldg(lens + w); }
};

// one scanner.Range / Count / Compact request, resolved to record indices
struct ReqDev {
    uint32_t lo, hi;       // record interval [lo, hi)
    uint32_t flat0;        // first slot of this request in the flat per-record scratch (multiple of TILE)
    uint32_t tile0;        // first tile of this request
    uint32_t ntiles;
    uint32_t sel_base;     // first slot of this request in the selection arrays
    uint64_t read_rev;
    int64_t  limit;
};

struct TileDev {
    uint32_t req;
    uint32_t rec0;   // first store record of the tile
    uint32_t n;      // records in the tile (<= TILE)
    uint32_t flat0;  // flat slot of rec0
    uint32_t lo;     // first record of the request (copy of ReqDev.lo: one load instead of two in the decode pass)
    uint32_t pad;
    uint64_t read_rev;
};

// The job table of an answer's copy: job_first[nreq + 1] (first kv of each request; [nreq] = the kvs) | arena_base[nreq + 1]
// (first arena byte of each request; [nreq] = the bytes) | the copy's work counter.  k_req_finalize writes a batch's; a
// one-request answer (range-stream page, point reads) has its request behind the table (jobtab_req) and is written by
// jobtab_write_one.
struct JobTable {
    uint64_t *job_first, *arena_base;
    unsigned long long *work_ctr;
    const uint64_t *n_kvs() const { return arena_base - 1; }  // job_first[nreq], right in front of arena_base
};
__host__ __device__ constexpr size_t jobtab_bytes(size_t nreq) { return (2 * (nreq + 1) + 1) * 8; }
__host__ __device__ __forceinline__ JobTable jobtab_at(void *p, size_t nreq)
{
    JobTable t;
    t.job_first = (uint64_t *)p;
    t.arena_base = t.job_first + nreq + 1;
    t.work_ctr = (unsigned long long *)(t.arena_base + nreq + 1);
    return t;
}
__host__ __device__ __forceinline__ ReqDev *jobtab_req(void *p) { return (ReqDev *)((uint8_t *)p + jobtab_bytes(1)); }

// a one-request table: kvs sel_base .. sel_base + nk - 1 of the selection, kv s placed at arena_base + slot[s]
__device__ __forceinline__ void jobtab_write_one(void *p, uint64_t nk, uint64_t arena_base, uint64_t bytes, uint32_t sel_base)
{
    const JobTable t = jobtab_at(p, 1);
    t.job_first[0] = 0;
    t.job_first[1] = nk;
    t.arena_base[0] = arena_base;
    t.arena_base[1] = bytes;
    *t.work_ctr = 0;
    ReqDev r;
    r.lo = r.hi = r.flat0 = r.tile0 = r.ntiles = 0;
    r.sel_base = sel_base;
    r.read_rev = 0;
    r.limit = 0;
    *jobtab_req(p) = r;
}

struct ScanMode {
    int      compact;      // workerConfig.compact
    int      ttl_scan;     // !SupportTTL() && timeoutRevision != 0
    uint64_t timeout_rev;
    int      wire;         // 0: padded [key][value] arena; KB_WIRE_KVS_I / KB_WIRE_EVENTS_I: etcd protobuf elements
    static ScanMode range(int wire) { return ScanMode{0, 0, 0, wire}; }
};
enum { KB_WIRE_NONE_I = 0, KB_WIRE_KVS_I = 1, KB_WIRE_EVENTS_I = 2 };

// per-record meta word produced by the decode pass
#define KB_M_LCP_MASK 0x0000FFFFu
#define KB_M_DEC_OK   (1u << 16)
#define KB_M_REV0     (1u << 17)   // revision == 0 (revision record)
#define KB_M_TRIG     (1u << 18)   // takes part as "cur": decodable, not TTL-expired, rev <= read_rev
#define KB_M_TOMB     (1u << 19)   // value == "tombstone"
#define KB_M_PREVOK   (1u << 20)   // becomes "prev" (TRIG and not the Q5 skip)
#define KB_M_REVDEL   (1u << 21)   // class 3 victim
#define KB_M_TTLREV   (1u << 22)   // class 4 victim
#define KB_M_TTLOBJ   (1u << 23)   // class 5 victim
// static bits of the scan-summary word (StoreDev::sword) besides KB_M_DEC_OK / KB_M_REV0
#define KB_S_TOMBV    KB_M_TOMB    // value == "tombstone" (the meta word keeps it only for visible records)
#define KB_S_VL9      (1u << 24)   // value is 9 bytes long
#define KB_S_VL8      (1u << 25)   // value is at least 8 bytes long
#define KB_S_EVENTS   (1u << 26)   // the user key contains "/events/"
#define KB_LCP_INF    0xFFFFu
#define KB_NONE       0xFFFFFFFFu

#define KB_TILE       1024          // records per tile (256 threads x 4)

// ------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ldg_stream(const uint4 *p)
{
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

__device__ __forceinline__ void stg_stream(uint4 *p, const uint4 &v)
{
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w)
                 : "memory");
}

// first differing byte (memory order) of two 16-byte chunks, 16 when equal
__device__ __forceinline__ int first_diff16(const uint4 &a, const uint4 &b)
{
    uint32_t x;
    x = a.x ^ b.x; if (x) return (__ffs(x) - 1) >> 3;
    x = a.y ^ b.y; if (x) return 4 + ((__ffs(x) - 1) >> 3);
    x = a.z ^ b.z; if (x) return 8 + ((__ffs(x) - 1) >> 3);
    x = a.w ^ b.w; if (x) return 12 + ((__ffs(x) - 1) >> 3);
    return 16;
}

__device__ __forceinline__ uint32_t byte_of(const uint4 &a, int i)
{
    uint32_t w = (i < 4) ? a.x : (i < 8) ? a.y : (i < 12) ? a.z : a.w;
    return (w >> ((i & 3) * 8)) & 0xffu;
}

__device__ __forceinline__ uint64_t be64_bytes(const uint8_t *p)
{
    uint64_t v = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) v = (v << 8) | (uint64_t)p[i];
    return v;
}

__device__ __forceinline__ uint32_t pad16(uint32_t x) { return (x + 15u) & ~15u; }

// every lane of a warp: do the first n bytes of the key at `a` (a record's) equal those of bound w?  32 lanes x 16 bytes
// per pass
__device__ __forceinline__ bool warp_prefix_eq(const uint4 *a, const BoundsDev &bounds, uint32_t w, uint32_t n)
{
    const uint4 *b = bounds.key(w);
    bool eq = true;
    for (uint32_t c = threadIdx.x & 31; c * 16 < n; c += 32) {
        uint4 x = a[c], y = __ldg(b + c);
        int p = first_diff16(x, y);
        if (p < 16 && c * 16 + p < n) eq = false;
    }
    return __all_sync(0xffffffffu, eq);
}

// Bounded mbarrier wait of the bulk-copy (TMA) kernels (a bulk copy that faults never completes its barrier): gives up
// after ~2 s of polling and raises the context's error flag (d_ctrs[8]) instead of hanging the stream; the results of
// that launch are then garbage.  k_wire_copy is its only user.  The flag is published as the error word of a LATER
// batch's rows or page cut (k_req_finalize / k_publish_rout / k_page_cut copy it) and is never cleared, so every range
// call that publishes after it fails.
__device__ __forceinline__ bool dmbar_wait(uint64_t *bar, uint32_t parity, unsigned int *err_flag)
{
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(bar);
    uint32_t done = 0;
    for (uint32_t spins = 0; spins < (1u << 26); spins++) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done)
            : "r"(a), "r"(parity)
            : "memory");
        if (done) return true;
    }
    atomicExch(err_flag, 1u);
    return false;
}

// Streaming copies: the bytes are read once per call, so they are the first to leave L2 (evict_first) -- the 50 MB L2
// then keeps what the latency-bound kernels running beside them re-read (directory arrays, summary and meta words, the
// fan-out's tables and scratch).
__device__ __forceinline__ uint64_t l2_evict_first_policy()
{
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}

// raise the epoch flag of a HostPub once everything the host reads with it has been stored
__device__ __forceinline__ void pub_raise(void *host, uint64_t epoch)
{
    __threadfence_system();
    *(volatile uint64_t *)host = epoch;
}

// ------------------------------------------------------------------------------------------------
// host plumbing
// ------------------------------------------------------------------------------------------------
struct DBuf {
    void  *p = nullptr;
    size_t cap = 0;
};

struct HBuf {  // pinned host
    void  *p = nullptr;
    size_t cap = 0;
};

// The value heap of the snapshot: HBM, or mapped pinned host memory when the context was opened with
// KB_CFG_HOST_VALUES.  p is what kernels read (the mapping's device pointer); host is the host address of a host heap
// (nullptr in HBM).  Only vheap_* in kb_store.cu allocate, grow, fill and free one.
struct VHeap {
    void    *p = nullptr;
    uint8_t *host = nullptr;
    size_t   cap = 0;
};

// Mapped pinned memory the device publishes results into, so that the host polls a flag instead of paying a stream /
// event synchronisation: [epoch flag u64 | error word u64 | payload].  The device stores the payload and the error word
// (0: no error), then raises the flag to the epoch of the publish (pub_raise); the host waits for it (hostpub_wait).
constexpr size_t KB_PUB_HEAD = 16;  // bytes in front of the payload
struct HostPub {
    uint8_t *p = nullptr;
    size_t cap = 0;
    uint64_t epoch = 0;  // of the last publish enqueued
    template <class T> T *payload() const { return (T *)(p + KB_PUB_HEAD); }
    uint64_t err() const { return ((volatile const uint64_t *)p)[1]; }
};

// the per-record arrays of one directory set (StoreDev's directory and scan summary), n + 1 entries each
struct DirSet {
    DBuf koff16, klen, voff16, vlen, srev, sword;
    // f(array, bytes per entry) for every array: a set is allocated, swapped and freed as a whole
    template <class F> void each(F &&f)
    {
        f(koff16, 4); f(klen, 2); f(voff16, 8); f(vlen, 4); f(srev, 8); f(sword, 4);
    }
};

struct ProfEntry {
    std::string name;
    uint64_t launches = 0;
    double   ms = 0;
    uint64_t bytes = 0;
};

struct ProfPending {
    int idx;
    cudaEvent_t a, b;
};

struct Watcher {
    std::string prefix;
    uint64_t min_rev;
    bool live;
};

struct WatchTablesDev;  // kb_watch.cu

// One bound search (k_search, kb_search.cu): the uploaded bound slab and its view, the device results, and their published
// copy (payload: results u32 x n; the error word stays zero) with its done counter d_ctrs[pub_ctr] (kb_open assigns it)
struct BoundSearch {
    DBuf d_bounds, d_bres;
    BoundsDev dev{};
    HostPub pub;
    uint32_t pub_ctr = 0;
};

// kb_range_prefetch: a bound search started ahead of the kb_range_batch that will use it
struct SearchSlot {
    HBuf stage;
    BoundSearch search;
    size_t ident_bytes = 0;
    uint64_t store_gen = 0, seq = 0;
    bool valid = false;
};

struct kb_pending;  // a submitted range batch (kb_batch.cu)

// A lane: everything a range batch owns between kb_range_submit and kb_range_collect.  kb_range_submit leaves its batch
// in flight on the current lane and moves the context to the next one (lane_swap), so that the next batch is laid out and
// launched on another stream / scratch set while the earlier ones' kernels run.  Lane i uses the work counters
// d_ctrs[64 + 16 i ..] and publishes its bound search through d_ctrs[16 + 2 + i].
// Every other entry point runs on the current lane's stream and uses its staging (h_stage, h_stage2, search, d_reqout).
// Before it may write them it waits for the lane's previous batch to publish its rows: ctx_quiesce does that for every
// lane, lane_take for the current one.
struct ScanLane {
    cudaStream_t stream = nullptr;   // created on the lane's first use (lane 0: by kb_open)
    cudaEvent_t ev_jobs = nullptr;   // end of the job construction of the lane's last batch (the copy stream waits on it)
    // the published per-request results of the lane's last batch (payload: ReqOut rows, none for a point-read batch;
    // error word: the context's error flag)
    HostPub rows;
    BoundSearch search;
    // request table (the tile table follows it, see tile_table in kb_scan.cu) and the per-batch scan scratch
    DBuf d_reqs, d_meta, d_tgt, d_tcnt /* look-back states */, d_tscan, d_reqout, d_sel, d_slot;
    // a point-read batch's copy: job table, copy jobs and the wire job kernel's per-kv scratch.  Its copy runs on the lane
    // stream, so these are free again once the batch's rows are published (they need no JobSet alternation)
    DBuf d_get;
    HBuf h_stage, h_stage2;          // pinned staging
    kb_pending *pending = nullptr;   // submitted on this lane (range or point-read batch), rows not yet read back
};
constexpr int KB_MAX_LANES = 4;

// The job buffers of a range batch's copy (gather / wire copy).  Two sets alternate between consecutive batches, so a
// batch's job construction may overlap the previous batch's copy; ev_gather marks the end of the last copy that read
// the set.
struct JobSet {
    DBuf jobs, gjobs;
    cudaEvent_t ev_gather = nullptr;
};

struct kb_ctx {
    int device = 0;
    uint32_t n_sms = 1;  // multiprocessors of `device`: caps the grid-stride launches, one fan-out CTA per SM
    ScanLane lanes[KB_MAX_LANES];
    int n_lanes = 1, cur_lane = 0;
    ScanLane &lane() { return lanes[cur_lane]; }  // the current lane
    int prio_lane = 0;                            // priority of the lane streams
    cudaStream_t stream2 = nullptr;  // bound search of a range batch: runs beside the tail (gather) of the previous batch
    // The gather / wire copy of a range batch runs on its own stream, so the next batch's decode .. placement (lane
    // stream) overlaps it.
    cudaStream_t stream_g = nullptr;
    JobSet jobsets[2];  // a range batch (or range-stream page) uses set batch_seq & 1; point reads use their lane's d_get
    uint64_t batch_seq = 0;
    cudaStream_t stream_h = nullptr;              // device -> host copies of KB_OUT_HOST answers (behind the gather's event)
    // watch match: payload [0] total deliveries, [1..5] phase spans (ns); error word: a grid barrier of k_fanout timed out
    HostPub wpub;
    HostPub ppub;  // k_partition_cut's report (kb_page.cu)
    // The last failure of any thread, its sequence number, and the sequence numbers of failures no kb_last_error has
    // returned yet (kb_core.cu).  err_mu, not mu, guards them: kb_fail also runs outside mu (kb_result_wait, refusals).
    std::string err;
    uint64_t err_seq = 0;
    std::vector<uint64_t> err_unread;
    uint64_t serial = 0;  // tags this context's failures in a thread's slot (a later context may reuse the address)
    std::mutex err_mu;
    std::mutex mu;

    // store (kb_store.cu): st points at the slabs and the live directory set; spare = the set the next merge or layout
    // compaction writes, then the two swap
    bool loaded = false;
    bool host_values = false;  // KB_CFG_HOST_VALUES: d_vslab is mapped pinned host memory (fixed at kb_open)
    StoreDev st{};
    DBuf d_kslab;
    VHeap d_vslab;
    DirSet live, spare;
    uint32_t max_kv_chunks = 0;  // largest padded [key][value] pair, in 16-byte chunks: sizes the wire copy's ring buffers
    // heap + sorted directory (kb_apply_batch): chunks in use at the slab tails, chunks no live record points at, records
    // appended out of key order since the last layout compaction
    uint64_t kused16 = 0, vused16 = 0, garbage_k16 = 0, garbage_v16 = 0, displaced = 0, layout_compactions = 0;
    // a batch changed the snapshot since the last canonical layout (both slabs contiguous in key order).  Apart from the
    // trigger's counters: a replacement of an empty value appends out of order and counts in none of them
    bool out_of_order = false;
    bool compact_present = false;
    uint64_t compact_rev = 0;
    // TTL puts: (expire_unix, internal key), ordered by time; ttl_of[key] = the expiry the key currently has (a later put
    // of the same key replaces or cancels it, a delete cancels it)
    std::multimap<uint64_t, std::string> ttl_queue;
    std::unordered_map<std::string, uint64_t> ttl_of;

    // scratch (grow only)
    DBuf d_flags, d_ctrs /* work-queue counters, kept at zero between kernels; [8] the wire copy's error flag */;

    // kb_range_prefetch: two bound searches in flight at most
    SearchSlot prefetch[2];
    uint32_t prefetch_next = 0;
    uint64_t store_gen = 0;  // bumped whenever the snapshot changes

    std::vector<kb_range_stream *> streams;  // open range streams (kb_close frees the ones nobody closed)
    std::vector<kb_compact_stream *> cstreams;  // open compaction streams (likewise)

    // buffer pools for results
    std::vector<DBuf> free_dev;
    std::vector<DBuf> free_arena;  // response arenas: only ever written by the gather stream (or after ctx_quiesce)
    // point-read arenas: written on a lane stream, complete before their result exists -- kept apart from free_arena, whose
    // buffers a range copy still running on the gather stream may be writing
    std::vector<DBuf> free_get_arena;
    std::vector<HBuf> free_host;

    // watchers
    std::vector<Watcher> watchers;
    std::vector<uint32_t> free_watch_ids;
    bool watch_dirty = true;
    WatchTablesDev *wt = nullptr;
    struct kb_events_dev *ev_scratch = nullptr;  // grow-only upload slab of kb_watch_match

    // NCCL (dlopen'ed)
    void *nccl_comm = nullptr;
    int nccl_rank = -1, nccl_nranks = 0;
    DBuf d_cursor;
    // peer-memory cursor exchange (set up by kb_nccl_init when every peer's slot buffer can be mapped over NVLink)
    bool p2p_ready = false;
    bool cursor_force_nccl = false;           // kb_cursor_force_nccl: measure / use the ncclAllGather path although peers map
    uint64_t p2p_epoch = 0;
    void *p2p_mine = nullptr;                 // this rank's slot buffer: 2 epochs x nranks x {value, flag}
    std::vector<void *> p2p_peer;             // every rank's slot buffer as seen from this device (own entry = p2p_mine)
    DBuf d_p2p_ptrs;                          // the same pointers on the device
    uint64_t *h_p2p_out = nullptr;            // pinned: [nranks] gathered cursors, [nranks] min, [nranks+1] status

    // profiling
    int prof_on = 0;  // 0 off, 1 every kernel, 2 only k_decode_lcp and k_gather
    std::vector<ProfEntry> prof;
    std::vector<ProfPending> prof_pending;
    std::vector<cudaEvent_t> ev_pool;
    uint64_t launches = 0;
    bool wire_attr_set = false;  // per-context (per-device) kernel attribute
};

// what a result answers: the kb_*_view_get that reads it, and the pool its device arena returns to
enum class ResultKind { range, compact_sweep, match, point_read, compact_page, partitions, reconcile };

// An answer and the pooled buffers it owns: per-item arrays (meta) and the arena, on the host and / or the device.  The
// device meta of a range answer and a sweep is capacity-sized; a point read's host meta holds its rows (GetRows in
// kb_batch.cu); a match's host meta always holds the offsets, its device meta offsets | delivery lists.
struct kb_result {
    ResultKind kind;
    int out_mode = 0;
    HBuf h_meta, h_arena;
    DBuf d_meta, d_arena;
    cudaEvent_t done_ev = nullptr;  // the device side is complete once this has fired (kb_result_wait, kb_sync)
    // range
    std::vector<uint64_t> req_first, req_count, req_examined;
    uint64_t n_kvs = 0, n_bytes = 0;
    const uint32_t *rec_idx = nullptr;
    const uint64_t *rev = nullptr, *key_off = nullptr, *val_off = nullptr;
    const uint32_t *key_len = nullptr, *val_len = nullptr;
    int wire = 0;                          // KB_WIRE_*_I
    const uint64_t *elem_off = nullptr;    // wire modes: n_kvs + 1 element offsets into the arena
    // compact (a compaction-stream page: its victims are [first, first + n_victims) of the sweep's list)
    uint64_t n_victims = 0, count = 0, examined = 0, vic_cap = 0, first = 0;
    // point reads
    uint64_t n_gets = 0;
    // partitions: host meta = key_off (n_parts + 2) | kv_first (n_parts + 1) | arena_first (n_parts + 1), host arena = borders
    uint64_t n_parts = 0;
    // match
    uint64_t n_watchers = 0, n_deliveries = 0;
    // reconcile: host meta = src_idx (n_diff) | key_off (n_diff + 1) | kind (n_diff bytes), host arena = the diff's keys
    uint64_t rc_n_engine = 0, rc_n_mirror = 0, rc_n_missing = 0, rc_n_extra = 0, rc_n_changed = 0, rc_n_diff = 0;
};

kb_result *kb_result_new(ResultKind kind, int out_mode);
// return every pooled buffer and the event of a result, then delete it; the caller holds ctx->mu (kb_copy.cu)
void result_release_locked(kb_ctx *ctx, kb_result *res);

// a pointer that a call hands out on success and releases with Drop when it fails part-way
template <class T, void (*Drop)(kb_ctx *, T *)> struct Held {
    kb_ctx *ctx;
    T *p;
    ~Held()
    {
        if (p) Drop(ctx, p);
    }
    T *release()
    {
        T *r = p;
        p = nullptr;
        return r;
    }
};
using HeldResult = Held<kb_result, result_release_locked>;

// one device piece of an answer's per-item arrays
struct D2HPiece {
    const void *src;
    size_t bytes;
};
// The KB_OUT_HOST copy of an answer on stream s, behind res->done_ev when it has one: the pieces land back to back in a
// new host meta (none drawn when they hold no bytes; an old one goes back to the pool), arena_bytes of the device arena in
// the host arena.  s is synchronised whether or not everything could be enqueued; the device meta and arena then go back
// to their pools.  `what` names a failed copy (kb_copy.cu).
int result_to_host(kb_ctx *ctx, kb_result *res, cudaStream_t s, std::initializer_list<D2HPiece> pieces,
                   uint64_t arena_bytes, const char *what);

int kb_fail(kb_ctx *ctx, int code, const char *fmt, ...);
// one committed batch -- kb_apply_batch without the argument checks and the lock -- and its TTL bookkeeping; the caller
// holds ctx->mu (kb_store.cu)
int write_batch_locked(kb_ctx *ctx, const kb_write_op *ops, uint64_t n_ops);
int kb_cuda_fail(kb_ctx *ctx, cudaError_t e, const char *what);

#define KB_CUDA(ctx, call)                                               \
    do {                                                                 \
        cudaError_t _e = (call);                                         \
        if (_e != cudaSuccess) return kb_cuda_fail((ctx), _e, #call);    \
    } while (0)

#define KB_TRY(expr)              \
    do {                          \
        int _rc = (expr);         \
        if (_rc != KB_OK) return _rc; \
    } while (0)

int dbuf_ensure(kb_ctx *ctx, DBuf &b, size_t bytes);
int hbuf_ensure(kb_ctx *ctx, HBuf &b, size_t bytes);
// release a value heap once no kernel can still read it (kb_store.cu)
void vheap_free(kb_ctx *ctx, VHeap &h);
int pool_get_dev(kb_ctx *ctx, size_t bytes, DBuf *out);
// get = true: the point-read pool (free_get_arena)
int pool_get_arena(kb_ctx *ctx, size_t bytes, DBuf *out, bool get = false);
void pool_put_arena(kb_ctx *ctx, DBuf b, bool get = false);
// read back the rows of every submitted range and point-read batch, then wait for the gather stream: the entry points that change the
// snapshot or read it outside the range calls start with it
int ctx_quiesce(kb_ctx *ctx);
int kb_pending_harvest_all(kb_ctx *ctx);  // kb_batch.cu
void kb_pending_drop_all(kb_ctx *ctx);
void kb_stream_drop_all(kb_ctx *ctx);  // kb_close, once every stream of the context is idle (kb_compact.cu)
// Open compaction streams address the heap by offsets (kb_compact.cu): while one that can still hand out pages is open, the
// write path leaves the heap in place (no layout compaction); load, restore and dump rewrite it and invalidate them.
bool compact_streams_pin_heap(const kb_ctx *ctx);
void compact_streams_invalidate(kb_ctx *ctx, const char *what);
// read back the rows of the current lane's previous batch, if it is still in flight: its staging is then free
int lane_take(kb_ctx *ctx);  // kb_batch.cu
void lane_swap(kb_ctx *ctx);
int pool_get_host(kb_ctx *ctx, size_t bytes, HBuf *out);
void pool_put_dev(kb_ctx *ctx, DBuf b);
void pool_put_host(kb_ctx *ctx, HBuf b);
// at least `bytes` of mapped pinned memory, zeroed with the epoch reset when it grows; an old buffer is freed once
// drain_stream (the stream that publishes into it) has finished
int hostpub_ensure(kb_ctx *ctx, HostPub &pub, size_t bytes, cudaStream_t drain_stream);
// wait until the device has raised the flag to `epoch`; `stream` (the publishing stream) is consulted now and then, so
// that a failed launch or kernel is noticed instead of spinning forever.  count_spins: add the spins to the
// host:search_wait_spins profiling counter
int hostpub_wait(kb_ctx *ctx, const HostPub &pub, uint64_t epoch, cudaStream_t stream, const char *what,
                 bool count_spins = false);
void hostpub_free(HostPub &pub);

// a bound slab packed into pinned staging (bounds_pack)
struct PackedBounds {
    const uint8_t *host = nullptr;
    uint64_t n = 0, chunks = 0;
    size_t bytes() const { return chunks * 16 + n * 8; }  // what the upload copies
};

// pack n bounds into `stage`: bound i is len(i) bytes, which put(i, dst) writes into its zeroed slot at dst
template <class Len, class Put>
int bounds_pack(kb_ctx *ctx, HBuf &stage, uint64_t n, Len &&len, Put &&put, PackedBounds *out)
{
    uint64_t chunks = 0;
    for (uint64_t i = 0; i < n; i++) chunks += bound_chunks(len(i));
    KB_TRY(hbuf_ensure(ctx, stage, chunks * 16 + n * 8 + 64));
    uint8_t *hs = (uint8_t *)stage.p;
    memset(hs, 0, chunks * 16);
    uint32_t *off16 = (uint32_t *)(hs + chunks * 16), *lens = off16 + n;
    uint64_t c = 0;
    for (uint64_t i = 0; i < n; i++) {
        const uint64_t l = len(i);
        off16[i] = (uint32_t)c;
        lens[i] = (uint32_t)l;
        put(i, hs + c * 16);
        c += bound_chunks(l);
    }
    *out = PackedBounds{hs, n, chunks};
    return KB_OK;
}

// Upload `pk` to s and run k_search on `strm` (kb_search.cu): s.d_bres gets the n lower bounds, followed by `extra_res`
// bytes the caller may use; s.dev is the uploaded slab.  publish: the results also go to s.pub, raised to ++s.pub.epoch.
int bound_search(kb_ctx *ctx, BoundSearch &s, const PackedBounds &pk, cudaStream_t strm, bool publish,
                 size_t extra_res = 0);

// profiling: bracket a kernel launch with events when enabled
int prof_index(kb_ctx *ctx, const char *name);
static inline bool prof_major(const char *n) { return n[0] == 'k' && n[1] == '_' && ((n[2] == 'd' && n[3] == 'e') || (n[2] == 'g' && n[3] == 'a' && n[8] == 0)); }
void prof_begin(kb_ctx *ctx, int idx, uint64_t alg_bytes, cudaStream_t strm);
// a completion event from ctx->ev_pool, or a new one; *ev stays nullptr when none can be had
int ev_take(kb_ctx *ctx, cudaEvent_t *ev);
void prof_end(kb_ctx *ctx, cudaStream_t strm);

#define KB_LAUNCH_S(ctx, strm, name, bytes, ...)              \
    do {                                                      \
        static thread_local int _pi = -1;                     \
        const bool _p = (ctx)->prof_on == 1 || ((ctx)->prof_on == 2 && prof_major(name)); \
        if (_p) {                                             \
            _pi = prof_index((ctx), (name));                  \
            prof_begin((ctx), _pi, (bytes), (strm));          \
        }                                                     \
        __VA_ARGS__;                                          \
        (ctx)->launches++;                                    \
        if (_p) prof_end((ctx), (strm));                      \
    } while (0)
#define KB_LAUNCH(ctx, name, bytes, ...) KB_LAUNCH_S(ctx, (ctx)->lane().stream, name, bytes, __VA_ARGS__)

// one polite spin of a host polling loop (the device publishes results into mapped pinned memory)
static inline void kb_cpu_relax()
{
#if defined(__x86_64__) || defined(__i386__)
    __builtin_ia32_pause();
#endif
}

// host wall-clock segments (with kb_prof_enable(ctx, 1 or 2)): where the non-kernel time of a call goes
typedef std::chrono::steady_clock::time_point kb_tp;
static inline kb_tp kb_now() { return std::chrono::steady_clock::now(); }
static inline void kb_seg(kb_ctx *ctx, const char *name, kb_tp &t)
{
    if (ctx->prof_on == 0) return;
    kb_tp n = kb_now();
    int i = prof_index(ctx, name);
    ctx->prof[i].launches++;
    ctx->prof[i].ms += std::chrono::duration<double, std::milli>(n - t).count();
    t = n;
}

// The lower bounds of a range batch's bounds (2 q: start of request q, 2 q + 1: its end) on the host, from a search
// kb_range_prefetch started for the same bounds on the same snapshot, or from a new one of lane L's (kb_search.cu).
// tseg: the host:range_* profiling segments
int range_bounds_find(kb_ctx *ctx, ScanLane &L, const kb_range_req *reqs, uint64_t nreq, const uint32_t **res,
                      kb_tp *tseg);

// kb_watch.cu
void watch_tables_free(kb_ctx *ctx);
