// kb_scan.cuh -- what the files of the scan path share: kb_scan.cu (the scan core), kb_copy.cu (the answer and its copy),
// kb_batch.cu (range batches and point reads), kb_page.cu (page cuts, range streams, partitions) and kb_compact.cu (the
// compaction sweep and its streams).  Every kernel is defined in exactly one of them.
#pragma once

#include "kb_internal.cuh"

namespace {

constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ uint64_t warp_incl_scan_u64(uint64_t v)
{
    const unsigned lane = threadIdx.x & 31;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint64_t o = __shfl_up_sync(FULL, v, d);
        if (lane >= (unsigned)d) v += o;
    }
    return v;
}

// exclusive scan of two u64 values per thread over 256 threads
__device__ __forceinline__ void block_excl_scan2(uint64_t a, uint64_t b, uint64_t &ea, uint64_t &eb, uint64_t &ta,
                                                 uint64_t &tb, uint64_t *ws /* 2*9 */)
{
    const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint64_t ia = warp_incl_scan_u64(a), ib = warp_incl_scan_u64(b);
    if (lane == 31) {
        ws[w] = ia;
        ws[9 + w] = ib;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t ra = 0, rb = 0;
        for (int k = 0; k < 8; k++) {
            uint64_t x = ws[k], y = ws[9 + k];
            ws[k] = ra;
            ws[9 + k] = rb;
            ra += x;
            rb += y;
        }
        ws[8] = ra;
        ws[17] = rb;
    }
    __syncthreads();
    ea = ia - a + ws[w];
    eb = ib - b + ws[9 + w];
    ta = ws[8];
    tb = ws[17];
    __syncthreads();
}

// Every lane of a warp: the first index in [lo, hi) where pred is false (hi when there is none); pred must hold for a
// prefix of the interval.  Each step tests 32 spread-out pivots and keeps the candidates between the last that holds and
// the first that does not; 32 candidates or fewer are tested at once.
template <class Pred>
__device__ __forceinline__ uint64_t warp_partition_point(uint64_t lo, uint64_t hi, Pred pred)
{
    const uint32_t lane = threadIdx.x & 31;
    while (hi > lo) {
        const uint64_t span = hi - lo;
        if (span <= 32) {
            lo += __popc(__ballot_sync(FULL, lane < span && pred(lo + lane)));
            break;
        }
        const uint64_t piv = lo + (span - 1) * lane / 31;
        const int c = __popc(__ballot_sync(FULL, pred(piv)));
        const uint64_t nlo = c > 0 ? __shfl_sync(FULL, piv, c - 1) + 1 : lo;
        const uint64_t nhi = c < 32 ? __shfl_sync(FULL, piv, c) : hi;
        lo = nlo;
        hi = nhi;
    }
    return lo;
}

// One warp: the padded key chunks of record rec into dst, every byte at or past `keep` zeroed.  Four chunk loads per lane
// stay in flight on long keys.
__device__ __forceinline__ void warp_copy_key(const StoreDev &st, uint32_t rec, uint4 *dst, uint32_t keep)
{
    const uint32_t kl = st.klen[rec];
    const uint4 *src = st.kslab + st.koff16[rec];
#pragma unroll 4
    for (uint32_t c = threadIdx.x & 31; c * 16 < kl; c += 32) {
        uint4 v = src[c];
        uint8_t *b = (uint8_t *)&v;
#pragma unroll
        for (uint32_t j = 0; j < 16; j++)
            if (c * 16 + j >= keep) b[j] = 0;
        dst[c] = v;
    }
}

}  // namespace

// one request's row of a scan
struct ReqOut {
    uint64_t total;        // emissions (range) / delete calls (compact)
    uint64_t total_aux;    // response bytes (range) / object count (compact)
    uint64_t capped_aux;   // response bytes of the first `limit` emissions (valid with KB_RO_CAPPED)
    uint32_t examined;     // records pulled from the iterator (valid with KB_RO_LIMIT_STOP, else hi - lo)
    uint32_t flags;
};
enum { KB_RO_LIMIT_STOP = 1u, KB_RO_CAPPED = 2u };

// the per-kv view arrays of a range answer
struct GatherOut {
    uint32_t *rec_idx;
    uint64_t *rev;
    uint64_t *key_off;
    uint32_t *key_len;
    uint64_t *val_off;
    uint32_t *val_len;
};

// one copy job per emitted kv (32 bytes): built thread-parallel so the per-kv lookups (request search, selection,
// offsets, lengths) do not sit in front of the streaming copy
struct GatherJob {
    uint64_t dst16;   // arena chunk index
    uint64_t vsrc16;  // value slab chunk index
    uint32_t ksrc16;  // key slab chunk index
    uint32_t nk, nv;  // 16-byte chunks of key / value
    uint32_t kl;      // exact key length
};

// requests resolved to record intervals and laid out as tiles
struct Resolved {
    std::vector<ReqDev> reqs;
    uint32_t nt = 0;  // tiles of the batch (the tile table itself is filled on the device, k_fill_tiles)
    uint64_t total_flat = 0, total_sel = 0, key_bytes = 0, n_records = 0;
};

// k_page_cut's report, a HostPub with the context's error flag as its error word: payload [end kv u64 | arena bytes u64 |
// key length u64], then from byte KB_PAGE_PUB_KEY the internal key of the page's last kv
constexpr size_t KB_PAGE_PUB_KEY = 64;
constexpr size_t KB_PAGE_PUB_BYTES = KB_PAGE_PUB_KEY + 65536 + 16;

// what a range stream and a compaction stream share: n entries (kvs / victims) of `total` arena bytes, handed out in pages
// of whole groups
struct PageStream {
    uint64_t group = 1;
    uint64_t n = 0, total = 0, pos = 0;  // entries, their arena bytes, entries handed out
    HostPub pub;                         // k_page_cut's report
};

// the next page of p: entries [p.pos, end) within max_bytes (at least one group), `bytes` of arena
struct PageCut {
    JobSet *J;  // holds the page's one-request job table
    uint64_t end, bytes;
};

// kb_scan.cu
int resolve_requests(kb_ctx *ctx, ScanLane &L, const kb_range_req *reqs, uint64_t nreq, bool cap_by_limit, Resolved &R,
                     kb_tp *tseg = nullptr);
int resolve_interval(kb_ctx *ctx, ScanLane &L, const uint8_t *start, uint64_t start_len, const uint8_t *end,
                     uint64_t end_len, uint64_t rev, Resolved &R);
int upload_layout(kb_ctx *ctx, ScanLane &L, const Resolved &R);
int sel_ensure(kb_ctx *ctx, ScanLane &L, const Resolved &R);
int launch_scan_core(kb_ctx *ctx, ScanLane &L, const Resolved &R, const ScanMode &mode, bool with_place,
                     uint32_t *vidx = nullptr, uint8_t *vcls = nullptr);
int scan_sync(kb_ctx *ctx, ScanLane &L, const Resolved &R, const ScanMode &mode, bool with_place, const ReqOut **rows,
              uint32_t *vidx = nullptr, uint8_t *vcls = nullptr);
int probe_limit_windows(kb_ctx *ctx, ScanLane &L, Resolved &R, int wire, bool *reused);

// kb_copy.cu
void result_put_device(kb_ctx *ctx, kb_result *res);
int pub_err_check(kb_ctx *ctx, const HostPub &pub);
int split_out_mode(int out_mode, int *base, int *wire);
uint64_t *om_layout(void *om, uint64_t cap, int wire, GatherOut &go);
int answer_new(kb_ctx *ctx, HeldResult &res, ResultKind kind, int out_mode, int wire, uint64_t cap_kvs,
               uint64_t arena_bytes, GatherOut *go = nullptr, uint64_t **elem_off = nullptr);
int answer_finish(kb_ctx *ctx, kb_result *res, const GatherOut &go, const uint64_t *d_elem_off, uint64_t nk,
                  uint64_t nbytes, kb_tp &tseg);
size_t copy_jobs_bytes(uint64_t n, int wire);
int copy_after_jobs(kb_ctx *ctx, ScanLane &L, cudaStream_t sg);
int copy_done(kb_ctx *ctx, cudaStream_t sg, cudaEvent_t ev_copied, kb_result *res);
int launch_gather(kb_ctx *ctx, cudaStream_t strm, const GatherJob *d_jobs, const JobTable &tab, uint4 *arena,
                  uint64_t n_jobs, uint64_t alg_bytes);
int launch_copy(kb_ctx *ctx, ScanLane &L, cudaStream_t sg, void *d_jobs, cudaEvent_t ev_copied, const ReqDev *d_reqs,
                uint32_t nreq, const JobTable &tab, const uint32_t *sel, const uint64_t *slot, uint64_t cap_kvs, int wire,
                const GatherOut &go, uint64_t *d_elem_off, kb_result *res);

// kb_batch.cu
int compact_race_check(kb_ctx *ctx, uint64_t rev);

// kb_page.cu
int page_cut(kb_ctx *ctx, PageStream &p, const uint32_t *sel, const uint64_t *slot, uint64_t max_bytes, const char *what,
             kb_tp &tseg, PageCut *out);
void stream_free(kb_range_stream *s);
