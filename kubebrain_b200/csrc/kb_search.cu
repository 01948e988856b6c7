// kb_search.cu -- the bound search: the lower bounds of a batch of keys in the sorted directory, for range batches and
// their prefetch (kb_range_prefetch), point reads and the write path.  The bound slab it reads is laid out by
// bounds_pack and read on the device through BoundsDev (kb_internal.cuh).
#include "kb_internal.cuh"

namespace {

constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ bool key_less(const StoreDev &st, uint32_t rec, const uint4 *b, uint32_t blen)
{
    const uint4 *a = st.kslab + st.koff16[rec];
    uint32_t la = st.klen[rec];
    uint32_t m = la < blen ? la : blen;
    // Kubernetes keys share ~30 leading bytes: fetch the first three chunks together instead of one per round trip
    // (both slabs are padded, so the loads are in bounds; positions at or beyond m are ignored)
    {
        uint4 x0 = a[0], x1 = a[1], x2 = a[2];
        uint4 y0 = __ldg(b), y1 = __ldg(b + 1), y2 = __ldg(b + 2);
        int p = first_diff16(x0, y0);
        if (p < 16) return p < (int)m ? byte_of(x0, p) < byte_of(y0, p) : la < blen;
        p = first_diff16(x1, y1);
        if (p < 16) return 16 + p < (int)m ? byte_of(x1, p) < byte_of(y1, p) : la < blen;
        p = first_diff16(x2, y2);
        if (p < 16) return 32 + p < (int)m ? byte_of(x2, p) < byte_of(y2, p) : la < blen;
    }
    for (uint32_t c = 3; c * 16 < m; c++) {
        uint4 x = a[c], y = __ldg(b + c);
        int p = first_diff16(x, y);
        if (p < 16 && c * 16 + p < m) return byte_of(x, p) < byte_of(y, p);
    }
    return la < blen;
}

// out[w] = index of the first record whose key >= bound w (bytes.Compare order)
// pub (optional): a HostPub whose payload is the results u32 x nb.  Every warp stores its result there too; the warp that
// completes the count raises the flag to `epoch` -- the host polls it instead of paying a stream / event synchronisation
// (slow for an already finished search while another host thread is busy in the driver).
struct SearchPub {
    uint8_t *host;          // nullptr: results only in `out`
    unsigned int *done;     // device counter, zero between searches
    uint64_t epoch;
};

__global__ void __launch_bounds__(128) k_search(StoreDev st, BoundsDev bounds, uint32_t *__restrict__ out, SearchPub pub)
{
    uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    uint32_t lane = threadIdx.x & 31;
    const uint32_t nb = bounds.n;
    if (w >= nb) return;
    const uint4 *b = bounds.key(w);
    uint32_t bl = bounds.len(w);
    uint32_t lo = 0, hi = st.n;
    for (;;) {
        uint32_t span = hi - lo;
        if (span == 0) break;
        if (span <= 32) {
            bool less = lane < span ? key_less(st, lo + lane, b, bl) : false;
            lo += __popc(__ballot_sync(FULL, less));
            break;
        }
        uint32_t piv = lo + (uint32_t)(((uint64_t)span * (lane + 1)) / 33);
        bool less = key_less(st, piv, b, bl);
        int k = __popc(__ballot_sync(FULL, less));  // sorted slab: `less` holds for a prefix of the pivots
        uint32_t nlo = lo, nhi = hi;
        if (k > 0) nlo = __shfl_sync(FULL, piv, k - 1) + 1;
        if (k < 32) nhi = __shfl_sync(FULL, piv, k);
        lo = nlo;
        hi = nhi;
    }
    if (lane == 0) {
        out[w] = lo;
        if (pub.host) {
            ((volatile uint32_t *)(pub.host + KB_PUB_HEAD))[w] = lo;
            __threadfence_system();
            if (atomicAdd(pub.done, 1u) == nb - 1) {
                *pub.done = 0;
                pub_raise(pub.host, pub.epoch);
            }
        }
    }
}

// the bounds of a range batch: [start, end) of every request
int range_bounds_pack(kb_ctx *ctx, const kb_range_req *reqs, uint64_t nreq, HBuf &stage, PackedBounds *pk)
{
    for (uint64_t q = 0; q < nreq; q++) {
        if ((!reqs[q].start && reqs[q].start_len) || (!reqs[q].end && reqs[q].end_len)) return KB_EINVAL;
        if (reqs[q].start_len > 65535 || reqs[q].end_len > 65535) return kb_fail(ctx, KB_ELIMIT, "bound key too long");
    }
    return bounds_pack(
        ctx, stage, 2 * nreq, [&](uint64_t i) { return i & 1 ? reqs[i / 2].end_len : reqs[i / 2].start_len; },
        [&](uint64_t i, uint8_t *dst) {
            const kb_range_req &r = reqs[i / 2];
            const uint64_t len = i & 1 ? r.end_len : r.start_len;
            if (len) memcpy(dst, i & 1 ? r.end : r.start, len);
        },
        pk);
}

}  // namespace

int bound_search(kb_ctx *ctx, BoundSearch &s, const PackedBounds &pk, cudaStream_t strm, bool publish, size_t extra_res)
{
    const uint64_t n = pk.n;
    KB_TRY(dbuf_ensure(ctx, s.d_bounds, pk.bytes() + 64));
    KB_TRY(dbuf_ensure(ctx, s.d_bres, n * 4 + extra_res + 16));
    if (publish) KB_TRY(hostpub_ensure(ctx, s.pub, KB_PUB_HEAD + n * 4, strm));
    KB_CUDA(ctx, cudaMemcpyAsync(s.d_bounds.p, pk.host, pk.bytes(), cudaMemcpyHostToDevice, strm));
    const uint32_t *off16 = (const uint32_t *)((const uint8_t *)s.d_bounds.p + pk.chunks * 16);
    s.dev = BoundsDev{(const uint4 *)s.d_bounds.p, off16, off16 + n, (uint32_t)n};
    const SearchPub pub{publish ? s.pub.p : nullptr, (unsigned int *)ctx->d_ctrs.p + s.pub_ctr, publish ? ++s.pub.epoch : 0};
    if (n == 0 && publish) *(volatile uint64_t *)s.pub.p = s.pub.epoch;  // nothing to search: already "published"
    if (n == 0) return KB_OK;
    KB_LAUNCH(ctx, "k_search", n * 64,
              (k_search<<<(unsigned)((n * 32 + 127) / 128), 128, 0, strm>>>(ctx->st, s.dev, (uint32_t *)s.d_bres.p, pub)));
    return KB_OK;
}

int range_bounds_find(kb_ctx *ctx, ScanLane &L, const kb_range_req *reqs, uint64_t nreq, const uint32_t **res, kb_tp *tseg)
{
    PackedBounds pk;
    KB_TRY(range_bounds_pack(ctx, reqs, nreq, L.h_stage, &pk));
    if (tseg) kb_seg(ctx, "host:range_pack_bounds", *tseg);
    SearchSlot *hit = nullptr;
    for (auto &sl : ctx->prefetch)  // the OLDEST matching one: a caller may already have submitted the batch after this one
        if (sl.valid && sl.ident_bytes == pk.bytes() && sl.store_gen == ctx->store_gen &&
            memcmp(sl.stage.p, pk.host, pk.bytes()) == 0 && (!hit || sl.seq < hit->seq))
            hit = &sl;
    if (ctx->prof_on == 1) hit = nullptr;
    BoundSearch &s = hit ? hit->search : L.search;
    // The search only reads the snapshot and its own bound slab, so it runs on the second stream: while the previous
    // batch's gather is still draining the host already learns the record intervals of this one.
    // (With every kernel bracketed by profiling events -- level 1 -- it stays on the lane stream.)
    cudaStream_t ss = ctx->prof_on == 1 ? L.stream : ctx->stream2;
    if (!hit) KB_TRY(bound_search(ctx, s, pk, ss, true));
    if (tseg) kb_seg(ctx, "host:range_search_enqueue", *tseg);
    KB_TRY(hostpub_wait(ctx, s.pub, s.pub.epoch, ss, "bound search", true));
    *res = s.pub.payload<const uint32_t>();
    if (hit) hit->valid = false;  // consumed
    if (tseg) kb_seg(ctx, "host:range_search_sync", *tseg);
    return KB_OK;
}

// Start the bound search of a batch that a later kb_range_batch will ask for (same bounds, same snapshot): a caller with a
// queue of pending requests submits batch n+1 before it waits for batch n, so the search's host round trip (the one
// synchronisation a range call needs before it can lay its requests out) overlaps the previous batch's kernels.
extern "C" int kb_range_prefetch(kb_ctx *ctx, const kb_range_req *reqs, uint64_t nreq)
{
    if (!ctx || (nreq && !reqs)) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->loaded) return kb_fail(ctx, KB_ESTATE, "no store loaded");
    cudaSetDevice(ctx->device);
    const int slot = (int)(ctx->prefetch_next++ & 1);
    SearchSlot &sl = ctx->prefetch[slot];
    if (ctx->prof_on) {  // diagnostic: is the OTHER slot's (older) submission already complete when the next one is made?
        SearchSlot &other = ctx->prefetch[slot ^ 1];
        if (other.valid && other.search.pub.p) {
            const bool ready = *(volatile uint64_t *)other.search.pub.p == other.search.pub.epoch;
            ctx->prof[prof_index(ctx, ready ? "host:prefetch_older_ready" : "host:prefetch_older_pending")].launches++;
        }
    }
    // an unconsumed older submission still owns the buffers
    if (sl.valid) KB_TRY(hostpub_wait(ctx, sl.search.pub, sl.search.pub.epoch, ctx->stream2, "bound search", true));
    sl.valid = false;
    PackedBounds pk;
    KB_TRY(range_bounds_pack(ctx, reqs, nreq, sl.stage, &pk));
    KB_TRY(bound_search(ctx, sl.search, pk, ctx->stream2, true));
    sl.ident_bytes = pk.bytes();
    sl.store_gen = ctx->store_gen;
    sl.seq = ctx->prefetch_next;
    sl.valid = true;
    return KB_OK;
}
