// kb_page.cu -- cuts of a placed answer by its arena offsets.  Both callers run the scan core's unlimited scan with
// placement (kb_scan.cu) on the current lane, then one single-CTA cut that publishes to mapped memory:
//   range streams     per page k_page_cut [S] -> the copy (kb_copy.cu): jobs [S], copy [SG]; compaction streams
//                     (kb_compact.cu) cut their pages with k_page_cut too
//   range partitions  k_partition_cut [S]: P equal shares of the answer's bytes at user-key borders
#include <algorithm>
#include <memory>

#include "kb_scan.cuh"

// ================================================================================================
// range streams: one unlimited scan at open, its answer handed out page by page within a byte budget
// ================================================================================================
namespace {

// One warp.  The page starting at kv a of the stream's selection ends at b = min(a + k * group, n) for the largest k >= 1
// whose arena bytes slot[b] - slot[a] (slot[n] = total) are at most max_bytes, or k = 1 when not even one group fits.
// Writes the page's one-request job table (kvs a .. b - 1 of the selection, arena base -slot[a]), then publishes b, the
// bytes and the page's last key to the host.  sel = nullptr: no last key (a compaction stream's victims are record
// indices of an older snapshot; the live directory may no longer hold them).
__global__ void __launch_bounds__(32)
k_page_cut(StoreDev st, const uint32_t *__restrict__ sel, const uint64_t *__restrict__ slot, uint64_t n, uint64_t total,
           uint64_t a, uint64_t group, uint64_t max_bytes, uint64_t *__restrict__ jobtab, uint8_t *host, uint64_t epoch,
           const unsigned int *__restrict__ err_flag)
{
    const uint32_t lane = threadIdx.x;
    const uint64_t base = slot[a];
    const uint64_t groups = (n - a + group - 1) / group;  // the last one may be partial
    auto end_of = [&](uint64_t k) { return n - a > k * group ? a + k * group : n; };
    auto bytes_of = [&](uint64_t k) {
        const uint64_t b = end_of(k);
        return (b == n ? total : slot[b]) - base;
    };
    // the largest k in [0, groups] whose page fits (k = 0 always does)
    const uint64_t k = warp_partition_point(1, groups + 1, [&](uint64_t k) { return bytes_of(k) <= max_bytes; }) - 1;
    const uint64_t b = end_of(k > 1 ? k : 1);
    const uint64_t bytes = bytes_of(k > 1 ? k : 1);
    uint32_t kl = 0;
    if (sel) {
        const uint32_t rec = sel[b - 1];
        kl = st.klen[rec];
        warp_copy_key(st, rec, (uint4 *)(host + KB_PAGE_PUB_KEY), kl);
    }
    if (lane == 0) {
        jobtab_write_one(jobtab, b - a, 0 - base, bytes, (uint32_t)a);  // the job kernels place kv s at 0 - base + slot[s]
        volatile uint64_t *h = (volatile uint64_t *)host;
        h[1] = *err_flag;  // a bulk copy of an earlier answer never completed
        h[2] = b;
        h[3] = bytes;
        h[4] = kl;
    }
    __threadfence_system();
    __syncwarp();
    if (lane == 0) pub_raise(host, epoch);
}

}  // namespace

// Cut the next page of p on the current lane: k_page_cut over the entries' arena offsets (slot; sel: the records of a
// range stream's kvs, whose last key it publishes) writes the page's job table into the next JobSet, which alternates
// with the range batches' as between two batches.
int page_cut(kb_ctx *ctx, PageStream &p, const uint32_t *sel, const uint64_t *slot, uint64_t max_bytes, const char *what,
             kb_tp &tseg, PageCut *out)
{
    ScanLane &L = ctx->lane();
    JobSet &J = ctx->jobsets[ctx->batch_seq++ & 1];
    KB_TRY(dbuf_ensure(ctx, J.jobs, jobtab_bytes(1) + sizeof(ReqDev)));
    KB_CUDA(ctx, cudaStreamWaitEvent(L.stream, J.ev_gather, 0));
    const uint64_t epoch = ++p.pub.epoch;
    KB_LAUNCH_S(ctx, L.stream, "k_page_cut", 64,
                (k_page_cut<<<1, 32, 0, L.stream>>>(ctx->st, sel, slot, p.n, p.total, p.pos,
                                                   std::min(p.group, p.n - p.pos),  // no overflow
                                                   max_bytes, (uint64_t *)J.jobs.p, p.pub.p, epoch,
                                                   (const unsigned int *)ctx->d_ctrs.p + 8)));
    KB_CUDA(ctx, cudaGetLastError());
    KB_TRY(hostpub_wait(ctx, p.pub, epoch, L.stream, what));
    KB_TRY(pub_err_check(ctx, p.pub));
    const volatile uint64_t *h = p.pub.payload<volatile uint64_t>();
    *out = PageCut{&J, h[0], h[1]};
    kb_seg(ctx, "host:page_cut", tseg);
    return KB_OK;
}

struct kb_range_stream : PageStream {
    std::string start, end;                // the bounds of the open (internal keys)
    uint64_t read_rev = 0;
    int out_mode = 0, wire = 0;            // KB_OUT_HOST / KB_OUT_DEVICE, KB_WIRE_*_I
    uint64_t gen = 0;                      // ctx->store_gen the scan was made on
    DBuf d_sel, d_slot;                    // the scan's selection (record per kv) and each kv's arena offset
    std::string last_key;                  // internal key of the last kv handed out
    bool started = false, done = false;
};

void stream_free(kb_range_stream *s)
{
    if (s->d_sel.p) cudaFree(s->d_sel.p);
    if (s->d_slot.p) cudaFree(s->d_slot.p);
    hostpub_free(s->pub);
    delete s;
}

// the least internal key greater than every key that starts with k: k + 0x00, or (k at the 65535-byte key limit) k with
// its trailing 0xff bytes dropped and the last byte left incremented.  false: no such key can exist.
static bool key_after(const std::string &k, std::string *out)
{
    if (k.size() < 65535) {
        *out = k;
        out->push_back('\0');
        return true;
    }
    *out = k;
    while (!out->empty() && (uint8_t)out->back() == 0xff) out->pop_back();
    if (out->empty()) return false;
    out->back() = (char)((uint8_t)out->back() + 1);
    return true;
}

// One unlimited scan of [start, s->end) at s->read_rev on the current lane (decode .. placement, as a range batch); its
// selection and arena offsets are copied into the stream's buffers, and the lane is free again when this returns.
static int stream_scan(kb_ctx *ctx, kb_range_stream *s, const std::string &start)
{
    KB_TRY(lane_take(ctx));
    ScanLane &L = ctx->lane();
    Resolved R;
    KB_TRY(resolve_interval(ctx, L, (const uint8_t *)start.data(), start.size(), (const uint8_t *)s->end.data(),
                            s->end.size(), s->read_rev, R));
    const ReqOut *rows = nullptr;
    KB_TRY(scan_sync(ctx, L, R, ScanMode::range(s->wire), true, &rows));
    const ReqOut ro = *rows;
    if (ro.total) {
        KB_TRY(dbuf_ensure(ctx, s->d_sel, ro.total * 4));
        KB_TRY(dbuf_ensure(ctx, s->d_slot, ro.total * 8));
        KB_CUDA(ctx, cudaMemcpyAsync(s->d_sel.p, L.d_sel.p, ro.total * 4, cudaMemcpyDeviceToDevice, L.stream));
        KB_CUDA(ctx, cudaMemcpyAsync(s->d_slot.p, L.d_slot.p, ro.total * 8, cudaMemcpyDeviceToDevice, L.stream));
        KB_CUDA(ctx, cudaStreamSynchronize(L.stream));
    }
    s->n = ro.total;
    s->total = ro.total_aux;
    s->pos = 0;
    s->gen = ctx->store_gen;
    return KB_OK;
}

extern "C" int kb_range_stream_open(kb_ctx *ctx, const kb_range_req *req, int out_mode, uint64_t group_kvs,
                                    kb_range_stream **out)
{
    if (!ctx || !req || !out) return KB_EINVAL;
    *out = nullptr;
    int base = 0, wire = 0;
    KB_TRY(split_out_mode(out_mode, &base, &wire));
    if (base != KB_OUT_HOST && base != KB_OUT_DEVICE) return KB_EINVAL;
    if (group_kvs == 0 || req->limit > 0) return KB_EINVAL;
    if ((!req->start && req->start_len) || (!req->end && req->end_len)) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->loaded) return kb_fail(ctx, KB_ESTATE, "no store loaded");
    KB_TRY(compact_race_check(ctx, req->read_rev));
    cudaSetDevice(ctx->device);
    std::unique_ptr<kb_range_stream, void (*)(kb_range_stream *)> s(new kb_range_stream(), stream_free);
    s->start.assign((const char *)req->start, req->start_len);
    s->end.assign((const char *)req->end, req->end_len);
    s->read_rev = req->read_rev;
    s->out_mode = base;
    s->wire = wire;
    s->group = group_kvs;
    KB_TRY(hostpub_ensure(ctx, s->pub, KB_PAGE_PUB_BYTES, ctx->lane().stream));
    KB_TRY(stream_scan(ctx, s.get(), s->start));
    ctx->streams.push_back(s.get());
    *out = s.release();
    return KB_OK;
}

extern "C" int kb_range_stream_next(kb_ctx *ctx, kb_range_stream *s, uint64_t max_bytes, kb_result **page)
{
    if (!ctx || !s || !page) return KB_EINVAL;
    *page = nullptr;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (s->done) return KB_OK;
    if (!ctx->loaded) return kb_fail(ctx, KB_ESTATE, "no store loaded");
    cudaSetDevice(ctx->device);
    if (s->gen != ctx->store_gen) {
        // The snapshot changed since the scan, so its record indices are stale: scan again what has not been handed out
        // yet.  worker.run emits a kv when it meets the next visible record of another user key, so a scan that starts
        // right behind the last kv handed out reaches every later emission in the same state.
        std::string from = s->start;
        if (s->started && !key_after(s->last_key, &from)) {
            s->done = true;
            return KB_OK;
        }
        // the job kernels of earlier pages read the selection: they are done once the copies that waited for them are
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->stream_g));
        KB_TRY(stream_scan(ctx, s, from));
    }
    if (s->pos >= s->n) {
        s->done = true;
        return KB_OK;
    }
    kb_tp tseg = kb_now();
    PageCut c;
    KB_TRY(page_cut(ctx, *s, (const uint32_t *)s->d_sel.p, (const uint64_t *)s->d_slot.p, max_bytes, "range stream", tseg,
                    &c));
    JobSet &J = *c.J;
    const uint64_t nk = c.end - s->pos, nbytes = c.bytes;

    // every buffer of the page is sized by the page: the cut is known before the copy is launched
    HeldResult res{ctx, nullptr};
    GatherOut go;
    uint64_t *d_elem_off = nullptr;
    KB_TRY(answer_new(ctx, res, ResultKind::range, s->out_mode, s->wire, nk, nbytes + 64, &go, &d_elem_off));
    KB_TRY(dbuf_ensure(ctx, J.gjobs, copy_jobs_bytes(nk, s->wire)));
    KB_TRY(launch_copy(ctx, ctx->lane(), ctx->stream_g, J.gjobs.p, J.ev_gather, jobtab_req(J.jobs.p), 1,
                       jobtab_at(J.jobs.p, 1), (const uint32_t *)s->d_sel.p, (const uint64_t *)s->d_slot.p, nk, s->wire, go,
                       d_elem_off, res.p));
    res.p->req_first = {0, nk};
    res.p->req_count = {nk};
    res.p->req_examined = {0};
    res.p->n_kvs = nk;
    res.p->n_bytes = nbytes;
    KB_TRY(answer_finish(ctx, res.p, go, d_elem_off, nk, nbytes, tseg));
    s->pos = c.end;
    s->last_key.assign((const char *)s->pub.p + KB_PAGE_PUB_KEY, s->pub.payload<volatile uint64_t>()[2]);
    s->started = true;
    *page = res.release();
    return KB_OK;
}

extern "C" void kb_range_stream_close(kb_ctx *ctx, kb_range_stream *s)
{
    if (!ctx || !s) return;
    std::lock_guard<std::mutex> g(ctx->mu);
    auto it = std::find(ctx->streams.begin(), ctx->streams.end(), s);
    if (it == ctx->streams.end()) return;
    ctx->streams.erase(it);
    cudaSetDevice(ctx->device);
    // the job kernels of its pages read its selection: they are done once the copies that waited for them are
    cudaStreamSynchronize(ctx->stream_g);
    stream_free(s);
}

// ================================================================================================
// range partitions: one unlimited scan with placement, then the answer cut into P equal byte shares at user-key borders
// ================================================================================================
namespace {

constexpr uint64_t KB_MAX_PARTS = 4096;
constexpr unsigned KB_PART_WARPS = 16;

// k_partition_cut's report in ctx->ppub (error word: the context's error flag): per cut k = 1 .. P-1 the u64 quadruple
// [kv index | arena offset | key length | above] at payload entry 4 (k - 1), then from payload byte part_keys_off(P) the
// revision-record key of cut k at (k - 1) * key_stride.  A cut with no kv (index n) has arena offset T and no key.
__host__ __device__ constexpr uint64_t part_keys_off(uint64_t parts) { return (parts - 1) * 32; }

// One warp: is the internal key of record b, every byte at or past b_keep read as 0, greater than that of record a?
__device__ __forceinline__ bool warp_key_greater(const StoreDev &st, uint32_t b, uint32_t b_keep, uint32_t a)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t bl = st.klen[b], al = st.klen[a], m = bl < al ? bl : al;
    const uint4 *pb = st.kslab + st.koff16[b], *pa = st.kslab + st.koff16[a];
    for (uint32_t c0 = 0; c0 * 16 < m; c0 += 32) {
        const uint32_t c = c0 + lane;
        int p = 16;
        uint4 x{}, y{};
        if (c * 16 < m) {
            x = pb[c];
            y = pa[c];
            uint8_t *xb = (uint8_t *)&x;
#pragma unroll
            for (uint32_t j = 0; j < 16; j++)
                if (c * 16 + j >= b_keep) xb[j] = 0;
            p = first_diff16(x, y);
            if (c * 16 + p >= m) p = 16;
        }
        const unsigned diff = __ballot_sync(FULL, p < 16);
        if (diff) {
            const int src = __ffs(diff) - 1;
            const bool gt = p < 16 && byte_of(x, p) > byte_of(y, p);
            return __shfl_sync(FULL, gt, src);
        }
    }
    return bl > al;  // one a prefix of the other: the longer is greater
}

// One CTA; warp w takes the cuts k = w + 1, w + 1 + KB_PART_WARPS, ...: the least i in [1, n) with slot[i] * P >= k * T
// (n when there is none) by the 32-ary search k_page_cut uses too, then the internal key of kv i with its 8 revision
// bytes zeroed (EncodeRevisionKey of its user key; every emitted record decodes, so its key is at least 13 bytes long),
// and whether that border is above kv i - 1's record.  It is not when kv i - 1's user key is kv i's + '$' + bytes that
// sort below kv i's revision bytes: the border would then run backwards, so the host drops the cut.
__global__ void __launch_bounds__(KB_PART_WARPS * 32)
k_partition_cut(StoreDev st, const uint32_t *__restrict__ sel, const uint64_t *__restrict__ slot, uint64_t n, uint64_t total,
                uint64_t parts, uint64_t key_stride, uint8_t *host, uint64_t epoch, const unsigned int *__restrict__ err_flag)
{
    const uint32_t lane = threadIdx.x & 31;
    uint64_t *cut = (uint64_t *)(host + KB_PUB_HEAD);
    uint8_t *keys = host + KB_PUB_HEAD + part_keys_off(parts);
    for (uint64_t k = 1 + (threadIdx.x >> 5); k < parts; k += KB_PART_WARPS) {
        const uint64_t want = k * total;
        const uint64_t i = warp_partition_point(1, n, [&](uint64_t i) { return slot[i] * parts < want; });
        uint32_t kl = 0;
        bool above = false;
        if (i < n) {
            const uint32_t rec = sel[i];
            kl = st.klen[rec];
            warp_copy_key(st, rec, (uint4 *)(keys + (k - 1) * key_stride), kl - 8);
            above = warp_key_greater(st, rec, kl - 8, sel[i - 1]);
        }
        if (lane == 0) {
            volatile uint64_t *h = cut + 4 * (k - 1);
            h[0] = i;
            h[1] = i < n ? slot[i] : total;
            h[2] = kl;
            h[3] = above;
        }
    }
    if (threadIdx.x == 0) *(volatile uint64_t *)(host + 8) = *err_flag;  // a bulk copy of an earlier answer never completed
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) pub_raise(host, epoch);
}

// bytes.Compare(a, b) < 0
bool host_key_less(const uint8_t *a, uint64_t al, const uint8_t *b, uint64_t bl)
{
    const uint64_t m = std::min(al, bl);
    const int c = m ? memcmp(a, b, m) : 0;
    return c < 0 || (c == 0 && al < bl);
}

}  // namespace

static int range_partitions_locked(kb_ctx *ctx, const kb_range_req *req, uint64_t part_bytes, uint64_t max_parts,
                                   kb_result **out)
{
    KB_TRY(lane_take(ctx));  // only the current lane: batches on the others stay in flight
    ScanLane &L = ctx->lane();
    Resolved R;
    KB_TRY(resolve_interval(ctx, L, req->start, req->start_len, req->end, req->end_len, req->read_rev, R));
    const ReqOut *rows = nullptr;
    KB_TRY(scan_sync(ctx, L, R, ScanMode::range(0), true, &rows));
    const uint64_t n = rows->total, T = rows->total_aux;

    uint64_t parts = 1;
    if (n > 1 && host_key_less(req->start, req->start_len, req->end, req->end_len)) {
        const uint64_t shares = std::max<uint64_t>(1, T / part_bytes + (T % part_bytes != 0));
        parts = std::min(std::min(max_parts, n), shares);
    }
    // kept cuts: (kv index, arena offset, key bytes in the report, key length)
    struct Cut {
        uint64_t kv, arena;
        const uint8_t *key;
        uint64_t klen;
    };
    std::vector<Cut> cuts;
    if (parts > 1) {
        const uint64_t stride = (uint64_t)ctx->max_kv_chunks * 16;
        KB_TRY(hostpub_ensure(ctx, ctx->ppub, KB_PUB_HEAD + part_keys_off(parts) + (parts - 1) * stride, L.stream));
        const uint64_t epoch = ++ctx->ppub.epoch;
        KB_LAUNCH_S(ctx, L.stream, "k_partition_cut", (parts - 1) * 64,
                    (k_partition_cut<<<1, KB_PART_WARPS * 32, 0, L.stream>>>(
                        ctx->st, (const uint32_t *)L.d_sel.p, (const uint64_t *)L.d_slot.p, n, T, parts, stride, ctx->ppub.p,
                        epoch, (const unsigned int *)ctx->d_ctrs.p + 8)));
        KB_CUDA(ctx, cudaGetLastError());
        KB_TRY(hostpub_wait(ctx, ctx->ppub, epoch, L.stream, "range partitions"));
        KB_TRY(pub_err_check(ctx, ctx->ppub));
        const uint64_t *h = ctx->ppub.payload<const uint64_t>();
        const uint8_t *keys = ctx->ppub.payload<const uint8_t>() + part_keys_off(parts);
        uint64_t prev = 0;
        for (uint64_t k = 1; k < parts; k++) {
            const uint64_t *c = h + 4 * (k - 1);
            // no kv reaches the share, the same kv as the cut before, or a border not above the kv in front of it
            if (c[0] >= n || c[0] == prev || !c[3]) continue;
            const uint64_t i = c[0];
            cuts.push_back(Cut{i, c[1], keys + (k - 1) * stride, c[2]});
            prev = i;
        }
    }

    const uint64_t np = cuts.size() + 1;
    HeldResult res{ctx, kb_result_new(ResultKind::partitions, KB_OUT_HOST)};
    uint64_t nbytes = req->start_len + req->end_len;
    for (const Cut &c : cuts) nbytes += c.klen;
    KB_TRY(pool_get_host(ctx, (np + 2 + 2 * (np + 1)) * 8, &res.p->h_meta));
    KB_TRY(pool_get_host(ctx, nbytes + 16, &res.p->h_arena));
    uint64_t *key_off = (uint64_t *)res.p->h_meta.p, *kv_first = key_off + np + 2, *arena_first = kv_first + np + 1;
    uint8_t *bytes = (uint8_t *)res.p->h_arena.p;
    uint64_t w = 0;
    auto put = [&](const uint8_t *p, uint64_t len) {
        if (len) memcpy(bytes + w, p, len);
        w += len;
    };
    key_off[0] = 0;
    kv_first[0] = arena_first[0] = 0;
    put(req->start, req->start_len);
    for (uint64_t k = 0; k < cuts.size(); k++) {
        key_off[k + 1] = w;
        put(cuts[k].key, cuts[k].klen);
        kv_first[k + 1] = cuts[k].kv;
        arena_first[k + 1] = cuts[k].arena;
    }
    key_off[np] = w;
    put(req->end, req->end_len);
    key_off[np + 1] = w;
    kv_first[np] = n;
    arena_first[np] = T;
    res.p->n_parts = np;
    res.p->n_bytes = nbytes;
    *out = res.release();
    return KB_OK;
}

extern "C" int kb_range_partitions(kb_ctx *ctx, const kb_range_req *req, uint64_t part_bytes, uint64_t max_parts,
                                   kb_result **out)
{
    if (!ctx || !req || !out) return KB_EINVAL;
    *out = nullptr;
    if (part_bytes == 0 || max_parts == 0 || req->limit > 0) return KB_EINVAL;
    if ((!req->start && req->start_len) || (!req->end && req->end_len)) return KB_EINVAL;
    if (max_parts > KB_MAX_PARTS) return KB_ELIMIT;  // bounds the report at 4096 keys of the store's largest padded pair
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->loaded) return kb_fail(ctx, KB_ESTATE, "no store loaded");
    cudaSetDevice(ctx->device);
    return range_partitions_locked(ctx, req, part_bytes, max_parts, out);
}

extern "C" int kb_partition_view_get(const kb_result *res, kb_partition_view *v)
{
    if (!res || !v || res->kind != ResultKind::partitions) return KB_EINVAL;
    const uint64_t np = res->n_parts;
    const uint64_t *meta = (const uint64_t *)res->h_meta.p;
    v->n_parts = np;
    v->key_off = meta;
    v->kv_first = meta + np + 2;
    v->arena_first = meta + np + 2 + np + 1;
    v->bytes = (const uint8_t *)res->h_arena.p;
    v->n_bytes = res->n_bytes;
    return KB_OK;
}
