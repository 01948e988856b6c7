// kb_compact.cu -- scanner.Compact's sweep and compaction streams.
//   sweep               the scan core in compact mode (kb_scan.cu): decode .. k_place_victims on the lane stream
//   compaction stream   the sweep and k_victim_capture at open; per page k_page_cut (kb_page.cu) -> k_victim_jobs [S] ->
//                       k_gather [SG] (kb_copy.cu)
#include <algorithm>
#include <memory>

#include "kb_scan.cuh"

// ------------------------------------------------------------------------------------------------
// compaction sweep
// ------------------------------------------------------------------------------------------------
// scanner.Compact's sweep of [start, end) at rev on the current lane (the caller holds ctx->mu, the store is loaded).  With
// want_victims the ordered delete calls go to *vic, a pooled buffer of victim_idx u32 x cap then victim_class u8 x cap
// (cap = *cap_v; none when the interval holds no record).  Records the compact revision.
static int sweep_locked(kb_ctx *ctx, const uint8_t *start, uint64_t start_len, const uint8_t *end, uint64_t end_len,
                        uint64_t rev, uint64_t timeout_rev, int support_ttl, bool want_victims, DBuf *vic,
                        uint64_t *cap_v, ReqOut *ro, uint64_t *examined)
{
    KB_TRY(ctx_quiesce(ctx));
    ScanLane &L = ctx->lane();
    Resolved R;
    KB_TRY(resolve_interval(ctx, L, start, start_len, end, end_len, rev, R));
    const ScanMode mode{1, (!support_ttl && timeout_rev != 0) ? 1 : 0, timeout_rev, 0};
    // One pass writes the ordered delete calls, so their buffer is sized before the count is known: a record is the
    // target of at most two calls (superseded as somebody's prev + tombstone / deleted revision record at its own turn,
    // or one TTL call).  The buffer is pooled; the host copy is cut to the real count.
    const uint64_t nrec = R.n_records;
    *cap_v = 2 * nrec;
    uint32_t *vidx = nullptr;
    uint8_t *vcls = nullptr;
    if (want_victims && nrec) {
        KB_TRY(pool_get_dev(ctx, *cap_v * 5 + 64, vic));
        vidx = (uint32_t *)vic->p;
        vcls = (uint8_t *)(vidx + *cap_v);
    }
    const ReqOut *rows = nullptr;
    KB_TRY(scan_sync(ctx, L, R, mode, vidx != nullptr, &rows, vidx, vcls));
    *ro = *rows;
    *examined = R.reqs[0].hi - R.reqs[0].lo;
    // scan(compact=true) blindly stores the compact revision (checkCompactRace, scanner.go:596-604)
    ctx->compact_present = true;
    ctx->compact_rev = rev;
    return KB_OK;
}

extern "C" int kb_compact_sweep(kb_ctx *ctx, const uint8_t *start, uint64_t start_len, const uint8_t *end,
                                uint64_t end_len, uint64_t rev, uint64_t timeout_rev, int support_ttl, int out_mode,
                                kb_result **out)
{
    if (!ctx || !out) return KB_EINVAL;
    if (out_mode != KB_OUT_HOST && out_mode != KB_OUT_DEVICE && out_mode != KB_OUT_COUNT) return KB_EINVAL;
    *out = nullptr;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->loaded) return kb_fail(ctx, KB_ESTATE, "no store loaded");
    cudaSetDevice(ctx->device);
    HeldResult res{ctx, kb_result_new(ResultKind::compact_sweep, out_mode)};
    ReqOut ro;
    uint64_t cap_v = 0;
    KB_TRY(sweep_locked(ctx, start, start_len, end, end_len, rev, timeout_rev, support_ttl, out_mode != KB_OUT_COUNT,
                        &res.p->d_meta, &cap_v, &ro, &res.p->examined));
    const uint64_t nv = ro.total;
    res.p->n_victims = nv;
    res.p->count = ro.total_aux;
    res.p->vic_cap = cap_v;
    if (out_mode == KB_OUT_HOST) {
        const uint32_t *vidx = (const uint32_t *)res.p->d_meta.p;
        KB_TRY(result_to_host(ctx, res.p, ctx->lane().stream, {{vidx, nv * 4}, {vidx + cap_v, nv}}, 0,
                              "compact sweep: victims D2H"));
    }
    *out = res.release();
    return KB_OK;
}

extern "C" int kb_compact_view_get(const kb_result *res, kb_compact_view *v)
{
    if (!res || !v || res->kind != ResultKind::compact_sweep) return KB_EINVAL;
    memset(v, 0, sizeof(*v));
    v->n_victims = res->n_victims;
    v->count = res->count;
    v->examined = res->examined;
    v->on_device = res->out_mode == KB_OUT_DEVICE;
    const uint8_t *base = v->on_device ? (const uint8_t *)res->d_meta.p : (const uint8_t *)res->h_meta.p;
    if (base && res->out_mode != KB_OUT_COUNT) {
        v->victim_idx = (const uint32_t *)base;
        // device-resident answers keep the capacity-sized layout the sweep wrote into; the host copy is compact
        v->victim_class = base + (v->on_device ? res->vic_cap : res->n_victims) * 4;
    }
    return KB_OK;
}

// ------------------------------------------------------------------------------------------------
// compaction streams: the sweep's victims handed out as internal keys (+ guards), page by page
// ------------------------------------------------------------------------------------------------
// At open every victim gets its heap location (VictimLoc) and its arena offset (an exclusive scan of the entry sizes).
// The heap only grows while a stream is open (kb_apply_batch / kb_expire append at the slab tails and defer the layout
// compaction), so these offsets address the same bytes on every page, however the directory has changed since.  A page is
// cut by k_page_cut over the arena offsets, k_victim_jobs turns its locations into GatherJobs, k_gather copies them.
namespace {

struct VictimLoc {    // 16 bytes; the victim's arena offset is kept beside it (24 bytes per victim)
    uint64_t vk;      // value chunk (classes 3 / 4, else 0) << 16 | key length
    uint32_t koff16;  // key chunk
    uint32_t vlen;    // guard length: the value's length for classes 3 / 4, else 0
};
static_assert(sizeof(VictimLoc) == 16, "VictimLoc is two 8-byte words");

// look-back state of a capture tile: flag in the top two bits, byte count below
constexpr unsigned long long VT_AGG = 1ull << 62, VT_PREFIX = 2ull << 62, VT_VAL = (1ull << 62) - 1;

// Thread per victim (four per thread, 1024 per tile; tiles in ticket order): the heap location of victim i's key (and, for
// classes 3 / 4, of its value: the guard) into loc[i], and its arena offset into off[i] -- an exclusive scan of the entry
// sizes pad16(key) + pad16(guard) by decoupled look-back over the tiles (warp 0 reads the states of 32 preceding tiles per
// step until it meets an inclusive prefix).  off[n] = the arena bytes of all victims.
__global__ void __launch_bounds__(256)
k_victim_capture(StoreDev st, const uint32_t *__restrict__ vidx, const uint8_t *__restrict__ vcls, uint64_t n,
                 VictimLoc *__restrict__ loc, uint64_t *__restrict__ off, unsigned long long *__restrict__ tstate,
                 unsigned int *__restrict__ ticket)
{
    __shared__ uint64_t ws2[18];
    __shared__ uint64_t tile_s, excl_s;
    if (threadIdx.x == 0) tile_s = atomicAdd(ticket, 1u);
    __syncthreads();
    const uint64_t t = tile_s;
    const uint64_t i0 = t * 1024 + threadIdx.x * 4;
    uint64_t sz[4], sum = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        sz[k] = 0;
        const uint64_t i = i0 + k;
        if (i < n) {
            const uint32_t rec = vidx[i], c = vcls[i];
            const bool guard = c == KB_V_REVRECORD || c == KB_V_TTL_REVREC;
            const uint32_t kl = st.klen[rec], vl = guard ? st.vlen[rec] : 0;
            VictimLoc v;
            v.vk = (guard ? st.voff16[rec] << 16 : 0) | kl;
            v.koff16 = st.koff16[rec];
            v.vlen = vl;
            loc[i] = v;
            sz[k] = pad16(kl) + (((uint64_t)vl + 15) & ~15ull);
            sum += sz[k];
        }
    }
    uint64_t ea, eb, ta, tb;
    block_excl_scan2(sum, 0, ea, eb, ta, tb, ws2);
    if (threadIdx.x < 32) {
        const uint32_t lane = threadIdx.x;
        volatile unsigned long long *ts = (volatile unsigned long long *)tstate;
        uint64_t excl = 0;
        if (t > 0) {
            if (lane == 0) ts[t] = VT_AGG | ta;
            for (uint64_t hi = t; hi > 0;) {  // tiles hi-1, hi-2, .. (lane 0 = nearest)
                const bool in = lane < hi;
                unsigned long long w;
                do {
                    w = VT_PREFIX;  // lanes past tile 0 stop nothing: their value does not count
                    if (in) w = ts[hi - 1 - lane];
                } while (!__all_sync(FULL, (w & ~VT_VAL) != 0));
                const unsigned pre = __ballot_sync(FULL, in && (w & ~VT_VAL) == VT_PREFIX);
                const uint32_t k = pre ? (uint32_t)(__ffs(pre) - 1) : 31u;  // nearest inclusive prefix
                uint64_t v = (in && lane <= k) ? (uint64_t)(w & VT_VAL) : 0;
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULL, v, d);
                excl += v;
                if (pre) break;
                hi -= hi < 32 ? hi : 32;
            }
        }
        if (lane == 0) {
            ts[t] = VT_PREFIX | (excl + ta);
            excl_s = excl;
        }
    }
    __syncthreads();
    uint64_t o = excl_s + ea;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const uint64_t i = i0 + k;
        if (i < n) {
            off[i] = o;
            o += sz[k];
            if (i == n - 1) off[n] = o;
        }
    }
}

// the per-victim arrays of a page (device, then copied as they are into the page's host layout)
struct VictimOut {
    uint64_t *key_off, *guard_off;
    uint32_t *key_len, *guard_len;
};

// Thread per victim of the page [a, a + nk): one GatherJob (the key's chunks, then the guard's) placed at off[i] - off[a],
// and the view's offsets and lengths.  The page's job table (count, work counter) is k_page_cut's.
__global__ void __launch_bounds__(256)
k_victim_jobs(const VictimLoc *__restrict__ loc, const uint64_t *__restrict__ off, uint64_t a, uint64_t nk,
              GatherJob *__restrict__ jobs, VictimOut out)
{
    const uint64_t base = off[a];
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < nk; k += (uint64_t)gridDim.x * blockDim.x) {
        const VictimLoc v = loc[a + k];
        const uint64_t dst = off[a + k] - base;
        const uint32_t kl = (uint32_t)(v.vk & 0xFFFFu);
        GatherJob j;
        j.dst16 = dst >> 4;
        j.vsrc16 = v.vk >> 16;
        j.ksrc16 = v.koff16;
        j.nk = (kl + 15) >> 4;
        j.nv = (uint32_t)(((uint64_t)v.vlen + 15) >> 4);
        j.kl = kl;
        jobs[k] = j;
        out.key_off[k] = dst;
        out.key_len[k] = kl;
        out.guard_off[k] = dst + (uint64_t)j.nk * 16;
        out.guard_len[k] = v.vlen;
    }
}

}  // namespace

struct kb_compact_stream : PageStream {  // n: the sweep's victims
    uint64_t count = 0, examined = 0;  // the sweep's count and examined records
    // n victims: arena offset u64 (n + 1) | VictimLoc | record u32 | class u8
    DBuf d;
    uint64_t *off() const { return (uint64_t *)d.p; }
    VictimLoc *loc() const { return (VictimLoc *)(off() + n + 1); }
    uint32_t *vidx() const { return (uint32_t *)(loc() + n); }
    uint8_t *vcls() const { return (uint8_t *)(vidx() + n); }
    const char *invalid = nullptr;  // the entry point that rewrote the heap since the open
};

static void cstream_free(kb_compact_stream *s)
{
    if (s->d.p) cudaFree(s->d.p);
    hostpub_free(s->pub);
    delete s;
}

bool compact_streams_pin_heap(const kb_ctx *ctx)
{
    for (const kb_compact_stream *s : ctx->cstreams)
        if (!s->invalid) return true;
    return false;
}

void compact_streams_invalidate(kb_ctx *ctx, const char *what)
{
    for (kb_compact_stream *s : ctx->cstreams) s->invalid = what;
}

void kb_stream_drop_all(kb_ctx *ctx)
{
    for (kb_range_stream *s : ctx->streams) stream_free(s);
    ctx->streams.clear();
    for (kb_compact_stream *s : ctx->cstreams) cstream_free(s);
    ctx->cstreams.clear();
}

// the sweep's n victims (vic: victim_idx u32 x cap_v | victim_class u8 x cap_v) -> the stream's arrays, with every
// victim's heap location and arena offset; the lane is free again when this returns
static int victims_capture(kb_ctx *ctx, kb_compact_stream *s, const DBuf &vic, uint64_t cap_v, uint64_t n)
{
    s->n = n;
    if (n == 0) return KB_OK;
    ScanLane &L = ctx->lane();
    const size_t bytes = (n + 1) * 8 + n * (sizeof(VictimLoc) + 5) + 64;
    KB_CUDA(ctx, cudaMalloc(&s->d.p, bytes));  // exact: it lives as long as the stream
    s->d.cap = bytes;
    KB_CUDA(ctx, cudaMemcpyAsync(s->vidx(), vic.p, n * 4, cudaMemcpyDeviceToDevice, L.stream));
    KB_CUDA(ctx, cudaMemcpyAsync(s->vcls(), (const uint8_t *)vic.p + cap_v * 4, n, cudaMemcpyDeviceToDevice, L.stream));
    const uint64_t ntiles = (n + 1023) / 1024;
    DBuf scratch;  // ticket, then one look-back state per tile
    KB_TRY(pool_get_dev(ctx, 16 + ntiles * 8, &scratch));
    int rc = KB_OK;
    do {
        if (cudaMemsetAsync(scratch.p, 0, 16 + ntiles * 8, L.stream) != cudaSuccess) {
            rc = kb_fail(ctx, KB_ECUDA, "compaction stream: scratch");
            break;
        }
        // per victim: record and class read, four directory entries gathered, 24 bytes written
        KB_LAUNCH_S(ctx, L.stream, "k_victim_capture", n * 47,
                    (k_victim_capture<<<(unsigned)ntiles, 256, 0, L.stream>>>(
                        ctx->st, s->vidx(), s->vcls(), n, s->loc(), s->off(),
                        (unsigned long long *)((uint8_t *)scratch.p + 16), (unsigned int *)scratch.p)));
        rc = hbuf_ensure(ctx, L.h_stage, 64);
        if (rc != KB_OK) break;
        cudaMemcpyAsync(L.h_stage.p, s->off() + n, 8, cudaMemcpyDeviceToHost, L.stream);
        const cudaError_t e = cudaStreamSynchronize(L.stream);
        if (e != cudaSuccess) {
            rc = kb_cuda_fail(ctx, e, "compaction stream: victim capture");
            break;
        }
        s->total = *(const uint64_t *)L.h_stage.p;
    } while (0);
    pool_put_dev(ctx, scratch);
    return rc;
}

extern "C" int kb_compact_stream_open(kb_ctx *ctx, const uint8_t *start, uint64_t start_len, const uint8_t *end,
                                      uint64_t end_len, uint64_t rev, uint64_t timeout_rev, int support_ttl,
                                      uint64_t group_victims, kb_compact_stream **out)
{
    if (!ctx || !out) return KB_EINVAL;
    *out = nullptr;
    if (group_victims == 0 || (!start && start_len) || (!end && end_len)) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->loaded) return kb_fail(ctx, KB_ESTATE, "no store loaded");
    cudaSetDevice(ctx->device);
    std::unique_ptr<kb_compact_stream, void (*)(kb_compact_stream *)> s(new kb_compact_stream(), cstream_free);
    s->group = group_victims;
    KB_TRY(hostpub_ensure(ctx, s->pub, KB_PAGE_PUB_KEY, ctx->lane().stream));
    DBuf vic;
    uint64_t cap_v = 0;
    ReqOut ro;
    int rc = sweep_locked(ctx, start, start_len, end, end_len, rev, timeout_rev, support_ttl, true, &vic, &cap_v, &ro,
                          &s->examined);
    if (rc == KB_OK) rc = victims_capture(ctx, s.get(), vic, cap_v, ro.total);
    pool_put_dev(ctx, vic);
    KB_TRY(rc);
    s->count = ro.total_aux;
    ctx->cstreams.push_back(s.get());
    *out = s.release();
    return KB_OK;
}

extern "C" int kb_compact_stream_info(const kb_compact_stream *s, uint64_t *n_victims, uint64_t *count, uint64_t *examined)
{
    if (!s) return KB_EINVAL;
    if (n_victims) *n_victims = s->n;
    if (count) *count = s->count;
    if (examined) *examined = s->examined;
    return KB_OK;
}

// the host layout of a page's per-victim arrays: key_off u64 | guard_off u64 | key_len u32 | guard_len u32 (the first 24
// bytes per victim are k_victim_jobs' device layout, copied as they are) | record u32 | class u8
static VictimOut victim_out_at(void *p, uint64_t nk)
{
    VictimOut o;
    o.key_off = (uint64_t *)p;
    o.guard_off = o.key_off + nk;
    o.key_len = (uint32_t *)(o.guard_off + nk);
    o.guard_len = o.key_len + nk;
    return o;
}

extern "C" int kb_compact_stream_next(kb_ctx *ctx, kb_compact_stream *s, uint64_t max_bytes, kb_result **page)
{
    if (!ctx || !s || !page) return KB_EINVAL;
    *page = nullptr;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (s->invalid)
        return kb_fail(ctx, KB_ESTATE, "compaction stream: %s rewrote the snapshot since the stream was opened; its victims "
                                       "can no longer be copied (close it and sweep again)", s->invalid);
    if (s->pos >= s->n) return KB_OK;
    cudaSetDevice(ctx->device);
    kb_tp tseg = kb_now();
    PageCut c;
    KB_TRY(page_cut(ctx, *s, nullptr, s->off(), max_bytes, "compaction stream", tseg, &c));
    JobSet &J = *c.J;
    ScanLane &L = ctx->lane();
    const uint64_t nk = c.end - s->pos, nbytes = c.bytes;

    HeldResult res{ctx, nullptr};
    KB_TRY(answer_new(ctx, res, ResultKind::compact_page, KB_OUT_HOST, 0, 0, nbytes + 64));
    KB_TRY(pool_get_dev(ctx, nk * 24 + 64, &res.p->d_meta));
    KB_TRY(dbuf_ensure(ctx, J.gjobs, nk * sizeof(GatherJob)));
    GatherJob *d_gj = (GatherJob *)J.gjobs.p;
    const unsigned jgrid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((nk + 255) / 256, (uint64_t)ctx->n_sms * 8));
    KB_LAUNCH_S(ctx, L.stream, "k_victim_jobs", nk * 72,
                (k_victim_jobs<<<jgrid, 256, 0, L.stream>>>(s->loc(), s->off(), s->pos, nk, d_gj,
                                                           victim_out_at(res.p->d_meta.p, nk))));
    KB_TRY(copy_after_jobs(ctx, L, ctx->stream_g));
    KB_TRY(launch_gather(ctx, ctx->stream_g, d_gj, jobtab_at(J.jobs.p, 1), (uint4 *)res.p->d_arena.p, nk, 2 * nbytes));
    KB_TRY(copy_done(ctx, ctx->stream_g, J.ev_gather, res.p));

    // the host copy, on the host-copy stream behind the gather (which waited for the per-victim arrays)
    const int rc = result_to_host(ctx, res.p, ctx->stream_h,
                                  {{res.p->d_meta.p, nk * 24}, {s->vidx() + s->pos, nk * 4}, {s->vcls() + s->pos, nk}},
                                  nbytes, "compaction page D2H");
    kb_seg(ctx, "host:compact_page_d2h", tseg);
    KB_TRY(rc);
    res.p->first = s->pos;
    res.p->n_victims = nk;
    res.p->n_bytes = nbytes;
    s->pos = c.end;
    *page = res.release();
    return KB_OK;
}

extern "C" void kb_compact_stream_close(kb_ctx *ctx, kb_compact_stream *s)
{
    if (!ctx || !s) return;
    std::lock_guard<std::mutex> g(ctx->mu);
    auto it = std::find(ctx->cstreams.begin(), ctx->cstreams.end(), s);
    if (it == ctx->cstreams.end()) return;
    ctx->cstreams.erase(it);
    cudaSetDevice(ctx->device);
    cstream_free(s);  // every kernel that read its arrays ended before the page that launched it was returned
}

extern "C" int kb_compact_page_view_get(const kb_result *res, kb_compact_page_view *v)
{
    if (!res || !v || res->kind != ResultKind::compact_page) return KB_EINVAL;
    memset(v, 0, sizeof(*v));
    const uint64_t n = res->n_victims;
    v->first = res->first;
    v->n = n;
    const VictimOut o = victim_out_at(res->h_meta.p, n);
    v->key_off = o.key_off;
    v->guard_off = o.guard_off;
    v->key_len = o.key_len;
    v->guard_len = o.guard_len;
    v->rec_idx = o.guard_len + n;
    v->victim_class = (const uint8_t *)(v->rec_idx + n);
    v->bytes = (const uint8_t *)res->h_arena.p;
    v->n_bytes = res->n_bytes;
    return KB_OK;
}
