// kb_batch.cu -- lane batches: range batches and point reads, each launched on the current lane and collected with one
// host wait on its published rows (streams: S2 = bound search, S = lane, SG = copy stream).
//   range batch  k_search [S2] -> the scan core (kb_scan.cu) [S] -> k_req_finalize [S] -> the copy (kb_copy.cu): jobs [S],
//                copy [SG], which overlaps the next batch's scan; count-only and empty answers publish with k_publish_rout
//   point reads  k_search -> k_get_resolve -> k_get_finalize -> k_gather (or k_wire_jobs -> k_wire_copy) -> k_publish_rout,
//                all on the lane stream (backend.get, pkg/backend/range.go:81-121)
#include <algorithm>
#include <memory>
#include <string_view>

#include "kb_scan.cuh"
#include "kb_wire.cuh"

namespace {

// ---- k_get_resolve: one warp per point read.  cand = (first record > EncodeObjectKey(key, revision)) - 1 is what the
// reference's reverse iterator yields first (range.go:97-107); it answers the read iff it decodes to the same user
// key with a non-zero revision (range.go:109-117); a tombstone value maps to ErrKeyNotFound (range.go:82-86).
struct GetOut {
    uint8_t *status;
    uint64_t *mod_rev;
    uint64_t *voff16;  // value slab chunk of the answering record (k_get_finalize builds the copy jobs from it)
    uint32_t *rec;
    uint32_t *vlen;
};

__global__ void __launch_bounds__(128)
k_get_resolve(StoreDev st, BoundsDev bounds, const uint32_t *__restrict__ ub, GetOut out)
{
    const uint32_t g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (g >= bounds.n) return;
    const uint32_t idx = ub[g];
    uint32_t status = KB_GET_NOT_FOUND, rec = 0, vl = 0;
    uint64_t mrev = 0, vo = 0;
    if (idx > 0) {
        rec = idx - 1;
        const uint32_t bl = bounds.len(g);     // magic + key + '$' + rev(8) + one 0x00 byte
        const uint32_t pre = bl - 9;           // magic + key + '$'
        const uint32_t kl = st.klen[rec];
        if (kl == pre + 8) {
            const uint4 *a = st.kslab + st.koff16[rec];
            if (warp_prefix_eq(a, bounds, g, pre)) {
                mrev = be64_bytes((const uint8_t *)a + kl - 8);
                if (mrev != 0) {
                    vl = st.vlen[rec];
                    vo = st.voff16[rec];
                    status = KB_GET_FOUND;
                    if (vl == 9) {
                        const uint4 v0 = st.vslab[vo];
                        if (v0.x == 0x626d6f74u && v0.y == 0x6e6f7473u && (v0.z & 0xffu) == 0x65u) status = KB_GET_TOMBSTONE;
                    }
                }
            }
        }
    }
    if (lane == 0) {
        out.status[g] = (uint8_t)status;
        out.mod_rev[g] = status == KB_GET_NOT_FOUND ? 0 : mrev;
        out.voff16[g] = vo;
        out.rec[g] = rec;
        out.vlen[g] = vl;
    }
}

// The per-read rows of a point-read batch: one layout on the device (k_get_resolve and k_get_finalize write it) and in
// the result's pinned host copy: [arena bytes u64][status u8 n, padded to 8][mod_rev u64 n][val_off u64 n][rec u32 n]
// [val_len u32 n][elem_off u64 n + 1, wire mode only]
struct GetRows {
    uint64_t *n_bytes;
    uint8_t *status;
    uint64_t *mod_rev, *val_off;
    uint32_t *rec, *val_len;
    uint64_t *elem_off;  // nullptr outside the wire mode
};

size_t get_rows_bytes(uint64_t n, bool wire) { return 8 + ((n + 7) & ~7ull) + 24 * n + (wire ? 8 * (n + 1) : 0); }

GetRows get_rows_at(void *base, uint64_t n, bool wire)
{
    GetRows r;
    r.n_bytes = (uint64_t *)base;
    r.status = (uint8_t *)base + 8;
    r.mod_rev = (uint64_t *)(r.status + ((n + 7) & ~7ull));
    r.val_off = r.mod_rev + n;
    r.rec = (uint32_t *)(r.val_off + n);
    r.val_len = r.rec + n;
    r.elem_off = wire ? (uint64_t *)(r.val_len + n) : nullptr;
    return r;
}

// single CTA: the arena of a point-read batch.  A read has an arena entry iff it is FOUND: its value padded to 16 bytes
// (raw modes, kb_get_batch's values-only arena) or its RangeResponse.kvs element (wire mode).  Loops over the reads in
// chunks of 256 with a block scan and a carry, as k_req_finalize does: compacts the FOUND reads, places each entry, and
// turns the resolve rows into the answer's rows (val_off, the value slab chunk until now, becomes the arena offset of the
// value; a missing read's val_len is cleared).  Raw modes: one values-only GatherJob per FOUND read (k_gather).  Wire
// mode: the selection and arena offsets for k_wire_jobs / k_wire_copy.  Both: a one-request job table over the FOUND reads.
__global__ void __launch_bounds__(256, 8)  // <= 32 registers: eight CTAs per SM, room for other lanes' batches beside the copy
k_get_finalize(StoreDev st, GetRows rows, uint32_t n, int wire, GatherJob *__restrict__ gjobs, uint32_t *__restrict__ sel,
               uint64_t *__restrict__ slot, uint64_t *__restrict__ jobtab)
{
    __shared__ uint64_t ws2[18];
    __shared__ uint64_t carry[2];
    if (threadIdx.x == 0) carry[0] = carry[1] = 0;
    __syncthreads();
    for (uint32_t c0 = 0; c0 < n; c0 += 256) {
        const uint32_t i = c0 + threadIdx.x;
        uint32_t status = KB_GET_NOT_FOUND, vl = 0;
        uint64_t size = 0;
        if (i < n) {
            status = rows.status[i];
            vl = rows.val_len[i];
            if (status == KB_GET_FOUND)
                size = wire ? wire_sizes(st.klen[rows.rec[i]] - 13, vl, rows.mod_rev[i], KB_WIRE_KVS_I).elem : pad16(vl);
        }
        const bool found = status == KB_GET_FOUND;
        uint64_t ek, eo, tk, to;
        block_excl_scan2(found ? 1 : 0, size, ek, eo, tk, to, ws2);
        const uint64_t k = carry[0] + ek, off = carry[1] + eo;
        if (i < n) {
            if (found && wire) {
                sel[k] = rows.rec[i];
                slot[k] = off;
            } else if (found) {
                GatherJob j;
                j.dst16 = off >> 4;
                j.vsrc16 = rows.val_off[i];
                j.ksrc16 = 0;
                j.nk = 0;
                j.nv = (vl + 15) >> 4;
                j.kl = 0;
                gjobs[k] = j;
            }
            rows.val_off[i] = found ? (wire ? off + size - vl : off) : 0;  // the value ends the element
            if (status == KB_GET_NOT_FOUND) rows.val_len[i] = 0;
            if (wire) rows.elem_off[i] = off;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            carry[0] += tk;
            carry[1] += to;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const uint64_t bytes = carry[1];
        *rows.n_bytes = bytes;
        if (wire) rows.elem_off[n] = bytes;
        jobtab_write_one(jobtab, carry[0], 0, bytes, 0);
    }
}

// The per-request rows are the only thing the host needs before it can return a device-resident answer: the device
// stores them into the lane's HostPub, with the context's error flag as the error word, and then raises the epoch flag;
// the host polls the flag -- no copy, no stream synchronisation, and the gather that follows keeps running after the
// call has returned.
__device__ __forceinline__ void publish_rout(const ReqOut *__restrict__ rout, uint32_t nreq, uint8_t *host, uint64_t epoch,
                                             const unsigned int *err_flag)
{
    const uint4 *src = (const uint4 *)rout;
    uint4 *dst = (uint4 *)(host + KB_PUB_HEAD);
    for (uint32_t i = threadIdx.x; i < nreq * 2; i += blockDim.x) dst[i] = src[i];
    if (threadIdx.x == 0) *(volatile uint64_t *)(host + 8) = *err_flag;  // a bulk copy of an earlier batch never completed
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) pub_raise(host, epoch);
}

__global__ void __launch_bounds__(256) k_publish_rout(const ReqOut *__restrict__ rout, uint32_t nreq, uint8_t *host,
                                                      uint64_t epoch, const unsigned int *err_flag)
{
    publish_rout(rout, nreq, host, epoch, err_flag);
}

// single CTA: per-request emitted count / response bytes (limit applied) and their exclusive prefixes over the
// requests, written as the batch's job table
__global__ void __launch_bounds__(256, 8)  // <= 32 registers: eight CTAs per SM, room for other lanes' batches beside the copy
k_req_finalize(const ReqDev *__restrict__ reqs, uint32_t nreq, const ReqOut *__restrict__ rout, JobTable tab,
               uint8_t *host_rout, uint64_t epoch, const unsigned int *__restrict__ err_flag)
{
    uint64_t *__restrict__ job_first = tab.job_first, *__restrict__ arena_base = tab.arena_base;
    if (threadIdx.x == 0) *tab.work_ctr = 0;  // the gather's block counter
    __shared__ uint64_t ws2[18];
    __shared__ uint64_t carry[2];
    if (threadIdx.x == 0) carry[0] = carry[1] = 0;
    __syncthreads();
    for (uint32_t c0 = 0; c0 < nreq; c0 += 256) {
        const uint32_t q = c0 + threadIdx.x;
        uint64_t ne = 0, nb = 0;
        if (q < nreq) {
            const ReqOut o = rout[q];
            const int64_t lim = reqs[q].limit;
            ne = (lim > 0 && o.total > (uint64_t)lim) ? (uint64_t)lim : o.total;
            nb = (lim > 0 && (o.flags & KB_RO_CAPPED)) ? o.capped_aux : o.total_aux;
        }
        uint64_t ea, eb, ta, tb;
        block_excl_scan2(ne, nb, ea, eb, ta, tb, ws2);
        const uint64_t ca = carry[0], cb = carry[1];
        if (q < nreq) {
            job_first[q] = ca + ea;
            arena_base[q] = cb + eb;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            carry[0] = ca + ta;
            carry[1] = cb + tb;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        job_first[nreq] = carry[0];
        arena_base[nreq] = carry[1];
    }
    publish_rout(rout, nreq, host_rout, epoch, err_flag);
}

}  // namespace

static_assert(sizeof(ReqOut) == 32, "publish_rout copies ReqOut rows as two 16-byte words");

// checkCompactRace (scanner.go:594-626): a read below the compact revision fails, with the text of the range path
int compact_race_check(kb_ctx *ctx, uint64_t rev)
{
    if (ctx->compact_present && ctx->compact_rev > rev)
        return kb_fail(ctx, KB_ECOMPACTED, "range stream revision %llu less than compact revision %llu",
                       (unsigned long long)rev, (unsigned long long)ctx->compact_rev);
    return KB_OK;
}

// a range or point-read batch between its submission and the collection of its answer
struct kb_pending {
    bool get = false;          // a point-read batch (kb_get_submit): its rows are copied into res->h_meta before they publish
    ScanLane *lane = nullptr;  // the lane it was submitted on: its rows arrive in lane->rows
    Resolved R;
    uint64_t nreq = 0;
    int out_mode = 0, wire = 0;
    bool want_kvs = false;
    kb_result *res = nullptr;  // owns the answer's buffers
    GatherOut go;              // the per-kv arrays (res->d_meta)
    uint64_t *d_elem_off = nullptr;
    uint64_t epoch = 0;        // of its publish; 0: the batch launched none
    kb_tp t_submit;
    std::vector<ReqOut> rout;         // rows, once read back
    bool harvested = false;
    int harvest_rc = KB_OK;
};
static int pending_harvest(kb_ctx *ctx, kb_pending *P);
static void pending_drop(kb_ctx *ctx, kb_pending *P);

using HeldPending = Held<kb_pending, pending_drop>;

// first half of a range call: everything up to the launch of the last kernel; the batch is then in flight on lane L (the
// current lane)
static int range_submit_locked(kb_ctx *ctx, ScanLane &L, const kb_range_req *reqs, uint64_t nreq, int out_mode, kb_pending **out)
{
    // wire modes: the arena holds etcd protobuf elements instead of padded [key][value] pairs (kb_wire.cuh)
    int wire = 0;
    KB_TRY(split_out_mode(out_mode, &out_mode, &wire));
    if (out_mode != KB_OUT_HOST && out_mode != KB_OUT_DEVICE && out_mode != KB_OUT_COUNT) return KB_EINVAL;
    if (wire && out_mode == KB_OUT_COUNT) return KB_EINVAL;
    *out = nullptr;
    if (!ctx->loaded) return kb_fail(ctx, KB_ESTATE, "no store loaded");
    cudaSetDevice(ctx->device);
    KB_TRY(lane_take(ctx));
    for (uint64_t q = 0; q < nreq; q++) KB_TRY(compact_race_check(ctx, reqs[q].read_rev));
    kb_tp tseg = kb_now();
    std::unique_ptr<kb_pending> P(new kb_pending());
    Resolved &R = P->R;
    KB_TRY(resolve_requests(ctx, L, reqs, nreq, true, R, &tseg));
    kb_seg(ctx, "host:range_layout", tseg);
    bool probe_is_final = false;
    if (out_mode != KB_OUT_COUNT) {
        KB_TRY(probe_limit_windows(ctx, L, R, wire, &probe_is_final));
        kb_seg(ctx, "host:range_limit_probe", tseg);
    }
    if (!probe_is_final) {
        KB_TRY(upload_layout(ctx, L, R));
        KB_TRY(sel_ensure(ctx, L, R));
        KB_TRY(launch_scan_core(ctx, L, R, ScanMode::range(wire), out_mode != KB_OUT_COUNT));
    }
    const ReqDev *d_reqs = (const ReqDev *)L.d_reqs.p;
    ReqOut *d_rout = (ReqOut *)L.d_reqout.p;
    KB_TRY(hostpub_ensure(ctx, L.rows, KB_PUB_HEAD + std::max<uint64_t>(nreq, 1) * sizeof(ReqOut), L.stream));
    const uint64_t epoch = nreq ? ++L.rows.epoch : 0;  // an empty batch publishes nothing

    // Response arena: sized by an upper bound the host knows without a round trip (all key+value bytes of the examined
    // record intervals), so the gather is enqueued right behind the placement and the only synchronisation left is
    // the final one (the arena is pooled, so steady-state calls reuse it).
    const bool want_kvs = out_mode != KB_OUT_COUNT && R.total_sel > 0;
    // (a heap has no "bytes of an interval": every examined record could be emitted with the store's largest pair, and
    // no answer can exceed one copy of everything per request that could return it all)
    uint64_t ub_bytes = 0;
    for (auto &r : R.reqs) {
        uint64_t cap = (uint64_t)(r.hi - r.lo);
        if (r.limit > 0) cap = std::min<uint64_t>(cap, (uint64_t)r.limit);
        ub_bytes += std::min<uint64_t>(cap * ctx->max_kv_chunks, ctx->kused16 + ctx->vused16) * 16;
    }
    // a wire element is at most 48 bytes of tags / varints longer than its key + value (and the key loses 13)
    if (wire) ub_bytes += (uint64_t)R.total_sel * 48;
    GatherOut go;
    memset(&go, 0, sizeof(go));
    const uint64_t cap_kvs = R.total_sel;
    uint64_t *d_elem_off = nullptr;
    // every early return below hands the pooled buffers back (the stream keeps later reuse ordered behind this call)
    HeldResult res{ctx, nullptr};
    KB_TRY(answer_new(ctx, res, ResultKind::range, out_mode, wire, cap_kvs, want_kvs ? ub_bytes + 64 : 0, &go,
                      &d_elem_off));
    // The copy into the arena runs on the gather stream.  Consecutive batches alternate between two sets of job
    // buffers, so this batch's job construction (main stream) may overlap the previous batch's copy; it only has to
    // wait for the copy that last READ this set (two batches ago).
    JobSet &J = ctx->jobsets[ctx->batch_seq++ & 1];
    if (want_kvs) {
        KB_TRY(dbuf_ensure(ctx, J.jobs, jobtab_bytes(nreq)));
        KB_TRY(dbuf_ensure(ctx, J.gjobs, copy_jobs_bytes(std::max<uint64_t>(cap_kvs, 1), wire)));
        const JobTable tab = jobtab_at(J.jobs.p, nreq);  // its work counter is zeroed by k_req_finalize
        KB_CUDA(ctx, cudaStreamWaitEvent(L.stream, J.ev_gather, 0));
        KB_LAUNCH_S(ctx, L.stream, "k_req_finalize", nreq * 64,
                    (k_req_finalize<<<1, 256, 0, L.stream>>>(d_reqs, (uint32_t)nreq, d_rout, tab, L.rows.p, epoch,
                                                             (const unsigned int *)ctx->d_ctrs.p + 8)));
        KB_TRY(launch_copy(ctx, L, ctx->stream_g, J.gjobs.p, J.ev_gather, d_reqs, (uint32_t)nreq, tab,
                           (const uint32_t *)L.d_sel.p, (const uint64_t *)L.d_slot.p, cap_kvs, wire, go, d_elem_off, res.p));
    } else if (nreq) {  // count-only / empty answers: nothing ran k_req_finalize, publish the rows directly
        KB_LAUNCH_S(ctx, L.stream, "k_publish_rout", nreq * 32,
                    (k_publish_rout<<<1, 256, 0, L.stream>>>(d_rout, (uint32_t)nreq, L.rows.p, epoch,
                                                             (const unsigned int *)ctx->d_ctrs.p + 8)));
    }
    kb_seg(ctx, "host:range_launch", tseg);
    P->lane = &L;
    P->nreq = nreq;
    P->out_mode = out_mode;
    P->wire = wire;
    P->want_kvs = want_kvs;
    P->res = res.release();
    P->go = go;
    P->d_elem_off = d_elem_off;
    P->epoch = epoch;
    P->t_submit = tseg;
    L.pending = P.get();
    *out = P.release();
    return KB_OK;
}

// wait for the rows of a submitted batch and keep them with it: afterwards the lane's buffers are free again
static int pending_harvest(kb_ctx *ctx, kb_pending *P)
{
    if (P->harvested) return P->harvest_rc;
    P->harvested = true;
    ScanLane &L = *P->lane;
    if (L.pending == P) L.pending = nullptr;
    if (P->epoch != 0) {
        P->harvest_rc = hostpub_wait(ctx, L.rows, P->epoch, L.stream, "range scan");
        if (P->harvest_rc != KB_OK) return P->harvest_rc;
        const ReqOut *rows = L.rows.payload<const ReqOut>();
        P->rout.assign(rows, rows + P->nreq);
        P->harvest_rc = pub_err_check(ctx, L.rows);
    }
    return P->harvest_rc;
}

int lane_take(kb_ctx *ctx)
{
    ScanLane &L = ctx->lane();
    return L.pending ? pending_harvest(ctx, L.pending) : KB_OK;
}

int kb_pending_harvest_all(kb_ctx *ctx)
{
    for (ScanLane &L : ctx->lanes)
        if (L.pending) KB_TRY(pending_harvest(ctx, L.pending));
    return KB_OK;
}

static void pending_drop(kb_ctx *ctx, kb_pending *P)
{
    if (P->lane->pending == P) P->lane->pending = nullptr;
    result_release_locked(ctx, P->res);
    delete P;
}

void kb_pending_drop_all(kb_ctx *ctx)  // kb_close: batches nobody collected
{
    for (ScanLane &L : ctx->lanes)
        if (kb_pending *P = L.pending) {
            pending_harvest(ctx, P);
            pending_drop(ctx, P);
        }
}

// second half: rows -> the result's per-request arrays, host copies for KB_OUT_HOST
static int range_collect_locked(kb_ctx *ctx, kb_pending *P, kb_result **out)
{
    *out = nullptr;
    cudaSetDevice(ctx->device);
    const uint64_t nreq = P->nreq;
    const int out_mode = P->out_mode, wire = P->wire;
    const bool want_kvs = P->want_kvs;
    Resolved &R = P->R;
    kb_result *res = P->res;
    GatherOut &go = P->go;
    uint64_t *d_elem_off = P->d_elem_off;
    kb_tp tseg = kb_now();
    HeldPending held{ctx, P};  // every return below ends the batch: a failed one hands its buffers back
    int rc = pending_harvest(ctx, P);
    if (rc != KB_OK) return rc;
    std::vector<ReqOut> &rout = P->rout;
    kb_seg(ctx, "host:range_sync", tseg);

    res->req_first.resize(nreq + 1);
    res->req_count.resize(nreq);
    res->req_examined.resize(nreq);
    uint64_t nk = 0, nbytes = 0;
    for (uint64_t q = 0; q < nreq; q++) {
        uint64_t ne = rout[q].total;
        bool capped = R.reqs[q].limit > 0 && ne > (uint64_t)R.reqs[q].limit;
        if (capped) ne = (uint64_t)R.reqs[q].limit;
        res->req_first[q] = nk;
        if (out_mode == KB_OUT_COUNT) {
            res->req_count[q] = rout[q].total;  // emptyResultReceiver never stops the loop
            res->req_examined[q] = R.reqs[q].hi - R.reqs[q].lo;
        } else {
            const bool stop = rout[q].flags & KB_RO_LIMIT_STOP;
            res->req_count[q] = stop ? 0 : ne;  // (0, nil) when the limit stopped the loop (Q4)
            res->req_examined[q] = stop ? rout[q].examined : R.reqs[q].hi - R.reqs[q].lo;
            nk += ne;
            nbytes += (R.reqs[q].limit > 0 && (rout[q].flags & KB_RO_CAPPED)) ? rout[q].capped_aux : rout[q].total_aux;
        }
    }
    res->req_first[nreq] = nk;
    res->n_kvs = nk;
    res->n_bytes = nbytes;
    if (ctx->prof_on) {  // the gather's algorithmic bytes are only known now
        int gi = prof_index(ctx, wire ? "k_wire_copy" : "k_gather");
        ctx->prof[gi].bytes += 2 * nbytes + nk * 40;
    }

    if (want_kvs && nk > 0) {
        rc = answer_finish(ctx, res, go, d_elem_off, nk, nbytes, tseg);
        if (rc != KB_OK) return rc;
    } else {
        result_put_device(ctx, res);
    }
    *out = res;
    delete held.release();
    kb_seg(ctx, "host:range_finish", tseg);
    return KB_OK;
}

extern "C" int kb_range_batch(kb_ctx *ctx, const kb_range_req *reqs, uint64_t nreq, int out_mode, kb_result **out)
{
    if (!ctx || !out || (nreq && !reqs)) return KB_EINVAL;
    *out = nullptr;
    std::lock_guard<std::mutex> g(ctx->mu);
    kb_pending *P = nullptr;
    KB_TRY(range_submit_locked(ctx, ctx->lane(), reqs, nreq, out_mode, &P));
    return range_collect_locked(ctx, P, out);
}

// The two halves on their own: a caller with a queue of batches submits batch n+1 before it collects batch n, so the
// host's part of n+1 (bound search round trip, layout, launches) and its first kernels overlap the kernels of n.  Each
// submission leaves its batch on the current lane and moves the context to the next one; KB_LANES batches in flight at
// most (a submission first reads back the rows of the batch that last used its lane).
extern "C" int kb_range_submit(kb_ctx *ctx, const kb_range_req *reqs, uint64_t nreq, int out_mode, kb_pending **out)
{
    if (!ctx || !out || (nreq && !reqs)) return KB_EINVAL;
    *out = nullptr;
    std::lock_guard<std::mutex> g(ctx->mu);
    KB_TRY(range_submit_locked(ctx, ctx->lane(), reqs, nreq, out_mode, out));
    lane_swap(ctx);
    return KB_OK;
}

extern "C" int kb_range_collect(kb_ctx *ctx, kb_pending *pending, kb_result **out)
{
    if (!ctx || !pending || !out) return KB_EINVAL;
    *out = nullptr;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (pending->get) return kb_fail(ctx, KB_EINVAL, "kb_range_collect: a point-read batch is collected by kb_get_collect");
    return range_collect_locked(ctx, pending, out);
}

// give up a submitted batch without reading its answer
extern "C" void kb_pending_free(kb_ctx *ctx, kb_pending *pending)
{
    if (!ctx || !pending) return;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaSetDevice(ctx->device);
    pending_harvest(ctx, pending);  // its kernels must be done before its buffers go back to the pools
    pending_drop(ctx, pending);
}

extern "C" int kb_range_view_get(const kb_result *res, kb_range_view *v)
{
    if (!res || !v || res->kind != ResultKind::range) return KB_EINVAL;
    memset(v, 0, sizeof(*v));
    v->n_req = res->req_count.size();
    v->req_first = res->req_first.data();
    v->req_count = res->req_count.data();
    v->req_examined = res->req_examined.data();
    v->n_kvs = res->n_kvs;
    v->rec_idx = res->rec_idx;
    v->rev = res->rev;
    v->key_off = res->key_off;
    v->key_len = res->key_len;
    v->val_off = res->val_off;
    v->val_len = res->val_len;
    v->n_bytes = res->n_bytes;
    v->elem_off = res->elem_off;
    v->wire = res->wire == KB_WIRE_KVS_I ? KB_WIRE_ETCD_KVS : res->wire == KB_WIRE_EVENTS_I ? KB_WIRE_ETCD_EVENTS : 0;
    v->on_device = res->out_mode == KB_OUT_DEVICE;
    v->bytes = res->out_mode == KB_OUT_DEVICE ? (const uint8_t *)res->d_arena.p : (const uint8_t *)res->h_arena.p;
    return KB_OK;
}

// ------------------------------------------------------------------------------------------------
// point reads
// ------------------------------------------------------------------------------------------------
// A point-read batch is a lane batch like a range batch: one launch chain on the lane stream -- bound upload, k_search,
// k_get_resolve, k_get_finalize, the rows' copy into the result's pinned buffer, the value / element copy, k_publish_rout --
// and one host wait in collect.  The rows publish after the copy, so that wait means the arena is complete, ctx_quiesce's
// harvest covers the copy before anything rewrites the slabs, and the copy never queues behind another lane's range copy
// on the copy stream.
static int get_submit_locked(kb_ctx *ctx, ScanLane &L, const kb_get_req *reqs, uint64_t n, int out_mode, kb_pending **out)
{
    int base = 0, wire_mode = 0;
    KB_TRY(split_out_mode(out_mode, &base, &wire_mode));
    if ((base != KB_OUT_HOST && base != KB_OUT_DEVICE) || wire_mode == KB_WIRE_EVENTS_I) return KB_EINVAL;
    const bool wire = wire_mode != 0;
    *out = nullptr;
    if (!ctx->loaded) return kb_fail(ctx, KB_ESTATE, "no store loaded");
    if (n >= 0x7FFFFFFFull) return kb_fail(ctx, KB_ELIMIT, "too many point reads in one batch");
    for (uint64_t i = 0; i < n; i++) {
        if (!reqs[i].key && reqs[i].key_len) return KB_EINVAL;
        // the longest user key a record can hold: its internal key (magic + key + '$' + revision) is at most 65535 bytes
        if (reqs[i].key_len > 65535 - 13) return kb_fail(ctx, KB_ELIMIT, "key too long");
    }
    cudaSetDevice(ctx->device);
    KB_TRY(lane_take(ctx));
    std::unique_ptr<kb_pending> P(new kb_pending());
    // Arena: sized by a bound the host knows without a round trip, as the range path does: n times the store's largest
    // pair (+ 48 bytes of tags per element in wire mode).  Reads of different user keys answer with different records,
    // so when that exceeds the slab, k reads of the most-read key bound the answer by k copies of the slab.
    uint64_t ub = n * ctx->max_kv_chunks * 16;
    const uint64_t slab = (ctx->kused16 + ctx->vused16) * 16;
    if (ub > slab) {
        std::unordered_map<std::string_view, uint64_t> reads;
        uint64_t most = 0;
        for (uint64_t i = 0; i < n; i++)
            most = std::max(most, ++reads[std::string_view((const char *)reqs[i].key, reqs[i].key_len)]);
        ub = std::min(ub, most * slab);
    }
    if (wire) ub += n * 48;
    HeldResult res{ctx, nullptr};  // every early return hands the result's pooled buffers back
    // an empty batch launches nothing
    KB_TRY(answer_new(ctx, res, ResultKind::point_read, base, wire_mode, 0, n ? ub + 64 : 0));
    res.p->n_gets = n;
    const size_t rows_bytes = get_rows_bytes(n, wire);
    KB_TRY(pool_get_host(ctx, rows_bytes + 64, &res.p->h_meta));
    const GetRows hrows = get_rows_at(res.p->h_meta.p, n, wire);
    *hrows.n_bytes = 0;
    if (wire) hrows.elem_off[0] = 0;
    uint64_t epoch = 0;
    if (n) {
        // bound of read i = EncodeObjectKey(key, revision or MaxUint64) + 0x00: its lower_bound is the first record
        // strictly greater than the start key of the reference's reverse iterator (the 0x00 is the zeroed slot's)
        PackedBounds pk;
        KB_TRY(bounds_pack(
            ctx, L.h_stage, n, [&](uint64_t i) { return reqs[i].key_len + 14; },
            [&](uint64_t i, uint8_t *b) {
                const uint64_t ul = reqs[i].key_len;
                const uint64_t rev = reqs[i].revision ? reqs[i].revision : ~0ull;
                b[0] = 0x57; b[1] = 0xfb; b[2] = 0x80; b[3] = 0x8b;
                if (ul) memcpy(b + 4, reqs[i].key, ul);
                b[4 + ul] = 0x24;
                for (int k = 0; k < 8; k++) b[5 + ul + k] = (uint8_t)(rev >> (8 * (7 - k)));
            },
            &pk));
        KB_TRY(dbuf_ensure(ctx, L.d_reqout, rows_bytes + 64));
        // L.d_get: [one-request job table | ReqDev][copy jobs][wire mode: the per-kv arrays k_wire_jobs writes (scratch)]
        const size_t tab_bytes = jobtab_bytes(1) + sizeof(ReqDev);
        static_assert((jobtab_bytes(1) + sizeof(ReqDev)) % 16 == 0, "the copy jobs start on a 16-byte boundary");
        const size_t jobs_bytes = copy_jobs_bytes(n, wire_mode);
        KB_TRY(dbuf_ensure(ctx, L.d_get, tab_bytes + jobs_bytes + (wire ? n * 44 + 72 : 0)));
        if (wire) {
            KB_TRY(dbuf_ensure(ctx, L.d_sel, n * 4));
            KB_TRY(dbuf_ensure(ctx, L.d_slot, n * 8));
        }
        KB_TRY(hostpub_ensure(ctx, L.rows, KB_PUB_HEAD + sizeof(ReqOut), L.stream));
        const JobTable tab = jobtab_at(L.d_get.p, 1);
        void *d_jobs = (uint8_t *)L.d_get.p + tab_bytes;
        const GetRows drows = get_rows_at(L.d_reqout.p, n, wire);

        KB_TRY(bound_search(ctx, L.search, pk, L.stream, false));
        GetOut go;
        go.status = drows.status;
        go.mod_rev = drows.mod_rev;
        go.voff16 = drows.val_off;  // k_get_finalize replaces the slab chunk by the arena offset
        go.rec = drows.rec;
        go.vlen = drows.val_len;
        KB_LAUNCH_S(ctx, L.stream, "k_get_resolve", n * 320,
                    (k_get_resolve<<<(unsigned)((n * 32 + 127) / 128), 128, 0, L.stream>>>(
                        ctx->st, L.search.dev, (const uint32_t *)L.search.d_bres.p, go)));
        KB_LAUNCH_S(ctx, L.stream, "k_get_finalize", n * 40,
                    (k_get_finalize<<<1, 256, 0, L.stream>>>(ctx->st, drows, (uint32_t)n, wire ? 1 : 0, (GatherJob *)d_jobs,
                                                             (uint32_t *)L.d_sel.p, (uint64_t *)L.d_slot.p, tab.job_first)));
        KB_CUDA(ctx, cudaMemcpyAsync(res.p->h_meta.p, L.d_reqout.p, rows_bytes, cudaMemcpyDeviceToHost, L.stream));
        if (wire) {
            GatherOut gout;
            uint64_t *d_elem_off = om_layout((uint8_t *)d_jobs + jobs_bytes, n, KB_WIRE_KVS_I, gout);
            KB_TRY(launch_copy(ctx, L, L.stream, d_jobs, nullptr, jobtab_req(L.d_get.p), 1, tab, (const uint32_t *)L.d_sel.p,
                               (const uint64_t *)L.d_slot.p, n, KB_WIRE_KVS_I, gout, d_elem_off, res.p));
        } else {
            KB_TRY(launch_gather(ctx, L.stream, (const GatherJob *)d_jobs, tab, (uint4 *)res.p->d_arena.p, n, 0));
        }
        epoch = ++L.rows.epoch;
        KB_LAUNCH_S(ctx, L.stream, "k_publish_rout", 32,
                    (k_publish_rout<<<1, 256, 0, L.stream>>>(nullptr, 0, L.rows.p, epoch,
                                                             (const unsigned int *)ctx->d_ctrs.p + 8)));
        KB_CUDA(ctx, cudaGetLastError());
    }
    P->get = true;
    P->lane = &L;
    P->out_mode = base;
    P->wire = wire_mode;
    P->res = res.release();
    P->epoch = epoch;
    L.pending = P.get();
    *out = P.release();
    return KB_OK;
}

// the rows are in res->h_meta once the batch has published; KB_OUT_HOST copies the arena to pinned memory
static int get_collect_locked(kb_ctx *ctx, kb_pending *P, kb_result **out)
{
    *out = nullptr;
    cudaSetDevice(ctx->device);
    HeldPending held{ctx, P};  // every return below ends the batch: a failed one hands its buffers back
    KB_TRY(pending_harvest(ctx, P));
    kb_result *res = P->res;
    const uint64_t nbytes = *get_rows_at(res->h_meta.p, res->n_gets, res->wire != 0).n_bytes;
    res->n_bytes = nbytes;
    if (ctx->prof_on && nbytes) ctx->prof[prof_index(ctx, res->wire ? "k_wire_copy" : "k_gather")].bytes += 2 * nbytes;
    if (nbytes && res->out_mode == KB_OUT_HOST)
        KB_TRY(result_to_host(ctx, res, ctx->stream_h, {}, nbytes, "point-read D2H"));
    else if (!nbytes)
        result_put_device(ctx, res);
    *out = res;
    delete held.release();
    return KB_OK;
}

extern "C" int kb_get_submit(kb_ctx *ctx, const kb_get_req *reqs, uint64_t n, int out_mode, kb_pending **out)
{
    if (!ctx || !out || (n && !reqs)) return KB_EINVAL;
    *out = nullptr;
    std::lock_guard<std::mutex> g(ctx->mu);
    KB_TRY(get_submit_locked(ctx, ctx->lane(), reqs, n, out_mode, out));
    lane_swap(ctx);
    return KB_OK;
}

extern "C" int kb_get_collect(kb_ctx *ctx, kb_pending *pending, kb_result **out)
{
    if (!ctx || !pending || !out) return KB_EINVAL;
    *out = nullptr;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!pending->get) return kb_fail(ctx, KB_EINVAL, "kb_get_collect: a range batch is collected by kb_range_collect");
    return get_collect_locked(ctx, pending, out);
}

// submit + collect on the current lane, as kb_range_batch is built; the raw modes only
extern "C" int kb_get_batch(kb_ctx *ctx, const kb_get_req *reqs, uint64_t n, int out_mode, kb_result **out)
{
    if (!ctx || !out || (n && !reqs)) return KB_EINVAL;
    if (out_mode != KB_OUT_HOST && out_mode != KB_OUT_DEVICE) return KB_EINVAL;
    *out = nullptr;
    std::lock_guard<std::mutex> g(ctx->mu);
    kb_pending *P = nullptr;
    KB_TRY(get_submit_locked(ctx, ctx->lane(), reqs, n, out_mode, &P));
    return get_collect_locked(ctx, P, out);
}

extern "C" int kb_get_view_get(const kb_result *res, kb_get_view *v)
{
    if (!res || !v || res->kind != ResultKind::point_read) return KB_EINVAL;
    memset(v, 0, sizeof(*v));
    const GetRows r = get_rows_at(res->h_meta.p, res->n_gets, res->wire != 0);
    v->n = res->n_gets;
    v->status = r.status;
    v->mod_rev = r.mod_rev;
    v->val_off = r.val_off;
    v->rec_idx = r.rec;
    v->val_len = r.val_len;
    v->n_bytes = res->n_bytes;
    v->on_device = res->out_mode == KB_OUT_DEVICE;
    v->bytes = v->on_device ? (const uint8_t *)res->d_arena.p : (const uint8_t *)res->h_arena.p;
    return KB_OK;
}

extern "C" int kb_get_elem_off(const kb_result *res, const uint64_t **elem_off)
{
    if (!res || !elem_off || res->kind != ResultKind::point_read || !res->wire) return KB_EINVAL;
    *elem_off = get_rows_at(res->h_meta.p, res->n_gets, true).elem_off;
    return KB_OK;
}
