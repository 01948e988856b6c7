// kb_store.cu -- the HBM snapshot of libkbb200.so: everything that creates, changes, dumps or restores it.
//
// Replaces (reference file:line):
//   storage.BatchWrite   pkg/storage/interface.go:62-106, badger batch.go:33-139  -> kb_apply_batch, kb_expire
//
// A snapshot is two slabs (keys and values, every record on a 16-byte boundary, zero padded) and one DirSet: per record
// the directory (koff16, klen, voff16, vlen) and the scan summary (srev, sword; see summarize_record).  A second DirSet,
// the spare, is what a committed batch or a layout compaction writes; then the two swap and store_bind points ctx->st
// at the new live set.
//   kb_load_sorted / kb_restore  the caller's packed arrays / a dump file -> directory + slabs; store_install then
//                                builds the summary and checks the key order
//   kb_apply_batch / kb_expire   the batch's bytes appended at the slab tails; k_dir_merge + k_summarize into the spare
//   store_compact_layout         both slabs rewritten contiguously in key order (k_relocate); what kb_dump writes
// The scan path (kb_scan.cu and the files that share kb_scan.cuh) only reads the snapshot: ctx->st, max_kv_chunks,
// kused16 / vused16 and store_gen.
// The value slab (the heap) is HBM or, under KB_CFG_HOST_VALUES, mapped pinned host memory: only the vheap_* functions
// and the places that fill it (load, restore, the write path's append) and write it out (dump) know which.  Kernels read
// both through StoreDev::vslab.
#include <algorithm>
#include <system_error>
#include <thread>

#include "kb_internal.cuh"

// A host heap is released only once every stream that may run a kernel reading it has drained: cudaFree synchronises
// the device, but cudaFreeHost is not relied on to wait for kernels still reading the mapping.
void vheap_free(kb_ctx *ctx, VHeap &h)
{
    if (!h.p) return;
    if (h.host) {
        for (ScanLane &L : ctx->lanes)
            if (L.stream) cudaStreamSynchronize(L.stream);
        for (cudaStream_t s : {ctx->stream2, ctx->stream_g, ctx->stream_h})
            if (s) cudaStreamSynchronize(s);
        cudaFreeHost(h.host);
    } else {
        cudaFree(h.p);
    }
    h = VHeap();
}

namespace {

// a new value heap of at least `bytes`, in the context's placement (the HBM one exactly as dbuf_ensure sizes it)
int vheap_alloc(kb_ctx *ctx, VHeap &h, size_t bytes)
{
    if (!ctx->host_values) {
        DBuf b;
        KB_TRY(dbuf_ensure(ctx, b, bytes));
        h.p = b.p;
        h.host = nullptr;
        h.cap = b.cap;
        return KB_OK;
    }
    size_t want = std::max(bytes + bytes / 4, (size_t)4096);
    want = (want + 255) & ~(size_t)255;
    void *host = nullptr, *dev = nullptr;
    cudaError_t e = cudaHostAlloc(&host, want, cudaHostAllocMapped);
    if (e == cudaSuccess) e = cudaHostGetDevicePointer(&dev, host, 0);
    if (e != cudaSuccess) {
        if (host) cudaFreeHost(host);
        cudaGetLastError();  // not sticky: the context stays usable
        return kb_fail(ctx, KB_ENOMEM, "cannot allocate %zu bytes of mapped pinned host memory for the value heap (%s)",
                       want, cudaGetErrorString(e));
    }
    h.p = dev;
    h.host = (uint8_t *)host;
    h.cap = want;
    return KB_OK;
}

// room for `bytes` in the context's heap; its content is not kept
int vheap_ensure(kb_ctx *ctx, size_t bytes)
{
    if (ctx->d_vslab.p && ctx->d_vslab.cap >= bytes) return KB_OK;
    if (ctx->d_vslab.p) {
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->lane().stream));
        if (ctx->stream_g) KB_CUDA(ctx, cudaStreamSynchronize(ctx->stream_g));
        vheap_free(ctx, ctx->d_vslab);
    }
    return vheap_alloc(ctx, ctx->d_vslab, bytes);
}

// zero bytes [off, off + n) of heap h: on the host, or on the lane stream
int vheap_zero(kb_ctx *ctx, const VHeap &h, size_t off, size_t n)
{
    if (h.host) {
        memset(h.host + off, 0, n);
        return KB_OK;
    }
    KB_CUDA(ctx, cudaMemsetAsync((uint8_t *)h.p + off, 0, n, ctx->lane().stream));
    return KB_OK;
}

// grow the context's heap to hold `need16` chunks (+ slack), keeping its first `used16` chunks
int vheap_reserve(kb_ctx *ctx, uint64_t used16, uint64_t need16)
{
    const size_t need = (size_t)need16 * 16 + 64;
    VHeap &h = ctx->d_vslab;
    if (h.p && h.cap >= need) return KB_OK;
    VHeap nb;
    KB_TRY(vheap_alloc(ctx, nb, need + need / 2));
    if (h.p && used16) {
        if (h.host) {
            memcpy(nb.host, h.host, (size_t)used16 * 16);
        } else {
            const cudaError_t e = cudaMemcpyAsync(nb.p, h.p, (size_t)used16 * 16, cudaMemcpyDeviceToDevice, ctx->lane().stream);
            if (e != cudaSuccess) {
                vheap_free(ctx, nb);
                return kb_cuda_fail(ctx, e, "value heap growth");
            }
        }
    }
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->lane().stream));
    vheap_free(ctx, h);
    h = nb;
    return KB_OK;
}

// ------------------------------------------------------------------------------------------------
// scan summary
// ------------------------------------------------------------------------------------------------
constexpr uint32_t MAGIC_LE = 0x8b80fb57u;  // bytes 57 fb 80 8b (coder/normal.go:26)

__device__ __forceinline__ uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

// Summary of record i of `st` against record i - 1 (record 0 gets KB_LCP_INF; the pass replaces the LCP of every
// request's first record by KB_LCP_INF anyway), computed by one warp; `lane` 0 stores it.
//   sword: the LCP in bits 0..15; KB_M_DEC_OK / KB_M_REV0 / KB_S_TOMBV (the value is "tombstone", util.go:28) at the
//          meta word's positions; KB_S_VL9, KB_S_VL8, KB_S_EVENTS (the user key contains "/events/") above them
//   srev:  the key's revision; for a revision record (revision 0) with a value of at least 8 bytes, the value's first
//          8 bytes big-endian (scanner.go:476-491, 566-591); 0 when the key does not decode
// The lanes compare 32 chunks of the two keys at a time and test 32 start positions of "/events/" at a time, so a
// record costs a few dependent round trips whatever its key length (the write path summarizes a few hundred records
// per batch, the load path all of them).
__device__ __forceinline__ void summarize_record(const StoreDev &st, uint32_t i, uint32_t lane, uint64_t *srev, uint32_t *sword)
{
    const unsigned FULLM = 0xffffffffu;
    const uint4 *kp = st.kslab + st.koff16[i];
    const uint32_t len = st.klen[i];
    uint32_t lcp = KB_LCP_INF;
    if (i > 0) {
        const uint4 *pp = st.kslab + st.koff16[i - 1];
        const uint32_t m = min(len, (uint32_t)st.klen[i - 1]);
        lcp = m;
        for (uint32_t c0 = 0; c0 * 16 < m; c0 += 32) {
            const uint32_t c = c0 + lane;
            const int p = c * 16 < m ? first_diff16(kp[c], pp[c]) : 16;
            const unsigned diff = __ballot_sync(FULLM, p < 16);
            if (diff) {
                const int src = __ffs(diff) - 1;
                lcp = min(m, (c0 + src) * 16 + (uint32_t)__shfl_sync(FULLM, p, src));
                break;
            }
        }
    }
    const uint8_t *kb = (const uint8_t *)kp;
    const uint32_t vl = st.vlen[i];
    uint32_t w = lcp;
    uint64_t s = 0;
    if (vl == 9) w |= KB_S_VL9;
    if (vl >= 8) w |= KB_S_VL8;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (vl >= 8) v = st.vslab[st.voff16[i]];
    if (vl == 9 && v.x == 0x626d6f74u && v.y == 0x6e6f7473u && (v.z & 0xffu) == 0x65u) w |= KB_S_TOMBV;
    if (len >= 13 && ((const uint32_t *)kp)[0] == MAGIC_LE && kb[len - 9] == 0x24) {  // coder.Decode (normal.go:58-70)
        w |= KB_M_DEC_OK;
        s = be64_bytes(kb + len - 8);
        if (s == 0) {
            w |= KB_M_REV0;
            if (vl >= 8) s = ((uint64_t)bswap32(v.x) << 32) | bswap32(v.y);
        }
        // bytes.Contains(rawKey, "/events/") over the user key kb[4 .. len - 9)
        const uint8_t *uk = kb + 4;
        const uint32_t n = len - 13;
        bool found = false;
        for (uint32_t p = lane; p + 8 <= n && !found; p += 32) found = be64_bytes(uk + p) == 0x2f6576656e74732full;
        if (__any_sync(FULLM, found)) w |= KB_S_EVENTS;
    }
    if (lane == 0) {
        *srev = s;
        *sword = w;
    }
}

// summary of records idx[0 .. n) (idx == nullptr: of records 0 .. n) into srev / sword, warp per record
__global__ void __launch_bounds__(256)
k_summarize(StoreDev st, const uint32_t *__restrict__ idx, uint32_t n, uint64_t *__restrict__ srev, uint32_t *__restrict__ sword)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t t = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; t < n; t += warps) {
        const uint32_t i = idx ? idx[t] : (uint32_t)t;
        summarize_record(st, i, lane, srev + i, sword + i);
    }
}

// ------------------------------------------------------------------------------------------------
// store ingest
// ------------------------------------------------------------------------------------------------
// one warp per record: copy the packed bytes into the 16-byte aligned slab (destination is pre-zeroed)
__global__ void k_repack(const uint8_t *__restrict__ src, const uint64_t *__restrict__ soff, uint8_t *__restrict__ dst,
                         const uint32_t *__restrict__ doff16_32, const uint64_t *__restrict__ doff16_64, uint32_t n)
{
    uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    uint32_t nw = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = w; i < n; i += nw) {
        uint64_t s = soff[i], e = soff[i + 1];
        uint64_t d = (doff16_32 ? (uint64_t)doff16_32[i] : doff16_64[i]) * 16ull;
        for (uint64_t b = lane; b < e - s; b += 32) dst[d + b] = src[s + b];
    }
}

// strict ascending order of adjacent keys (storage.Iter contract); thread per record
__global__ void k_check_sorted(StoreDev st, uint32_t *bad)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0 || i >= st.n) return;
    const uint4 *a = st.kslab + st.koff16[i - 1];
    const uint4 *b = st.kslab + st.koff16[i];
    uint32_t la = st.klen[i - 1], lb = st.klen[i];
    uint32_t m = la < lb ? la : lb;
    bool less = la < lb;  // all common bytes equal -> shorter first; equal length -> duplicate -> not less
    for (uint32_t c = 0; c * 16 < m; c++) {
        uint4 x = a[c], y = b[c];
        int p = first_diff16(x, y);
        if (p < 16 && c * 16 + p < m) {
            less = byte_of(x, p) < byte_of(y, p);
            break;
        }
    }
    if (!less) atomicMin(bad, i);
}

// ------------------------------------------------------------------------------------------------
// kb_apply_batch kernels
// ------------------------------------------------------------------------------------------------
// exists[i] = 1 iff the record at pos[i] (lower_bound of op key i) carries exactly that key; old_vchunks[i] = its value's
// 16-byte chunks (they become garbage when the op replaces or deletes the record)
__global__ void __launch_bounds__(128)
k_key_exists(StoreDev st, BoundsDev bounds, const uint32_t *__restrict__ pos, uint8_t *__restrict__ exists,
             uint32_t *__restrict__ old_vchunks)
{
    const uint32_t g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (g >= bounds.n) return;
    const uint32_t r = pos[g];
    bool eq = r < st.n;
    if (eq) {
        const uint32_t bl = bounds.len(g);
        eq = st.klen[r] == bl && warp_prefix_eq(st.kslab + st.koff16[r], bounds, g, bl);
    }
    if (lane == 0) {
        exists[g] = eq ? 1 : 0;
        old_vchunks[g] = eq ? (st.vlen[r] + 15) >> 4 : 0;
    }
}

// The store is a HEAP of key / value bytes plus a directory sorted by key.  A committed batch appends the bytes of its
// puts at the slab tails and rebuilds only the directory: every surviving record moves by (#inserts at or before it) -
// (#deletes before it), every insert lands at (its lower bound) + (#inserts before it) - (#deletes before it).
// ins_pos / del_pos / rep_pos are ascending.
struct DirEntry {  // an inserted record; a replacement uses voff16 / vlen only (its key stays where it is)
    uint64_t voff16;
    uint32_t koff16, vlen;
    uint32_t klen, pad;
};

struct DirArrays {
    uint32_t *koff16;
    uint16_t *klen;
    uint64_t *voff16;
    uint32_t *vlen;
    uint64_t *srev;
    uint32_t *sword;
};

__device__ __forceinline__ uint32_t lower_bound_u32(const uint32_t *a, uint32_t n, uint32_t v)
{
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (a[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(256)
k_dir_merge(StoreDev old, const uint32_t *__restrict__ ins_pos, const DirEntry *__restrict__ ins_ent, uint32_t n_ins,
            const uint32_t *__restrict__ del_pos, uint32_t n_del, const uint32_t *__restrict__ rep_pos,
            const DirEntry *__restrict__ rep_ent, uint32_t n_rep, DirArrays out)
{
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < old.n) {
        const uint32_t i = (uint32_t)t;
        const uint32_t db = lower_bound_u32(del_pos, n_del, i);
        if (db < n_del && del_pos[db] == i) return;  // deleted
        const uint32_t ib = lower_bound_u32(ins_pos, n_ins, i + 1);  // inserts with pos <= i sort in front of record i
        const uint32_t at = i + ib - db;
        out.koff16[at] = old.koff16[i];
        out.klen[at] = old.klen[i];
        const uint32_t rb = lower_bound_u32(rep_pos, n_rep, i);
        if (rb < n_rep && rep_pos[rb] == i) {  // same key, new value
            out.voff16[at] = rep_ent[rb].voff16;
            out.vlen[at] = rep_ent[rb].vlen;
        } else {
            out.voff16[at] = old.voff16[i];
            out.vlen[at] = old.vlen[i];
        }
        out.srev[at] = old.srev[i];  // the summary travels with the record; k_summarize redoes the ones the batch changed
        out.sword[at] = old.sword[i];
    } else if (t < (uint64_t)old.n + n_ins) {
        const uint32_t k = (uint32_t)(t - old.n);
        const uint32_t p = ins_pos[k];
        const uint32_t at = p + k - lower_bound_u32(del_pos, n_del, p);
        const DirEntry e = ins_ent[k];
        out.koff16[at] = e.koff16;
        out.klen[at] = (uint16_t)e.klen;
        out.voff16[at] = e.voff16;
        out.vlen[at] = e.vlen;
    }
}

// layout compaction: every record's key and value copied to its place in fresh, contiguous, sorted slabs (warp per record)
__global__ void __launch_bounds__(256)
k_relocate(StoreDev old, const uint32_t *__restrict__ nkoff16, const uint64_t *__restrict__ nvoff16, uint4 *__restrict__ nk,
           uint4 *__restrict__ nv)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t r = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < old.n; r += warps) {
        const uint32_t kc = ((uint32_t)old.klen[r] + 15) >> 4, vc = (old.vlen[r] + 15) >> 4;
        const uint4 *ks = old.kslab + old.koff16[r], *vs = old.vslab + old.voff16[r];
        uint4 *kd = nk + nkoff16[r], *vd = nv + nvoff16[r];
        for (uint32_t c = lane; c < kc; c += 32) kd[c] = ldg_stream(ks + c);
        for (uint32_t c = lane; c < vc; c += 32) stg_stream(vd + c, ldg_stream(vs + c));
    }
}

// ------------------------------------------------------------------------------------------------
// host: directory sets and the install path
// ------------------------------------------------------------------------------------------------
// a record directory on the host: n + 1 offsets (the last one = the slab's used chunks), n lengths
struct HostDir {
    std::vector<uint32_t> koff16, vlen;
    std::vector<uint16_t> klen;
    std::vector<uint64_t> voff16;
    explicit HostDir(uint64_t n) : koff16(n + 1), vlen(n + 1), klen(n + 1), voff16(n + 1) {}
};

int dirset_ensure(kb_ctx *ctx, DirSet &d, uint64_t n)
{
    int rc = KB_OK;
    d.each([&](DBuf &b, size_t elem) {
        if (rc == KB_OK) rc = dbuf_ensure(ctx, b, (n + 1) * elem);
    });
    return rc;
}

// the slabs with the directory set `d` of n records
StoreDev store_view(const kb_ctx *ctx, const DirSet &d, uint64_t n)
{
    StoreDev st;
    st.kslab = (const uint4 *)ctx->d_kslab.p;
    st.koff16 = (const uint32_t *)d.koff16.p;
    st.klen = (const uint16_t *)d.klen.p;
    st.vslab = (const uint4 *)ctx->d_vslab.p;
    st.voff16 = (const uint64_t *)d.voff16.p;
    st.vlen = (const uint32_t *)d.vlen.p;
    st.srev = (const uint64_t *)d.srev.p;
    st.sword = (const uint32_t *)d.sword.p;
    st.n = (uint32_t)n;
    return st;
}

// ctx->st = the slabs and the live set; the snapshot changed, so bound searches prefetched against the old one are void
void store_bind(kb_ctx *ctx, uint64_t n)
{
    ctx->st = store_view(ctx, ctx->live, n);
    ctx->store_gen++;
}

// Room for a snapshot of n records whose directory is `d`: both slabs, each with a zeroed 64-byte slack behind its tail
// (key_less reads up to three chunks from a key's start), and the live directory set, which gets the directory.  The
// caller fills the slabs.
int store_alloc(kb_ctx *ctx, const HostDir &d, uint64_t n)
{
    const uint64_t kc = d.koff16[n], vc = d.voff16[n];
    KB_TRY(dbuf_ensure(ctx, ctx->d_kslab, kc * 16 + 64));
    KB_TRY(vheap_ensure(ctx, vc * 16 + 64));
    KB_TRY(dirset_ensure(ctx, ctx->live, n));
    KB_CUDA(ctx, cudaMemsetAsync((uint8_t *)ctx->d_kslab.p + kc * 16, 0, 64, ctx->lane().stream));
    KB_TRY(vheap_zero(ctx, ctx->d_vslab, vc * 16, 64));
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->live.koff16.p, d.koff16.data(), (n + 1) * 4, cudaMemcpyHostToDevice, ctx->lane().stream));
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->live.klen.p, d.klen.data(), n * 2, cudaMemcpyHostToDevice, ctx->lane().stream));
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->live.voff16.p, d.voff16.data(), (n + 1) * 8, cudaMemcpyHostToDevice, ctx->lane().stream));
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->live.vlen.p, d.vlen.data(), n * 4, cudaMemcpyHostToDevice, ctx->lane().stream));
    return KB_OK;
}

// The slabs and directory store_alloc made, now filled, become the snapshot: the scan summary is built (it is not part
// of a dump: it derives from the keys and values), the iterator contract is checked (strictly ascending unique keys),
// the heap counters and TTL maps start afresh.  `what` prefixes the error message.
int store_install(kb_ctx *ctx, const HostDir &d, uint64_t n, uint64_t max_kv, const char *what)
{
    store_bind(ctx, n);
    // per record: two keys' offsets and lengths, the value's, a 16-byte value probe and the 12-byte summary (the key
    // bytes themselves are not counted)
    if (n)
        KB_LAUNCH(ctx, "k_summarize", n * 48,
                  (k_summarize<<<(unsigned)std::min<uint64_t>((n + 7) / 8, (uint64_t)ctx->n_sms * 16), 256, 0, ctx->lane().stream>>>(
                      ctx->st, nullptr, (uint32_t)n, (uint64_t *)ctx->live.srev.p, (uint32_t *)ctx->live.sword.p)));
    KB_CUDA(ctx, cudaGetLastError());
    uint32_t init = KB_NONE, bad = KB_NONE;
    if (n > 1) {
        KB_TRY(dbuf_ensure(ctx, ctx->d_flags, 64));
        KB_CUDA(ctx, cudaMemcpyAsync(ctx->d_flags.p, &init, 4, cudaMemcpyHostToDevice, ctx->lane().stream));
        k_check_sorted<<<(unsigned)((n + 255) / 256), 256, 0, ctx->lane().stream>>>(ctx->st, (uint32_t *)ctx->d_flags.p);
        KB_CUDA(ctx, cudaMemcpyAsync(&bad, ctx->d_flags.p, 4, cudaMemcpyDeviceToHost, ctx->lane().stream));
    }
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->lane().stream));
    if (bad != KB_NONE) return kb_fail(ctx, KB_EUNSORTED, "%srecord %u is not greater than its predecessor", what, bad);
    ctx->kused16 = d.koff16[n];
    ctx->vused16 = d.voff16[n];
    ctx->max_kv_chunks = (uint32_t)std::min<uint64_t>(max_kv, 0xFFFFFFFFu);
    ctx->garbage_k16 = ctx->garbage_v16 = ctx->displaced = 0;
    ctx->out_of_order = false;
    ctx->ttl_queue.clear();
    ctx->ttl_of.clear();
    ctx->loaded = true;
    return KB_OK;
}

// A host heap is filled on the host: record i's value into its zero-padded 16-byte slots, in parallel chunks of records
// (the value bytes never pass through HBM)
void vheap_fill_host(kb_ctx *ctx, const HostDir &d, const uint8_t *vals, const uint64_t *val_off, uint64_t n)
{
    uint8_t *heap = ctx->d_vslab.host;
    auto fill = [&](uint64_t a, uint64_t b) {
        for (uint64_t i = a; i < b; i++) {
            const uint64_t vl = d.vlen[i], pad = ((vl + 15) & ~15ull) - vl;
            uint8_t *dst = heap + d.voff16[i] * 16;
            if (vl) memcpy(dst, vals + val_off[i], vl);
            if (pad) memset(dst + vl, 0, pad);
        }
    };
    const uint64_t bytes = d.voff16[n] * 16;
    const uint64_t nt = std::max<uint64_t>(1, std::min<uint64_t>({(uint64_t)std::thread::hardware_concurrency(), 16,
                                                                   bytes / (8u << 20)}));
    std::vector<std::thread> th;
    for (uint64_t t = 1; t < nt; t++) {
        try {
            th.emplace_back(fill, n * t / nt, n * (t + 1) / nt);
        } catch (const std::system_error &) {
            fill(n * t / nt, n * (t + 1) / nt);  // no thread to be had: this one does the chunk
        }
    }
    fill(0, n / nt);
    for (std::thread &x : th) x.join();
}
}  // namespace

extern "C" int kb_load_sorted(kb_ctx *ctx, const uint8_t *keys, const uint64_t *key_off, const uint8_t *vals,
                              const uint64_t *val_off, uint64_t n)
{
    if (!ctx || (n && (!keys || !key_off || !vals || !val_off))) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaSetDevice(ctx->device);
    KB_TRY(ctx_quiesce(ctx));
    compact_streams_invalidate(ctx, "kb_load_sorted");
    if (n >= 0xFFFFFFFEull) return kb_fail(ctx, KB_ELIMIT, "too many records (%llu)", (unsigned long long)n);
    ctx->loaded = false;

    // destination offsets (host): every record padded to a 16-byte multiple
    HostDir d(n);
    uint64_t kacc = 0, vacc = 0, max_kv = 0;
    for (uint64_t i = 0; i < n; i++) {
        uint64_t kl = key_off[i + 1] - key_off[i], vl = val_off[i + 1] - val_off[i];
        if (kl > 65535) return kb_fail(ctx, KB_ELIMIT, "key %llu longer than 65535 bytes", (unsigned long long)i);
        if (vl > 0xFFFFFFFFull) return kb_fail(ctx, KB_ELIMIT, "value %llu too long", (unsigned long long)i);
        d.koff16[i] = (uint32_t)kacc;
        d.voff16[i] = vacc;
        d.klen[i] = (uint16_t)kl;
        d.vlen[i] = (uint32_t)vl;
        kacc += (kl + 15) / 16;
        vacc += (vl + 15) / 16;
        max_kv = std::max<uint64_t>(max_kv, (kl + 15) / 16 + (vl + 15) / 16);
        if (kacc > 0xFFFFFFF0ull) return kb_fail(ctx, KB_ELIMIT, "key slab exceeds 64 GiB");
    }
    d.koff16[n] = (uint32_t)kacc;
    d.voff16[n] = vacc;

    KB_TRY(store_alloc(ctx, d, n));
    // k_repack writes only the bytes of each record: the padding behind them is zeroed first (a host heap is filled
    // with its padding by vheap_fill_host)
    KB_CUDA(ctx, cudaMemsetAsync(ctx->d_kslab.p, 0, kacc * 16, ctx->lane().stream));
    if (!ctx->host_values) KB_CUDA(ctx, cudaMemsetAsync(ctx->d_vslab.p, 0, vacc * 16, ctx->lane().stream));

    // packed source bytes -> device (temporary), then repack on the device
    uint64_t ksrc = n ? key_off[n] - key_off[0] : 0, vsrc = n ? val_off[n] - val_off[0] : 0;
    DBuf tmp_b, tmp_o;
    uint64_t maxsrc = ctx->host_values ? ksrc : std::max(ksrc, vsrc);
    KB_TRY(dbuf_ensure(ctx, tmp_b, maxsrc + 16));
    KB_TRY(dbuf_ensure(ctx, tmp_o, (n + 1) * 8));
    const int TB = 256;
    int rg = (int)std::min<uint64_t>((n * 32 + TB - 1) / TB + 1, (uint64_t)ctx->n_sms * 16);
    int rc = KB_OK;
    do {
        if (n == 0) break;
        // keys (offsets rebased to 0 if the caller's first offset is not 0)
        std::vector<uint64_t> rebased;
        const uint64_t *ko = key_off, *vo = val_off;
        if (key_off[0] != 0) {
            rebased.resize(n + 1);
            for (uint64_t i = 0; i <= n; i++) rebased[i] = key_off[i] - key_off[0];
            ko = rebased.data();
        }
        if (cudaMemcpyAsync(tmp_b.p, keys + key_off[0], ksrc, cudaMemcpyHostToDevice, ctx->lane().stream) != cudaSuccess ||
            cudaMemcpyAsync(tmp_o.p, ko, (n + 1) * 8, cudaMemcpyHostToDevice, ctx->lane().stream) != cudaSuccess) {
            rc = kb_fail(ctx, KB_ECUDA, "H2D of keys failed");
            break;
        }
        k_repack<<<rg, TB, 0, ctx->lane().stream>>>((const uint8_t *)tmp_b.p, (const uint64_t *)tmp_o.p,
                                             (uint8_t *)ctx->d_kslab.p, (const uint32_t *)ctx->live.koff16.p, nullptr,
                                             (uint32_t)n);
        if (cudaStreamSynchronize(ctx->lane().stream) != cudaSuccess) {
            rc = kb_fail(ctx, KB_ECUDA, "key repack failed: %s", cudaGetErrorString(cudaGetLastError()));
            break;
        }
        if (ctx->host_values) {
            vheap_fill_host(ctx, d, vals, val_off, n);
            break;
        }
        std::vector<uint64_t> rebased_v;
        if (val_off[0] != 0) {
            rebased_v.resize(n + 1);
            for (uint64_t i = 0; i <= n; i++) rebased_v[i] = val_off[i] - val_off[0];
            vo = rebased_v.data();
        }
        if (cudaMemcpyAsync(tmp_b.p, vals + val_off[0], vsrc, cudaMemcpyHostToDevice, ctx->lane().stream) != cudaSuccess ||
            cudaMemcpyAsync(tmp_o.p, vo, (n + 1) * 8, cudaMemcpyHostToDevice, ctx->lane().stream) != cudaSuccess) {
            rc = kb_fail(ctx, KB_ECUDA, "H2D of values failed");
            break;
        }
        k_repack<<<rg, TB, 0, ctx->lane().stream>>>((const uint8_t *)tmp_b.p, (const uint64_t *)tmp_o.p,
                                             (uint8_t *)ctx->d_vslab.p, nullptr, (const uint64_t *)ctx->live.voff16.p,
                                             (uint32_t)n);
        if (cudaStreamSynchronize(ctx->lane().stream) != cudaSuccess) {
            rc = kb_fail(ctx, KB_ECUDA, "value repack failed: %s", cudaGetErrorString(cudaGetLastError()));
            break;
        }
    } while (0);
    cudaFree(tmp_b.p);
    cudaFree(tmp_o.p);
    if (rc != KB_OK) return rc;
    return store_install(ctx, d, n, max_kv, "");
}

extern "C" int kb_store_info(kb_ctx *ctx, uint64_t *n_records, uint64_t *key_bytes, uint64_t *val_bytes)
{
    if (!ctx) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);  // a write or an expiry moves all three together
    if (!ctx->loaded) return kb_fail(ctx, KB_ESTATE, "no store loaded");
    if (n_records) *n_records = ctx->st.n;
    if (key_bytes) *key_bytes = ctx->kused16 * 16;
    if (val_bytes) *val_bytes = ctx->vused16 * 16;
    return KB_OK;
}

extern "C" int kb_store_mem(kb_ctx *ctx, uint64_t *device_bytes, uint64_t *host_bytes)
{
    if (!ctx) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->loaded) return kb_fail(ctx, KB_ESTATE, "no store loaded");
    uint64_t dev = ctx->d_kslab.cap, host = 0;
    (ctx->d_vslab.host ? host : dev) += ctx->d_vslab.cap;
    for (DirSet *d : {&ctx->live, &ctx->spare}) d->each([&](DBuf &b, size_t) { dev += b.cap; });
    if (device_bytes) *device_bytes = dev;
    if (host_bytes) *host_bytes = host;
    return KB_OK;
}

extern "C" int kb_set_compact_revision(kb_ctx *ctx, int present, uint64_t rev)
{
    if (!ctx) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    ctx->compact_present = present != 0;
    ctx->compact_rev = rev;
    return KB_OK;
}

// ------------------------------------------------------------------------------------------------
// kb_apply_batch: one committed BatchWrite merged into the HBM snapshot.
//
// Round 1 rebuilt both slabs and merged the whole directory on the host for every batch (O(store bytes)).  Now the
// store is a heap + a sorted directory: the bytes of the batch's puts are appended at the slab tails (a value that
// replaces an existing key leaves the old bytes behind as garbage; the key bytes are reused), and only the directory
// and the scan summary (18 + 12 bytes per record) are rebuilt, on the device, by k_dir_merge; k_summarize then redoes the
// summary of the records whose key, value or predecessor the batch changed.  When more than 1/32 of the records are out
// of place, or a quarter of a slab is garbage, store_compact_layout rewrites the slabs contiguously in key order
// (O(store), amortised O(1) per op).
// ------------------------------------------------------------------------------------------------
namespace {
struct ApplyOp {
    std::string key, val;
    uint32_t type;
    uint64_t order;
};

// grow the key slab to hold `need16` chunks (+ slack), keeping its first `used16` chunks (the value heap: vheap_reserve)
int slab_reserve(kb_ctx *ctx, DBuf &slab, uint64_t used16, uint64_t need16)
{
    const size_t need = (size_t)need16 * 16 + 64;
    if (slab.p && slab.cap >= need) return KB_OK;
    DBuf nb;
    KB_TRY(dbuf_ensure(ctx, nb, need + need / 2));
    if (slab.p && used16)
        KB_CUDA(ctx, cudaMemcpyAsync(nb.p, slab.p, (size_t)used16 * 16, cudaMemcpyDeviceToDevice, ctx->lane().stream));
    KB_CUDA(ctx, cudaStreamSynchronize(ctx->lane().stream));
    if (slab.p) cudaFree(slab.p);
    slab = nb;
    return KB_OK;
}

// rewrite both slabs contiguously in key order (also what kb_dump writes), unless no batch changed them since they last
// were; the caller holds ctx->mu
int store_compact_layout(kb_ctx *ctx)
{
    const uint64_t n = ctx->st.n;
    if (!ctx->out_of_order) return KB_OK;
    std::vector<uint16_t> klen(std::max<uint64_t>(n, 1));
    std::vector<uint32_t> vlen(std::max<uint64_t>(n, 1)), nko(n + 1);
    std::vector<uint64_t> nvo(n + 1);
    if (n) {
        KB_CUDA(ctx, cudaMemcpyAsync(klen.data(), ctx->st.klen, n * 2, cudaMemcpyDeviceToHost, ctx->lane().stream));
        KB_CUDA(ctx, cudaMemcpyAsync(vlen.data(), ctx->st.vlen, n * 4, cudaMemcpyDeviceToHost, ctx->lane().stream));
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->lane().stream));
    }
    uint64_t kacc = 0, vacc = 0;
    for (uint64_t i = 0; i < n; i++) {
        nko[i] = (uint32_t)kacc;
        nvo[i] = vacc;
        kacc += ((uint32_t)klen[i] + 15) / 16;
        vacc += ((uint64_t)vlen[i] + 15) / 16;
    }
    nko[n] = (uint32_t)kacc;
    nvo[n] = vacc;
    DBuf nk;
    VHeap nv;
    KB_TRY(dbuf_ensure(ctx, nk, kacc * 16 + 64));
    int rc = vheap_alloc(ctx, nv, vacc * 16 + 64);
    if (rc == KB_OK) rc = dirset_ensure(ctx, ctx->spare, n);
    if (rc != KB_OK) {
        cudaFree(nk.p);
        vheap_free(ctx, nv);
        return rc;
    }
    const DirSet &s = ctx->spare;
    cudaMemsetAsync((uint8_t *)nk.p + kacc * 16, 0, 64, ctx->lane().stream);
    vheap_zero(ctx, nv, vacc * 16, 64);
    // a host heap is read and written by k_relocate across the host link: one implementation for both placements
    cudaMemcpyAsync(s.koff16.p, nko.data(), (n + 1) * 4, cudaMemcpyHostToDevice, ctx->lane().stream);
    cudaMemcpyAsync(s.voff16.p, nvo.data(), (n + 1) * 8, cudaMemcpyHostToDevice, ctx->lane().stream);
    if (n) {
        KB_LAUNCH(ctx, "k_relocate", 2 * (kacc + vacc) * 16,
                  (k_relocate<<<ctx->n_sms * 8, 256, 0, ctx->lane().stream>>>(ctx->st, (const uint32_t *)s.koff16.p,
                                                               (const uint64_t *)s.voff16.p, (uint4 *)nk.p, (uint4 *)nv.p)));
        cudaMemcpyAsync(s.klen.p, ctx->st.klen, n * 2, cudaMemcpyDeviceToDevice, ctx->lane().stream);
        cudaMemcpyAsync(s.vlen.p, ctx->st.vlen, n * 4, cudaMemcpyDeviceToDevice, ctx->lane().stream);
        // the order stays, and the summary holds no offsets: it moves as it is
        cudaMemcpyAsync(s.srev.p, ctx->st.srev, n * 8, cudaMemcpyDeviceToDevice, ctx->lane().stream);
        cudaMemcpyAsync(s.sword.p, ctx->st.sword, n * 4, cudaMemcpyDeviceToDevice, ctx->lane().stream);
    }
    cudaError_t e = cudaStreamSynchronize(ctx->lane().stream);  // the host vectors die here; the old slabs are released below
    if (e != cudaSuccess) {
        cudaFree(nk.p);
        vheap_free(ctx, nv);
        ctx->loaded = false;
        return kb_cuda_fail(ctx, e, "layout compaction");
    }
    cudaFree(ctx->d_kslab.p);
    vheap_free(ctx, ctx->d_vslab);
    ctx->d_kslab = nk;
    ctx->d_vslab = nv;
    std::swap(ctx->live, ctx->spare);
    store_bind(ctx, n);
    ctx->kused16 = kacc;
    ctx->vused16 = vacc;
    ctx->garbage_k16 = ctx->garbage_v16 = ctx->displaced = 0;
    ctx->out_of_order = false;
    ctx->layout_compactions++;
    return KB_OK;
}
}  // namespace

static int apply_batch_locked(kb_ctx *ctx, const kb_write_op *ops, uint64_t n_ops);

extern "C" int kb_apply_batch(kb_ctx *ctx, const kb_write_op *ops, uint64_t n_ops)
{
    if (!ctx || (n_ops && !ops)) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    return write_batch_locked(ctx, ops, n_ops);
}

int write_batch_locked(kb_ctx *ctx, const kb_write_op *ops, uint64_t n_ops)
{
    KB_TRY(apply_batch_locked(ctx, ops, n_ops));
    // TTL bookkeeping, in op order: the last op on a key decides whether (and when) it expires
    for (uint64_t i = 0; i < n_ops; i++) {
        std::string k((const char *)ops[i].key, ops[i].key_len);
        if (ops[i].type == KB_OP_PUT && ops[i].expire_unix) {
            ctx->ttl_of[k] = ops[i].expire_unix;
            ctx->ttl_queue.emplace(ops[i].expire_unix, std::move(k));
        } else if (!ctx->ttl_of.empty()) {
            ctx->ttl_of.erase(k);  // deleted, or rewritten without a ttl: stale queue entries are skipped by kb_expire
        }
    }
    return KB_OK;
}

extern "C" int kb_expire(kb_ctx *ctx, uint64_t now_unix, uint64_t *n_dropped)
{
    if (!ctx) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (n_dropped) *n_dropped = 0;
    if (!ctx->loaded) return kb_fail(ctx, KB_ESTATE, "no store loaded");
    std::vector<std::string> due;
    auto end = ctx->ttl_queue.upper_bound(now_unix);
    for (auto it = ctx->ttl_queue.begin(); it != end; ++it) {
        auto cur = ctx->ttl_of.find(it->second);
        if (cur != ctx->ttl_of.end() && cur->second == it->first) {  // still the expiry the key has
            due.push_back(it->second);
            ctx->ttl_of.erase(cur);
        }
    }
    ctx->ttl_queue.erase(ctx->ttl_queue.begin(), end);
    if (due.empty()) return KB_OK;
    std::vector<kb_write_op> ops(due.size());
    for (size_t i = 0; i < due.size(); i++) {
        memset(&ops[i], 0, sizeof(kb_write_op));
        ops[i].type = KB_OP_DEL;
        ops[i].key = (const uint8_t *)due[i].data();
        ops[i].key_len = due[i].size();
    }
    const uint64_t before = ctx->st.n;
    KB_TRY(apply_batch_locked(ctx, ops.data(), ops.size()));
    if (n_dropped) *n_dropped = before - ctx->st.n;
    return KB_OK;
}

static int apply_batch_locked(kb_ctx *ctx, const kb_write_op *ops, uint64_t n_ops)
{
    if (!ctx->loaded) return kb_fail(ctx, KB_ESTATE, "no store loaded");
    cudaSetDevice(ctx->device);
    KB_TRY(ctx_quiesce(ctx));
    if (n_ops == 0) return KB_OK;
    // 1. last op per key wins; sort by key (bytes.Compare order)
    std::vector<ApplyOp> all(n_ops);
    for (uint64_t i = 0; i < n_ops; i++) {
        if ((!ops[i].key && ops[i].key_len) || (ops[i].type == KB_OP_PUT && !ops[i].val && ops[i].val_len)) return KB_EINVAL;
        if (ops[i].key_len > 65535) return kb_fail(ctx, KB_ELIMIT, "key longer than 65535 bytes");
        if (ops[i].val_len > 0xFFFFFFFFull) return kb_fail(ctx, KB_ELIMIT, "value too long");
        if (ops[i].type != KB_OP_PUT && ops[i].type != KB_OP_DEL) return KB_EINVAL;
        all[i].key.assign((const char *)ops[i].key, ops[i].key_len);
        if (ops[i].type == KB_OP_PUT) all[i].val.assign((const char *)ops[i].val, ops[i].val_len);
        all[i].type = ops[i].type;
        all[i].order = i;
    }
    std::sort(all.begin(), all.end(), [](const ApplyOp &a, const ApplyOp &b) {
        const int c = a.key.compare(b.key);  // std::string::compare is lexicographic on unsigned char via char_traits
        return c != 0 ? c < 0 : a.order < b.order;
    });
    std::vector<ApplyOp> m;
    for (size_t i = 0; i < all.size(); i++)
        if (i + 1 == all.size() || all[i + 1].key != all[i].key) m.push_back(std::move(all[i]));
    const uint64_t M = m.size();

    // 2. op keys as a bound slab on the device; lower bound and exact-match test of every op key
    PackedBounds pk;
    KB_TRY(bounds_pack(
        ctx, ctx->lane().h_stage, M, [&](uint64_t i) { return (uint64_t)m[i].key.size(); },
        [&](uint64_t i, uint8_t *dst) { memcpy(dst, m[i].key.data(), m[i].key.size()); }, &pk));
    BoundSearch &s = ctx->lane().search;
    KB_TRY(bound_search(ctx, s, pk, ctx->lane().stream, false, M * 5));  // pos (the results) | oldv | exists
    uint32_t *d_pos = (uint32_t *)s.d_bres.p, *d_oldv = d_pos + M;
    uint8_t *d_exists = (uint8_t *)(d_oldv + M);
    const unsigned sg = (unsigned)((M * 32 + 127) / 128);
    KB_LAUNCH(ctx, "k_key_exists", M * 320,
              (k_key_exists<<<sg, 128, 0, ctx->lane().stream>>>(ctx->st, s.dev, d_pos, d_exists, d_oldv)));
    std::vector<uint32_t> pos(M), oldv(M);
    std::vector<uint8_t> exists(M);
    KB_CUDA(ctx, cudaMemcpyAsync(pos.data(), d_pos, M * 4, cudaMemcpyDeviceToHost, ctx->lane().stream));
    KB_CUDA(ctx, cudaMemcpyAsync(oldv.data(), d_oldv, M * 4, cudaMemcpyDeviceToHost, ctx->lane().stream));
    KB_CUDA(ctx, cudaMemcpyAsync(exists.data(), d_exists, M, cudaMemcpyDeviceToHost, ctx->lane().stream));
    cudaError_t e = cudaStreamSynchronize(ctx->lane().stream);
    if (e != cudaSuccess) return kb_cuda_fail(ctx, e, "apply: search");

    // 3. classify; lay the appended bytes out behind the slab tails
    const uint64_t N = ctx->st.n;
    std::vector<uint32_t> ins_pos, del_pos, rep_pos;
    std::vector<DirEntry> ins_ent, rep_ent;
    std::vector<uint8_t> kimg, vimg;  // images of the appended key / value chunks
    uint64_t ktail = ctx->kused16, vtail = ctx->vused16, garbage_k = 0, garbage_v = 0;
    uint32_t max_kv = ctx->max_kv_chunks;
    auto append = [](std::vector<uint8_t> &img, const std::string &b) {
        const size_t at = img.size(), n16 = (b.size() + 15) / 16;
        img.resize(at + n16 * 16, 0);
        if (!b.empty()) memcpy(img.data() + at, b.data(), b.size());
        return (uint64_t)n16;
    };
    for (uint64_t i = 0; i < M; i++) {
        if (m[i].type == KB_OP_PUT) {
            const uint64_t vo = vtail;
            const uint64_t nv = append(vimg, m[i].val);
            vtail += nv;
            const uint64_t nk = (m[i].key.size() + 15) / 16;
            if (exists[i]) {  // same key: the key bytes stay where they are, the old value becomes garbage
                rep_pos.push_back(pos[i]);
                rep_ent.push_back(DirEntry{vo, 0, (uint32_t)m[i].val.size(), 0, 0});
                garbage_v += oldv[i];
            } else {
                ins_pos.push_back(pos[i]);
                ins_ent.push_back(DirEntry{vo, (uint32_t)ktail, (uint32_t)m[i].val.size(), (uint32_t)m[i].key.size(), 0});
                ktail += append(kimg, m[i].key);
            }
            max_kv = std::max<uint32_t>(max_kv, (uint32_t)std::min<uint64_t>(nk + nv, 0xFFFFFFFFu));
        } else if (exists[i]) {
            del_pos.push_back(pos[i]);
            garbage_k += (m[i].key.size() + 15) / 16;
            garbage_v += oldv[i];
        }
    }
    const uint64_t n_ins = ins_pos.size(), n_del = del_pos.size(), n_rep = rep_pos.size();
    const uint64_t N2 = N + n_ins - n_del;
    if (N2 >= 0xFFFFFFFEull) return kb_fail(ctx, KB_ELIMIT, "too many records");
    if (ktail > 0xFFFFFFF0ull) return kb_fail(ctx, KB_ELIMIT, "key slab exceeds 64 GiB");
    if (n_ins + n_del + n_rep == 0) return KB_OK;  // only deletes of absent keys
    // records of the new directory whose summary the merge cannot carry: every insert and the record behind it, the
    // record behind every deleted one (their predecessor changed), every replaced value
    std::vector<uint32_t> fix;
    fix.reserve(2 * n_ins + n_del + n_rep);
    auto dels_before = [&](uint32_t p) { return (uint32_t)(std::lower_bound(del_pos.begin(), del_pos.end(), p) - del_pos.begin()); };
    auto ins_upto = [&](uint32_t p) { return (uint32_t)(std::upper_bound(ins_pos.begin(), ins_pos.end(), p) - ins_pos.begin()); };
    for (uint64_t k = 0; k < n_ins; k++) {
        const uint32_t q = ins_pos[k] + (uint32_t)k - dels_before(ins_pos[k]);
        fix.push_back(q);
        if (q + 1 < N2) fix.push_back(q + 1);
    }
    for (uint32_t d : del_pos) {
        const uint32_t q = d - dels_before(d) + ins_upto(d);
        if (q < N2) fix.push_back(q);
    }
    for (uint32_t r : rep_pos) fix.push_back(r - dels_before(r) + ins_upto(r));
    std::sort(fix.begin(), fix.end());
    fix.erase(std::unique(fix.begin(), fix.end()), fix.end());
    const uint64_t n_fix = fix.size();

    // 4. bytes to the slab tails (growing a slab copies its used part once; the live store is untouched until step 6)
    KB_TRY(slab_reserve(ctx, ctx->d_kslab, ctx->kused16, ktail));
    KB_TRY(vheap_reserve(ctx, ctx->vused16, vtail));
    store_bind(ctx, N);
    const size_t tab_bytes = (n_ins + n_rep) * sizeof(DirEntry) + (n_ins + n_del + n_rep + n_fix) * 4 + 64;
    // The value image is staged for the upload below, or, into a host heap, copied straight to the heap tail: a host copy
    // that is done before the k_dir_merge / k_summarize launches that read it.  Nothing in flight reads the heap behind
    // vused16 (ctx_quiesce).
    const size_t vstage = ctx->d_vslab.host ? 0 : vimg.size();
    KB_TRY(hbuf_ensure(ctx, ctx->lane().h_stage2, kimg.size() + vstage + tab_bytes + 256));
    uint8_t *h2 = (uint8_t *)ctx->lane().h_stage2.p;
    if (!kimg.empty()) memcpy(h2, kimg.data(), kimg.size());
    if (!vimg.empty()) memcpy(vstage ? h2 + kimg.size() : ctx->d_vslab.host + ctx->vused16 * 16, vimg.data(), vimg.size());
    uint8_t *ht = h2 + ((kimg.size() + vstage + 15) & ~(size_t)15);
    DirEntry *t_ins_ent = (DirEntry *)ht, *t_rep_ent = t_ins_ent + n_ins;
    uint32_t *t_ins_pos = (uint32_t *)(t_rep_ent + n_rep), *t_del_pos = t_ins_pos + n_ins, *t_rep_pos = t_del_pos + n_del;
    uint32_t *t_fix = t_rep_pos + n_rep;
    if (n_ins) memcpy(t_ins_ent, ins_ent.data(), n_ins * sizeof(DirEntry)), memcpy(t_ins_pos, ins_pos.data(), n_ins * 4);
    if (n_rep) memcpy(t_rep_ent, rep_ent.data(), n_rep * sizeof(DirEntry)), memcpy(t_rep_pos, rep_pos.data(), n_rep * 4);
    if (n_del) memcpy(t_del_pos, del_pos.data(), n_del * 4);
    if (n_fix) memcpy(t_fix, fix.data(), n_fix * 4);
    KB_TRY(dbuf_ensure(ctx, ctx->lane().search.d_bounds, tab_bytes + 64));  // the bound slab is no longer needed: reuse it for the tables
    KB_TRY(dirset_ensure(ctx, ctx->spare, N2));
    if (!kimg.empty())
        KB_CUDA(ctx, cudaMemcpyAsync((uint8_t *)ctx->d_kslab.p + ctx->kused16 * 16, h2, kimg.size(), cudaMemcpyHostToDevice, ctx->lane().stream));
    if (vstage)
        KB_CUDA(ctx, cudaMemcpyAsync((uint8_t *)ctx->d_vslab.p + ctx->vused16 * 16, h2 + kimg.size(), vstage,
                                     cudaMemcpyHostToDevice, ctx->lane().stream));
    // key_less / decode read up to three chunks past a key: keep the slack behind the tails zero
    KB_CUDA(ctx, cudaMemsetAsync((uint8_t *)ctx->d_kslab.p + ktail * 16, 0, 64, ctx->lane().stream));
    KB_TRY(vheap_zero(ctx, ctx->d_vslab, vtail * 16, 64));
    KB_CUDA(ctx, cudaMemcpyAsync(ctx->lane().search.d_bounds.p, ht, tab_bytes - 64, cudaMemcpyHostToDevice, ctx->lane().stream));
    // 5. the directory, rebuilt on the device into the spare set
    const DirEntry *d_ins_ent = (const DirEntry *)ctx->lane().search.d_bounds.p, *d_rep_ent = d_ins_ent + n_ins;
    const uint32_t *d_ins_pos = (const uint32_t *)(d_rep_ent + n_rep), *d_del_pos = d_ins_pos + n_ins, *d_rep_pos = d_del_pos + n_del;
    const uint32_t *d_fix = d_rep_pos + n_rep;
    const StoreDev nst = store_view(ctx, ctx->spare, N2);  // the slabs as they are now, the directory the merge writes
    const DirArrays out{(uint32_t *)nst.koff16, (uint16_t *)nst.klen, (uint64_t *)nst.voff16, (uint32_t *)nst.vlen,
                        (uint64_t *)nst.srev, (uint32_t *)nst.sword};
    const uint64_t threads = N + n_ins;
    // per record read (N) and written (N2): 18 bytes of directory and 12 of summary
    KB_LAUNCH(ctx, "k_dir_merge", (N + N2) * 30,
              (k_dir_merge<<<(unsigned)((threads + 255) / 256), 256, 0, ctx->lane().stream>>>(ctx->st, d_ins_pos, d_ins_ent, (uint32_t)n_ins,
                                                                                       d_del_pos, (uint32_t)n_del, d_rep_pos,
                                                                                       d_rep_ent, (uint32_t)n_rep, out)));
    if (n_fix)
        KB_LAUNCH(ctx, "k_summarize", n_fix * 48,
                  (k_summarize<<<(unsigned)std::min<uint64_t>((n_fix + 7) / 8, (uint64_t)ctx->n_sms * 16), 256, 0, ctx->lane().stream>>>(
                      nst, d_fix, (uint32_t)n_fix, out.srev, out.sword)));
    e = cudaStreamSynchronize(ctx->lane().stream);  // the staging buffers are reused by the next call
    if (e != cudaSuccess) {
        ctx->loaded = false;
        return kb_cuda_fail(ctx, e, "apply: directory merge");
    }
    // 6. the new snapshot becomes visible
    std::swap(ctx->live, ctx->spare);
    store_bind(ctx, N2);
    ctx->kused16 = ktail;
    ctx->vused16 = vtail;
    ctx->garbage_k16 += garbage_k;
    ctx->garbage_v16 += garbage_v;
    ctx->displaced += n_ins;
    ctx->out_of_order = true;
    ctx->max_kv_chunks = max_kv;
    // an open compaction stream still copies keys and guards from where its sweep found them: the layout compaction
    // waits for the first batch after the last such stream closed (the garbage counters keep growing meanwhile)
    if (compact_streams_pin_heap(ctx)) return KB_OK;
    if (ctx->displaced > std::max<uint64_t>(4096, N2 / 32) || ctx->garbage_k16 * 4 > ktail || ctx->garbage_v16 * 4 > vtail)
        KB_TRY(store_compact_layout(ctx));
    return KB_OK;
}

// ------------------------------------------------------------------------------------------------
// durable dump / restore of the snapshot (device layout, so restore is file -> pinned staging -> HBM with no repack)
// ------------------------------------------------------------------------------------------------
namespace {
struct DumpHeader {
    char     magic[8];  // "KBB200D1"
    uint32_t version, header_bytes;
    uint64_t n, key_chunks, val_chunks;
    uint64_t compact_present, compact_rev;
    uint32_t max_kv_chunks, pad;
    uint64_t sum_dir, sum_keys, sum_vals;  // FNV-1a 64 of the directory section and of the two slabs
};
constexpr size_t DUMP_STAGE = 64u << 20;  // bytes per host <-> device hop

inline uint64_t fnv1a64_update(uint64_t h, const uint8_t *p, size_t n)
{
    // 8 bytes per step (word-wise FNV-1a variant): the checksum only has to detect torn or foreign files
    size_t i = 0;
    for (; i + 8 <= n; i += 8) {
        uint64_t w;
        memcpy(&w, p + i, 8);
        h = (h ^ w) * 0x100000001b3ull;
    }
    for (; i < n; i++) h = (h ^ p[i]) * 0x100000001b3ull;
    return h;
}

// device -> file through the pinned staging buffer, or straight from `host` (a host heap) when it is given; returns the
// checksum of the bytes written
int dump_section(kb_ctx *ctx, FILE *f, const void *dev, const uint8_t *host, uint64_t bytes, uint64_t *sum)
{
    uint64_t h = 0xcbf29ce484222325ull;
    for (uint64_t off = 0; off < bytes; off += DUMP_STAGE) {
        const size_t n = (size_t)std::min<uint64_t>(DUMP_STAGE, bytes - off);
        const uint8_t *src = host ? host + off : (const uint8_t *)ctx->lane().h_stage.p;
        if (!host) {
            KB_CUDA(ctx, cudaMemcpyAsync(ctx->lane().h_stage.p, (const uint8_t *)dev + off, n, cudaMemcpyDeviceToHost, ctx->lane().stream));
            KB_CUDA(ctx, cudaStreamSynchronize(ctx->lane().stream));
        }
        h = fnv1a64_update(h, src, n);
        if (fwrite(src, 1, n, f) != n) return kb_fail(ctx, KB_EIO, "dump: short write");
    }
    *sum = h;
    return KB_OK;
}

// file -> device through the pinned staging buffer, or straight into `host` (a host heap) when it is given
int restore_section(kb_ctx *ctx, FILE *f, void *dev, uint8_t *host, uint64_t bytes, uint64_t *sum)
{
    uint64_t h = 0xcbf29ce484222325ull;
    for (uint64_t off = 0; off < bytes; off += DUMP_STAGE) {
        const size_t n = (size_t)std::min<uint64_t>(DUMP_STAGE, bytes - off);
        uint8_t *dst = host ? host + off : (uint8_t *)ctx->lane().h_stage.p;
        if (fread(dst, 1, n, f) != n) return kb_fail(ctx, KB_EINVAL, "restore: file truncated");
        h = fnv1a64_update(h, dst, n);
        if (!host) {
            KB_CUDA(ctx, cudaMemcpyAsync((uint8_t *)dev + off, dst, n, cudaMemcpyHostToDevice, ctx->lane().stream));
            KB_CUDA(ctx, cudaStreamSynchronize(ctx->lane().stream));  // the staging buffer is reused by the next hop
        }
    }
    *sum = h;
    return KB_OK;
}
}  // namespace

extern "C" int kb_dump(kb_ctx *ctx, const char *path)
{
    if (!ctx || !path) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->loaded) return kb_fail(ctx, KB_ESTATE, "no store loaded");
    cudaSetDevice(ctx->device);
    KB_TRY(ctx_quiesce(ctx));
    compact_streams_invalidate(ctx, "kb_dump");
    KB_TRY(store_compact_layout(ctx));  // the file holds the contiguous, key-ordered layout
    KB_TRY(hbuf_ensure(ctx, ctx->lane().h_stage, DUMP_STAGE));
    // the record directory lives on the device only: fetch it for the directory section
    const uint64_t n = ctx->st.n;
    HostDir d(n);
    if (n) {
        KB_CUDA(ctx, cudaMemcpyAsync(d.koff16.data(), ctx->st.koff16, n * 4, cudaMemcpyDeviceToHost, ctx->lane().stream));
        KB_CUDA(ctx, cudaMemcpyAsync(d.klen.data(), ctx->st.klen, n * 2, cudaMemcpyDeviceToHost, ctx->lane().stream));
        KB_CUDA(ctx, cudaMemcpyAsync(d.voff16.data(), ctx->st.voff16, n * 8, cudaMemcpyDeviceToHost, ctx->lane().stream));
        KB_CUDA(ctx, cudaMemcpyAsync(d.vlen.data(), ctx->st.vlen, n * 4, cudaMemcpyDeviceToHost, ctx->lane().stream));
        KB_CUDA(ctx, cudaStreamSynchronize(ctx->lane().stream));
    }
    d.koff16[n] = (uint32_t)ctx->kused16;
    d.voff16[n] = ctx->vused16;
    const std::string tmp = std::string(path) + ".tmp";
    FILE *f = fopen(tmp.c_str(), "wb");
    if (!f) return kb_fail(ctx, KB_EIO, "dump: cannot create %s", tmp.c_str());
    DumpHeader h;
    memset(&h, 0, sizeof(h));
    memcpy(h.magic, "KBB200D1", 8);
    h.version = 1;
    h.header_bytes = (uint32_t)sizeof(DumpHeader);
    h.n = n;
    h.key_chunks = ctx->kused16;
    h.val_chunks = ctx->vused16;
    h.compact_present = ctx->compact_present ? 1 : 0;
    h.compact_rev = ctx->compact_rev;
    h.max_kv_chunks = ctx->max_kv_chunks;
    int rc = KB_OK;
    if (fwrite(&h, 1, sizeof(h), f) != sizeof(h)) rc = kb_fail(ctx, KB_EIO, "dump: short write");
    uint64_t hd = 0xcbf29ce484222325ull;
    auto put = [&](const void *p, size_t bytes) {
        if (rc != KB_OK) return;
        hd = fnv1a64_update(hd, (const uint8_t *)p, bytes);
        if (bytes && fwrite(p, 1, bytes, f) != bytes) rc = kb_fail(ctx, KB_EIO, "dump: short write");
    };
    put(d.koff16.data(), (n + 1) * 4);
    put(d.klen.data(), n * 2);
    put(d.voff16.data(), (n + 1) * 8);
    put(d.vlen.data(), n * 4);
    h.sum_dir = hd;
    if (rc == KB_OK) rc = dump_section(ctx, f, ctx->d_kslab.p, nullptr, ctx->kused16 * 16, &h.sum_keys);
    if (rc == KB_OK) rc = dump_section(ctx, f, ctx->d_vslab.p, ctx->d_vslab.host, ctx->vused16 * 16, &h.sum_vals);
    if (rc == KB_OK && (fseek(f, 0, SEEK_SET) != 0 || fwrite(&h, 1, sizeof(h), f) != sizeof(h)))
        rc = kb_fail(ctx, KB_EIO, "dump: cannot finish the header");
    if (fclose(f) != 0 && rc == KB_OK) rc = kb_fail(ctx, KB_EIO, "dump: close failed");
    if (rc == KB_OK && rename(tmp.c_str(), path) != 0) rc = kb_fail(ctx, KB_EIO, "dump: cannot rename to %s", path);
    if (rc != KB_OK) remove(tmp.c_str());
    return rc;
}

extern "C" int kb_restore(kb_ctx *ctx, const char *path)
{
    if (!ctx || !path) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaSetDevice(ctx->device);
    KB_TRY(ctx_quiesce(ctx));
    compact_streams_invalidate(ctx, "kb_restore");
    FILE *f = fopen(path, "rb");
    if (!f) return kb_fail(ctx, KB_EIO, "restore: cannot open %s", path);
    struct Closer {
        FILE *f;
        ~Closer() { fclose(f); }
    } closer{f};
    DumpHeader h;
    if (fread(&h, 1, sizeof(h), f) != sizeof(h) || memcmp(h.magic, "KBB200D1", 8) != 0 || h.version != 1 ||
        h.header_bytes != sizeof(DumpHeader))
        return kb_fail(ctx, KB_EINVAL, "restore: %s is not a kb_b200 dump (version 1)", path);
    const uint64_t n = h.n;
    if (n >= 0xFFFFFFFEull || h.key_chunks > 0xFFFFFFF0ull) return kb_fail(ctx, KB_ELIMIT, "restore: dump exceeds the format limits");
    ctx->loaded = false;
    HostDir d(n);
    uint64_t hd = 0xcbf29ce484222325ull;
    bool ok = true;
    auto get = [&](void *p, size_t bytes) {
        if (!ok) return;
        if (bytes && fread(p, 1, bytes, f) != bytes) ok = false;
        else hd = fnv1a64_update(hd, (const uint8_t *)p, bytes);
    };
    get(d.koff16.data(), (n + 1) * 4);
    get(d.klen.data(), n * 2);
    get(d.voff16.data(), (n + 1) * 8);
    get(d.vlen.data(), n * 4);
    if (!ok) return kb_fail(ctx, KB_EINVAL, "restore: file truncated");
    if (hd != h.sum_dir) return kb_fail(ctx, KB_EINVAL, "restore: directory checksum mismatch");
    // the directory must describe exactly the slabs that follow: monotone offsets, every record inside its slab
    if (d.koff16[0] != 0 || d.voff16[0] != 0 || d.koff16[n] != h.key_chunks || d.voff16[n] != h.val_chunks) ok = false;
    uint64_t max_kv = 0;
    for (uint64_t i = 0; ok && i < n; i++) {
        const uint64_t nk = ((uint32_t)d.klen[i] + 15) / 16, nv = ((uint64_t)d.vlen[i] + 15) / 16;
        if (d.koff16[i + 1] < d.koff16[i] || d.koff16[i + 1] - d.koff16[i] != nk) ok = false;
        if (d.voff16[i + 1] < d.voff16[i] || d.voff16[i + 1] - d.voff16[i] != nv) ok = false;
        max_kv = std::max(max_kv, nk + nv);
    }
    if (!ok) return kb_fail(ctx, KB_EINVAL, "restore: inconsistent record directory");
    KB_TRY(hbuf_ensure(ctx, ctx->lane().h_stage, DUMP_STAGE));
    KB_TRY(store_alloc(ctx, d, n));
    uint64_t sk = 0, sv = 0;
    KB_TRY(restore_section(ctx, f, ctx->d_kslab.p, nullptr, h.key_chunks * 16, &sk));
    KB_TRY(restore_section(ctx, f, ctx->d_vslab.p, ctx->d_vslab.host, h.val_chunks * 16, &sv));
    if (sk != h.sum_keys || sv != h.sum_vals) return kb_fail(ctx, KB_EINVAL, "restore: slab checksum mismatch");
    KB_TRY(store_install(ctx, d, n, max_kv, "restore: "));
    ctx->compact_present = h.compact_present != 0;
    ctx->compact_rev = h.compact_rev;
    return KB_OK;
}
