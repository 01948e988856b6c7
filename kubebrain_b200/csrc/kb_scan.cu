// kb_scan.cu -- the MVCC range-scan, point-read and compaction-sweep path.  It only reads the snapshot (ctx->st, the
// slab bounds, store_gen); kb_store.cu builds and changes it.
//
// Replaces (reference file:line):
//   storage.Iter over badger            pkg/storage/badger/iter.go:27-98        -> HBM slab + k_search
//   coder.Decode                        pkg/backend/coder/normal.go:58-70       -> k_decode_lcp
//   worker.run (range + compact)        pkg/backend/scanner/scanner.go:389-516  -> k_decode_lcp, k_emit, k_place
//   commonResultReceiver (limit)        pkg/backend/scanner/receiver.go:62-103  -> k_tile_scan, k_place, k_gather
//
// Kernel pipeline for one batch of requests (streams: S2 = bound search, S = main, SG = copy stream):
//   k_search      [S2] (kb_search.cu) lower_bound of every [start,end) bound in the sorted slab (warp per bound,
//                 32-ary); the only step the host waits for before it lays the requests out as tiles
//   k_decode_lcp  [S] element-wise pass over the store's scan summary (kb_decode.cuh: LCP with the preceding key, decode /
//                 tombstone / value facts, revision): visibility at the request's read revision, TTL expiry, deleted-flag
//                 revision records -> one 32-bit meta word per record
//   k_emit        [S] per tile: segmented "last visible version" scan over the meta words (prev pointer + running
//                 min-LCP; the cross-tile carry by decoupled look-back) decides which record every key change emits /
//                 supersedes
//   k_tile_scan   [S] prefix sums of the per-tile counts / bytes (one CTA per 1024 tiles); k_req_totals: per-request rows
//   k_place       [S] ordered placement of the selection (limit applied) / ordered victim list
//   k_req_finalize [S] per-request prefix sums; publishes the per-request rows to mapped pinned memory (the host
//                 returns device-resident answers on that flag)
//   k_gather_jobs / k_wire_jobs [S] one copy job per emitted kv + the per-kv view arrays
//   k_gather / k_wire_copy [SG] bulk-TMA copy of the winners' key+value into the response arena (padded pairs, or
//                 etcd protobuf elements); overlaps the next batch's k_decode_lcp .. k_place
// A batch of point reads (backend.get, pkg/backend/range.go:81-121) is a lane batch too, all on the lane stream:
//   k_search -> k_get_resolve -> k_get_finalize -> k_gather (or k_wire_jobs -> k_wire_copy) -> k_publish_rout
// A compaction stream: the sweep (decode .. k_place_victims) and k_victim_capture at open; per page k_page_cut ->
// k_victim_jobs [S] -> k_gather [SG]
// Range partitions (kb_range_partitions): a range batch's decode .. k_place on the lane stream, then k_partition_cut [S]
// over the placement's arena offsets
#include <algorithm>
#include <memory>
#include <string_view>

#include "kb_internal.cuh"
#include "kb_decode.cuh"
#include "kb_wire.cuh"

namespace {


constexpr unsigned FULL = 0xffffffffu;

// ------------------------------------------------------------------------------------------------
// block-wide exclusive scan of the (last-prev slot, min-LCP-since) state
//   combine(A, B) = B.L != NONE ? B : (A.L, min(A.m, B.m))
// ------------------------------------------------------------------------------------------------
struct LM {
    uint32_t L, m;
};

__device__ __forceinline__ LM lm_combine(LM a, LM b)
{
    if (b.L != KB_NONE) return b;
    LM r;
    r.L = a.L;
    r.m = min(a.m, b.m);
    return r;
}

__device__ __forceinline__ LM block_excl_scan_lm(LM v, LM *warp_tot /* 8 */)
{
    const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    LM inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        LM o;
        o.L = __shfl_up_sync(FULL, inc.L, d);
        o.m = __shfl_up_sync(FULL, inc.m, d);
        if (lane >= (unsigned)d) inc = lm_combine(o, inc);
    }
    if (lane == 31) warp_tot[w] = inc;
    __syncthreads();
    LM ex;  // exclusive within the warp
    ex.L = __shfl_up_sync(FULL, inc.L, 1);
    ex.m = __shfl_up_sync(FULL, inc.m, 1);
    if (lane == 0) {
        ex.L = KB_NONE;
        ex.m = KB_LCP_INF;
    }
    LM pre;
    pre.L = KB_NONE;
    pre.m = KB_LCP_INF;
    for (unsigned k = 0; k < w; k++) pre = lm_combine(pre, warp_tot[k]);
    __syncthreads();
    return lm_combine(pre, ex);
}

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

// ------------------------------------------------------------------------------------------------
// k_emit: the worker.run state machine, data-parallel.
// For every TRIG record i with prev p = last PREVOK record before it (inside the request):
//   same key  <=> klen[i] == klen[p] && min LCP over (p, i] >= klen[i] - 9
//   range  : key change && rev[p] > 0 && value[p] != tombstone  -> emit p         (scanner.go:457-462)
//   compact: same key && rev[p] > 0                             -> p superseded   (scanner.go:463-469)
// After the last record of a request the trailing prev is emitted (scanner.go:503-507).
// tgt[i] = flat slot of the emitted (range) / superseded (compact) record, or NONE.
// tcnt[2t] = emissions (range) or delete calls (compact) of tile t; tcnt[2t+1] = response bytes (range) or object
// count (compact).
//
// The (last PREVOK slot, min LCP since) carry into a tile comes from DECOUPLED LOOK-BACK over per-tile states: a tile
// (taken in ticket order) publishes its own aggregate at once, then warp 0 reads the states of up to 32 preceding tiles
// of the request per step until it meets an inclusive prefix or a tile that holds a PREVOK record (nothing before such a
// tile can matter).  Round 1 walked the sub-tile aggregates backwards with one thread until it met a visible record: a
// scan whose records are mostly invisible (read revision below the versions, compact at an old revision) cost O(tiles)
// dependent loads per tile; now it costs one step per tile.
// (Resolving the output positions by look-back in the same pass -- one kernel instead of three -- was tried: with
// ~1 200 tiles of 1 024 records in flight every tile walked several windows back to the frontier of resolved prefixes,
// and the single pass was slower than emit + scan + place.)
// ------------------------------------------------------------------------------------------------
struct ReqOut {
    uint64_t total;        // emissions (range) / delete calls (compact)
    uint64_t total_aux;    // response bytes (range) / object count (compact)
    uint64_t capped_aux;   // response bytes of the first `limit` emissions (valid with KB_RO_CAPPED)
    uint32_t examined;     // records pulled from the iterator (valid with KB_RO_LIMIT_STOP, else hi - lo)
    uint32_t flags;
};
enum { KB_RO_LIMIT_STOP = 1u, KB_RO_CAPPED = 2u };

struct __align__(16) TileState {  // 32 bytes; zeroed by one memset per batch
    unsigned long long lm_agg, lm_pre;  // (last PREVOK slot | min LCP << 32): the tile alone / request start .. this tile
    uint32_t st_lm;                     // 0 empty, 1 aggregate valid, 2 inclusive prefix valid
    uint32_t pad[3];
};
enum { TS_EMPTY = 0, TS_AGG = 1, TS_PREFIX = 2 };

__device__ __forceinline__ unsigned long long lm_pack(LM v) { return ((unsigned long long)v.m << 32) | v.L; }
__device__ __forceinline__ LM lm_unpack(unsigned long long w)
{
    LM r;
    r.L = (uint32_t)w;
    r.m = (uint32_t)(w >> 32);
    return r;
}
__device__ __forceinline__ void ts_publish(uint32_t *status, uint32_t v)
{
    __threadfence();
    *(volatile uint32_t *)status = v;
}

// warp 0: exclusive (L, m) carry of tile t inside its request (tiles [t0, t))
__device__ __forceinline__ LM lookback_lm(TileState *ts, uint32_t t, uint32_t t0, uint32_t lane)
{
    LM acc;
    acc.L = KB_NONE;
    acc.m = KB_LCP_INF;
    for (uint32_t hi = t; hi > t0;) {  // this step looks at tiles hi-1, hi-2, .. (lane 0 = nearest)
        const bool in = lane < hi - t0;
        TileState *p = ts + (hi - 1 - (in ? lane : 0));
        uint32_t st;
        do {
            st = in ? *(volatile uint32_t *)&p->st_lm : (uint32_t)TS_PREFIX;
        } while (!__all_sync(FULL, st != TS_EMPTY));
        __threadfence();
        LM v;
        v.L = KB_NONE;
        v.m = KB_LCP_INF;
        if (in) v = lm_unpack(*(volatile unsigned long long *)(st == TS_PREFIX ? &p->lm_pre : &p->lm_agg));
        const unsigned term = __ballot_sync(FULL, in && (st == TS_PREFIX || v.L != KB_NONE));
        const uint32_t k = term ? (uint32_t)(__ffs(term) - 1) : 31u;  // farthest lane that still matters
        const uint32_t mm = __reduce_min_sync(FULL, (in && lane <= k) ? v.m : KB_LCP_INF);
        const uint32_t Lk = __shfl_sync(FULL, v.L, k);
        // combine(farther, nearer): nearer tiles (already in acc) hold no PREVOK, so only the minimum accumulates
        acc.m = min(acc.m, mm);
        if (term) {
            acc.L = Lk;
            break;
        }
        hi -= min(32u, hi - t0);
    }
    return acc;
}

template <bool COMPACT>
__global__ void __launch_bounds__(256, 8)  // <= 32 registers: eight CTAs per SM, room for other lanes' batches beside the copy
k_emit(StoreDev st, const ReqDev *__restrict__ reqs, const TileDev *__restrict__ tiles, const uint32_t *__restrict__ meta,
       TileState *__restrict__ ts, unsigned int *__restrict__ ticket, uint32_t *__restrict__ tgt,
       uint32_t *__restrict__ tail_tgt, uint64_t *__restrict__ tcnt, int wire, unsigned int *__restrict__ decode_ctr)
{
    __shared__ LM warp_tot[8];
    __shared__ LM carry_s, agg_s;
    __shared__ uint64_t ws2[18];
    __shared__ uint32_t tile_s;
    if (threadIdx.x == 0) tile_s = atomicAdd(ticket, 1u);  // ticket order: every preceding tile has started
    if (blockIdx.x == 0 && threadIdx.x == 0) *decode_ctr = 0;  // leave k_decode_lcp's work counter at zero
    __syncthreads();
    const uint32_t tix = tile_s;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const TileDev tile = tiles[tix];
    const ReqDev req = reqs[tile.req];
    const bool first_tile = tix == req.tile0, last_tile = tix == req.tile0 + req.ntiles - 1;
    TileState *my = ts + tix;
    const uint32_t base = threadIdx.x * 4;
    const uint32_t flat = tile.flat0 + base;
    uint32_t w[4];
    {
        uint4 mw = make_uint4(KB_LCP_INF, KB_LCP_INF, KB_LCP_INF, KB_LCP_INF);
        if (base < tile.n) mw = *(const uint4 *)(meta + flat);
        w[0] = base + 0 < tile.n ? mw.x : KB_LCP_INF;
        w[1] = base + 1 < tile.n ? mw.y : KB_LCP_INF;
        w[2] = base + 2 < tile.n ? mw.z : KB_LCP_INF;
        w[3] = base + 3 < tile.n ? mw.w : KB_LCP_INF;
    }
    LM mine;
    mine.L = KB_NONE;
    mine.m = KB_LCP_INF;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (w[k] & KB_M_PREVOK) {
            mine.L = flat + k;
            mine.m = KB_LCP_INF;
        } else {
            mine.m = min(mine.m, w[k] & KB_M_LCP_MASK);
        }
    }
    const LM ex = block_excl_scan_lm(mine, warp_tot);
    if (threadIdx.x == 255) agg_s = lm_combine(ex, mine);
    __syncthreads();
    if (warp == 0) {
        const LM agg = agg_s;
        LM carry;
        carry.L = KB_NONE;
        carry.m = KB_LCP_INF;
        bool resolved = first_tile;
        if (!first_tile) {
            // Fast path: the meta words in front of this tile are complete (the decode pass has finished), so the last
            // PREVOK record is looked for directly in the 256 records before the tile -- 32 per step, nearest first.
            // Almost every tile ends here without waiting for anybody.
            for (uint32_t back = 0; back < 256 && !resolved; back += 32) {
                const uint32_t wd = meta[tile.flat0 - 1 - back - lane];  // lane 0 = the record right in front
                const unsigned pm = __ballot_sync(FULL, wd & KB_M_PREVOK);
                const uint32_t k = pm ? (uint32_t)(__ffs(pm) - 1) : 32u;  // nearest PREVOK lane; records nearer than it count
                const uint32_t mm = __reduce_min_sync(FULL, lane < k ? (wd & KB_M_LCP_MASK) : KB_LCP_INF);
                carry.m = min(carry.m, mm);
                if (pm) {
                    carry.L = tile.flat0 - 1 - back - k;
                    resolved = true;
                }
            }
        }
        if (resolved) {
            if (lane == 0) {
                my->lm_pre = lm_pack(lm_combine(carry, agg));
                ts_publish(&my->st_lm, TS_PREFIX);
            }
        } else {
            // long run without a visible record: decoupled look-back over the tile states
            if (lane == 0) {
                my->lm_agg = lm_pack(agg);
                ts_publish(&my->st_lm, TS_AGG);
            }
            carry = lookback_lm(ts, tix, req.tile0, lane);
            if (lane == 0) {
                my->lm_pre = lm_pack(lm_combine(carry, agg));
                ts_publish(&my->st_lm, TS_PREFIX);
            }
        }
        if (lane == 0) carry_s = carry;
    }
    __syncthreads();
    LM x = lm_combine(carry_s, ex);

    uint64_t cnt = 0, aux = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (base + k >= tile.n) break;
        const uint32_t i = flat + k;
        const uint32_t word = w[k];
        uint32_t t = KB_NONE;
        if (word & KB_M_TRIG) {
            if (x.L != KB_NONE) {
                const uint32_t mm = min(x.m, word & KB_M_LCP_MASK);
                const uint32_t irec = req.lo + (i - req.flat0), prec = req.lo + (x.L - req.flat0);
                const uint32_t pw = meta[x.L];
                const uint32_t kl = st.klen[irec], pkl = st.klen[prec];
                const bool same = (kl == pkl) && (mm >= kl - 9);
                if (!same) {
                    if (!(pw & KB_M_REV0) && !(pw & KB_M_TOMB)) {
                        if (COMPACT) {
                            aux++;  // count++ only
                        } else {
                            t = x.L;
                            cnt++;
                            aux += kv_resp_bytes(st, prec, wire);
                        }
                    }
                } else if (COMPACT && !(pw & KB_M_REV0)) {
                    t = x.L;  // superseded version
                    cnt++;
                }
            }
            if (COMPACT) {
                if (word & KB_M_TOMB) cnt++;
                if (word & KB_M_REVDEL) cnt++;
            }
        }
        if (COMPACT && (word & (KB_M_TTLREV | KB_M_TTLOBJ))) cnt++;
        if (word & KB_M_PREVOK) {
            x.L = i;
            x.m = KB_LCP_INF;
        } else {
            x.m = min(x.m, word & KB_M_LCP_MASK);
        }
        tgt[i] = t;
        if (last_tile && base + k == tile.n - 1) {
            // end of the request's iterator: the trailing prev (scanner.go:503-507)
            uint32_t tt = KB_NONE;
            if (x.L != KB_NONE) {
                const uint32_t pw = meta[x.L];
                if (!(pw & KB_M_REV0) && !(pw & KB_M_TOMB)) {
                    if (COMPACT) {
                        aux++;
                    } else {
                        const uint32_t prec = req.lo + (x.L - req.flat0);
                        tt = x.L;
                        cnt++;
                        aux += kv_resp_bytes(st, prec, wire);
                    }
                }
            }
            tail_tgt[tile.req] = tt;
        }
    }
    uint64_t ea, eb, ta, tb;
    block_excl_scan2(cnt, aux, ea, eb, ta, tb, ws2);
    if (threadIdx.x == 0) {
        tcnt[2 * tix] = ta;
        tcnt[2 * tix + 1] = tb;
    }
}

// tile table from the request table: tile t belongs to the last request whose tile0 <= t (requests without records own
// no tile; their tile0 equals their successor's)
__global__ void __launch_bounds__(256)
k_fill_tiles(const ReqDev *__restrict__ reqs, uint32_t nreq, uint32_t nt, TileDev *__restrict__ tiles)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    uint32_t lo = 0, hi = nreq;  // invariant: reqs[lo].tile0 <= t
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (reqs[mid].tile0 <= t) lo = mid; else hi = mid;
    }
    const ReqDev r = reqs[lo];  // among equal tile0 the LAST request is found: the one that really owns tile t
    const uint32_t k = t - r.tile0, n = r.hi - r.lo;
    TileDev td;
    td.req = lo;
    td.rec0 = r.lo + k * KB_TILE;
    td.n = min((uint32_t)KB_TILE, n - k * KB_TILE);
    td.flat0 = r.flat0 + k * KB_TILE;
    td.lo = r.lo;
    td.pad = 0;
    td.read_rev = r.read_rev;
    tiles[t] = td;
}

// ------------------------------------------------------------------------------------------------
// k_tile_scan: exclusive prefix of the per-tile (count, aux) pairs over ALL tiles of the batch, tscan[2 * (T + 1)].
// One CTA per chunk of 1024 tiles (rather than one CTA for everything): a chunk scans its tiles,
// publishes its total, and adds the totals of the chunks in front of it (at most a few hundred: plain look-back).
// ------------------------------------------------------------------------------------------------
struct __align__(16) ChunkState {
    unsigned long long cnt, aux;
    uint32_t ready;
    uint32_t pad[3];
};

__global__ void __launch_bounds__(256, 8)  // <= 32 registers: eight CTAs per SM, room for other lanes' batches beside the copy
k_tile_scan(const uint64_t *__restrict__ tcnt, uint64_t *__restrict__ tscan, uint32_t ntiles, ChunkState *__restrict__ cs)
{
    __shared__ uint64_t ws2[18];
    __shared__ uint64_t base_s[2];
    const uint32_t c = blockIdx.x, t0 = c * 1024 + threadIdx.x * 4;
    uint64_t a[4], b[4], sa = 0, sb = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        a[k] = t0 + k < ntiles ? tcnt[2 * (t0 + k)] : 0;
        b[k] = t0 + k < ntiles ? tcnt[2 * (t0 + k) + 1] : 0;
        sa += a[k];
        sb += b[k];
    }
    uint64_t ea, eb, ta, tb;
    block_excl_scan2(sa, sb, ea, eb, ta, tb, ws2);
    if (threadIdx.x == 0) {
        cs[c].cnt = ta;
        cs[c].aux = tb;
        ts_publish(&cs[c].ready, 1u);
    }
    if (threadIdx.x < 32) {
        // totals of the chunks in front, 32 at a time (each is ready as soon as its own 1024 counts are summed)
        const uint32_t lane = threadIdx.x;
        uint64_t pa = 0, pb = 0;
        for (uint32_t p0 = 0; p0 < c; p0 += 32) {
            const uint32_t p = p0 + lane;
            if (p < c) {
                while (*(volatile uint32_t *)&cs[p].ready == 0) {}
                __threadfence();
                pa += *(volatile unsigned long long *)&cs[p].cnt;
                pb += *(volatile unsigned long long *)&cs[p].aux;
            }
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            pa += __shfl_xor_sync(FULL, pa, d);
            pb += __shfl_xor_sync(FULL, pb, d);
        }
        if (lane == 0) {
            base_s[0] = pa;
            base_s[1] = pb;
        }
    }
    __syncthreads();
    uint64_t ra = base_s[0] + ea, rb = base_s[1] + eb;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (t0 + k < ntiles) {
            tscan[2 * (t0 + k)] = ra;
            tscan[2 * (t0 + k) + 1] = rb;
        }
        ra += a[k];
        rb += b[k];
        if (t0 + k == ntiles - 1) {
            tscan[2 * ntiles] = ra;
            tscan[2 * ntiles + 1] = rb;
        }
    }
}

// per-request totals from the tile prefix sums; every field of the row is written (no memset needed)
__global__ void __launch_bounds__(256)
k_req_totals(const ReqDev *__restrict__ reqs, uint32_t nreq, const uint64_t *__restrict__ tscan, ReqOut *__restrict__ rout)
{
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nreq) return;
    const ReqDev r = reqs[q];
    ReqOut o;
    o.total = o.total_aux = 0;
    if (r.ntiles) {
        o.total = tscan[2 * (r.tile0 + r.ntiles)] - tscan[2 * r.tile0];
        o.total_aux = tscan[2 * (r.tile0 + r.ntiles) + 1] - tscan[2 * r.tile0 + 1];
    }
    o.capped_aux = 0;
    o.examined = 0;
    o.flags = 0;
    rout[q] = o;
}

// ------------------------------------------------------------------------------------------------
// k_place: ordered selection (range) -- position = emissions before it in the request; the first `limit`
// positions are kept (commonResultReceiver.needMore, receiver.go:82-87).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, 8)  // <= 32 registers: eight CTAs per SM, room for other lanes' batches beside the copy
k_place(StoreDev st, const ReqDev *__restrict__ reqs, const TileDev *__restrict__ tiles,
        const uint32_t *__restrict__ tgt, const uint32_t *__restrict__ tail_tgt,
        const uint64_t *__restrict__ tscan, uint32_t *__restrict__ sel, uint64_t *__restrict__ slot,
        ReqOut *__restrict__ rout, int wire)
{
    __shared__ uint64_t ws2[18];
    const TileDev tile = tiles[blockIdx.x];
    const ReqDev req = reqs[tile.req];
    const uint32_t base = threadIdx.x * 4;
    const uint32_t flat = tile.flat0 + base;
    const bool last_tile = (blockIdx.x == req.tile0 + req.ntiles - 1);
    uint32_t t[5];
    uint32_t sz[5];
    uint64_t cnt = 0, bytes = 0;
#pragma unroll
    for (int k = 0; k < 5; k++) {
        t[k] = KB_NONE;
        sz[k] = 0;
    }
    if (base < tile.n) {
        uint4 tw = *(const uint4 *)(tgt + flat);
        t[0] = tw.x;
        t[1] = base + 1 < tile.n ? tw.y : KB_NONE;
        t[2] = base + 2 < tile.n ? tw.z : KB_NONE;
        t[3] = base + 3 < tile.n ? tw.w : KB_NONE;
        if (last_tile && tile.n - 1 >= base && tile.n - 1 < base + 4) t[4] = tail_tgt[tile.req];
    }
#pragma unroll
    for (int k = 0; k < 5; k++) {
        if (t[k] != KB_NONE) {
            const uint32_t prec = req.lo + (t[k] - req.flat0);
            sz[k] = (uint32_t)kv_resp_bytes(st, prec, wire);
            cnt++;
            bytes += sz[k];
        }
    }
    uint64_t ea, eb, ta, tb;
    block_excl_scan2(cnt, bytes, ea, eb, ta, tb, ws2);
    uint64_t pos = tscan[2 * blockIdx.x] - tscan[2 * req.tile0] + ea;
    uint64_t off = tscan[2 * blockIdx.x + 1] - tscan[2 * req.tile0 + 1] + eb;
    const bool limited = req.limit > 0;
#pragma unroll
    for (int k = 0; k < 5; k++) {
        if (t[k] == KB_NONE) continue;
        if (!limited || pos < (uint64_t)req.limit) {
            sel[req.sel_base + pos] = req.lo + (t[k] - req.flat0);
            slot[req.sel_base + pos] = off;
            if (limited && pos == (uint64_t)req.limit - 1) {
                rout[tile.req].capped_aux = off + sz[k];
                uint32_t fl = KB_RO_CAPPED;
                if (k < 4) {
                    // the limit-th append happened inside the loop: the iterator stops here (Q4)
                    rout[tile.req].examined = (flat + k) - req.flat0 + 1;
                    fl |= KB_RO_LIMIT_STOP;
                }
                rout[tile.req].flags = fl;
            }
        }
        pos++;
        off += sz[k];
    }
}

// ordered delete calls (compact): per record [superseded prev] [tombstone] [revision record] | [ttl]
__global__ void __launch_bounds__(256, 8)  // <= 32 registers: eight CTAs per SM, room for other lanes' batches beside the copy
k_place_victims(const ReqDev *__restrict__ reqs, const TileDev *__restrict__ tiles,
                const uint32_t *__restrict__ meta, const uint32_t *__restrict__ tgt,
                const uint64_t *__restrict__ tscan, uint32_t *__restrict__ vidx, uint8_t *__restrict__ vcls)
{
    __shared__ uint64_t ws2[18];
    const TileDev tile = tiles[blockIdx.x];
    const ReqDev req = reqs[tile.req];
    const uint32_t base = threadIdx.x * 4;
    const uint32_t flat = tile.flat0 + base;
    uint32_t t[4], w[4];
    uint64_t cnt = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        t[k] = KB_NONE;
        w[k] = 0;
    }
    if (base < tile.n) {
        const uint4 tw = *(const uint4 *)(tgt + flat), mw = *(const uint4 *)(meta + flat);
        t[0] = tw.x, w[0] = mw.x;
        if (base + 1 < tile.n) t[1] = tw.y, w[1] = mw.y;
        if (base + 2 < tile.n) t[2] = tw.z, w[2] = mw.z;
        if (base + 3 < tile.n) t[3] = tw.w, w[3] = mw.w;
    }
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (t[k] != KB_NONE) cnt++;
        if ((w[k] & KB_M_TRIG) && (w[k] & KB_M_TOMB)) cnt++;
        if (w[k] & KB_M_REVDEL) cnt++;
        if (w[k] & (KB_M_TTLREV | KB_M_TTLOBJ)) cnt++;
    }
    uint64_t ea, eb, ta, tb;
    block_excl_scan2(cnt, 0, ea, eb, ta, tb, ws2);
    uint64_t pos = req.sel_base + tscan[2 * blockIdx.x] - tscan[2 * req.tile0] + ea;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        if (base + k >= tile.n) break;
        const uint32_t irec = req.lo + (flat + k - req.flat0);
        if (t[k] != KB_NONE) {
            vidx[pos] = req.lo + (t[k] - req.flat0);
            vcls[pos++] = KB_V_SUPERSEDED;
        }
        if ((w[k] & KB_M_TRIG) && (w[k] & KB_M_TOMB)) {
            vidx[pos] = irec;
            vcls[pos++] = KB_V_TOMBSTONE;
        }
        if (w[k] & KB_M_REVDEL) {
            vidx[pos] = irec;
            vcls[pos++] = KB_V_REVRECORD;
        }
        if (w[k] & KB_M_TTLREV) {
            vidx[pos] = irec;
            vcls[pos++] = KB_V_TTL_REVREC;
        }
        if (w[k] & KB_M_TTLOBJ) {
            vidx[pos] = irec;
            vcls[pos++] = KB_V_TTL_OBJECT;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// k_gather: one warp per emitted kv; key (internal key, padded) then value (padded), 16-byte vector copies
// ------------------------------------------------------------------------------------------------
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

__global__ void __launch_bounds__(256)
k_gather_jobs(StoreDev st, const ReqDev *__restrict__ reqs, uint32_t nreq, const uint64_t *__restrict__ job_first,
              const uint64_t *__restrict__ arena_base, const uint32_t *__restrict__ sel,
              const uint64_t *__restrict__ slot, GatherJob *__restrict__ jobs, GatherOut out)
{
    const uint64_t n_kvs = job_first[nreq];  // written by k_req_finalize
    for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n_kvs; k += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = nreq;  // request of kv k: last q with job_first[q] <= k
    while (hi - lo > 1) {
        uint32_t mid = (lo + hi) >> 1;
        if (job_first[mid] <= k) lo = mid; else hi = mid;
    }
    const uint32_t q = lo;
    const uint64_t s = reqs[q].sel_base + (k - job_first[q]);
    const uint32_t rec = sel[s];
    const uint64_t dst_byte = arena_base[q] + slot[s];
    const uint32_t kl = st.klen[rec], vl = st.vlen[rec];
    GatherJob j;
    j.dst16 = dst_byte >> 4;
    j.vsrc16 = st.voff16[rec];
    j.ksrc16 = st.koff16[rec];
    j.nk = (kl + 15) >> 4;
    j.nv = (vl + 15) >> 4;
    j.kl = kl;
    jobs[k] = j;
    out.rec_idx[k] = rec;
    out.key_off[k] = dst_byte + 4;
    out.key_len[k] = kl - 13;
    out.val_off[k] = dst_byte + (uint64_t)j.nk * 16;
    out.val_len[k] = vl;
    out.rev[k] = be64_bytes((const uint8_t *)(st.kslab + j.ksrc16) + kl - 8);
    }
}

// ---- k_gather: copy of every winner's [internal key, padded][value, padded] into the response arena, staged through
// registers.  One warp per kv: every lane loads up to GATHER_U 16-byte chunks of the pair (all loads of a round are
// issued before its first store), then stores them; a kv larger than 32 x GATHER_U chunks takes several rounds.  Blocks
// of 32 jobs are handed out through a global counter (zeroed by the kernel that builds the jobs), so a CTA that starts
// late -- the SM was still busy with another stream's kernel -- simply takes fewer blocks.
// No shared memory and 40 registers: the copy runs beside the next batch's short kernels and the fan-out CTA instead of
// holding the SM's shared memory (the bulk-TMA ring it replaces held 2 x 111 KB per SM), and on a 2 320-byte kv it is
// faster with the GPU to itself too (profiles/h100_ab_gather.txt).
constexpr int GATHER_WARPS = 8;
constexpr int GATHER_U = 5;  // chunks per lane and round: 160 chunks (2560 B), a typical kv in one round

__device__ __forceinline__ uint4 ldg_evict_first(const uint4 *p, uint64_t pol)
{
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p), "l"(pol));
    return r;
}
__device__ __forceinline__ void stg_evict_first(uint4 *p, const uint4 &v, uint64_t pol)
{
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y),
                 "r"(v.z), "r"(v.w), "l"(pol)
                 : "memory");
}

__global__ void __launch_bounds__(GATHER_WARPS * 32, 6)  // 40 registers: two CTAs fit beside the fan-out CTA and the short kernels
k_gather(StoreDev st, const GatherJob *__restrict__ jobs, const uint64_t *__restrict__ n_kvs_dev, uint4 *__restrict__ arena,
         unsigned long long *__restrict__ work_ctr)
{
    static_assert(sizeof(GatherJob) == 32, "lanes 0..7 hold the eight words of a job");
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_kvs = *n_kvs_dev;
    const uint64_t l2pol = l2_evict_first_policy();  // both directions stream: the copy must not flush L2 for its neighbours
    for (;;) {
        unsigned long long b = 0;
        if (lane == 0) b = atomicAdd(work_ctr, 32ull);
        const uint64_t base = __shfl_sync(0xffffffffu, b, 0);
        if (base >= n_kvs) break;
        const uint32_t cnt = n_kvs - base < 32 ? (uint32_t)(n_kvs - base) : 32u;
        // word (lane & 7) of the current job; the next kv's is loaded while this one is copied
        const uint32_t *jw = (const uint32_t *)(jobs + base) + (lane & 7);
        uint32_t w = __ldg(jw);
        for (uint32_t j = 0; j < cnt; j++) {
            const uint64_t dst16 = ((uint64_t)__shfl_sync(0xffffffffu, w, 1) << 32) | __shfl_sync(0xffffffffu, w, 0);
            const uint64_t vsrc16 = ((uint64_t)__shfl_sync(0xffffffffu, w, 3) << 32) | __shfl_sync(0xffffffffu, w, 2);
            const uint32_t ksrc16 = __shfl_sync(0xffffffffu, w, 4);
            const uint32_t nk = __shfl_sync(0xffffffffu, w, 5), n = nk + __shfl_sync(0xffffffffu, w, 6);
            if (j + 1 < cnt) w = __ldg(jw + 8 * (j + 1));
            for (uint32_t c0 = 0; c0 < n; c0 += 32 * GATHER_U) {
                uint4 v[GATHER_U];
#pragma unroll
                for (int u = 0; u < GATHER_U; u++) {
                    const uint32_t c = c0 + lane + 32 * u;
                    if (c < n) v[u] = ldg_evict_first(c < nk ? st.kslab + ksrc16 + c : st.vslab + vsrc16 + (c - nk), l2pol);
                }
#pragma unroll
                for (int u = 0; u < GATHER_U; u++) {
                    const uint32_t c = c0 + lane + 32 * u;
                    if (c < n) stg_evict_first(arena + dst16 + c, v[u], l2pol);
                }
            }
        }
    }
}

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

// ================================================================================================
// host orchestration
// ================================================================================================
kb_result *kb_result_new(ResultKind kind, int out_mode)
{
    kb_result *r = new kb_result();
    r->kind = kind;
    r->out_mode = out_mode;
    return r;
}

// the device meta and arena back to their pools
static void result_put_device(kb_ctx *ctx, kb_result *res)
{
    pool_put_dev(ctx, res->d_meta);
    res->d_meta = DBuf();
    pool_put_arena(ctx, res->d_arena, res->kind == ResultKind::point_read);
    res->d_arena = DBuf();
}

void result_release_locked(kb_ctx *ctx, kb_result *res)
{
    if (!res) return;
    if (ctx) {
        pool_put_host(ctx, res->h_meta);
        pool_put_host(ctx, res->h_arena);
        result_put_device(ctx, res);
        if (res->done_ev) ctx->ev_pool.push_back(res->done_ev);
    }
    delete res;
}

int result_to_host(kb_ctx *ctx, kb_result *res, cudaStream_t s, std::initializer_list<D2HPiece> pieces,
                   uint64_t arena_bytes, const char *what)
{
    size_t meta = 0;
    for (const D2HPiece &p : pieces) meta += p.bytes;
    int rc = KB_OK;
    cudaError_t e = res->done_ev ? cudaStreamWaitEvent(s, res->done_ev, 0) : cudaSuccess;
    if (meta) {
        pool_put_host(ctx, res->h_meta);
        res->h_meta = HBuf();
        rc = pool_get_host(ctx, meta + 64, &res->h_meta);
    }
    if (rc == KB_OK && arena_bytes) rc = pool_get_host(ctx, arena_bytes + 16, &res->h_arena);
    if (rc == KB_OK) {
        size_t off = 0;
        for (const D2HPiece &p : pieces) {
            if (p.bytes && e == cudaSuccess)
                e = cudaMemcpyAsync((uint8_t *)res->h_meta.p + off, p.src, p.bytes, cudaMemcpyDeviceToHost, s);
            off += p.bytes;
        }
        if (arena_bytes && e == cudaSuccess)
            e = cudaMemcpyAsync(res->h_arena.p, res->d_arena.p, arena_bytes, cudaMemcpyDeviceToHost, s);
    }
    const cudaError_t es = cudaStreamSynchronize(s);  // also after a failure: nothing may still be writing the buffers
    if (e == cudaSuccess) e = es;
    if (rc == KB_OK && e != cudaSuccess) rc = kb_cuda_fail(ctx, e, what);
    result_put_device(ctx, res);
    return rc;
}

extern "C" void kb_result_free(kb_ctx *ctx, kb_result *res)
{
    if (!res) return;
    if (ctx) {
        std::lock_guard<std::mutex> g(ctx->mu);
        result_release_locked(ctx, res);
    } else {
        delete res;
    }
}

namespace {

struct Resolved {
    std::vector<ReqDev> reqs;
    uint32_t nt = 0;  // tiles of the batch (the tile table itself is filled on the device, k_fill_tiles)
    uint64_t total_flat = 0, total_sel = 0, key_bytes = 0, n_records = 0;
};

// lay the requests ([lo,hi) already known) out as tiles of KB_TILE records that never span two requests
int layout_requests(kb_ctx *ctx, bool cap_by_limit, Resolved &R)
{
    R.n_records = 0;
    uint64_t flat = 0, selb = 0, nt = 0;
    for (size_t q = 0; q < R.reqs.size(); q++) {
        ReqDev &r = R.reqs[q];
        r.flat0 = (uint32_t)flat;
        r.tile0 = (uint32_t)nt;
        uint32_t n = r.hi - r.lo;
        r.ntiles = (n + KB_TILE - 1) / KB_TILE;
        r.sel_base = (uint32_t)selb;
        nt += r.ntiles;
        flat += (uint64_t)r.ntiles * KB_TILE;
        uint64_t cap = n;
        if (cap_by_limit && r.limit > 0) cap = std::min<uint64_t>(cap, (uint64_t)r.limit);
        selb += cap;
        R.n_records += n;
        if (flat >= 0xFFFFF000ull || selb >= 0xFFFFF000ull)
            return kb_fail(ctx, KB_ELIMIT, "batch examines more than 2^32 records; split it");
    }
    R.total_flat = flat;
    R.total_sel = selb;
    R.nt = (uint32_t)nt;
    return KB_OK;
}

// the bound search (or the one kb_range_prefetch started for exactly these bounds), then the requests laid out as tiles
int resolve_requests(kb_ctx *ctx, ScanLane &L, const kb_range_req *reqs, uint64_t nreq, bool cap_by_limit, Resolved &R,
                     kb_tp *tseg = nullptr)
{
    const uint32_t *hres = nullptr;
    KB_TRY(range_bounds_find(ctx, L, reqs, nreq, &hres, tseg));
    R.reqs.resize(nreq);
    for (uint64_t q = 0; q < nreq; q++) {
        ReqDev &r = R.reqs[q];
        r.lo = hres[2 * q];
        r.hi = std::max(hres[2 * q + 1], r.lo);
        r.read_rev = reqs[q].read_rev;
        r.limit = reqs[q].limit;
    }
    return layout_requests(ctx, cap_by_limit, R);
}

// the tile table starts on a 32-byte boundary behind the lane's `nreq` requests; only the requests travel, the device
// derives the tiles from them (a 100M-record sweep has 97 656 tiles: 0.4 ms of host loop + 3 MB of upload in round 1)
size_t tile_table_off(size_t nreq) { return (nreq * sizeof(ReqDev) + 31) & ~(size_t)31; }
TileDev *tile_table(const ScanLane &L, size_t nreq) { return (TileDev *)((uint8_t *)L.d_reqs.p + tile_table_off(nreq)); }

int upload_layout(kb_ctx *ctx, ScanLane &L, const Resolved &R)
{
    const size_t nreq = R.reqs.size(), nt = R.nt;
    KB_TRY(dbuf_ensure(ctx, L.d_reqs, tile_table_off(nreq) + std::max<size_t>(nt, 1) * sizeof(TileDev) + 64));
    KB_TRY(dbuf_ensure(ctx, L.d_meta, std::max<uint64_t>(R.total_flat, 4) * 4));
    KB_TRY(dbuf_ensure(ctx, L.d_tgt, std::max<uint64_t>(R.total_flat, 4) * 4 + nreq * 4 + 16));
    // one zeroed region per batch: [ticket, padded to 64 bytes][one ChunkState per 1024 tiles][one TileState per tile]
    KB_TRY(dbuf_ensure(ctx, L.d_tscan, 64 + (std::max<size_t>(nt, 1) / 1024 + 1) * sizeof(ChunkState) +
                                           std::max<size_t>(nt, 1) * sizeof(TileState)));
    KB_TRY(dbuf_ensure(ctx, L.d_tcnt, (std::max<size_t>(nt, 1) * 2 + (nt + 1) * 2) * 8));  // tcnt | tscan
    KB_TRY(dbuf_ensure(ctx, L.d_reqout, std::max<size_t>(nreq, 1) * sizeof(ReqOut)));
    // pinned staging so the async copies really are asynchronous
    const size_t bytes = nreq * sizeof(ReqDev);
    KB_TRY(hbuf_ensure(ctx, L.h_stage2, bytes + 64));
    uint8_t *h = (uint8_t *)L.h_stage2.p;
    memcpy(h, R.reqs.data(), bytes);
    if (bytes) KB_CUDA(ctx, cudaMemcpyAsync(L.d_reqs.p, h, bytes, cudaMemcpyHostToDevice, L.stream));
    if (nt)
        KB_LAUNCH_S(ctx, L.stream, "k_fill_tiles", nt * 32,
                    (k_fill_tiles<<<(unsigned)((nt + 255) / 256), 256, 0, L.stream>>>((const ReqDev *)L.d_reqs.p, (uint32_t)nreq,
                                                                                      (uint32_t)nt, tile_table(L, nreq))));
    return KB_OK;
}

}  // namespace

// the per-batch pass over the scan summary: one CTA per tile (kb_decode.cuh)
static int launch_decode(kb_ctx *ctx, cudaStream_t strm, uint32_t ntiles, uint64_t n_rec, const ScanMode &mode,
                         const TileDev *d_tiles, uint32_t *d_meta)
{
    // 12 bytes of summary read (the revision only for decodable keys) and the 4-byte meta word written per record
    KB_LAUNCH_S(ctx, strm, "k_decode_lcp", n_rec * 16,
                (k_decode_lcp<<<ntiles, 256, 0, strm>>>(ctx->st, d_tiles, mode, d_meta)));
    return KB_OK;
}

// gather of `n_jobs` (upper bound; the count is the table's kvs) copy jobs into `arena`
static int launch_gather(kb_ctx *ctx, cudaStream_t strm, const GatherJob *d_jobs, const JobTable &tab, uint4 *arena,
                         uint64_t n_jobs, uint64_t alg_bytes)
{
    // two CTAs per SM (16 warps, one 2.3 KB kv each in flight) reach the copy rate; a third takes HBM from the fan-out,
    // and one showed no gain (profiles/h100_ab.txt)
    const unsigned ggrid =
        (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((n_jobs + GATHER_WARPS * 32 - 1) / (GATHER_WARPS * 32), 2 * ctx->n_sms));
    KB_LAUNCH_S(ctx, strm, "k_gather", alg_bytes,
                (k_gather<<<ggrid, GATHER_WARPS * 32, 0, strm>>>(ctx->st, d_jobs, tab.n_kvs(), arena, tab.work_ctr)));
    return KB_OK;
}

// decode -> emit -> tile scan -> request totals -> (place) for a layout uploaded to lane L; everything stays enqueued on
// L.stream.  Range: the selection goes to L.d_sel / d_slot; compact: the delete calls go to vidx / vcls.
static int launch_scan_core(kb_ctx *ctx, ScanLane &L, const Resolved &R, const ScanMode &mode, bool with_place,
                            uint32_t *vidx = nullptr, uint8_t *vcls = nullptr)
{
    const uint32_t nt = R.nt;
    const uint32_t nreq = (uint32_t)R.reqs.size();
    const ReqDev *d_reqs = (const ReqDev *)L.d_reqs.p;
    const TileDev *d_tiles = tile_table(L, nreq);
    uint32_t *d_meta = (uint32_t *)L.d_meta.p;
    uint32_t *d_tgt = (uint32_t *)L.d_tgt.p;
    uint32_t *d_tail = d_tgt + std::max<uint64_t>(R.total_flat, 4);
    const uint32_t nchunks = nt / 1024 + 1;
    unsigned int *d_ticket = (unsigned int *)L.d_tscan.p;
    ChunkState *d_cs = (ChunkState *)((uint8_t *)L.d_tscan.p + 64);
    TileState *d_ts = (TileState *)(d_cs + nchunks);
    uint64_t *d_tcnt = (uint64_t *)L.d_tcnt.p, *d_tscan = d_tcnt + (size_t)std::max<uint32_t>(nt, 1) * 2;
    ReqOut *d_rout = (ReqOut *)L.d_reqout.p;
    const uint32_t ctr_base = 64 + 16 * (uint32_t)(&L - ctx->lanes);  // this lane's work counters
    if (nt) {
        // the ticket and the look-back states start empty
        KB_CUDA(ctx, cudaMemsetAsync(L.d_tscan.p, 0, 64 + (size_t)nchunks * sizeof(ChunkState) + (size_t)nt * sizeof(TileState),
                                     L.stream));
        KB_TRY(launch_decode(ctx, L.stream, nt, R.n_records, mode, d_tiles, d_meta));
        if (mode.compact) {
            KB_LAUNCH_S(ctx, L.stream, "k_emit_compact", R.n_records * 8,
                        (k_emit<true><<<nt, 256, 0, L.stream>>>(ctx->st, d_reqs, d_tiles, d_meta, d_ts, d_ticket, d_tgt, d_tail,
                                                                d_tcnt, 0, (unsigned int *)ctx->d_ctrs.p + ctr_base)));
        } else {
            KB_LAUNCH_S(ctx, L.stream, "k_emit", R.n_records * 8,
                        (k_emit<false><<<nt, 256, 0, L.stream>>>(ctx->st, d_reqs, d_tiles, d_meta, d_ts, d_ticket, d_tgt, d_tail,
                                                                 d_tcnt, mode.wire, (unsigned int *)ctx->d_ctrs.p + ctr_base)));
        }
        KB_LAUNCH_S(ctx, L.stream, "k_tile_scan", (uint64_t)nt * 32,
                    (k_tile_scan<<<nchunks, 256, 0, L.stream>>>(d_tcnt, d_tscan, nt, d_cs)));
    }
    if (nreq)
        KB_LAUNCH_S(ctx, L.stream, "k_req_totals", (uint64_t)nreq * 64,
                    (k_req_totals<<<(nreq + 255) / 256, 256, 0, L.stream>>>(d_reqs, nreq, d_tscan, d_rout)));
    if (nt && with_place) {
        if (mode.compact) {
            KB_LAUNCH_S(ctx, L.stream, "k_place_victims", R.n_records * 8,
                        (k_place_victims<<<nt, 256, 0, L.stream>>>(d_reqs, d_tiles, d_meta, d_tgt, d_tscan, vidx, vcls)));
        } else {
            KB_LAUNCH_S(ctx, L.stream, "k_place", R.n_records * 4,
                        (k_place<<<nt, 256, 0, L.stream>>>(ctx->st, d_reqs, d_tiles, d_tgt, d_tail, d_tscan,
                                                           (uint32_t *)L.d_sel.p, (uint64_t *)L.d_slot.p, d_rout,
                                                           mode.wire)));
        }
    }
    KB_CUDA(ctx, cudaGetLastError());
    return KB_OK;
}

// the selection arrays k_place writes for a range layout
static int sel_ensure(kb_ctx *ctx, ScanLane &L, const Resolved &R)
{
    KB_TRY(dbuf_ensure(ctx, L.d_sel, std::max<uint64_t>(R.total_sel, 1) * 4));
    return dbuf_ensure(ctx, L.d_slot, std::max<uint64_t>(R.total_sel, 1) * 8);
}

// A scan whose request rows the host reads at once: R's layout is uploaded to lane L (with its selection arrays for a
// range), scanned, and the rows come back through L.h_stage once the lane stream has drained
static int scan_sync(kb_ctx *ctx, ScanLane &L, const Resolved &R, const ScanMode &mode, bool with_place, const ReqOut **rows,
                     uint32_t *vidx = nullptr, uint8_t *vcls = nullptr)
{
    KB_TRY(upload_layout(ctx, L, R));
    if (!mode.compact) KB_TRY(sel_ensure(ctx, L, R));
    KB_TRY(launch_scan_core(ctx, L, R, mode, with_place, vidx, vcls));
    const size_t bytes = R.reqs.size() * sizeof(ReqOut);
    KB_TRY(hbuf_ensure(ctx, L.h_stage, bytes + 64));
    KB_CUDA(ctx, cudaMemcpyAsync(L.h_stage.p, L.d_reqout.p, bytes, cudaMemcpyDeviceToHost, L.stream));
    KB_CUDA(ctx, cudaStreamSynchronize(L.stream));
    *rows = (const ReqOut *)L.h_stage.p;
    return KB_OK;
}

// `limit` requests over intervals much larger than the limit: find how far the reference's loop would read
// (worker.run stops pulling from the iterator once the receiver is full, scanner.go:416 / receiver.go:82-87) by
// scanning geometrically growing windows, then clip the request to exactly those records.  The final pass then
// sees what the reference saw, with work proportional to the answer instead of to the interval.
constexpr uint32_t KB_LIMIT_WINDOW_MIN = 8192;

// *reused: the probe pass WAS the final pass (every request of the batch was probed, all of them were settled by the first
// window, padded-arena sizes): its selection and request rows are already on the device, the caller skips its own scan
static int probe_limit_windows(kb_ctx *ctx, ScanLane &L, Resolved &R, int wire, bool *reused)
{
    *reused = false;
    struct Todo {
        uint32_t q, true_hi;
        uint64_t w;
    };
    std::vector<Todo> todo;
    for (uint32_t q = 0; q < R.reqs.size(); q++) {
        const ReqDev &r = R.reqs[q];
        if (r.limit <= 0) continue;
        uint64_t w0 = std::max<uint64_t>(KB_LIMIT_WINDOW_MIN, (uint64_t)r.limit * 8);
        w0 = (w0 + KB_TILE - 1) / KB_TILE * KB_TILE;
        if ((uint64_t)(r.hi - r.lo) > w0) todo.push_back(Todo{q, r.hi, w0});
    }
    if (todo.empty()) return KB_OK;
    for (int round = 0; !todo.empty(); round++) {
        Resolved P;
        P.reqs.resize(todo.size());
        for (size_t i = 0; i < todo.size(); i++) {
            P.reqs[i] = R.reqs[todo[i].q];
            P.reqs[i].hi = (uint32_t)std::min<uint64_t>(todo[i].true_hi, (uint64_t)P.reqs[i].lo + todo[i].w);
        }
        KB_TRY(layout_requests(ctx, true, P));
        const ReqOut *ro = nullptr;
        KB_TRY(scan_sync(ctx, L, P, ScanMode::range(0), true, &ro));
        std::vector<Todo> next;
        for (size_t i = 0; i < todo.size(); i++) {
            ReqDev &r = R.reqs[todo[i].q];
            if (ro[i].flags & KB_RO_LIMIT_STOP)
                r.hi = r.lo + ro[i].examined;  // exactly the records the reference's loop pulled
            else if (P.reqs[i].hi != todo[i].true_hi)
                next.push_back(Todo{todo[i].q, todo[i].true_hi, todo[i].w * 8});
            // else: the whole interval was examined and the limit was not reached inside the loop
        }
        if (round == 0 && next.empty() && wire == 0 && todo.size() == R.reqs.size()) {
            // every request of the batch sits in P in the same order; for a request the limit stopped, the window holds
            // more records than the reference's loop pulled, but the first `limit` emissions, the bytes of those and the
            // examined count (all in its request row) are the ones the clipped scan would produce
            R = P;
            *reused = true;
            return KB_OK;
        }
        todo.swap(next);
    }
    return layout_requests(ctx, true, R);
}

static_assert(sizeof(ReqOut) == 32, "publish_rout copies ReqOut rows as two 16-byte words");

// The context's error flag, as a lane batch's rows or a page cut published it (its HostPub's error word): raised by an
// EARLIER wire copy of this context and never cleared
static int pub_err_check(kb_ctx *ctx, const HostPub &pub)
{
    if (pub.err() == 0) return KB_OK;
    return kb_fail(ctx, KB_ECUDA, "range scan: an earlier wire copy of this context timed out on a bulk copy (the "
                                  "context's error flag stays raised)");
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

// the per-kv view arrays of an answer of at most `cap` kvs inside one device buffer of cap * (wire ? 44 : 36) + 72 bytes;
// returns the element offsets (wire modes: cap + 1 entries)
static uint64_t *om_layout(void *om, uint64_t cap, int wire, GatherOut &go)
{
    go.rev = (uint64_t *)om;
    go.key_off = go.rev + cap;
    go.val_off = go.key_off + cap;
    uint64_t *elem_off = go.val_off + cap;
    go.rec_idx = (uint32_t *)(wire ? elem_off + cap + 1 : elem_off);
    go.key_len = go.rec_idx + cap;
    go.val_len = go.key_len + cap;
    return elem_off;
}

// A new result (held by `res`) and the buffers of its answer: an arena of arena_bytes (none when 0) and, for a range
// answer (batch or page) of at most cap_kvs kvs, its per-kv arrays (res->d_meta, laid out into go; *elem_off: the element
// offsets).  A point-read result takes only the arena, from the point-read pool.
static int answer_new(kb_ctx *ctx, HeldResult &res, ResultKind kind, int out_mode, int wire, uint64_t cap_kvs,
                      uint64_t arena_bytes, GatherOut *go = nullptr, uint64_t **elem_off = nullptr)
{
    res.p = kb_result_new(kind, out_mode);
    res.p->wire = wire;
    if (!arena_bytes) return KB_OK;
    if (cap_kvs) {
        KB_TRY(pool_get_dev(ctx, cap_kvs * (wire ? 44 : 36) + 64 + 8, &res.p->d_meta));
        *elem_off = om_layout(res.p->d_meta.p, cap_kvs, wire, *go);
    }
    return pool_get_arena(ctx, arena_bytes, &res.p->d_arena, kind == ResultKind::point_read);
}

// out_mode -> the base mode (KB_OUT_*) and the wire mode (KB_WIRE_*_I); KB_EINVAL when both wire flags are set.  Each
// entry point checks which combinations it accepts.
static int split_out_mode(int out_mode, int *base, int *wire)
{
    const int flags = out_mode & (KB_WIRE_ETCD_KVS | KB_WIRE_ETCD_EVENTS);
    *base = out_mode & ~(KB_WIRE_ETCD_KVS | KB_WIRE_ETCD_EVENTS);
    *wire = flags == KB_WIRE_ETCD_KVS ? KB_WIRE_KVS_I : flags == KB_WIRE_ETCD_EVENTS ? KB_WIRE_EVENTS_I : 0;
    return flags == (KB_WIRE_ETCD_KVS | KB_WIRE_ETCD_EVENTS) ? KB_EINVAL : KB_OK;
}

// the copy on stream sg starts behind the copy jobs enqueued on L.stream
static int copy_after_jobs(kb_ctx *ctx, ScanLane &L, cudaStream_t sg)
{
    if (sg == L.stream) return KB_OK;
    KB_CUDA(ctx, cudaEventRecord(L.ev_jobs, L.stream));
    KB_CUDA(ctx, cudaStreamWaitEvent(sg, L.ev_jobs, 0));
    return KB_OK;
}

// the end of a copy just enqueued on the copy stream sg: recorded in ev_copied (its JobSet's ev_gather) and in
// res->done_ev, which completes the answer (kb_result_wait, kb_sync)
static int copy_done(kb_ctx *ctx, cudaStream_t sg, cudaEvent_t ev_copied, kb_result *res)
{
    KB_CUDA(ctx, cudaEventRecord(ev_copied, sg));
    KB_TRY(ev_take(ctx, &res->done_ev));
    KB_CUDA(ctx, cudaEventRecord(res->done_ev, sg));
    return KB_OK;
}

// The copy of an answer whose job table (job_first[nreq + 1] | arena_base[nreq + 1] | work counter) is being written on
// L.stream: the copy jobs (into d_jobs) and the per-kv arrays on L.stream, the copy into res->d_arena on stream sg.  A
// range answer copies on the copy stream and passes ev_copied (its JobSet's ev_gather): the end of the copy is recorded
// there and in res->done_ev.  A point-read answer copies on the lane stream itself (ev_copied = nullptr): the batch
// publishes its rows behind the copy, so the arena is complete when they arrive.
static int launch_copy(kb_ctx *ctx, ScanLane &L, cudaStream_t sg, void *d_jobs, cudaEvent_t ev_copied, const ReqDev *d_reqs,
                       uint32_t nreq, const JobTable &tab, const uint32_t *sel, const uint64_t *slot, uint64_t cap_kvs,
                       int wire, const GatherOut &go, uint64_t *d_elem_off, kb_result *res)
{
    const uint64_t *d_jobfirst = tab.job_first, *d_arenabase = tab.arena_base;
    const unsigned jgrid = (unsigned)std::min<uint64_t>((cap_kvs + 255) / 256, (uint64_t)ctx->n_sms * 8);
    if (wire) {
        WireOut wo;
        wo.rec_idx = go.rec_idx;
        wo.rev = go.rev;
        wo.key_off = go.key_off;
        wo.key_len = go.key_len;
        wo.val_off = go.val_off;
        wo.val_len = go.val_len;
        wo.elem_off = d_elem_off;
        WireJob *d_wj = (WireJob *)d_jobs;
        KB_LAUNCH_S(ctx, L.stream, "k_wire_jobs", cap_kvs * 20,
                    (k_wire_jobs<<<jgrid, 256, 0, L.stream>>>(ctx->st, d_reqs, nreq, d_jobfirst, d_arenabase, sel, slot,
                                                              wire, d_wj, wo)));
        KB_TRY(copy_after_jobs(ctx, L, sg));
        uint32_t slot_chunks, wstages;
        wire_geometry(ctx->max_kv_chunks, &slot_chunks, &wstages);
        const size_t wsmem = (size_t)WIRE_WARPS * wstages * slot_chunks * 16;
        if (!ctx->wire_attr_set) {
            cudaFuncSetAttribute(k_wire_copy, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)(WIRE_WARPS * WIRE_WARP_CHUNKS * 16));
            ctx->wire_attr_set = true;
        }
        const unsigned wgrid =
            (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((cap_kvs + WIRE_WARPS - 1) / WIRE_WARPS, 2 * (uint64_t)ctx->n_sms));
        KB_LAUNCH_S(ctx, sg, "k_wire_copy", 0,
                    (k_wire_copy<<<wgrid, WIRE_WARPS * 32, wsmem, sg>>>(ctx->st, d_wj, tab.n_kvs(),
                                                                      (uint8_t *)res->d_arena.p, slot_chunks, wstages,
                                                                      (unsigned int *)ctx->d_ctrs.p + 8)));
    } else {
        GatherJob *d_gj = (GatherJob *)d_jobs;
        KB_LAUNCH_S(ctx, L.stream, "k_gather_jobs", cap_kvs * 20,
                    (k_gather_jobs<<<jgrid, 256, 0, L.stream>>>(ctx->st, d_reqs, nreq, d_jobfirst, d_arenabase, sel, slot,
                                                                d_gj, go)));
        KB_TRY(copy_after_jobs(ctx, L, sg));
        KB_TRY(launch_gather(ctx, sg, d_gj, tab, (uint4 *)res->d_arena.p, cap_kvs, 0));
    }
    return ev_copied ? copy_done(ctx, sg, ev_copied, res) : KB_OK;
}

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
    for (uint64_t q = 0; q < nreq; q++) {
        // checkCompactRace (scanner.go:594-626)
        if (ctx->compact_present && ctx->compact_rev > reqs[q].read_rev)
            return kb_fail(ctx, KB_ECOMPACTED, "range stream revision %llu less than compact revision %llu",
                           (unsigned long long)reqs[q].read_rev, (unsigned long long)ctx->compact_rev);
    }
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
        KB_TRY(dbuf_ensure(ctx, J.gjobs, std::max<uint64_t>(cap_kvs, 1) * (wire ? sizeof(WireJob) : sizeof(GatherJob))));
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

// The per-kv arrays and the arena of an answer of nk > 0 kvs and nbytes arena bytes become the result's: KB_OUT_HOST
// copies them to pinned host memory (and hands the device meta and arena back), KB_OUT_DEVICE keeps them in HBM
static int answer_finish(kb_ctx *ctx, kb_result *res, const GatherOut &go, const uint64_t *d_elem_off, uint64_t nk,
                         uint64_t nbytes, kb_tp &tseg)
{
    const int wire = res->wire;
    if (res->out_mode == KB_OUT_HOST) {
        // per-kv arrays: six strided pieces of the capacity-sized device layout -> one compact host layout, on the
        // host-copy stream behind this batch's gather (which waited for the per-kv arrays): a later batch's gather (already
        // queued on the copy stream when batches are submitted ahead) does not sit between the answer and the host
        const int rc = result_to_host(ctx, res, ctx->stream_h,
                                      {{go.rev, nk * 8}, {go.key_off, nk * 8}, {go.val_off, nk * 8},
                                       {d_elem_off, wire ? (nk + 1) * 8 : 0}, {go.rec_idx, nk * 4}, {go.key_len, nk * 4},
                                       {go.val_len, nk * 4}},
                                      nbytes, "range D2H");
        kb_seg(ctx, "host:range_d2h", tseg);
        KB_TRY(rc);
        uint8_t *hm = (uint8_t *)res->h_meta.p;
        res->rev = (const uint64_t *)hm;
        res->key_off = res->rev + nk;
        res->val_off = res->key_off + nk;
        res->elem_off = wire ? res->val_off + nk : nullptr;
        res->rec_idx = (const uint32_t *)(res->val_off + nk + (wire ? nk + 1 : 0));
        res->key_len = res->rec_idx + nk;
        res->val_len = res->key_len + nk;
    } else {
        res->rev = go.rev;
        res->key_off = go.key_off;
        res->val_off = go.val_off;
        res->rec_idx = go.rec_idx;
        res->key_len = go.key_len;
        res->val_len = go.val_len;
        res->elem_off = wire ? d_elem_off : nullptr;
    }
    return KB_OK;
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

extern "C" int kb_result_wait(kb_ctx *ctx, const kb_result *res, void *cuda_stream)
{
    if (!ctx || !res) return KB_EINVAL;
    if (!res->done_ev) return KB_OK;
    cudaSetDevice(ctx->device);
    if (cuda_stream) {
        KB_CUDA(ctx, cudaStreamWaitEvent((cudaStream_t)cuda_stream, res->done_ev, 0));
    } else {
        KB_CUDA(ctx, cudaEventSynchronize(res->done_ev));
    }
    return KB_OK;
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

// ================================================================================================
// range streams: one unlimited scan at open, its answer handed out page by page within a byte budget
// ================================================================================================
namespace {

// k_page_cut's report, a HostPub with the context's error flag as its error word: payload [end kv u64 | arena bytes u64 |
// key length u64], then from byte KB_PAGE_PUB_KEY the internal key of the page's last kv
constexpr size_t KB_PAGE_PUB_KEY = 64;
constexpr size_t KB_PAGE_PUB_BYTES = KB_PAGE_PUB_KEY + 65536 + 16;

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
    // largest k in [0, groups] whose page fits (k = 0 always does); `fits` holds for a prefix of the candidates, so each
    // step tests 32 spread-out pivots and keeps the interval between the last that fits and the first that does not
    uint64_t lo = 0, hi = groups + 1;
    while (hi - lo > 1) {
        const uint64_t span = hi - lo - 1;  // candidates lo + 1 .. hi - 1
        if (span <= 32) {
            const bool f = lane < span && bytes_of(lo + 1 + lane) <= max_bytes;
            lo += __popc(__ballot_sync(FULL, f));
            break;
        }
        const uint64_t piv = lo + 1 + (span - 1) * lane / 31;
        const int c = __popc(__ballot_sync(FULL, bytes_of(piv) <= max_bytes));
        const uint64_t nlo = c > 0 ? __shfl_sync(FULL, piv, c - 1) : lo;
        const uint64_t nhi = c < 32 ? __shfl_sync(FULL, piv, c) : hi;
        lo = nlo;
        hi = nhi;
    }
    const uint64_t b = end_of(lo > 1 ? lo : 1);
    const uint64_t bytes = bytes_of(lo > 1 ? lo : 1);
    uint32_t kl = 0;
    if (sel) {
        const uint32_t rec = sel[b - 1];
        kl = st.klen[rec];
        const uint4 *src = st.kslab + st.koff16[rec];
        uint4 *dst = (uint4 *)(host + KB_PAGE_PUB_KEY);
        for (uint32_t c = lane; c * 16 < kl; c += 32) dst[c] = src[c];
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

// Cut the next page of p on the current lane: k_page_cut over the entries' arena offsets (slot; sel: the records of a
// range stream's kvs, whose last key it publishes) writes the page's job table into the next JobSet, which alternates
// with the range batches' as between two batches.
static int page_cut(kb_ctx *ctx, PageStream &p, const uint32_t *sel, const uint64_t *slot, uint64_t max_bytes,
                    const char *what, kb_tp &tseg, PageCut *out)
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

static void stream_free(kb_range_stream *s)
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
    kb_range_req q;
    q.start = (const uint8_t *)start.data();
    q.start_len = start.size();
    q.end = (const uint8_t *)s->end.data();
    q.end_len = s->end.size();
    q.read_rev = s->read_rev;
    q.limit = 0;
    Resolved R;
    KB_TRY(resolve_requests(ctx, L, &q, 1, false, R));
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
    // checkCompactRace (scanner.go:594-626), with the text of the range path
    if (ctx->compact_present && ctx->compact_rev > req->read_rev)
        return kb_fail(ctx, KB_ECOMPACTED, "range stream revision %llu less than compact revision %llu",
                       (unsigned long long)req->read_rev, (unsigned long long)ctx->compact_rev);
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
    KB_TRY(dbuf_ensure(ctx, J.gjobs, nk * (s->wire ? sizeof(WireJob) : sizeof(GatherJob))));
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

// k_partition_cut's report in ctx->ppub (error word: the context's error flag): per cut k = 1 .. P-1 the u64 triple
// [kv index | arena offset | key length] at payload entry 3 (k - 1), then from payload byte part_keys_off(P) the
// revision-record key of cut k at (k - 1) * key_stride.  A cut with no kv (index n) has arena offset T and no key.
__host__ __device__ constexpr uint64_t part_keys_off(uint64_t parts) { return ((parts - 1) * 24 + 15) & ~(uint64_t)15; }

// One CTA; warp w takes the cuts k = w + 1, w + 1 + KB_PART_WARPS, ...: the least i in [1, n) with slot[i] * P >= k * T
// (n when there is none) by the 32-ary lower-bound search of k_page_cut, then the internal key of kv i with its 8 revision
// bytes zeroed (EncodeRevisionKey of its user key; every emitted record decodes, so its key is at least 13 bytes long).
__global__ void __launch_bounds__(KB_PART_WARPS * 32)
k_partition_cut(StoreDev st, const uint32_t *__restrict__ sel, const uint64_t *__restrict__ slot, uint64_t n, uint64_t total,
                uint64_t parts, uint64_t key_stride, uint8_t *host, uint64_t epoch, const unsigned int *__restrict__ err_flag)
{
    const uint32_t lane = threadIdx.x & 31;
    uint64_t *cut = (uint64_t *)(host + KB_PUB_HEAD);
    uint8_t *keys = host + KB_PUB_HEAD + part_keys_off(parts);
    for (uint64_t k = 1 + (threadIdx.x >> 5); k < parts; k += KB_PART_WARPS) {
        const uint64_t want = k * total;
        auto below = [&](uint64_t i) { return slot[i] * parts < want; };  // false from the cut on
        uint64_t lo = 1, hi = n;  // the cut lies in [lo, hi]; hi = n: none found yet
        while (hi > lo) {
            const uint64_t span = hi - lo;  // candidates lo .. hi - 1
            if (span <= 32) {
                lo += __popc(__ballot_sync(FULL, lane < span && below(lo + lane)));
                break;
            }
            const uint64_t piv = lo + (span - 1) * lane / 31;
            const int c = __popc(__ballot_sync(FULL, below(piv)));
            const uint64_t nlo = c > 0 ? __shfl_sync(FULL, piv, c - 1) + 1 : lo;
            const uint64_t nhi = c < 32 ? __shfl_sync(FULL, piv, c) : hi;
            lo = nlo;
            hi = nhi;
        }
        const uint64_t i = lo;
        uint32_t kl = 0;
        if (i < n) {
            const uint32_t rec = sel[i];
            kl = st.klen[rec];
            const uint4 *src = st.kslab + st.koff16[rec];
            uint4 *dst = (uint4 *)(keys + (k - 1) * key_stride);
            for (uint32_t c = lane; c * 16 < kl; c += 32) {
                uint4 v = src[c];
                uint8_t *b = (uint8_t *)&v;
#pragma unroll
                for (uint32_t j = 0; j < 16; j++)
                    if (c * 16 + j + 8 >= kl) b[j] = 0;
                dst[c] = v;
            }
        }
        if (lane == 0) {
            volatile uint64_t *h = cut + 3 * (k - 1);
            h[0] = i;
            h[1] = i < n ? slot[i] : total;
            h[2] = kl;
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
    kb_range_req q = *req;
    q.limit = 0;
    Resolved R;
    KB_TRY(resolve_requests(ctx, L, &q, 1, false, R));
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
            const uint64_t i = h[3 * (k - 1)];
            if (i >= n || i == prev) continue;  // no kv reaches the share, or the same kv as the cut before
            cuts.push_back(Cut{i, h[3 * (k - 1) + 1], keys + (k - 1) * stride, h[3 * (k - 1) + 2]});
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

// ---- framing of the wire elements (host): etcdserverpb.ResponseHeader{revision} (pkg/server/etcd/kv.go:253-257) is
// field 1 of both responses; a header with revision 0 is still emitted (non-nil message of length 0)
static uint64_t host_put_varint(uint8_t *out, uint64_t v)
{
    uint64_t n = 0;
    while (v >= 0x80) {
        out[n++] = (uint8_t)(v | 0x80);
        v >>= 7;
    }
    out[n++] = (uint8_t)v;
    return n;
}

static uint64_t host_put_header(uint64_t header_rev, uint8_t *out)
{
    uint8_t body[12];
    uint64_t nb = 0;
    if (header_rev) {
        body[nb++] = 0x18;  // ResponseHeader.revision = 3, varint
        nb += host_put_varint(body + nb, header_rev);
    }
    uint64_t w = 0;
    out[w++] = 0x0a;  // field 1, length-delimited
    w += host_put_varint(out + w, nb);
    memcpy(out + w, body, nb);
    return w + nb;
}

extern "C" uint64_t kb_wire_range_head(uint64_t header_rev, uint8_t *out)
{
    return out ? host_put_header(header_rev, out) : 0;
}

extern "C" uint64_t kb_wire_range_tail(int more, int64_t count, uint8_t *out)
{
    if (!out) return 0;
    uint64_t w = 0;
    if (more) {  // RangeResponse.more = 3
        out[w++] = 0x18;
        out[w++] = 1;
    }
    if (count) {  // RangeResponse.count = 4
        out[w++] = 0x20;
        w += host_put_varint(out + w, (uint64_t)count);
    }
    return w;
}

extern "C" uint64_t kb_wire_watch_head(uint64_t header_rev, int canceled, const uint8_t *reason, uint64_t reason_len,
                                       uint8_t *out)
{
    if (!out || (reason_len && !reason)) return 0;
    uint64_t w = host_put_header(header_rev, out);
    if (canceled) {  // WatchResponse.canceled = 4
        out[w++] = 0x20;
        out[w++] = 1;
    }
    if (reason_len) {  // WatchResponse.cancel_reason = 6
        out[w++] = 0x32;
        w += host_put_varint(out + w, reason_len);
        memcpy(out + w, reason, reason_len);
        w += reason_len;
    }
    return w;
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
        const size_t jobs_bytes = n * (wire ? sizeof(WireJob) : sizeof(GatherJob));
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
    kb_range_req rq;
    rq.start = start;
    rq.start_len = start_len;
    rq.end = end;
    rq.end_len = end_len;
    rq.read_rev = rev;
    rq.limit = 0;
    Resolved R;
    KB_TRY(resolve_requests(ctx, L, &rq, 1, false, R));
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
