// kb_scan.cu -- the scan core every reader of the snapshot runs: requests resolved to record intervals and laid out as
// tiles, then one launch chain that finds what each request emits and places it.  It only reads the snapshot (ctx->st,
// the slab bounds, store_gen); kb_store.cu builds and changes it.
//
// Replaces (reference file:line):
//   storage.Iter over badger            pkg/storage/badger/iter.go:27-98        -> HBM slab + k_search
//   coder.Decode                        pkg/backend/coder/normal.go:58-70       -> k_decode_lcp
//   worker.run (range + compact)        pkg/backend/scanner/scanner.go:389-516  -> k_decode_lcp, k_emit, k_place
//   commonResultReceiver (limit)        pkg/backend/scanner/receiver.go:62-103  -> k_tile_scan, k_place, k_gather
//
// On the lane stream, behind the bound search (k_search, kb_search.cu) and k_fill_tiles:
//   k_decode_lcp  element-wise pass over the store's scan summary (kb_decode.cuh): one 32-bit meta word per record
//   k_emit        per tile: segmented "last visible version" scan over the meta words (prev pointer + running min-LCP;
//                 the cross-tile carry by decoupled look-back) decides which record every key change emits / supersedes
//   k_tile_scan   prefix sums of the per-tile counts / bytes (one CTA per 1024 tiles); k_req_totals: per-request rows
//   k_place       ordered placement of the selection (limit applied), or k_place_victims: the ordered victim list
#include <algorithm>

#include "kb_scan.cuh"
#include "kb_decode.cuh"
#include "kb_wire.cuh"

namespace {

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

}  // namespace

// lay the requests ([lo,hi) already known) out as tiles of KB_TILE records that never span two requests
static int layout_requests(kb_ctx *ctx, bool cap_by_limit, Resolved &R)
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
                     kb_tp *tseg)
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

// one unlimited request over [start, end) at rev, resolved on lane L
int resolve_interval(kb_ctx *ctx, ScanLane &L, const uint8_t *start, uint64_t start_len, const uint8_t *end,
                     uint64_t end_len, uint64_t rev, Resolved &R)
{
    kb_range_req q;
    q.start = start;
    q.start_len = start_len;
    q.end = end;
    q.end_len = end_len;
    q.read_rev = rev;
    q.limit = 0;
    return resolve_requests(ctx, L, &q, 1, false, R);
}

// the tile table starts on a 32-byte boundary behind the lane's `nreq` requests; only the requests travel, the device
// derives the tiles from them (a 100M-record sweep has 97 656 tiles: 0.4 ms of host loop + 3 MB of upload in round 1)
static size_t tile_table_off(size_t nreq) { return (nreq * sizeof(ReqDev) + 31) & ~(size_t)31; }
static TileDev *tile_table(const ScanLane &L, size_t nreq) { return (TileDev *)((uint8_t *)L.d_reqs.p + tile_table_off(nreq)); }

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

// the per-batch pass over the scan summary: one CTA per tile (kb_decode.cuh)
static int launch_decode(kb_ctx *ctx, cudaStream_t strm, uint32_t ntiles, uint64_t n_rec, const ScanMode &mode,
                         const TileDev *d_tiles, uint32_t *d_meta)
{
    // 12 bytes of summary read (the revision only for decodable keys) and the 4-byte meta word written per record
    KB_LAUNCH_S(ctx, strm, "k_decode_lcp", n_rec * 16,
                (k_decode_lcp<<<ntiles, 256, 0, strm>>>(ctx->st, d_tiles, mode, d_meta)));
    return KB_OK;
}

// decode -> emit -> tile scan -> request totals -> (place) for a layout uploaded to lane L; everything stays enqueued on
// L.stream.  Range: the selection goes to L.d_sel / d_slot; compact: the delete calls go to vidx / vcls.
int launch_scan_core(kb_ctx *ctx, ScanLane &L, const Resolved &R, const ScanMode &mode, bool with_place, uint32_t *vidx,
                     uint8_t *vcls)
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
int sel_ensure(kb_ctx *ctx, ScanLane &L, const Resolved &R)
{
    KB_TRY(dbuf_ensure(ctx, L.d_sel, std::max<uint64_t>(R.total_sel, 1) * 4));
    return dbuf_ensure(ctx, L.d_slot, std::max<uint64_t>(R.total_sel, 1) * 8);
}

// A scan whose request rows the host reads at once: R's layout is uploaded to lane L (with its selection arrays for a
// range), scanned, and the rows come back through L.h_stage once the lane stream has drained
int scan_sync(kb_ctx *ctx, ScanLane &L, const Resolved &R, const ScanMode &mode, bool with_place, const ReqOut **rows,
              uint32_t *vidx, uint8_t *vcls)
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
int probe_limit_windows(kb_ctx *ctx, ScanLane &L, Resolved &R, int wire, bool *reused)
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
