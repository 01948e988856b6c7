// kb_reconcile.cu -- the snapshot reconciled with the engine's content of one key interval (kb_reconcile).
//
// The caller hands in the engine's records of [start, end); the diff is the merge of them with the snapshot's records of
// the interval, compared on the device:
//   upload        the input keys as one bound slab (bounds_pack: [start, end, key 0 .. key n-1]), the values as one
//                 16-byte-padded image with per-record offsets and lengths
//   bound_search  one k_search launch: [lo, hi) of the interval and the lower bound of every input key
//   k_reconcile_match  warp per input record: exact key match at its lower bound, then length and value chunks (the
//                 snapshot's value through StoreDev::vslab, so both heap placements); a one-byte verdict, and the matched
//                 position marked (and counted per tile of [lo, hi))
//   k_reconcile_extra  block per tile: the unmarked positions of [lo, hi), in order, at the tile's base
//   k_reconcile_keys   warp per EXTRA record: its key gathered into a padded image
// The host reads back the bounds, the verdicts and the tile counts, then the EXTRA positions and their keys: key and value
// bytes of records that match never leave the device.  A non-empty diff that is not a dry run is committed as one
// kb_apply_batch of the diff in key order (write_batch_locked, kb_store.cu).
#include <algorithm>

#include "kb_internal.cuh"

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr uint32_t RECON_TILE = KB_TILE;  // positions of [lo, hi) per block of k_reconcile_extra (256 threads x 4)

// bres = the bound search's results: [0] lo, [1] hi, [2 + g] the lower bound of input key g (bound 2 + g)
__global__ void __launch_bounds__(128)
k_reconcile_match(StoreDev st, BoundsDev bounds, const uint32_t *__restrict__ bres, const uint4 *__restrict__ vimg,
                  const uint64_t *__restrict__ ivoff16, const uint32_t *__restrict__ ivlen, uint32_t n,
                  uint8_t *__restrict__ verdict, uint8_t *__restrict__ mark, uint32_t *__restrict__ tile_matched)
{
    const uint32_t g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (g >= n) return;
    const uint32_t lo = bres[0], hi = bres[1], r = bres[2 + g], bl = bounds.len(2 + g);
    // every input key lies in [start, end), so its lower bound lies in [lo, hi]
    const bool eq = r < hi && st.klen[r] == bl && warp_prefix_eq(st.kslab + st.koff16[r], bounds, 2 + g, bl);
    uint8_t v = KB_DIFF_MISSING;
    if (eq) {
        const uint32_t vl = st.vlen[r];
        bool same = vl == __ldg(ivlen + g);
        if (same) {  // equal lengths: the zero padding of both images is equal too, so whole chunks compare
            const uint4 *a = st.vslab + st.voff16[r], *b = vimg + __ldg(ivoff16 + g);
            bool d = false;
            for (uint64_t c = lane; c < ((uint64_t)vl + 15) / 16; c += 32) {
                const uint4 x = a[c], y = __ldg(b + c);
                d |= ((x.x ^ y.x) | (x.y ^ y.y) | (x.z ^ y.z) | (x.w ^ y.w)) != 0;
            }
            same = !__any_sync(FULL, d);
        }
        v = same ? 0 : KB_DIFF_CHANGED;
        if (lane == 0) {
            mark[r - lo] = 1;
            atomicAdd(tile_matched + (r - lo) / RECON_TILE, 1u);
        }
    }
    if (lane == 0) verdict[g] = v;
}

// Block t: the positions of tile t of [lo, hi) that no input record matched, in ascending order from tile_base[t], with
// their key lengths
__global__ void __launch_bounds__(256)
k_reconcile_extra(StoreDev st, const uint32_t *__restrict__ bres, const uint8_t *__restrict__ mark,
                  const uint32_t *__restrict__ tile_base, uint32_t *__restrict__ xpos, uint32_t *__restrict__ xklen)
{
    __shared__ uint32_t warp_sum[8];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t lo = bres[0], hi = bres[1];
    const uint64_t rel0 = (uint64_t)blockIdx.x * RECON_TILE + threadIdx.x * 4;
    uint32_t bits = 0;
#pragma unroll
    for (uint32_t j = 0; j < 4; j++)
        if (lo + rel0 + j < hi && !mark[rel0 + j]) bits |= 1u << j;
    const uint32_t c = __popc(bits);
    uint32_t x = c;  // inclusive scan over the warp
#pragma unroll
    for (uint32_t o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(FULL, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sum[warp] = x;
    __syncthreads();
    uint32_t at = tile_base[blockIdx.x] + x - c;
    for (uint32_t w = 0; w < warp; w++) at += warp_sum[w];
#pragma unroll
    for (uint32_t j = 0; j < 4; j++)
        if (bits >> j & 1) {
            const uint32_t r = (uint32_t)(lo + rel0 + j);
            xpos[at] = r;
            xklen[at] = st.klen[r];
            at++;
        }
}

// warp per EXTRA record k: its key, zero padded, at chunk xkoff16[k] of `out`
__global__ void __launch_bounds__(128)
k_reconcile_keys(StoreDev st, const uint32_t *__restrict__ xpos, const uint64_t *__restrict__ xkoff16, uint32_t nx,
                 uint4 *__restrict__ out)
{
    const uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (k >= nx) return;
    const uint32_t r = xpos[k], kc = ((uint32_t)st.klen[r] + 15) >> 4;
    const uint4 *src = st.kslab + st.koff16[r];
    uint4 *dst = out + xkoff16[k];
    for (uint32_t c = lane; c < kc; c += 32) dst[c] = src[c];
}

// bytes.Compare(a, b) < 0
bool key_less(const uint8_t *a, uint64_t al, const uint8_t *b, uint64_t bl)
{
    const uint64_t m = std::min(al, bl);
    const int c = m ? memcmp(a, b, m) : 0;
    return c < 0 || (c == 0 && al < bl);
}

// the pooled scratch of one call, returned when it ends; on a failure part-way a launch may still read it, so the lane
// stream is drained first (a no-op after the call's own last synchronisation)
struct Scratch {
    kb_ctx *ctx;
    DBuf d[3];
    HBuf h[3];
    ~Scratch()
    {
        cudaStreamSynchronize(ctx->lane().stream);
        for (DBuf &b : d) pool_put_dev(ctx, b);
        for (HBuf &b : h) pool_put_host(ctx, b);
    }
};

uint64_t al16(uint64_t x) { return (x + 15) & ~15ull; }

}  // namespace

static int reconcile_locked(kb_ctx *ctx, const uint8_t *start, uint64_t start_len, const uint8_t *end, uint64_t end_len,
                            const uint8_t *keys, const uint64_t *key_off, const uint8_t *vals, const uint64_t *val_off,
                            uint64_t n, int dry_run, kb_result **out)
{
    if (!ctx->loaded) return kb_fail(ctx, KB_ESTATE, "no store loaded");
    if (start_len > 65535 || end_len > 65535) return kb_fail(ctx, KB_ELIMIT, "reconcile: bound key too long");
    if (n >= 0xFFFFFFFEull) return kb_fail(ctx, KB_ELIMIT, "reconcile: too many records (%llu)", (unsigned long long)n);
    kb_tp t0 = kb_now();
    // the input: lengths, the iterator contract, the interval
    uint64_t v16 = 0;
    for (uint64_t i = 0; i < n; i++) {
        const uint64_t kl = key_off[i + 1] - key_off[i], vl = val_off[i + 1] - val_off[i];
        if (kl > 65535) return kb_fail(ctx, KB_ELIMIT, "reconcile: key %llu longer than 65535 bytes", (unsigned long long)i);
        if (vl > 0xFFFFFFFFull) return kb_fail(ctx, KB_ELIMIT, "reconcile: value %llu too long", (unsigned long long)i);
        v16 += (vl + 15) / 16;
    }
    const bool interval = key_less(start, start_len, end, end_len);
    if (n && !interval) return kb_fail(ctx, KB_EINVAL, "reconcile: records given for an empty interval");
    auto key = [&](uint64_t i) { return keys + key_off[i]; };
    auto klen = [&](uint64_t i) { return key_off[i + 1] - key_off[i]; };
    for (uint64_t i = 1; i < n; i++)
        if (!key_less(key(i - 1), klen(i - 1), key(i), klen(i)))
            return kb_fail(ctx, KB_EUNSORTED, "reconcile: key %llu is not greater than its predecessor", (unsigned long long)i);
    if (n && (key_less(key(0), klen(0), start, start_len) || !key_less(key(n - 1), klen(n - 1), end, end_len)))
        return kb_fail(ctx, KB_EINVAL, "reconcile: a key lies outside [start, end)");
    cudaSetDevice(ctx->device);
    KB_TRY(ctx_quiesce(ctx));

    HeldResult res{ctx, kb_result_new(ResultKind::reconcile, KB_OUT_HOST)};
    kb_result &R = *res.p;
    R.rc_n_engine = n;
    std::vector<uint32_t> pos;      // lower bound of every input key
    std::vector<uint8_t> verdict;   // 0 (equal) or KB_DIFF_MISSING / _CHANGED per input record
    std::vector<uint32_t> xpos;     // EXTRA positions, ascending
    std::vector<uint64_t> xkoff;    // n_extra + 1 byte offsets of their keys in xkeys
    std::vector<uint8_t> xkeys;
    uint32_t lo = 0, hi = 0;
    Scratch sc{ctx, {}, {}};  // d[0] / h[0]: input and first readback; [1]: EXTRA positions; [2]: EXTRA keys
    if (interval) {
        ScanLane &L = ctx->lane();
        cudaStream_t s = L.stream;
        PackedBounds pk;
        KB_TRY(bounds_pack(
            ctx, L.h_stage, n + 2, [&](uint64_t i) { return i == 0 ? start_len : i == 1 ? end_len : klen(i - 2); },
            [&](uint64_t i, uint8_t *dst) {
                const uint64_t l = i == 0 ? start_len : i == 1 ? end_len : klen(i - 2);
                if (l) memcpy(dst, i == 0 ? start : i == 1 ? end : key(i - 2), l);
            },
            &pk));
        // device scratch: value image | ivoff16 u64 x n | ivlen u32 x n | verdict u8 x n | mark u8 x N | tile counts |
        // tile bases; the first three are staged on the host as they lie on the device (one upload)
        const uint64_t N = ctx->st.n, T = N / RECON_TILE + 1;
        const uint64_t o_ivoff = v16 * 16, o_ivlen = o_ivoff + n * 8, o_verdict = al16(o_ivlen + n * 4);
        const uint64_t o_mark = al16(o_verdict + n), o_tcnt = al16(o_mark + N + 1), o_tbase = o_tcnt + T * 4;
        const uint64_t d_bytes = o_tbase + T * 4;
        KB_TRY(pool_get_dev(ctx, d_bytes + 64, &sc.d[0]));
        KB_TRY(pool_get_host(ctx, std::max(o_verdict, (n + 2) * 4 + n + T * 4) + 64, &sc.h[0]));
        uint8_t *hin = (uint8_t *)sc.h[0].p, *dw = (uint8_t *)sc.d[0].p;
        uint64_t *ivoff = (uint64_t *)(hin + o_ivoff);
        uint32_t *ivlen = (uint32_t *)(hin + o_ivlen);
        uint64_t c16 = 0;
        for (uint64_t i = 0; i < n; i++) {
            const uint64_t vl = val_off[i + 1] - val_off[i], pad = al16(vl) - vl;
            uint8_t *dst = hin + c16 * 16;
            if (vl) memcpy(dst, vals + val_off[i], vl);
            if (pad) memset(dst + vl, 0, pad);
            ivoff[i] = c16;
            ivlen[i] = (uint32_t)vl;
            c16 += al16(vl) / 16;
        }
        kb_seg(ctx, "host:reconcile_pack", t0);
        KB_CUDA(ctx, cudaMemcpyAsync(dw, hin, o_verdict, cudaMemcpyHostToDevice, s));
        KB_CUDA(ctx, cudaMemsetAsync(dw + o_mark, 0, o_tbase - o_mark, s));  // marks and tile counts
        BoundSearch &bs = L.search;
        KB_TRY(bound_search(ctx, bs, pk, s, false));
        const uint32_t *d_bres = (const uint32_t *)bs.d_bres.p;
        if (n)
            // per input record: its key (twice: search and match), its value and the snapshot's
            KB_LAUNCH(ctx, "k_reconcile_match", (pk.chunks * 16 + c16 * 16) * 2,
                      (k_reconcile_match<<<(unsigned)((n * 32 + 127) / 128), 128, 0, s>>>(
                          ctx->st, bs.dev, d_bres, (const uint4 *)dw, (const uint64_t *)(dw + o_ivoff),
                          (const uint32_t *)(dw + o_ivlen), (uint32_t)n, dw + o_verdict, dw + o_mark,
                          (uint32_t *)(dw + o_tcnt))));
        // readback: the bounds, the verdicts, the tile counts
        uint32_t *h_bres = (uint32_t *)hin;
        uint8_t *h_verdict = hin + (n + 2) * 4;
        uint8_t *h_tcnt = h_verdict + n;  // read with memcpy: not 4-byte aligned
        KB_CUDA(ctx, cudaMemcpyAsync(h_bres, d_bres, (n + 2) * 4, cudaMemcpyDeviceToHost, s));
        if (n) KB_CUDA(ctx, cudaMemcpyAsync(h_verdict, dw + o_verdict, n, cudaMemcpyDeviceToHost, s));
        KB_CUDA(ctx, cudaMemcpyAsync(h_tcnt, dw + o_tcnt, T * 4, cudaMemcpyDeviceToHost, s));
        KB_CUDA(ctx, cudaStreamSynchronize(s));
        lo = h_bres[0];
        hi = std::max(h_bres[0], h_bres[1]);
        pos.assign(h_bres + 2, h_bres + 2 + n);
        verdict.assign(h_verdict, h_verdict + n);
        // EXTRA per tile = the tile's positions - the matched ones; their bases
        const uint64_t span = hi - lo, tiles = (span + RECON_TILE - 1) / RECON_TILE;
        std::vector<uint32_t> tbase(tiles + 1);
        uint64_t nx = 0;
        for (uint64_t t = 0; t < tiles; t++) {
            uint32_t matched;
            memcpy(&matched, h_tcnt + t * 4, 4);
            tbase[t] = (uint32_t)nx;
            nx += std::min<uint64_t>(RECON_TILE, span - t * RECON_TILE) - matched;
        }
        if (nx) {
            memcpy(hin, tbase.data(), tiles * 4);  // the staged input is on the device already: its staging is free
            KB_CUDA(ctx, cudaMemcpyAsync(dw + o_tbase, hin, tiles * 4, cudaMemcpyHostToDevice, s));
            // d[1] = xpos u32 x nx | xklen u32 x nx | xkoff16 u64 x nx; h[1] the same on the host
            const uint64_t o_xkoff = al16(nx * 8);
            KB_TRY(pool_get_dev(ctx, o_xkoff + nx * 8 + 64, &sc.d[1]));
            KB_TRY(pool_get_host(ctx, o_xkoff + nx * 8 + 64, &sc.h[1]));
            uint8_t *dx = (uint8_t *)sc.d[1].p;
            uint32_t *hx = (uint32_t *)sc.h[1].p, *hxlen = hx + nx;
            uint64_t *hkoff16 = (uint64_t *)((uint8_t *)hx + o_xkoff);
            KB_LAUNCH(ctx, "k_reconcile_extra", span + nx * 8,
                      (k_reconcile_extra<<<(unsigned)tiles, 256, 0, s>>>(ctx->st, d_bres, dw + o_mark,
                                                                          (const uint32_t *)(dw + o_tbase),
                                                                          (uint32_t *)dx, (uint32_t *)dx + nx)));
            KB_CUDA(ctx, cudaMemcpyAsync(hx, dx, nx * 8, cudaMemcpyDeviceToHost, s));
            KB_CUDA(ctx, cudaStreamSynchronize(s));
            xpos.assign(hx, hx + nx);
            xkoff.resize(nx + 1);
            uint64_t k16 = 0;
            xkoff[0] = 0;
            for (uint64_t k = 0; k < nx; k++) {
                hkoff16[k] = k16;
                k16 += (hxlen[k] + 15) / 16;
                xkoff[k + 1] = xkoff[k] + hxlen[k];
            }
            // d[2] / h[2]: the EXTRA keys, each zero padded to 16 bytes
            KB_TRY(pool_get_dev(ctx, k16 * 16 + 64, &sc.d[2]));
            KB_TRY(pool_get_host(ctx, k16 * 16 + 64, &sc.h[2]));
            KB_CUDA(ctx, cudaMemcpyAsync(dx + o_xkoff, hkoff16, nx * 8, cudaMemcpyHostToDevice, s));
            KB_LAUNCH(ctx, "k_reconcile_keys", k16 * 32,
                      (k_reconcile_keys<<<(unsigned)((nx * 32 + 127) / 128), 128, 0, s>>>(
                          ctx->st, (const uint32_t *)dx, (const uint64_t *)(dx + o_xkoff), (uint32_t)nx,
                          (uint4 *)sc.d[2].p)));
            KB_CUDA(ctx, cudaMemcpyAsync(sc.h[2].p, sc.d[2].p, k16 * 16, cudaMemcpyDeviceToHost, s));
            KB_CUDA(ctx, cudaStreamSynchronize(s));
            xkeys.resize(xkoff[nx]);
            for (uint64_t k = 0; k < nx; k++)
                if (hxlen[k]) memcpy(xkeys.data() + xkoff[k], (const uint8_t *)sc.h[2].p + hkoff16[k] * 16, hxlen[k]);
        }
        KB_CUDA(ctx, cudaGetLastError());
        kb_seg(ctx, "host:reconcile_compare", t0);
    }

    // the diff in key order: EXTRA position p goes in front of input record g iff p < pos[g]
    const uint64_t nx = xpos.size();
    uint64_t nmiss = 0, nchg = 0, kbytes = xkeys.size();
    for (uint64_t g = 0; g < n; g++) {
        if (verdict[g] == KB_DIFF_MISSING) nmiss++;
        if (verdict[g] == KB_DIFF_CHANGED) nchg++;
        if (verdict[g]) kbytes += klen(g);
    }
    const uint64_t nd = nmiss + nchg + nx;
    R.rc_n_mirror = hi - lo;
    R.rc_n_missing = nmiss;
    R.rc_n_extra = nx;
    R.rc_n_changed = nchg;
    R.rc_n_diff = nd;
    KB_TRY(pool_get_host(ctx, nd * 8 + (nd + 1) * 8 + nd + 64, &R.h_meta));
    KB_TRY(pool_get_host(ctx, kbytes + 16, &R.h_arena));
    uint64_t *src_idx = (uint64_t *)R.h_meta.p, *koff = src_idx + nd;
    uint8_t *kind = (uint8_t *)(koff + nd + 1), *bytes = (uint8_t *)R.h_arena.p;
    std::vector<kb_write_op> ops(dry_run ? 0 : nd);
    uint64_t d = 0, w = 0, x = 0;
    auto emit = [&](uint8_t kd, uint64_t src, const uint8_t *k, uint64_t kl) {
        kind[d] = kd;
        src_idx[d] = src;
        koff[d] = w;
        if (kl) memcpy(bytes + w, k, kl);
        if (!dry_run) {
            kb_write_op &op = ops[d];
            memset(&op, 0, sizeof(op));
            op.type = kd == KB_DIFF_EXTRA ? KB_OP_DEL : KB_OP_PUT;
            op.key = bytes + w;
            op.key_len = kl;
            if (kd != KB_DIFF_EXTRA) {
                op.val = vals + val_off[src];
                op.val_len = val_off[src + 1] - val_off[src];
            }
        }
        w += kl;
        d++;
    };
    auto emit_extra = [&](uint64_t k) { emit(KB_DIFF_EXTRA, UINT64_MAX, xkeys.data() + xkoff[k], xkoff[k + 1] - xkoff[k]); };
    for (uint64_t g = 0; g < n; g++) {
        if (!verdict[g]) continue;
        while (x < nx && xpos[x] < pos[g]) emit_extra(x++);
        emit(verdict[g], g, key(g), klen(g));
    }
    while (x < nx) emit_extra(x++);
    koff[nd] = w;
    R.n_bytes = w;
    if (!dry_run && nd) {
        kb_tp ta = kb_now();
        KB_TRY(write_batch_locked(ctx, ops.data(), nd));
        kb_seg(ctx, "host:reconcile_apply", ta);
    }
    *out = res.release();
    return KB_OK;
}

extern "C" int kb_reconcile(kb_ctx *ctx, const uint8_t *start, uint64_t start_len, const uint8_t *end, uint64_t end_len,
                            const uint8_t *keys, const uint64_t *key_off, const uint8_t *vals, const uint64_t *val_off,
                            uint64_t n, int dry_run, kb_result **out)
{
    if (!ctx || !out) return KB_EINVAL;
    *out = nullptr;
    if (n && (!keys || !key_off || !vals || !val_off)) return KB_EINVAL;
    if ((!start && start_len) || (!end && end_len)) return KB_EINVAL;
    std::lock_guard<std::mutex> g(ctx->mu);
    return reconcile_locked(ctx, start, start_len, end, end_len, keys, key_off, vals, val_off, n, dry_run, out);
}

extern "C" int kb_reconcile_view_get(const kb_result *res, kb_reconcile_view *v)
{
    if (!res || !v || res->kind != ResultKind::reconcile) return KB_EINVAL;
    const uint64_t nd = res->rc_n_diff;
    const uint64_t *meta = (const uint64_t *)res->h_meta.p;
    v->n_engine = res->rc_n_engine;
    v->n_mirror = res->rc_n_mirror;
    v->n_missing = res->rc_n_missing;
    v->n_extra = res->rc_n_extra;
    v->n_changed = res->rc_n_changed;
    v->n_diff = nd;
    v->src_idx = meta;
    v->key_off = meta + nd;
    v->kind = (const uint8_t *)(meta + nd + nd + 1);
    v->bytes = (const uint8_t *)res->h_arena.p;
    v->n_bytes = res->n_bytes;
    return KB_OK;
}
