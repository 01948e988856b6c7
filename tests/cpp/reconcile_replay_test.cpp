// reconcile_replay_test.cpp -- replays, call for call, what the Go storage adaptor does to keep the HBM mirror equal to
// the engine (go/pkg/storage/b200/storage.go Verify / verifyChunk / repairLoop -> kb.go Engine.Reconcile), against a
// std::map engine, and checks every answer in between against the CPU oracle (oracle/libkboracle.so):
//   Verify(start, end, chunk, repair): per chunk Iter(cursor, end, chunk) of the engine, then
//     kb_reconcile(cursor, to, records, dry_run = !repair) with to = lastKey + 0x00, or end once the engine has fewer
//     records than the chunk; after a repair, kb_apply_batch of the repaired /events/ keys with the full TTL
//   an uncertain commit: the batch reaches the engine and not the mirror; the retry queue finds it landed and rewrites
//     the value at a new revision through the commit hook (engine, then kb_apply_batch); the suspect repair then runs
//     Verify(key, key + 0x00, 1, true) for every key of the uncertain batch
// Between the steps: answers at revisions between the two writes, and the compaction sweep's victims, from the mirror
// against the oracle on the engine's records -- they differ while the record of the uncertain revision is stranded in
// the engine, and agree once it is repaired.
// usage: reconcile_replay_test   (needs a CUDA device; tests/test_gpu_reconcile.py builds and runs it)
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "../../include/kb_b200.h"
#include "../../oracle/kb_oracle.h"

#define CHECK(c)                                                                                         \
    do {                                                                                                 \
        if (!(c)) {                                                                                      \
            std::printf("FAIL %s:%d: %s  [%s]\n", __FILE__, __LINE__, #c, ctx ? kb_last_error(ctx) : ""); \
            std::exit(1);                                                                                \
        }                                                                                                \
    } while (0)

typedef std::string Bytes;
static kb_ctx *ctx = nullptr;
static std::map<Bytes, Bytes> engine;  // the durable engine's records
static const uint64_t kTTL = 3600;      // cfg.TTL of the /events/ keys, seconds
static const uint64_t kNow = 1700000000;

static Bytes be64(uint64_t v)
{
    Bytes b(8, '\0');
    for (int i = 0; i < 8; i++) b[i] = (char)(v >> (8 * (7 - i)));
    return b;
}
static Bytes ikey(const Bytes &uk, uint64_t rev) { return Bytes("\x57\xfb\x80\x8b", 4) + uk + "$" + be64(rev); }
static const Bytes kMagic("\x57\xfb\x80\x8b", 4), kMagicEnd("\x57\xfb\x80\x8c", 4);

struct Op {
    bool del;
    Bytes key, val;
    uint64_t expire;
};

static void mirror_apply(const std::vector<Op> &ops)
{
    std::vector<kb_write_op> raw(ops.size());
    for (size_t i = 0; i < ops.size(); i++) {
        memset(&raw[i], 0, sizeof raw[i]);
        raw[i].type = ops[i].del ? KB_OP_DEL : KB_OP_PUT;
        raw[i].key = (const uint8_t *)ops[i].key.data();
        raw[i].key_len = ops[i].key.size();
        raw[i].val = (const uint8_t *)ops[i].val.data();
        raw[i].val_len = ops[i].val.size();
        raw[i].expire_unix = ops[i].expire;
    }
    CHECK(kb_apply_batch(ctx, raw.data(), raw.size()) == KB_OK);
}

static void engine_apply(const std::vector<Op> &ops)
{
    for (const Op &o : ops) {
        if (o.del)
            engine.erase(o.key);
        else
            engine[o.key] = o.val;
    }
}

// batch.Commit: engine first, mirror second; uncertain = the engine took it, the mirror never hears of it
static void commit(const std::vector<Op> &ops, bool uncertain = false)
{
    engine_apply(ops);
    if (!uncertain) mirror_apply(ops);
}

struct Packed {
    std::vector<uint8_t> keys, vals;
    std::vector<uint64_t> koff{0}, voff{0};
    void add(const Bytes &k, const Bytes &v)
    {
        keys.insert(keys.end(), k.begin(), k.end());
        vals.insert(vals.end(), v.begin(), v.end());
        koff.push_back(keys.size());
        voff.push_back(vals.size());
    }
    uint64_t n() const { return koff.size() - 1; }
    Bytes key(uint64_t i) const { return Bytes((const char *)keys.data() + koff[i], koff[i + 1] - koff[i]); }
    Bytes val(uint64_t i) const { return Bytes((const char *)vals.data() + voff[i], voff[i + 1] - voff[i]); }
    ko_store view() const { return ko_store{keys.data(), koff.data(), vals.data(), voff.data(), n()}; }
};

static Packed pack_engine()
{
    Packed p;
    for (auto &it : engine) p.add(it.first, it.second);
    return p;
}

struct Report {
    uint64_t chunks = 0, missing = 0, extra = 0, changed = 0;
};

// storage.go verifyChunk: the engine's records of [cur, end) up to `chunk`, compared (and repaired); returns the next cursor
static bool verify_chunk(const Bytes &cur, const Bytes &end, uint64_t chunk, bool repair, Report &rep, Bytes *next)
{
    Packed p;
    for (auto it = engine.lower_bound(cur); it != engine.end() && it->first < end && p.n() < chunk; ++it)
        p.add(it->first, it->second);
    const bool done = p.n() < chunk;
    const Bytes to = done ? end : p.key(p.n() - 1) + Bytes(1, '\0');
    kb_result *res = nullptr;
    CHECK(kb_reconcile(ctx, (const uint8_t *)cur.data(), cur.size(), (const uint8_t *)to.data(), to.size(), p.keys.data(),
                       p.koff.data(), p.vals.data(), p.voff.data(), p.n(), repair ? 0 : 1, &res) == KB_OK);
    kb_reconcile_view v;
    CHECK(kb_reconcile_view_get(res, &v) == KB_OK);
    CHECK(v.n_engine == p.n() && v.n_diff == v.n_missing + v.n_extra + v.n_changed);
    rep.chunks++;
    rep.missing += v.n_missing;
    rep.extra += v.n_extra;
    rep.changed += v.n_changed;
    std::vector<Op> ttl;
    for (uint64_t k = 0; k < v.n_diff; k++) {
        const Bytes key((const char *)v.bytes + v.key_off[k], v.key_off[k + 1] - v.key_off[k]);
        if (k) CHECK(Bytes((const char *)v.bytes + v.key_off[k - 1], v.key_off[k] - v.key_off[k - 1]) < key);
        if (v.kind[k] == KB_DIFF_EXTRA) {
            CHECK(v.src_idx[k] == UINT64_MAX && !engine.count(key));
        } else {
            CHECK(p.key(v.src_idx[k]) == key);
            if (key.find("/events/") != Bytes::npos) ttl.push_back(Op{false, key, p.val(v.src_idx[k]), kNow + kTTL});
        }
    }
    kb_result_free(ctx, res);
    if (repair && !ttl.empty()) mirror_apply(ttl);  // registerTTL
    *next = to;
    return done;
}

static Report verify(const Bytes &start, const Bytes &end, uint64_t chunk, bool repair)
{
    Report rep;
    Bytes cur = start, next;
    while (!verify_chunk(cur, end, chunk, repair, rep, &next)) cur = next;
    return rep;
}

// (user key, value, revision) of the whole key space at `rev`: from the mirror, and from the oracle on the engine
typedef std::vector<std::pair<Bytes, Bytes>> KVs;
static KVs mirror_range(uint64_t rev)
{
    kb_range_req rq{(const uint8_t *)kMagic.data(), 4, (const uint8_t *)kMagicEnd.data(), 4, rev, 0};
    kb_result *res = nullptr;
    CHECK(kb_range_batch(ctx, &rq, 1, KB_OUT_HOST, &res) == KB_OK);
    kb_range_view v;
    CHECK(kb_range_view_get(res, &v) == KB_OK);
    KVs out;
    for (uint64_t k = 0; k < v.n_kvs; k++)
        out.emplace_back(Bytes((const char *)v.bytes + v.key_off[k], v.key_len[k]) + "@" + std::to_string(v.rev[k]),
                         Bytes((const char *)v.bytes + v.val_off[k], v.val_len[k]));
    kb_result_free(ctx, res);
    return out;
}

static KVs oracle_range(uint64_t rev)
{
    const Packed p = pack_engine();
    const ko_store st = p.view();
    ko_result r;
    ko_result_init(&r);
    CHECK(ko_range(&st, (const uint8_t *)kMagic.data(), 4, (const uint8_t *)kMagicEnd.data(), 4, rev, 0, 0, 0, &r) == 0);
    KVs out;
    for (uint64_t i = 0; i < r.n_emit; i++) {
        const Bytes k = p.key(r.emit[i]);
        uint64_t kr = 0;
        for (int b = 0; b < 8; b++) kr = (kr << 8) | (uint8_t)k[k.size() - 8 + b];
        out.emplace_back(k.substr(4, k.size() - 13) + "@" + std::to_string(kr), p.val(r.emit[i]));
    }
    ko_result_free(&r);
    return out;
}

// the keys the compaction sweep at `rev` deletes: from the mirror's compaction stream, and from the oracle on the engine
static std::set<Bytes> mirror_victims(uint64_t rev)
{
    kb_compact_stream *cs = nullptr;
    CHECK(kb_compact_stream_open(ctx, (const uint8_t *)kMagic.data(), 4, (const uint8_t *)kMagicEnd.data(), 4, rev, 0, 1, 64,
                                 &cs) == KB_OK);
    std::set<Bytes> out;
    for (;;) {
        kb_result *page = nullptr;
        CHECK(kb_compact_stream_next(ctx, cs, 1 << 20, &page) == KB_OK);
        if (!page) break;
        kb_compact_page_view v;
        CHECK(kb_compact_page_view_get(page, &v) == KB_OK);
        for (uint64_t k = 0; k < v.n; k++) out.insert(Bytes((const char *)v.bytes + v.key_off[k], v.key_len[k]));
        kb_result_free(ctx, page);
    }
    kb_compact_stream_close(ctx, cs);
    CHECK(kb_set_compact_revision(ctx, 0, 0) == KB_OK);  // the sweep recorded it: later reads below it must not fail
    return out;
}

static std::set<Bytes> oracle_victims(uint64_t rev)
{
    const Packed p = pack_engine();
    const ko_store st = p.view();
    ko_worker_cfg cfg{rev, 0, 1, 0, 1, 0};
    ko_result r;
    ko_result_init(&r);
    CHECK(ko_worker_run(&st, (const uint8_t *)kMagic.data(), 4, (const uint8_t *)kMagicEnd.data(), 4, &cfg, &r) == 0);
    std::set<Bytes> out;
    for (uint64_t i = 0; i < r.n_victim; i++) out.insert(p.key(r.victim[i]));
    ko_result_free(&r);
    return out;
}

// the backend's write of user key uk at revision rev: CAS(revision record) + Put(object record)
static std::vector<Op> write(const Bytes &uk, uint64_t rev, const Bytes &val, uint64_t expire = 0)
{
    return {Op{false, ikey(uk, 0), be64(rev), expire}, Op{false, ikey(uk, rev), val, expire}};
}

int main()
{
    CHECK(kb_open(0, nullptr, &ctx) == KB_OK);
    for (int j = 0; j < 400; j++) {
        char uk[64];
        std::snprintf(uk, sizeof uk, "/registry/pods/ns-%02d/pod-%04d", j % 13, j);
        for (auto &o : write(uk, 10 + j, Bytes(100 + j % 50, (char)('a' + j % 26)))) engine[o.key] = o.val;
    }
    {
        const Packed p = pack_engine();
        CHECK(kb_load_sorted(ctx, p.keys.data(), p.koff.data(), p.vals.data(), p.voff.data(), p.n()) == KB_OK);
    }
    // in sync: a chunked walk finds nothing, at every chunk size
    for (uint64_t chunk : {(uint64_t)1, (uint64_t)7, (uint64_t)4096}) {
        const Report r = verify(kMagic, kMagicEnd, chunk, false);
        CHECK(r.missing + r.extra + r.changed == 0 && r.chunks == (chunk == 4096 ? 1 : 800 / chunk + 1));
    }

    // /events/ records the mirror never saw, and one it holds that the engine dropped
    std::vector<Op> ev;
    for (int j = 0; j < 6; j++) {
        char uk[64];
        std::snprintf(uk, sizeof uk, "/registry/events/ns-00/ev-%02d", j);
        for (auto &o : write(uk, 1000 + j, "event " + std::to_string(j), kNow + kTTL)) ev.push_back(o);
    }
    engine_apply(ev);
    const Bytes gone = ikey("/registry/pods/ns-03/pod-0003", 13);
    engine.erase(gone);
    Report r = verify(kMagic, kMagicEnd, 7, true);
    CHECK(r.missing == 12 && r.extra == 1 && r.changed == 0);
    CHECK(mirror_range(UINT64_MAX) == oracle_range(UINT64_MAX));
    r = verify(kMagic, kMagicEnd, 7, false);
    CHECK(r.missing + r.extra + r.changed == 0);
    // the repaired /events/ keys carry the full TTL again: they expire together at now + TTL, not before
    uint64_t dropped = 0;
    CHECK(kb_expire(ctx, kNow + kTTL - 1, &dropped) == KB_OK && dropped == 0);
    CHECK(kb_expire(ctx, kNow + kTTL, &dropped) == KB_OK && dropped == 12);
    for (const Op &o : ev) engine.erase(o.key);  // the engine's own TTL ran out too

    // the uncertain-commit story: user key K written at r1 (uncertain, landed), rewritten at r2 by the retry queue
    const Bytes K = "/registry/pods/ns-05/pod-0005";
    const uint64_t r0 = 15, r1 = 2000, r2 = 2001;
    const std::vector<Op> uncertain = write(K, r1, "written at r1");
    commit(uncertain, true);
    commit(write(K, r2, "written at r1"));  // the retry queue's rewrite of the value it read back, through the hook
    // answers at revisions between the two writes differ: the engine has K at r1, the mirror still K at r0
    CHECK(mirror_range(r1) != oracle_range(r1));
    CHECK(mirror_range(r0) == oracle_range(r0) && mirror_range(r2) == oracle_range(r2));
    // the compaction sweep names the stranded record in the engine, never in the mirror
    std::set<Bytes> mv = mirror_victims(r2), ov = oracle_victims(r2);
    CHECK(ov.count(ikey(K, r1)) && !mv.count(ikey(K, r1)) && mv != ov);
    // the suspect repair: Verify(key, key + 0x00, 1, true) for each key of the uncertain batch
    uint64_t missing = 0;
    for (const Op &o : uncertain) {
        const Report s = verify(o.key, o.key + Bytes(1, '\0'), 1, true);
        CHECK(s.extra == 0 && s.changed == 0);
        missing += s.missing;
    }
    CHECK(missing == 1);  // the object record at r1; the revision record already holds r2
    for (uint64_t rev : {r0, r1, r2, UINT64_MAX}) CHECK(mirror_range(rev) == oracle_range(rev));
    CHECK(mirror_victims(r2) == oracle_victims(r2));
    r = verify(kMagic, kMagicEnd, 4096, false);
    CHECK(r.missing + r.extra + r.changed == 0);
    kb_close(ctx);
    ctx = nullptr;
    std::printf("reconcile replay OK\n");
    return 0;
}
