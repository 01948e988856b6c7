// compact_replay_test.cpp -- replays, call for call, what the Go shim's compaction does through the C ABI
// (go/pkg/backend/scanner/b200/kb.go Compact, go/pkg/storage/b200/storage.go ApplyVictimPage), with a std::map standing
// in for the durable engine, and checks the victims against the CPU oracle (oracle/libkboracle.so):
//   kb_expire(now)                            the mirror drops what the TTL engine no longer returns
//   kb_compact_stream_open(..., 1024)         the sweep (classes, count) -- checked against ko_scan
//   kb_compact_stream_next(64 MiB) until NULL each page's keys, guards and classes copied out, kb_result_free
//   ApplyVictimPage(page)                     per group of 1024: classes 1 / 2 / 5 in one engine batch, then the mirror;
//                                             classes 3 / 4 one at a time: the engine's value against the guard
//                                             (DelCurrent; a mismatch is a failed CAS and is skipped), then the mirror
//   kb_compact_stream_close
// with the context lock released between the calls: the backend's writes land between pages, including a rewrite of a
// revision record whose DelCurrent victim has not been applied yet.  Every run ends with the mirror equal to the engine.
// usage: compact_replay_test            (needs a CUDA device; tests/test_gpu_compact_stream.py builds and runs it)
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
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

static Bytes be64(uint64_t v)
{
    Bytes b(8, '\0');
    for (int i = 0; i < 8; i++) b[i] = (char)(v >> (8 * (7 - i)));
    return b;
}
static Bytes ikey(const Bytes &uk, uint64_t rev) { return Bytes("\x57\xfb\x80\x8b", 4) + uk + "$" + be64(rev); }

// ---- the durable engine: a sorted map with per-key expiry ---------------------------------------------------------
struct MiniEngine {
    std::map<Bytes, Bytes> kv;
    std::map<Bytes, uint64_t> expire;
    void put(const Bytes &k, const Bytes &v, uint64_t exp)
    {
        kv[k] = v;
        if (exp) expire[k] = exp; else expire.erase(k);
    }
    void del(const Bytes &k)
    {
        kv.erase(k);
        expire.erase(k);
    }
    void advance(uint64_t now)
    {
        for (auto it = expire.begin(); it != expire.end();)
            if (it->second <= now) {
                kv.erase(it->first);
                it = expire.erase(it);
            } else
                ++it;
    }
};

struct Packed {
    std::vector<uint8_t> keys, vals;
    std::vector<uint64_t> koff{0}, voff{0};
    uint64_t n() const { return koff.size() - 1; }
    ko_store view() const { return ko_store{keys.data(), koff.data(), vals.data(), voff.data(), n()}; }
};

static Packed iterate(const MiniEngine &e)
{
    Packed p;
    for (auto &it : e.kv) {
        p.keys.insert(p.keys.end(), it.first.begin(), it.first.end());
        p.vals.insert(p.vals.end(), it.second.begin(), it.second.end());
        p.koff.push_back(p.keys.size());
        p.voff.push_back(p.vals.size());
    }
    if (p.keys.empty()) p.keys.push_back(0);
    if (p.vals.empty()) p.vals.push_back(0);
    return p;
}

struct WriteOp {
    bool del;
    Bytes key, val;
    uint64_t expire_unix;
};
static void apply_batch(const std::vector<WriteOp> &ops)  // kb.go ApplyBatch: the commit hook
{
    if (ops.empty()) return;
    std::vector<kb_write_op> raw(ops.size());
    for (size_t i = 0; i < ops.size(); i++) {
        memset(&raw[i], 0, sizeof(raw[i]));
        raw[i].type = ops[i].del ? KB_OP_DEL : KB_OP_PUT;
        raw[i].key = (const uint8_t *)ops[i].key.data();
        raw[i].key_len = ops[i].key.size();
        raw[i].val = ops[i].val.empty() ? nullptr : (const uint8_t *)ops[i].val.data();
        raw[i].val_len = ops[i].val.size();
        raw[i].expire_unix = ops[i].expire_unix;
    }
    CHECK(kb_apply_batch(ctx, raw.data(), raw.size()) == KB_OK);
}

struct Backend {  // the reference's record formats (pkg/backend/txn.go)
    MiniEngine eng;
    uint64_t rev = 1000;
    void write(const Bytes &uk, const Bytes &val, uint64_t exp)
    {
        const uint64_t r = ++rev;
        std::vector<WriteOp> ops = {{false, ikey(uk, 0), be64(r), exp}, {false, ikey(uk, r), val, exp}};
        for (auto &o : ops) eng.put(o.key, o.val, o.expire_unix);
        apply_batch(ops);
    }
    void remove(const Bytes &uk)
    {
        const uint64_t r = ++rev;
        std::vector<WriteOp> ops = {{false, ikey(uk, 0), be64(r) + Bytes(1, '\0'), 0}, {false, ikey(uk, r), "tombstone", 0}};
        for (auto &o : ops) eng.put(o.key, o.val, 0);
        apply_batch(ops);
    }
};

// ---- kb.go Compact + storage.go ApplyVictimPage --------------------------------------------------------------------
struct Page {  // kb.go CompactPage
    std::vector<Bytes> keys, guards;
    std::vector<uint8_t> classes;
    std::vector<uint32_t> records;
};

struct Stats {
    uint64_t pages = 0, victims = 0, deleted = 0, skipped = 0, count = 0;
    std::vector<uint32_t> records;
    std::vector<uint8_t> classes;
};

static void apply_victim_page(Backend &be, const Page &p, uint64_t group, Stats &st)
{
    for (size_t g = 0; g < p.keys.size(); g += group) {
        const size_t h = std::min<size_t>(p.keys.size(), g + group);
        std::vector<WriteOp> dels;  // one engine batch: store.Del of classes 1, 2, 5
        for (size_t i = g; i < h; i++)
            if (p.classes[i] != KB_V_REVRECORD && p.classes[i] != KB_V_TTL_REVREC) dels.push_back({true, p.keys[i], "", 0});
        for (auto &d : dels) be.eng.del(d.key);  // inner.Commit succeeded ...
        apply_batch(dels);                       // ... then the mirror, through the commit hook
        st.deleted += dels.size();
        for (size_t i = g; i < h; i++) {  // DelCurrent: an Iter positioned on the key, its value against the guard
            if (p.classes[i] != KB_V_REVRECORD && p.classes[i] != KB_V_TTL_REVREC) continue;
            auto it = be.eng.kv.find(p.keys[i]);
            if (it == be.eng.kv.end() || it->second != p.guards[i]) {
                st.skipped++;  // ErrCASFailed: a skip, not an error
                continue;
            }
            be.eng.del(p.keys[i]);
            apply_batch({{true, p.keys[i], "", 0}});
            st.deleted++;
        }
    }
}

static Stats compact(Backend &be, const Bytes &s, const Bytes &t, uint64_t crev, uint64_t page_bytes, uint64_t group,
                     uint64_t now, const std::function<void(uint64_t)> &between_pages = nullptr)
{
    Stats st;
    be.eng.advance(now);
    CHECK(kb_expire(ctx, now, nullptr) == KB_OK);  // what the engine no longer returns must not be classified
    kb_compact_stream *cs = nullptr;
    CHECK(kb_compact_stream_open(ctx, (const uint8_t *)s.data(), s.size(), (const uint8_t *)t.data(), t.size(), crev, 0, 1,
                                 group, &cs) == KB_OK);
    uint64_t nv = 0, examined = 0;
    CHECK(kb_compact_stream_info(cs, &nv, &st.count, &examined) == KB_OK);
    for (;;) {
        if (between_pages) between_pages(st.pages);
        kb_result *res = nullptr;
        CHECK(kb_compact_stream_next(ctx, cs, page_bytes, &res) == KB_OK);
        if (!res) break;
        kb_compact_page_view v;
        CHECK(kb_compact_page_view_get(res, &v) == KB_OK);
        CHECK(v.first == st.victims && v.n > 0);
        CHECK(v.n % group == 0 || v.first + v.n == nv);
        Page p;
        for (uint64_t i = 0; i < v.n; i++) {
            p.keys.push_back(Bytes((const char *)v.bytes + v.key_off[i], v.key_len[i]));
            p.guards.push_back(Bytes((const char *)v.bytes + v.guard_off[i], v.guard_len[i]));
            p.classes.push_back(v.victim_class[i]);
            p.records.push_back(v.rec_idx[i]);
        }
        kb_result_free(ctx, res);
        st.records.insert(st.records.end(), p.records.begin(), p.records.end());
        st.classes.insert(st.classes.end(), p.classes.begin(), p.classes.end());
        st.victims += v.n;
        st.pages++;
        apply_victim_page(be, p, group, st);
    }
    kb_compact_stream_close(ctx, cs);
    CHECK(st.victims == nv);
    return st;
}

// the sweep's victims on the engine's content at open, by the oracle
static void check_victims(const Packed &p, const Bytes &s, const Bytes &t, uint64_t crev, const Stats &st)
{
    const ko_store kst = p.view();
    std::vector<uint8_t> borders(s.begin(), s.end());
    borders.insert(borders.end(), t.begin(), t.end());
    const uint64_t boff[3] = {0, s.size(), s.size() + t.size()};
    ko_worker_cfg cfg{crev, 0, 1, 0, 1, 0};
    ko_result exp;
    ko_result_init(&exp);
    int total = 0;
    CHECK(ko_scan(&kst, borders.data(), boff, 2, &cfg, 0, 0, 1, &exp, &total) == 0);
    CHECK(st.records.size() == exp.n_victim && st.count == (uint64_t)total);
    for (uint64_t i = 0; i < exp.n_victim; i++) CHECK(st.records[i] == exp.victim[i] && st.classes[i] == exp.vclass[i]);
    ko_result_free(&exp);
}

// the mirror holds exactly the engine: record count and the full range at the newest revision
static void check_store_equals(const MiniEngine &e)
{
    uint64_t n = 0;
    CHECK(kb_store_info(ctx, &n, nullptr, nullptr) == KB_OK);
    CHECK(n == e.kv.size());
    const Packed p = iterate(e);
    const ko_store st = p.view();
    const Bytes s = ikey("/registry/", 0), t = ikey("/registry0", 0);
    ko_result r;
    ko_result_init(&r);
    CHECK(ko_range(&st, (const uint8_t *)s.data(), s.size(), (const uint8_t *)t.data(), t.size(), ~0ull >> 1, 0, 0, 0, &r) == 0);
    kb_range_req rq{(const uint8_t *)s.data(), s.size(), (const uint8_t *)t.data(), t.size(), ~0ull >> 1, 0};
    kb_result *res = nullptr;
    CHECK(kb_range_batch(ctx, &rq, 1, KB_OUT_HOST, &res) == KB_OK);
    kb_range_view v;
    CHECK(kb_range_view_get(res, &v) == KB_OK);
    CHECK(v.n_kvs == r.n_emit);
    for (uint64_t i = 0; i < r.n_emit; i++) CHECK(v.rec_idx[i] == r.emit[i]);
    kb_result_free(ctx, res);
    ko_result_free(&r);
}

int main()
{
    if (kb_open(0, nullptr, &ctx) != KB_OK) {
        std::printf("no CUDA device: the shim has no CPU fallback\n");
        return 2;
    }
    {  // the mirror follows the writes from an empty engine on (LoadSorted(n = 0) as kb.go sends it)
        const uint64_t zero = 0;
        CHECK(kb_load_sorted(ctx, nullptr, &zero, nullptr, &zero, 0) == KB_OK);
    }
    Backend be;
    const uint64_t now = 1700000000;
    const char *res[] = {"pods", "configmaps", "events"};
    auto name = [&](int i) {
        char b[96];
        std::snprintf(b, sizeof b, "/registry/%s/ns-%02d/obj-%05d", res[i % 3], i % 7, i);
        return Bytes(b);
    };
    for (int i = 0; i < 3000; i++) be.write(name(i), Bytes(40 + i % 50, 'a' + i % 26), i % 3 == 2 ? now + 10 + i % 20 : 0);
    for (int r = 0; r < 3; r++)
        for (int i = r; i < 3000; i += 3) be.write(name(i), Bytes(30 + r, 'A' + r), 0);
    for (int i = 0; i < 3000; i += 5) be.remove(name(i));
    {
        const Packed p = iterate(be.eng);
        CHECK(kb_load_sorted(ctx, p.keys.data(), p.koff.data(), p.vals.data(), p.voff.data(), p.n()) == KB_OK);
        std::vector<WriteOp> ops;
        for (auto &x : be.eng.expire) ops.push_back({false, x.first, be.eng.kv[x.first], x.second});
        apply_batch(ops);
    }
    check_store_equals(be.eng);
    const Bytes s = ikey("/registry/", 0), t = ikey("/registry0", 0);

    // 1. kb.go's page size and group, one TTL tick later; a write lands between open and the first page, and it rewrites
    //    the revision record of a deleted object: that DelCurrent victim carries the old guard and is skipped
    {
        const uint64_t crev = be.rev - 100, tnow = now + 15;
        be.eng.advance(tnow);
        const Packed at_open = iterate(be.eng);
        const Stats st = compact(be, s, t, crev, 64ull << 20, 1024, tnow, [&](uint64_t page) {
            if (page == 0) be.write(name(0), "recreated", 0);  // name(0) was removed: its revision record is a class-3 victim
        });
        check_victims(at_open, s, t, crev, st);
        CHECK(st.pages == 1 && st.skipped == 1 && st.deleted + st.skipped == st.victims && st.victims > 3000);
        check_store_equals(be.eng);
    }
    // 2. small pages: writes and deletes (new DelCurrent victims above the compact revision are not part of this sweep)
    //    between every two pages, and one rewritten revision record whose victim comes in a later page
    for (int i = 3000; i < 3600; i++) be.write(name(i), Bytes(60, 'q'), 0);
    for (int i = 3000; i < 3600; i += 2) be.remove(name(i));
    {
        const uint64_t crev = be.rev;
        const Packed at_open = iterate(be.eng);
        int next_obj = 5000;
        const Stats st = compact(be, s, t, crev, 4096, 8, now + 16, [&](uint64_t page) {
            if (page == 0) be.write(name(3598), "recreated", 0);  // a removed object near the end of the key space
            be.write(name(next_obj++), Bytes(70, 'n'), 0);
            if (page % 3 == 2) be.remove(name(next_obj - 2));
        });
        check_victims(at_open, s, t, crev, st);
        CHECK(st.pages > 10 && st.skipped == 1 && st.deleted + st.skipped == st.victims);
        check_store_equals(be.eng);
    }
    // 3. an empty interval: the first page is NULL
    {
        const Stats st = compact(be, s, s, be.rev, 64ull << 20, 1024, now + 17);
        CHECK(st.pages == 0 && st.victims == 0);
        check_store_equals(be.eng);
    }
    kb_close(ctx);
    ctx = nullptr;
    std::printf("compact replay OK\n");
    return 0;
}
