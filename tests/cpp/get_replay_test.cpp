// get_replay_test.cpp -- replays, call for call, what the Go shim's point reads (go/pkg/backend/scanner/b200/kb.go
// Engine.Get / GetResponseWire) do through the C ABI, and checks the answers against the CPU oracle
// (oracle/libkboracle.so).  Go cannot be compiled in the build image, so this is the executable form of that sequence:
//   lock; kb_get_submit(1 read, KB_OUT_HOST [| KB_WIRE_ETCD_KVS]); unlock
//   lock; kb_get_collect; unlock -> status / mod_rev / value (or the element), kb_result_free
// including a Get whose two critical sections fall between another goroutine's kb_range_submit and kb_range_collect.
// usage: get_replay_test            (needs a CUDA device; tests/test_gpu_get_pipeline.py builds and runs it)
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/kb_b200.h"
#include "../../kubebrain_b200/host/kubebrain.hpp"
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

// the store, packed once for the library and the oracle
struct Store {
    Bytes keys, vals;
    std::vector<uint64_t> ko{0}, vo{0};
    ko_store os{};
    explicit Store(const std::map<Bytes, Bytes> &items)
    {
        for (auto &kv : items) {
            keys += kv.first;
            vals += kv.second;
            ko.push_back(keys.size());
            vo.push_back(vals.size());
        }
        os = ko_store{(const uint8_t *)keys.data(), ko.data(), (const uint8_t *)vals.data(), vo.data(), items.size()};
    }
};

enum { kNotFound = 1 };
struct GetAns {
    int err = 0;  // 0, or kNotFound (storage.ErrKeyNotFound)
    Bytes val;
    uint64_t mod_rev = 0;
};

// kb.go Engine.Get, first half: submit under the context lock
static kb_pending *get_submit(const Bytes &key, uint64_t rev, int mode)
{
    kb_get_req rq{(const uint8_t *)key.data(), key.size(), rev};
    kb_pending *p = nullptr;
    CHECK(kb_get_submit(ctx, &rq, 1, mode, &p) == KB_OK && p);
    return p;
}

// ... second half: collect under the lock, copy out, free
static GetAns get_collect(kb_pending *p)
{
    kb_result *res = nullptr;
    CHECK(kb_get_collect(ctx, p, &res) == KB_OK && res);
    kb_get_view v;
    CHECK(kb_get_view_get(res, &v) == KB_OK && v.n == 1 && !v.on_device);
    GetAns a;
    a.mod_rev = v.mod_rev[0];  // valid for a tombstone too (backend.get returns it with ErrKeyNotFound)
    if (v.status[0] == KB_GET_FOUND)
        a.val.assign((const char *)v.bytes + v.val_off[0], v.val_len[0]);
    else
        a.err = kNotFound;
    kb_result_free(ctx, res);
    return a;
}

// kb.go Engine.GetResponseWire: head(max(curRev, modRev) if found else curRev) | element | tail(false, found ? 1 : 0)
static Bytes get_response_wire(const Bytes &key, uint64_t rev, uint64_t cur_rev)
{
    kb_pending *p = get_submit(key, rev, KB_OUT_HOST | KB_WIRE_ETCD_KVS);
    kb_result *res = nullptr;
    CHECK(kb_get_collect(ctx, p, &res) == KB_OK && res);
    kb_get_view v;
    const uint64_t *eo = nullptr;
    CHECK(kb_get_view_get(res, &v) == KB_OK && kb_get_elem_off(res, &eo) == KB_OK);
    const bool found = v.status[0] == KB_GET_FOUND;
    uint8_t head[32], tail[32];
    const uint64_t nh = kb_wire_range_head(found && v.mod_rev[0] > cur_rev ? v.mod_rev[0] : cur_rev, head);
    const uint64_t nt = kb_wire_range_tail(0, found ? 1 : 0, tail);
    Bytes out((const char *)head, nh);
    if (found) out.append((const char *)v.bytes + eo[0], eo[1] - eo[0]);
    out.append((const char *)tail, nt);
    kb_result_free(ctx, res);
    return out;
}

static void expect_get(const Store &s, const Bytes &key, uint64_t rev, const GetAns &a)
{
    uint64_t mod = 0;
    const int64_t idx = ko_get(&s.os, (const uint8_t *)key.data(), key.size(), rev, &mod);
    if (idx >= 0) {
        CHECK(a.err == 0 && a.mod_rev == mod);
        CHECK(a.val == Bytes(s.vals.data() + s.vo[idx], s.vo[idx + 1] - s.vo[idx]));
    } else {
        CHECK(a.err == kNotFound && a.mod_rev == (idx == -2 ? mod : 0));
    }
}

static Bytes oracle_response(const Store &s, const Bytes &key, uint64_t rev, uint64_t cur_rev)
{
    uint64_t mod = 0;
    const int64_t idx = ko_get(&s.os, (const uint8_t *)key.data(), key.size(), rev, &mod);
    uint8_t buf[64];
    Bytes out((const char *)buf, ko_wire_range_head(idx >= 0 && mod > cur_rev ? mod : cur_rev, buf));
    if (idx >= 0) {
        const uint64_t r = (uint64_t)idx;
        uint64_t off[2];
        std::vector<uint8_t> el(ko_wire_encode(&s.os, &r, 1, KO_WIRE_KVS, nullptr, off) + 1);
        ko_wire_encode(&s.os, &r, 1, KO_WIRE_KVS, el.data(), off);
        out.append((const char *)el.data(), off[1]);
    }
    out.append((const char *)buf, ko_wire_range_tail(0, idx >= 0 ? 1 : 0, buf));
    return out;
}

int main()
{
    CHECK(kb_open(0, nullptr, &ctx) == KB_OK);
    // objects with versions, a deleted one (tombstone + deleted-flag revision record), an empty value, a key that is a
    // prefix of another
    std::map<Bytes, Bytes> items;
    for (int i = 0; i < 300; i++) {
        char uk[64];
        std::snprintf(uk, sizeof uk, "/registry/pods/ns-%02d/pod-%04d", i % 7, i);
        const uint64_t r0 = 1000 + 3 * i;
        items[ikey(uk, 0)] = be64(r0 + (i % 5 == 0 ? 2 : 1)) + (i % 11 == 0 ? Bytes(1, '\0') : Bytes());
        items[ikey(uk, r0)] = Bytes(40 + i % 90, (char)('a' + i % 26));
        items[ikey(uk, r0 + 1)] = i % 11 == 0 ? Bytes("tombstone") : i % 13 == 0 ? Bytes() : Bytes(i % 200, 'v');
    }
    items[ikey("/registry/pods/ns-00", 990)] = "prefix";
    Store s(items);
    CHECK(kb_load_sorted(ctx, (const uint8_t *)s.keys.data(), s.ko.data(), (const uint8_t *)s.vals.data(), s.vo.data(),
                         items.size()) == KB_OK);
    std::vector<std::pair<Bytes, uint64_t>> reads;
    for (int i = 0; i < 300; i += 7) {
        char uk[64];
        std::snprintf(uk, sizeof uk, "/registry/pods/ns-%02d/pod-%04d", i % 7, i);
        const uint64_t r0 = 1000 + 3 * i;
        for (uint64_t rev : {(uint64_t)0, r0 - 1, r0, r0 + 1, r0 + 2, ~(uint64_t)0}) reads.push_back({uk, rev});
    }
    reads.push_back({"/registry/pods/ns-00", 0});
    reads.push_back({"/registry/pods/ns-0", 0});
    reads.push_back({"/nothing", 0});
    const uint64_t cur_rev = 1500;

    // Get / GetResponseWire one after the other
    for (auto &r : reads) {
        expect_get(s, r.first, r.second, get_collect(get_submit(r.first, r.second, KB_OUT_HOST)));
        CHECK(get_response_wire(r.first, r.second, cur_rev) == oracle_response(s, r.first, r.second, cur_rev));
    }
    // a Get between another goroutine's range submit and collect, both ways round
    const Bytes lo = ikey("/registry/", 0), hi = ikey("/registry0", 0);
    kb_range_req rq{(const uint8_t *)lo.data(), lo.size(), (const uint8_t *)hi.data(), hi.size(), 2000, 0};
    uint64_t range_kvs = 0;
    for (size_t i = 0; i < reads.size(); i++) {
        const Bytes &k = reads[i].first;
        const uint64_t rev = reads[i].second;
        kb_pending *rp = nullptr;
        kb_result *rr = nullptr;
        if (i % 2 == 0) {
            CHECK(kb_range_submit(ctx, &rq, 1, KB_OUT_HOST | KB_WIRE_ETCD_KVS, &rp) == KB_OK);
            kb_pending *gp = get_submit(k, rev, KB_OUT_HOST);
            const GetAns a = get_collect(gp);
            CHECK(kb_range_collect(ctx, rp, &rr) == KB_OK);
            expect_get(s, k, rev, a);
        } else {
            kb_pending *gp = get_submit(k, rev, KB_OUT_HOST);
            CHECK(kb_range_submit(ctx, &rq, 1, KB_OUT_HOST, &rp) == KB_OK);
            CHECK(kb_range_collect(ctx, rp, &rr) == KB_OK);
            expect_get(s, k, rev, get_collect(gp));
        }
        kb_range_view v;
        CHECK(kb_range_view_get(rr, &v) == KB_OK && v.n_req == 1 && v.n_kvs > 0);
        if (i == 0) range_kvs = v.n_kvs;
        CHECK(v.n_kvs == range_kvs);  // the List beside the Gets answers the same every time
        kb_result_free(ctx, rr);
    }
    // the C++ host layer on the same store: Backend::GetResponseWire and the batched GetMany
    {
        kb::Engine e(0);
        e.LoadSorted(std::vector<std::pair<Bytes, Bytes>>(items.begin(), items.end()));
        kb::Backend be(e, "/registry");
        be.SetCurrentRevision(cur_rev);
        for (auto &r : reads) CHECK(be.GetResponseWire(r.first, r.second) == oracle_response(s, r.first, r.second, cur_rev));
        const auto many = be.GetMany(reads);
        CHECK(many.size() == reads.size());
        for (size_t i = 0; i < reads.size(); i++) {
            uint64_t mod = 0;
            const int64_t idx = ko_get(&s.os, (const uint8_t *)reads[i].first.data(), reads[i].first.size(), reads[i].second, &mod);
            CHECK(many[i].Found == (idx >= 0));
            if (idx >= 0)
                CHECK(many[i].Kv.Key == reads[i].first && many[i].Kv.Revision == mod &&
                      many[i].Kv.Value == Bytes(s.vals.data() + s.vo[idx], s.vo[idx + 1] - s.vo[idx]));
        }
    }
    kb_close(ctx);
    ctx = nullptr;
    std::printf("get replay OK (%zu reads)\n", reads.size());
    return 0;
}
