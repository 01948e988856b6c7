// stream_replay_test.cpp -- replays, call for call, what the Go shim's RangeStream (go/pkg/backend/scanner/b200/kb.go
// RangeStream / rangePages) does through the C ABI, and checks its messages against the CPU oracle
// (oracle/libkboracle.so).  Go cannot be compiled in the build image, so this is the executable form of that sequence:
//   kb_range_stream_open(KB_OUT_HOST, 300)  -> KB_ECOMPACTED: the end marker carries the message
//   kb_range_stream_next(64 MiB) until NULL -> copyKvs of every page, kb_result_free, cut into 300-kv messages
//   kb_range_stream_close
// with the context lock released between pages: a write above the read revision between two pages (what the backend
// commits meanwhile) leaves the messages unchanged.
// usage: stream_replay_test            (needs a CUDA device; tests/test_gpu_range_stream.py builds and runs it)
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

static const uint64_t kBatch = 300;             // rangeStreamBatch
static const uint64_t kPageBytes = 64ull << 20;  // rangeStreamPageBytes

static Bytes be64(uint64_t v)
{
    Bytes b(8, '\0');
    for (int i = 0; i < 8; i++) b[i] = (char)(v >> (8 * (7 - i)));
    return b;
}
static Bytes ikey(const Bytes &uk, uint64_t rev) { return Bytes("\x57\xfb\x80\x8b", 4) + uk + "$" + be64(rev); }

struct KV {
    Bytes key, val;
    uint64_t rev;
    bool operator==(const KV &o) const { return key == o.key && val == o.val && rev == o.rev; }
};
struct Msg {  // proto.StreamRangeResponse
    uint64_t header_rev;
    std::vector<KV> kvs;
    bool more;
    Bytes err;
};

// kb.go RangeStream: rangePages + the cut into 300-kv messages + the end marker
static std::vector<Msg> range_stream(const Bytes &s, const Bytes &t, uint64_t revision,
                                     const std::function<void(int)> &between_pages = nullptr)
{
    std::vector<Msg> out;
    kb_range_req rq{(const uint8_t *)s.data(), s.size(), (const uint8_t *)t.data(), t.size(), revision, 0};
    kb_range_stream *rs = nullptr;
    Bytes err;
    if (kb_range_stream_open(ctx, &rq, KB_OUT_HOST, kBatch, &rs) != KB_OK) {
        err = kb_last_error(ctx);
    } else {
        for (int page_no = 0;; page_no++) {
            kb_result *page = nullptr;
            if (kb_range_stream_next(ctx, rs, kPageBytes, &page) != KB_OK) {
                err = kb_last_error(ctx);
                break;
            }
            if (!page) break;
            kb_range_view v;
            CHECK(kb_range_view_get(page, &v) == KB_OK);
            CHECK(v.n_req == 1 && v.req_first[0] == 0 && v.req_first[1] == v.n_kvs && !v.on_device);
            std::vector<KV> kvs(v.n_kvs);  // copyKvs
            for (uint64_t k = 0; k < v.n_kvs; k++)
                kvs[k] = KV{Bytes((const char *)v.bytes + v.key_off[k], v.key_len[k]),
                            Bytes((const char *)v.bytes + v.val_off[k], v.val_len[k]), v.rev[k]};
            kb_result_free(ctx, page);
            for (uint64_t i = 0; i < kvs.size(); i += kBatch)
                out.push_back(Msg{0, std::vector<KV>(kvs.begin() + i, kvs.begin() + std::min<uint64_t>(kvs.size(), i + kBatch)),
                                  true, ""});
            if (between_pages) between_pages(page_no);
        }
        kb_range_stream_close(ctx, rs);
    }
    out.push_back(Msg{revision, {}, false, err});
    return out;
}

// ---- the snapshot: a sorted map, bulk-loaded as storage.Iter hands it over -------------------------------------
static std::map<Bytes, Bytes> kv;

struct Packed {
    std::vector<uint8_t> keys, vals;
    std::vector<uint64_t> koff{0}, voff{0};
    ko_store view() const { return ko_store{keys.data(), koff.data(), vals.data(), voff.data(), koff.size() - 1}; }
};

static Packed pack()
{
    Packed p;
    for (auto &it : kv) {
        p.keys.insert(p.keys.end(), it.first.begin(), it.first.end());
        p.vals.insert(p.vals.end(), it.second.begin(), it.second.end());
        p.koff.push_back(p.keys.size());
        p.voff.push_back(p.vals.size());
    }
    return p;
}

// the messages RangeStream sends for the oracle's answer on the current map
static std::vector<Msg> want(const Bytes &s, const Bytes &t, uint64_t revision)
{
    const Packed p = pack();
    const ko_store st = p.view();
    ko_result r;
    ko_result_init(&r);
    CHECK(ko_range(&st, (const uint8_t *)s.data(), s.size(), (const uint8_t *)t.data(), t.size(), revision, 0, 0, 0, &r) == 0);
    std::vector<KV> kvs;
    for (uint64_t i = 0; i < r.n_emit; i++) {
        const uint64_t rec = r.emit[i];
        const Bytes k((const char *)p.keys.data() + p.koff[rec], p.koff[rec + 1] - p.koff[rec]);
        uint64_t rev = 0;
        for (int b = 0; b < 8; b++) rev = (rev << 8) | (uint8_t)k[k.size() - 8 + b];
        kvs.push_back(KV{k.substr(4, k.size() - 13), Bytes((const char *)p.vals.data() + p.voff[rec], p.voff[rec + 1] - p.voff[rec]),
                         rev});
    }
    ko_result_free(&r);
    std::vector<Msg> out;
    for (size_t i = 0; i < kvs.size(); i += kBatch)
        out.push_back(Msg{0, std::vector<KV>(kvs.begin() + i, kvs.begin() + std::min<size_t>(kvs.size(), i + kBatch)), true, ""});
    out.push_back(Msg{revision, {}, false, ""});
    return out;
}

static bool same(const std::vector<Msg> &a, const std::vector<Msg> &b)
{
    if (a.size() != b.size()) return false;
    for (size_t i = 0; i < a.size(); i++)
        if (a[i].header_rev != b[i].header_rev || !(a[i].kvs == b[i].kvs) || a[i].more != b[i].more || a[i].err != b[i].err)
            return false;
    return true;
}

static void load()
{
    const Packed p = pack();
    CHECK(kb_load_sorted(ctx, p.keys.data(), p.koff.data(), p.vals.data(), p.voff.data(), p.koff.size() - 1) == KB_OK);
}

int main()
{
    CHECK(kb_open(0, nullptr, &ctx) == KB_OK);
    // 36 000 objects with 2 KiB values in two versions and a revision record: the answer (~80 MB of arena) takes two
    // 64 MiB pages
    const uint64_t read_rev = 5000;
    for (int j = 0; j < 36000; j++) {
        char uk[64];
        std::snprintf(uk, sizeof uk, "/registry/pods/ns-%03d/pod-%06d", j % 97, j);
        const uint64_t r1 = 100 + j % 1000, r2 = 2000 + j % 2000;
        kv[ikey(uk, 0)] = be64(r2);
        kv[ikey(uk, r1)] = Bytes(2000 + j % 33, (char)('a' + j % 26));
        kv[ikey(uk, r2)] = Bytes(2048 + j % 17, (char)('A' + j % 26));
    }
    load();
    const Bytes s = ikey("/registry/", 0), t = ikey("/registry0", 0);
    const std::vector<Msg> exp = want(s, t, read_rev);
    CHECK(exp.size() == 36000 / kBatch + 1);
    int pages = 0;
    CHECK(same(range_stream(s, t, read_rev, [&](int n) { pages = n + 1; }), exp));
    CHECK(pages == 2);
    // a commit above the read revision between the two pages: new versions, new keys
    CHECK(same(range_stream(s, t, read_rev,
                            [&](int n) {
                                if (n != 0) return;
                                std::vector<Bytes> keys, vals;
                                for (int j = 0; j < 36000; j += 7) {
                                    char uk[64];
                                    std::snprintf(uk, sizeof uk, "/registry/pods/ns-%03d/pod-%06d", j % 97, j);
                                    keys.push_back(ikey(uk, read_rev + 1 + j));
                                    vals.push_back(Bytes(100, 'n'));
                                    keys.push_back(ikey(Bytes(uk) + "x", read_rev + 1 + j));
                                    vals.push_back(Bytes(10, 'k'));
                                }
                                std::vector<kb_write_op> ops(keys.size());
                                for (size_t i = 0; i < keys.size(); i++) {
                                    memset(&ops[i], 0, sizeof(ops[i]));
                                    ops[i].type = KB_OP_PUT;
                                    ops[i].key = (const uint8_t *)keys[i].data();
                                    ops[i].key_len = keys[i].size();
                                    ops[i].val = (const uint8_t *)vals[i].data();
                                    ops[i].val_len = vals[i].size();
                                    kv[keys[i]] = vals[i];
                                }
                                CHECK(kb_apply_batch(ctx, ops.data(), ops.size()) == KB_OK);
                            }),
               exp));
    // an empty range and a range that holds fewer than 300 kvs
    CHECK(same(range_stream(s, s, read_rev), want(s, s, read_rev)));
    const Bytes s2 = ikey("/registry/pods/ns-001/", 0), t2 = ikey("/registry/pods/ns-0010", 0);
    CHECK(same(range_stream(s2, t2, read_rev), want(s2, t2, read_rev)));
    // checkCompactRace at open: the end marker carries the range path's message
    CHECK(kb_set_compact_revision(ctx, 1, read_rev + 1) == KB_OK);
    const std::vector<Msg> c = range_stream(s, t, read_rev);
    CHECK(c.size() == 1 && !c[0].more && c[0].header_rev == read_rev);
    CHECK(c[0].err == "range stream revision 5000 less than compact revision 5001");
    kb_close(ctx);
    ctx = nullptr;
    std::printf("stream replay OK\n");
    return 0;
}
