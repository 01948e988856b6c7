// host_values_replay_test.cpp -- replays, call for call, what the Go storage adaptor does with Config.HostValues
// (go/pkg/storage/b200/storage.go NewKvStorage -> kb.OpenConfig(device, kb.CfgHostValues)), through the C ABI:
//   kb_open(flags = KB_CFG_HOST_VALUES); kb_load_sorted; kb_range_batch (List: KB_OUT_HOST | KB_WIRE_ETCD_KVS, and the
//   raw arena); kb_apply_batch (the commit hook); kb_dump (shutdown); kb_restore into a context in device placement
// and checks it against the same calls on a device-placement context: the same answers, the same dump file, and
// kb_store_mem reporting the value heap as host bytes.  Go cannot be compiled in the build image, so this is the
// executable form of that sequence.
// usage: host_values_replay_test <dir for the dump files>   (needs a CUDA device; tests/test_gpu_host_values_replay.py)
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/kb_b200.h"

static kb_ctx *ctx = nullptr;  // the context the last failed check was about

#define CHECK(c)                                                                                         \
    do {                                                                                                 \
        if (!(c)) {                                                                                      \
            std::printf("FAIL %s:%d: %s  [%s]\n", __FILE__, __LINE__, #c, ctx ? kb_last_error(ctx) : ""); \
            std::exit(1);                                                                                \
        }                                                                                                \
    } while (0)

typedef std::string Bytes;

static Bytes be64(uint64_t v)
{
    Bytes b(8, '\0');
    for (int i = 0; i < 8; i++) b[i] = (char)(v >> (8 * (7 - i)));
    return b;
}
static Bytes ikey(const Bytes &uk, uint64_t rev) { return Bytes("\x57\xfb\x80\x8b", 4) + uk + "$" + be64(rev); }

static kb_ctx *open_ctx(uint32_t flags)
{
    kb_ctx *c = nullptr;
    const kb_config cfg{(uint32_t)sizeof(kb_config), flags};
    CHECK(kb_open(0, &cfg, &c) == KB_OK);
    return c;
}

// one List of [start, end) at rev in `mode`: rows, record indices and the arena, as one string
static Bytes list(kb_ctx *c, const Bytes &s, const Bytes &e, uint64_t rev, int64_t limit, int mode)
{
    ctx = c;
    kb_range_req r{(const uint8_t *)s.data(), s.size(), (const uint8_t *)e.data(), e.size(), rev, limit};
    kb_result *res = nullptr;
    CHECK(kb_range_batch(c, &r, 1, mode, &res) == KB_OK);
    kb_range_view v;
    CHECK(kb_range_view_get(res, &v) == KB_OK);
    Bytes out = std::to_string(v.n_kvs) + "/" + std::to_string(v.req_count[0]) + "/" + std::to_string(v.req_examined[0]) + ":";
    for (uint64_t k = 0; k < v.n_kvs; k++) out += std::to_string(v.rec_idx[k]) + "," + std::to_string(v.rev[k]) + ";";
    out.append((const char *)v.bytes, v.n_bytes);
    kb_result_free(c, res);
    return out;
}

static Bytes slurp(const std::string &path)
{
    FILE *f = std::fopen(path.c_str(), "rb");
    CHECK(f);
    Bytes b;
    char buf[1 << 16];
    size_t n;
    while ((n = std::fread(buf, 1, sizeof buf, f)) > 0) b.append(buf, n);
    std::fclose(f);
    return b;
}

int main(int argc, char **argv)
{
    if (argc < 2) {
        std::printf("usage: %s <dir>\n", argv[0]);
        return 2;
    }
    const std::string dir = argv[1];
    // the engine's content as storage.Iter hands it over: revision records and object records, 1 000 objects
    std::vector<std::pair<Bytes, Bytes>> items;
    for (int i = 0; i < 1000; i++) {
        char uk[64];
        std::snprintf(uk, sizeof uk, "/registry/pods/ns%d/p%05d", i % 7, i);
        const uint64_t rev = 100 + i;
        items.push_back({ikey(uk, 0), be64(rev)});
        items.push_back({ikey(uk, rev), Bytes(40 + (i * 37) % 3000, (char)('a' + i % 26))});
    }
    std::sort(items.begin(), items.end());
    Bytes keys, vals;
    std::vector<uint64_t> ko{0}, vo{0};
    for (auto &kv : items) {
        keys += kv.first;
        vals += kv.second;
        ko.push_back(keys.size());
        vo.push_back(vals.size());
    }
    kb_ctx *host = open_ctx(KB_CFG_HOST_VALUES), *dev = open_ctx(0);
    for (kb_ctx *c : {host, dev}) {
        ctx = c;
        uint64_t d = 0, h = 0;
        CHECK(kb_store_mem(c, &d, &h) == KB_ESTATE);
        CHECK(kb_load_sorted(c, (const uint8_t *)keys.data(), ko.data(), (const uint8_t *)vals.data(), vo.data(), items.size()) == KB_OK);
        CHECK(kb_store_mem(c, &d, &h) == KB_OK);
        CHECK(d > 0);
        CHECK(c == host ? h >= vals.size() : h == 0);
    }
    const Bytes lo = ikey("/registry/", 0), hi = ikey("/registry0", 0);
    const int modes[] = {KB_OUT_HOST, KB_OUT_HOST | KB_WIRE_ETCD_KVS, KB_OUT_HOST | KB_WIRE_ETCD_EVENTS};
    for (int m : modes)
        for (uint64_t rev : {(uint64_t)0, (uint64_t)600, ~(uint64_t)0})
            for (int64_t lim : {(int64_t)0, (int64_t)17}) CHECK(list(host, lo, hi, rev, lim, m) == list(dev, lo, hi, rev, lim, m));

    // the commit hook: CAS(revision record) + Put(object record) per write, and a delete, as one batch each
    for (int b = 0; b < 3; b++) {
        std::vector<Bytes> ks, vs;
        for (int i = 0; i < 200; i++) {
            char uk[64];
            std::snprintf(uk, sizeof uk, "/registry/pods/ns%d/p%05d", i % 7, (i * 13 + b) % 1200);
            const uint64_t rev = 5000 + b * 1000 + i;
            ks.push_back(ikey(uk, 0));
            vs.push_back(be64(rev));
            ks.push_back(ikey(uk, rev));
            vs.push_back(Bytes(10 + (i * 101) % 6000, (char)('A' + b)));
        }
        std::vector<kb_write_op> ops(ks.size() + 1);
        for (size_t i = 0; i < ks.size(); i++)
            ops[i] = kb_write_op{KB_OP_PUT, (const uint8_t *)ks[i].data(), ks[i].size(), (const uint8_t *)vs[i].data(), vs[i].size(), 0};
        const Bytes del = items[2 * b + 1].first;
        ops.back() = kb_write_op{KB_OP_DEL, (const uint8_t *)del.data(), del.size(), nullptr, 0, 0};
        for (kb_ctx *c : {host, dev}) {
            ctx = c;
            CHECK(kb_apply_batch(c, ops.data(), ops.size()) == KB_OK);
        }
        for (int m : modes) CHECK(list(host, lo, hi, ~(uint64_t)0, 0, m) == list(dev, lo, hi, ~(uint64_t)0, 0, m));
    }
    // shutdown dump, restart in the other placement
    const std::string ph = dir + "/host.kbd", pd = dir + "/dev.kbd";
    ctx = host;
    CHECK(kb_dump(host, ph.c_str()) == KB_OK);
    ctx = dev;
    CHECK(kb_dump(dev, pd.c_str()) == KB_OK);
    CHECK(slurp(ph) == slurp(pd));
    kb_ctx *dev2 = open_ctx(0), *host2 = open_ctx(KB_CFG_HOST_VALUES);
    ctx = dev2;
    CHECK(kb_restore(dev2, ph.c_str()) == KB_OK);
    ctx = host2;
    CHECK(kb_restore(host2, pd.c_str()) == KB_OK);
    for (int m : modes)
        for (uint64_t rev : {(uint64_t)600, ~(uint64_t)0}) {
            const Bytes want = list(dev, lo, hi, rev, 0, m);
            CHECK(list(dev2, lo, hi, rev, 0, m) == want);
            CHECK(list(host2, lo, hi, rev, 0, m) == want);
        }
    uint64_t d2 = 0, h2 = 0;
    CHECK(kb_store_mem(host2, &d2, &h2) == KB_OK && h2 > 0);
    for (kb_ctx *c : {host, dev, dev2, host2}) kb_close(c);
    std::printf("host values replay ok\n");
    return 0;
}
