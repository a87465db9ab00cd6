// Host-side zone builder: snapshot JSON-lines -> bb::ZoneImage.
//
// Replaces the ingest half of lib/zk.js (TreeNode ctor :78-97, onChildrenChanged :120-138,
// onDataChanged :139-194) for a whole-subtree snapshot, and pre-evaluates the query-independent
// parts of lib/server.js resolve()/resolvePtr() per node (see zone_image.h).
//
// JSON handling is a single-pass "tape" parser (no per-value allocation): 10M-znode
// snapshots (~1.1 GB of text) build in seconds.
#include "zone_image.h"
#include "../../include/binder_b200.h"

#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

namespace {

using namespace bb;

// ---------------------------------------------------------------------------------------
// JSON tape
// ---------------------------------------------------------------------------------------
enum JT : uint8_t { J_NULL, J_FALSE, J_TRUE, J_NUM, J_STR, J_ARR, J_OBJ };
struct Tok {
    uint8_t  type;
    uint32_t a, b;       // J_STR: [a, a+b) in pool.  J_ARR/J_OBJ: b = number of children (pairs for OBJ)
    uint32_t next;       // index of the token after this value's subtree
    double   num;
};
struct Tape {
    std::vector<Tok> t;
    std::string pool;
    const char* p; const char* e;

    void ws() { while (p < e && (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r')) ++p; }
    static void put_utf8(std::string& o, uint32_t c) {
        if (c < 0x80) o.push_back((char)c);
        else if (c < 0x800) { o.push_back((char)(0xC0 | c >> 6)); o.push_back((char)(0x80 | (c & 63))); }
        else if (c < 0x10000) { o.push_back((char)(0xE0 | c >> 12)); o.push_back((char)(0x80 | ((c >> 6) & 63))); o.push_back((char)(0x80 | (c & 63))); }
        else { o.push_back((char)(0xF0 | c >> 18)); o.push_back((char)(0x80 | ((c >> 12) & 63))); o.push_back((char)(0x80 | ((c >> 6) & 63))); o.push_back((char)(0x80 | (c & 63))); }
    }
    bool hex4(uint32_t& v) {
        if (e - p < 4) return false;
        v = 0;
        for (int i = 0; i < 4; i++) {
            unsigned c = (unsigned char)p[i], d;
            if (c - '0' < 10) d = c - '0'; else if ((c | 32) - 'a' < 6) d = (c | 32) - 'a' + 10; else return false;
            v = v << 4 | d;
        }
        p += 4; return true;
    }
    bool str(Tok& k) {
        ++p;                                    // opening quote
        k.type = J_STR; k.a = (uint32_t)pool.size();
        for (;;) {
            const char* s = p;
            while (p < e && *p != '"' && *p != '\\' && (unsigned char)*p >= 0x20) ++p;
            pool.append(s, p - s);
            if (p >= e || (unsigned char)*p < 0x20) return false;
            if (*p == '"') { ++p; break; }
            ++p; if (p >= e) return false;
            char x = *p++;
            switch (x) {
            case '"': case '\\': case '/': pool.push_back(x); break;
            case 'b': pool.push_back('\b'); break; case 'f': pool.push_back('\f'); break;
            case 'n': pool.push_back('\n'); break; case 'r': pool.push_back('\r'); break;
            case 't': pool.push_back('\t'); break;
            case 'u': {
                uint32_t v; if (!hex4(v)) return false;
                if (v >= 0xD800 && v < 0xDC00 && e - p >= 6 && p[0] == '\\' && p[1] == 'u') {
                    const char* save = p; p += 2; uint32_t lo;
                    if (hex4(lo) && lo >= 0xDC00 && lo < 0xE000) v = 0x10000 + ((v - 0xD800) << 10) + (lo - 0xDC00);
                    else p = save;
                }
                put_utf8(pool, v); break; }
            default: return false;
            }
        }
        k.b = (uint32_t)pool.size() - k.a;
        return true;
    }
    bool num(Tok& k) {
        const char* s = p;
        if (p < e && *p == '-') ++p;
        if (p >= e) return false;
        if (*p == '0') ++p;
        else if (*p >= '1' && *p <= '9') { while (p < e && (unsigned)(*p - '0') < 10) ++p; }
        else return false;
        if (p < e && *p == '.') { ++p; if (p >= e || (unsigned)(*p - '0') >= 10) return false; while (p < e && (unsigned)(*p - '0') < 10) ++p; }
        if (p < e && (*p == 'e' || *p == 'E')) {
            ++p; if (p < e && (*p == '+' || *p == '-')) ++p;
            if (p >= e || (unsigned)(*p - '0') >= 10) return false;
            while (p < e && (unsigned)(*p - '0') < 10) ++p;
        }
        char buf[64]; size_t n = (size_t)(p - s);
        k.type = J_NUM;
        if (n < sizeof buf) { memcpy(buf, s, n); buf[n] = 0; k.num = strtod(buf, nullptr); }
        else { std::string tmp(s, n); k.num = strtod(tmp.c_str(), nullptr); }
        return true;
    }
    bool lit(const char* w, size_t n) { if ((size_t)(e - p) < n || memcmp(p, w, n)) return false; p += n; return true; }
    bool value(int depth) {
        if (depth > 200) return false;
        ws(); if (p >= e) return false;
        size_t me = t.size(); t.emplace_back();
        Tok k; k.a = k.b = k.next = 0; k.num = 0;
        bool ok = true;
        switch (*p) {
        case '{': {
            ++p; k.type = J_OBJ; ws();
            if (p < e && *p == '}') { ++p; break; }
            for (;;) {
                ws(); if (p >= e || *p != '"') return false;
                size_t ki = t.size(); t.emplace_back(); Tok kk; kk.next = 0; kk.num = 0;
                if (!str(kk)) return false;
                kk.next = (uint32_t)t.size(); t[ki] = kk;
                ws(); if (p >= e || *p != ':') return false; ++p;
                if (!value(depth + 1)) return false;
                ++k.b; ws(); if (p >= e) return false;
                if (*p == ',') { ++p; continue; }
                if (*p == '}') { ++p; break; }
                return false;
            }
            break; }
        case '[': {
            ++p; k.type = J_ARR; ws();
            if (p < e && *p == ']') { ++p; break; }
            for (;;) {
                if (!value(depth + 1)) return false;
                ++k.b; ws(); if (p >= e) return false;
                if (*p == ',') { ++p; continue; }
                if (*p == ']') { ++p; break; }
                return false;
            }
            break; }
        case '"': ok = str(k); break;
        case 't': k.type = J_TRUE; ok = lit("true", 4); break;
        case 'f': k.type = J_FALSE; ok = lit("false", 5); break;
        case 'n': k.type = J_NULL; ok = lit("null", 4); break;
        default: ok = num(k);
        }
        if (!ok) return false;
        k.next = (uint32_t)t.size();
        t[me] = k;
        return true;
    }
    // parse [b, e) as one JSON document appended to the tape; returns root index or -1
    int parse(const char* b, const char* end) {
        size_t t0 = t.size(), p0 = pool.size();
        p = b; e = end;
        bool ok = value(0);
        if (ok) { ws(); ok = (p == e); }
        if (!ok) { t.resize(t0); pool.resize(p0); return -1; }
        return (int)t0;
    }
    void clear() { t.clear(); pool.clear(); }
    bool is_obj(int v) const { return v >= 0 && (t[v].type == J_OBJ || t[v].type == J_ARR); }   // typeof 'object', non-null
    // own-property read; JSON.parse keeps the last duplicate
    int get(int v, const char* key, size_t klen) const {
        if (v < 0 || t[v].type != J_OBJ) return -1;
        int found = -1; uint32_t i = (uint32_t)v + 1;
        for (uint32_t c = 0; c < t[v].b; c++) {
            const Tok& k = t[i];
            uint32_t val = i + 1;
            if (k.b == klen && memcmp(pool.data() + k.a, key, klen) == 0) found = (int)val;
            i = t[val].next;
        }
        return found;
    }
    int get(int v, const char* key) const { return get(v, key, strlen(key)); }
    bool str_eq(int v, const char* s) const { return v >= 0 && t[v].type == J_STR && t[v].b == strlen(s) && memcmp(pool.data() + t[v].a, s, t[v].b) == 0; }
};

// ---------------------------------------------------------------------------------------
// contract predicates (DESIGN.md "Contract": what mname's record constructors accept)
// ---------------------------------------------------------------------------------------
bool uint_ok(const Tape& J, int v, double limit, uint32_t& out) {
    if (v < 0 || J.t[v].type != J_NUM) return false;
    double d = J.t[v].num;
    if (!(d >= 0.0) || !(d < limit) || std::floor(d) != d) return false;
    out = (uint32_t)d; return true;
}
bool ipv4_ok(const char* s, size_t n, uint32_t& out) {
    size_t i = 0; uint32_t acc = 0;
    for (int o = 0; o < 4; o++) {
        size_t st = i; unsigned v = 0;
        while (i < n && (unsigned)(s[i] - '0') < 10 && i - st < 4) { v = v * 10 + (unsigned)(s[i] - '0'); ++i; }
        size_t nd = i - st;
        if (nd < 1 || nd > 3 || v > 255 || (nd > 1 && s[st] == '0')) return false;
        acc = acc << 8 | v;
        if (o < 3) { if (i >= n || s[i] != '.') return false; ++i; }
    }
    if (i != n) return false;
    out = acc; return true;
}
// hostname of scheme://[userinfo@]host[:port][/...]  (url.parse at lib/server.js:297-298)
bool url_host_ipv4(const char* s, size_t n, uint32_t& out) {
    size_t i = 0;
    if (n == 0 || !(((unsigned)(s[0] | 32) - 'a') < 26)) return false;
    while (i < n && ((((unsigned)(s[i] | 32) - 'a') < 26) || (unsigned)(s[i] - '0') < 10 || s[i] == '+' || s[i] == '.' || s[i] == '-')) ++i;
    if (n - i < 3 || memcmp(s + i, "://", 3)) return false;
    i += 3;
    size_t e = i;
    while (e < n && s[e] != '/' && s[e] != '?' && s[e] != '#') ++e;
    for (size_t k = e; k > i; k--) if (s[k - 1] == '@') { i = k; break; }
    for (size_t k = e; k > i; k--) if (s[k - 1] == ':') { e = k - 1; break; }
    return ipv4_ok(s + i, e - i, out);          // digits and dots: lower-casing is a no-op
}

const char* const kHostLike[] = { "db_host", "host", "load_balancer", "moray_host", "redis_host", "ops_host", "rr_host" };
const char* const kSvcKid[] = { "load_balancer", "moray_host", "ops_host", "rr_host", "redis_host" };

// ---------------------------------------------------------------------------------------
// flattened nodes
// ---------------------------------------------------------------------------------------
enum : uint16_t {
    NF_KIDTYPE = 1,      // data.type passes the service child filter (lib/server.js:352-360)
    NF_SUB_OBJ = 2,      // data[data.type] is a non-null object
    NF_HAS_TTL = 4,      // data.ttl or data[type].ttl defined
    NF_TTL_OK = 8,
    NF_ADDR_NULL = 16,
    NF_ADDR_OK = 32,
    NF_PORTS_LIST = 64,  // ports is a non-empty list of valid ports (stored in `ports`)
    NF_PORTS_BAD = 128,  // ports present but unusable
    NF_REV = 256,        // registers in ca_revLookup
    NF_HOSTLIKE = 512,
    NF_DEAD = 1024,      // unbound (lib/zk.js:195-208): out of the tree, but a reverse entry may still name it
    NF_REV_LOST = 2048,  // another node's address change deleted this node's reverse entry (tn_ip itself stays, :183-185)
};
struct Node {
    uint32_t parent, name_off, name_len;
    uint32_t first_kid = 0, last_kid = 0, next_sib = 0;      // 0 = none (node 0 is the root)
    uint32_t ttl = 30, addr = 0, extra = 0xFFFFFFFFu;        // extra: index into svcs / ports
    uint32_t rev_off = 0, rev_len = 0;                        // address string in pool (reverse key)
    uint32_t rev_seq = 0;                                     // when this node last wrote its reverse entry (event order)
    uint16_t flags = 0; uint8_t kind = K_INVALID; uint8_t pad = 0;
};
struct SvcInfo { std::string srvce, proto; bool has_srvce = false, has_proto = false, port_ok = false; uint32_t port = 0; uint32_t ttl = 30; };

struct Builder {
    std::string dns_domain;                 // lower-cased root domain
    std::vector<Node> nodes;
    std::string pool;                       // names + address strings
    std::vector<SvcInfo> svcs;
    std::vector<std::vector<uint16_t>> ports;
    std::vector<uint32_t> child_tab;        // open-addressed (parent,name) -> node index + 1
    uint32_t child_mask = 0;
    Tape J;

    static uint64_t mix(uint64_t h) { h ^= h >> 33; h *= 0xff51afd7ed558ccdULL; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ULL; h ^= h >> 33; return h; }
    uint64_t child_hash(uint32_t parent, const char* s, size_t n) const {
        uint64_t h = 0x9E3779B97F4A7C15ULL ^ parent;
        for (size_t i = 0; i < n; i++) h = (h ^ (unsigned char)s[i]) * 0x100000001B3ULL;
        return mix(h);
    }
    void child_grow() {
        uint32_t cap = child_tab.empty() ? 1024 : (uint32_t)child_tab.size() * 2;
        std::vector<uint32_t> nt(cap, 0);
        uint32_t m = cap - 1;
        for (uint32_t v : child_tab) if (v) {
            const Node& nd = nodes[v - 1];
            uint64_t h = child_hash(nd.parent, pool.data() + nd.name_off, nd.name_len);
            uint32_t i = (uint32_t)h & m; while (nt[i]) i = (i + 1) & m; nt[i] = v;
        }
        child_tab.swap(nt); child_mask = m;
    }
    int find_child(uint32_t parent, const char* s, size_t n) const {
        if (child_tab.empty()) return -1;
        uint32_t i = (uint32_t)child_hash(parent, s, n) & child_mask;
        while (child_tab[i]) {
            const Node& nd = nodes[child_tab[i] - 1];
            if (nd.parent == parent && nd.name_len == n && !(nd.flags & NF_DEAD) && memcmp(pool.data() + nd.name_off, s, n) == 0) return (int)(child_tab[i] - 1);
            i = (i + 1) & child_mask;
        }
        return -1;
    }
    uint32_t add_node(uint32_t parent, const char* s, size_t n) {
        Node nd; nd.parent = parent; nd.name_off = (uint32_t)pool.size(); nd.name_len = (uint32_t)n;
        pool.append(s, n);
        uint32_t id = (uint32_t)nodes.size();
        nodes.push_back(nd);
        if (id != 0) {
            if ((nodes.size() + 1) * 2 > child_tab.size()) child_grow();
            uint32_t i = (uint32_t)child_hash(parent, s, n) & child_mask;
            while (child_tab[i]) i = (i + 1) & child_mask;
            child_tab[i] = id + 1;
            Node& p = nodes[parent];
            if (p.last_kid) nodes[p.last_kid].next_sib = id; else p.first_kid = id;
            p.last_kid = id;
        }
        return id;
    }

    // what the last ingest() did to the node's tn_ip (lib/zk.js:176-189)
    bool ip_event = false, old_ip_valid = false; uint32_t old_ip_off = 0, old_ip_len = 0;
    uint32_t rev_clock = 0;                 // orders reverse-map writes across nodes

    // lib/zk.js:139-194 + the query-independent half of lib/server.js:249-274,296-332
    void ingest(uint32_t id, int v) {
        Node& nd = nodes[id];
        const uint16_t keep = nd.flags & (NF_REV | NF_REV_LOST);   // tn_ip outlives data that never reaches the address branch
        ip_event = false;
        nd.kind = K_INVALID; nd.flags = keep; nd.ttl = 30;
        // ttl of whatever is stored — record.ttl, then record[type].ttl (:270-274; resolvePtr reads it the
        // same way at :123-128, whatever the record's shape); kept even when unusable so that a service
        // child can tell "has its own ttl" from "inherits" (:389-393)
        int type = -1, sub = -1, tv = -1; const char* ts = nullptr; size_t tl = 0;
        if (v >= 0 && J.t[v].type == J_OBJ) {
            int a = J.get(v, "ttl");
            if (a >= 0) tv = a;
            type = J.get(v, "type");
            if (type >= 0 && J.t[type].type == J_STR) {
                ts = J.pool.data() + J.t[type].a; tl = J.t[type].b;
                sub = J.get(v, ts, tl);
                if (J.is_obj(sub)) { int b = J.get(sub, "ttl"); if (b >= 0) tv = b; }
            }
        }
        bool ttl_ok = true;
        if (tv >= 0) { nd.flags |= NF_HAS_TTL; ttl_ok = uint_ok(J, tv, 2147483648.0, nd.ttl); }
        if (ttl_ok) nd.flags |= NF_TTL_OK;
        if (v < 0 || J.t[v].type != J_OBJ) return;           // null, array (no .type), or nothing stored
        if (type < 0 || J.t[type].type != J_STR) return;
        bool hostlike = false, kidtype = false;
        for (auto h : kHostLike) if (strlen(h) == tl && !memcmp(h, ts, tl)) hostlike = true;
        for (auto h : kSvcKid) if (strlen(h) == tl && !memcmp(h, ts, tl)) kidtype = true;
        if (kidtype) nd.flags |= NF_KIDTYPE;
        if (hostlike) nd.flags |= NF_HOSTLIKE;
        if (!J.is_obj(sub)) return;                           // :251-253 / :366-368
        nd.flags |= NF_SUB_OBJ;
        bool is_service = tl == 7 && !memcmp(ts, "service", 7);
        bool is_db = tl == 8 && !memcmp(ts, "database", 8);
        if (hostlike) {
            // the old address leaves the reverse map, the new one enters it (lib/zk.js:183-188; strings only)
            ip_event = true; old_ip_valid = (keep & NF_REV) != 0; old_ip_off = nd.rev_off; old_ip_len = nd.rev_len;
            nd.flags &= ~(NF_REV | NF_REV_LOST);
            int ad = J.get(sub, "address");
            if (ad >= 0 && J.t[ad].type == J_NULL) nd.flags |= NF_ADDR_NULL;
            if (ad >= 0 && J.t[ad].type == J_STR) {
                const char* as = J.pool.data() + J.t[ad].a; size_t al = J.t[ad].b;
                if (ipv4_ok(as, al, nd.addr)) nd.flags |= NF_ADDR_OK;
                if (al > 0) {                                  // lib/zk.js:183-188 (strings only)
                    nd.flags |= NF_REV; nd.rev_off = (uint32_t)pool.size(); nd.rev_len = (uint32_t)al; nd.rev_seq = ++rev_clock;
                    pool.append(as, al);
                }
            }
            int pv = J.get(sub, "ports");
            if (pv >= 0 && !(J.t[pv].type == J_ARR && J.t[pv].b == 0)) {     // :383-385
                bool ok = J.t[pv].type == J_ARR;
                std::vector<uint16_t> pl;
                if (ok) {
                    uint32_t i = (uint32_t)pv + 1;
                    for (uint32_t c = 0; c < J.t[pv].b; c++) { uint32_t p; if (uint_ok(J, (int)i, 65536.0, p)) pl.push_back((uint16_t)p); else ok = false; i = J.t[i].next; }
                    if (pl.size() > 255) ok = false;
                }
                if (ok) { nd.flags |= NF_PORTS_LIST; nd.extra = (uint32_t)ports.size(); ports.push_back(std::move(pl)); }
                else nd.flags |= NF_PORTS_BAD;
            }
        }
        if (!ttl_ok) return;                                  // K_INVALID (contract)
        if (hostlike) { nd.kind = (nd.flags & NF_ADDR_OK) ? K_ADDR : K_ADDR_BAD; return; }
        if (is_db) {
            int pr = J.get(sub, "primary");
            nd.kind = (pr >= 0 && J.t[pr].type == J_STR && url_host_ipv4(J.pool.data() + J.t[pr].a, J.t[pr].b, nd.addr)) ? K_ADDR : K_ADDR_BAD;
            return;
        }
        if (is_service) {
            int s = sub;
            int inner = J.get(s, "service");
            if (inner >= 0 && J.t[inner].type == J_NULL) return;             // contract: null.ttl throws
            if (J.is_obj(inner)) s = inner;                                   // :324-325
            SvcInfo si; si.ttl = nd.ttl;
            int st = J.get(s, "ttl");
            if (st >= 0 && !uint_ok(J, st, 2147483648.0, si.ttl)) return;     // :331-332 (contract)
            int sv = J.get(s, "srvce"), pr = J.get(s, "proto"), po = J.get(s, "port");
            if (sv >= 0 && J.t[sv].type == J_STR) { si.has_srvce = true; si.srvce.assign(J.pool.data() + J.t[sv].a, J.t[sv].b); }
            if (pr >= 0 && J.t[pr].type == J_STR) { si.has_proto = true; si.proto.assign(J.pool.data() + J.t[pr].a, J.t[pr].b); }
            si.port_ok = uint_ok(J, po, 65536.0, si.port);
            nd.kind = K_SERVICE; nd.extra = (uint32_t)svcs.size(); svcs.push_back(std::move(si));
            return;
        }
        nd.kind = K_UNKNOWN;
    }

    // lower-cased fqdn of a node (lib/zk.js:80-84): name + '.' + parent's domain
    void domain_of(uint32_t id, std::string& out) const {
        out.clear();
        for (uint32_t cur = id;; cur = nodes[cur].parent) {
            if (cur == 0) { out += dns_domain; break; }
            size_t at = out.size();
            out.append(pool.data() + nodes[cur].name_off, nodes[cur].name_len);
            for (size_t i = at; i < out.size(); i++) if (out[i] >= 'A' && out[i] <= 'Z') out[i] = (char)(out[i] + 32);
            out.push_back('.');
        }
    }
};

// dotted name -> wire labels (no terminator); false if a label is empty or > 63
bool to_wire(const char* s, size_t n, std::string& out) {
    out.clear();
    size_t st = 0;
    for (size_t i = 0; i <= n; i++) {
        if (i == n || s[i] == '.') {
            size_t l = i - st;
            if (l < 1 || l > 63) return false;
            out.push_back((char)l); out.append(s + st, l);
            st = i + 1;
        }
    }
    return true;
}

struct TableBuilder {
    ZoneImage* z = nullptr;
    std::vector<uint8_t> arena;
    uint32_t mask = 0;
    std::string suffix;          // '.' + dnsDomain: what every reachable forward key ends with
    uint32_t arena_put(const void* p, size_t n, size_t align = 4) {
        while (arena.size() & (align - 1)) arena.push_back(0);
        uint32_t off = (uint32_t)arena.size();
        arena.insert(arena.end(), (const uint8_t*)p, (const uint8_t*)p + n);
        return off;
    }
    // A key as the callers spell it (forward: lower-cased dotted fqdn, reverse: address string) -> the form the
    // table stores and the kernel derives from a query (zone_image.h): forward = wire labels of what precedes
    // '.' + dnsDomain (the root domain itself = the empty key, which no query can spell).  false: a forward name no
    // query can reach (empty or over-long label in front of the suffix) — it is not stored.
    bool canon(uint32_t ns, const uint8_t* k, uint32_t len, std::string& out) const {
        if (ns != NS_FORWARD) { out.assign((const char*)k, len); return true; }
        out.clear();
        if (len + 1 == suffix.size() && memcmp(k, suffix.data() + 1, len) == 0) return true;         // the root
        if (len <= suffix.size() || memcmp(k + len - suffix.size(), suffix.data(), suffix.size())) return false;
        return to_wire((const char*)k, len - suffix.size(), out);
    }
    bool key_eq(const Slot& s, uint32_t ns, uint32_t h, const uint8_t* k, uint32_t len) const {
        if ((uint32_t)s.ns != ns) return false;
        if (len <= KEY_INLINE_MAX) return s.klen == len && memcmp(s.key, k, len) == 0;
        if (s.klen != KLEN_OVERFLOW) return false;
        uint32_t off, l, sh; memcpy(&off, s.key, 4); memcpy(&l, s.key + 4, 4); memcpy(&sh, s.key + 8, 4);
        return l == len && sh == h && memcmp(arena.data() + off, k, len) == 0;
    }
    uint32_t nranks = 1, rank = 0;
    bool mine(uint32_t ns, const uint8_t* dk, uint32_t dlen) const {
        if (nranks == 1) return true;
        std::string c;
        if (!canon(ns, dk, dlen, c)) return false;
        return owner_of(hash_key(ns, (const uint8_t*)c.data(), (uint32_t)c.size()), nranks) == rank;
    }
    bool failed = false;         // a cuckoo insertion ran out of kicks: the caller rebuilds with a larger table
    // host-side only, per slot: both hashes of the resident key (evictions need them) and the node that wrote it
    std::vector<uint32_t> h1s, h2s, own;
    uint64_t count = 0;          // resident keys
    // slots changed since the device last saw the table (bb_zone_apply -> bb_engine_apply_update)
    bool track = false; std::vector<uint32_t> dirty; std::vector<uint8_t> dirty_mark;
    void touch(uint32_t pos) { if (track && !dirty_mark[pos]) { dirty_mark[pos] = 1; dirty.push_back(pos); } }
    void reset(ZoneImage* img, uint32_t nslots) {
        z = img; mask = nslots - 1; failed = false; count = 0;
        h1s.assign(nslots, 0); h2s.assign(nslots, 0); own.assign(nslots, 0); disp.assign(nslots, 0);
        dirty.clear(); dirty_mark.assign(nslots, 0);
        arena.assign(32, 0);                                  // offset 0 is never a valid record
    }
    void fill(Slot& s, uint32_t h, uint32_t ns, const uint8_t* k, uint32_t len, uint8_t kind, uint32_t ttl, uint32_t val) {
        memset(&s, 0, sizeof s);
        bool clean = ns == NS_FORWARD;
        for (uint32_t i = 0; clean && i < len;) {             // wire labels: length byte, then that many label bytes
            const uint32_t l = k[i++];
            for (uint32_t j = 0; j < l && i < len; j++, i++) {
                const uint8_t c = k[i];
                if (!((c >= 'a' && c <= 'z') || (c >= '0' && c <= '9') || c == '_' || c == '-')) clean = false;
            }
        }
        s.ns = (uint8_t)ns;
        s.flags = clean ? SLOT_KEY_CLEAN : 0;
        if (len <= KEY_INLINE_MAX) { s.klen = (uint8_t)len; memcpy(s.key, k, len); }
        else { s.klen = KLEN_OVERFLOW; uint32_t off = arena_put(k, len); memcpy(s.key, &off, 4); memcpy(s.key + 4, &len, 4); memcpy(s.key + 8, &h, 4); }
        s.kind = kind; s.ttl = ttl; s.val = val;
    }
    int64_t find_canon(uint32_t ns, const uint8_t* k, uint32_t len) const {
        uint32_t h2;
        const uint32_t h = hash_key2(ns, k, len, &h2);
        for (uint32_t i : { slot1_of(h, mask), slot2_of(h, h2, mask) }) {
            const Slot& s = z->slots[i];
            if (s.kind != K_EMPTY && key_eq(s, ns, h, k, len)) return i;
        }
        return -1;
    }
    // slot holding the key (as the caller spells it), or -1
    int64_t find(uint32_t ns, const uint8_t* dk, uint32_t dlen) const {
        std::string c;
        if (!canon(ns, dk, dlen, c)) return -1;
        return find_canon(ns, (const uint8_t*)c.data(), (uint32_t)c.size());
    }
    // ---- residents and the SLOT_DISPLACED flag of their first slots -------------------------------------------
    // disp[p] = keys whose first slot is p but which live in their second slot; the flag at p mirrors disp[p] > 0.
    std::vector<uint32_t> disp;
    void set_resident(uint32_t pos, const Slot& c, uint32_t h1, uint32_t h2, uint32_t owner) {
        Slot& s = z->slots[pos];
        const uint8_t posflag = s.flags & SLOT_DISPLACED;
        s = c; s.flags = (uint8_t)((c.flags & ~SLOT_DISPLACED) | posflag);
        h1s[pos] = h1; h2s[pos] = h2; own[pos] = owner;
        touch(pos);
        const uint32_t first = slot1_of(h1, mask);
        if (first != pos && disp[first]++ == 0) { z->slots[first].flags |= SLOT_DISPLACED; touch(first); }
    }
    // the resident of pos leaves it (erased, or evicted by a kick); returns what it was
    Slot take_resident(uint32_t pos) {
        Slot& s = z->slots[pos];
        Slot was = s;
        const uint8_t posflag = s.flags & SLOT_DISPLACED;
        const uint32_t first = slot1_of(h1s[pos], mask);
        if (first != pos && --disp[first] == 0) { z->slots[first].flags &= (uint8_t)~SLOT_DISPLACED; touch(first); }
        memset(&s, 0, sizeof s); s.flags = posflag;
        h1s[pos] = 0; h2s[pos] = 0; own[pos] = 0;
        touch(pos);
        was.flags &= (uint8_t)~SLOT_DISPLACED;
        return was;
    }
    // a cuckoo table needs no tombstones: a lookup only ever reads the key's two slots
    void erase(uint32_t pos) { take_resident(pos); --count; }
    // insert or overwrite ("last writer wins", like assigning into a JS object); 2-choice cuckoo, first slot preferred.
    // Returns true when the key is new.
    bool put(uint32_t ns, const uint8_t* dk, uint32_t dlen, uint8_t kind, uint32_t ttl, uint32_t val, uint32_t owner) {
        std::string c;
        if (!canon(ns, dk, dlen, c)) return false;
        const uint8_t* k = (const uint8_t*)c.data(); const uint32_t len = (uint32_t)c.size();
        uint32_t h2;
        const uint32_t h = hash_key2(ns, k, len, &h2);
        const uint32_t i1 = slot1_of(h, mask), i2 = slot2_of(h, h2, mask);
        for (uint32_t i : { i1, i2 }) {
            Slot& s = z->slots[i];
            if (s.kind != K_EMPTY && key_eq(s, ns, h, k, len)) { s.kind = kind; s.ttl = ttl; s.val = val; own[i] = owner; touch(i); return false; }
        }
        Slot cur; fill(cur, h, ns, k, len, kind, ttl, val);
        uint32_t cur_h1 = h, cur_h2 = h2, cur_own = owner;
        uint32_t pos = z->slots[i1].kind == K_EMPTY ? i1 : (z->slots[i2].kind == K_EMPTY ? i2 : i1);
        ++count;
        for (int kick = 0; kick < 2000; kick++) {
            if (z->slots[pos].kind == K_EMPTY) { set_resident(pos, cur, cur_h1, cur_h2, cur_own); return true; }
            // evict the resident, move it to its other slot
            const uint32_t ev_h1 = h1s[pos], ev_h2 = h2s[pos], ev_own = own[pos];
            const Slot ev = take_resident(pos);
            set_resident(pos, cur, cur_h1, cur_h2, cur_own);
            cur = ev; cur_h1 = ev_h1; cur_h2 = ev_h2; cur_own = ev_own;
            const uint32_t a = slot1_of(cur_h1, mask), b = slot2_of(cur_h1, cur_h2, mask);
            pos = pos == a ? b : a;
        }
        if (getenv("BB_DEBUG")) fprintf(stderr, "cuckoo fail: ns=%u len=%u h=%08x i1=%u i2=%u mask=%u\n", ns, len, h, i1, i2, mask);
        failed = true;                                           // one key fell out: the caller lays the table out again
        return true;
    }
};

}  // namespace

// ---------------------------------------------------------------------------------------
// a zone: the flattened tree (kept, so that deltas can be applied) + its table image
// ---------------------------------------------------------------------------------------
struct bb_zone {
    bb::ZoneImage img;
    Builder B; TableBuilder T;
    std::string root_path;
    uint32_t nranks = 1, rank = 0;
    bool relaid = false;             // the table was laid out again since the device last saw it: full upload
    uint64_t arena_synced = 0;       // arena bytes the device already has
    uint64_t arena_base = 0;         // arena bytes right after the last full layout (no garbage yet)
    uint64_t sync_gen = 0;           // bumped whenever an engine takes the pending changes
};

namespace {

// ---- one node's forward key (lib/zk.js:96) and its payload ------------------------------------
// Returns false only for a snapshot the image cannot express (> 65535 children in a service).
bool emit_forward(bb_zone& zn, uint32_t id) {
    Builder& B = zn.B; TableBuilder& T = zn.T;
    const Node& nd = B.nodes[id];
    std::string dom, dom_wire, kw;
    B.domain_of(id, dom);
    const bool dom_ok = to_wire(dom.data(), dom.size(), dom_wire) && dom_wire.size() + 1 <= 255;
    // unspellable names are unreachable; other ranks own the rest
    if (!dom_ok || !T.mine(NS_FORWARD, (const uint8_t*)dom.data(), (uint32_t)dom.size())) return true;
    uint32_t val = nd.addr;
    if (nd.kind == K_SERVICE) {
        const SvcInfo& si = B.svcs[nd.extra];
        std::vector<uint32_t> kids;
        for (uint32_t k = nd.first_kid; k; k = B.nodes[k].next_sib)
            if ((B.nodes[k].flags & (NF_KIDTYPE | NF_DEAD)) == NF_KIDTYPE) kids.push_back(k);
        if (kids.size() > 65535) return false;
        // header | kid_info | A answers | KidRecs | additional RRs | SRV answers: ready wire bytes, one section per kind (zone_image.h)
        SvcHdr h; memset(&h, 0, sizeof h);
        h.ttl = si.ttl; h.nkids = (uint16_t)kids.size();
        h.dom_wl = (uint8_t)(dom_wire.size() + 1);
        {
            std::string sp;
            const bool s_ok = si.has_srvce && si.srvce.size() >= 1 && si.srvce.size() <= 63;
            const bool p_ok = si.has_proto && si.proto.size() >= 1 && si.proto.size() <= 63;
            if (!s_ok || !p_ok) h.hflags |= SVC_SP_NEVER;
            else {
                sp.push_back((char)si.srvce.size()); sp += si.srvce; sp.push_back((char)si.proto.size()); sp += si.proto;
                h.sp_len = (uint8_t)sp.size();
                if (sp.size() <= sizeof h.sp) memcpy(h.sp, sp.data(), sp.size());
                else { h.hflags |= SVC_SP_EXT; const uint32_t off = T.arena_put(sp.data(), sp.size()); memcpy(h.sp, &off, 4); }
            }
        }
        auto be16 = [](std::vector<uint8_t>& v, uint32_t x) { v.push_back((uint8_t)(x >> 8)); v.push_back((uint8_t)x); };
        auto be32 = [](std::vector<uint8_t>& v, uint32_t x) { v.push_back((uint8_t)(x >> 24)); v.push_back((uint8_t)(x >> 16)); v.push_back((uint8_t)(x >> 8)); v.push_back((uint8_t)x); };
        uint64_t n_valid = 0, sum_ports = 0, sum_wl = 0, sum_wl_ports = 0, jobs_srv = 0;
        std::vector<std::vector<uint8_t>> a_rr(kids.size()), add_rr(kids.size()), srv_rr(kids.size());
        std::vector<KidRec> recs(kids.size());
        std::vector<uint32_t> info(kids.size(), 0);
        size_t add_stride = 16, srv_stride = 16;
        for (size_t ki = 0; ki < kids.size(); ki++) {
            const Node& kn = B.nodes[kids[ki]];
            KidRec kr; memset(&kr, 0, sizeof kr);
            std::vector<uint16_t> pl;
            bool name_ok = to_wire(B.pool.data() + kn.name_off, kn.name_len, kw) && kw.size() + dom_wire.size() + 1 <= 255;
            if (!(kn.flags & NF_SUB_OBJ)) kr.flags = KID_BAD_A | KID_BAD_SRV;            // :366-376
            else if (kn.flags & NF_ADDR_NULL) kr.flags = KID_ADDR_NULL;                    // :378-381
            else {
                bool bad = !(kn.flags & NF_ADDR_OK) || !(kn.flags & NF_TTL_OK);
                bool bad_srv = bad || !name_ok || (kn.flags & NF_PORTS_BAD);
                if (kn.flags & NF_PORTS_LIST) pl = B.ports[kn.extra];
                else if (si.port_ok) pl.push_back((uint16_t)si.port);                     // :383-385
                else bad_srv = true;
                kr.flags = (bad ? KID_BAD_A : 0) | (bad_srv ? KID_BAD_SRV : 0);
                if (kn.flags & NF_HAS_TTL) kr.flags |= KID_HAS_RTTL;
                kr.addr = kn.addr; kr.rttl = kn.ttl;
                if (bad_srv) pl.clear();
            }
            if (!name_ok) kw.clear();
            kr.wire_len = (uint8_t)kw.size(); kr.nports = (uint8_t)pl.size();
            if (kr.flags & KID_BAD_A) h.hflags |= SVC_BAD_A;
            if (kr.flags & KID_BAD_SRV) h.hflags |= SVC_BAD_SRV;
            if (!(kr.flags & KID_ADDR_NULL)) {
                ++n_valid; sum_ports += pl.size(); sum_wl += kw.size(); sum_wl_ports += pl.size() * kw.size();
                // the pieces a whole SRV answer copies from this child: its run of SRV RRs and its additional RR, 64 bytes per job
                jobs_srv += (pl.size() * kid_srv_len((uint32_t)kw.size(), (uint32_t)dom_wire.size() + 1) + 63) / 64 + (kid_add_len((uint32_t)kw.size()) + 63) / 64;
            }
            info[ki] = (uint32_t)kr.flags | (uint32_t)kr.wire_len << 8 | (uint32_t)kr.nports << 16;
            // the child's pieces: KidRec, A answer, additional RR, SRV answers
            recs[ki] = kr;
            const uint32_t rttl = (kr.flags & KID_HAS_RTTL) ? kr.rttl : si.ttl;
            std::vector<uint8_t>& ar = a_rr[ki];
            be16(ar, 0xC00C); be16(ar, 1); be16(ar, 1); be32(ar, si.ttl < rttl ? si.ttl : rttl); be16(ar, 4); be32(ar, kr.addr);
            std::vector<uint8_t>& ad = add_rr[ki];
            ad.insert(ad.end(), kw.begin(), kw.end());
            be16(ad, 0xC000u | (12u + h.sp_len)); be16(ad, 1); be16(ad, 1); be32(ad, rttl); be16(ad, 4); be32(ad, kr.addr);
            std::vector<uint8_t>& sr = srv_rr[ki];
            for (uint16_t port : pl) {
                be16(sr, 0xC00C); be16(sr, 33); be16(sr, 1); be32(sr, si.ttl); be16(sr, (uint32_t)(6 + kw.size() + dom_wire.size() + 1));
                be16(sr, 0); be16(sr, 10); be16(sr, port);
                sr.insert(sr.end(), kw.begin(), kw.end());
                sr.insert(sr.end(), dom_wire.begin(), dom_wire.end()); sr.push_back(0);
            }
            if (((ad.size() + 15) & ~(size_t)15) > add_stride) add_stride = (ad.size() + 15) & ~(size_t)15;
            if (((sr.size() + 15) & ~(size_t)15) > srv_stride) srv_stride = (sr.size() + 15) & ~(size_t)15;
        }
        if (srv_stride / 16 > 0xFFFF || add_stride > SVC_ADD_STRIDE_MAX) return false;
        if (add_stride > 240) add_stride = SVC_ADD_STRIDE_MAX;          // the one stride over 15 units the header can name
        h.stride16 = (uint16_t)(srv_stride / 16);
        h.hflags |= (uint8_t)svc_add_stride_bits((uint32_t)add_stride);
        // sums the kernel sizes an answer from without walking the children; a service too large for them is walked
        if (n_valid > 0xFFFF || sum_ports > 0xFFFF || sum_wl > 0xFFFF || sum_wl_ports > 0xFFFF || jobs_srv > 0xFFFF) h.hflags |= SVC_BAD_A | SVC_BAD_SRV;
        h.n_valid = (uint16_t)n_valid; h.sum_ports = (uint16_t)sum_ports; h.sum_wl = (uint16_t)sum_wl; h.sum_wl_ports = (uint16_t)sum_wl_ports;
        h.jobs_srv = (uint16_t)jobs_srv;
        const uint32_t nk = (uint32_t)kids.size();
        std::vector<uint8_t> rec(svc_record_len(nk, (uint32_t)add_stride, (uint32_t)srv_stride), 0);     // zero padded throughout
        memcpy(rec.data(), &h, sizeof h);
        if (!info.empty()) memcpy(rec.data() + sizeof h, info.data(), 4 * info.size());
        for (size_t ki = 0; ki < kids.size(); ki++) {
            memcpy(rec.data() + svc_a_off(nk) + 16 * ki, a_rr[ki].data(), 16);
            memcpy(rec.data() + svc_rec_off(nk) + 16 * ki, &recs[ki], sizeof(KidRec));
            memcpy(rec.data() + svc_add_off(nk) + add_stride * ki, add_rr[ki].data(), add_rr[ki].size());
            memcpy(rec.data() + svc_srv_off(nk, (uint32_t)add_stride) + srv_stride * ki, srv_rr[ki].data(), srv_rr[ki].size());
        }
        val = T.arena_put(rec.data(), rec.size(), 32);
    }
    uint32_t ttl = nd.kind == K_SERVICE ? B.svcs[nd.extra].ttl : nd.ttl;
    if (T.put(NS_FORWARD, (const uint8_t*)dom.data(), (uint32_t)dom.size(), nd.kind, ttl, val, id)) zn.img.n_fwd++;
    return true;
}

// ---- the reverse key a node registered (lib/zk.js:183-188), answered as lib/server.js:123-130 ----
void emit_reverse(bb_zone& zn, uint32_t id) {
    Builder& B = zn.B; TableBuilder& T = zn.T;
    const Node nd = B.nodes[id];
    if ((nd.flags & (NF_REV | NF_REV_LOST)) != NF_REV || nd.rev_len > 253) return;
    const uint8_t* key = (const uint8_t*)B.pool.data() + nd.rev_off;
    if (!T.mine(NS_REVERSE, key, nd.rev_len)) return;
    std::string dom, dom_wire;
    B.domain_of(id, dom);
    const bool dom_ok = to_wire(dom.data(), dom.size(), dom_wire) && dom_wire.size() + 1 <= 255;
    uint8_t kind = K_PTR_BAD; uint32_t val = 0;
    if ((nd.flags & NF_TTL_OK) && dom_ok) {
        std::string t; t.push_back((char)(dom_wire.size() + 1)); t += dom_wire; t.push_back(0);
        val = T.arena_put(t.data(), t.size()); kind = K_PTR;
    }
    // assignment into ca_revLookup replaces whoever was there: that node's entry is gone for good, even if
    // this one later moves to another address (:183-188)
    const int64_t prev = T.find(NS_REVERSE, key, nd.rev_len);
    if (prev >= 0 && T.own[prev] != id) B.nodes[T.own[prev]].flags |= NF_REV_LOST;
    if (T.put(NS_REVERSE, key, nd.rev_len, kind, nd.ttl, val, id)) zn.img.n_rev++;
}

// ---- (re)build the whole table from the tree -----------------------------------------------------
int layout(bb_zone& zn) {
    Builder& B = zn.B; TableBuilder& T = zn.T; ZoneImage& Z = zn.img;
    for (uint32_t grow = 0;; grow++) {      // cuckoo insertion can (rarely) fail: rebuild one size up
        uint64_t nkeys = 0;
        for (auto& nd : B.nodes) nkeys += ((nd.flags & NF_DEAD) ? 0 : 1) + ((nd.flags & NF_REV) ? 1 : 0);
        // 2-choice cuckoo needs a load factor below 0.5: size for <= 0.45 (a shard holds ~1/nranks of the keys)
        uint64_t want = (nkeys * 22 / 10) / zn.nranks + (zn.nranks > 1 ? nkeys / (4 * zn.nranks) : 0) + 64; uint32_t ns = 64;
        while (ns < want) { ns <<= 1; if (ns == 0) return BB_ERR_NOMEM; }
        ns <<= grow;
        if (ns == 0) return BB_ERR_NOMEM;
        free(Z.slots); Z.slots = nullptr; Z.n_fwd = Z.n_rev = 0;
        Z.nslots = ns;
        Z.slots = (Slot*)aligned_alloc(64, (size_t)ns * sizeof(Slot));
        if (!Z.slots) return BB_ERR_NOMEM;
        memset(Z.slots, 0, (size_t)ns * sizeof(Slot));
        const bool track = T.track;
        T.track = false;
        T.reset(&Z, ns); T.nranks = zn.nranks; T.rank = zn.rank;
        Z.n_nodes = B.nodes.size();
        // Forward keys in creation order: the TreeNode constructor takes the key from an earlier node
        // that spells it the same (:96); an unbound node that held it took it along (:205-207).
        std::string dom;
        for (uint32_t id = 0; id < B.nodes.size(); id++) {
            if (!(B.nodes[id].flags & NF_DEAD)) { if (!emit_forward(zn, id)) return BB_ERR_SNAPSHOT; continue; }
            B.domain_of(id, dom);
            const int64_t pos = T.find(NS_FORWARD, (const uint8_t*)dom.data(), (uint32_t)dom.size());
            if (pos >= 0) { T.erase((uint32_t)pos); Z.n_fwd--; }
        }
        // Reverse keys in the order they were written (last writer wins, :187-188); an unbound node
        // keeps its entry (unbind never removes it).
        std::vector<std::pair<uint32_t, uint32_t>> rev;
        for (uint32_t id = 0; id < B.nodes.size(); id++) if (B.nodes[id].flags & NF_REV) rev.emplace_back(B.nodes[id].rev_seq, id);
        std::sort(rev.begin(), rev.end());
        for (auto& e : rev) emit_reverse(zn, e.second);
        T.track = track;
        if (!T.failed) break;
        if (grow > 3) return BB_ERR_NOMEM;
    }
    while (T.arena.size() & 31) T.arena.push_back(0);
    Z.arena = T.arena.data(); Z.arena_len = T.arena.size();
    Z.ready = 1;                                              // the root TreeNode exists (lib/zk.js:55-58)
    zn.relaid = true; zn.arena_synced = 0; zn.arena_base = Z.arena_len;
    T.dirty.clear(); std::fill(T.dirty_mark.begin(), T.dirty_mark.end(), 0);
    return BB_OK;
}

// ---- one snapshot / delta line ---------------------------------------------------------------------
enum { LINE_SKIP = 0, LINE_DATA = 1, LINE_DELETE = 2, LINE_BAD = -1 };
// Parses the line into B.J and resolves its path.  LINE_DATA: *id = the node (created when its parent is
// mirrored and `create` allows), *v = tape index of the accepted value or -1 when the content is ignored
// (lib/zk.js:141-155: unparsable, or neither null nor an object).  *created reports a new node.
int read_line(bb_zone& zn, const char* a, const char* b, uint32_t* id, int* v, bool* created) {
    Builder& B = zn.B;
    B.J.clear();
    *created = false; *v = -1;
    int ent = B.J.parse(a, b);
    if (ent < 0 || B.J.t[ent].type != J_OBJ) return LINE_BAD;
    int path = B.J.get(ent, "path");
    if (path < 0 || B.J.t[path].type != J_STR) return LINE_BAD;
    const int del = B.J.get(ent, "deleted");
    const bool deleting = del >= 0 && B.J.t[del].type == J_TRUE;
    const char* ps = B.J.pool.data() + B.J.t[path].a; size_t pl = B.J.t[path].b;
    const std::string& root_path = zn.root_path;
    if (pl == root_path.size() && !memcmp(ps, root_path.data(), pl)) *id = 0;
    else {
        if (pl <= root_path.size() + 1 || memcmp(ps, root_path.data(), root_path.size()) || ps[root_path.size()] != '/') return LINE_SKIP;
        size_t i = root_path.size() + 1; uint32_t cur = 0; int found = -1;
        for (;;) {
            size_t j = i; while (j < pl && ps[j] != '/') ++j;
            if (j == i) return LINE_SKIP;                          // empty component
            found = B.find_child(cur, ps + i, j - i);
            if (j == pl) {                                         // last component: the znode itself
                if (found < 0) {
                    if (deleting) return LINE_SKIP;
                    found = (int)B.add_node(cur, ps + i, j - i); *created = true;
                }
                break;
            }
            if (found < 0) return LINE_SKIP;                       // parent not mirrored
            cur = (uint32_t)found; i = j + 1;
            if (i >= pl) return LINE_SKIP;                         // trailing '/'
        }
        *id = (uint32_t)found;
    }
    if (deleting) return LINE_DELETE;
    int raw = B.J.get(ent, "raw"), data = B.J.get(ent, "data");
    if (raw >= 0 && B.J.t[raw].type == J_STR) {
        // the znode's bytes: JSON.parse them (lib/zk.js:141-148); failure = ignored
        std::string rs(B.J.pool.data() + B.J.t[raw].a, B.J.t[raw].b);
        int pv = B.J.parse(rs.data(), rs.data() + rs.size());
        if (pv >= 0 && (B.J.t[pv].type == J_NULL || B.J.is_obj(pv))) *v = pv;      // :149-155
    } else if (data >= 0) {
        if (B.J.t[data].type == J_NULL || B.J.is_obj(data)) *v = data;
    }
    return LINE_DATA;
}

template <class F>
int for_each_line(const char* buf, size_t len, F&& f) {
    const char* p = buf; const char* end = buf + len;
    while (p < end) {
        const char* nl = (const char*)memchr(p, '\n', (size_t)(end - p));
        const char* a = p; const char* b = nl ? nl : end;
        p = nl ? nl + 1 : end;
        while (a < b && (*a == ' ' || *a == '\t' || *a == '\r')) ++a;
        while (b > a && (b[-1] == ' ' || b[-1] == '\t' || b[-1] == '\r')) --b;
        if (a == b) continue;
        int rc = f(a, b);
        if (rc != BB_OK) return rc;
    }
    return BB_OK;
}

}  // namespace

// ---------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------
extern "C" void bb_zone_free(bb_zone* z);

extern "C" bb_zone* bb_zone_build_shard(const char* buf, size_t len, const char* dns_domain, uint32_t nranks,
                                        uint32_t rank, int* err) {
    auto fail = [&](int e) -> bb_zone* { if (err) *err = e; return nullptr; };
    if (err) *err = BB_OK;
    if ((!buf && len) || !dns_domain || nranks == 0 || rank >= nranks) return fail(BB_ERR_ARG);
    bb_zone* zone = new bb_zone();
    memset(&zone->img, 0, sizeof zone->img);
    zone->nranks = nranks; zone->rank = rank;
    Builder& B = zone->B;
    auto bail = [&](int e) -> bb_zone* { bb_zone_free(zone); return fail(e); };
    B.dns_domain = dns_domain;
    zone->T.suffix = std::string(".") + dns_domain;
    // ZKCache.isReady() compares with options.domain verbatim (lib/zk.js:55-58) while keys are
    // lower-cased (:84): an upper-case domain is never ready.  We require lower case instead.
    for (char c : B.dns_domain) if (c >= 'A' && c <= 'Z') return bail(BB_ERR_DOMAIN);
    std::string w;
    if (B.dns_domain.empty() || !to_wire(B.dns_domain.data(), B.dns_domain.size(), w) || w.size() + 1 > 244) return bail(BB_ERR_DOMAIN);
    // root node (lib/zk.js:68-76): exists as soon as the cache is built, data null
    size_t dot = B.dns_domain.find('.');
    std::string first = B.dns_domain.substr(0, dot);
    B.add_node(0, first.data(), first.size());
    {                                                              // lib/zk.js:225-228
        std::vector<std::string> parts; size_t s = 0;
        for (;;) { size_t d = B.dns_domain.find('.', s); parts.push_back(B.dns_domain.substr(s, d == std::string::npos ? d : d - s)); if (d == std::string::npos) break; s = d + 1; }
        for (size_t i = parts.size(); i-- > 0;) { zone->root_path += "/"; zone->root_path += parts[i]; }
    }
    std::vector<uint8_t> seen_data(1, 0);
    int rc = for_each_line(buf, len, [&](const char* a, const char* b) -> int {
        uint32_t id; int v; bool created;
        const int what = read_line(*zone, a, b, &id, &v, &created);
        if (what == LINE_BAD || what == LINE_DELETE) return BB_ERR_SNAPSHOT;   // a snapshot states what exists
        if (what == LINE_SKIP) return BB_OK;
        if (seen_data.size() < B.nodes.size()) seen_data.resize(B.nodes.size(), 0);
        if (seen_data[id]) return BB_ERR_SNAPSHOT;                 // one line per znode
        seen_data[id] = 1;
        if (v >= 0) B.ingest(id, v);
        return BB_OK;
    });
    if (rc != BB_OK) return bail(rc);
    rc = layout(*zone);
    if (rc != BB_OK) return bail(rc);
    zone->T.track = true;
    return zone;
}

extern "C" bb_zone* bb_zone_build(const char* buf, size_t len, const char* dns_domain, int* err) {
    return bb_zone_build_shard(buf, len, dns_domain, 1, 0, err);
}

// Apply a delta — the batched analogue of the ZooKeeper watch events lib/zk.js handles — to a built zone:
//   {"path": P, "data": D} / {"path": P, "raw": "<znode bytes>"}   the znode now holds this content
//       (dataChanged, :139-194); a path not seen before is a new child appended to its parent's child
//       list (childrenChanged, :120-130) — its parent must already be mirrored
//   {"path": P, "deleted": true}                                       the znode and its subtree are gone
//       (childrenChanged -> unbind, :131-133,195-208)
// Only the keys that depend on the touched nodes are re-derived: the node's own key, the reverse-map
// entry of its address, and its parent's service record.  The changed slots and the arena tail are
// what bb_engine_apply_update ships to the device.
extern "C" int bb_zone_apply(bb_zone* zone, const char* buf, size_t len) {
    if (!zone || (!buf && len)) return BB_ERR_ARG;
    Builder& B = zone->B; TableBuilder& T = zone->T;
    std::vector<uint32_t> stack;
    auto refresh_parent = [&](uint32_t id) -> bool {               // the parent's answer lists its children (:352-417)
        if (id == 0) return true;
        const uint32_t p = B.nodes[id].parent;
        const Node& pn = B.nodes[p];
        if ((pn.flags & NF_DEAD) || pn.kind != K_SERVICE) return true;
        std::string dom; B.domain_of(p, dom);
        const int64_t pos = T.find(NS_FORWARD, (const uint8_t*)dom.data(), (uint32_t)dom.size());
        if (pos < 0 || T.own[pos] != p) return true;               // the key belongs to a case-twin (or another rank)
        return emit_forward(*zone, p);
    };
    int rc = for_each_line(buf, len, [&](const char* a, const char* b) -> int {
        uint32_t id; int v; bool created;
        const int what = read_line(*zone, a, b, &id, &v, &created);
        if (what == LINE_BAD) return BB_ERR_SNAPSHOT;
        if (what == LINE_SKIP) return BB_OK;
        if (what == LINE_DELETE) {
            if (id == 0) return BB_ERR_SNAPSHOT;                   // the root of the mirrored subtree stays
            stack.assign(1, id);
            while (!stack.empty()) {                               // unbind(): the node and everything below it
                const uint32_t cur = stack.back(); stack.pop_back();
                for (uint32_t k = B.nodes[cur].first_kid; k; k = B.nodes[k].next_sib) if (!(B.nodes[k].flags & NF_DEAD)) stack.push_back(k);
                std::string dom; B.domain_of(cur, dom);
                const int64_t pos = T.find(NS_FORWARD, (const uint8_t*)dom.data(), (uint32_t)dom.size());
                if (pos >= 0 && T.own[pos] == cur) { T.erase((uint32_t)pos); zone->img.n_fwd--; }   // `=== this` (:205-207)
                B.nodes[cur].flags |= NF_DEAD;                     // its reverse entry, if any, stays (never removed)
            }
            return refresh_parent(id) ? BB_OK : BB_ERR_SNAPSHOT;
        }
        // LINE_DATA
        const bool had_rev = (B.nodes[id].flags & NF_REV) != 0;
        if (v >= 0) {
            B.ingest(id, v);
            if (B.ip_event) {
                if (B.old_ip_valid && B.old_ip_len <= 253) {       // `delete ca_revLookup[this.tn_ip]`, whoever wrote it last
                    const uint8_t* ok = (const uint8_t*)B.pool.data() + B.old_ip_off;
                    const int64_t pos = T.find(NS_REVERSE, ok, B.old_ip_len);
                    if (pos >= 0) {
                        if (T.own[pos] != id) B.nodes[T.own[pos]].flags |= NF_REV_LOST;   // that node's tn_ip stays, its entry is gone
                        T.erase((uint32_t)pos); zone->img.n_rev--;
                    }
                }
                emit_reverse(*zone, id);                           // `ca_revLookup[addr] = this`
            } else if (had_rev) {                                  // the entry (if still ours) answers with the new ttl
                const Node& nd = B.nodes[id];
                const int64_t pos = nd.rev_len <= 253 ? T.find(NS_REVERSE, (const uint8_t*)B.pool.data() + nd.rev_off, nd.rev_len) : -1;
                if (pos >= 0 && T.own[pos] == id) emit_reverse(*zone, id);
            }
        }
        if (created) {                                             // the TreeNode constructor takes the key (:96)
            if (!emit_forward(*zone, id)) return BB_ERR_SNAPSHOT;
        } else if (v >= 0) {                                       // data changed: only the node that holds the key answers
            std::string dom; B.domain_of(id, dom);
            const int64_t pos = T.find(NS_FORWARD, (const uint8_t*)dom.data(), (uint32_t)dom.size());
            if (pos >= 0 && T.own[pos] == id && !emit_forward(*zone, id)) return BB_ERR_SNAPSHOT;
        }
        if ((created || v >= 0) && !refresh_parent(id)) return BB_ERR_SNAPSHOT;
        return BB_OK;
    });
    // Whatever happened to the lines — earlier lines of a delta stay applied when a later one is bad — the image must
    // describe the builder's state again before anyone reads it: records appended above may have moved the arena.
    // A cuckoo insertion that failed, a table filling past what two choices sustain, or an arena that is mostly
    // superseded records (every re-derived service / PTR record is appended): lay it out again.
    int rc2 = BB_OK;
    if (T.failed || T.count * 100 > (uint64_t)zone->img.nslots * 47 || T.arena.size() > 2 * zone->arena_base + (16u << 20))
        rc2 = layout(*zone);
    while (T.arena.size() & 31) T.arena.push_back(0);
    zone->img.arena = T.arena.data(); zone->img.arena_len = T.arena.size();
    zone->img.n_nodes = B.nodes.size();
    return rc != BB_OK ? rc : rc2;
}

// What the device has not seen yet (used by bb_engine_apply_update in engine.cu).
extern "C" int bb_zone_pending(const bb_zone* z, const uint32_t** slots, uint32_t* n_slots, uint64_t* arena_from, int* relaid) {
    if (!z) return BB_ERR_ARG;
    *slots = z->T.dirty.data(); *n_slots = (uint32_t)z->T.dirty.size(); *arena_from = z->arena_synced; *relaid = z->relaid ? 1 : 0;
    return BB_OK;
}
extern "C" void bb_zone_mark_synced(bb_zone* z) {
    if (!z) return;
    for (uint32_t pos : z->T.dirty) z->T.dirty_mark[pos] = 0;
    z->T.dirty.clear(); z->relaid = false; z->arena_synced = z->img.arena_len; z->sync_gen++;
}
extern "C" uint64_t bb_zone_sync_gen(const bb_zone* z) { return z ? z->sync_gen : 0; }

extern "C" void bb_zone_free(bb_zone* z) {
    if (!z) return;
    free(z->img.slots);                                        // img.arena is the table builder's vector
    delete z;
}

extern "C" uint64_t bb_zone_stat(const bb_zone* z, int what) {
    if (!z) return 0;
    switch (what) {
    case 0: return z->img.n_nodes;
    case 1: return z->img.n_fwd;
    case 2: return z->img.n_rev;
    case 3: return z->img.nslots;
    case 4: return (uint64_t)z->img.nslots * sizeof(bb::Slot) + z->img.arena_len;
    case 5: return z->img.arena_len;
    case 6: return z->T.dirty.size();                          // slots changed since the device last saw the table
    case 7: return z->relaid ? 1 : 0;
    case 8: { uint64_t d = 0; for (uint32_t v : z->T.disp) d += v; return d; }      // keys living in their second slot
    }
    return 0;
}

// Diagnostics: what the image holds for a key (host side; the tests compare an updated zone with a fresh
// build through it).  rec = the payload in a position-independent form: service header + srvce + proto
// + every child (KidRec, ports, name); PTR target wire bytes.  Returns 1 when the key is present.
extern "C" int bb_zone_probe(const bb_zone* z, uint32_t ns, const uint8_t* key, uint32_t len, uint8_t* kind, uint32_t* ttl,
                             uint32_t* val, uint8_t* rec, uint32_t rec_cap, uint32_t* rec_len) {
    if (!z || !key) return 0;
    const int64_t pos = z->T.find(ns, key, len);
    if (pos < 0) return 0;
    const bb::Slot& s = z->img.slots[pos];
    if (kind) *kind = s.kind;
    if (ttl) *ttl = s.ttl;
    if (val) *val = (s.kind == bb::K_SERVICE || s.kind == bb::K_PTR) ? 0 : s.val;
    std::string out;
    const uint8_t* A = z->T.arena.data();
    if (s.kind == bb::K_SERVICE) {
        bb::SvcHdr h; memcpy(&h, A + s.val, sizeof h);
        std::string ext;
        if (h.hflags & bb::SVC_SP_EXT) { uint32_t off; memcpy(&off, h.sp, 4); ext.assign((const char*)A + off, h.sp_len); memset(h.sp, 0, 4); }
        out.append((const char*)&h, sizeof h); out += ext;                 // offsets are relative to the record: position independent
        const size_t body = bb::svc_record_len(h.nkids, bb::svc_add_stride(h.hflags), (uint32_t)h.stride16 * 16) - sizeof h;
        out.append((const char*)(A + s.val + sizeof h), body);
    } else if (s.kind == bb::K_PTR) {
        out.append((const char*)(A + s.val + 1), A[s.val]);
    }
    if (rec_len) *rec_len = (uint32_t)out.size();
    if (rec && out.size() <= rec_cap) memcpy(rec, out.data(), out.size());
    return 1;
}

// used by engine.cu
extern "C" const bb::ZoneImage* bb_zone_image(const bb_zone* z) { return z ? &z->img : nullptr; }
