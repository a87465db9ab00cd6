// TEST INFRASTRUCTURE — CPU oracle for the binder resolve path.  NOT the product.
//
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
// may build, load or call this file.  binder_b200/ never includes or links it.
//
// PARITY STATUS: the resolve logic (lib/server.js, lib/zk.js) is restated from sources that
// are in the reference tree (TritonDataCenter/binder) and is pinned by the reference's own 13 integration-test cases
// (tests/golden/).  The byte-level codec lives in the un-vendored npm dependency
// mname@1.5.1 (package.json:15, package-lock.json:1124-1126): its layout decisions are
// restated here from DESIGN.md "Wire spec" and are PARITY-UNPINNED at byte level (the
// reference's tests only pin rcode / answer count / owner / ttl / type / rdata via dig text).
//
// Restates (file:line in the reference tree):
//   lib/zk.js:78-97,108-114   TreeNode (lower-cased domain key, case-preserved name, child order)
//   lib/zk.js:139-194         onDataChanged: JSON.parse ingest + reverse map
//   lib/zk.js:55-67           isReady / lookup / reverseLookup
//   lib/server.js:40-53       shuffle            lib/server.js:55-65  isSuffix
//   lib/server.js:67-134      resolvePtr         lib/server.js:136-429 resolve
//   lib/server.js:471-507     onQuery dispatch
//   mname call sites          lib/server.js:74,116,130,146,286,299,310,398-402,413-414,427
//
// Style: literal.  Records stay a parsed-JSON DOM and every query walks it the way the
// JavaScript does (property reads, typeof tests); nothing is pre-flattened.
#include <cstdint>
#include <cstring>
#include <cstdlib>
#include <cmath>
#include <string>
#include <vector>
#include <unordered_map>
#include <memory>
#include <thread>
#include <algorithm>

namespace {

// ---------------------------------------------------------------------------------------
// JSON.parse
// ---------------------------------------------------------------------------------------
struct JVal;
using JObj = std::vector<std::pair<std::string, JVal>>;
struct JVal {
    enum T : uint8_t { UNDEF, NUL, BOOL, NUM, STR, ARR, OBJ } t = UNDEF;
    bool b = false;
    double num = 0;
    std::string str;
    std::unique_ptr<std::vector<JVal>> arr;
    std::unique_ptr<JObj> obj;
    bool is_object() const { return t == ARR || t == OBJ; }   // typeof 'object' && !== null
    const JVal& get(const char* key) const;                  // own-property read
    const JVal& get(const std::string& key) const { return get(key.c_str()); }
};
const JVal kUndef;
const JVal& JVal::get(const char* key) const {
    if (t != OBJ) return kUndef;
    for (auto& kv : *obj) if (kv.first == key) return kv.second;
    return kUndef;
}

struct JParser {
    const char* p; const char* e; bool ok = true;
    JParser(const char* b, const char* end) : p(b), e(end) {}
    void ws() { while (p < e && (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r')) ++p; }
    bool lit(const char* s) {
        size_t n = strlen(s);
        if ((size_t)(e - p) < n || memcmp(p, s, n) != 0) return false;
        p += n; return true;
    }
    static void utf8(std::string& o, uint32_t c) {
        if (c < 0x80) o += (char)c;
        else if (c < 0x800) { o += (char)(0xC0 | (c >> 6)); o += (char)(0x80 | (c & 0x3F)); }
        else if (c < 0x10000) { o += (char)(0xE0 | (c >> 12)); o += (char)(0x80 | ((c >> 6) & 0x3F)); o += (char)(0x80 | (c & 0x3F)); }
        else { o += (char)(0xF0 | (c >> 18)); o += (char)(0x80 | ((c >> 12) & 0x3F)); o += (char)(0x80 | ((c >> 6) & 0x3F)); o += (char)(0x80 | (c & 0x3F)); }
    }
    bool hex4(uint32_t& v) {
        if (e - p < 4) return false;
        v = 0;
        for (int i = 0; i < 4; i++) {
            char c = p[i]; v <<= 4;
            if (c >= '0' && c <= '9') v |= c - '0';
            else if (c >= 'a' && c <= 'f') v |= c - 'a' + 10;
            else if (c >= 'A' && c <= 'F') v |= c - 'A' + 10;
            else return false;
        }
        p += 4; return true;
    }
    bool string(std::string& o) {
        if (p >= e || *p != '"') return false;
        ++p;
        while (p < e) {
            unsigned char c = (unsigned char)*p++;
            if (c == '"') return true;
            if (c < 0x20) return false;
            if (c != '\\') { o += (char)c; continue; }
            if (p >= e) return false;
            char x = *p++;
            switch (x) {
            case '"': o += '"'; break;   case '\\': o += '\\'; break;
            case '/': o += '/'; break;   case 'b': o += '\b'; break;
            case 'f': o += '\f'; break;  case 'n': o += '\n'; break;
            case 'r': o += '\r'; break;  case 't': o += '\t'; break;
            case 'u': {
                uint32_t v; if (!hex4(v)) return false;
                if (v >= 0xD800 && v < 0xDC00 && e - p >= 6 && p[0] == '\\' && p[1] == 'u') {
                    const char* save = p; p += 2; uint32_t lo;
                    if (hex4(lo) && lo >= 0xDC00 && lo < 0xE000) v = 0x10000 + ((v - 0xD800) << 10) + (lo - 0xDC00);
                    else p = save;
                }
                utf8(o, v); break; }
            default: return false;
            }
        }
        return false;
    }
    bool number(double& d) {
        const char* s = p;
        if (p < e && *p == '-') ++p;
        if (p >= e) return false;
        if (*p == '0') ++p;
        else if (*p >= '1' && *p <= '9') { while (p < e && *p >= '0' && *p <= '9') ++p; }
        else return false;
        if (p < e && *p == '.') { ++p; if (p >= e || *p < '0' || *p > '9') return false; while (p < e && *p >= '0' && *p <= '9') ++p; }
        if (p < e && (*p == 'e' || *p == 'E')) {
            ++p; if (p < e && (*p == '+' || *p == '-')) ++p;
            if (p >= e || *p < '0' || *p > '9') return false;
            while (p < e && *p >= '0' && *p <= '9') ++p;
        }
        std::string tmp(s, p - s);
        d = strtod(tmp.c_str(), nullptr);
        return true;
    }
    bool value(JVal& v, int depth = 0) {
        if (depth > 200) return false;
        ws();
        if (p >= e) return false;
        char c = *p;
        if (c == '{') {
            ++p; v.t = JVal::OBJ; v.obj.reset(new JObj());
            ws();
            if (p < e && *p == '}') { ++p; return true; }
            for (;;) {
                ws(); std::string k;
                if (!string(k)) return false;
                ws(); if (p >= e || *p != ':') return false; ++p;
                JVal child; if (!value(child, depth + 1)) return false;
                bool dup = false;
                for (auto& kv : *v.obj) if (kv.first == k) { kv.second = std::move(child); dup = true; break; }
                if (!dup) v.obj->emplace_back(std::move(k), std::move(child));
                ws(); if (p >= e) return false;
                if (*p == ',') { ++p; continue; }
                if (*p == '}') { ++p; return true; }
                return false;
            }
        }
        if (c == '[') {
            ++p; v.t = JVal::ARR; v.arr.reset(new std::vector<JVal>());
            ws();
            if (p < e && *p == ']') { ++p; return true; }
            for (;;) {
                JVal child; if (!value(child, depth + 1)) return false;
                v.arr->push_back(std::move(child));
                ws(); if (p >= e) return false;
                if (*p == ',') { ++p; continue; }
                if (*p == ']') { ++p; return true; }
                return false;
            }
        }
        if (c == '"') { v.t = JVal::STR; return string(v.str); }
        if (c == 't') { v.t = JVal::BOOL; v.b = true; return lit("true"); }
        if (c == 'f') { v.t = JVal::BOOL; v.b = false; return lit("false"); }
        if (c == 'n') { v.t = JVal::NUL; return lit("null"); }
        v.t = JVal::NUM; return number(v.num);
    }
    bool document(JVal& v) { if (!value(v)) return false; ws(); return p == e; }
};

// ---------------------------------------------------------------------------------------
// lib/zk.js restated
// ---------------------------------------------------------------------------------------
std::string ascii_lower(const std::string& s) {
    std::string o = s;
    for (auto& c : o) if (c >= 'A' && c <= 'Z') c = (char)(c + 32);
    return o;
}

struct TreeNode {
    std::string tn_name;            // child label, original case   (lib/zk.js:79)
    std::string tn_domain;          // lower-cased fqdn             (lib/zk.js:84)
    std::vector<int> tn_kids;       // insertion order              (lib/zk.js:108-114)
    JVal tn_data;                   // NUL = null                   (lib/zk.js:88,155)
    bool has_ip = false; std::string tn_ip;
    TreeNode() { tn_data.t = JVal::NUL; }
};

const char* const kHostLike[] = { "db_host", "host", "load_balancer", "moray_host", "redis_host",
                                  "ops_host", "rr_host" };
const char* const kServiceKid[] = { "load_balancer", "moray_host", "ops_host", "rr_host", "redis_host" };
bool in_list(const std::string& s, const char* const* l, int n) {
    for (int i = 0; i < n; i++) if (s == l[i]) return true;
    return false;
}

struct ZKCache {
    std::string ca_domain;
    std::vector<std::unique_ptr<TreeNode>> nodes;
    std::unordered_map<std::string, int> ca_treeNodes;   // lower-cased fqdn -> node
    std::unordered_map<std::string, int> ca_revLookup;   // address string -> node
    std::unordered_map<std::string, int> by_path;
    bool loaded = false;

    int new_node(const std::string& pdomain, const std::string& name) {   // lib/zk.js:78-97
        std::unique_ptr<TreeNode> n(new TreeNode());
        n->tn_name = name;
        std::string d = name;
        if (!pdomain.empty()) d += "." + pdomain;
        n->tn_domain = ascii_lower(d);
        int id = (int)nodes.size();
        ca_treeNodes[n->tn_domain] = id;
        nodes.push_back(std::move(n));
        return id;
    }
    void on_data_changed(int id, JVal&& parsed) {                         // lib/zk.js:139-194
        TreeNode& n = *nodes[id];
        if (!(parsed.t == JVal::NUL || parsed.is_object())) return;       // :149-154
        n.tn_data = std::move(parsed);
        const JVal& d = n.tn_data;
        const JVal& type = d.get("type");
        if (d.t == JVal::NUL || type.t != JVal::STR) return;              // :157-165
        if (!in_list(type.str, kHostLike, 7)) return;
        const JVal& rec = d.get(type.str);
        if (!rec.is_object()) return;                                     // :181-182
        const JVal& addr = rec.get("address");
        if (n.has_ip) { auto it = ca_revLookup.find(n.tn_ip); if (it != ca_revLookup.end()) ca_revLookup.erase(it); }
        n.has_ip = false;
        if (addr.t == JVal::STR && !addr.str.empty()) {                   // contract: strings only
            n.has_ip = true; n.tn_ip = addr.str;
            ca_revLookup[addr.str] = id;
        }
    }
    static std::string domain_to_path(const std::string& domain) {       // lib/zk.js:225-228
        std::vector<std::string> parts; size_t s = 0;
        for (;;) { size_t d = domain.find('.', s); parts.push_back(domain.substr(s, d == std::string::npos ? d : d - s)); if (d == std::string::npos) break; s = d + 1; }
        std::string o;
        for (size_t i = parts.size(); i-- > 0;) { o += "/"; o += parts[i]; }
        return o;
    }
    // lib/zk.js:195-208: the node and its subtree leave ca_treeNodes (each only if the key is still its
    // own); ca_revLookup is never touched.
    void unbind(int id) {
        TreeNode& n = *nodes[id];
        for (int k : n.tn_kids) unbind(k);
        auto it = ca_treeNodes.find(n.tn_domain);
        if (it != ca_treeNodes.end() && it->second == id) ca_treeNodes.erase(it);
    }
    void forget_paths(int id, const std::string& path) {
        for (int k : nodes[id]->tn_kids) forget_paths(k, path + "/" + nodes[k]->tn_name);
        by_path.erase(path);
    }
    // Snapshot = JSON lines {"path":..., "data":<value>} | {"path":..., "raw":"<znode bytes>"}.
    int load(const char* buf, size_t len) {
        size_t dot = ca_domain.find('.');
        std::string first = ca_domain.substr(0, dot);
        std::string rest = dot == std::string::npos ? "" : ca_domain.substr(dot + 1);
        int root = new_node(rest, first);                                 // lib/zk.js:68-76
        by_path[domain_to_path(ca_domain)] = root;
        if (apply(buf, len, false) != 0) return -1;
        loaded = true;
        return 0;
    }
    // The same lines as watch events on a live cache: a known path = dataChanged (:139-194), a new
    // path = a child appended by childrenChanged (:120-130) followed by its data, and
    // {"path":..., "deleted":true} = the child vanishing from its parent's list (:131-133).
    int apply(const char* buf, size_t len, bool allow_delete) {
        std::string root_path = domain_to_path(ca_domain);
        int root = by_path[root_path];
        const char* p = buf; const char* end = buf + len;
        while (p < end) {
            const char* nl = (const char*)memchr(p, '\n', end - p);
            const char* le = nl ? nl : end;
            const char* a = p; const char* b = le;
            while (a < b && (*a == ' ' || *a == '\t' || *a == '\r')) ++a;
            while (b > a && (b[-1] == ' ' || b[-1] == '\t' || b[-1] == '\r')) --b;
            p = nl ? nl + 1 : end;
            if (a == b) continue;
            JVal ent; JParser jp(a, b);
            if (!jp.document(ent) || ent.t != JVal::OBJ) return -1;
            const JVal& path = ent.get("path");
            if (path.t != JVal::STR) return -1;
            const JVal& dv = ent.get("deleted");
            const bool deleting = dv.t == JVal::BOOL && dv.b;
            if (deleting && !allow_delete) return -1;
            int id;
            if (path.str == root_path) { if (deleting) return -1; id = root; }
            else {
                size_t sl = path.str.rfind('/');
                if (sl == std::string::npos) continue;
                std::string ppath = path.str.substr(0, sl), name = path.str.substr(sl + 1);
                auto it = by_path.find(ppath);
                if (it == by_path.end() || name.empty()) continue;         // not under the watched root
                int parent = it->second;
                auto self = by_path.find(path.str);
                if (deleting) {
                    if (self == by_path.end()) continue;
                    id = self->second;
                    unbind(id);
                    forget_paths(id, path.str);
                    auto& kids = nodes[parent]->tn_kids;
                    kids.erase(std::find(kids.begin(), kids.end(), id));
                    continue;
                }
                if (self != by_path.end()) id = self->second;
                else {
                    std::string pdom = nodes[parent]->tn_domain;
                    id = new_node(pdom, name);
                    nodes[parent]->tn_kids.push_back(id);
                    by_path[path.str] = id;
                }
            }
            JVal* data = nullptr;
            for (auto& kv : *ent.obj) if (kv.first == "data") data = &kv.second;
            const JVal& raw = ent.get("raw");
            if (raw.t == JVal::STR) {
                JVal parsed; JParser rp(raw.str.data(), raw.str.data() + raw.str.size());
                if (rp.document(parsed)) on_data_changed(id, std::move(parsed));   // :141-148 parse error: ignore
            } else if (data) {
                on_data_changed(id, std::move(*data));
            }
        }
        return 0;
    }
    bool isReady() const { return loaded && ca_treeNodes.count(ca_domain) != 0; }   // lib/zk.js:55-58
    const TreeNode* lookup(const std::string& d) const {                             // lib/zk.js:62-64
        auto it = ca_treeNodes.find(d); return it == ca_treeNodes.end() ? nullptr : nodes[it->second].get();
    }
    const TreeNode* reverseLookup(const std::string& ip) const {                      // lib/zk.js:65-67
        auto it = ca_revLookup.find(ip); return it == ca_revLookup.end() ? nullptr : nodes[it->second].get();
    }
};

// ---------------------------------------------------------------------------------------
// contract helpers (values mname's record constructors would reject; DESIGN.md "Contract")
// ---------------------------------------------------------------------------------------
bool valid_uint(const JVal& v, double limit, uint32_t& out) {
    if (v.t != JVal::NUM) return false;
    double d = v.num;
    if (!(d >= 0) || !(d < limit) || d != std::floor(d)) return false;
    out = (uint32_t)d; return true;
}
bool valid_ipv4(const JVal& v, uint8_t out[4]) {
    if (v.t != JVal::STR) return false;
    const std::string& s = v.str; size_t i = 0;
    for (int o = 0; o < 4; o++) {
        size_t st = i; unsigned val = 0;
        while (i < s.size() && s[i] >= '0' && s[i] <= '9' && i - st < 4) { val = val * 10 + (s[i] - '0'); ++i; }
        size_t nd = i - st;
        if (nd < 1 || nd > 3 || val > 255 || (nd > 1 && s[st] == '0')) return false;
        out[o] = (uint8_t)val;
        if (o < 3) { if (i >= s.size() || s[i] != '.') return false; ++i; }
    }
    return i == s.size();
}
// url.parse(x).hostname for scheme://[user[:pw]@]host[:port][/...]   (lib/server.js:297-298)
bool url_hostname(const JVal& v, JVal& host) {
    if (v.t != JVal::STR) return false;
    const std::string& s = v.str; size_t i = 0;
    if (s.empty() || !isalpha((unsigned char)s[0])) return false;
    while (i < s.size() && (isalnum((unsigned char)s[i]) || s[i] == '+' || s[i] == '.' || s[i] == '-')) ++i;
    if (s.compare(i, 3, "://") != 0) return false;
    i += 3;
    size_t e = s.find_first_of("/?#", i);
    std::string auth = s.substr(i, e == std::string::npos ? e : e - i);
    size_t at = auth.rfind('@');
    if (at != std::string::npos) auth = auth.substr(at + 1);
    size_t colon = auth.rfind(':');
    if (colon != std::string::npos) auth = auth.substr(0, colon);
    host.t = JVal::STR; host.str = ascii_lower(auth);
    return true;
}
// a dotted name every label of which fits the wire format
bool encodable(const std::string& name) {
    if (name.empty()) return true;
    size_t s = 0, wire = 1;
    for (;;) {
        size_t d = name.find('.', s);
        size_t l = (d == std::string::npos ? name.size() : d) - s;
        if (l < 1 || l > 63) return false;
        wire += 1 + l;
        if (d == std::string::npos) break;
        s = d + 1;
    }
    return wire <= 255;
}

// ---------------------------------------------------------------------------------------
// mname codec restated (DESIGN.md "Wire spec")
// ---------------------------------------------------------------------------------------
enum { ST_ANSWERED = 0, ST_MISS_RECURSE = 1, ST_DROPPED = 2 };
enum { RC_NOERROR = 0, RC_SERVFAIL = 2, RC_NXDOMAIN = 3, RC_NOTIMP = 4, RC_REFUSED = 5 };
enum { T_A = 1, T_SOA = 6, T_PTR = 12, T_SRV = 33, T_OPT = 41 };

struct Query {
    const uint8_t* pkt; uint32_t len;
    uint16_t id; uint8_t opcode; bool rd;
    uint32_t qname_len;                 // wire bytes incl. terminating 0
    std::vector<std::pair<uint32_t, uint32_t>> labels;   // (offset in packet, length)
    uint16_t qtype, qclass;
    uint32_t q_end;                     // end of question section
    bool edns; uint16_t adv;
    bool tcp = false;                   // arrived over TCP: no UDP size limit (RFC 1035 4.2.2)
    bool label_dot;
    std::string name;                   // query.name(): labels joined by '.', latin-1 bytes
};

bool decode(const uint8_t* p, uint32_t len, Query& q) {
    // a DNS message is at most 65,535 bytes (RFC 1035 4.2.2 framing; the engine's u16 response length): anything longer is not a query
    if (len < 12 || len > 65535) return false;
    q.pkt = p; q.len = len;
    q.id = (uint16_t)(p[0] << 8 | p[1]);
    if (p[2] & 0x80) return false;                        // QR=1: not a query
    q.opcode = (p[2] >> 3) & 0xF; q.rd = p[2] & 1;
    unsigned qd = p[4] << 8 | p[5], an = p[6] << 8 | p[7], ns = p[8] << 8 | p[9], ar = p[10] << 8 | p[11];
    if (qd != 1 || an != 0 || ns != 0 || ar > 1) return false;
    uint32_t pos = 12; q.label_dot = false; q.name.clear(); q.labels.clear();
    for (;;) {
        if (pos >= len) return false;
        unsigned c = p[pos];
        if (c == 0) { ++pos; break; }
        if (c > 63) return false;                          // pointers / extended labels
        if (pos + 1 + c > len) return false;
        q.labels.emplace_back(pos + 1, c);
        if (!q.name.empty() || q.labels.size() > 1) q.name += '.';
        for (unsigned i = 0; i < c; i++) { char ch = (char)p[pos + 1 + i]; if (ch == '.') q.label_dot = true; q.name += ch; }
        pos += 1 + c;
        if (pos - 12 + 1 > 255) return false;
    }
    q.qname_len = pos - 12;
    if (pos + 4 > len) return false;
    q.qtype = (uint16_t)(p[pos] << 8 | p[pos + 1]); q.qclass = (uint16_t)(p[pos + 2] << 8 | p[pos + 3]);
    pos += 4; q.q_end = pos;
    if (q.qclass != 1) return false;
    q.edns = false; q.adv = 0;
    if (ar == 1) {
        if (pos + 11 > len) return false;
        if (p[pos] != 0) return false;
        if ((p[pos + 1] << 8 | p[pos + 2]) != T_OPT) return false;
        q.adv = (uint16_t)(p[pos + 3] << 8 | p[pos + 4]);
        unsigned rdlen = p[pos + 9] << 8 | p[pos + 10];
        if (pos + 11 + rdlen > len) return false;
        q.edns = true;
    }
    return true;
}

struct RR {
    int section;                // 0 answer, 1 authority, 2 additional
    std::string owner; uint16_t type; uint32_t ttl;
    std::vector<uint8_t> rdata;
};

void put16(std::vector<uint8_t>& o, unsigned v) { o.push_back((uint8_t)(v >> 8)); o.push_back((uint8_t)v); }
void put32(std::vector<uint8_t>& o, uint32_t v) { put16(o, v >> 16); put16(o, v & 0xFFFF); }
void put_name_plain(std::vector<uint8_t>& o, const std::string& n) {
    size_t s = 0;
    if (!n.empty()) for (;;) {
        size_t d = n.find('.', s);
        size_t l = (d == std::string::npos ? n.size() : d) - s;
        o.push_back((uint8_t)l);
        o.insert(o.end(), n.begin() + s, n.begin() + s + l);
        if (d == std::string::npos) break;
        s = d + 1;
    }
    o.push_back(0);
}

struct Responder {
    const Query& q; int rcode = -1; int status = ST_ANSWERED;
    std::vector<RR> rrs; size_t n_answers = 0;
    uint32_t dom_label0 = 0;    // index of the first QNAME label of the "domain part"
    explicit Responder(const Query& qq) : q(qq) {}
    void setError(int rc) { rcode = rc; }
    void add(int section, const std::string& owner, uint16_t type, uint32_t ttl, std::vector<uint8_t>&& rd) {
        RR r; r.section = section; r.owner = owner; r.type = type; r.ttl = ttl; r.rdata = std::move(rd);
        rrs.push_back(std::move(r));
        if (section == 0) ++n_answers;
    }
    // owner-name compression: pointer 0xC00C when byte-identical to the QNAME, else longest
    // label-aligned suffix shared with the QNAME's domain part (labels >= dom_label0)
    void put_owner(std::vector<uint8_t>& o, const std::string& n) const {
        if (n == q.name && !q.labels.empty()) { put16(o, 0xC00C); return; }
        size_t s = 0;
        for (;;) {
            // does n[s:] equal the QNAME suffix that starts at some label k >= dom_label0?
            size_t off = 0;
            for (size_t k = 0; k < q.labels.size(); k++) {
                if (k >= dom_label0 && q.name.size() - off == n.size() - s &&
                    q.name.compare(off, std::string::npos, n, s, std::string::npos) == 0) {
                    put16(o, 0xC000 | (q.labels[k].first - 1));
                    return;
                }
                off += q.labels[k].second + 1;
            }
            size_t d = n.find('.', s);
            size_t l = (d == std::string::npos ? n.size() : d) - s;
            o.push_back((uint8_t)l);
            o.insert(o.end(), n.begin() + s, n.begin() + s + l);
            if (d == std::string::npos) break;
            s = d + 1;
        }
        o.push_back(0);
    }
    size_t encode(uint8_t* out, size_t cap) const {
        int rc = rcode >= 0 ? rcode : (n_answers ? RC_NOERROR : RC_NOTIMP);
        size_t maxsz = 512;
        if (q.edns) maxsz = std::min<size_t>(std::max<size_t>(q.adv, 512), 1200);
        if (q.tcp) maxsz = 65535;
        std::vector<uint8_t> fixed(12, 0);
        fixed.insert(fixed.end(), q.pkt + 12, q.pkt + q.q_end);         // question echoed verbatim
        std::vector<uint8_t> opt;
        if (q.edns) { opt = { 0, 0, T_OPT, 0x04, 0xB0, 0, 0, 0, 0, 0, 0 }; }
        std::vector<std::vector<uint8_t>> enc(rrs.size());
        for (size_t i = 0; i < rrs.size(); i++) {
            auto& o = enc[i]; const RR& r = rrs[i];
            put_owner(o, r.owner); put16(o, r.type); put16(o, 1); put32(o, r.ttl);
            put16(o, (unsigned)r.rdata.size()); o.insert(o.end(), r.rdata.begin(), r.rdata.end());
        }
        // emission order: answers, authority, [OPT,] additional.  Keep the longest prefix of
        // the RR sequence that fits (OPT always kept); TC if anything was dropped.
        std::vector<size_t> order;
        for (int sec = 0; sec < 3; sec++) for (size_t i = 0; i < rrs.size(); i++) if (rrs[i].section == sec) order.push_back(i);
        size_t total = fixed.size() + opt.size(), keep = 0;
        for (; keep < order.size(); keep++) { if (total + enc[order[keep]].size() > maxsz) break; total += enc[order[keep]].size(); }
        bool tc = keep < order.size();
        unsigned cnt[3] = { 0, 0, 0 };
        for (size_t i = 0; i < keep; i++) cnt[rrs[order[i]].section]++;
        if (q.edns) cnt[2]++;
        fixed[0] = (uint8_t)(q.id >> 8); fixed[1] = (uint8_t)q.id;
        fixed[2] = (uint8_t)(0x80 | (q.opcode << 3) | 0x04 | (tc ? 0x02 : 0) | (q.rd ? 1 : 0));
        fixed[3] = (uint8_t)rc;
        fixed[4] = 0; fixed[5] = 1;
        fixed[6] = (uint8_t)(cnt[0] >> 8); fixed[7] = (uint8_t)cnt[0];
        fixed[8] = (uint8_t)(cnt[1] >> 8); fixed[9] = (uint8_t)cnt[1];
        fixed[10] = (uint8_t)(cnt[2] >> 8); fixed[11] = (uint8_t)cnt[2];
        if (total > cap) return (size_t)-1;
        size_t w = 0;
        memcpy(out + w, fixed.data(), fixed.size()); w += fixed.size();
        bool opt_done = !q.edns;
        for (size_t i = 0; i < keep; i++) {
            const RR& r = rrs[order[i]];
            if (r.section == 2 && !opt_done) { memcpy(out + w, opt.data(), opt.size()); w += opt.size(); opt_done = true; }
            memcpy(out + w, enc[order[i]].data(), enc[order[i]].size()); w += enc[order[i]].size();
        }
        if (!opt_done) { memcpy(out + w, opt.data(), opt.size()); w += opt.size(); }
        return w;
    }
};

// ---------------------------------------------------------------------------------------
// lib/server.js restated
// ---------------------------------------------------------------------------------------
// Recursion.resolve()'s quick rejects (lib/recursion.js:329-344,377-379) as a pre-filter on misses: would
// the miss be forwarded anywhere?  dcs = the keys of self.dcs that keep an upstream after the own-address
// filter (:360-379); ptr = any such upstream exists (PTR asks every datacenter, :346-354).
struct RecursionFilter {
    bool enabled = false, ptr = false;
    std::string dnsDomain;
    std::vector<std::string> dcs;
    bool forwards(const std::string& domain, bool is_ptr) const {
        if (is_ptr) return ptr;
        long from = (long)domain.size() - (long)dnsDomain.size();             // indexOf clamps a negative start to 0
        if (domain.find(dnsDomain, (size_t)(from < 0 ? 0 : from)) == std::string::npos) return false;   // :330-333
        long end = (long)domain.size() - (long)dnsDomain.size() - 1;           // substring clamps it too
        std::string p = domain.substr(0, (size_t)(end < 0 ? 0 : end));         // :338-339
        size_t dot = p.rfind('.');
        std::string dc = p.substr(dot == std::string::npos ? 0 : dot + 1);     // :340
        return std::find(dcs.begin(), dcs.end(), dc) != dcs.end();             // :341-343
    }
};
struct Options {
    ZKCache* zkCache = nullptr;
    std::string dnsDomain, datacenterName;
    bool recursion = false;
    RecursionFilter rf;
};

uint32_t fmix32(uint32_t x) { x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16; return x; }
// replacement for Math.random() at lib/server.js:46 -> j = floor(u * (i + 1))
uint32_t shuffle_rand(uint64_t seed, uint32_t qidx, uint32_t i) {
    uint32_t lo = (uint32_t)seed, hi = (uint32_t)(seed >> 32);
    uint32_t r = fmix32(fmix32(fmix32(lo) ^ hi ^ (qidx * 0x9E3779B1u)) + i * 0x85EBCA77u);
    return (uint32_t)(((uint64_t)r * (i + 1)) >> 32);
}
template <class T> void shuffle(std::vector<T>& arr, uint64_t seed, uint32_t qidx) {   // lib/server.js:40-53
    if (arr.empty()) return;
    size_t i = arr.size();
    while (--i > 0) { uint32_t j = shuffle_rand(seed, qidx, (uint32_t)i); std::swap(arr[i], arr[j]); }
}
bool isSuffix(const std::string& suffix, const std::string& str) {                      // lib/server.js:55-58
    size_t idx = str.rfind(suffix);
    return idx != std::string::npos && idx + suffix.size() == str.size();
}
// ttl = 30; record.ttl; record[record.type].ttl   (lib/server.js:270-274, 124-128)
bool record_ttl(const JVal& record, uint32_t& ttl) {
    JVal def; def.t = JVal::NUM; def.num = 30;
    const JVal* t = &def;
    const JVal& a = record.get("ttl");
    if (a.t != JVal::UNDEF) t = &a;
    const JVal& type = record.get("type");
    if (type.t == JVal::STR) { const JVal& b = record.get(type.str).get("ttl"); if (b.t != JVal::UNDEF) t = &b; }
    return valid_uint(*t, 2147483648.0, ttl);
}
std::vector<uint8_t> rdata_a(const uint8_t ip[4]) { return std::vector<uint8_t>(ip, ip + 4); }

void resolvePtr(const Options& o, const Query& q, Responder& r) {                       // lib/server.js:67-134
    const std::string& domain = q.name;
    std::vector<std::string> parts; size_t s = 0;
    for (;;) { size_t d = domain.find('.', s); parts.push_back(domain.substr(s, d == std::string::npos ? d : d - s)); if (d == std::string::npos) break; s = d + 1; }
    std::reverse(parts.begin(), parts.end());
    if (parts.size() < 2 || parts[0] != "arpa" || parts[1] != "in-addr") { r.setError(RC_REFUSED); return; }
    std::string ip;
    for (size_t i = 2; i < parts.size(); i++) { if (i > 2) ip += '.'; ip += parts[i]; }
    if (!o.zkCache || !o.zkCache->isReady()) { r.setError(RC_SERVFAIL); return; }
    const TreeNode* node = o.zkCache->reverseLookup(ip);
    if (!node) {
        if (o.recursion && q.rd) {
            if (o.rf.enabled && !o.rf.forwards(q.name, true)) { r.setError(RC_REFUSED); return; }   // recursion.js would refuse
            r.status = ST_MISS_RECURSE; return;
        }
        r.setError(RC_REFUSED); return;
    }
    uint32_t ttl;
    if (!record_ttl(node->tn_data, ttl) || !encodable(node->tn_domain)) { r.setError(RC_SERVFAIL); return; }   // contract
    std::vector<uint8_t> rd; put_name_plain(rd, node->tn_domain);
    r.add(0, domain, T_PTR, ttl, std::move(rd));
}

void resolve(const Options& o, const Query& q, Responder& r, uint64_t seed, uint32_t qidx) {   // lib/server.js:136-429
    std::string domain = q.name;
    bool have_srv = false; std::string service, protocol;
    // /^(_[^_.]*)[.](_[^_.]*)[.](.*)/  — '.' stops at \n and \r, no '$'
    bool m = false; size_t g1e = 0, g2s = 0, g2e = 0, g3s = 0, g3e = 0;
    {
        const std::string& d = q.name; size_t i = 0;
        if (i < d.size() && d[i] == '_') {
            ++i; while (i < d.size() && d[i] != '_' && d[i] != '.') ++i;
            g1e = i;
            if (i < d.size() && d[i] == '.') {
                ++i; g2s = i;
                if (i < d.size() && d[i] == '_') {
                    ++i; while (i < d.size() && d[i] != '_' && d[i] != '.') ++i;
                    g2e = i;
                    if (i < d.size() && d[i] == '.') {
                        ++i; g3s = i; while (i < d.size() && d[i] != '\n' && d[i] != '\r') ++i;
                        g3e = i; m = true;
                    }
                }
            }
        }
    }
    if (q.qtype == T_SRV) {
        if (!m || g3e - g3s < 1) { r.setError(RC_REFUSED); return; }
        service = q.name.substr(0, g1e); protocol = q.name.substr(g2s, g2e - g2s);
        domain = q.name.substr(g3s, g3e - g3s); have_srv = true;
        r.dom_label0 = 2;
    }
    if (!o.dnsDomain.empty()) {
        if (!isSuffix("." + o.dnsDomain, domain)) { r.setError(RC_REFUSED); return; }
        // lib/server.js:167-175 is dead code (stripSuffix appends '...'): no refusal here.
    }
    if (!o.zkCache || !o.zkCache->isReady()) { r.setError(RC_SERVFAIL); return; }
    if (domain.size() < 1) { r.setError(RC_REFUSED); return; }
    domain = ascii_lower(domain);
    for (unsigned char c : domain)
        if (!((c >= 'a' && c <= 'z') || (c >= '0' && c <= '9') || c == '_' || c == '.' || c == '-')) { r.setError(RC_REFUSED); return; }
    const TreeNode* node = o.zkCache->lookup(domain);
    if (!node) {
        if (o.recursion && q.rd) {
            if (o.rf.enabled && !o.rf.forwards(q.name, false)) { r.setError(RC_REFUSED); return; }  // recursion.js would refuse
            r.status = ST_MISS_RECURSE; return;
        }
        r.setError(RC_REFUSED); return;
    }
    const JVal& record = node->tn_data;
    const JVal& rtype = record.get("type");
    if (record.t == JVal::NUL || rtype.t != JVal::STR || !record.get(rtype.str).is_object()) { r.setError(RC_SERVFAIL); return; }
    uint32_t ttl;
    if (!record_ttl(record, ttl)) { r.setError(RC_SERVFAIL); return; }                 // contract
    if (have_srv && rtype.str != "service") {
        r.setError(RC_NOERROR);
        std::vector<uint8_t> rd;
        put_name_plain(rd, o.dnsDomain);
        put_name_plain(rd, o.dnsDomain.empty() ? std::string("hostmaster") : "hostmaster." + o.dnsDomain);
        put32(rd, 0); put32(rd, 10); put32(rd, 10); put32(rd, 10); put32(rd, ttl);
        r.add(1, domain, T_SOA, ttl, std::move(rd));
        return;
    }
    uint8_t ip[4];
    if (rtype.str == "database") {
        JVal host;
        if (!url_hostname(record.get("database").get("primary"), host) || !valid_ipv4(host, ip)) { r.setError(RC_SERVFAIL); return; }
        r.add(0, domain, T_A, ttl, rdata_a(ip));
    } else if (in_list(rtype.str, kHostLike, 7)) {
        if (!valid_ipv4(record.get(rtype.str).get("address"), ip)) { r.setError(RC_SERVFAIL); return; }
        r.add(0, domain, T_A, ttl, rdata_a(ip));
    } else if (rtype.str == "service") {
        const JVal* s = &record.get("service");
        const JVal& inner = s->get("service");
        if (inner.t == JVal::NUL) { r.setError(RC_SERVFAIL); return; }                  // contract
        if (inner.is_object()) s = &inner;
        const JVal& sttl = s->get("ttl");
        if (sttl.t != JVal::UNDEF) { if (!valid_uint(sttl, 2147483648.0, ttl)) { r.setError(RC_SERVFAIL); return; } }
        if (have_srv) {
            const JVal& sv = s->get("srvce"); const JVal& pr = s->get("proto");
            if (sv.t != JVal::STR || sv.str != service || pr.t != JVal::STR || pr.str != protocol) { r.setError(RC_NXDOMAIN); return; }
        }
        r.setError(RC_NOERROR);
        std::vector<const TreeNode*> kids;
        for (int k : node->tn_kids) {
            const TreeNode* sub = o.zkCache->nodes[k].get();
            const JVal& kt = sub->tn_data.get("type");
            if (sub->tn_data.is_object() && kt.t == JVal::STR && in_list(kt.str, kServiceKid, 5)) kids.push_back(sub);
        }
        shuffle(kids, seed, qidx);
        for (const TreeNode* knode : kids) {
            const JVal& krec = knode->tn_data;
            const JVal& ksub = krec.get(krec.get("type").str);
            if (!ksub.is_object()) { r.setError(RC_SERVFAIL); break; }                  // :366-376
            const JVal& a = ksub.get("address");
            if (a.t == JVal::NUL) continue;                                             // :378-381
            const JVal* ports = &ksub.get("ports");
            bool use_sport = ports->t == JVal::UNDEF || (ports->t == JVal::ARR && ports->arr->size() < 1);
            uint32_t rttl = ttl; bool bad = false;
            const JVal* rt = nullptr;
            if (krec.get("ttl").t != JVal::UNDEF) rt = &krec.get("ttl");
            if (ksub.get("ttl").t != JVal::UNDEF) rt = &ksub.get("ttl");
            if (rt && !valid_uint(*rt, 2147483648.0, rttl)) bad = true;
            if (!valid_ipv4(a, ip)) bad = true;
            std::vector<uint32_t> plist;
            std::string nm = knode->tn_name + "." + domain;
            if (have_srv) {
                uint32_t pv;
                if (use_sport) { if (valid_uint(s->get("port"), 65536.0, pv)) plist.push_back(pv); else bad = true; }
                else if (ports->t != JVal::ARR) bad = true;
                else for (auto& pj : *ports->arr) { if (valid_uint(pj, 65536.0, pv)) plist.push_back(pv); else bad = true; }
                if (!encodable(nm)) bad = true;
            }
            if (bad) { r.setError(RC_SERVFAIL); break; }                                // contract -> "bad zk info"
            if (have_srv) {
                for (uint32_t pv : plist) {
                    std::vector<uint8_t> rd; put16(rd, 0); put16(rd, 10); put16(rd, pv); put_name_plain(rd, nm);
                    r.add(0, q.name, T_SRV, ttl, std::move(rd));
                }
                r.add(2, nm, T_A, rttl, rdata_a(ip));
            } else {
                if (ttl < rttl) rttl = ttl;
                r.add(0, domain, T_A, rttl, rdata_a(ip));
            }
        }
    }
    // else: unknown record.type — nothing added, nothing set (lib/server.js:419-424)
}

void onQuery(const Options& o, const Query& q, Responder& r, uint64_t seed, uint32_t qidx) {   // lib/server.js:471-507
    bool handled = q.opcode == 0 && (q.qtype == T_A || q.qtype == T_SRV || q.qtype == T_PTR);
    if (!handled) { r.setError(RC_NOTIMP); return; }
    if (q.label_dot) { r.setError(RC_REFUSED); return; }          // DESIGN.md "in-label dots"
    if (q.qtype == T_PTR) resolvePtr(o, q, r);
    else resolve(o, q, r, seed, qidx);
}

struct Engine { Options opt; std::unique_ptr<ZKCache> zk; };

}  // namespace

extern "C" {

void* orc_create(const char* dns_domain, const char* datacenter_name, int recursion) {
    Engine* e = new Engine();
    e->opt.dnsDomain = dns_domain ? dns_domain : "";
    e->opt.datacenterName = datacenter_name ? datacenter_name : "";
    e->opt.recursion = recursion != 0;
    return e;
}
void orc_destroy(void* h) { delete (Engine*)h; }

// (Re)build the cache from a snapshot; the cache's root is `dns_domain`.
int orc_load_snapshot(void* h, const char* buf, size_t len) {
    Engine* e = (Engine*)h;
    std::unique_ptr<ZKCache> zk(new ZKCache());
    zk->ca_domain = e->opt.dnsDomain;
    if (zk->load(buf, len) != 0) return -1;
    e->zk = std::move(zk);
    e->opt.zkCache = e->zk.get();
    return 0;
}
// Recursion pre-filter (see RecursionFilter); region_domain NULL removes it.
int orc_set_recursion_filter(void* h, const char* region_domain, const char* const* dcs, uint32_t n, int ptr) {
    Engine* e = (Engine*)h;
    e->opt.rf = RecursionFilter();
    if (!region_domain) return 0;
    e->opt.rf.enabled = true; e->opt.rf.ptr = ptr != 0; e->opt.rf.dnsDomain = region_domain;
    for (uint32_t i = 0; i < n; i++) e->opt.rf.dcs.push_back(dcs[i]);
    return 0;
}
// Watch events on the loaded cache (see ZKCache::apply).
int orc_apply_delta(void* h, const char* buf, size_t len) {
    Engine* e = (Engine*)h;
    if (!e->zk) return -1;
    return e->zk->apply(buf, len, true);
}
long orc_node_count(void* h) { Engine* e = (Engine*)h; return e->zk ? (long)e->zk->nodes.size() : 0; }

// Same batch container as bb_resolve_batch (include/binder_b200.h).  nthreads<=1: scalar.
// flags: 1 = the batch arrived over TCP
int orc_resolve_batch_ex(void* h, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n, uint64_t seed,
                         uint32_t qidx_base, uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint8_t* status,
                         uint32_t* miss_idx, uint32_t* n_miss, int nthreads, uint32_t flags) {
    Engine* e = (Engine*)h;
    const bool tcp = (flags & 1u) != 0;
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > n) nthreads = n ? (int)n : 1;
    struct Part { std::vector<uint8_t> bytes; std::vector<uint32_t> lens; };
    std::vector<Part> parts(nthreads);
    auto work = [&](int t) {
        uint32_t lo = (uint32_t)((uint64_t)n * t / nthreads), hi = (uint32_t)((uint64_t)n * (t + 1) / nthreads);
        Part& P = parts[t]; P.lens.resize(hi - lo);
        std::vector<uint8_t> tmpv(tcp ? 65536 : 1300);
        uint8_t* const tmp = tmpv.data();
        for (uint32_t i = lo; i < hi; i++) {
            Query q; size_t w = 0;
            if (!decode(pkts + pkt_off[i], pkt_off[i + 1] - pkt_off[i], q)) status[i] = ST_DROPPED;
            else {
                q.tcp = tcp;
                Responder r(q);
                onQuery(e->opt, q, r, seed, qidx_base + i);
                status[i] = (uint8_t)r.status;
                if (r.status == ST_ANSWERED) w = r.encode(tmp, tmpv.size());
            }
            P.lens[i - lo] = (uint32_t)w;
            P.bytes.insert(P.bytes.end(), tmp, tmp + w);
        }
    };
    if (nthreads == 1) work(0);
    else { std::vector<std::thread> th; for (int t = 0; t < nthreads; t++) th.emplace_back(work, t); for (auto& x : th) x.join(); }
    uint64_t pos = 0; uint32_t i = 0, nm = 0;
    for (int t = 0; t < nthreads; t++) {
        Part& P = parts[t];
        if (pos + P.bytes.size() > out_cap) return -2;
        memcpy(out + pos, P.bytes.data(), P.bytes.size());
        for (uint32_t l : P.lens) { out_off[i] = (uint32_t)pos; pos += l; if (status[i] == ST_MISS_RECURSE) miss_idx[nm++] = i; ++i; }
    }
    out_off[n] = (uint32_t)pos;
    *n_miss = nm;
    return 0;
}
int orc_resolve_batch(void* h, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n, uint64_t seed,
                      uint32_t qidx_base, uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint8_t* status,
                      uint32_t* miss_idx, uint32_t* n_miss, int nthreads) {
    return orc_resolve_batch_ex(h, pkts, pkt_off, n, seed, qidx_base, out, out_cap, out_off, status, miss_idx, n_miss, nthreads, 0);
}

}  // extern "C"
