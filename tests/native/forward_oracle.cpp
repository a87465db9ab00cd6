// TEST INFRASTRUCTURE — CPU oracle of the recursion forward and match (DESIGN.md section 14).  NOT the product.
//
// Restates what recursion.py's _exchange does for a batch of misses (lib/recursion.js:253-280,335-354,382-387) with the
// GPU path's ID scheme and grouping: the route of each miss from its dotted name (the string operations of Recursion's
// quick rejects, as the resolve oracle's RecursionFilter does them), its upstream query, the queries grouped by route
// with a stable sort, and for each miss the first received datagram that passes the match rules.  The query decoder
// is the resolve oracle's own (oracle/oracle.cpp, included unchanged).  Built and loaded by tests/forward_oracle.py.
#include "../../oracle/oracle.cpp"

namespace {

constexpr uint32_t R_PTR = 16, R_NONE = 17, N_ROUTES = 18;

uint32_t mix(uint32_t h) { h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16; return h; }

// the keyed 16-bit bijection: 4 Feistel rounds over (high byte, low byte)
struct Feistel {
    uint32_t k[4];
    explicit Feistel(uint64_t key) {
        for (uint32_t i = 0; i < 4; i++) k[i] = mix((uint32_t)key ^ mix((uint32_t)(key >> 32) + 0x9E3779B9u * (i + 1)));
    }
    uint32_t f(int i, uint32_t x) const { return mix(x ^ k[i]) & 0xFF; }
    uint32_t enc(uint32_t j) const {
        uint32_t a = j >> 8 & 0xFF, b = j & 0xFF;
        for (int i = 0; i < 4; i++) { const uint32_t t = a ^ f(i, b); a = b; b = t; }
        return a << 8 | b;
    }
    uint32_t dec(uint32_t id) const {
        uint32_t a = id >> 8 & 0xFF, b = id & 0xFF;
        for (int i = 3; i >= 0; i--) { const uint32_t t = b ^ f(i, a); b = a; a = t; }
        return a << 8 | b;
    }
};

struct Table {
    RecursionFilter rf;
    std::vector<uint32_t> ip; std::vector<uint16_t> port; std::vector<uint8_t> dc;
    Table(const char* region, const char* const* dcs, uint32_t n_dc, const uint32_t* ip_, const uint16_t* port_, const uint8_t* dc_, uint32_t n_up) {
        rf.enabled = true; rf.dnsDomain = region;
        for (uint32_t i = 0; i < n_dc; i++) rf.dcs.push_back(dcs[i]);
        ip.assign(ip_, ip_ + n_up); port.assign(port_, port_ + n_up); dc.assign(dc_, dc_ + n_up);
    }
    // Recursion.resolve's choice of upstreams (:329-379) as a route
    uint32_t route(const Query& q) const {
        if (q.qtype == T_PTR) return ip.empty() ? R_NONE : R_PTR;
        const std::string& d = q.name;
        long from = (long)d.size() - (long)rf.dnsDomain.size();
        if (d.find(rf.dnsDomain, (size_t)(from < 0 ? 0 : from)) == std::string::npos) return R_NONE;
        long end = (long)d.size() - (long)rf.dnsDomain.size() - 1;
        std::string p = d.substr(0, (size_t)(end < 0 ? 0 : end));
        size_t dot = p.rfind('.');
        std::string name = p.substr(dot == std::string::npos ? 0 : dot + 1);
        auto it = std::find(rf.dcs.begin(), rf.dcs.end(), name);
        if (it == rf.dcs.end()) return R_NONE;
        const uint32_t k = (uint32_t)(it - rf.dcs.begin());
        for (uint8_t x : dc) if (x == k) return k;
        return R_NONE;
    }
    bool source_ok(uint32_t rt, uint32_t sip, uint32_t sport) const {
        for (size_t i = 0; i < ip.size(); i++)
            if (ip[i] == sip && port[i] == sport && (rt == R_PTR || dc[i] == rt)) return true;
        return false;
    }
};

// question bytes (QNAME labels, QTYPE, QCLASS) of a packet, or 0
uint32_t question_bytes(const uint8_t* p, uint32_t len) {
    uint32_t pos = 12;
    while (pos < len && p[pos] != 0) {
        if (p[pos] > 63) return 0;
        pos += 1 + p[pos];
    }
    if (pos >= len || pos + 5 > len) return 0;
    return pos + 5 - 12;
}

}  // namespace

extern "C" {

uint32_t orc_fwd_id(uint64_t key, uint32_t x, int inverse) { Feistel F(key); return inverse ? F.dec(x) : F.enc(x); }

// Forward: miss j = pkts[off[j] .. off[j+1]).  Outputs as bb_forward_batch (uq packed by output position).
int orc_forward_batch(const char* region, const char* const* dcs, uint32_t n_dc, const uint32_t* ip, const uint16_t* port, const uint8_t* dc,
                      uint32_t n_up, const uint8_t* pkts, const uint32_t* off, uint32_t n, uint64_t key, uint8_t* uq, uint32_t* uq_off,
                      uint32_t* order, uint32_t* group_off, uint8_t* route) {
    Table tb(region, dcs, n_dc, ip, port, dc, n_up);
    Feistel F(key);
    std::vector<std::vector<uint8_t>> msg(n);
    for (uint32_t j = 0; j < n; j++) {
        Query q;
        route[j] = (uint8_t)R_NONE;
        if (off[j + 1] < off[j] || !decode(pkts + off[j], off[j + 1] - off[j], q)) continue;
        route[j] = (uint8_t)tb.route(q);
        std::vector<uint8_t>& m = msg[j];
        put16(m, F.enc(j));
        put16(m, (unsigned)((q.pkt[2] << 8 | q.pkt[3]) & 0x7800));        // opcode; msg.clearFlag('rd')
        put16(m, 1); put16(m, 0); put16(m, 0); put16(m, 0);
        m.insert(m.end(), q.pkt + 12, q.pkt + q.q_end);                      // QNAME, QTYPE, QCLASS
    }
    uint32_t k = 0, at = 0;
    for (uint32_t r = 0; r < N_ROUTES; r++) {
        group_off[r] = k;
        for (uint32_t j = 0; j < n; j++) {
            if (route[j] != r) continue;
            order[k] = j; uq_off[k] = at;
            memcpy(uq + at, msg[j].data(), msg[j].size());
            at += (uint32_t)msg[j].size(); k++;
        }
    }
    group_off[N_ROUTES] = k; uq_off[n] = at;
    return 0;
}

// Match: response r = resp[resp_off[r] .. resp_off[r+1]) from src_ip[r]:src_port[r]; the misses' client queries in miss
// order (q / q_off) and routes.  -> up / up_off in miss order (the first accepted response of each miss, or nothing).
int orc_match(const char* region, const char* const* dcs, uint32_t n_dc, const uint32_t* ip, const uint16_t* port, const uint8_t* dc,
              uint32_t n_up, const uint8_t* resp, const uint32_t* resp_off, const uint32_t* src_ip, const uint16_t* src_port, uint32_t n_resp,
              const uint8_t* q, const uint32_t* q_off, const uint8_t* route, uint32_t n, uint64_t key, uint8_t* up, uint32_t* up_off) {
    Table tb(region, dcs, n_dc, ip, port, dc, n_up);
    Feistel F(key);
    std::vector<int64_t> win(n, -1);
    for (uint32_t r = 0; r < n_resp; r++) {
        const uint8_t* u = resp + resp_off[r];
        const uint32_t len = resp_off[r + 1] - resp_off[r];
        if (len < 12 || !(u[2] & 0x80)) continue;                            // too short for a header / not a response
        const uint32_t j = F.dec((uint32_t)(u[0] << 8 | u[1]));
        if (j >= n || win[j] >= 0 || route[j] >= R_NONE) continue;           // foreign ID / answered already / never sent
        if (!tb.source_ok(route[j], src_ip[r], src_port[r])) continue;       // not an upstream this miss went to
        if ((u[4] << 8 | u[5]) == 0) continue;                               // no question
        const uint8_t* c = q + q_off[j];
        const uint32_t ql = question_bytes(c, q_off[j + 1] - q_off[j]);
        if (ql == 0 || len < 12 + ql || memcmp(u + 12, c + 12, ql) != 0) continue;   // not the question that was asked
        win[j] = r;
    }
    uint32_t at = 0;
    for (uint32_t j = 0; j < n; j++) {
        up_off[j] = at;
        if (win[j] < 0) continue;
        const uint32_t r = (uint32_t)win[j], len = resp_off[r + 1] - resp_off[r];
        memcpy(up + at, resp + resp_off[r], len);
        at += len;
    }
    up_off[n] = at;
    return 0;
}

}  // extern "C"
