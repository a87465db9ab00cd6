// TEST INFRASTRUCTURE — CPU oracle of the recursion relay (DESIGN.md section 13).  NOT the product.
//
// Restates Recursion.prototype.resolve's respond() (lib/recursion.js:287-327) literally: a byte-serial decoder turns the
// upstream response into records shaped like what mname-client's getAnswers() hands to respond(), respond() re-wraps
// them (query.setError / query.addAnswer), and the reply is encoded by DESIGN.md section 3's rules.  The query decoder
// and the byte helpers are the resolve oracle's own (oracle/oracle.cpp, included unchanged), so a query is accepted or
// dropped exactly as the resolve path does it.  Built and loaded by tests/relay_oracle.py.
#include "../../oracle/oracle.cpp"

namespace {

// One record of the upstream's answer section, as getAnswers() would give it: type name, target (address bytes, TXT
// bytes, or a name as labels), SRV fields, ttl.
struct UpRecord {
    std::string type; uint16_t klass = 0; uint32_t ttl = 0;
    std::vector<uint8_t> bytes; std::vector<std::string> labels;
    uint16_t priority = 0, weight = 0, port = 0;
};

// Byte-serial decode of the upstream response (DESIGN.md section 13, "upstream decode"); false = the lookup failed
// (recursion.js then keeps answers = []: `if (!err) answers = ans` is skipped).
struct UpstreamDecoder {
    const uint8_t* p; size_t len;
    bool name(size_t pos, std::vector<std::string>& labels, size_t& next) const {
        size_t wire = 1; bool jumped = false;
        for (;;) {
            if (pos >= len) return false;
            const uint8_t c = p[pos];
            if ((c & 0xC0) == 0xC0) {                                      // pointer: strictly backwards
                if (pos + 2 > len) return false;
                const size_t to = (size_t)(c & 0x3F) << 8 | p[pos + 1];
                if (to >= pos) return false;
                if (!jumped) { next = pos + 2; jumped = true; }
                pos = to; continue;
            }
            if (c & 0xC0) return false;
            if (c == 0) { if (!jumped) next = pos + 1; return true; }
            if (pos + 1 + c > len) return false;
            labels.emplace_back((const char*)p + pos + 1, c);
            wire += 1 + c;
            if (wire > 255) return false;
            pos += 1 + c;
        }
    }
    static std::string type_name(unsigned t) {
        switch (t) {
        case 1: return "A"; case 5: return "CNAME"; case 12: return "PTR"; case 16: return "TXT";
        case 28: return "AAAA"; case 33: return "SRV";
        }
        return "TYPE" + std::to_string(t);
    }
    bool answers(std::vector<UpRecord>& out) const {
        if (len < 12 || len > 65535 || !(p[2] & 0x80)) return false;
        const unsigned qd = p[4] << 8 | p[5], an = p[6] << 8 | p[7];
        size_t pos = 12;
        for (unsigned i = 0; i < qd; i++) {
            std::vector<std::string> l; size_t next = 0;
            if (!name(pos, l, next) || next + 4 > len) return false;
            pos = next + 4;
        }
        for (unsigned i = 0; i < an; i++) {
            std::vector<std::string> owner; size_t next = 0;
            if (!name(pos, owner, next) || next + 10 > len) return false;
            const uint8_t* h = p + next;
            const unsigned type = h[0] << 8 | h[1], rdlen = h[8] << 8 | h[9];
            const size_t rd = next + 10;
            if (rd + rdlen > len) return false;
            UpRecord r;
            r.type = type_name(type); r.klass = (uint16_t)(h[2] << 8 | h[3]);
            r.ttl = (uint32_t)h[4] << 24 | (uint32_t)h[5] << 16 | (uint32_t)h[6] << 8 | h[7];
            size_t end = 0;
            if (type == 1 || type == 28) {
                if (rdlen != (type == 1 ? 4u : 16u)) return false;
                r.bytes.assign(p + rd, p + rd + rdlen);
            } else if (type == 16) {
                r.bytes.assign(p + rd, p + rd + rdlen);
            } else if (type == 5 || type == 12) {
                if (!name(rd, r.labels, end) || end > rd + rdlen) return false;
            } else if (type == 33) {
                if (rdlen < 7) return false;
                r.priority = (uint16_t)(p[rd] << 8 | p[rd + 1]); r.weight = (uint16_t)(p[rd + 2] << 8 | p[rd + 3]);
                r.port = (uint16_t)(p[rd + 4] << 8 | p[rd + 5]);
                if (!name(rd + 6, r.labels, end) || end > rd + rdlen) return false;
            }
            out.push_back(std::move(r));
            pos = rd + rdlen;
        }
        return true;
    }
};

std::vector<uint8_t> wire_labels(const std::vector<std::string>& labels) {
    std::vector<uint8_t> o;
    for (auto& l : labels) { o.push_back((uint8_t)l.size()); o.insert(o.end(), l.begin(), l.end()); }
    o.push_back(0);
    return o;
}

// The reply respond() builds: every RR is an answer with owner query.name() (DESIGN.md section 3 rule (1): the pointer
// 0xC00C, or the root name itself for a root QNAME), then query.respond() encodes it.
struct RelayReply {
    const Query& q; int rcode = -1;
    struct Answer { uint16_t type; uint32_t ttl; std::vector<uint8_t> rdata; };
    std::vector<Answer> answers;
    explicit RelayReply(const Query& qq) : q(qq) {}
    void setError(int rc) { rcode = rc; }
    void addAnswer(uint16_t type, uint32_t ttl, std::vector<uint8_t>&& rd) { answers.push_back({ type, ttl, std::move(rd) }); }
    // DESIGN.md section 3: header, question verbatim, the longest prefix of the answers that fits, TC if one was cut,
    // the OPT echoed last; RCODE = the one set, else NOERROR if an answer was added, else NOTIMP
    size_t encode(uint8_t* out) const {
        const int rc = rcode >= 0 ? rcode : (answers.empty() ? RC_NOTIMP : RC_NOERROR);
        size_t maxsz = 512;
        if (q.edns) maxsz = std::min<size_t>(std::max<size_t>(q.adv, 512), 1200);
        if (q.tcp) maxsz = 65535;
        const size_t fixed = 12 + (q.q_end - 12) + (q.edns ? 11 : 0);
        std::vector<uint8_t> owner = q.labels.empty() ? std::vector<uint8_t>{ 0 } : std::vector<uint8_t>{ 0xC0, 0x0C };
        size_t total = fixed, keep = 0;
        for (; keep < answers.size(); keep++) {
            const size_t sz = owner.size() + 10 + answers[keep].rdata.size();
            if (total + sz > maxsz) break;
            total += sz;
        }
        const bool tc = keep < answers.size();
        std::vector<uint8_t> o;
        put16(o, q.id);
        o.push_back((uint8_t)(0x80 | (q.opcode << 3) | 0x04 | (tc ? 0x02 : 0) | (q.rd ? 1 : 0)));
        o.push_back((uint8_t)rc);
        put16(o, 1); put16(o, (unsigned)keep); put16(o, 0); put16(o, q.edns ? 1 : 0);
        o.insert(o.end(), q.pkt + 12, q.pkt + q.q_end);
        for (size_t i = 0; i < keep; i++) {
            const Answer& a = answers[i];
            o.insert(o.end(), owner.begin(), owner.end());
            put16(o, a.type); put16(o, 1); put32(o, a.ttl); put16(o, (unsigned)a.rdata.size());
            o.insert(o.end(), a.rdata.begin(), a.rdata.end());
        }
        if (q.edns) { const uint8_t opt[11] = { 0, 0, T_OPT, 0x04, 0xB0, 0, 0, 0, 0, 0, 0 }; o.insert(o.end(), opt, opt + 11); }
        memcpy(out, o.data(), o.size());
        return o.size();
    }
};

// respond() (lib/recursion.js:292-326) once lookup() has called back.
void relay_respond(const std::vector<UpRecord>& answers, RelayReply& r) {
    if (answers.empty()) { r.setError(RC_REFUSED); return; }                  // :293-295
    for (const UpRecord& rec : answers) {                                     // :299-323
        if (rec.klass != 1) continue;                                         // only class IN is re-wrapped
        uint16_t type;
        std::vector<uint8_t> rd;
        if (rec.type == "A" || rec.type == "AAAA" || rec.type == "TXT") {
            type = rec.type == "A" ? 1 : rec.type == "AAAA" ? 28 : 16;
            rd = rec.bytes;
        } else if (rec.type == "PTR" || rec.type == "CNAME") {
            type = rec.type == "PTR" ? 12 : 5;
            rd = wire_labels(rec.labels);
        } else if (rec.type == "SRV") {
            type = 33;
            put16(rd, rec.priority); put16(rd, rec.weight); put16(rd, rec.port);
            std::vector<uint8_t> t = wire_labels(rec.labels);
            rd.insert(rd.end(), t.begin(), t.end());
        } else continue;                                                      // :316-320 unsupported type: dropped
        r.addAnswer(type, rec.ttl, std::move(rd));                            // query.addAnswer(domain, inst, rec.ttl)
    }
}

}  // namespace

extern "C" {

// Relay batch (bb_relay_batch's container): query i = q_pkts[q_off[i] .. q_off[i+1]), its upstream response
// up_pkts[up_off[i] .. up_off[i+1]) (empty: the lookup failed or was not made).  Replies packed in order.
// flags: 1 = the queries arrived over TCP.  Returns -2 when out_cap is too small.
int orc_relay_batch(const uint8_t* q_pkts, const uint32_t* q_off, const uint8_t* up_pkts, const uint32_t* up_off, uint32_t n,
                    uint32_t flags, uint8_t* out, uint64_t out_cap, uint32_t* out_off, uint8_t* status, int nthreads) {
    const bool tcp = (flags & 1u) != 0;
    if (nthreads < 1) nthreads = 1;
    if ((uint32_t)nthreads > n) nthreads = n ? (int)n : 1;
    struct Part { std::vector<uint8_t> bytes; std::vector<uint32_t> lens; };
    std::vector<Part> parts(nthreads);
    auto work = [&](int t) {
        uint32_t lo = (uint32_t)((uint64_t)n * t / nthreads), hi = (uint32_t)((uint64_t)n * (t + 1) / nthreads);
        Part& P = parts[t]; P.lens.resize(hi - lo);
        std::vector<uint8_t> tmp(65536);
        for (uint32_t i = lo; i < hi; i++) {
            Query q; size_t w = 0;
            if (!decode(q_pkts + q_off[i], q_off[i + 1] - q_off[i], q)) status[i] = ST_DROPPED;
            else {
                q.tcp = tcp;
                RelayReply r(q);
                std::vector<UpRecord> answers;
                UpstreamDecoder up{ up_pkts + up_off[i], (size_t)(up_off[i + 1] - up_off[i]) };
                if (!up.answers(answers)) answers.clear();                   // error / timeout (:382-386)
                relay_respond(answers, r);
                status[i] = ST_ANSWERED;
                w = r.encode(tmp.data());
            }
            P.lens[i - lo] = (uint32_t)w;
            P.bytes.insert(P.bytes.end(), tmp.data(), tmp.data() + w);
        }
    };
    if (nthreads == 1) work(0);
    else { std::vector<std::thread> th; for (int t = 0; t < nthreads; t++) th.emplace_back(work, t); for (auto& x : th) x.join(); }
    uint64_t pos = 0; uint32_t i = 0;
    for (int t = 0; t < nthreads; t++) {
        Part& P = parts[t];
        if (pos + P.bytes.size() > out_cap) return -2;
        memcpy(out + pos, P.bytes.data(), P.bytes.size());
        for (uint32_t l : P.lens) { out_off[i++] = (uint32_t)pos; pos += l; }
    }
    out_off[n] = (uint32_t)pos;
    return 0;
}

}  // extern "C"
