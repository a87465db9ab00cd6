// Per-response device code of the query log (DESIGN.md section 15, lib/server.js:509-591): binder's "DNS query" record
// of one response, as two JSON fragments.  Included by engine.cu after relay_device.cuh, whose bounds-checked up_name
// and up_rr it decodes with; like them it also compiles with g++ against tests/native/cuda_shim.h
// (tests/native/emu_log.cpp runs it on the CPU).
//
// The response bytes come from the caller (relayed replies carry upstream-derived names): every read is checked against
// the response's length.  The record is written by one function in two passes: sizing (Txt::o == nullptr) and emit.
// Text is rendered from immediates and arithmetic: no tables in global memory.
#ifndef BB_LOG_DEVICE_CUH
#define BB_LOG_DEVICE_CUH

namespace bbk {

enum { UT_NS = 2, UT_SOA = 6, UT_MX = 15, UT_OPT = 41, UT_AXFR = 252, UT_ANY = 255 };
// summary word: qtype | rcode << 16 | edns << 20 | tc << 21 | bad << 22
constexpr uint32_t LOG_BAD = 1u << 22;

__device__ __forceinline__ uint32_t hex_digit(uint32_t d) { return d < 10 ? '0' + d : 'a' - 10 + d; }

// A text cursor: o == nullptr counts the bytes only.
struct Txt {
    uint8_t* o; uint32_t n;
    __device__ __forceinline__ void b(uint32_t c) { if (o) o[n] = (uint8_t)c; n++; }
    // a literal: unrolled, so that its bytes become immediates
    template <int N> __device__ __forceinline__ void s(const char (&z)[N]) {
#pragma unroll
        for (int i = 0; i < N - 1; i++) b((uint8_t)z[i]);
    }
    // one latin-1 byte inside a JSON string, as JSON.stringify writes it and bunyan's UTF-8 stream encodes it
    __device__ void esc(uint32_t c) {
        if (c >= 0x80) { b(0xC0 | c >> 6); b(0x80 | (c & 0x3F)); return; }
        if (c >= 0x20) { if (c == '"' || c == '\\') b('\\'); b(c); return; }
        b('\\');
        switch (c) {
        case 8: b('b'); break;
        case 9: b('t'); break;
        case 10: b('n'); break;
        case 12: b('f'); break;
        case 13: b('r'); break;
        default: b('u'); b('0'); b('0'); b(hex_digit(c >> 4)); b(hex_digit(c & 15));
        }
    }
    __device__ void dec(uint32_t v) {
        uint32_t d = 1;
        for (uint32_t x = v; x >= 10; x /= 10) d++;
        if (o) for (uint32_t i = d, x = v; i--; x /= 10) o[n + i] = (uint8_t)('0' + x % 10);
        n += d;
    }
    __device__ void hex16(uint32_t v) {              // lower case, no leading zeros
        int sh = 12;
        while (sh && !(v >> sh)) sh -= 4;
        for (; sh >= 0; sh -= 4) b(hex_digit((v >> sh) & 15));
    }
};

// up_name's sink: the labels as query.name()'s dotted string, escaped into t (t == nullptr: not written).  Dotted bytes
// from index `cut` on are compared with sfx instead (stripSuffix); `match` stays true while they are equal.
struct DotSink {
    Txt* t; const uint8_t* sfx; uint32_t k, cut; bool match;
    __device__ void put(uint32_t c) {
        if (k >= cut) match &= c == sfx[k - cut];
        else if (t) t->esc(c);
        k++;
    }
    __device__ void u8(uint32_t c) { if (c && k) put('.'); }     // labels are not empty: k == 0 only before the first
    __device__ void copy(const uint8_t* p, uint32_t c) { for (uint32_t i = 0; i < c; i++) put(p[i]); }
};

// The (validated) name at `pos` as escaped JSON string content.  sl != 0: stripSuffix(sfx, name) (lib/server.js:55-65)
// with sfx = '.' + dnsDomain, sl bytes: a dotted name ending in it, case-sensitively, ends in "..." instead.
__device__ void log_name(Txt& t, const uint8_t* u, uint32_t len, uint32_t pos, const uint8_t* sfx, uint32_t sl) {
    uint32_t end = 0, wl = 0;
    up_name<Out>(u, len, pos, end, wl, nullptr);
    const uint32_t dl = wl > 1 ? wl - 2 : 0;                         // dotted length: labels and the dots between them
    DotSink d{ nullptr, sfx, 0, ~0u, true };
    if (sl && dl >= sl) {
        d.cut = dl - sl;
        up_name(u, len, pos, end, wl, &d);
        if (!d.match) d.cut = ~0u;
    }
    d.t = &t; d.k = 0;
    up_name(u, len, pos, end, wl, &d);
    if (d.cut != ~0u) t.s("...");
}

// "<mnemonic>" of a type, RFC 3597's "TYPE<n>" for the rest
__device__ void log_type(Txt& t, uint32_t type) {
    switch (type) {
    case UT_A: t.s("\"A\""); return;
    case UT_NS: t.s("\"NS\""); return;
    case UT_CNAME: t.s("\"CNAME\""); return;
    case UT_SOA: t.s("\"SOA\""); return;
    case UT_PTR: t.s("\"PTR\""); return;
    case UT_MX: t.s("\"MX\""); return;
    case UT_TXT: t.s("\"TXT\""); return;
    case UT_AAAA: t.s("\"AAAA\""); return;
    case UT_SRV: t.s("\"SRV\""); return;
    case UT_OPT: t.s("\"OPT\""); return;
    case UT_AXFR: t.s("\"AXFR\""); return;
    case UT_ANY: t.s("\"ANY\""); return;
    }
    t.s("\"TYPE"); t.dec(type); t.b('"');
}

// the address of an A (dotted quad) or AAAA RR (RFC 5952: the first longest run of two or more zero groups is "::")
__device__ void log_addr(Txt& t, const uint8_t* u, const UpRR& rr) {
    const uint8_t* a = u + rr.rd;
    if (rr.type == UT_A) {
        for (int i = 0; i < 4; i++) { if (i) t.b('.'); t.dec(a[i]); }
        return;
    }
    int z0 = 8, zn = 0;
    for (int i = 0; i < 8;) {
        int j = i;
        while (j < 8 && be16(a + 2 * j) == 0) j++;
        if (j - i > zn) { z0 = i; zn = j - i; }
        i = j > i ? j : i + 1;
    }
    if (zn < 2) z0 = 8;
    for (int i = 0; i < 8; i++) {
        if (i == z0) { t.s("::"); i += zn - 1; continue; }
        if (i && i != z0 + zn) t.b(':');
        t.hex16(be16(a + 2 * i));
    }
}

// TXT RDATA: one or more character-strings that fill RDLEN exactly (what dnspython accepts)
__device__ bool txt_ok(const uint8_t* u, const UpRR& rr) {
    uint32_t p = rr.rd;
    const uint32_t e = rr.rd + rr.rdlen;
    if (rr.rdlen == 0) return false;
    while (p < e) p += 1 + u[p];
    return p == e;
}

// The object form of an RR (Object.keys(rdata) then type): PTR and CNAME {"target":name}, TXT {"target":the strings
// concatenated}, anything else only its type.
__device__ void log_obj(Txt& t, const uint8_t* u, uint32_t len, const UpRR& rr) {
    t.b('{');
    if (rr.type == UT_PTR || rr.type == UT_CNAME || rr.type == UT_TXT) {
        t.s("\"target\":\"");
        if (rr.type == UT_TXT) {
            for (uint32_t p = rr.rd, e = rr.rd + rr.rdlen; p < e; p += 1 + u[p])
                for (uint32_t i = 1; i <= u[p]; i++) t.esc(u[p + i]);
        } else {
            log_name(t, u, len, rr.rd, nullptr, 0);
        }
        t.s("\",");
    }
    t.s("\"type\":"); log_type(t, rr.type); t.b('}');
}

// The record of response u[0, len) -> its summary word.  t receives head then body (hl = the head's length); a response
// that breaks a decode rule (DESIGN.md section 15) gives LOG_BAD and must not be emitted: its record is empty.
//   head  "query":{"name":N,"type":T},"edns":true|false
//   body  "rcode":R,"answers":[...],"additional":[...]
__device__ uint32_t log_record(const uint8_t* u, uint32_t len, const uint8_t* sfx, uint32_t sl, Txt& t, uint32_t& hl) {
    hl = 0;
    if (len < 12 || !(u[2] & 0x80) || be16(u + 4) != 1) return LOG_BAD;
    uint32_t qend = 0, wl = 0;
    // end == 12 + wl only without a pointer: one would leave at least 2 decompressed bytes past it for its 2 wire bytes
    if (!up_name<Out>(u, len, 12, qend, wl, nullptr) || qend != 12 + wl || qend + 4 > len) return LOG_BAD;
    const uint32_t an = be16(u + 6), ns = be16(u + 8), ar = be16(u + 10), rr0 = qend + 4;
    uint32_t edns = 0, pos = rr0;
    for (uint32_t i = 0; i < an + ns + ar; i++) {               // every RR inside the response, OPT seen
        UpRR rr;
        if (!up_rr(u, len, pos, rr) || (rr.type == UT_TXT && !txt_ok(u, rr))) return LOG_BAD;
        if (i >= an + ns && rr.type == UT_OPT) edns = 1;
    }
    const uint32_t qtype = be16(u + qend), rcode = u[3] & 15, tc = (u[2] >> 1) & 1;

    t.s("\"query\":{\"name\":\""); log_name(t, u, len, 12, nullptr, 0);
    t.s("\",\"type\":"); log_type(t, qtype);
    if (edns) t.s("},\"edns\":true"); else t.s("},\"edns\":false");
    hl = t.n;
    t.s("\"rcode\":"); t.dec(rcode);
    t.s(",\"answers\":[");
    pos = rr0;
    for (uint32_t i = 0; i < an; i++) {
        UpRR rr;
        up_rr(u, len, pos, rr);
        if (i) t.b(',');
        if (rr.type == UT_A || rr.type == UT_AAAA) {
            if (rr.type == UT_A) t.s("\"A "); else t.s("\"AAAA ");
            log_addr(t, u, rr); t.b('"');
        } else if (rr.type == UT_SRV) {
            t.s("\"SRV "); log_name(t, u, len, rr.rd + 6, sfx, sl);
            t.b(':'); t.dec(be16(u + rr.rd + 4)); t.b('"');
        } else {
            log_obj(t, u, len, rr);
        }
    }
    t.s("],\"additional\":[");
    for (uint32_t i = 0; i < ns; i++) { UpRR rr; up_rr(u, len, pos, rr); }      // the authority section is not logged
    bool first = true;
    for (uint32_t i = 0; i < ar; i++) {
        const uint32_t owner = pos;
        UpRR rr;
        up_rr(u, len, pos, rr);
        if (rr.type == UT_OPT) continue;
        if (!first) t.b(',');
        first = false;
        if (rr.type == UT_A || rr.type == UT_AAAA) {
            t.b('"'); log_name(t, u, len, owner, sfx, sl);
            if (rr.type == UT_A) t.s(" A "); else t.s(" AAAA ");
            log_addr(t, u, rr); t.b('"');
        } else {
            log_obj(t, u, len, rr);
        }
    }
    t.b(']');
    return qtype | rcode << 16 | edns << 20 | tc << 21;
}

}  // namespace bbk

#endif
