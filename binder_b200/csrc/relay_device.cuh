// Per-relay device code of the recursion relay (DESIGN.md section 13, lib/recursion.js:287-327): decode of an untrusted
// upstream response, sizing with truncation, emit.  Included by engine.cu after resolve_device.cuh (it reuses that file's
// query decode() and byte emitter Out); like it, it also compiles with g++ against tests/native/cuda_shim.h
// (tests/native/emu_relay.cpp runs it on the CPU).
//
// The upstream packet arrives from the network: every read of it is checked against its length.  The query packet has
// been accepted by decode() first, which checks its own bounds.
#ifndef BB_RELAY_DEVICE_CUH
#define BB_RELAY_DEVICE_CUH

namespace bbk {

enum { UT_A = 1, UT_CNAME = 5, UT_PTR = 12, UT_TXT = 16, UT_AAAA = 28, UT_SRV = 33 };

// The name at `pos` of the upstream packet u[0, len).  Labels are 1..63 bytes, a pointer (two bytes, 0b11 prefix) must
// point strictly before its own position, the decompressed name is at most 255 wire bytes; anything else -> false.
// `end` = first byte after the name's bytes at `pos` (its terminator or its first pointer), `wl` = decompressed wire
// length with the terminator.  With `w`, the decompressed labels are written out (original case, no compression).
// Termination: a run of pointers strictly decreases, and every label in between adds to the 255-byte budget.
// W is any sink with u8() (a length byte, 0 for the terminator) and copy() (a label's bytes): the relay writes the labels
// with Out, the query log (log_device.cuh) renders them as a dotted string.
template <class W>
__device__ bool up_name(const uint8_t* u, uint32_t len, uint32_t pos, uint32_t& end, uint32_t& wl, W* w) {
    uint32_t p = pos, n = 0;
    bool jumped = false;
    for (;;) {
        if (p >= len) return false;
        const uint32_t c = u[p];
        if (c >= 0xC0) {
            if (p + 1 >= len) return false;
            const uint32_t t = ((c & 0x3Fu) << 8) | u[p + 1];
            if (t >= p) return false;
            if (!jumped) { end = p + 2; jumped = true; }
            p = t;
            continue;
        }
        if (c > 63) return false;                        // 0b01 / 0b10 label types
        if (c == 0) {
            if (!jumped) end = p + 1;
            if (w) w->u8(0);
            wl = n + 1;
            return true;
        }
        if (p + 1 + c > len) return false;
        n += 1 + c;
        if (n + 1 > 255) return false;
        if (w) { w->u8(c); w->copy(u + p + 1, c); }
        p += 1 + c;
    }
}

// one answer RR of the upstream
struct UpRR { uint32_t type, klass, ttl, rd, rdlen, nwl; };

// The RR at `pos`: it and its RDATA lie inside the packet; A has RDLEN 4, AAAA 16, SRV >= 7; the name in the RDATA of
// CNAME, PTR and SRV is valid and ends inside RDLEN.  -> false when malformed; else `pos` moves past the RR.
__device__ bool up_rr(const uint8_t* u, uint32_t len, uint32_t& pos, UpRR& rr) {
    uint32_t end = 0, wl = 0;
    if (!up_name<Out>(u, len, pos, end, wl, nullptr) || end + 10 > len) return false;
    rr.type = be16(u + end); rr.klass = be16(u + end + 2);
    rr.ttl = be16(u + end + 4) << 16 | be16(u + end + 6);
    rr.rdlen = be16(u + end + 8); rr.rd = end + 10; rr.nwl = 0;
    const uint32_t rdend = rr.rd + rr.rdlen;
    if (rdend > len) return false;
    switch (rr.type) {
    case UT_A: if (rr.rdlen != 4) return false; break;
    case UT_AAAA: if (rr.rdlen != 16) return false; break;
    case UT_SRV: if (rr.rdlen < 7 || !up_name<Out>(u, len, rr.rd + 6, end, rr.nwl, nullptr) || end > rdend) return false; break;
    case UT_CNAME: case UT_PTR: if (!up_name<Out>(u, len, rr.rd, end, rr.nwl, nullptr) || end > rdend) return false; break;
    }
    pos = rdend;
    return true;
}
// the types recursion.js re-wraps (:299-315), class IN only; everything else is dropped (:316-320)
__device__ __forceinline__ bool up_kept(const UpRR& rr) {
    return rr.klass == 1 && (rr.type == UT_A || rr.type == UT_AAAA || rr.type == UT_TXT || rr.type == UT_PTR ||
                             rr.type == UT_CNAME || rr.type == UT_SRV);
}
// RDLEN of the reply's RR: names are written decompressed; SRV keeps the upstream's priority, weight and port
__device__ __forceinline__ uint32_t up_out_rdlen(const UpRR& rr) {
    return rr.type == UT_SRV ? 6 + rr.nwl : (rr.type == UT_PTR || rr.type == UT_CNAME) ? rr.nwl : rr.rdlen;
}

// per-relay state carried from the sizing pass to the emit pass
struct Relay {
    uint32_t status, rcode, tc, rlen;
    uint32_t opcode, rd, edns, qn_len;   // of the query (decode())
    uint32_t keep;                       // answer RRs written
    uint32_t an0, nan;                   // first answer RR of the upstream and ANCOUNT (read again by the emit pass)
};

// Decode both packets and size the reply (query.respond() after respond(), lib/recursion.js:292-326, with DESIGN.md
// section 3's header, EDNS and truncation rules).  An empty or malformed upstream, or one without answer RRs, gives
// REFUSED; answers that are all dropped give no answer and no error, hence NOTIMP.
__device__ void relay_size(const uint8_t* q, uint32_t qlen, const uint8_t* u, uint32_t ulen, bool tcp, Relay& R) {
    R.rlen = 0; R.keep = 0; R.tc = 0; R.nan = 0; R.an0 = 0; R.rcode = RC_REFUSED;
    Res d;
    if (qlen > 65535u || !decode(q, qlen, d)) { R.status = ST_DROPPED; return; }
    R.status = ST_ANSWERED; R.opcode = d.opcode; R.rd = d.rd; R.edns = d.edns; R.qn_len = d.qn_len;
    const uint32_t maxsz = tcp ? 65535u : d.edns ? min(max((uint32_t)d.adv, 512u), 1200u) : 512u;
    const uint32_t fixed = 12 + d.qn_len + 4 + (d.edns ? 11 : 0), own = d.qn_len > 1 ? 2 : 1;
    R.rlen = fixed;
    bool ok = ulen >= 12 && ulen <= 65535u && (u[2] & 0x80), full = false;
    uint32_t pos = 12, an = 0, kept = 0, total = fixed, keep = 0;
    if (ok) {
        const uint32_t qd = be16(u + 4);
        an = be16(u + 6);
        for (uint32_t i = 0; ok && i < qd; i++) {                 // questions: skipped, but they must be well formed
            uint32_t end = 0, wl = 0;
            ok = up_name<Out>(u, ulen, pos, end, wl, nullptr) && end + 4 <= ulen;
            pos = end + 4;
        }
        R.an0 = pos;
        for (uint32_t i = 0; ok && i < an; i++) {                 // every answer is checked, also past a truncation
            UpRR rr;
            ok = up_rr(u, ulen, pos, rr);
            if (!ok || !up_kept(rr)) continue;
            ++kept;
            const uint32_t sz = own + 10 + up_out_rdlen(rr);
            if (!full && total + sz <= maxsz) { total += sz; ++keep; }
            else full = true;
        }
    }
    if (!ok || an == 0) return;                                   // REFUSED, no answers
    if (kept == 0) { R.rcode = RC_NOTIMP; return; }
    R.rcode = RC_NOERROR; R.tc = full; R.rlen = total; R.keep = keep; R.nan = an;
}

// The reply relay_size() sized, R.rlen bytes at dst.
__device__ void relay_emit(const uint8_t* q, const uint8_t* u, uint32_t ulen, const Relay& R, uint8_t* dst) {
    Out w; w.o = dst;
    w.u8(q[0]); w.u8(q[1]);
    w.u8(0x80 | (R.opcode << 3) | 0x04 | (R.tc ? 0x02 : 0) | R.rd);          // QR AA TC RD
    w.u8(R.rcode);                                                            // RA=0 Z=0
    w.u16(1); w.u16(R.keep); w.u16(0); w.u16(R.edns);
    w.copy(q + 12, R.qn_len + 4);                                             // question, verbatim
    uint32_t pos = R.an0;
    for (uint32_t i = 0, k = 0; k < R.keep && i < R.nan; i++) {
        UpRR rr;
        up_rr(u, ulen, pos, rr);                                              // validated by relay_size()
        if (!up_kept(rr)) continue;
        if (R.qn_len > 1) w.u16(0xC00C); else w.u8(0);                       // owner = query.name()
        w.u16(rr.type); w.u16(1); w.u32(rr.ttl); w.u16(up_out_rdlen(rr));
        uint32_t end = 0, wl = 0;
        if (rr.type == UT_SRV) { w.copy(u + rr.rd, 6); up_name(u, ulen, rr.rd + 6, end, wl, &w); }
        else if (rr.type == UT_PTR || rr.type == UT_CNAME) up_name(u, ulen, rr.rd, end, wl, &w);
        else w.copy(u + rr.rd, rr.rdlen);                                     // A, AAAA, TXT
        ++k;
    }
    if (R.edns) { const uint8_t* opt = c_opt_rr; w.copy(opt, 11); }
}

}  // namespace bbk

#endif
