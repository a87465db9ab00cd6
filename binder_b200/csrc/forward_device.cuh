// Per-miss device code of the recursion forward and match kernels (DESIGN.md section 14, lib/recursion.js:253-280,
// 335-354,382-387): the upstream query a miss sends, the datacenter it goes to, its ID, and whether an upstream response
// belongs to it.  Included by engine.cu after resolve_device.cuh (it reuses decode() and the pre-filter's rf_dc_index());
// like those files it also compiles with g++ against tests/native/cuda_shim.h (tests/native/emu_forward.cpp).
//
// The upstream responses arrive from the network: every read of one is checked against its length.
#ifndef BB_FORWARD_DEVICE_CUH
#define BB_FORWARD_DEVICE_CUH

namespace bbk {

constexpr uint32_t FWD_MAX = 65536;                    // misses per forward call: the 16-bit ID space
// routes: 0 .. RF_MAX_DC - 1 = the datacenter with that index in the filter, then "every datacenter" (PTR), then none
constexpr uint32_t RT_PTR = RF_MAX_DC, RT_NONE = RF_MAX_DC + 1, NROUTE = RF_MAX_DC + 2;
constexpr uint32_t NO_MATCH = 0xFFFFFFFFu;

// ---- upstream IDs: a keyed bijection on 16 bits ------------------------------------------------------------------
// A 4-round Feistel network over the two bytes of j.  Round i's function is fmix32(x ^ k[i]) & 0xFF with
// k[i] = fmix32(lo ^ fmix32(hi + 0x9E3779B9 * (i + 1))) of the 64-bit key (lo, hi): distinct j give distinct IDs, and the
// ID of a miss cannot be told without the key (recursion.py draws them from os.urandom for the same reason).
struct IdKey { uint32_t k[4]; };
__host__ __device__ inline IdKey id_key_rounds(uint64_t key) {
    IdKey K;
    const uint32_t lo = (uint32_t)key, hi = (uint32_t)(key >> 32);
    for (uint32_t i = 0; i < 4; i++) K.k[i] = fmix32(lo ^ fmix32(hi + 0x9E3779B9u * (i + 1)));
    return K;
}
__device__ __forceinline__ uint32_t id_enc(const IdKey& K, uint32_t j) {
    uint32_t L = (j >> 8) & 0xFF, R = j & 0xFF;
#pragma unroll
    for (int i = 0; i < 4; i++) { const uint32_t t = L ^ (fmix32(R ^ K.k[i]) & 0xFF); L = R; R = t; }
    return L << 8 | R;
}
__device__ __forceinline__ uint32_t id_dec(const IdKey& K, uint32_t id) {
    uint32_t L = (id >> 8) & 0xFF, R = id & 0xFF;
#pragma unroll
    for (int i = 3; i >= 0; i--) { const uint32_t t = R ^ (fmix32(L ^ K.k[i]) & 0xFF); R = L; L = t; }
    return L << 8 | R;
}

// ---- forward: route and upstream query of one miss -----------------------------------------------------------------
// The route of a miss decode() accepted (d): PTR asks every upstream (:346-354); any other type the datacenter the
// pre-filter's scan finds (:329-344), when the upstream table has an upstream there; otherwise none.
__device__ __forceinline__ uint32_t fwd_route(const EngineConst* E, const uint8_t* q, const Res& d) {
    if (d.qtype == QT_PTR) return E->fu_n ? RT_PTR : RT_NONE;
    const int k = rf_dc_index(E, q + 12, d.qn_len - 1);
    return (k >= 0 && ((E->fu_dcmask >> k) & 1u)) ? (uint32_t)k : RT_NONE;
}
// The upstream query recursion.py's _exchange sends (lib/recursion.js:253-262): ID, the client's flags & 0x7800 (opcode
// kept, RD cleared), QD = 1, AN = NS = AR = 0, the client's QNAME wire bytes, QTYPE and QCLASS; no OPT.  12 + qn_len + 4 bytes.
__device__ __forceinline__ void fwd_emit(const uint8_t* q, uint32_t qn_len, uint32_t id, uint8_t* dst) {
    dst[0] = (uint8_t)(id >> 8); dst[1] = (uint8_t)id;
    dst[2] = (uint8_t)(q[2] & 0x78); dst[3] = 0;
    dst[4] = 0; dst[5] = 1;
    for (int i = 6; i < 12; i++) dst[i] = 0;
    for (uint32_t i = 0; i < qn_len + 4; i++) dst[12 + i] = q[12 + i];
}

// ---- match: which miss an upstream response answers ----------------------------------------------------------------
// Bytes of the question of a client query c[0, clen): QNAME (uncompressed labels) + QTYPE + QCLASS, or 0 if malformed.
__device__ __forceinline__ uint32_t client_question_len(const uint8_t* c, uint32_t clen) {
    uint32_t pos = 12;
    for (;;) {
        if (pos >= clen) return 0;
        const uint32_t l = c[pos];
        if (l == 0) break;
        if (l > 63) return 0;
        pos += 1 + l;
    }
    return pos + 1 + 4 <= clen ? pos + 1 + 4 - 12 : 0;
}
// Response u[0, ulen) from src_ip:src_port -> the miss j it answers, or NO_MATCH.  Accepted when the ID decodes to a
// j < n, the length is at least 12 and QR is set, the source is an upstream of route[j] (any upstream for PTR), as in
// recursion.py, QDCOUNT >= 1 and the first question equals the forwarded one byte for byte (no compression pointer,
// same case).  c / c_off: the client queries in j order (the forward kernel's packed copy).
__device__ __forceinline__ uint32_t match_one(const EngineConst* E, const IdKey& K, const uint8_t* u, uint32_t ulen, uint32_t src_ip,
                                              uint32_t src_port, uint32_t n, const uint8_t* route, const uint8_t* c, const uint32_t* c_off) {
    if (ulen < 12 || !(u[2] & 0x80)) return NO_MATCH;
    const uint32_t j = id_dec(K, be16(u));
    if (j >= n) return NO_MATCH;
    const uint32_t rt = route[j];
    if (rt >= RT_NONE) return NO_MATCH;
    bool src = false;
    for (uint32_t i = 0; i < E->fu_n; i++)
        src |= E->fu_ip[i] == src_ip && E->fu_port[i] == src_port && (rt == RT_PTR || E->fu_dc[i] == rt);
    if (!src || be16(u + 4) == 0) return NO_MATCH;
    const uint32_t c0 = c_off[j], c1 = c_off[j + 1];
    if (c1 < c0) return NO_MATCH;
    const uint8_t* cq = c + c0;
    const uint32_t ql = client_question_len(cq, c1 - c0);
    if (ql == 0 || 12 + ql > ulen) return NO_MATCH;
    for (uint32_t i = 0; i < ql; i++) if (u[12 + i] != cq[12 + i]) return NO_MATCH;
    return j;
}

}  // namespace bbk

#endif
