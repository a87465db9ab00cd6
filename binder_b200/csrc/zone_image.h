// Zone image: the HBM-resident, flattened form of binder's ZKCache (lib/zk.js:20-119).
//
// One 2-choice cuckoo table (power-of-two, load factor < 0.46) of 32-byte slots — ONE DRAM sector each —
// holds BOTH of ZKCache's maps.  A key lives in slot hash & mask (its first slot, where the builder puts it
// whenever it can: ~87 % of the keys at these load factors) or in slot hash2 & mask — two independent hashes of
// the key — never anywhere else; the first slot's position carries a flag when some key had to go to its second
// slot.  A lookup — hit or miss — therefore reads ONE random sector, and a second one only behind that flag:
// random DRAM accesses (row activations; tools/micro/probe_gran.cu measures their rate), not bytes,
// are what bounds a hash probe in HBM:
//   forward  ca_treeNodes[lower-cased fqdn]  (lib/zk.js:62-64, keys written at :84,96)
//   reverse  ca_revLookup[address string]    (lib/zk.js:65-67, keys written at :187-188)
// distinguished by a namespace bit that also seeds the hash.
//
// Forward keys are stored in CANONICAL form: the lower-cased fqdn minus the '.' + dnsDomain every reachable
// key ends with, as DNS wire labels (length byte + bytes per label).  resolve() only looks a name up after its
// case-sensitive suffix gate (lib/server.js:157-166) has shown that the name ends with '.' + dnsDomain, so
// string equality of the full names is equality of what precedes the suffix; and a query name without a '.'
// inside a label equals a key string exactly when their label sequences are equal.  The kernel therefore
// hashes and compares the query's own wire bytes (lower-cased; length bytes 1..63 are not letters) and never
// builds the dotted string: "h0001234.g0012.dc1.example.com" is the 15-byte key \x08h0001234\x05g0012.
// Reverse keys are the address strings themselves.
//
// Everything lib/server.js computes per query from the JSON record that does not depend on the query (record
// validation :251-260, ttl selection :270-274, url.parse :297-298, the service child filter :352-360 and
// per-child validation :366-393) is evaluated once at build time and stored as a `kind` + payload, so the
// kernel never touches JSON.
#ifndef BB_ZONE_IMAGE_H
#define BB_ZONE_IMAGE_H

#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define BB_HD __host__ __device__ __forceinline__
#else
#define BB_HD inline
#endif

namespace bb {

enum : uint8_t {
    K_EMPTY = 0,
    // forward namespace
    K_INVALID = 1,    // lib/server.js:251-260 fails (or a ttl mname would reject): SERVFAIL
    K_ADDR = 2,       // host-like / database with a usable IPv4: one A record (:296-311)
    K_ADDR_BAD = 3,   // typed + ttl fine, address unusable: A -> SERVFAIL, SRV -> NODATA (:276-292)
    K_SERVICE = 4,    // val = arena offset of a SvcHdr (:313-417)
    K_UNKNOWN = 5,    // record.type not in the switch (:419-424): A -> default rcode, SRV -> NODATA
    // reverse namespace
    K_PTR = 6,        // val = arena offset of {u8 wire_len, target name wire bytes} (:123-130)
    K_PTR_BAD = 7,    // ttl / target unusable: SERVFAIL
};

constexpr uint32_t NS_FORWARD = 0;
constexpr uint32_t NS_REVERSE = 1;
constexpr uint32_t KEY_INLINE_MAX = 20;
constexpr uint8_t  KLEN_OVERFLOW = 0xFF;      // key bytes live in the arena
constexpr uint8_t  SLOT_KEY_CLEAN = 1;
constexpr uint8_t  SLOT_DISPLACED = 2;        // a property of the POSITION, not of the resident: some key whose first slot is this
                                              // one lives in its second slot — only then does a lookup read a second slot

struct alignas(32) Slot {
    uint8_t  klen;       // key length 0..20 (0: the root domain's own key, which no query can spell), or KLEN_OVERFLOW
    uint8_t  kind;       // K_*
    uint8_t  ns;         // NS_*
    uint8_t  flags;      // SLOT_KEY_CLEAN: every label byte of a forward key is in [a-z0-9_-] (lib/server.js:208)
    uint32_t ttl;        // record ttl (lib/server.js:270-274)
    uint32_t val;        // IPv4 (network order bytes packed big-endian) or arena offset
    uint8_t  key[20];    // inline key, zero padded; overflow: key[0..3] = arena offset, [4..7] = length, [8..11] = hash
};
static_assert(sizeof(Slot) == 32, "slot must be one 32-byte sector");

// ---- service record in the arena (32-byte aligned) ---------------------------------------------------------
//   SvcHdr (32 B) | kid_info[nkids] (4 B each, padded to 16) | A answers (16 B per child) | KidRec (16 B per child) |
//   additional RRs (add_stride per child) | SRV answers (srv_stride per child) — every section in child order.
// Sizing a service answer is one header read unless a child is malformed or the answer must be truncated:
// the sums over the children that answer are taken at build time.  So are the resource records themselves:
// everything in an answer RR except the bytes of the question is known when the zone is built (the SRV target is
// the child's name + the service's own lower-cased fqdn — which the query's name equals, or it would not have hit —
// the ttls, the ports, the owner pointers), so each child carries its RRs as ready wire bytes and answering is
// copying them in shuffled child order (lib/server.js:361-416):
//   A answer       C00C | A IN | min(ttl, rttl) | 4 | addr                                             (:411-414)
//   additional     child labels | C0 ptr to the domain part of the QNAME | A IN | rttl | 4 | addr      (:401-402)
//   SRV answers    per port: C00C | SRV IN | ttl | rdlen | 0 | 10 | port | child labels | fqdn | 0     (:396-400)
// SECTIONS, not per-child blocks: an A query on a service reads header + kid_info + its children's 16-byte A answers —
// one or two 128-byte lines — instead of one sector out of every child's block; an SRV query reads the additional and the
// SRV sections, both dense.  kid_info (flags | wire_len << 8 | nports << 16 per child) sits next to the header so that one
// memory round trip tells how long every child's pieces are; their positions follow from the section strides, and the
// kernel turns an answer into a list of independent copy jobs (engine.cu) instead of walking the children one load after
// another.  A query whose domain part carries upper-case letters (the owner pointers then land elsewhere), a truncated
// answer or a malformed child take the field-by-field writer instead, which reads names and ports out of the same bytes.
// Every slot of the additional and SRV sections is padded with zeros up to its stride.
enum : uint8_t {
    SVC_BAD_A = 1,       // some child is "bad zk info" for an A query (:366-376): the walk must find where
    SVC_BAD_SRV = 2,     // same for SRV
    SVC_SP_NEVER = 4,    // s.srvce / s.proto absent, not strings, or not spellable as labels: never equal (:334-335)
    SVC_SP_EXT = 8,      // the two labels do not fit `sp`: sp[0..3] = arena offset of the bytes
};
// hflags >> 4: additional-section stride / 16.  A child is a znode path component and may contain dots, so its wire name is
// up to 255 - dom_wl <= 252 bytes (several labels) and its additional RR (wire name + 16) up to 268: a stride of 1..17 units.
// Four bits hold 1..15 as the count; 0 is never a count and stands for 17 (272 bytes), the stride of every child whose
// additional RR is over 240 bytes.
constexpr uint32_t SVC_ADD_STRIDE_SHIFT = 4;
constexpr uint32_t SVC_ADD_STRIDE_MAX = 272;
BB_HD uint32_t svc_add_stride(uint32_t hflags) {       // min(u - 1, 16) + 1 units: 0 wraps to 17 (an unsigned min, no branch)
    const uint32_t m = ((hflags & 0xFF) >> SVC_ADD_STRIDE_SHIFT) - 1u;
    return ((m < 16u ? m : 16u) + 1u) << 4;
}
BB_HD uint32_t svc_add_stride_bits(uint32_t stride) { return stride > 240 ? 0u : (stride >> 4) << SVC_ADD_STRIDE_SHIFT; }   // stride: 16..240 or 272
struct alignas(32) SvcHdr {
    uint32_t ttl;            // after record.ttl / service.ttl / service.service.ttl (:270-274,331-332)
    uint16_t nkids;          // children that pass the type filter (:352-360), in child order
    uint16_t n_valid;        // of those, the ones with an address (not KID_ADDR_NULL): one A / one additional each
    uint16_t sum_ports;      // sum of nports over them: SRV answers
    uint16_t sum_wl;         // sum of wire_len over them
    uint16_t sum_wl_ports;   // sum of nports * wire_len over them
    uint16_t jobs_srv;       // copy jobs of a whole SRV answer (resolve_device.cuh: a piece is ceil(len / 64) jobs), OPT not counted
    uint8_t  hflags;         // SVC_* | bytes per child of the additional section, encoded by svc_add_stride_bits
    uint8_t  sp_len;         // bytes of "_srvce._proto." on the wire = where the domain part of a matching SRV QNAME starts
    uint8_t  dom_wl;         // the service's fqdn as wire labels + terminator (what every SRV target ends with)
    uint8_t  sp[11];         // len, srvce bytes, len, proto bytes — as the query spells them
    uint16_t stride16;       // bytes per child of the SRV section / 16
};
static_assert(sizeof(SvcHdr) == 32, "service header is one sector");
enum : uint8_t {
    KID_BAD_A = 1,       // "bad zk info" when serving A        (:366-376 + contract)
    KID_BAD_SRV = 2,     // "bad zk info" when serving SRV
    KID_ADDR_NULL = 4,   // address === null -> skipped          (:378-381)
    KID_HAS_RTTL = 8,    // child carries its own ttl            (:389-393)
};
struct alignas(16) KidRec {
    uint32_t addr;           // IPv4 packed big-endian
    uint32_t rttl;
    uint8_t  flags;          // KID_*
    uint8_t  wire_len;       // child name as wire labels, no terminator (knode.name, :396)
    uint8_t  nports;         // SRV ports: krec[type].ports or [s.port]  (:383-385)
    uint8_t  pad;
    uint32_t pad2;
};
static_assert(sizeof(KidRec) == 16, "child record is one 16-byte load");
BB_HD uint32_t kid_add_len(uint32_t wire_len) { return wire_len + 16; }                            // additional RR
BB_HD uint32_t kid_srv_len(uint32_t wire_len, uint32_t dom_wl) { return 18 + wire_len + dom_wl; }  // one SRV answer RR
// offsets of the sections inside a record (every piece 16-byte aligned: they are streamed with 16-byte loads)
BB_HD uint32_t svc_a_off(uint32_t nkids) { return 32 + ((4 * nkids + 15) & ~15u); }               // A answers
BB_HD uint32_t svc_rec_off(uint32_t nkids) { return svc_a_off(nkids) + 16 * nkids; }                // KidRec
BB_HD uint32_t svc_add_off(uint32_t nkids) { return svc_rec_off(nkids) + 16 * nkids; }              // additional RRs
BB_HD uint32_t svc_srv_off(uint32_t nkids, uint32_t add_stride) { return svc_add_off(nkids) + add_stride * nkids; }      // SRV answers
BB_HD uint32_t svc_record_len(uint32_t nkids, uint32_t add_stride, uint32_t srv_stride) { return svc_srv_off(nkids, add_stride) + srv_stride * nkids; }

// ---- key hash: two independent multiply-fold accumulators over little-endian words, zero-padded tail -----
// (one IMAD.WIDE + one LOP3 per accumulator per word on the device)
BB_HD uint32_t fmix32(uint32_t h) {
    h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16; return h;
}
BB_HD uint32_t mulfold(uint32_t x, uint32_t k) { const uint64_t p = (uint64_t)x * k; return (uint32_t)p ^ (uint32_t)(p >> 32); }
BB_HD uint32_t hash_init(uint32_t ns) { return ns ? 0x52455631u : 0x42494E44u; }
BB_HD uint32_t hash_word(uint32_t h, uint32_t w) { return mulfold(h ^ w, 0x9E3779B1u); }
BB_HD uint32_t hash_finish(uint32_t h, uint32_t len) { return fmix32(h ^ len); }
// Second hash over the same words: it picks the key's second cuckoo slot, so two keys whose 32-bit
// hashes collide do not also share both of their slots.
BB_HD uint32_t hash2_init(uint32_t ns) { return ns ? 0x7F4A7C15u : 0x2545F491u; }
BB_HD uint32_t hash2_word(uint32_t g, uint32_t w) { return mulfold(g ^ w, 0x85EBCA77u); }
BB_HD uint32_t hash2_finish(uint32_t g, uint32_t len) { return fmix32(g + len * 0xC2B2AE3Du); }

// -> primary hash; *h2 = second hash
inline uint32_t hash_key2(uint32_t ns, const uint8_t* k, uint32_t len, uint32_t* h2) {
    uint32_t h = hash_init(ns), g = hash2_init(ns);
    uint32_t i = 0;
    for (; i + 4 <= len; i += 4) {
        const uint32_t w = (uint32_t)k[i] | (uint32_t)k[i + 1] << 8 | (uint32_t)k[i + 2] << 16 | (uint32_t)k[i + 3] << 24;
        h = hash_word(h, w); g = hash2_word(g, w);
    }
    if (i < len) {
        uint32_t w = 0;
        for (uint32_t j = 0; i + j < len; j++) w |= (uint32_t)k[i + j] << (8 * j);
        h = hash_word(h, w); g = hash2_word(g, w);
    }
    *h2 = hash2_finish(g, len);
    return hash_finish(h, len);
}
inline uint32_t hash_key(uint32_t ns, const uint8_t* k, uint32_t len) { uint32_t h2; return hash_key2(ns, k, len, &h2); }

// ---- cuckoo: the two slots a key may live in -------------------------------------------------
BB_HD uint32_t slot1_of(uint32_t key_hash, uint32_t mask) { return key_hash & mask; }
BB_HD uint32_t slot2_of(uint32_t key_hash, uint32_t key_hash2, uint32_t mask) {
    const uint32_t a = key_hash & mask, b = key_hash2 & mask;
    return b != a ? b : (a ^ 1u) & mask;
}

// ---- sharding: which rank owns a key (multi-GPU, SURVEY.md §8e) -------------------------------
// A second mix decorrelates the owner from the slot index (both derive from the key hash).
BB_HD uint32_t owner_of(uint32_t key_hash, uint32_t nranks) {
    return (uint32_t)(((uint64_t)fmix32(key_hash * 0x9E3779B1u + 0x7F4A7C15u) * nranks) >> 32);
}

// ---- shuffle RNG: the seeded stand-in for Math.random() at lib/server.js:46 ------------
BB_HD uint32_t shuffle_rand(uint64_t seed, uint32_t qidx, uint32_t i) {
    uint32_t lo = (uint32_t)seed, hi = (uint32_t)(seed >> 32);
    uint32_t r = fmix32(fmix32(fmix32(lo) ^ hi ^ (qidx * 0x9E3779B1u)) + i * 0x85EBCA77u);
    return (uint32_t)(((uint64_t)r * (i + 1)) >> 32);
}

// ---- per-engine constants (createServer options, lib/server.js:435-441) ----------------
constexpr uint32_t RF_MAX_DC = 16;
struct EngineConst {
    uint32_t suffix_len;         // strlen('.' + dnsDomain); 0 when dnsDomain === '' (:157)
    uint32_t soa_len;            // SOA rdata up to (not including) the trailing 5 x u32
    uint32_t recursion;          // options.recursion present (:110,222)
    uint32_t lean_ok;            // every dnsDomain byte is in [a-z0-9_.-]: the charset test of lib/server.js:208 can only fail in front of it
    uint8_t  suffix[256];        // '.' + dnsDomain, as query.name() would spell it
    uint8_t  soa[528];           // mname wire + rname wire of SOARecord(dnsDomain) (:286-287)
    uint8_t  wire_tail[256];     // dnsDomain as wire labels (no terminator), right-aligned: ends at wire_tail[256]
    // recursion pre-filter (lib/recursion.js:329-344; engaged when `recursion` == 2): which misses
    // Recursion.resolve() would forward at all
    uint32_t rf_dom_len;         // strlen(recursion's dnsDomain), compared case-sensitively as a string suffix
    uint32_t rf_ndc;             // datacenters with at least one upstream resolver that is not this host
    uint32_t rf_ptr;             // a PTR miss has somewhere to go (any such upstream in any datacenter)
    uint32_t rf_pad;
    uint8_t  rf_dom[256];        // that domain, dotted
    uint8_t  rf_dc_len[16];
    uint8_t  rf_dc[16][64];      // datacenter names (self.dcs keys), case-sensitive
    // upstream resolvers of the forward and match kernels (bb_engine_set_recursion_upstreams): what is left of self.dcs
    // after the own-address filter (lib/recursion.js:205-240,360-379); fu_dc[i] indexes rf_dc
    uint32_t fu_n;               // entries (0: no table)
    uint32_t fu_dcmask;          // bit d: datacenter d has at least one upstream
    uint32_t fu_ip[64];          // IPv4, host byte order (127.0.0.1 = 0x7F000001)
    uint16_t fu_port[64];
    uint8_t  fu_dc[64];
};
constexpr uint32_t FU_MAX = 64;

// ---- building the per-engine constants (host side; shared by the engine and the CPU emulation harness) ----
// dotted name -> wire labels without terminator; false if a label is empty or longer than 63 bytes
inline bool name_to_wire_labels(const char* s, size_t n, uint8_t* out, size_t cap, size_t* len) {
    size_t st = 0, w = 0;
    if (n == 0) return false;
    for (size_t i = 0; i <= n; i++) if (i == n || s[i] == '.') {
        const size_t l = i - st;
        if (l < 1 || l > 63 || w + 1 + l > cap) return false;
        out[w++] = (uint8_t)l;
        for (size_t k = 0; k < l; k++) out[w++] = (uint8_t)s[st + k];
        st = i + 1;
    }
    *len = w;
    return true;
}
// createServer options -> EngineConst (lib/server.js:435-441; SOARecord(dnsDomain) of :286-287: mname = dnsDomain,
// rname = hostmaster.<dnsDomain>, both uncompressed).  false: dns_domain is not a lower-case, encodable name.
inline bool make_engine_const(const char* dns_domain, bool recursion, EngineConst& C) {
    size_t n = 0; while (dns_domain[n]) ++n;
    for (size_t i = 0; i < n; i++) if (dns_domain[i] >= 'A' && dns_domain[i] <= 'Z') return false;
    uint8_t w[256], hw[300]; size_t wl = 0, hl = 0;
    char hm[300]; const char pre[] = "hostmaster.";
    if (n + sizeof pre > sizeof hm) return false;
    for (size_t i = 0; i < sizeof pre - 1; i++) hm[i] = pre[i];
    for (size_t i = 0; i < n; i++) hm[sizeof pre - 1 + i] = dns_domain[i];
    if (!name_to_wire_labels(dns_domain, n, w, sizeof w, &wl) || !name_to_wire_labels(hm, sizeof pre - 1 + n, hw, sizeof hw, &hl) || hl + 1 > 255)
        return false;
    C = EngineConst();
    unsigned char* z = (unsigned char*)&C; for (size_t i = 0; i < sizeof C; i++) z[i] = 0;
    C.suffix_len = (uint32_t)n + 1;
    C.suffix[0] = '.'; for (size_t i = 0; i < n; i++) C.suffix[1 + i] = (uint8_t)dns_domain[i];
    for (size_t i = 0; i < wl; i++) C.soa[i] = w[i];
    C.soa[wl] = 0;
    for (size_t i = 0; i < hl; i++) C.soa[wl + 1 + i] = hw[i];
    C.soa[wl + 1 + hl] = 0;
    C.soa_len = (uint32_t)(wl + 1 + hl + 1);
    for (size_t i = 0; i < wl; i++) C.wire_tail[256 - wl + i] = w[i];     // word-wise suffix gate compares the name's tail with this
    C.recursion = recursion ? 1 : 0;
    C.lean_ok = 1;
    for (size_t i = 0; i < n; i++) { const char c = dns_domain[i]; if (!((c >= 'a' && c <= 'z') || (c >= '0' && c <= '9') || c == '_' || c == '-' || c == '.')) C.lean_ok = 0; }
    return true;
}
inline void clear_upstreams_const(EngineConst& C) {
    C.fu_n = 0; C.fu_dcmask = 0;
    for (uint32_t i = 0; i < 64; i++) { C.fu_ip[i] = 0; C.fu_port[i] = 0; C.fu_dc[i] = 0; }
}
// lib/recursion.js:329-344 pre-filter fields (see bb_engine_set_recursion_filter).  false: bad arguments.
// Setting or removing the filter also clears the upstream table: its datacenter indices refer to the old list.
inline bool set_recursion_filter_const(EngineConst& C, const char* region_domain, const char* const* dc_names, uint32_t n_dc, bool ptr) {
    if (!region_domain) { if (C.recursion) C.recursion = 1; clear_upstreams_const(C); return true; }
    if (!C.recursion || n_dc > RF_MAX_DC || (n_dc && !dc_names)) return false;
    size_t L = 0; while (region_domain[L]) ++L;
    if (L > 255) return false;
    for (uint32_t k = 0; k < n_dc; k++) { size_t l = 0; if (dc_names[k]) while (dc_names[k][l]) ++l; if (l < 1 || l > 63) return false; }
    C.rf_dom_len = (uint32_t)L;
    for (size_t i = 0; i < sizeof C.rf_dom; i++) C.rf_dom[i] = i < L ? (uint8_t)region_domain[i] : 0;
    C.rf_ndc = n_dc;
    for (uint32_t k = 0; k < RF_MAX_DC; k++) {
        size_t l = 0; if (k < n_dc) while (dc_names[k][l]) ++l;
        C.rf_dc_len[k] = (uint8_t)l;
        for (size_t i = 0; i < 64; i++) C.rf_dc[k][i] = i < l ? (uint8_t)dc_names[k][i] : 0;
    }
    C.rf_ptr = ptr ? 1 : 0;
    C.recursion = 2;
    clear_upstreams_const(C);
    return true;
}
// bb_engine_set_recursion_upstreams: false on an engine without recursion, more than FU_MAX entries, or a dc[i] that
// is not in the filter's list.  n == 0 clears the table.
inline bool set_recursion_upstreams_const(EngineConst& C, const uint32_t* ip, const uint16_t* port, const uint8_t* dc, uint32_t n) {
    if (!C.recursion || n > FU_MAX || (n && (!ip || !port || !dc))) return false;
    for (uint32_t i = 0; i < n; i++) if (C.recursion != 2 || dc[i] >= C.rf_ndc) return false;
    C.fu_n = n; C.fu_dcmask = 0;
    for (uint32_t i = 0; i < FU_MAX; i++) {
        C.fu_ip[i] = i < n ? ip[i] : 0; C.fu_port[i] = i < n ? port[i] : 0; C.fu_dc[i] = i < n ? dc[i] : 0;
        if (i < n) C.fu_dcmask |= 1u << dc[i];
    }
    return true;
}

// host-side container of a built zone
struct ZoneImage {
    uint32_t  nslots;            // power of two
    Slot*     slots;             // malloc'd, 64-byte aligned
    uint8_t*  arena;
    uint64_t  arena_len;
    uint64_t  n_nodes, n_fwd, n_rev;
    int       ready;             // root domain node exists (lib/zk.js:55-58)
};

}  // namespace bb
#endif
