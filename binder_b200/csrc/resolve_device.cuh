// Per-query device code of the resolve path: decode, zkCache lookup, resolve()/resolvePtr() decisions, sizing and
// the response writers.  Included by engine.cu (the kernels and the host side of the C ABI); kept apart so that a
// host build can compile the same source against tests/native/cuda_shim.h (BB_HOST_EMU) and run it on the CPU.
#ifndef BB_RESOLVE_DEVICE_CUH
#define BB_RESOLVE_DEVICE_CUH

namespace bbk {
using namespace bb;

constexpr int T = 128;                    // queries (= threads) per tile
constexpr int S_IN = 8192;                // staged input bytes per tile
#ifndef BB_CAPW
#define BB_CAPW 12288
#endif
constexpr int CAPW = BB_CAPW;             // output staging window per flush round
constexpr int MAXRESP = 1232;             // >= the largest response (1200)
constexpr int S_OUT = ((CAPW + 32 + 127) / 128 + 1) * 128;   // whole 128-byte rows (the staging buffer is swizzled per row)
constexpr int WIN = CAPW - MAXRESP;        // output window of one emit round: a response STARTING in it ends inside the buffer
// copy jobs of a big tile (the service variant of the kernel): ONE list in tile-offset order (a thread's jobs sit at the
// exclusive prefix of the job counts, so the list is sorted by destination and every emit round owns a contiguous run
// of it); a response whose jobs do not fit is written whole by its thread
constexpr int TASKCAP = 1024;             // jobs = 8 KB of shared memory
constexpr int TASK_BYTES = 64;            // a job copies at most this much: four 16-byte chunks, all loaded before the first is written
constexpr int NROUNDS = 16;               // emit rounds of a big tile
static_assert(T * MAXRESP <= NROUNDS * (CAPW - MAXRESP), "a tile of maximal responses fits the rounds");
constexpr uint32_t NONE16 = 0xFFFF;

constexpr uint64_t D_FLAG_A = 1ull << 62, D_FLAG_P = 2ull << 62, D_VAL = (1ull << 62) - 1;
constexpr int D_MISS_SHIFT = 40;

enum { ST_ANSWERED = 0, ST_MISS = 1, ST_DROPPED = 2 };
enum { RC_NOERROR = 0, RC_SERVFAIL = 2, RC_NXDOMAIN = 3, RC_NOTIMP = 4, RC_REFUSED = 5 };
enum { QT_A = 1, QT_SOA = 6, QT_PTR = 12, QT_SRV = 33, QT_OPT = 41 };
enum { RK_NONE = 0, RK_HEADER = 1, RK_A1 = 2, RK_PTR = 3, RK_SOA = 4, RK_SVC_A = 5, RK_SVC_SRV = 6 };

// A tile kernel's placement state: desc[0, ntiles_cap) holds each tile's published prefix, desc[ntiles_cap] the arrival
// cursor, and the upper word of desc[ntiles_cap + 1] the finished-block counter; epoch is the launch number, which marks
// totals[2] (overflow) / totals[3] (done) of THIS launch.
struct Place {
    unsigned long long* desc;
    uint32_t ntiles_cap, epoch;
};

struct Params {
    const uint8_t* pkts; const uint32_t* pkt_off; uint32_t n;
    uint64_t seed; uint32_t qidx_base;
    uint8_t* out; uint32_t out_cap; uint32_t* out_off; uint16_t* out_len; uint8_t* status; uint32_t* miss_idx; uint32_t* totals;
    const Slot* table; uint32_t mask; const uint8_t* arena; int ready;
    const EngineConst* eng;
    Place place; uint32_t ntiles;
    unsigned long long* stage_log;   // optional [ntiles][8] globaltimer stamps (bb_engine_set_stage_log)
    const uint32_t* n_dev;           // when set, the batch size is read from device memory (routed batches)
    const uint32_t* qidx_map;        // when set, query i's shuffle index is qidx_map[i] (routed batches)
    uint32_t route, nranks, rank;    // route != 0: compute the owner rank of each query instead of probing
    uint32_t suffix_len, soa_len, recursion;   // copies of EngineConst scalars (constant bank instead of a global load)
    uint32_t lean_ok;        // dnsDomain is made of [a-z0-9_.-] only: a clean key hit proves the whole name passes lib/server.js:208
    uint32_t tcp;            // the batch arrived over TCP: no 512-byte / EDNS size limit (RFC 1035 4.2.2)
    uint32_t* fb;            // when set (pinned host memory): the last block also leaves {response bytes, queries, -, epoch} here — what the
                             // host picks the next batch's kernel variant from, without a copy or a synchronisation
    uint32_t* qidx_out;      // multi-region: each result's ingress index is also written here (host result mirrors)
    const uint32_t* err_in;  // multi-region: the shard's wait-timeout word, copied into totals[6]
    uint8_t* bounce;         // zero-copy results: device buffer (same offsets as `out`) that direct-emit tiles write to
                             // before copying their range to the host buffer with coalesced stores
    // multi-region launch (grid.y = regions): every per-batch pointer advances by its stride per region
    uint32_t regions;
    size_t in_stride, out_stride, off_stride, len_stride, status_stride, miss_stride, totals_stride, desc_stride;
};

// per-thread state carried from the sizing pass to the emit pass
struct Res {
    const uint8_t* p;        // packet bytes (shared memory, or global when the tile did not fit)
    uint32_t sp;             // shared-memory address of the packet (0 when not staged)
    uint32_t qn_len;         // QNAME wire length incl. terminator
    uint32_t ttl, val;
    uint64_t perm;           // shuffled child order, 4 bits each (nk <= 16)
    // one 32-bit register each: narrower fields cost a mask or a byte-permute at every write
    uint32_t rlen, maxsz, qtype, adv;
    uint32_t d_off, d_end;   // domain part [d_off, d_end) in QNAME wire coordinates
    uint32_t ptr_tgt;        // label boundary the owner's compression pointer targets, or NONE16
    uint32_t lastlen;        // position of the domain's last length byte
    uint32_t keep_ans, keep_add, n_walk, nk;
    uint32_t status, rk, rcode, tc, opcode, rd, edns, trunc;
    uint32_t owner;          // route mode: rank that owns this query's lookup key
    uint32_t ntask;          // != 0: a service answer that can be assembled from copy jobs (plan_service): header + question by this thread, the
                             // RRs by anyone.  It is 2 + n for n jobs (size_service counts them)
};

__device__ __forceinline__ uint32_t lower8(uint32_t c) { return (c - 'A' < 26u) ? c + 32 : c; }
__device__ __forceinline__ uint32_t be16(const uint8_t* p) { return (uint32_t)p[0] << 8 | p[1]; }
__device__ __forceinline__ uint32_t ld32(const uint8_t* p) { return *(const uint32_t*)p; }    // 4-byte aligned
__device__ __forceinline__ uint32_t ld16a(const uint8_t* p) { return *(const uint16_t*)p; }   // 2-byte aligned
#ifndef BB_HOST_EMU        /* the host emulation (tests/native/cuda_shim.h) supplies these over an emulated shared memory */
__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t lds8(uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ void sts32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void sts8(uint32_t a, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void sts_or(uint32_t a, uint32_t v) { asm volatile("red.shared.or.b32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
#endif

// byte-fed murmur (same result as bb::hash_key over the materialised key)
struct KeyHash {
    uint32_t h, g, acc, n;
    __device__ void init(uint32_t ns) { h = hash_init(ns); g = hash2_init(ns); acc = 0; n = 0; }
    __device__ void feed(uint32_t c) {
        acc |= c << (8 * (n & 3)); ++n;
        if ((n & 3) == 0) { h = hash_word(h, acc); g = hash2_word(g, acc); acc = 0; }
    }
    // -> primary hash; h2 = second hash (second cuckoo slot)
    __device__ uint32_t finish(uint32_t& h2) {
        if (n & 3) { h = hash_word(h, acc); g = hash2_word(g, acc); }
        h2 = hash2_finish(g, n);
        return hash_finish(h, n);
    }
};

// ---- mname decode (DESIGN.md "Wire spec: decode") ---------------------------------------
__device__ bool decode(const uint8_t* p, uint32_t len, Res& r) {
    if (len < 12) return false;
    if (p[2] & 0x80) return false;
    r.opcode = (p[2] >> 3) & 0xF; r.rd = p[2] & 1;
    uint32_t qd = be16(p + 4), an = be16(p + 6), ns = be16(p + 8), ar = be16(p + 10);
    if (qd != 1 || an != 0 || ns != 0 || ar > 1) return false;
    uint32_t pos = 12;
    for (;;) {
        if (pos >= len) return false;
        uint32_t c = p[pos];
        if (c == 0) { ++pos; break; }
        if (c > 63 || pos + 1 + c > len) return false;
        pos += 1 + c;
        if (pos - 12 + 1 > 255) return false;
    }
    r.qn_len = pos - 12;
    if (pos + 4 > len) return false;
    r.qtype = be16(p + pos);
    if (be16(p + pos + 2) != 1) return false;
    pos += 4;
    r.edns = 0; r.adv = 0;
    if (ar == 1) {
        if (pos + 11 > len || p[pos] != 0 || be16(p + pos + 1) != QT_OPT) return false;
        r.adv = be16(p + pos + 3);
        if (pos + 11 + be16(p + pos + 9) > len) return false;
        r.edns = 1;
    }
    return true;
}

// ---- zkCache.lookup / reverseLookup ------------------------------------------------------
// The key is produced twice (hash, then compare) by the same generator so that nothing is
// materialised.  Forward keys (zone_image.h): the wire labels in front of the dnsDomain suffix,
// lower-cased (length bytes are below 'A').  Reverse keys: the labels before "in-addr.arpa",
// reversed, joined by '.'.
struct FwdKey {
    const uint8_t* nm; uint32_t k0, k1;      // wire range [k0, k1) of the QNAME
    uint32_t pos;
    __device__ uint32_t length() const { return k1 - k0; }
    __device__ void start() { pos = k0; }
    __device__ uint32_t next() { return lower8(nm[pos++]); }
};
struct RevKey {
    const uint8_t* nm; uint32_t nlab;       // labels before in-addr.arpa
    uint32_t len_;
    int k; uint32_t pos, rem; bool dot;
    __device__ uint32_t label_pos(int idx) const { uint32_t q = 0; for (int i = 0; i < idx; i++) q += 1 + nm[q]; return q; }
    __device__ void measure() { len_ = 0; uint32_t q = 0; for (uint32_t i = 0; i < nlab; i++) { len_ += nm[q] + (i ? 1 : 0); q += 1 + nm[q]; } }
    __device__ uint32_t length() const { return len_; }
    __device__ void start() { k = (int)nlab - 1; dot = false; if (k >= 0) { pos = label_pos(k); rem = nm[pos]; ++pos; } }
    __device__ uint32_t next() {
        if (dot) { dot = false; return '.'; }
        uint32_t c = nm[pos++]; --rem;
        if (rem == 0 && k > 0) { --k; pos = label_pos(k); rem = nm[pos]; ++pos; dot = true; }
        return c;
    }
};

template <class KG>
__device__ bool probe(const Params& P, Res& r, uint32_t ns, KG& kg, uint32_t& kind, uint32_t& ttl, uint32_t& val) {
    uint32_t klen = kg.length();
    KeyHash kh; kh.init(ns);
    kg.start();
    for (uint32_t i = 0; i < klen; i++) kh.feed(kg.next());
    uint32_t h2;
    uint32_t h = kh.finish(h2);
    if (P.route) { r.owner = owner_of(h, P.nranks); return false; }   // sharding: who would answer
    // 2-choice cuckoo: the key is in slot1_of(h), or — only when that position says some key was displaced — in
    // slot2_of(h), or nowhere
    const uint32_t cand[2] = { slot1_of(h, P.mask), slot2_of(h, h2, P.mask) };
    for (int c = 0; c < 2; c++) {
        const Slot* s = P.table + cand[c];
        uint4 hd = __ldg((const uint4*)s);                  // klen,kind,ns,flags | ttl | val | key[0..3]
        const bool more = c == 0 && ((hd.x >> 24) & SLOT_DISPLACED);
        uint32_t sk = (hd.x >> 8) & 0xFF;
        if (sk != K_EMPTY && ((hd.x >> 16) & 0xFF) == ns) {
            uint32_t sl = hd.x & 0xFF;
            const uint8_t* kb = nullptr;
            if (sl == KLEN_OVERFLOW) {
                uint32_t off = hd.w, l = __ldg((const uint32_t*)(s->key + 4)), sh = __ldg((const uint32_t*)(s->key + 8));
                if (l == klen && sh == h) kb = P.arena + off;
            } else if (sl == klen) kb = s->key;
            if (kb) {
                kg.start();
                bool eq = true;
                for (uint32_t j = 0; j < klen; j++) if (__ldg(kb + j) != kg.next()) { eq = false; break; }
                if (eq) { kind = sk; ttl = hd.y; val = hd.z; return true; }
            }
        }
        if (!more) break;
    }
    return false;
}

// ---- shuffle (lib/server.js:40-53) --------------------------------------------------------
__device__ uint64_t make_perm(uint32_t n, uint64_t seed, uint32_t qidx) {     // n <= 16
    uint64_t perm = 0xFEDCBA9876543210ull;
    for (uint32_t i = n; i-- > 1;) {
        uint32_t j = shuffle_rand(seed, qidx, i);
        uint64_t x = ((perm >> (4 * i)) ^ (perm >> (4 * j))) & 15;
        perm ^= (x << (4 * i)) | (x << (4 * j));
    }
    return perm;
}
// element that ends up at position `p`, for any n: undo the swaps in reverse order
__device__ uint32_t perm_at_slow(uint32_t p, uint32_t n, uint64_t seed, uint32_t qidx) {
    uint32_t pos = p;
    for (uint32_t i = 1; i < n; i++) {
        uint32_t j = shuffle_rand(seed, qidx, i);
        if (pos == i) pos = j; else if (pos == j) pos = i;
    }
    return pos;
}
__device__ __forceinline__ uint32_t perm_at(const Res& r, uint32_t t, uint64_t seed, uint32_t qidx) {
    return r.nk <= 16 ? (uint32_t)(r.perm >> (4 * t)) & 15 : perm_at_slow(t, r.nk, seed, qidx);
}

// 16 bytes of a record that is read front to back (a service's header, child records and ready RRs): ask L2 to bring the
// surrounding 256 bytes in from DRAM.  The engine runs with sector-granular L2 fetches (bb_engine_create: a probe wants
// one 32-byte slot of a table far larger than L2), which would otherwise turn such a walk into one DRAM round trip per sector.
#if defined(BB_HOST_EMU)
static inline uint4 ldg_stream(const uint4* p) { return *p; }
#elif defined(BB_NO_STREAM_HINT)    /* experiment switch */
__device__ __forceinline__ uint4 ldg_stream(const uint4* p) { return __ldg(p); }
#else
__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
    uint4 v;
    asm volatile("ld.global.nc.L2::256B.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
#endif

// A service record in the arena (zone_image.h): 32-byte header, kid_info, then one section per kind of piece.
struct SvcView {
    const uint8_t* base; const uint8_t* arena;
    uint4 h0, h1;            // ttl | nkids,n_valid | sum_ports,sum_wl | sum_wl_ports,jobs_srv ; hflags,sp_len,dom_wl,sp[11],stride16
    __device__ void open(const uint8_t* arena_, uint32_t off) {
        arena = arena_; base = arena_ + off;
        h0 = ldg_stream((const uint4*)base); h1 = ldg_stream((const uint4*)base + 1);
#ifndef BB_HOST_EMU
        // kid_info follows the header: have its first sector (8 children) on the way while the header is still in flight
        asm volatile("prefetch.global.L1 [%0];" :: "l"(base + sizeof(SvcHdr)));
#endif
    }
    __device__ uint32_t ttl() const { return h0.x; }
    __device__ uint32_t nkids() const { return h0.y & 0xFFFF; }
    __device__ uint32_t n_valid() const { return h0.y >> 16; }
    __device__ uint32_t sum_ports() const { return h0.z & 0xFFFF; }
    __device__ uint32_t sum_wl() const { return h0.z >> 16; }
    __device__ uint32_t sum_wl_ports() const { return h0.w & 0xFFFF; }
    __device__ uint32_t jobs_srv() const { return h0.w >> 16; }
    __device__ uint32_t hflags() const { return h1.x & 0xFF; }
    __device__ uint32_t sp_len() const { return (h1.x >> 8) & 0xFF; }
    __device__ uint32_t dom_wl() const { return (h1.x >> 16) & 0xFF; }
    __device__ uint32_t srv_stride() const { return (h1.w >> 16) << 4; }
    __device__ uint32_t add_stride() const { return svc_add_stride(h1.x); }
    __device__ uint32_t a_off() const { return svc_a_off(nkids()); }
    __device__ uint32_t rec_off() const { return svc_rec_off(nkids()); }
    __device__ uint32_t add_off() const { return svc_add_off(nkids()); }
    __device__ uint32_t srv_off() const { return svc_srv_off(nkids(), add_stride()); }
    // flags | wire_len << 8 | nports << 16 of child i
    __device__ uint32_t info(uint32_t i) const { return __ldg((const uint32_t*)(base + sizeof(SvcHdr)) + i); }
    // byte i of "_srvce._proto." as wire labels
    __device__ uint32_t sp_byte(uint32_t i) const {
        if (hflags() & SVC_SP_EXT) { const uint32_t off = (h1.x >> 24) | (h1.y << 8); return __ldg(arena + off + i); }
        const uint32_t j = i + 3;                                   // sp starts at byte 3 of h1
        const uint32_t w = j < 4 ? h1.x : j < 8 ? h1.y : j < 12 ? h1.z : h1.w;
        return (w >> (8 * (j & 3))) & 0xFF;
    }
};
// One child's pieces: its KidRec and where its A answer, additional RR and SRV answers sit (the field-by-field paths read
// them through this).
struct KidView {
    uint4 a;                 // addr | rttl | flags,wire_len,nports,pad | -
    const uint8_t* a_; const uint8_t* add_; const uint8_t* srv_;
    uint32_t dwl;            // the service's dom_wl
    __device__ void load(const SvcView& sv, uint32_t i) {
        a = ldg_stream((const uint4*)(sv.base + sv.rec_off() + 16 * (size_t)i));
        a_ = sv.base + sv.a_off() + 16 * (size_t)i;
        add_ = sv.base + sv.add_off() + (size_t)sv.add_stride() * i;
        srv_ = sv.base + sv.srv_off() + (size_t)sv.srv_stride() * i;
        dwl = sv.dom_wl();
    }
    __device__ uint32_t addr() const { return a.x; }
    __device__ uint32_t rttl() const { return a.y; }
    __device__ uint32_t flags() const { return a.z & 0xFF; }
    __device__ uint32_t wire_len() const { return (a.z >> 8) & 0xFF; }
    __device__ uint32_t nports() const { return (a.z >> 16) & 0xFF; }
    __device__ const uint8_t* a_rr() const { return a_; }
    __device__ const uint8_t* add_rr() const { return add_; }                                      // starts with the child's labels
    __device__ const uint8_t* srv_rr() const { return srv_; }
    __device__ uint32_t srv_len() const { return kid_srv_len(wire_len(), dwl); }
    __device__ uint32_t port(uint32_t c) const { const uint8_t* p = srv_rr() + c * srv_len() + 16; return (uint32_t)__ldg(p) << 8 | __ldg(p + 1); }
    __device__ uint32_t name_byte(uint32_t i) const { return __ldg(add_rr() + i); }
};

// owner-name sizes for this query's domain part (DESIGN.md "Wire spec: compression")
__device__ __forceinline__ uint32_t dom_owner_len(const Res& r) {
    return r.ptr_tgt != NONE16 ? (uint32_t)(r.ptr_tgt - r.d_off) + 2 : (uint32_t)(r.d_end - r.d_off) + 1;
}
__device__ __forceinline__ uint32_t dom_wire_len(const Res& r) { return (uint32_t)(r.d_end - r.d_off) + 1; }

// One step of a walk over a service's children in sizing or planning.  Counted only by the host emulation built with
// -DBB_EMU_WALKS (tests/native/emu_service_jobs.cpp, tools/walk_counts.py).
#if defined(BB_HOST_EMU) && defined(BB_EMU_WALKS)
extern thread_local unsigned long long bb_emu_walk_steps;
#define BB_WALK_STEP() (++bb_emu_walk_steps)
#else
#define BB_WALK_STEP() ((void)0)
#endif

// copy jobs of a piece of `len` bytes (run_tasks copies at most TASK_BYTES per job)
__device__ __forceinline__ uint32_t piece_jobs(uint32_t len) { return (len + TASK_BYTES - 1) / TASK_BYTES; }

// Sizing of a service answer (lib/server.js:361-416).  When no child is malformed for this query type the
// sums taken at build time size it from the header alone; the children are walked (in shuffled order) only to
// find where a malformed child cuts the answer short, or which prefix of the RRs survives truncation.
// An answer that can be assembled from copy jobs (`jobs_ok`) leaves with its exact job count, r.ntask = 2 + jobs: the
// same pieces plan_service() makes, counted by the walk that sizes the answer, so that no second walk has to count them.
__device__ void size_service(const Params& P, Res& r, const SvcView& sv, uint32_t qidx, bool srv, uint32_t fixed) {
    const uint32_t nk = sv.nkids();
    r.nk = nk; r.ntask = 0;
    r.perm = nk <= 16 ? make_perm(nk, P.seed, qidx) : 0;
    const uint32_t dol = dom_owner_len(r), dwl = dom_wire_len(r);
    uint32_t ans_b = 0, add_b = 0, n_ans = 0, n_add = 0, n_walk = nk, jobs = 0;
    const uint32_t badbit = srv ? KID_BAD_SRV : KID_BAD_A;
    const bool sums = !(sv.hflags() & (srv ? SVC_BAD_SRV : SVC_BAD_A));
    // The answer is the header, the question and (a prefix of) the children's ready RRs: it can be assembled as
    // independent copy jobs (engine.cu) when the prebuilt owner pointers are this query's — no upper-case letter in its
    // domain part — whether or not it is truncated or cut short by a malformed child.
    const bool jobs_ok = nk <= 16 && r.ptr_tgt == r.d_off;
    if (sums) {
        // a whole answer's job count is a build-time sum too (an A answer is one 16-byte RR per child)
        if (srv) {
            n_ans = sv.sum_ports(); ans_b = n_ans * (18 + dwl) + sv.sum_wl_ports();
            n_add = sv.n_valid(); add_b = sv.sum_wl() + n_add * (dol + 14);
            jobs = sv.jobs_srv();
        } else { n_ans = sv.n_valid(); ans_b = n_ans * (dol + 14); jobs = n_ans; }
    } else {
        for (uint32_t t = 0; t < nk; t++) {
            BB_WALK_STEP();
            const uint32_t inf = sv.info(perm_at(r, t, P.seed, qidx)), fl = inf & 0xFF, wl = (inf >> 8) & 0xFF, np = (inf >> 16) & 0xFF;
            if (fl & badbit) { r.rcode = RC_SERVFAIL; n_walk = t; break; }      // :366-376
            if (fl & KID_ADDR_NULL) continue;                                    // :378-381
            if (srv) {
                const uint32_t a = np * (18 + wl + dwl), d = wl + dol + 14;
                ans_b += a; n_ans += np; add_b += d; n_add++; jobs += piece_jobs(a) + piece_jobs(d);
            } else { ans_b += dol + 14; n_ans++; jobs++; }
        }
    }
    r.n_walk = n_walk;
    const uint32_t opt_job = r.edns ? 1u : 0u;                                  // the OPT is a job of its own
    if (fixed + ans_b + add_b <= r.maxsz) {
        r.keep_ans = n_ans; r.keep_add = n_add; r.rlen = fixed + ans_b + add_b;
        if (jobs_ok && (n_ans + n_add) && r.rlen <= (uint32_t)MAXRESP) r.ntask = 2 + jobs + opt_job;
        return;
    }
    // Truncation: keep the longest prefix of [answers..., additionals...] that fits.  Whether all the answers fit is
    // known before the walk (fixed + ans_b), so ONE walk finds the cut: inside the answers (no additional survives), or
    // inside the additionals (an A answer has none, so that is SRV only).  Its job count is the kept answer RRs' —
    // every child's whole SRV run when the answers fit, which keeps a job-mode walk going past the additionals' cut.
    r.tc = 1;
    const bool ans_fit = fixed + ans_b <= r.maxsz;
    uint32_t total = ans_fit ? fixed + ans_b : fixed, ka = ans_fit ? n_ans : 0, kd = 0;
    bool add_cut = false;
    jobs = 0;
    for (uint32_t t = 0; t < n_walk; t++) {
        BB_WALK_STEP();
        const uint32_t inf = sv.info(perm_at(r, t, P.seed, qidx)), wl = (inf >> 8) & 0xFF, np = (inf >> 16) & 0xFF;
        if (inf & KID_ADDR_NULL) continue;
        const uint32_t each = srv ? 18 + wl + dwl : dol + 14, cnt = srv ? np : 1;
        if (!ans_fit) {
            uint32_t take = 0;                                                    // how many of this child's RRs still fit (cnt is 1..3 in practice:
            while (take < cnt && total + each <= r.maxsz) { total += each; ++take; }   // a compare per RR beats an integer division per child)
            ka += take; jobs += piece_jobs(take * each);
            if (take < cnt) break;
        } else {
            jobs += piece_jobs(cnt * each);
            const uint32_t d = wl + dol + 14;
            if (!add_cut && total + d <= r.maxsz) { total += d; ++kd; jobs += piece_jobs(d); }
            else if (!jobs_ok) break;
            else add_cut = true;
        }
    }
    r.keep_ans = ka; r.keep_add = kd; r.rlen = total;
    if (jobs_ok && (ka + kd) && total <= (uint32_t)MAXRESP) r.ntask = 2 + jobs + opt_job;
}

// one RR that either fits or is dropped (TC)
__device__ __forceinline__ void size_single(Res& r, uint32_t fixed, uint32_t rr) {
    if (fixed + rr <= r.maxsz) { r.rlen = (fixed + rr); r.keep_ans = 1; }
    else { r.rlen = fixed; r.keep_ans = 0; r.tc = 1; }
}

// Recursion.resolve()'s quick rejects (lib/recursion.js:329-344), for a miss that would otherwise be handed
// to the host: would it be forwarded anywhere?  nm = QNAME wire bytes — query.name() in its original case,
// SRV prefix included — W = its length without the terminator.  The dotted string is the wire bytes with each
// label boundary written as a '.', so the string operations map one to one onto wire positions; a '.' inside a
// label is a '.' of that string like any other (query.name() does not escape it), both in the suffix compare and
// as the start of dc:
//   domain.indexOf(dnsDomain, domain.length - dnsDomain.length) === -1            -> not ours   (:330-333)
//   p = domain minus the suffix and the one character before it; dc = p after its last '.';
//   self.dcs[dc] === undefined (or every upstream of dc is this host)              -> nowhere to ask (:338-343,377-379)
// rf_scan() is the scan itself: IDX -> the index of dc in the filter's list or -1 (rf_dc_index(), the forward kernel's
// route, forward_device.cuh); !IDX -> 1 or 0 (recursion_forwardable(), kept out of line: it runs for misses only and must
// not cost the hit path registers; this form compiles to the same instructions as the scan written with bool returns).
template <bool IDX>
__device__ __forceinline__ int rf_scan(const EngineConst* E, const uint8_t* nm, uint32_t W) {
    constexpr int NO = IDX ? -1 : 0;
    const uint32_t L = E->rf_dom_len;
    if (W < 1 + L) return NO;                          // name shorter than the suffix
    const uint32_t s0 = W - L;                         // wire index where the suffix must start
    if (s0 < 2) return NO;                             // nothing before it: dc = ''
    const uint32_t cw = s0 - 1;                        // the character substring() drops (normally the '.')
    uint32_t nlp = 1u + nm[0], last_b = 0;             // next length byte; last '.' of the dotted string before cw
    bool ok = true;
    for (uint32_t w = 1; w < W; w++) {
        const bool boundary = w == nlp;
        if (boundary) nlp = w + 1u + nm[w];
        if ((boundary || nm[w] == '.') && w < cw) last_b = w;
        if (w >= s0) ok &= E->rf_dom[w - s0] == (boundary ? (uint8_t)'.' : nm[w]);
    }
    if (!ok) return NO;
    const uint32_t d0 = last_b + 1, dl = cw - d0;      // dc = dotted[d0 .. cw)
    if (dl == 0 || dl > 63) return NO;
    for (uint32_t k = 0; k < E->rf_ndc; k++) {
        if (E->rf_dc_len[k] != dl) continue;
        bool eq = true;
        for (uint32_t i = 0; i < dl; i++) eq &= E->rf_dc[k][i] == nm[d0 + i];
        if (eq) return IDX ? (int)k : 1;
    }
    return NO;
}
__device__ __forceinline__ int rf_dc_index(const EngineConst* E, const uint8_t* nm, uint32_t W) { return rf_scan<true>(E, nm, W); }
__device__ __noinline__ bool recursion_forwardable(const EngineConst* E, const uint8_t* nm, uint32_t W) {
    return rf_scan<false>(E, nm, W) != 0;
}

// What resolve() does once zk.lookup() has answered (lib/server.js:219-424); shared by the
// generic and the word-wise front ends.
__device__ void finish_forward(const Params& P, Res& r, uint32_t qidx, uint32_t fixed, bool srv, bool hit,
                               uint32_t kind, uint32_t ttl, uint32_t val, uint32_t l0, uint32_t l1) {
    const uint8_t* nm = r.p + 12;
    const EngineConst* E = P.eng;
    if (!hit) {                                                               // :219-247
        if (P.recursion && r.rd) {
            // pre-filter: a miss recursion.js would refuse without asking anyone is refused here (same bytes)
            if (P.recursion == 2 && !recursion_forwardable(E, nm, r.qn_len - 1)) { r.rcode = RC_REFUSED; return; }
            r.status = ST_MISS; r.rk = RK_NONE; r.rlen = 0; return;
        }
        r.rcode = RC_REFUSED; return;
    }
    r.ttl = ttl; r.val = val;
    if (kind == K_INVALID) { r.rcode = RC_SERVFAIL; return; }                 // :251-260
    if (srv && kind != K_SERVICE) {                                           // :276-292 NODATA + SOA
        r.rcode = RC_NOERROR; r.rk = RK_SOA;
        uint32_t rr = dom_owner_len(r) + 10 + E->soa_len + 20;
        if (fixed + rr <= r.maxsz) { r.rlen = (fixed + rr); r.keep_ans = 1; }
        else { r.keep_ans = 0; r.tc = 1; }
        return;
    }
    if (kind == K_ADDR) { r.rcode = RC_NOERROR; r.rk = RK_A1; size_single(r, fixed, dom_owner_len(r) + 14); return; }
    if (kind == K_ADDR_BAD) { r.rcode = RC_SERVFAIL; return; }                // contract
    if (kind == K_UNKNOWN) { r.rcode = RC_NOTIMP; return; }                   // :419-424 + :346-350
    // K_SERVICE (:313-417)
    SvcView sv; sv.open(P.arena, val);
    r.ttl = sv.ttl();
    if (srv) {                                                                // :334-345: service === s.srvce && protocol === s.proto
        const uint32_t n = sv.sp_len();
        bool match = !(sv.hflags() & SVC_SP_NEVER) && n == l0 + l1 + 2;      // the two length bytes are part of the comparison
        if (match && r.sp && !(sv.hflags() & SVC_SP_EXT)) {
            // the 11 bytes of sp sit in the header's registers (bytes 3..13 of h1): three word compares against the QNAME's
            // first bytes, the last one masked to n
            const uint32_t a = r.sp + 12, b = a & ~3u, sh = (a & 3u) * 8;
            const uint32_t t0 = lds32(b), t1 = lds32(b + 4), t2 = lds32(b + 8), t3 = lds32(b + 12);
            const uint32_t q0 = __funnelshift_r(t0, t1, sh), q1 = __funnelshift_r(t1, t2, sh), q2 = __funnelshift_r(t2, t3, sh);
            const uint32_t s0 = __funnelshift_r(sv.h1.x, sv.h1.y, 24), s1 = __funnelshift_r(sv.h1.y, sv.h1.z, 24), s2 = __funnelshift_r(sv.h1.z, sv.h1.w, 24);
            const uint32_t m0 = n >= 4 ? 0xFFFFFFFFu : (1u << (8 * n)) - 1, m1 = n >= 8 ? 0xFFFFFFFFu : n > 4 ? (1u << (8 * (n - 4))) - 1 : 0u;
            const uint32_t m2 = n >= 12 ? 0xFFFFFFFFu : n > 8 ? (1u << (8 * (n - 8))) - 1 : 0u;
            match = (((q0 ^ s0) & m0) | ((q1 ^ s1) & m1) | ((q2 ^ s2) & m2)) == 0;
        } else
            for (uint32_t i = 0; match && i < n; i++) if (sv.sp_byte(i) != nm[i]) match = false;
        if (!match) { r.rcode = RC_NXDOMAIN; return; }
    }
    r.rcode = RC_NOERROR;                                                     // :351
    r.rk = srv ? RK_SVC_SRV : RK_SVC_A;
    size_service(P, r, sv, qidx, srv, fixed);
}

#ifndef BB_HOST_EMU
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#endif
// per-stage stamps of one tile, the batched analogue of query._stamp() (lib/server.js:479-483)
constexpr int NSTAGE = 16;
// Compiled in only with -DBB_STAGE_LOG (tools/stage_times.py builds such a library): eleven tests of a kernel parameter
// per query are ~5 % of the hot path's instructions.
#ifdef BB_STAGE_LOG
#define STAMP(k) do { if (P.stage_log && threadIdx.x == 0) P.stage_log[(size_t)blockIdx.x * NSTAGE + (k)] = gtime(); } while (0)
#else
#define STAMP(k) ((void)0)
#endif

// ---- word-wise front end of resolve() -----------------------------------------------------
// Same decisions as resolve_forward() below, four name bytes per step, for the common case:
// packet staged in shared memory, QNAME <= 64 wire bytes, lookup key <= 48 bytes (inline slot
// keys).  Anything else returns false and takes the generic path.
// unaligned 32-bit load from shared memory (the staging buffers carry read slack)
__device__ __forceinline__ uint32_t ldsu32(uint32_t a) {
    const uint32_t b = a & ~3u;
    return __funnelshift_r(lds32(b), lds32(b + 4), (a & 3u) * 8);
}
// v << n with PTX semantics: any n > 31 (including a wrapped-around negative) gives 0
#ifndef BB_HOST_EMU
__device__ __forceinline__ uint32_t shl_clamp(uint32_t v, uint32_t n) { uint32_t r; asm("shl.b32 %0, %1, %2;" : "=r"(r) : "r"(v), "r"(n)); return r; }
#endif
// 0x80 in every byte of v that is zero
__device__ __forceinline__ uint32_t zero_bytes(uint32_t v) { return ~(((v & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | v | 0x7F7F7F7Fu); }
// 0x80 in every byte of x7 (7-bit bytes) that is >= k
__device__ __forceinline__ uint32_t ge7(uint32_t x7, uint32_t k) { return (x7 + (0x80u - k) * 0x01010101u) & 0x80808080u; }
// 0x80 in every byte that is 'A'..'Z'
__device__ __forceinline__ uint32_t upper_bytes(uint32_t x) {
    const uint32_t x7 = x & 0x7F7F7F7Fu;
    return ge7(x7, 0x41) & ~ge7(x7, 0x5B) & ~x;
}

// Decode of a packet staged in shared memory, word-wise (same acceptance as decode()).
__device__ bool decode_staged(uint32_t sp, uint32_t len, Res& r) {
    if (len < 17) return false;                                               // header + root name + type/class at least
    const uint32_t hb = sp & ~3u, hs = (sp & 3u) * 8;
    const uint32_t t0 = lds32(hb), t1 = lds32(hb + 4), t2 = lds32(hb + 8), t3 = lds32(hb + 12);
    const uint32_t w0 = __funnelshift_r(t0, t1, hs), w1 = __funnelshift_r(t1, t2, hs), w2 = __funnelshift_r(t2, t3, hs);
    const uint32_t fl = (w0 >> 16) & 0xFF;                                    // byte 2: QR opcode AA TC RD
    if (fl & 0x80) return false;
    r.opcode = (fl >> 3) & 0xF; r.rd = fl & 1;
    if (w1 != 0x00000100u) return false;                                      // QDCOUNT=1, ANCOUNT=0
    if (w2 != 0u && w2 != 0x01000000u) return false;                          // NSCOUNT=0, ARCOUNT<=1
    const uint32_t nm = sp + 12, lim = len - 12;                              // name bytes available
    // label hop: one dependent shared-memory byte per label; validity is accumulated, not branched on
    uint32_t pos = 0, bad = 0, c = lds8(nm);
#pragma unroll 1
    while (c != 0) {
        bad |= c > 63;                                                        // pointers / extended label types
        pos += 1 + c;
        if (pos >= lim || pos > 254) { bad = 1; break; }
        c = lds8(nm + pos);
    }
    if (bad) return false;
    if (pos + 1 + 4 > lim) return false;
    r.qn_len = pos + 1;
    const uint32_t tc = ldsu32(nm + pos + 1);                                 // QTYPE, QCLASS (big-endian)
    r.qtype = (((tc & 0xFF) << 8) | ((tc >> 8) & 0xFF));
    if ((tc >> 16) != 0x0100u) return false;                                  // class IN
    r.edns = 0; r.adv = 0;
    if (w2) {
        const uint32_t q = nm + pos + 5;                                      // the one additional RR
        if (pos + 5 + 11 > lim) return false;
        const uint32_t a = ldsu32(q), b = ldsu32(q + 4), c2 = ldsu32(q + 8);
        if ((a & 0xFFFFFF) != 0x290000u) return false;                        // root owner, TYPE 41
        r.adv = (((a >> 24) << 8) | (b & 0xFF));
        const uint32_t rdlen = (((c2 >> 8) & 0xFF) << 8) | ((c2 >> 16) & 0xFF);
        if (pos + 5 + 11 + rdlen > lim) return false;
        r.edns = 1;
    }
    return true;
}

// 0x80 in every byte of the lower-cased dotted word `lo` that is NOT in [a-z0-9_-] ('.' counts as bad:
// the caller masks out the label-boundary positions)
__device__ __forceinline__ uint32_t bad_chars(uint32_t lo) {
    const uint32_t y7 = lo & 0x7F7F7F7Fu;
    const uint32_t ok = ((ge7(y7, 0x61) & ~ge7(y7, 0x7B)) | (ge7(y7, 0x30) & ~ge7(y7, 0x3A)) |
                         zero_bytes(lo ^ 0x2D2D2D2Du) | zero_bytes(lo ^ 0x5F5F5F5Fu)) & ~lo;
    return ~ok & 0x80808080u;
}

// Classification of a name the lean path could not settle with a clean hit, the way resolve() does before its
// lookup: a character outside [a-z0-9_.-] after toLowerCase (lib/server.js:207-215) or a '.' inside a label
// (DESIGN.md "in-label dots") -> bit 0; a line terminator in a label (the SRV regex's group 3 stops there, :141)
// -> bit 1.  Walks the labels of QNAME wire range [k0, k1) (already validated).  Out of line: it runs for misses
// and unusual keys only and must not cost the hit path registers.
__device__ __noinline__ uint32_t classify_labels(uint32_t nm, uint32_t k0, uint32_t k1) {
    uint32_t res = 0;
    for (uint32_t pos = k0; pos < k1;) {
        const uint32_t l = lds8(nm + pos); ++pos;
        for (uint32_t i = 0; i < l && pos < k1; i++, pos++) {
            const uint32_t c = lower8(lds8(nm + pos));
            if (!((c - 'a' < 26u) || (c - '0' < 10u) || c == '_' || c == '-')) res |= 1u;
            if (c == '\n' || c == '\r') res |= 2u;
        }
    }
    return res;
}
// Where the owner name's compression pointer may land when the domain carries upper-case letters: the first label
// boundary after the last upper-case byte of [k0, k1) — k1 (the start of the dnsDomain suffix, all lower case) at the latest.
__device__ __noinline__ uint32_t ptr_target_after_upper(uint32_t nm, uint32_t k0, uint32_t k1) {
    uint32_t tgt = k0;
    for (uint32_t pos = k0; pos < k1;) {
        const uint32_t l = lds8(nm + pos);
        bool up = false;
        for (uint32_t i = 1; i <= l; i++) { const uint32_t c = lds8(nm + pos + i); up |= (c - 'A' < 26u); }
        pos += 1 + l;
        if (up) tgt = pos;
    }
    return tgt;
}

// ---- the lean front end of onQuery/resolve() -------------------------------------------------------------
// The common shape, settled in one pass over the packet's words: a query staged in shared memory, QDCOUNT 1, no
// trailing bytes (ARCOUNT 0, or one bare OPT), QNAME <= 64 wire bytes that ENDS with dnsDomain's wire labels.
// Because the terminator's position follows from the packet length, the name is validated without hopping over
// every label: the bytes in front of the terminator must equal dnsDomain's labels (a word compare, which is also
// resolve()'s case-sensitive suffix gate, lib/server.js:157-166), and walking the labels in FRONT of them must
// land exactly on their first length byte.  Walking from the start is what decode() does, so a name accepted
// here is exactly the name decode() accepts (and its fields are the same); anything else returns 0 and takes the
// complete decoder and the generic path.  The lookup key is those front labels, lower-cased (zone_image.h).
// Returns 1 when r is complete (answer sized, or DROPPED), 0 when the caller must run the general path.
// RTCP: whether the batch arrived over TCP is `tcp`, not P.tcp (resolve_query).
template <bool RTCP>
__device__ int lean_query(const Params& P, Res& r, uint32_t len, uint32_t qidx, uint32_t s_sfx, uint32_t tcp) {
    const uint32_t sp = r.sp;
    if (len < 12 + 2 + 5) return 0;
    const uint32_t hb = sp & ~3u, hs = (sp & 3u) * 8;
    const uint32_t t0w = lds32(hb), t1w = lds32(hb + 4), t2w = lds32(hb + 8), t3w = lds32(hb + 12);
    const uint32_t w0 = __funnelshift_r(t0w, t1w, hs), w1 = __funnelshift_r(t1w, t2w, hs), w2 = __funnelshift_r(t2w, t3w, hs);
    const uint32_t fl = (w0 >> 16) & 0xFF;                                    // byte 2: QR opcode AA TC RD
    if ((fl & 0x80) || w1 != 0x00000100u || (w2 != 0u && w2 != 0x01000000u)) { r.status = ST_DROPPED; return 1; }   // as decode()
    r.opcode = (fl >> 3) & 0xF; r.rd = fl & 1;
    const uint32_t nm = sp + 12;
    uint32_t tail = 5;                                                        // terminator + QTYPE + QCLASS
    r.edns = 0; r.adv = 0;
    if (w2) {                                                                 // one additional RR: a bare OPT at the very end?
        if (len < 12 + 2 + 5 + 11) return 0;
        const uint32_t q = sp + len - 11;
        const uint32_t a = ldsu32(q), b = ldsu32(q + 4), c2 = ldsu32(q + 8);
        if ((a & 0xFFFFFFu) != 0x290000u) return 0;                           // root owner, TYPE 41
        if ((c2 >> 8) & 0xFFFFu) return 0;                                    // RDLEN != 0: options follow
        r.adv = (((a >> 24) << 8) | (b & 0xFF));
        r.edns = 1; tail = 16;
    }
    const uint32_t d_end = len - 12 - tail;                                   // where the terminator must be
    if (d_end > 63) return 0;
    const uint32_t tq = ldsu32(nm + d_end);                                   // 00 | QTYPE | QCLASS hi
    if ((tq & 0xFFu) != 0 || (tq >> 24) != 0 || lds8(nm + d_end + 4) != 1) return 0;
    const uint32_t qtype = ((tq >> 8) & 0xFF) << 8 | ((tq >> 16) & 0xFF);
    const bool srv = qtype == QT_SRV;
    // SRV: /^(_[^_.]*)[.](_[^_.]*)[.](.*)/ (:141-154) — the first two labels
    uint32_t d_off = 0, l0 = 0, l1 = 0;
    bool refuse = false;
    if (srv) {
        l0 = lds8(nm);
        if (l0 == 0 || l0 > 63 || 1 + l0 >= d_end) return 0;
        const uint32_t p1 = 1 + l0; l1 = lds8(nm + p1);
        if (l1 == 0 || l1 > 63 || p1 + 1 + l1 >= d_end) return 0;
        for (uint32_t i = 1; i <= l0; i++) { const uint32_t c = lds8(nm + i); refuse |= (i == 1) ? (c != '_') : (c == '_' || c == '.'); }
        for (uint32_t i = 1; i <= l1; i++) { const uint32_t c = lds8(nm + p1 + i); refuse |= (i == 1) ? (c != '_') : (c == '_' || c == '.'); }
        d_off = p1 + 1 + l1;
    }
    // the name must end with dnsDomain's labels, with at least one label in front of them
    const uint32_t sl = P.suffix_len;
    if (d_end < d_off + sl + 2) return 0;
    const uint32_t k1 = d_end - sl;                                           // the suffix's first length byte
    {
        uint32_t bad = 0;
        const uint32_t nw = (sl + 3) >> 2;
        // words right-aligned to the end of the name, from the end backwards; consecutive unaligned words share
        // their aligned halves (one LDS per word)
        const uint32_t ea = nm + d_end, eb = ea & ~3u, esh = (ea & 3u) * 8;
        uint32_t hi = lds32(eb);
        for (uint32_t j = 0; j < nw; j++) {
            const uint32_t lo = lds32(eb - 4 * (j + 1));
            const uint32_t x = __funnelshift_r(lo, hi, esh);                  // bytes [ea - 4(j+1), ea - 4j)
            hi = lo;
            const uint32_t e = lds32(s_sfx + 256 - 4 * (j + 1));
            const uint32_t rem = sl - 4 * j;                                  // bytes of this word that belong to the suffix
            const uint32_t cm = rem >= 4 ? 0xFFFFFFFFu : (0xFFFFFFFFu << (8 * (4 - rem)));
            bad |= (x ^ e) & cm;
        }
        if (bad) return 0;
    }
    {                                                                         // the labels in front: must land on k1
        uint32_t pos = d_off;
#pragma unroll 1
        while (pos < k1) { const uint32_t c = lds8(nm + pos); if (c == 0 || c > 63) return 0; pos += 1 + c; }
        if (pos != k1) return 0;
    }
    // ---- a valid query (what decode() returns for it) ----
    r.qn_len = d_end + 1; r.qtype = qtype;
    r.maxsz = (RTCP ? tcp : P.tcp) ? 65535 : r.edns ? min(max((uint32_t)r.adv, 512u), 1200u) : 512;
    const uint32_t fixed = 12 + r.qn_len + 4 + (r.edns ? 11 : 0);
    r.rk = RK_HEADER; r.rlen = fixed;
    if (r.opcode != 0 || !(qtype == QT_A || srv)) {
        if (r.opcode == 0 && qtype == QT_PTR) return 0;                       // resolvePtr: general path
        r.rcode = RC_NOTIMP; return 1;                                        // :500-505
    }
    if (!P.ready && !P.route) return 0;                // not-ready engines: exact ordering of refusals lives in the generic path
    STAMP(3);
    // lower-case + hash the key bytes [d_off, k1), four at a time (length bytes < 'A' pass through unchanged)
    const uint32_t pl = k1 - d_off;
    if (pl > 48) return 0;
    const uint32_t nwords = (pl + 3) >> 2;
    const uint32_t tailm = (pl & 3) ? ((1u << (8 * (pl & 3))) - 1) : 0xFFFFFFFFu;
    const uint32_t ka = nm + d_off, kb = ka & ~3u, ksh = (ka & 3u) * 8;
    uint32_t kw[5];
    uint32_t h = hash_init(NS_FORWARD), g = hash2_init(NS_FORWARD), anyup = 0;
    uint32_t wprev = lds32(kb);
#pragma unroll
    for (int i = 0; i < 5; i++) {
        kw[i] = 0;
        if ((uint32_t)i < nwords) {
            const uint32_t wnext = lds32(kb + 4 * (i + 1));
            uint32_t x = __funnelshift_r(wprev, wnext, ksh);
            wprev = wnext;
            if ((uint32_t)i == nwords - 1) x &= tailm;
            const uint32_t up = upper_bytes(x);
            anyup |= up;
            const uint32_t lo = x | (up >> 2);
            kw[i] = lo;
            h = hash_word(h, lo); g = hash2_word(g, lo);
        }
    }
#pragma unroll 1
    for (uint32_t i = 5; i < nwords; i++) {                                   // keys over 20 bytes (they live in the arena)
        const uint32_t wnext = lds32(kb + 4 * (i + 1));
        uint32_t x = __funnelshift_r(wprev, wnext, ksh);
        wprev = wnext;
        if (i == nwords - 1) x &= tailm;
        const uint32_t up = upper_bytes(x);
        anyup |= up;
        const uint32_t lo = x | (up >> 2);
        h = hash_word(h, lo); g = hash2_word(g, lo);
    }
    h = hash_finish(h, pl);
    const uint32_t h2 = hash2_finish(g, pl);
    STAMP(4);
    if (refuse) { r.rcode = RC_REFUSED; return 1; }
    if (P.route) { r.owner = owner_of(h, P.nranks); return 1; }      // sharding: who would answer
    r.d_off = d_off; r.d_end = d_end; r.trunc = 0; r.lastlen = d_off;
    r.ptr_tgt = anyup ? ptr_target_after_upper(nm, d_off, k1) : d_off;
    // zk.lookup(domain): the key's first slot — one 32-byte sector, one random DRAM access — and its second slot only
    // when the first position is flagged (some key was displaced from it): ~1.1 accesses per lookup, hit or miss
    uint32_t kind = 0, ttl = 0, val = 0;
    bool hit = false, clean = false;
    {
        const uint4* sa = (const uint4*)(P.table + slot1_of(h, P.mask));
        uint4 a0 = __ldg(sa), a1 = __ldg(sa + 1);
#pragma unroll 1
        for (int c = 0; c < 2; c++) {
            uint32_t da;
            if (pl <= KEY_INLINE_MAX) {
                // header: klen | kind | ns | flags; an empty slot has klen 0 and cannot equal `want` (pl >= 2)
                const uint32_t want = pl | (NS_FORWARD << 16);
                da = ((a0.x & 0x00FF00FFu) ^ want) | (kw[0] ^ a0.w) | (kw[1] ^ a1.x) | (kw[2] ^ a1.y) | (kw[3] ^ a1.z) | (kw[4] ^ a1.w);
            } else {
                // the slot names the key by arena offset, length and hash; the bytes are compared in the arena
                const uint32_t want = KLEN_OVERFLOW | (NS_FORWARD << 16);
                da = ((a0.x & 0x00FF00FFu) ^ want) | (a1.x ^ pl) | (a1.y ^ h);
                if (da == 0) {
                    const uint32_t* kp = (const uint32_t*)(P.arena + a0.w);                  // 4-byte aligned, zero padded
                    uint32_t wp2 = lds32(kb);
#pragma unroll 1
                    for (uint32_t i = 0; i < nwords; i++) {
                        const uint32_t wnext = lds32(kb + 4 * (i + 1));
                        uint32_t x = __funnelshift_r(wp2, wnext, ksh);
                        wp2 = wnext;
                        if (i == nwords - 1) x &= tailm;
                        x |= upper_bytes(x) >> 2;
                        uint32_t kwd = __ldg(kp + i);
                        if (i == nwords - 1) kwd &= tailm;
                        da |= x ^ kwd;
                    }
                }
            }
            if (da == 0) { hit = true; kind = (a0.x >> 8) & 0xFF; ttl = a0.y; val = a0.z; clean = (a0.x >> 24) & SLOT_KEY_CLEAN; break; }
            if (c || !((a0.x >> 24) & SLOT_DISPLACED)) break;
            const uint4* sb = (const uint4*)(P.table + slot2_of(h, h2, P.mask));
            a0 = __ldg(sb); a1 = __ldg(sb + 1);
        }
    }
    STAMP(5);
    if (!(hit && clean)) {
        // Not a clean hit: classify the name the way resolve() does before its lookup — a character outside
        // [a-z0-9_.-], a '.' inside a label -> REFUSED (:208-215); an SRV name with a line terminator goes to
        // the generic path (its regex group stops there, :141)
        const uint32_t cls = classify_labels(nm, d_off, k1);
        if (srv && (cls & 2u)) return 0;
        if (cls & 1u) { r.rcode = RC_REFUSED; return 1; }
    }
    finish_forward(P, r, qidx, fixed, srv, hit, kind, ttl, val, l0, l1);
    return 1;
}

// ---- resolve (lib/server.js:136-429) -------------------------------------------------------
__device__ void resolve_forward(const Params& P, Res& r, uint32_t qidx, uint32_t fixed) {
    const uint8_t* nm = r.p + 12;
    const EngineConst* E = P.eng;
    const bool srv = r.qtype == QT_SRV;
    uint32_t d_off = 0, d_end = r.qn_len - 1;
    uint32_t l0 = 0, l1 = 0;
    r.trunc = 0;
    if (srv) {
        // /^(_[^_.]*)[.](_[^_.]*)[.](.*)/ on query.name() (:141-154); labels hold no '.' here
        l0 = nm[0];
        if (l0 == 0 || nm[1] != '_') { r.rcode = RC_REFUSED; return; }
        for (uint32_t i = 2; i <= l0; i++) if (nm[i] == '_') { r.rcode = RC_REFUSED; return; }
        uint32_t p1 = 1 + l0; l1 = nm[p1];
        if (l1 == 0 || nm[p1 + 1] != '_') { r.rcode = RC_REFUSED; return; }
        for (uint32_t i = 2; i <= l1; i++) if (nm[p1 + i] == '_') { r.rcode = RC_REFUSED; return; }
        d_off = p1 + 1 + l1;
        if (nm[d_off] == 0) { r.rcode = RC_REFUSED; return; }                 // no third part
        // group 3 stops at the first \n or \r (JS '.' excludes line terminators, no '$')
        uint32_t nlp = d_off;
        for (uint32_t pos = d_off; pos < d_end; pos++) {
            if (pos == nlp) { nlp = pos + 1 + nm[pos]; continue; }
            if (nm[pos] == '\n' || nm[pos] == '\r') { d_end = pos; r.trunc = 1; break; }
        }
        if (d_end - d_off - 1 < 1 || d_end <= d_off + 1) { r.rcode = RC_REFUSED; return; }   // :144
    }
    r.d_off = d_off; r.d_end = d_end;
    if (d_end <= d_off + 1 && !srv) {                                         // root name: ''
        // isSuffix('.dom', '') is false -> refused; with no dnsDomain: length < 1 -> refused (:198)
        r.rcode = P.ready || E->suffix_len ? RC_REFUSED : RC_SERVFAIL; return;
    }
    // one pass over the domain in dotted view: suffix gate (:157-166, case-sensitive), charset
    // after toLowerCase (:207-215), and where an owner-name pointer may land
    const uint32_t dl = d_end - d_off - 1;
    const uint32_t sl = E->suffix_len;
    bool suffix_ok = sl == 0 || dl >= sl, charset_ok = true, need_b = false;
    uint32_t pos0 = d_end - sl, ptr_tgt = d_off, lastlen = d_off;
    {
        uint32_t nlp = d_off + 1 + nm[d_off];
        for (uint32_t pos = d_off + 1; pos < d_end; pos++) {
            uint32_t c, raw;
            if (pos == nlp) { raw = c = '.'; nlp = pos + 1 + nm[pos]; lastlen = pos; if (need_b) { ptr_tgt = pos; need_b = false; } }
            else {
                raw = nm[pos]; c = lower8(raw);
                if (raw != c) need_b = true;
                if (!((c - 'a' < 26u) || (c - '0' < 10u) || c == '_' || c == '-')) charset_ok = false;
            }
            if (suffix_ok && sl && pos >= pos0 && raw != E->suffix[pos - pos0]) suffix_ok = false;
        }
    }
    if (!suffix_ok) { r.rcode = RC_REFUSED; return; }
    if (!P.ready && !P.route) { r.rcode = RC_SERVFAIL; return; }             // :186-192
    if (!charset_ok) { r.rcode = RC_REFUSED; return; }
    r.ptr_tgt = (need_b || r.trunc) ? NONE16 : ptr_tgt;
    r.lastlen = lastlen;

    // the lookup key (zone_image.h): the labels in front of the suffix the gate has just matched
    FwdKey kg; kg.nm = nm; kg.k0 = d_off; kg.k1 = d_end - sl;
    uint32_t kind = 0, ttl = 0, val = 0;
    const bool hit = probe(P, r, NS_FORWARD, kg, kind, ttl, val);
    finish_forward(P, r, qidx, fixed, srv, hit, kind, ttl, val, l0, l1);
}

// ---- resolvePtr (lib/server.js:67-134) -----------------------------------------------------
__device__ void resolve_ptr(const Params& P, Res& r, uint32_t fixed) {
    const uint8_t* nm = r.p + 12;
    uint32_t nlab = 0, last = 0, prev = 0;
    for (uint32_t q = 0; nm[q]; q += 1 + nm[q]) { prev = last; last = q; ++nlab; }
    // parts.reverse(): [0] must be 'arpa', [1] 'in-addr' — case-sensitive (:71-78)
    bool ok = nlab >= 2 && nm[last] == 4 && nm[last + 1] == 'a' && nm[last + 2] == 'r' && nm[last + 3] == 'p' && nm[last + 4] == 'a' &&
              nm[prev] == 7 && nm[prev + 1] == 'i' && nm[prev + 2] == 'n' && nm[prev + 3] == '-' && nm[prev + 4] == 'a' &&
              nm[prev + 5] == 'd' && nm[prev + 6] == 'd' && nm[prev + 7] == 'r';
    if (!ok) { r.rcode = RC_REFUSED; return; }
    if (!P.ready && !P.route) { r.rcode = RC_SERVFAIL; return; }              // :86-92
    RevKey kg; kg.nm = nm; kg.nlab = nlab - 2; kg.measure();
    uint32_t kind = 0, ttl = 0, val = 0;
    bool hit = kg.length() > 0 && probe(P, r, NS_REVERSE, kg, kind, ttl, val);
    if (!hit) {                                                               // :107-121
        if (P.recursion && r.rd) {                                            // a PTR miss asks every datacenter (:346-354)
            if (P.recursion == 2 && !P.eng->rf_ptr) { r.rcode = RC_REFUSED; return; }
            r.status = ST_MISS; r.rk = RK_NONE; r.rlen = 0; return;
        }
        r.rcode = RC_REFUSED; return;
    }
    if (kind != K_PTR) { r.rcode = RC_SERVFAIL; return; }                     // contract
    r.ttl = ttl; r.val = val; r.rcode = RC_NOERROR; r.rk = RK_PTR;
    size_single(r, fixed, 2 + 10 + P.arena[val]);
}

// onQuery (lib/server.js:471-507) + sizing.  Leaves r ready for emit_response().
__device__ __forceinline__ void res_init(Res& r) {
    r.status = ST_ANSWERED; r.rk = RK_NONE; r.rlen = 0; r.tc = 0; r.keep_ans = r.keep_add = 0; r.nk = 0; r.n_walk = 0; r.ntask = 0;
    r.ptr_tgt = NONE16; r.trunc = 0; r.perm = 0; r.ttl = r.val = 0; r.d_off = r.d_end = r.lastlen = 0;
}
#ifdef BB_HOST_EMU        /* the CPU emulation counts which front end settled each query (tests/test_host_emulation.py) */
extern thread_local unsigned long long bb_emu_lean_count, bb_emu_general_count;
#define BB_EMU_COUNT(x) (++(x))
#else
#define BB_EMU_COUNT(x) ((void)0)
#endif
// RTCP (the multi-region kernel): whether the query arrived over TCP is `tcp`, the flag of its region's header, instead
// of the launch's P.tcp.  Every other caller keeps the constant-bank flag (and the code it compiled to).
template <bool RTCP = false>
__device__ void resolve_query(const Params& P, Res& r, uint32_t len, uint32_t qidx, uint32_t s_sfx, uint32_t tcp = 0) {
    res_init(r);
    if (r.sp && P.lean_ok && lean_query<RTCP>(P, r, len, qidx, s_sfx, tcp)) { BB_EMU_COUNT(bb_emu_lean_count); return; }
    BB_EMU_COUNT(bb_emu_general_count);
    res_init(r);
    if (!(r.sp ? decode_staged(r.sp, len, r) : decode(r.p, len, r))) { r.status = ST_DROPPED; return; }
    r.maxsz = (RTCP ? tcp : P.tcp) ? 65535 : r.edns ? min(max((uint32_t)r.adv, 512u), 1200u) : 512;
    const uint32_t fixed = 12 + r.qn_len + 4 + (r.edns ? 11 : 0);
    r.rk = RK_HEADER; r.rlen = fixed;
    const bool handled = r.opcode == 0 && (r.qtype == QT_A || r.qtype == QT_SRV || r.qtype == QT_PTR);
    if (!handled) { r.rcode = RC_NOTIMP; return; }                            // :500-505
    const uint8_t* nm = r.p + 12;
    for (uint32_t q = 0; nm[q];) {                                            // DESIGN.md "in-label dots"
        uint32_t l = nm[q];
        for (uint32_t i = 1; i <= l; i++) if (nm[q + i] == '.') { r.rcode = RC_REFUSED; return; }
        q += 1 + l;
    }
    if (r.qtype == QT_PTR) resolve_ptr(P, r, fixed);
    else resolve_forward(P, r, qidx, fixed);
}

// ---- mname encode (DESIGN.md "Wire spec: encode") ------------------------------------------
// OPT echoed when the query carried one: root owner, type 41, udp size 1200, ttl 0, rdlen 0
__constant__ uint8_t c_opt_rr[11] = { 0, 0, QT_OPT, 0x04, 0xB0, 0, 0, 0, 0, 0, 0 };
// The response staging buffer is XOR-swizzled: 16-byte chunk index ^ (128-byte row & 7).  With one
// 64-byte response per lane, word w of every lane would otherwise fall into 2 of the 32 banks (a
// 16-way conflict on every store); swizzled, a warp's stores spread over more banks, and the flush
// (consecutive 16-byte chunks) still reads each row as a permutation of itself.
__device__ __forceinline__ uint32_t swz(uint32_t off) { return off ^ (((off >> 7) & 7u) << 4); }

// byte emitter of the generic path: writes the response straight to its place in global memory
struct Out {
    uint8_t* o;
    __device__ void u8(uint32_t v) { *o++ = (uint8_t)v; }
    __device__ void u16(uint32_t v) { o[0] = (uint8_t)(v >> 8); o[1] = (uint8_t)v; o += 2; }
    __device__ void u32(uint32_t v) { o[0] = (uint8_t)(v >> 24); o[1] = (uint8_t)(v >> 16); o[2] = (uint8_t)(v >> 8); o[3] = (uint8_t)v; o += 4; }
    __device__ void copy(const uint8_t* s, uint32_t n) { for (uint32_t i = 0; i < n; i++) o[i] = s[i]; o += n; }
};
// the domain part, lower-cased, as wire labels up to `stop` (no terminator)
__device__ void put_dom_labels(Out& w, const Res& r, uint32_t stop) {
    const uint8_t* nm = r.p + 12;
    uint8_t* start = w.o;
    for (uint32_t pos = r.d_off; pos < stop; pos++) w.u8(lower8(nm[pos]));    // length bytes (<64) are unaffected
    if (r.trunc && stop > r.lastlen) start[r.lastlen - r.d_off] = (uint8_t)(r.d_end - r.lastlen - 1);
}
__device__ void put_dom_owner(Out& w, const Res& r) {
    if (r.ptr_tgt != NONE16) { put_dom_labels(w, r, r.ptr_tgt); w.u16(0xC000 | (12 + r.ptr_tgt)); }
    else { put_dom_labels(w, r, r.d_end); w.u8(0); }
}
__device__ void put_rr_head(Out& w, uint32_t type, uint32_t ttl, uint32_t rdlen) { w.u16(type); w.u16(1); w.u32(ttl); w.u16(rdlen); }

__device__ void emit_response(const Params& P, const Res& r, uint8_t* dst, uint32_t qidx) {
    Out w; w.o = dst;
    const uint8_t* p = r.p;
    uint32_t an = 0, ns = 0, ar = r.edns ? 1 : 0;
    switch (r.rk) {
    case RK_A1: case RK_PTR: an = r.keep_ans; break;
    case RK_SOA: ns = r.keep_ans; break;
    case RK_SVC_A: case RK_SVC_SRV: an = r.keep_ans; ar += r.keep_add; break;
    }
    w.u8(p[0]); w.u8(p[1]);
    w.u8(0x80 | (r.opcode << 3) | 0x04 | (r.tc ? 0x02 : 0) | r.rd);          // QR AA TC RD
    w.u8(r.rcode);                                                            // RA=0 Z=0
    w.u16(1); w.u16(an); w.u16(ns); w.u16(ar);
    w.copy(p + 12, r.qn_len + 4);                                             // question, verbatim
    const uint8_t* opt = c_opt_rr;
    bool opt_done = !r.edns;
    if (r.rk == RK_A1 && r.keep_ans) {                                        // :299,310
        put_dom_owner(w, r); put_rr_head(w, QT_A, r.ttl, 4); w.u32(r.val);
    } else if (r.rk == RK_PTR && r.keep_ans) {                                // :130
        w.u16(0xC00C); uint32_t tl = P.arena[r.val]; put_rr_head(w, QT_PTR, r.ttl, tl); w.copy(P.arena + r.val + 1, tl);
    } else if (r.rk == RK_SOA && r.keep_ans) {                                // :286-287
        const EngineConst* E = P.eng;
        put_dom_owner(w, r); put_rr_head(w, QT_SOA, r.ttl, E->soa_len + 20);
        w.copy(E->soa, E->soa_len); w.u32(0); w.u32(10); w.u32(10); w.u32(10); w.u32(r.ttl);
    } else if (r.rk == RK_SVC_A || r.rk == RK_SVC_SRV) {
        const bool srv = r.rk == RK_SVC_SRV;
        SvcView sv; sv.open(P.arena, r.val);
        uint32_t left = r.keep_ans;
        for (uint32_t t = 0; t < r.n_walk && left; t++) {
            KidView k; k.load(sv, perm_at(r, t, P.seed, qidx));
            if (k.flags() & KID_ADDR_NULL) continue;
            if (srv) {                                                        // :396-400
                const uint32_t np = k.nports(), wl = k.wire_len();
                for (uint32_t c = 0; c < np && left; c++, left--) {
                    w.u16(0xC00C); put_rr_head(w, QT_SRV, r.ttl, 6 + wl + dom_wire_len(r));
                    w.u16(0); w.u16(10); w.u16(k.port(c));
                    for (uint32_t i = 0; i < wl; i++) w.u8(k.name_byte(i));
                    put_dom_labels(w, r, r.d_end); w.u8(0);
                }
            } else {                                                          // :411-414
                uint32_t rttl = (k.flags() & KID_HAS_RTTL) ? k.rttl() : r.ttl;
                if (r.ttl < rttl) rttl = r.ttl;
                put_dom_owner(w, r); put_rr_head(w, QT_A, rttl, 4); w.u32(k.addr()); --left;
            }
        }
        if (srv) {
            if (!opt_done) { w.copy(opt, 11); opt_done = true; }
            left = r.keep_add;
            for (uint32_t t = 0; t < r.n_walk && left; t++) {                 // :401-402
                KidView k; k.load(sv, perm_at(r, t, P.seed, qidx));
                if (k.flags() & KID_ADDR_NULL) continue;
                const uint32_t wl = k.wire_len();
                uint32_t rttl = (k.flags() & KID_HAS_RTTL) ? k.rttl() : r.ttl;
                for (uint32_t i = 0; i < wl; i++) w.u8(k.name_byte(i));
                put_dom_owner(w, r); put_rr_head(w, QT_A, rttl, 4); w.u32(k.addr()); --left;
            }
        }
    }
    if (!opt_done) w.copy(opt, 11);
}

// ---- word-wise response writer -------------------------------------------------------------
// A byte stream into shared memory at an arbitrary byte address, stored as aligned 32-bit words;
// only the bytes shared with the neighbouring responses (first / last partial word) go out as
// single bytes, so two threads never write the same word.
// MODE 0: plain shared buffer, 1: XOR-swizzled shared staging (buffer 1024-byte aligned, so the
// swizzle applies to the address itself), 2: global memory (gbase + offset), 3: like 1 for a ZEROED buffer that
// copy jobs also fill (put16_or): single bytes — the words shared with a neighbouring piece — are OR-ed in; 4: like 3
// without the swizzle (the service variant's big tiles: lanes write pieces ~50 bytes apart, which spread over the banks by themselves).
// HEADCHK: any put may be the one that completes the first word.  Without it the stream must open
// with put4_first(), and every later store is a plain aligned word.
template <int MODE, bool HEADCHK = false>
struct WrT {
    uint32_t base;       // shared address of the buffer (mode 0)
    uint8_t* gbase;      // global destination (mode 2)
    uint32_t wp;         // position of the aligned word being filled: offset (modes 0, 2) or shared address (mode 1)
    uint32_t acc, fill;  // its bytes so far (fill = 0..3 of them)
    uint32_t head;       // bytes of the FIRST word that belong to the previous response (0..3)
    __device__ void begin(uint32_t buf, uint32_t off) {
        gbase = nullptr; head = off & 3u; acc = 0; fill = head;
        if (MODE == 1 || MODE == 3 || MODE == 4) { base = 0; wp = buf + off - head; } else { base = buf; wp = off - head; }
    }
    // global: `g` must be 4-byte aligned (the output buffer is 16-byte aligned), off = byte offset in it
    __device__ void begin_global(uint8_t* g, uint32_t off) { base = 0; gbase = g; head = off & 3u; wp = off - head; acc = 0; fill = head; }
    __device__ __forceinline__ void st32(uint32_t pos, uint32_t v) {
        if (MODE == 2) *(uint32_t*)(gbase + pos) = v;
        else if (MODE == 1 || MODE == 3) sts32(pos ^ ((pos >> 3) & 0x70u), v);
        else if (MODE == 4) sts32(pos, v);
        else sts32(base + pos, v);
    }
    __device__ __forceinline__ void st8(uint32_t pos, uint32_t v) {
        if (MODE == 2) gbase[pos] = (uint8_t)v;
        else if (MODE == 3) { const uint32_t a = pos & ~3u; sts_or(a ^ ((a >> 3) & 0x70u), (v & 0xFFu) << (8 * (pos & 3u))); }   // a word shared with a piece that is OR-ed in
        else if (MODE == 4) sts_or(pos & ~3u, (v & 0xFFu) << (8 * (pos & 3u)));
        else if (MODE == 1) sts8(pos ^ ((pos >> 3) & 0x70u), v & 0xFF);
        else sts8(base + pos, v & 0xFF);
    }
    __device__ __forceinline__ void store(uint32_t v) {
        if (HEADCHK && head) { for (uint32_t b = head; b < 4; b++) st8(wp + b, (v >> (8 * b)) & 0xFF); head = 0; }
        else st32(wp, v);
        wp += 4;
    }
    // the first four bytes of the stream: the only word that may be shared with the previous response
    __device__ __forceinline__ void put4_first(uint32_t v) {
        const uint32_t s8 = 8 * head, w = v << s8;
        if (head == 0) st32(wp, w);
        else for (uint32_t b = head; b < 4; b++) st8(wp + b, (w >> (8 * b)) & 0xFF);
        acc = __funnelshift_l(v, 0u, s8);
        wp += 4; head = 0;
    }
    // four bytes in memory order: the word being filled completes, `fill` bytes carry over
    __device__ __forceinline__ void put4(uint32_t v) {
        const uint32_t s8 = 8 * fill;
        store(acc | (v << s8));
        acc = __funnelshift_l(v, 0u, s8);                // v >> (32 - s8), 0 when s8 == 0
    }
    // v holds n (1..4) bytes in memory order (little-endian integer), upper bytes zero
    __device__ __forceinline__ void put(uint32_t v, uint32_t n) {
        const uint32_t s8 = 8 * fill;
        const uint32_t w = acc | (v << s8);
        if (fill + n >= 4) { store(w); acc = __funnelshift_l(v, 0u, s8); fill = fill + n - 4; }
        else { acc = w; fill += n; }
    }
    __device__ void end() { for (uint32_t b = head; b < fill; b++) st8(wp + b, (acc >> (8 * b)) & 0xFF); }
    // n bytes from shared memory (consecutive unaligned words share their aligned halves)
    __device__ void copy(uint32_t src, uint32_t n) {
        const uint32_t b = src & ~3u, sh = (src & 3u) * 8;
        if ((sh | fill) == 0 && !(HEADCHK && head)) {     // word-aligned on both sides: no shifting, no carry
            uint32_t i = 0;
            for (; i + 4 <= n; i += 4) { st32(wp, lds32(b + i)); wp += 4; }
            if (i < n) { acc = lds32(b + i) & ((1u << (8 * (n - i))) - 1); fill = n - i; }
            return;
        }
        uint32_t prev = lds32(b), i = 0, k = 1;
        for (; i + 4 <= n; i += 4, k++) { const uint32_t nx = lds32(b + 4 * k); put4(__funnelshift_r(prev, nx, sh)); prev = nx; }
        if (i < n) { const uint32_t nx = lds32(b + 4 * k); put(__funnelshift_r(prev, nx, sh) & ((1u << (8 * (n - i))) - 1), n - i); }
    }
};
__device__ __forceinline__ uint32_t bswap32(uint32_t v) { return __byte_perm(v, 0, 0x0123); }

// emit_response() with the word-wise writer, for every response shape of a packet staged in shared
// memory (everything except the SRV line-terminator quirk, which keeps the byte emitter).
__device__ __forceinline__ uint32_t bswap16(uint32_t v) { return ((v & 0xFF) << 8) | ((v >> 8) & 0xFF); }

// domain labels [d_off, stop) of the QNAME, lower-cased (length bytes < 64 are unaffected)
template <class W>
__device__ void put_dom_labels_w(W& w, const Res& r, uint32_t stop) {
    const uint32_t n = stop - r.d_off;
    const uint32_t src = r.sp + 12 + r.d_off, b = src & ~3u, sh = (src & 3u) * 8;
    uint32_t prev = lds32(b), i = 0, k = 1;
    for (; i < n; i += 4, k++) {
        const uint32_t nx = lds32(b + 4 * k);
        uint32_t x = __funnelshift_r(prev, nx, sh);
        prev = nx;
        x |= upper_bytes(x) >> 2;
        const uint32_t nb = n - i;
        if (nb >= 4) w.put4(x); else w.put(x & ((1u << (8 * nb)) - 1), nb);
    }
}
template <class W>
__device__ void put_dom_owner_w(W& w, const Res& r) {
    if (r.ptr_tgt != NONE16) {
        if (r.ptr_tgt != r.d_off) put_dom_labels_w(w, r, r.ptr_tgt);
        const uint32_t ptr = 0xC000u | (12u + r.ptr_tgt);
        w.put(bswap16(ptr), 2);
    } else { put_dom_labels_w(w, r, r.d_end); w.put(0, 1); }
}
template <class W>
__device__ __forceinline__ void put_global_bytes(W& w, const uint8_t* s, uint32_t n) {
    for (uint32_t i = 0; i < n; i++) w.put(__ldg(s + i), 1);
}

// up to 16 bytes held in registers into the stream
template <class W>
__device__ __forceinline__ void put_chunk_w(W& w, const uint4 x, uint32_t rem) {
    if (rem >= 16) { w.put4(x.x); w.put4(x.y); w.put4(x.z); w.put4(x.w); return; }
    if (rem >= 4) w.put4(x.x); else { w.put(x.x & ((1u << (8 * rem)) - 1), rem); return; }
    if (rem >= 8) w.put4(x.y); else { if (rem > 4) w.put(x.y & ((1u << (8 * (rem - 4))) - 1), rem - 4); return; }
    if (rem >= 12) w.put4(x.z); else { if (rem > 8) w.put(x.z & ((1u << (8 * (rem - 8))) - 1), rem - 8); return; }
    if (rem > 12) w.put(x.w & ((1u << (8 * (rem - 12))) - 1), rem - 12);
}
// n bytes from the arena (16-byte aligned source, readable up to the next multiple of 16) into the stream; up to four
// 16-byte loads are in flight before the first byte is written (one memory round trip per 64 bytes, not per 16)
template <class W>
__device__ __forceinline__ void copy_arena_w(W& w, const uint8_t* src, uint32_t n) {
    const uint4* q = (const uint4*)src;
#pragma unroll 1
    while (n) {
        const uint32_t m = n < 64 ? n : 64;
        const uint4 z = make_uint4(0, 0, 0, 0);
        const uint4 x0 = ldg_stream(q);
        const uint4 x1 = m > 16 ? ldg_stream(q + 1) : z;
        const uint4 x2 = m > 32 ? ldg_stream(q + 2) : z;
        const uint4 x3 = m > 48 ? ldg_stream(q + 3) : z;
        put_chunk_w(w, x0, m);
        if (m > 16) put_chunk_w(w, x1, m - 16);
        if (m > 32) put_chunk_w(w, x2, m - 32);
        if (m > 48) put_chunk_w(w, x3, m - 48);
        q += 4; n -= m;
    }
}

// ---- copy jobs: a service answer as independent pieces (engine.cu runs them, any thread any job) ---------------
// word 1: tile offset of the first byte (18 bits) | length 1..TASK_BYTES (7 bits) << 18 | source is a shared address << 25 |
// the source does not end in zero padding << 26 (a run of SRV answers cut short by truncation: its tail is masked)
struct Task { uint32_t src, w; };
__device__ __forceinline__ uint32_t task_word(uint32_t dst, uint32_t len, uint32_t sm, uint32_t exact) { return dst | (len << 18) | (sm << 25) | (exact << 26); }
__device__ __forceinline__ uint32_t task_dst(const Task& t) { return t.w & 0x3FFFFu; }
__device__ __forceinline__ uint32_t task_len(const Task& t) { return (t.w >> 18) & 0x7Fu; }
__device__ __forceinline__ bool task_smem(const Task& t) { return (t.w >> 25) & 1u; }
__device__ __forceinline__ bool task_exact(const Task& t) { return (t.w >> 26) & 1u; }
// The pieces of one job-mode response, given where the response starts in its tile: (a prefix of) the children's ready RRs
// in shuffled child order (lib/server.js:361-416) — the same walk as emit_fast's, counters included — and, for EDNS, the
// OPT (from `opt_sp`, a shared address holding its 11 bytes, zero padded to 16).  The header and the question are the
// owning thread's.  Every arena piece ends in zero padding up to the next multiple of 16 (zone_build.cpp pads each slot of
// the additional and SRV sections with zeros up to its stride) unless it is a run of SRV answers cut short (`exact`).
template <class Sink>
__device__ void plan_service(const Params& P, const Res& r, uint32_t qidx, uint32_t my_o, uint32_t opt_sp, Sink& sink) {
    const bool srv = r.rk == RK_SVC_SRV;
    SvcView sv; sv.open(P.arena, r.val);
    const uint32_t dwl = sv.dom_wl(), add_stride = sv.add_stride(), srv_stride = sv.srv_stride();
    const uint32_t a0 = r.val + sv.a_off(), add0 = r.val + sv.add_off(), srv0 = r.val + sv.srv_off();
    uint32_t dst = my_o + 12 + r.qn_len + 4;
    uint32_t left = r.keep_ans;
    uint64_t pm = r.perm;                                                     // job mode implies nk <= 16: four bits per position
    for (uint32_t t = 0; t < r.n_walk && left; t++, pm >>= 4) {
        BB_WALK_STEP();
        const uint32_t k = (uint32_t)pm & 15u, inf = sv.info(k);
        if (inf & KID_ADDR_NULL) continue;
        const uint32_t wl = (inf >> 8) & 0xFF, np = (inf >> 16) & 0xFF;
        if (srv) {
            const uint32_t n = min(np, left), len = n * kid_srv_len(wl, dwl);
            if (len) sink.put(srv0 + srv_stride * k, dst, len, 0, n < np);
            dst += len; left -= n;
        } else { sink.put(a0 + 16 * k, dst, 16, 0, 0); dst += 16; --left; }
    }
    if (r.edns) { sink.put(opt_sp, dst, 11, 1, 0); dst += 11; }               // the OPT leads the additional section
    if (srv) {
        left = r.keep_add; pm = r.perm;
        for (uint32_t t = 0; t < r.n_walk && left; t++, pm >>= 4) {
            BB_WALK_STEP();
            const uint32_t k = (uint32_t)pm & 15u, inf = sv.info(k);
            if (inf & KID_ADDR_NULL) continue;
            const uint32_t wl = (inf >> 8) & 0xFF;
            sink.put(add0 + add_stride * k, dst, kid_add_len(wl), 0, 0); dst += kid_add_len(wl); --left;
        }
    }
}
// a piece becomes ceil(len / TASK_BYTES) jobs (the kernel takes the count from size_service; the tests hold it to this walk)
struct TaskCount {
    uint32_t n;
    __device__ void put(uint32_t, uint32_t, uint32_t len, uint32_t, uint32_t) { n += piece_jobs(len); }
};
struct TaskFill {
    Task* tl;
    __device__ void put(uint32_t src, uint32_t dst, uint32_t len, uint32_t sm, uint32_t exact) {
        for (uint32_t off = 0; off < len; off += TASK_BYTES, tl++) {
            const uint32_t l = min((uint32_t)TASK_BYTES, len - off);
            tl->src = src + off; tl->w = task_word(dst + off, l, sm, exact && off + TASK_BYTES >= len);
        }
    }
};
// 16 bytes held in x to byte position pos of the (linear, zeroed) staging buffer: shifted into place over five words and
// OR-ed in, so a word shared with the neighbouring piece — some other thread's — needs no byte stores and no branches.
// Bytes of x beyond the piece must be zero (zero padding in the arena, or masked by the caller).
#ifndef BB_HOST_EMU
__device__ __forceinline__ void sts_or5(uint32_t base, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t w4) {
    asm volatile("{\n\t.reg .pred p0, p1, p2, p3, p4;\n\t"
                 "setp.ne.u32 p0, %1, 0;\n\tsetp.ne.u32 p1, %2, 0;\n\tsetp.ne.u32 p2, %3, 0;\n\tsetp.ne.u32 p3, %4, 0;\n\tsetp.ne.u32 p4, %5, 0;\n\t"
                 "@p0 red.shared.or.b32 [%0], %1;\n\t@p1 red.shared.or.b32 [%0+4], %2;\n\t@p2 red.shared.or.b32 [%0+8], %3;\n\t"
                 "@p3 red.shared.or.b32 [%0+12], %4;\n\t@p4 red.shared.or.b32 [%0+16], %5;\n\t}"
                 :: "r"(base), "r"(w0), "r"(w1), "r"(w2), "r"(w3), "r"(w4) : "memory");
}
#endif
__device__ __forceinline__ void put16_or(uint32_t pos, const uint4 x) {
    const uint32_t h = pos & 3u, s8 = 8 * h, base = pos - h;
    const uint32_t w0 = x.x << s8, w1 = __funnelshift_l(x.x, x.y, s8), w2 = __funnelshift_l(x.y, x.z, s8);
    const uint32_t w3 = __funnelshift_l(x.z, x.w, s8), w4 = __funnelshift_l(x.w, 0u, s8);
    sts_or5(base, w0, w1, w2, w3, w4);
}
// zero the bytes of x from byte nb (0..16) on
__device__ __forceinline__ uint4 keep_bytes(uint4 x, uint32_t nb) {
    x.x &= nb >= 4 ? 0xFFFFFFFFu : (1u << (8 * nb)) - 1;
    x.y &= nb >= 8 ? 0xFFFFFFFFu : nb > 4 ? (1u << (8 * (nb - 4))) - 1 : 0u;
    x.z &= nb >= 12 ? 0xFFFFFFFFu : nb > 8 ? (1u << (8 * (nb - 8))) - 1 : 0u;
    x.w &= nb >= 16 ? 0xFFFFFFFFu : nb > 12 ? (1u << (8 * (nb - 12))) - 1 : 0u;
    return x;
}
// Run the copy jobs [t0, t1) of one emit round into the staging buffer, a thread per job: up to four 16-byte loads, all
// issued before the first write (one memory round trip per job, and every job of the tile's round is in flight at once:
// the walk child by child that a thread per response would do is one dependent DRAM round trip after another), then the
// realigned writes.  Tile byte x lives at shared address delta + x.
__device__ __forceinline__ void run_tasks(const Params& P, const Task* tl, uint32_t t0, uint32_t t1, uint32_t tid, uint32_t delta) {
#pragma unroll 1
    for (uint32_t i = t0 + tid; i < t1; i += T) {
        const Task t = tl[i];
        const uint32_t len = task_len(t), pos = delta + task_dst(t);
        uint4 x0, x1 = make_uint4(0, 0, 0, 0), x2 = x1, x3 = x1;
        if (task_smem(t)) {                                                   // the OPT: one chunk
            x0.x = lds32(t.src); x0.y = lds32(t.src + 4); x0.z = lds32(t.src + 8); x0.w = lds32(t.src + 12);
        } else {
            const uint4* q = (const uint4*)(P.arena + t.src);
            x0 = ldg_stream(q);
            if (len > 16) x1 = ldg_stream(q + 1);
            if (len > 32) x2 = ldg_stream(q + 2);
            if (len > 48) x3 = ldg_stream(q + 3);
        }
        if (task_exact(t)) {                                                  // rare: the source runs on past the piece
            x0 = keep_bytes(x0, min(len, 16u)); x1 = keep_bytes(x1, len > 16 ? min(len - 16, 16u) : 0u);
            x2 = keep_bytes(x2, len > 32 ? min(len - 32, 16u) : 0u); x3 = keep_bytes(x3, len > 48 ? len - 48 : 0u);
        }
        put16_or(pos, x0);
        if (len > 16) put16_or(pos + 16, x1);
        if (len > 32) put16_or(pos + 32, x2);
        if (len > 48) put16_or(pos + 48, x3);
    }
}

// header + question (verbatim) of a response; the stream stays open
template <class W>
__device__ __forceinline__ void emit_head_w(const Res& r, W& w) {
    const uint32_t p = r.sp;
    uint32_t an = 0, ns = 0, ar = r.edns ? 1 : 0;
    switch (r.rk) {
    case RK_A1: case RK_PTR: an = r.keep_ans; break;
    case RK_SOA: ns = r.keep_ans; break;
    case RK_SVC_A: case RK_SVC_SRV: an = r.keep_ans; ar += r.keep_add; break;
    }
    const uint32_t flags = 0x80u | ((uint32_t)r.opcode << 3) | 0x04u | (r.tc ? 0x02u : 0u) | r.rd;
    w.put4_first((ldsu32(p) & 0xFFFFu) | (flags << 16) | ((uint32_t)r.rcode << 24));   // id, QR AA TC RD, rcode
    w.put4(0x00000100u | (bswap16(an) << 16));                                  // QDCOUNT=1, ANCOUNT
    w.put4(bswap16(ns) | (bswap16(ar) << 16));                                  // NSCOUNT, ARCOUNT
    w.copy(p + 12, r.qn_len + 4);                                               // question, verbatim
}

template <class W>
__device__ void emit_fast(const Params& P, const Res& r, W& w, uint32_t qidx) {
    emit_head_w(r, w);
    bool opt_done = !r.edns;
    if (r.rk == RK_A1 && r.keep_ans) {                                          // :299,310
        const uint32_t bt = bswap32(r.ttl);
        if (r.ptr_tgt == r.d_off) {              // owner is a bare pointer: the 16-byte RR as four whole words
            w.put4(bswap16(0xC000u | (12u + r.ptr_tgt)) | 0x01000000u);        // ptr | TYPE A ...
            w.put4(0x00000100u | (bt << 16));                                    // ... CLASS IN | ttl (high half)
            w.put4((bt >> 16) | 0x04000000u);                                    // ttl (low half) | RDLENGTH 4
            w.put4(bswap32(r.val));
        } else {
            put_dom_owner_w(w, r);
            w.put4(0x01000100u); w.put4(bt); w.put(0x0400u, 2); w.put4(bswap32(r.val));
        }
    } else if (r.rk == RK_PTR && r.keep_ans) {                                  // :130
        const uint32_t tl = P.arena[r.val];
        w.put(0x0CC0u, 2); w.put4(0x01000C00u); w.put4(bswap32(r.ttl)); w.put(bswap16(tl), 2);
        put_global_bytes(w, P.arena + r.val + 1, tl);
    } else if (r.rk == RK_SOA && r.keep_ans) {                                  // :286-287
        const EngineConst* E = P.eng;
        put_dom_owner_w(w, r);
        w.put4(0x01000600u); w.put4(bswap32(r.ttl)); w.put(bswap16(P.soa_len + 20), 2);
        put_global_bytes(w, E->soa, P.soa_len);
        w.put4(0); w.put4(bswap32(10)); w.put4(bswap32(10)); w.put4(bswap32(10)); w.put4(bswap32(r.ttl));
    } else if (r.rk == RK_SVC_A || r.rk == RK_SVC_SRV) {
        // The children's RRs are ready wire bytes in the service record (zone_image.h): answering is copying them in
        // shuffled child order.  SRV answers never depend on how the query is spelled; the A answers and the additional
        // RRs carry an owner pointer that is this query's only when its domain part has no upper-case letter
        // (`lower`) — otherwise they are written field by field.
        const bool srv = r.rk == RK_SVC_SRV;
        const bool lower = r.ptr_tgt == r.d_off;
        SvcView sv; sv.open(P.arena, r.val);
        uint32_t left = r.keep_ans;
        for (uint32_t t = 0; t < r.n_walk && left; t++) {
            KidView k; k.load(sv, perm_at(r, t, P.seed, qidx));
            const uint32_t fl = k.flags();
            if (fl & KID_ADDR_NULL) continue;
            if (srv) {                                                          // :396-400
                const uint32_t n = min(k.nports(), left);
                copy_arena_w(w, k.srv_rr(), n * k.srv_len());
                left -= n;
            } else if (lower) {                                                 // :411-414
                const uint4 x = ldg_stream((const uint4*)k.a_rr());
                w.put4(x.x); w.put4(x.y); w.put4(x.z); w.put4(x.w); --left;
            } else {
                uint32_t rttl = (fl & KID_HAS_RTTL) ? k.rttl() : r.ttl;
                if (r.ttl < rttl) rttl = r.ttl;
                put_dom_owner_w(w, r);
                w.put4(0x01000100u); w.put4(bswap32(rttl)); w.put(0x0400u, 2); w.put4(bswap32(k.addr())); --left;
            }
        }
        if (srv) {
            if (!opt_done) { w.put4(0x04290000u); w.put4(0x000000B0u); w.put(0, 3); opt_done = true; }
            left = r.keep_add;
            for (uint32_t t = 0; t < r.n_walk && left; t++) {                   // :401-402
                KidView k; k.load(sv, perm_at(r, t, P.seed, qidx));
                const uint32_t fl = k.flags();
                if (fl & KID_ADDR_NULL) continue;
                if (lower) copy_arena_w(w, k.add_rr(), kid_add_len(k.wire_len()));
                else {
                    const uint32_t rttl = (fl & KID_HAS_RTTL) ? k.rttl() : r.ttl;
                    copy_arena_w(w, k.add_rr(), k.wire_len());
                    put_dom_owner_w(w, r);
                    w.put4(0x01000100u); w.put4(bswap32(rttl)); w.put(0x0400u, 2); w.put4(bswap32(k.addr()));
                }
                --left;
            }
        }
    }
    if (!opt_done) { w.put4(0x04290000u); w.put4(0x000000B0u); w.put(0, 3); }   // OPT: 00 | 00 29 | 04 B0 | ttl 0 | rdlen 0
    w.end();
}

}  // namespace bbk

#endif
