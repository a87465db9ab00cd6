/*
 * binder_b200 — C ABI of the GPU-native (H100) DNS resolve engine.
 *
 * This is the drop-in boundary for ONE path of TritonDataCenter/binder: raw DNS query
 * packet -> parse -> zone-cache lookup -> answer wire bytes.  Each entry point names the
 * reference interface it replaces (paths relative to the reference tree).  Plain pointers
 * and sizes only; nothing here throws, allocates on behalf of the caller, or exposes torch
 * / CUDA types (a stream is passed as an opaque pointer).
 *
 * A Node.js host binds these through an N-API addon (addon/binder_b200_napi.cc,
 * INTEGRATION.md); the tests and bench bind them through ctypes.
 */
#ifndef BINDER_B200_H
#define BINDER_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BB_ABI_VERSION 1

/* ---- error codes (negative) ------------------------------------------------------- */
enum {
    BB_OK = 0,
    BB_ERR_ARG = -1,        /* null / out-of-range argument                              */
    BB_ERR_SNAPSHOT = -2,   /* snapshot is not valid JSON-lines                          */
    BB_ERR_CUDA = -3,       /* CUDA runtime error (bb_last_cuda_error has the text)      */
    BB_ERR_NOMEM = -4,      /* host or device allocation failed                          */
    BB_ERR_CAPACITY = -5,   /* out_cap too small for this batch's responses              */
    BB_ERR_NO_DEVICE = -6,  /* no CUDA device: there is NO CPU fallback                   */
    BB_ERR_DOMAIN = -7,     /* dns_domain is not an encodable DNS name                   */
    BB_ERR_PROTOCOL = -8    /* balancer frame stream: unknown type, INBOUND_TCP, oversized packet;
                               TCP hub session: a first frame other than INBOUND_TCP, a zero-length message */
};
const char* bb_strerror(int err);
const char* bb_last_cuda_error(void);
int bb_abi_version(void);

/* ---- per-query status, written to status[i] ---------------------------------------- */
enum {
    BB_ANSWERED = 0,        /* out[out_off[i] .. out_off[i+1]) is the response packet:
                               query.respond() was called (lib/server.js:75,...,427)      */
    BB_MISS_RECURSE = 1,    /* cache miss, RD set, recursion enabled: no bytes; index is in
                               miss_idx[] for options.recursion.resolve(query, cb)
                               (lib/server.js:110-113, 222-225)                           */
    BB_DROPPED = 2          /* not a decodable query (mname never emits 'query'): no bytes */
};

/* ---- zone: replaces the read side of lib/zk.js ZKCache ----------------------------- */
/*
 * An immutable, flattened image of the ZooKeeper subtree binder mirrors
 * (lib/zk.js:20-48 ZKCache, :78-119 TreeNode, :139-194 onDataChanged ingest):
 *   forward keys  = ca_treeNodes  (lower-cased fqdn  -> node)   lib/zk.js:62-64
 *   reverse keys  = ca_revLookup  (address string    -> node)   lib/zk.js:65-67
 * built from a snapshot: JSON lines {"path": "/com/foo/x", "data": <JSON.parse result>}
 * (or "raw": "<znode bytes>"), parents before children, children in ZK child order.
 * `dns_domain` is ZKCache's options.domain (main.js:158-162): the subtree root.
 */
typedef struct bb_zone bb_zone;
bb_zone* bb_zone_build(const char* snapshot_jsonl, size_t len, const char* dns_domain, int* err);
/* Shard `rank` of `nranks` of the same zone: only the keys this rank owns are inserted
 * (owner = owner_of(hash(key)), zone_image.h); a service's child list lives with the service. */
bb_zone* bb_zone_build_shard(const char* snapshot_jsonl, size_t len, const char* dns_domain,
                             uint32_t nranks, uint32_t rank, int* err);
void     bb_zone_free(bb_zone* z);
/* introspection: znodes mirrored (root included), forward keys, reverse keys, table bytes */
uint64_t bb_zone_stat(const bb_zone* z, int what);   /* what: 0 nodes 1 fwd 2 rev 3 slots 4 image bytes 5 arena bytes
                                                         6 slots changed since the device last saw the table 7 table laid out again
                                                         8 keys living in their second cuckoo slot (a lookup reads a second sector for these) */
/*
 * Watch events on a built zone (lib/zk.js:120-208), batched as JSON lines:
 *   {"path": P, "data": D} | {"path": P, "raw": "<znode bytes>"}   the znode now holds this content (dataChanged,
 *        :139-194: unparsable or non-object content is ignored and the previous data kept); a path not seen before is
 *        a new child appended to its parent's child list (childrenChanged, :120-130) — the parent must be mirrored
 *   {"path": P, "deleted": true}    the znode and its subtree are gone (childrenChanged -> unbind, :131-133,195-208;
 *        like the reference, a reverse-map entry the node registered is NOT removed)
 * Only what depends on the touched znodes is re-derived: the node's own key, the reverse entry of its address, its
 * parent's service record.  Superseded arena records are garbage until the table is laid out again (which happens
 * when they outweigh the live records, when the table fills past its load limit, or on a cuckoo failure).  Deviation: the
 * reference re-orders a node's children to ZooKeeper's list on every childrenChanged; here a new child goes last.
 * Returns BB_OK, or BB_ERR_SNAPSHOT for a line that is not a JSON object with a string "path" (earlier lines of
 * the delta stay applied).
 */
int bb_zone_apply(bb_zone* z, const char* delta_jsonl, size_t len);
/* Diagnostics (host side): what the image holds for a key.  ns 0 = forward (lower-cased fqdn), 1 = reverse (address
 * string).  rec = the payload in a position-independent form (service header, srvce, proto, every child record;
 * PTR target as wire labels).  Returns 1 when the key is present. */
int bb_zone_probe(const bb_zone* z, uint32_t ns, const uint8_t* key, uint32_t len, uint8_t* kind, uint32_t* ttl,
                  uint32_t* val, uint8_t* rec, uint32_t rec_cap, uint32_t* rec_len);

/* ---- engine: replaces lib/server.js createServer()'s query handler ----------------- */
/*
 * Options mirror createServer(options) (lib/server.js:435-441, main.js:204-214):
 *   dns_domain       options.dnsDomain        (suffix gate, SOA host)  lib/server.js:157-166,286
 *   datacenter_name  options.datacenterName   (only read by dead code, lib/server.js:167-175)
 *   recursion        options.recursion != null (miss hand-off)          lib/server.js:110,222
 *   device           CUDA device ordinal
 */
typedef struct bb_engine bb_engine;
typedef struct bb_engine_opts {
    const char* dns_domain;
    const char* datacenter_name;
    int32_t     recursion;
    int32_t     device;
    uint32_t    max_batch;       /* largest n per call (0 -> 1<<20)                      */
    uint32_t    max_batch_bytes; /* largest packed query bytes per call (0 -> 64*max_batch) */
    int32_t     ordered_output;  /* 0: "arrival" packing — responses packed in the order tiles of
                                    128 queries finish (fastest; layout varies run to run, each
                                    response's bytes do not).  1: packed in query order, out_off
                                    monotonic, miss_idx ascending (tiles wait for predecessors). */
} bb_engine_opts;

bb_engine* bb_engine_create(const bb_engine_opts* opts, int* err);
void       bb_engine_destroy(bb_engine* e);

/*
 * Publish a zone (the "ZK session established / watcher fired" analogue,
 * lib/zk.js:45-47,68-76).  Uploads the image to HBM and swaps it in; batches submitted
 * afterwards see the new zone.  Until the first swap the engine is "not ready" and A / SRV /
 * PTR queries that pass the early refusals are answered SERVFAIL (lib/server.js:86-92,186-192).
 * The engine keeps its own device copy; the caller may free `z` afterwards.
 */
int bb_engine_swap_zone(bb_engine* e, const bb_zone* z);
/* After bb_zone_apply: ship only what changed (the touched 32-byte slots, scattered by a small kernel, and the arena
 * tail) instead of the whole image; batches in flight finish on the old state first.  Falls back to a full swap when
 * the table had to be laid out again, the arena outgrew its device allocation, or another engine took the zone's
 * previous changes (a zone feeds ONE engine incrementally). */
int bb_engine_apply_update(bb_engine* e, bb_zone* z);
/*
 * Recursion pre-filter (SURVEY.md section 8f row 3).  Recursion.resolve() (lib/recursion.js:285-388) refuses a
 * handed-off miss without asking anyone when the name is outside its dnsDomain (:330-333), when the label in front
 * of that suffix is not a datacenter it knows (:338-343), or when every upstream of that datacenter is this host
 * itself (:360-379).  With a filter set, the kernel evaluates those string operations on query.name() exactly as
 * the reference does and answers such misses REFUSED itself (the same bytes recursion.js would send); only misses
 * that have somewhere to go enter miss_idx.
 *   region_domain     Recursion's opts.dnsDomain (case-sensitive string suffix; NULL removes the filter)
 *   dc_names[n_dc]    keys of self.dcs that keep at least one upstream after the own-address filter (n_dc <= 16)
 *   ptr_forwardable   any such upstream exists (a PTR miss asks every datacenter, :346-354)
 * The host refreshes it whenever lib/recursion.js refreshes self.dcs (:205-240).  Requires opts.recursion.
 */
int bb_engine_set_recursion_filter(bb_engine* e, const char* region_domain, const char* const* dc_names,
                                   uint32_t n_dc, int ptr_forwardable);
int bb_engine_is_ready(const bb_engine* e);          /* zkCache.isReady(), lib/zk.js:55-58 */
/* Two variants of the resolve kernel answer every batch identically: one sized for short answers (6 tiles of 128 queries
 * per SM) and one for long service answers (copy jobs and emit rounds in shared memory, 5 tiles per SM).  0 (default): chosen
 * per batch from the mean response size of the latest batch whose totals are known; 1: always the first; 2: always the second. */
int bb_engine_set_kernel_profile(bb_engine* e, int profile);
uint32_t bb_engine_max_batch(const bb_engine* e);        /* the limits the engine was created with */
uint32_t bb_engine_max_batch_bytes(const bb_engine* e);

/*
 * Resolve one batch of raw DNS query packets held in HOST memory: the batched form of
 * mname's 'query' event -> onQuery(query, cb) (lib/server.js:471-507) -> resolve /
 * resolvePtr (lib/server.js:67-429) -> query.respond().
 *
 *   pkts, pkt_off[n+1]   packed packets; packet i = pkts[pkt_off[i] .. pkt_off[i+1])
 *   shuffle_seed         seeds the service-answer shuffle (lib/server.js:40-53, Math.random
 *                        replaced by a counter RNG keyed on (seed, qidx_base + i))
 *   out, out_cap         response bytes, packed (no gaps; see ordered_output)
 *   out_off[n+1]         response i = out[out_off[i] .. out_off[i] + out_len[i]); out_off[n] = total bytes
 *   out_len[n]           response length, 0 unless ANSWERED
 *   status[n]            BB_ANSWERED / BB_MISS_RECURSE / BB_DROPPED
 *   miss_idx[n], n_miss  indices of the BB_MISS_RECURSE queries (ascending when ordered_output)
 *
 * Host<->device copies happen inside the call (pinned buffers from bb_host_alloc make
 * them asynchronous DMA).  Returns BB_OK or a negative error; never partial results.
 */
int bb_resolve_batch(bb_engine* e, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n,
                     uint64_t shuffle_seed, uint32_t qidx_base,
                     uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status,
                     uint32_t* miss_idx, uint32_t* n_miss);

/*
 * Pipelined form of bb_resolve_batch: up to bb_engine_slots() batches in flight, each on
 * its own stream (H2D, kernel and D2H of different batches overlap).  submit() returns at
 * once; wait() blocks until that slot's results are in the caller's buffers.
 */
int bb_engine_slots(const bb_engine* e);
int bb_resolve_submit(bb_engine* e, int slot, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n,
                      uint64_t shuffle_seed, uint32_t qidx_base,
                      uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status,
                      uint32_t* miss_idx, uint32_t* n_miss);
int bb_resolve_wait(bb_engine* e, int slot);

/*
 * Batches that arrived over TCP (mname's listenTcp, lib/server.js:643-652; RFC 1035 4.2.2 two-byte length framing is
 * the host's job — binder_b200/server.py mirrors it): flags = BB_BATCH_TCP lifts the 512-byte / EDNS size limit, a
 * response may be up to 65,535 bytes and is truncated (TC) only beyond that.  flags = 0 is bb_resolve_batch/submit.
 * out_cap must allow for the larger answers (BB_ERR_CAPACITY otherwise; the engine's own staging holds 512 bytes
 * per query of max_batch on average).
 */
#define BB_BATCH_TCP 1u
int bb_resolve_batch_ex(bb_engine* e, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n,
                        uint64_t shuffle_seed, uint32_t qidx_base,
                        uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status,
                        uint32_t* miss_idx, uint32_t* n_miss, uint32_t flags);
int bb_resolve_submit_ex(bb_engine* e, int slot, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n,
                         uint64_t shuffle_seed, uint32_t qidx_base,
                         uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status,
                         uint32_t* miss_idx, uint32_t* n_miss, uint32_t flags);

/*
 * Device-resident form (inputs and outputs already in HBM; used for kernel-only timing and
 * by the multi-GPU router).  All pointers are device pointers; d_pkts must be 16-byte
 * aligned and readable up to the next multiple of 16 past pkt_off[n]; d_out must be 16-byte
 * aligned.  d_totals[4] receives {total response bytes, n_miss, overflow marker, done
 * marker}: the markers equal bb_engine_launch_epoch() of this call when set (out_cap too
 * small / launch finished).  Launches on up to 16 distinct streams may overlap; launches on one
 * stream run in order.  `stream` is a cudaStream_t (NULL = default
 * stream).  Asynchronous: returns after the launch.
 */
int bb_resolve_batch_device(bb_engine* e, const uint8_t* d_pkts, const uint32_t* d_pkt_off, uint32_t n,
                            uint64_t shuffle_seed, uint32_t qidx_base,
                            uint8_t* d_out, uint32_t out_cap, uint32_t* d_out_off, uint16_t* d_out_len, uint8_t* d_status,
                            uint32_t* d_miss_idx, uint32_t* d_totals, void* stream);
/*
 * bb_resolve_batch_device for batches that arrived over TCP: flags = BB_BATCH_TCP lifts the 512-byte / EDNS size limit
 * exactly as in bb_resolve_batch_ex (a response up to 65,535 bytes, TC only beyond that; out_cap must allow for the larger
 * answers, else the overflow marker is set).  Other bits are ignored; flags = 0 is bb_resolve_batch_device.
 */
int bb_resolve_batch_device_ex(bb_engine* e, const uint8_t* d_pkts, const uint32_t* d_pkt_off, uint32_t n,
                               uint64_t shuffle_seed, uint32_t qidx_base,
                               uint8_t* d_out, uint32_t out_cap, uint32_t* d_out_off, uint16_t* d_out_len, uint8_t* d_status,
                               uint32_t* d_miss_idx, uint32_t* d_totals, void* stream, uint32_t flags);

/*
 * Recursion relay: the reply binder sends for a forwarded miss, built from the upstream resolver's response.
 * Replaces the reply construction of Recursion.prototype.resolve (lib/recursion.js:287-327): the upstream's answer RRs
 * of type A, AAAA, TXT, PTR, CNAME and SRV with class IN are re-wrapped with owner query.name() and the upstream's TTL
 * (names in RDATA decompressed, SRV with the upstream's priority, weight and port); other types and classes are dropped
 * (:316-320).  A failed lookup — an empty upstream (up_off[i] == up_off[i+1]), one that is malformed, or one without
 * answer RRs — gives REFUSED; answers that are all dropped give NOTIMP (respond() neither sets an error nor adds an
 * answer).  Header, question echo, EDNS and truncation follow the resolve path's wire rules (DESIGN.md sections 3, 13);
 * flags = BB_BATCH_TCP lifts the size limit to 65,535 bytes.  The upstream packets are untrusted: every read of them is
 * bounds-checked.  Matching an upstream response to its query (ID, question) is the caller's job.
 *
 *   q_pkts, q_off[n+1]    the clients' query packets, packed; a query that does not decode is BB_DROPPED (no bytes)
 *   up_pkts, up_off[n+1]  relay i's upstream response = up_pkts[up_off[i] .. up_off[i+1])
 *   out, out_off, out_len, status   as bb_resolve_batch (status BB_ANSWERED or BB_DROPPED)
 * Offsets must not decrease (BB_ERR_ARG).  BB_ERR_ARG also for n > max_batch and on an engine created without
 * `recursion`; BB_ERR_CAPACITY when the replies do not fit out_cap.  When out, out_off, out_len and status are all
 * pinned host memory (bb_host_alloc) the kernel writes the results into them directly.  Synchronous.
 */
int bb_relay_batch(bb_engine* e, const uint8_t* q_pkts, const uint32_t* q_off, const uint8_t* up_pkts, const uint32_t* up_off,
                   uint32_t n, uint32_t flags, uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status);
/*
 * Device-resident form of bb_relay_batch (lib/recursion.js:287-327), with the contract of bb_resolve_batch_device:
 * d_q_pkts, d_up_pkts and d_out 16-byte aligned, the packet buffers readable up to the next multiple of 16 past their
 * last offset; d_totals[4] = {total reply bytes, 0, overflow marker, done marker}, the markers equal to
 * bb_engine_launch_epoch() of this call when set; up to 16 streams (shared with bb_resolve_batch_device).  Asynchronous.
 */
int bb_relay_batch_device(bb_engine* e, const uint8_t* d_q_pkts, const uint32_t* d_q_off, const uint8_t* d_up_pkts,
                          const uint32_t* d_up_off, uint32_t n, uint32_t flags, uint8_t* d_out, uint32_t out_cap, uint32_t* d_out_off,
                          uint16_t* d_out_len, uint8_t* d_status, uint32_t* d_totals, void* stream);

/* ---- query log (lib/server.js:509-591, DESIGN.md section 15) ----------------------------------------------------------
 * bb_log_batch: binder's per-query "DNS query" log record of every response of a result set, the output of
 * bb_resolve_batch* (either packing, UDP or TCP) or bb_relay_batch*: response i = resp[out_off[i] .. +out_len[i]) with
 * status[i].  An answered response gets a record of two fragments, the parts of bunyan's line the response decides:
 *   head   "query":{"name":N,"type":T},"edns":true|false
 *   body   "rcode":R,"answers":[...],"additional":[...]
 * Record i = log[log_off[i] .. log_off[i] + log_len[i]), its first head_len[i] bytes the head; log_off[n] = the total.
 * A miss or a dropped query has no record.  The response bytes are untrusted: every read is bounds-checked, and a
 * response that does not decode (or lies outside resp_bytes) gets an empty record and the bad bit of its summary.
 *   summary[i] (may be NULL): qtype | rcode << 16 | edns << 20 | tc << 21 | bad << 22; 0 without a record
 * BB_ERR_ARG for n > max_batch; BB_ERR_CAPACITY when the records do not fit log_cap.  When log, log_off, log_len,
 * head_len and summary are all pinned host memory (bb_host_alloc) the kernel writes the results into them directly.
 * Synchronous.
 */
int bb_log_batch(bb_engine* e, const uint8_t* resp, uint32_t resp_bytes, const uint32_t* out_off, const uint16_t* out_len,
                 const uint8_t* status, uint32_t n, uint8_t* log, uint32_t log_cap, uint32_t* log_off /* n+1 */,
                 uint32_t* log_len, uint16_t* head_len, uint32_t* summary /* may be NULL */);
/*
 * Device-resident form of bb_log_batch, with the contract of bb_resolve_batch_device: d_resp and d_log 16-byte aligned,
 * d_resp readable up to the next multiple of 16 past its last response; d_totals[4] = {log bytes, records, overflow
 * marker, done marker}, the markers equal to bb_engine_launch_epoch() of this call when set; up to 16 streams (shared
 * with bb_resolve_batch_device).  With d_resp_totals (a resolve or relay launch's d_totals, on the same stream) the
 * response byte count is d_resp_totals[0], read on the device, bounded by resp_bytes: a resolve -> log chain needs no
 * host round trip.  Asynchronous.
 */
int bb_log_batch_device(bb_engine* e, const uint8_t* d_resp, uint32_t resp_bytes, const uint32_t* d_resp_totals,
                        const uint32_t* d_out_off, const uint16_t* d_out_len, const uint8_t* d_status, uint32_t n,
                        uint8_t* d_log, uint32_t log_cap, uint32_t* d_log_off, uint32_t* d_log_len, uint16_t* d_head_len,
                        uint32_t* d_summary, uint32_t* d_totals, void* stream);

/*
 * Recursion forward: the upstream queries of a batch of misses, grouped by datacenter, and the matching of the upstream
 * responses to them.  Replaces Recursion.prototype.resolve's lookup (lib/recursion.js:253-280,335-354,382-387) up to the
 * point where the replies are built (bb_relay_batch).  DESIGN.md section 14.
 *
 * bb_engine_set_recursion_upstreams: the upstream resolvers, what is left of self.dcs after the own-address filter
 * (:205-240,360-379).  Entry i is ip[i]:port[i] (IPv4 and port in host byte order: 127.0.0.1 = 0x7F000001) of the
 * datacenter with index dc[i] in the list last passed to bb_engine_set_recursion_filter.  At most 64 entries; n = 0 clears
 * the table.  Batches already in flight finish on the old table.  BB_ERR_ARG on an engine without `recursion`, without a
 * filter, or for a dc[i] that is not in the filter.
 */
int bb_engine_set_recursion_upstreams(bb_engine* e, const uint32_t* ip, const uint16_t* port, const uint8_t* dc, uint32_t n);

#define BB_FORWARD_MAX 65536            /* misses per forward call: the 16-bit ID space */
#define BB_ROUTE_PTR 16                 /* route of a PTR miss: every upstream */
#define BB_ROUTE_NONE 17                /* route of a miss with no upstream to ask (answered REFUSED through the relay) */
#define BB_MATCH_MAX_RESPONSES 1048576  /* received datagrams per match call */
/*
 * bb_forward_batch: miss j = pkts[pkt_off[j] .. pkt_off[j+1]), n <= BB_FORWARD_MAX (and <= max_batch).  For each miss:
 *   route[j]    the index of its datacenter in the filter's list, BB_ROUTE_PTR for a PTR query, BB_ROUTE_NONE when the
 *               upstream table has no upstream for it or the packet does not decode.  The datacenter is found as
 *               lib/recursion.js:329-344 finds it in the dotted name, labels joined with '.' and a '.' inside a label
 *               kept as it is: the name must end with the region domain (compared as bytes), and the datacenter is the
 *               rest of the name without the character before that suffix, after its last '.'
 *   its upstream query, byte for byte what recursion.py's _exchange sends except the ID: the client's flags & 0x7800
 *               (opcode kept, RD cleared), QDCOUNT 1, no other records, the client's QNAME, QTYPE and QCLASS; no OPT.
 *               ID = F(j), a keyed bijection on 16 bits (4-round Feistel network, round keys from id_key): the IDs of
 *               one call are distinct and cannot be predicted without the key.  Pick a fresh key for every call.
 * The upstream queries are grouped by route with a stable sort: route r's queries are output positions
 * group_off[r] .. group_off[r+1] (group_off has BB_ROUTE_NONE + 2 entries), each run in miss order; position k holds
 * miss order[k], at uq[uq_off[k] .. uq_off[k+1]) (an undecodable packet has an empty query).  A run can be sent to every
 * upstream of its datacenter with one vector of messages.  BB_ERR_ARG without a filter or an upstream table, for
 * n > BB_FORWARD_MAX or decreasing offsets; BB_ERR_CAPACITY when the queries do not fit uq_cap.  Synchronous.
 */
int bb_forward_batch(bb_engine* e, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n, uint64_t id_key, uint8_t* uq,
                     uint32_t uq_cap, uint32_t* uq_off, uint32_t* order, uint32_t* group_off, uint8_t* route);
/*
 * Device-resident form of bb_forward_batch, straight from a resolve launch (bb_resolve_batch_device): miss j is packet
 * d_miss_idx[j] of d_pkts / d_pkt_off, the miss count is d_resolve_totals[1], read on the device (no host round trip
 * between the launches); n_cap bounds it (the resolve batch's size; more than min(n_cap, BB_FORWARD_MAX) misses is an
 * error).  Besides the outputs of bb_forward_batch it writes each miss's client query packed in miss order,
 * d_q[d_q_off[j] .. d_q_off[j+1]): the query input of bb_relay_batch_device and bb_match_upstreams_device.
 * d_totals[5] = {upstream query bytes, n, error marker, done marker, client query bytes}; the markers equal
 * bb_engine_launch_epoch() of this call when set (too many misses, or uq_cap / q_cap too small).  Streams as
 * bb_resolve_batch_device.  Asynchronous.
 */
int bb_forward_batch_device(bb_engine* e, const uint8_t* d_pkts, const uint32_t* d_pkt_off, const uint32_t* d_miss_idx,
                            const uint32_t* d_resolve_totals, uint32_t n_cap, uint64_t id_key, uint8_t* d_uq, uint32_t uq_cap,
                            uint32_t* d_uq_off, uint32_t* d_order, uint32_t* d_group_off, uint8_t* d_route, uint8_t* d_q,
                            uint32_t q_cap, uint32_t* d_q_off, uint32_t* d_totals, void* stream);
/*
 * bb_match_upstreams: the datagrams received for a forward call, packed in arrival order — response r =
 * resp[resp_off[r] .. resp_off[r+1]) from src_ip[r]:src_port[r] (host byte order), n_resp <= BB_MATCH_MAX_RESPONSES —
 * against that call's misses: the client queries q_pkts / q_off and route[] in miss order, n, and its id_key.
 * Response r is accepted for miss j = F^-1(ID) when j < n, it is at least 12 bytes with QR set, its source is an
 * upstream of route[j] (any upstream for BB_ROUTE_PTR), QDCOUNT >= 1 and its first question equals the forwarded one
 * byte for byte (no compression pointer, same case).  The earliest accepted response of each miss wins.  Output: the
 * winners packed in miss order, up[up_off[j] .. up_off[j+1]), empty for a miss without one — bb_relay_batch's upstream
 * input as it stands (an empty upstream is a failed lookup: REFUSED, :382-386).  The datagrams are untrusted: every read
 * is bounds-checked.  BB_ERR_ARG as bb_forward_batch; BB_ERR_CAPACITY when the winners do not fit up_cap.  Synchronous.
 */
int bb_match_upstreams(bb_engine* e, const uint8_t* resp, const uint32_t* resp_off, const uint32_t* src_ip, const uint16_t* src_port,
                       uint32_t n_resp, const uint8_t* q_pkts, const uint32_t* q_off, const uint8_t* route, uint32_t n, uint64_t id_key,
                       uint8_t* up, uint32_t up_cap, uint32_t* up_off);
/*
 * Device-resident form of bb_match_upstreams: the forward launch's d_q, d_q_off and d_route, its miss count read on the
 * device from d_forward_totals[1] (bounded by n_cap as in bb_forward_batch_device).  d_totals[4] = {response bytes,
 * misses answered, overflow marker, done marker}.  Streams as bb_resolve_batch_device.  Asynchronous.
 */
int bb_match_upstreams_device(bb_engine* e, const uint8_t* d_resp, const uint32_t* d_resp_off, const uint32_t* d_src_ip,
                              const uint16_t* d_src_port, uint32_t n_resp, const uint8_t* d_q, const uint32_t* d_q_off,
                              const uint8_t* d_route, const uint32_t* d_forward_totals, uint32_t n_cap, uint64_t id_key, uint8_t* d_up,
                              uint32_t up_cap, uint32_t* d_up_off, uint32_t* d_totals, void* stream);

/* Number of kernel launches bb_* calls have issued so far on this engine. */
uint64_t bb_engine_launch_count(const bb_engine* e);
/* Epoch (launch number, low 32 bits) of the most recent resolve call on this engine. */
uint32_t bb_engine_launch_epoch(const bb_engine* e);
/*
 * Stage timers, the batched analogue of query._stamp() (lib/server.js:479-483); compiled in only when the library is
 * built with -DBB_STAGE_LOG (tools/stage_times.py does that; the default build has no stamps): when d_log is
 * a device buffer of ceil(n/128) x 16 uint64, every 128-query tile of later launches stores
 * %globaltimer (ns) at: 0 start, 1 offsets in, 2 packets staged, 3 decoded, 4 normalised+hashed,
 * 5 probed, 6 sized, 7 tile scan, 8 placed (claim / look-back), 9 responses assembled,
 * 10 flushed; 11-14 service sizing: entered, record opened, permutation built, children walked
 * (thread 0's view of its tile).  NULL turns it off.  bb_shard_route_push stamps the same log (which
 * then needs one more row): 0 start, 1 offsets in, 2 packets staged, 3-4 decoded/hashed, 6 routed,
 * 7 space claimed, 8 grouped by owner, 9 peer stores issued, 10 system fence done + block counted;
 * row ntiles, slot 0: epoch flags published.
 */
void bb_engine_set_stage_log(bb_engine* e, unsigned long long* d_log);

/* ---- multi-GPU: hash-sharded zone, one process per GPU (SURVEY.md section 8e) ------------------ */
/*
 * The reference scales out with full replicas behind a balancer (boot/setup.sh:136-149); here the
 * zone is sharded by key hash and a batch is routed with ONE exchange: the ingress rank parses
 * each query far enough to know its lookup key and stores the packet directly into the owner
 * rank's HBM over NVLink peer memory (route + push, one kernel); the owner resolves and answers.
 * Queries that need no lookup (NOTIMP, refusals, malformed) are answered on the ingress rank.
 *
 *   bb_shard_create        receive regions (one per source rank) + per-region output buffers
 *   bb_shard_get_ipc_handle / bb_shard_open_peers
 *                          exchange CUDA IPC handles of the receive buffers (the host passes the
 *                          opaque bytes between processes, e.g. torch.distributed.all_gather)
 *   bb_shard_route_push    ingress: device-resident batch -> owners' regions (asynchronous); its last
 *                          block publishes, after system-scope fences, an epoch flag per region
 *   bb_shard_resolve       owner: resolve all regions (asynchronous; joins back into `stream`).
 *                          wait_for_peers=1: first waits on the device (bounded spin) for every
 *                          source's flag of this step — no collective anywhere on the data path;
 *                          wait_for_peers=0: the caller has put its own cross-rank barrier on the
 *                          stream.  All ranks must call route_push/resolve the same number of times.
 *   bb_shard_fetch         one region's results to host memory; qidx[] = ingress index of each
 *                          query on the source rank (qidx_base + position), which also keys the
 *                          service shuffle, so answers are identical to the unsharded engine's.
 *                          BB_ERR_CAPACITY: the source overflowed a region (cap_q queries or cap_b =
 *                          max_batch x bytes_per_query packet bytes) in this step, or the region's
 *                          answers overflowed the shard's output; the step after is unaffected.
 *                          BB_ERR_CUDA: this step's wait for the peers timed out.
 *   bb_shard_host_results  enable=1: the shard keeps pinned host mirrors of its result set and every
 *                          later bb_shard_resolve writes responses, offsets, lengths, statuses, ingress
 *                          indices, miss lists and totals straight into them (zero-copy: no device-to-
 *                          host copies, no size round trip).  bb_shard_fetch is then unavailable.
 *   bb_shard_results       pointers into the mirrors for region `src` of the last bb_shard_resolve,
 *                          once the caller has waited for the work it enqueued on that stream.  Valid
 *                          until the next bb_shard_resolve on this shard.
 */
typedef struct bb_shard bb_shard;
bb_shard* bb_shard_create(bb_engine* e, uint32_t nranks, uint32_t rank, uint32_t max_batch,
                          uint32_t bytes_per_query, int* err);
void      bb_shard_destroy(bb_shard* s);
uint32_t  bb_shard_ipc_handle_size(void);
uint32_t  bb_shard_region_capacity(const bb_shard* s);
int bb_shard_get_ipc_handle(bb_shard* s, void* handle_out);
int bb_shard_open_peers(bb_shard* s, const void* handles);
int bb_shard_route_push(bb_shard* s, const uint8_t* d_pkts, const uint32_t* d_pkt_off, uint32_t n,
                        uint32_t qidx_base, void* stream);
/*
 * bb_shard_route_push for a batch of TCP queries: flags = BB_BATCH_TCP makes every query of this push a TCP query.  The
 * flag travels in each region header of the step, so each owner answers each region under its own source's limit: one
 * step may mix ranks that push TCP with ranks that push UDP, and every push rewrites the flag.  TCP answers share the
 * region's output room, out_cap = cap_q x 256 bytes (cap_q = max_batch): a region whose answers do not fit is
 * BB_ERR_CAPACITY from bb_shard_fetch / bb_shard_results for that step only.  Other bits are ignored; flags = 0 is
 * bb_shard_route_push.
 */
int bb_shard_route_push_ex(bb_shard* s, const uint8_t* d_pkts, const uint32_t* d_pkt_off, uint32_t n,
                           uint32_t qidx_base, uint32_t flags, void* stream);
int bb_shard_resolve(bb_shard* s, uint64_t shuffle_seed, int wait_for_peers, void* stream);
int bb_shard_fetch(bb_shard* s, uint32_t src, uint8_t* out, uint32_t out_cap, uint32_t* out_off,
                   uint16_t* out_len, uint8_t* status, uint32_t* qidx, uint32_t* miss_idx,
                   uint32_t* n_out, uint32_t* n_miss, uint32_t* total_out);

/* The collective baseline (SURVEY.md section 8e: "one all-to-all of routed records"): with caller-owned exchange buffers
 * route_push fills LOCAL send regions (region d of the current set = the records for rank d, in the receive-region layout)
 * and bb_shard_resolve(wait_for_peers = 0) reads the receive buffer the caller's collective filled — ncclSend/ncclRecv of
 * the header, offset, ingress-index and packet arrays of every region (binder_b200/shard.py, sync='nccl_a2a').
 *   bb_shard_exchange_bytes   size of each buffer (2 sets x nranks regions)
 *   bb_shard_exchange_set     set (0/1) the last route_push wrote = the one the next resolve reads
 *   bb_shard_region_layout    out[5] = {bytes per region, capacity in queries, offset of the u32 offsets array (cap+1), of the
 *                             u32 ingress-index array (cap), of the packet bytes}; a region starts with the 16-byte header
 *                             {count, packet bytes, epoch, flags}; flags bit 0 = the sender overflowed a region in this
 *                             step, bit 1 = the push was TCP (bb_shard_route_push_ex) */
int      bb_shard_use_exchange_buffers(bb_shard* s, void* d_send, void* d_recv);
size_t   bb_shard_exchange_bytes(const bb_shard* s);
uint32_t bb_shard_exchange_set(const bb_shard* s);
void     bb_shard_region_layout(const bb_shard* s, uint64_t out[5]);

int bb_shard_host_results(bb_shard* s, int enable);
int bb_shard_results(bb_shard* s, uint32_t src, const uint8_t** out, const uint32_t** out_off,
                     const uint16_t** out_len, const uint8_t** status, const uint32_t** qidx,
                     const uint32_t** miss_idx, uint32_t* n_out, uint32_t* n_miss, uint32_t* total_out);

/* ---- mname-balancer backend frames (SURVEY.md section 8f row 1) -------------------------------------
 * The balancer relays UDP packets to a backend over an AF_UNIX stream as frames of little-endian u32 words
 * (deps/mname-balancer/backend.c:22-113, bbal.h:80-87): INBOUND_UDP {2, src ip, src port, len, bytes} in,
 * OUTBOUND_UDP {1002, dst ip, dst port, len, bytes} out, HELLO 1 -> 1001, HEARTBEAT 4 -> 1004.
 *   bb_frames_parse   byte stream -> batch container (+ source addresses, control frames in order).  Only whole
 *                     frames are consumed (*consumed); stops early when the batch or the control list is full.
 *                     BB_ERR_PROTOCOL on an unknown type, INBOUND_TCP (which turns the session into a TCP proxy,
 *                     backend.c:60-75) or a packet over 1500 bytes (udp_proxy.c:159-170) — what was parsed before
 *                     it is still returned.
 *   bb_frames_build   results -> one SERVER_HELLO/HEARTBEAT per control frame, then an OUTBOUND_UDP frame per answered
 *                     query (misses and drops produce no frame).  *out_len = bytes needed; BB_ERR_CAPACITY if out_cap
 *                     is smaller (call with out = NULL to size).
 *   bb_backend_*      a session: feed() the bytes read from the socket, get the bytes to write back; every complete
 *                     INBOUND_UDP frame fed so far is resolved in batches of up to max_batch through bb_resolve_batch,
 *                     a partial trailing frame is kept for the next call.  *out and the miss arrays point into the
 *                     session and stay valid until the next feed.  Handed-off misses (lib/server.js:110-113,222-225)
 *                     come back as packets + source addresses for the host's recursion.
 *   bb_backend_relay  the session's replies to those misses, once the host's upstream exchange has an upstream response
 *                     for each (q = the miss packets, up = upstream i, empty = the lookup failed): bb_relay_batch with
 *                     flags 0 (the UDP path: 512-byte / EDNS limits) in batches of max_batch, then bb_frames_build: one
 *                     OUTBOUND_UDP frame per answered relay, addressed to (dst_ip[i], dst_port[i]).  *out points into the
 *                     session, valid until the next relay call; it does not invalidate bb_backend_feed's output.  Call
 *                     it from the thread that feeds the session (they share its result buffers).  A failed batch
 *                     (capacity, CUDA, an engine without `recursion`) loses its relays, counts them (stat 7) and the
 *                     call goes on with the next batch; the return value is then the first batch's error.  BB_ERR_ARG
 *                     for null arrays or decreasing offsets.
 *   bb_query_log_backend_enable / bb_query_log_backend   binder's "DNS query" log records (lib/server.js:509-591) of the
 *                     answers a session sends: see bb_query_log_records below.  Off by default; stats 8 and 9.
 */
enum { BB_FRAME_CLIENT_HELLO = 1, BB_FRAME_INBOUND_UDP = 2, BB_FRAME_INBOUND_TCP = 3, BB_FRAME_CLIENT_HEARTBEAT = 4,
       BB_FRAME_SERVER_HELLO = 1001, BB_FRAME_OUTBOUND_UDP = 1002, BB_FRAME_INBOUND_TCP_OK = 1003, BB_FRAME_SERVER_HEARTBEAT = 1004 };
int bb_frames_parse(const uint8_t* in, size_t in_len, uint8_t* pkts, uint32_t cap_bytes, uint32_t* pkt_off,
                    uint32_t* src_ip, uint32_t* src_port, uint32_t cap_n, uint32_t* n,
                    uint32_t* control, uint32_t cap_ctrl, uint32_t* n_ctrl, size_t* consumed);
int bb_frames_build(const uint8_t* resp, const uint32_t* resp_off, const uint16_t* resp_len, const uint8_t* status,
                    const uint32_t* dst_ip, const uint32_t* dst_port, uint32_t n, const uint32_t* control, uint32_t n_ctrl,
                    uint8_t* out, size_t out_cap, size_t* out_len);
typedef struct bb_backend bb_backend;
typedef struct bb_backend_misses {
    uint32_t n; const uint8_t* pkts; const uint32_t* pkt_off /* n+1 */; const uint32_t* src_ip; const uint32_t* src_port;
} bb_backend_misses;
bb_backend* bb_backend_create(bb_engine* e, uint32_t max_batch, int* err);
void        bb_backend_destroy(bb_backend* b);
int         bb_backend_feed(bb_backend* b, const uint8_t* in, size_t in_len, uint64_t shuffle_seed,
                            const uint8_t** out, size_t* out_len, bb_backend_misses* misses);
int         bb_backend_relay(bb_backend* b, const uint8_t* q_pkts, const uint32_t* q_off, const uint8_t* up_pkts,
                             const uint32_t* up_off, const uint32_t* dst_ip, const uint32_t* dst_port, uint32_t n,
                             const uint8_t** out, size_t* out_len);
/* 0 udp frames 1 answered 2 missed 3 dropped 4 pending bytes 5 queries of failed batches 6 replies relayed
 * 7 queries of failed relay batches 8 query-log records 9 answers whose query-log call failed (lost records) */
uint64_t    bb_backend_stat(const bb_backend* b, int what);

/* ---- query log of the balancer sessions (DESIGN.md section 15) -------------------------------------------------------
 * With the query log on, every resolve or relay batch a session (bb_backend, bb_tcp_hub) runs that succeeds and has an
 * answer gets one bb_log_batch call over its own result set.  The records of one call (a feed or flush: which = 0; a
 * relay: which = 1) share one pinned buffer of the session, written by the kernel in place: batch k's records start
 * where batch k-1's end (rounded up to 16 bytes).  Record i = log[log_off[i] .. log_off[i] + log_len[i]), its first
 * head_len[i] bytes the head fragment, the rest the body; an answer that does not decode has an empty record.  One
 * record per answer sent, in the order the answers were written: a feed's OUTBOUND_UDP frames (control replies have no
 * record), a backend relay's frames, a flush's answers across sessions in the order they were appended, a hub relay's
 * replies that were appended (a reply to a session closed meanwhile is not sent and has no record).  The client is the
 * query's INBOUND_UDP source, the relay's (dst_ip, dst_port), or the hub session's INBOUND_TCP peer.  The records stay
 * valid until the next call of the same kind: a feed does not invalidate the last relay's, nor a relay the last feed's.
 * A log call that fails with BB_ERR_CAPACITY grows the buffer and runs once more; a batch whose log call still fails
 * keeps its answers (they are sent), and they count in `lost` and in the lost-records stat.  The query log never
 * changes a call's frames, outputs, misses, other stats or return code.
 *   ..._enable      enable != 0: on (allocates the buffers; BB_ERR_NOMEM); 0: off (frees them; no records, no calls).
 *   bb_query_log_backend / bb_query_log_tcp_hub   the records of the last call of kind `which`; n = 0 with the log off.
 *                   BB_ERR_ARG for which > 1.
 */
typedef struct bb_query_log_records {
    uint32_t n;                  /* records */
    const uint8_t*  log;         /* the call's record bytes */
    const uint32_t* log_off;     /* n: record i = log[log_off[i] .. log_off[i] + log_len[i]) */
    const uint32_t* log_len;     /* n */
    const uint16_t* head_len;    /* n: the first head_len[i] bytes are the head fragment */
    const uint16_t* req_id;      /* n: the response's DNS ID */
    const uint32_t* client_ip;   /* n: IPv4 as the frame carries it (127.0.0.1 = 0x7F000001) */
    const uint32_t* client_port; /* n */
    const uint32_t* session;     /* n for a hub: the record's session id; NULL for a backend */
    uint32_t lost;               /* answered responses of the call whose log call failed */
} bb_query_log_records;
int         bb_query_log_backend_enable(bb_backend* b, int enable);
int         bb_query_log_backend(const bb_backend* b, int which /* 0: last feed, 1: last relay */, bb_query_log_records* r);

/* ---- mname-balancer TCP proxy sessions (deps/mname-balancer/backend.c:22-113, tcp_proxy.c:160-300) ----------------
 * The balancer hands every DNS-over-TCP client connection to a backend as its own AF_UNIX session.  The session opens
 * with INBOUND_TCP {3, src ip, src port} (12 bytes, u32 little-endian); the backend answers INBOUND_TCP_OK (u32 1003), its
 * last frame on that session, and from then on the session carries the client's raw DNS-over-TCP stream both ways
 * (2-byte big-endian length prefixes, RFC 1035 4.2.2).  A host routes a new AF_UNIX connection by its first frame:
 * CLIENT_HELLO goes to a bb_backend, INBOUND_TCP to a TCP hub.  A hub owns many such sessions of one engine; the messages
 * that complete on ALL of them between two flushes are resolved together.
 *   create   max_batch is clamped to the engine's limits; query bytes per batch: max(64 x max_batch, 65,536), at most
 *            the engine's max_batch_bytes (a message larger than that is dropped).  Answer bytes per batch (stat 10):
 *            16 KB x max_batch, at least 1 MB, at most the engine's own response buffer (512 x its max_batch, >= 1 MB).
 *   open     a new session; ids are not reused.
 *   feed     bytes read from the session.  Before the handshake only a complete INBOUND_TCP frame is accepted: it records
 *            the source address and queues INBOUND_TCP_OK as the session's first output.  Any other first frame, and a
 *            zero-length DNS message later, is BB_ERR_PROTOCOL for this session only: it reads nothing more, messages
 *            that completed before the error are still answered, and the session may close once they are written.
 *            BB_ERR_ARG for a session that is unknown, closed, or past eof.
 *   eof      the peer half-closed: complete messages are still answered, a partial one is discarded.
 *   flush    every message completed since the last flush, in arrival order, through bb_resolve_batch_ex(BB_BATCH_TCP) in
 *            batches split at max_batch or the query-byte limit; qidx_base runs 0, n0, n0 + n1, ... over the batches of
 *            one flush.  Each answer is appended, length-prefixed, to its session's output: per session in arrival order.
 *            Misses (BB_MISS_RECURSE) come back in *misses (packets + session ids, valid until the next flush) and stay
 *            owed until relayed.  A failed batch (capacity, CUDA) loses its queries, counts them, and the flush goes on
 *            with the next batch; the return value is then the first batch's error.
 *   output   the bytes to write to the session (valid until the next hub call that changes it) and whether the session
 *            may be closed: eof or protocol error seen, no message queued or owed a relay, nothing left to write.
 *   consume  n bytes of that output were written.
 *   close    forget the session; its queued messages and outstanding relays are dropped (counted).
 *   relay    the host's upstream responses for misses (q = the miss packets, up = upstream i, empty = the lookup failed)
 *            through bb_relay_batch(BB_BATCH_TCP), each reply appended length-prefixed to sessions[i]: RFC 7766 allows
 *            out-of-order answers and the ID matches them.  Batches of max_batch; a failed one is counted as in flush.
 *   bb_query_log_tcp_hub_enable / bb_query_log_tcp_hub   the "DNS query" log records of the answers appended by the last
 *            flush (which = 0) or relay (which = 1), with each record's session id: bb_query_log_records above.  Off by
 *            default; stats 11, 12.
 */
typedef struct bb_tcp_hub bb_tcp_hub;
typedef struct bb_tcp_hub_misses {
    uint32_t n; const uint8_t* pkts; const uint32_t* pkt_off /* n+1 */; const uint32_t* session;
} bb_tcp_hub_misses;
bb_tcp_hub* bb_tcp_hub_create(bb_engine* e, uint32_t max_batch, int* err);
void        bb_tcp_hub_destroy(bb_tcp_hub* h);
int         bb_tcp_hub_open(bb_tcp_hub* h, uint32_t* session);
int         bb_tcp_hub_feed(bb_tcp_hub* h, uint32_t session, const uint8_t* in, size_t in_len);
int         bb_tcp_hub_eof(bb_tcp_hub* h, uint32_t session);
int         bb_tcp_hub_flush(bb_tcp_hub* h, uint64_t shuffle_seed, bb_tcp_hub_misses* misses);
int         bb_tcp_hub_output(bb_tcp_hub* h, uint32_t session, const uint8_t** out, size_t* out_len, int* closable);
int         bb_tcp_hub_consume(bb_tcp_hub* h, uint32_t session, size_t n);
int         bb_tcp_hub_close(bb_tcp_hub* h, uint32_t session);
int         bb_tcp_hub_relay(bb_tcp_hub* h, const uint8_t* q_pkts, const uint32_t* q_off, const uint8_t* up_pkts,
                             const uint32_t* up_off, const uint32_t* sessions, uint32_t n);
/* the client's address from the session's INBOUND_TCP frame (0, 0 before the handshake) */
int         bb_tcp_hub_peer(const bb_tcp_hub* h, uint32_t session, uint32_t* ip, uint32_t* port);
/* 0 sessions opened 1 DNS messages received 2 answered 3 missed 4 dropped (undecodable, oversized, or of a closed session)
 * 5 protocol errors 6 queries of failed batches 7 relay replies appended 8 sessions open 9 messages queued for the next flush
 * 10 answer bytes per batch 11 query-log records 12 answers whose query-log call failed (lost records) */
uint64_t    bb_tcp_hub_stat(const bb_tcp_hub* h, int what);
int         bb_query_log_tcp_hub_enable(bb_tcp_hub* h, int enable);
int         bb_query_log_tcp_hub(const bb_tcp_hub* h, int which /* 0: last flush, 1: last relay */, bb_query_log_records* r);

/* pinned host memory for the batch containers */
void* bb_host_alloc(size_t bytes);
void  bb_host_free(void* p);

#ifdef __cplusplus
}
#endif
#endif /* BINDER_B200_H */
