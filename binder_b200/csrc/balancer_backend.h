// One mname-balancer UDP session around an engine: the state bb_backend_feed (balancer_frames.cpp) and
// bb_backend_relay (balancer_relay.cpp) share; and the query-log records that both sessions, this one and the TCP hub
// (balancer_tcp.cpp), keep of their calls (switched on and read in balancer_query_log.cpp).  Host code only.
#pragma once
#include "../../include/binder_b200.h"

#include <algorithm>
#include <cstring>
#include <vector>

// The "DNS query" log records of a session's last call of one kind (a feed or flush, a relay): one bb_log_batch call per
// batch with an answer, into a pinned buffer (zero-copy: the kernel writes the records where they stay).  Batch k's
// records start at the end of batch k-1's, rounded up to 16 bytes (bb_log_batch writes pinned memory directly only from
// a 16-byte-aligned start).  The per-record arrays hold the answered responses only, in the order the answers were sent.
// The log call goes through `log_fn`, which only switching the log on sets (balancer_query_log.cpp): the session sources
// themselves do not depend on the log kernel and link without it.
struct bb_log_set {
    static constexpr uint32_t INITIAL = 1u << 20;      // bytes; grown on BB_ERR_CAPACITY
    using log_fn_t = int (*)(bb_engine*, const uint8_t*, uint32_t, const uint32_t*, const uint16_t*, const uint8_t*, uint32_t,
                             uint8_t*, uint32_t, uint32_t*, uint32_t*, uint16_t*, uint32_t*);
    log_fn_t log_fn = nullptr;                         // bb_log_batch
    uint32_t max_batch = 0;                            // responses per batch (the session's)
    uint8_t* log = nullptr; uint32_t cap = 0, used = 0;
    uint32_t* b_off = nullptr; uint32_t* b_len = nullptr; uint16_t* b_head = nullptr;    // one batch's bb_log_batch output (pinned)
    std::vector<uint32_t> off, len, ip, port, session; std::vector<uint16_t> head, req_id;
    uint32_t lost = 0;
    uint64_t n_records = 0, n_lost = 0;                // over the session's life (the stats)

    bool on() const { return log != nullptr; }
    void clear() { used = 0; lost = 0; off.clear(); len.clear(); ip.clear(); port.clear(); session.clear(); head.clear(); req_id.clear(); }
    void release() {
        bb_host_free(log); bb_host_free(b_off); bb_host_free(b_len); bb_host_free(b_head);
        log = nullptr; b_off = nullptr; b_len = nullptr; b_head = nullptr; cap = 0;
        clear();
    }
    // enable: the buffers for batches of up to max_batch responses, records made by `fn`; disable: none (and no records)
    int set(int enable, log_fn_t fn) {
        if (!enable) { release(); return BB_OK; }
        log_fn = fn;
        if (on()) return BB_OK;
        log = (uint8_t*)bb_host_alloc(INITIAL); b_off = (uint32_t*)bb_host_alloc(((size_t)max_batch + 1) * 4);
        b_len = (uint32_t*)bb_host_alloc((size_t)max_batch * 4 + 16); b_head = (uint16_t*)bb_host_alloc((size_t)max_batch * 2 + 16);
        if (!log || !b_off || !b_len || !b_head) { release(); return BB_ERR_NOMEM; }
        cap = INITIAL;
        return BB_OK;
    }
    // One batch's result set (n responses, statuses in `status`): bb_log_batch over all of it, then for each answered
    // response, in index order, keep(i, ip, port, session) says whether it was sent and to which client.  A failed log
    // call leaves the answers alone and counts the sent ones in `lost`.
    template <class Keep>
    void batch(bb_engine* e, const uint8_t* resp, const uint32_t* resp_off, const uint16_t* resp_len, const uint8_t* status,
               uint32_t n, Keep keep) {
        uint32_t answered = 0;
        for (uint32_t i = 0; i < n; i++) answered += status[i] == BB_ANSWERED;
        if (!on() || answered == 0) return;            // a batch without an answer needs no call
        const uint32_t at = (used + 15u) & ~15u;
        int rc = BB_ERR_CAPACITY;
        for (int attempt = 0; attempt < 2 && rc == BB_ERR_CAPACITY; attempt++) {
            if (attempt && grow(at, b_off[n]) != BB_OK) break;
            b_off[n] = 0;                              // the kernel leaves the bytes it needed here, also when they do not fit
            rc = at <= cap ? log_fn(e, resp, resp_off[n], resp_off, resp_len, status, n, log + at, cap - at, b_off, b_len, b_head, nullptr)
                           : BB_ERR_CAPACITY;
        }
        uint32_t kept = 0;
        for (uint32_t i = 0; i < n; i++) {
            uint32_t cip = 0, cport = 0, sid = 0;
            if (status[i] != BB_ANSWERED || !keep(i, cip, cport, sid)) continue;
            if (rc != BB_OK) { kept++; continue; }
            const uint8_t* r = resp + resp_off[i];
            off.push_back(at + b_off[i]); len.push_back(b_len[i]); head.push_back(b_head[i]);
            req_id.push_back(resp_len[i] >= 2 ? (uint16_t)(r[0] << 8 | r[1]) : 0);
            ip.push_back(cip); port.push_back(cport); session.push_back(sid);
            kept++;
        }
        if (rc != BB_OK) { lost += kept; n_lost += kept; return; }
        n_records += kept;
        used = at + b_off[n];
    }
    // room for `need` more bytes from `at`, the records before `at` kept
    int grow(uint32_t at, uint32_t need) {
        const uint64_t want = std::max<uint64_t>((uint64_t)cap * 2, (uint64_t)at + need + 64);
        if (want > 0xFFFFFF00ull) return BB_ERR_CAPACITY;
        uint8_t* p = (uint8_t*)bb_host_alloc((size_t)want);
        if (!p) return BB_ERR_NOMEM;
        if (used) memcpy(p, log, used);
        bb_host_free(log);
        log = p; cap = (uint32_t)want;
        return BB_OK;
    }
    void get(bb_query_log_records* r, bool with_session) const {
        r->n = (uint32_t)off.size(); r->log = log; r->log_off = off.data(); r->log_len = len.data(); r->head_len = head.data();
        r->req_id = req_id.data(); r->client_ip = ip.data(); r->client_port = port.data();
        r->session = with_session ? session.data() : nullptr; r->lost = lost;
    }
};

struct bb_backend {
    bb_engine* e = nullptr; uint32_t max_batch = 0, max_bytes = 0;
    std::vector<uint8_t> pending;                      // bytes of an incomplete trailing frame
    // batch containers (pinned: the engine then writes results straight into them)
    uint8_t* pkts = nullptr; uint32_t* pkt_off = nullptr; uint32_t* ip = nullptr; uint32_t* port = nullptr;
    uint8_t* resp = nullptr; uint32_t resp_cap = 0; uint32_t* resp_off = nullptr; uint16_t* resp_len = nullptr;
    uint8_t* status = nullptr; uint32_t* miss = nullptr;
    std::vector<uint8_t> out;                          // frames to write back
    std::vector<uint8_t> m_pkts; std::vector<uint32_t> m_off, m_ip, m_port;    // handed-off misses of the last feed
    std::vector<uint8_t> r_out;                        // frames of the last relay call (apart from `out`: both stay valid)
    std::vector<uint32_t> r_qoff, r_upoff;             // a relay batch's offsets, rebased
    uint64_t n_udp = 0, n_answered = 0, n_missed = 0, n_dropped = 0, n_failed = 0, n_relayed = 0, n_relay_failed = 0;
    uint32_t qidx_next = 0;                             // query index of the next batch's first query within the current feed (keys the shuffle)
    bb_log_set qlog[2];                                // query-log records of the last feed [0] and the last relay [1]
};

// the TCP hub's query-log records of its last flush [0] and last relay [1] (struct bb_tcp_hub: balancer_tcp.cpp)
bb_log_set* tcp_hub_log_sets(bb_tcp_hub* h);
