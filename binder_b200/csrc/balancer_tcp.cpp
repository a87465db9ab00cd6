// mname-balancer TCP proxy sessions, natively: the bb_tcp_hub of include/binder_b200.h.
//
// The balancer hands every DNS-over-TCP client connection to a backend as its own AF_UNIX session
// (deps/mname-balancer/backend.c:22-113, tcp_proxy.c:160-300): INBOUND_TCP {3, src ip, src port} in, INBOUND_TCP_OK (1003)
// out, then the client's raw stream of 2-byte big-endian length-prefixed messages both ways (RFC 1035 4.2.2).  A hub
// holds many such sessions of one engine: feed() de-frames each session's bytes into one queue, flush() resolves the
// whole queue as TCP batches (bb_resolve_batch_ex with BB_BATCH_TCP) and appends each answer, length-prefixed, to its
// session's output.  The host keeps the sockets.  Host code only: no CUDA in this file.
#include "balancer_backend.h"                          // bb_log_set: the query-log records

#include <algorithm>
#include <cstring>
#include <unordered_map>
#include <vector>

namespace {
inline uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
constexpr size_t HANDSHAKE = 12;                       // INBOUND_TCP {type, src ip, src port}

struct TcpSession {
    uint32_t ip = 0, port = 0;
    bool shook = false, eof = false, bad = false;      // handshake done / peer half-closed / protocol error (reads nothing more)
    uint32_t queued = 0, relays = 0;                   // messages waiting for a flush, misses waiting for their relay
    std::vector<uint8_t> in;                           // an incomplete frame or message
    std::vector<uint8_t> out; size_t head = 0;         // bytes to write: out[head..)

    void put(const uint8_t* msg, uint32_t len) {      // one length-prefixed DNS message
        out.push_back((uint8_t)(len >> 8)); out.push_back((uint8_t)len);
        out.insert(out.end(), msg, msg + len);
    }
};
}  // namespace

struct bb_tcp_hub {
    bb_engine* e = nullptr; uint32_t max_batch = 0, max_bytes = 0, resp_cap = 0;
    uint32_t next_id = 1;                              // 0 is never a session
    std::unordered_map<uint32_t, TcpSession> sess;
    // messages completed since the last flush, all sessions, in arrival order
    std::vector<uint8_t> q_bytes; std::vector<uint32_t> q_off{0}, q_sid;
    // batch containers (pinned: the engine then writes results straight into them)
    uint8_t* pkts = nullptr; uint32_t* pkt_off = nullptr;
    uint8_t* resp = nullptr; uint32_t* resp_off = nullptr; uint16_t* resp_len = nullptr; uint8_t* status = nullptr; uint32_t* miss = nullptr;
    std::vector<uint32_t> b_sid;                       // session of each query of the current batch
    std::vector<uint8_t> m_pkts; std::vector<uint32_t> m_off, m_sid;    // misses of the last flush
    std::vector<uint32_t> r_qoff, r_upoff;             // a relay batch's offsets, rebased
    uint64_t n_sessions = 0, n_msgs = 0, n_answered = 0, n_missed = 0, n_dropped = 0, n_proto = 0, n_failed = 0, n_relayed = 0;
    bb_log_set qlog[2];                                // query-log records of the last flush [0] and the last relay [1]

    TcpSession* find(uint32_t id) { auto it = sess.find(id); return it == sess.end() ? nullptr : &it->second; }
};

bb_log_set* tcp_hub_log_sets(bb_tcp_hub* h) { return h->qlog; }

extern "C" {

bb_tcp_hub* bb_tcp_hub_create(bb_engine* e, uint32_t max_batch, int* err) {
    if (err) *err = BB_OK;
    if (!e || max_batch == 0) { if (err) *err = BB_ERR_ARG; return nullptr; }
    // never build a batch the engine would refuse, nor ask for answer room its own response buffer does not have
    const uint32_t emb = bb_engine_max_batch(e);
    if (max_batch > emb) max_batch = emb;
    const uint64_t qbytes = std::min<uint64_t>(std::max<uint64_t>((uint64_t)max_batch * 64, 1u << 16), bb_engine_max_batch_bytes(e));
    const uint64_t ecap = std::min<uint64_t>(std::max<uint64_t>((uint64_t)emb * 512, 1u << 20), 0xFFFFFF00ull);
    const uint64_t rcap = std::min<uint64_t>(std::max<uint64_t>((uint64_t)max_batch * 16384, 1u << 20), ecap);
    bb_tcp_hub* h = new bb_tcp_hub();
    h->e = e; h->max_batch = max_batch; h->max_bytes = (uint32_t)qbytes; h->resp_cap = (uint32_t)rcap;
    h->pkts = (uint8_t*)bb_host_alloc((size_t)h->max_bytes + 64); h->pkt_off = (uint32_t*)bb_host_alloc(((size_t)max_batch + 1) * 4);
    h->resp = (uint8_t*)bb_host_alloc((size_t)h->resp_cap + 64); h->resp_off = (uint32_t*)bb_host_alloc(((size_t)max_batch + 1) * 4);
    h->resp_len = (uint16_t*)bb_host_alloc((size_t)max_batch * 2 + 16); h->status = (uint8_t*)bb_host_alloc((size_t)max_batch + 16);
    h->miss = (uint32_t*)bb_host_alloc((size_t)max_batch * 4);
    if (!h->pkts || !h->pkt_off || !h->resp || !h->resp_off || !h->resp_len || !h->status || !h->miss) {
        bb_tcp_hub_destroy(h); if (err) *err = BB_ERR_NOMEM; return nullptr;
    }
    memset(h->pkts, 0, (size_t)h->max_bytes + 64);
    h->b_sid.resize(max_batch);
    h->qlog[0].max_batch = h->qlog[1].max_batch = max_batch;
    return h;
}

void bb_tcp_hub_destroy(bb_tcp_hub* h) {
    if (!h) return;
    bb_host_free(h->pkts); bb_host_free(h->pkt_off); bb_host_free(h->resp); bb_host_free(h->resp_off);
    bb_host_free(h->resp_len); bb_host_free(h->status); bb_host_free(h->miss);
    h->qlog[0].release(); h->qlog[1].release();
    delete h;
}

int bb_tcp_hub_open(bb_tcp_hub* h, uint32_t* session) {
    if (!h || !session) return BB_ERR_ARG;
    if (h->next_id == 0) h->next_id = 1;
    while (h->sess.count(h->next_id)) h->next_id++;    // only after 2^32 sessions: skip ids still open
    const uint32_t id = h->next_id++;
    h->sess[id];
    h->n_sessions++;
    *session = id;
    return BB_OK;
}

int bb_tcp_hub_feed(bb_tcp_hub* h, uint32_t session, const uint8_t* in, size_t in_len) {
    if (!h || (!in && in_len)) return BB_ERR_ARG;
    TcpSession* s = h->find(session);
    if (!s || s->eof) return BB_ERR_ARG;               // past eof nothing can arrive
    if (s->bad) return BB_ERR_PROTOCOL;                // the session reads nothing more
    if (in_len) s->in.insert(s->in.end(), in, in + in_len);
    const uint8_t* b = s->in.data(); const size_t len = s->in.size();
    size_t pos = 0;
    if (!s->shook) {
        if (len < 4) return BB_OK;
        if (rd32(b) != BB_FRAME_INBOUND_TCP) {          // CLIENT_HELLO, INBOUND_UDP, anything else: this is no TCP session
            s->bad = true; h->n_proto++; s->in.clear();
            return BB_ERR_PROTOCOL;
        }
        if (len < HANDSHAKE) return BB_OK;
        s->ip = rd32(b + 4); s->port = rd32(b + 8); s->shook = true;
        const uint8_t ok[4] = { (uint8_t)BB_FRAME_INBOUND_TCP_OK, (uint8_t)(BB_FRAME_INBOUND_TCP_OK >> 8), 0, 0 };
        s->out.insert(s->out.end(), ok, ok + 4);       // the last frame the backend sends; raw DNS from here on
        pos = HANDSHAKE;
    }
    while (len - pos >= 2) {
        const uint32_t ln = (uint32_t)b[pos] << 8 | b[pos + 1];
        if (ln == 0) { s->bad = true; h->n_proto++; break; }     // as TcpFramer: what completed before is still answered
        if (len - pos - 2 < ln) break;
        h->q_bytes.insert(h->q_bytes.end(), b + pos + 2, b + pos + 2 + ln);
        h->q_off.push_back((uint32_t)h->q_bytes.size()); h->q_sid.push_back(session);
        s->queued++; h->n_msgs++;
        pos += 2 + (size_t)ln;
    }
    if (s->bad) s->in.clear();
    else s->in.erase(s->in.begin(), s->in.begin() + (long)pos);
    return s->bad ? BB_ERR_PROTOCOL : BB_OK;
}

int bb_tcp_hub_eof(bb_tcp_hub* h, uint32_t session) {
    TcpSession* s = h ? h->find(session) : nullptr;
    if (!s) return BB_ERR_ARG;
    s->eof = true;
    s->in.clear();                                     // a partial message never completes
    return BB_OK;
}

int bb_tcp_hub_flush(bb_tcp_hub* h, uint64_t shuffle_seed, bb_tcp_hub_misses* misses) {
    if (!h) return BB_ERR_ARG;
    h->m_pkts.clear(); h->m_off.assign(1, 0); h->m_sid.clear(); h->qlog[0].clear();
    const size_t total = h->q_sid.size();
    int rc = BB_OK;
    uint32_t qidx = 0;                                 // (seed, qidx) keys the service shuffle: it does not repeat across batches
    for (size_t i = 0; i < total;) {
        uint32_t n = 0, bytes = 0;
        h->pkt_off[0] = 0;
        while (i < total && n < h->max_batch) {
            const uint32_t a = h->q_off[i], ln = h->q_off[i + 1] - a;
            TcpSession* s = h->find(h->q_sid[i]);
            if (!s || ln > h->max_bytes) {              // its session is gone / it fits no batch
                h->n_dropped++; if (s) s->queued--; i++; continue;
            }
            if (bytes + ln > h->max_bytes) break;
            memcpy(h->pkts + bytes, h->q_bytes.data() + a, ln);
            bytes += ln; h->pkt_off[n + 1] = bytes; h->b_sid[n] = h->q_sid[i];
            n++; i++;
        }
        if (n == 0) continue;
        uint32_t n_miss = 0;
        const int r = bb_resolve_batch_ex(h->e, h->pkts, h->pkt_off, n, shuffle_seed, qidx, h->resp, h->resp_cap, h->resp_off,
                                          h->resp_len, h->status, h->miss, &n_miss, BB_BATCH_TCP);
        qidx += n;
        if (r != BB_OK) {                               // the batch's queries are lost (counted); the next batch still runs
            if (rc == BB_OK) rc = r;
            h->n_failed += n;
            for (uint32_t k = 0; k < n; k++) h->find(h->b_sid[k])->queued--;
            continue;
        }
        // the answers are appended below in query order, each to the session that asked
        h->qlog[0].batch(h->e, h->resp, h->resp_off, h->resp_len, h->status, n, [h](uint32_t k, uint32_t& ip, uint32_t& port, uint32_t& sid) {
            const TcpSession* s = h->find(h->b_sid[k]);
            ip = s->ip; port = s->port; sid = h->b_sid[k]; return true;
        });
        // per session in arrival order; misses in query order whatever the packing
        TcpSession* s = nullptr; uint32_t sid = 0;
        for (uint32_t k = 0; k < n; k++) {
            if (!s || sid != h->b_sid[k]) { sid = h->b_sid[k]; s = h->find(sid); }
            s->queued--;
            if (h->status[k] == BB_ANSWERED) {
                h->n_answered++;
                s->put(h->resp + h->resp_off[k], h->resp_len[k]);
            } else if (h->status[k] == BB_MISS_RECURSE) {
                h->n_missed++; s->relays++;
                h->m_pkts.insert(h->m_pkts.end(), h->pkts + h->pkt_off[k], h->pkts + h->pkt_off[k + 1]);
                h->m_off.push_back((uint32_t)h->m_pkts.size()); h->m_sid.push_back(sid);
            } else {
                h->n_dropped++;
            }
        }
    }
    h->q_bytes.clear(); h->q_off.assign(1, 0); h->q_sid.clear();
    if (misses) {
        misses->n = (uint32_t)h->m_sid.size(); misses->pkts = h->m_pkts.data(); misses->pkt_off = h->m_off.data();
        misses->session = h->m_sid.data();
    }
    return rc;
}

int bb_tcp_hub_output(bb_tcp_hub* h, uint32_t session, const uint8_t** out, size_t* out_len, int* closable) {
    TcpSession* s = h ? h->find(session) : nullptr;
    if (!s || !out || !out_len) return BB_ERR_ARG;
    *out = s->out.data() + s->head; *out_len = s->out.size() - s->head;
    if (closable) *closable = (s->eof || s->bad) && !s->queued && !s->relays && *out_len == 0;
    return BB_OK;
}

int bb_tcp_hub_consume(bb_tcp_hub* h, uint32_t session, size_t n) {
    TcpSession* s = h ? h->find(session) : nullptr;
    if (!s || n > s->out.size() - s->head) return BB_ERR_ARG;
    s->head += n;
    if (s->head == s->out.size()) { s->out.clear(); s->head = 0; }
    else if (s->head >= (1u << 16) && s->head * 2 >= s->out.size()) {      // keep the written prefix from piling up
        s->out.erase(s->out.begin(), s->out.begin() + (long)s->head); s->head = 0;
    }
    return BB_OK;
}

int bb_tcp_hub_close(bb_tcp_hub* h, uint32_t session) {
    if (!h || !h->sess.erase(session)) return BB_ERR_ARG;
    return BB_OK;
}

int bb_tcp_hub_relay(bb_tcp_hub* h, const uint8_t* q_pkts, const uint32_t* q_off, const uint8_t* up_pkts,
                     const uint32_t* up_off, const uint32_t* sessions, uint32_t n) {
    if (!h) return BB_ERR_ARG;
    h->qlog[1].clear();
    if (n == 0) return BB_OK;
    if (!q_off || !up_off || !sessions || (q_off[n] != q_off[0] && !q_pkts) || (up_off[n] != up_off[0] && !up_pkts)) return BB_ERR_ARG;
    for (uint32_t i = 0; i < n; i++) if (q_off[i + 1] < q_off[i] || up_off[i + 1] < up_off[i]) return BB_ERR_ARG;
    int rc = BB_OK;
    for (uint32_t k0 = 0; k0 < n; k0 += h->max_batch) {
        const uint32_t m = std::min(h->max_batch, n - k0);
        h->r_qoff.resize(m + 1); h->r_upoff.resize(m + 1);
        for (uint32_t j = 0; j <= m; j++) { h->r_qoff[j] = q_off[k0 + j] - q_off[k0]; h->r_upoff[j] = up_off[k0 + j] - up_off[k0]; }
        const int r = bb_relay_batch(h->e, q_pkts ? q_pkts + q_off[k0] : nullptr, h->r_qoff.data(), up_pkts ? up_pkts + up_off[k0] : nullptr,
                                     h->r_upoff.data(), m, BB_BATCH_TCP, h->resp, h->resp_cap, h->resp_off, h->resp_len, h->status);
        // a reply is appended (and has a record) when its session is still open
        if (r == BB_OK)
            h->qlog[1].batch(h->e, h->resp, h->resp_off, h->resp_len, h->status, m, [&](uint32_t j, uint32_t& ip, uint32_t& port, uint32_t& sid) {
                const TcpSession* s = h->find(sessions[k0 + j]);
                if (!s) return false;
                ip = s->ip; port = s->port; sid = sessions[k0 + j]; return true;
            });
        for (uint32_t j = 0; j < m; j++) {
            TcpSession* s = h->find(sessions[k0 + j]);
            if (s && s->relays) s->relays--;
            if (r != BB_OK) { h->n_failed++; continue; }
            if (!s || h->status[j] != BB_ANSWERED) { h->n_dropped++; continue; }     // closed meanwhile / query does not decode
            s->put(h->resp + h->resp_off[j], h->resp_len[j]);
            h->n_relayed++;
        }
        if (r != BB_OK && rc == BB_OK) rc = r;
    }
    return rc;
}

int bb_tcp_hub_peer(const bb_tcp_hub* h, uint32_t session, uint32_t* ip, uint32_t* port) {
    if (!h || !ip || !port) return BB_ERR_ARG;
    auto it = h->sess.find(session);
    if (it == h->sess.end()) return BB_ERR_ARG;
    *ip = it->second.ip; *port = it->second.port;      // 0, 0 until the handshake
    return BB_OK;
}

uint64_t bb_tcp_hub_stat(const bb_tcp_hub* h, int what) {
    if (!h) return 0;
    switch (what) {
    case 0: return h->n_sessions; case 1: return h->n_msgs; case 2: return h->n_answered; case 3: return h->n_missed;
    case 4: return h->n_dropped; case 5: return h->n_proto; case 6: return h->n_failed; case 7: return h->n_relayed;
    case 8: return h->sess.size(); case 9: return h->q_sid.size(); case 10: return h->resp_cap;
    case 11: return h->qlog[0].n_records + h->qlog[1].n_records; case 12: return h->qlog[0].n_lost + h->qlog[1].n_lost;
    }
    return 0;
}

}  // extern "C"
