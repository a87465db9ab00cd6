// mname-balancer backend protocol, natively (SURVEY.md section 8f row 1).
//
// The balancer (deps/mname-balancer) relays every UDP packet it receives to a backend process over an
// AF_UNIX stream socket as a frame, all integers u32 little-endian (backend.c:22-113, types bbal.h:80-87):
//     INBOUND_UDP   { type = 2,    source IPv4, source port, length, packet bytes }
//     OUTBOUND_UDP  { type = 1002, dest IPv4,   dest port,   length, packet bytes }        (the answer)
//     CLIENT_HELLO 1 -> SERVER_HELLO 1001, CLIENT_HEARTBEAT 4 -> SERVER_HEARTBEAT 1004    (bare type words)
// which is already "batched raw packets + source address".  bb_frames_parse turns a byte stream into the
// engine's batch container, bb_frames_build turns results back into frames, and bb_backend is a session that
// does both around bb_resolve_batch, so a native backend can sit on the socket where a Node backend
// (lib/server.js:621-631 -> mname) sits today (its relays, bb_backend_relay: balancer_relay.cpp).  Host code only: no
// CUDA in this file.
#include "balancer_backend.h"

#include <cstring>

namespace {
inline uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
inline void wr32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }
constexpr uint32_t MAX_UDP = 1500;             // deps/mname-balancer/udp_proxy.c:159-170, backend.c:709-716
}

extern "C" {

int bb_frames_parse(const uint8_t* in, size_t in_len, uint8_t* pkts, uint32_t cap_bytes, uint32_t* pkt_off,
                    uint32_t* src_ip, uint32_t* src_port, uint32_t cap_n, uint32_t* n_out,
                    uint32_t* control, uint32_t cap_ctrl, uint32_t* n_ctrl_out, size_t* consumed) {
    if ((!in && in_len) || !pkt_off || !n_out || !n_ctrl_out || !consumed || (cap_n && (!pkts || !src_ip || !src_port)) || (cap_ctrl && !control))
        return BB_ERR_ARG;
    size_t pos = 0; uint32_t n = 0, nc = 0, bytes = 0;
    pkt_off[0] = 0;
    int rc = BB_OK;
    while (pos + 4 <= in_len) {
        const uint32_t t = rd32(in + pos);
        if (t == BB_FRAME_CLIENT_HELLO || t == BB_FRAME_CLIENT_HEARTBEAT) {
            if (nc == cap_ctrl) break;                              // the caller drains and calls again
            control[nc++] = t; pos += 4;
        } else if (t == BB_FRAME_INBOUND_UDP) {
            if (pos + 16 > in_len) break;
            const uint32_t ln = rd32(in + pos + 12);
            if (ln > MAX_UDP) { rc = BB_ERR_PROTOCOL; break; }
            if (pos + 16 + (size_t)ln > in_len) break;
            if (n == cap_n || bytes + ln > cap_bytes) break;        // batch full: the rest stays for the next call
            src_ip[n] = rd32(in + pos + 4); src_port[n] = rd32(in + pos + 8);
            memcpy(pkts + bytes, in + pos + 16, ln);
            bytes += ln; pkt_off[++n] = bytes;
            pos += 16 + (size_t)ln;
        } else {                                                    // INBOUND_TCP turns the session into a TCP proxy; anything else is noise
            rc = BB_ERR_PROTOCOL; break;
        }
    }
    *n_out = n; *n_ctrl_out = nc; *consumed = pos;
    return rc;
}

int bb_frames_build(const uint8_t* resp, const uint32_t* resp_off, const uint16_t* resp_len, const uint8_t* status,
                    const uint32_t* dst_ip, const uint32_t* dst_port, uint32_t n, const uint32_t* control, uint32_t n_ctrl,
                    uint8_t* out, size_t out_cap, size_t* out_len) {
    if (!out_len || (n && (!resp_off || !resp_len || !status || !dst_ip || !dst_port)) || (n_ctrl && !control)) return BB_ERR_ARG;
    size_t need = 4 * (size_t)n_ctrl;
    for (uint32_t i = 0; i < n; i++) if (status[i] == BB_ANSWERED) need += 16 + (size_t)resp_len[i];
    *out_len = need;
    if (need > out_cap || (need && !out)) return BB_ERR_CAPACITY;
    uint8_t* w = out;
    for (uint32_t c = 0; c < n_ctrl; c++, w += 4) wr32(w, control[c] == BB_FRAME_CLIENT_HELLO ? BB_FRAME_SERVER_HELLO : BB_FRAME_SERVER_HEARTBEAT);
    for (uint32_t i = 0; i < n; i++) {
        if (status[i] != BB_ANSWERED) continue;                     // misses go to recursion, drops get no answer
        wr32(w, BB_FRAME_OUTBOUND_UDP); wr32(w + 4, dst_ip[i]); wr32(w + 8, dst_port[i]); wr32(w + 12, resp_len[i]);
        if (resp_len[i]) { if (!resp) return BB_ERR_ARG; memcpy(w + 16, resp + resp_off[i], resp_len[i]); }
        w += 16 + (size_t)resp_len[i];
    }
    return BB_OK;
}

}  // extern "C"

// ---- one balancer session around an engine (struct bb_backend: balancer_backend.h) -------------------
extern "C" {

bb_backend* bb_backend_create(bb_engine* e, uint32_t max_batch, int* err) {
    if (err) *err = BB_OK;
    if (!e || max_batch == 0) { if (err) *err = BB_ERR_ARG; return nullptr; }
    // never parse a batch the engine would refuse: its own limits bound the session's
    if (max_batch > bb_engine_max_batch(e)) max_batch = bb_engine_max_batch(e);
    bb_backend* b = new bb_backend();
    b->e = e; b->max_batch = max_batch; b->max_bytes = max_batch * 64u > (1u << 16) ? max_batch * 64u : (1u << 16);
    if (b->max_bytes > bb_engine_max_batch_bytes(e)) b->max_bytes = bb_engine_max_batch_bytes(e);
    b->resp_cap = max_batch * 512u > (1u << 20) ? max_batch * 512u : (1u << 20);
    b->pkts = (uint8_t*)bb_host_alloc(b->max_bytes + 64); b->pkt_off = (uint32_t*)bb_host_alloc(((size_t)max_batch + 1) * 4);
    b->ip = (uint32_t*)bb_host_alloc((size_t)max_batch * 4); b->port = (uint32_t*)bb_host_alloc((size_t)max_batch * 4);
    b->resp = (uint8_t*)bb_host_alloc(b->resp_cap); b->resp_off = (uint32_t*)bb_host_alloc(((size_t)max_batch + 1) * 4);
    b->resp_len = (uint16_t*)bb_host_alloc((size_t)max_batch * 2 + 16); b->status = (uint8_t*)bb_host_alloc((size_t)max_batch + 16);
    b->miss = (uint32_t*)bb_host_alloc((size_t)max_batch * 4);
    if (!b->pkts || !b->pkt_off || !b->ip || !b->port || !b->resp || !b->resp_off || !b->resp_len || !b->status || !b->miss) {
        bb_backend_destroy(b); if (err) *err = BB_ERR_NOMEM; return nullptr;
    }
    memset(b->pkts, 0, b->max_bytes + 64);
    b->qlog[0].max_batch = b->qlog[1].max_batch = max_batch;
    return b;
}

void bb_backend_destroy(bb_backend* b) {
    if (!b) return;
    bb_host_free(b->pkts); bb_host_free(b->pkt_off); bb_host_free(b->ip); bb_host_free(b->port); bb_host_free(b->resp);
    bb_host_free(b->resp_off); bb_host_free(b->resp_len); bb_host_free(b->status); bb_host_free(b->miss);
    b->qlog[0].release(); b->qlog[1].release();
    delete b;
}

int bb_backend_feed(bb_backend* b, const uint8_t* in, size_t in_len, uint64_t shuffle_seed,
                    const uint8_t** out, size_t* out_len, bb_backend_misses* misses) {
    if (!b || (!in && in_len) || !out || !out_len) return BB_ERR_ARG;
    b->pending.insert(b->pending.end(), in, in + in_len);
    b->out.clear(); b->m_pkts.clear(); b->m_off.assign(1, 0); b->m_ip.clear(); b->m_port.clear(); b->qlog[0].clear();
    size_t pos = 0; int rc = BB_OK;
    b->qidx_next = 0;                                   // (seed, index) keys the shuffle: indices run over the queries of this feed
    for (;;) {
        uint32_t n = 0, nc = 0, control[64]; size_t used = 0;
        rc = bb_frames_parse(b->pending.data() + pos, b->pending.size() - pos, b->pkts, b->max_bytes, b->pkt_off, b->ip, b->port,
                             b->max_batch, &n, control, 64, &nc, &used);
        pos += used;
        if (n == 0 && nc == 0) break;
        uint32_t n_miss = 0;
        if (n) {
            // qidx_base advances per batch: the service shuffle (keyed on seed and query index) does not repeat across the
            // batches of one feed
            int r2 = bb_resolve_batch(b->e, b->pkts, b->pkt_off, n, shuffle_seed, b->qidx_next, b->resp, b->resp_cap, b->resp_off, b->resp_len,
                                      b->status, b->miss, &n_miss);
            b->qidx_next += n;
            if (r2 != BB_OK) {
                // the batch's queries are lost (counted), the control frames parsed with it are still answered
                rc = r2; b->n_failed += n;
                size_t need = 0;
                bb_frames_build(b->resp, b->resp_off, b->resp_len, b->status, b->ip, b->port, 0, control, nc, nullptr, 0, &need);
                const size_t at = b->out.size();
                b->out.resize(at + need);
                if (need) bb_frames_build(b->resp, b->resp_off, b->resp_len, b->status, b->ip, b->port, 0, control, nc, b->out.data() + at, need, &need);
                break;
            }
            // record i of the batch goes with its OUTBOUND_UDP frame, which bb_frames_build below writes in index order
            b->qlog[0].batch(b->e, b->resp, b->resp_off, b->resp_len, b->status, n, [b](uint32_t i, uint32_t& ip, uint32_t& port, uint32_t&) {
                ip = b->ip[i]; port = b->port[i]; return true;
            });
            b->n_udp += n; b->n_missed += n_miss;
            for (uint32_t i = 0; i < n; i++) { b->n_answered += b->status[i] == BB_ANSWERED; b->n_dropped += b->status[i] == BB_DROPPED; }
            for (uint32_t k = 0; k < n_miss; k++) {                     // lib/server.js:110-113,222-225: these go to recursion
                const uint32_t i = b->miss[k];
                b->m_pkts.insert(b->m_pkts.end(), b->pkts + b->pkt_off[i], b->pkts + b->pkt_off[i + 1]);
                b->m_off.push_back((uint32_t)b->m_pkts.size()); b->m_ip.push_back(b->ip[i]); b->m_port.push_back(b->port[i]);
            }
        }
        size_t need = 0;
        bb_frames_build(b->resp, b->resp_off, b->resp_len, b->status, b->ip, b->port, n, control, nc, nullptr, 0, &need);
        const size_t at = b->out.size();
        b->out.resize(at + need);
        if (need) bb_frames_build(b->resp, b->resp_off, b->resp_len, b->status, b->ip, b->port, n, control, nc, b->out.data() + at, need, &need);
        if (rc != BB_OK) break;
    }
    b->pending.erase(b->pending.begin(), b->pending.begin() + (long)pos);
    *out = b->out.data(); *out_len = b->out.size();
    if (misses) {
        misses->n = (uint32_t)b->m_ip.size(); misses->pkts = b->m_pkts.data(); misses->pkt_off = b->m_off.data();
        misses->src_ip = b->m_ip.data(); misses->src_port = b->m_port.data();
    }
    return rc;
}

uint64_t bb_backend_stat(const bb_backend* b, int what) {
    if (!b) return 0;
    switch (what) { case 0: return b->n_udp; case 1: return b->n_answered; case 2: return b->n_missed; case 3: return b->n_dropped; case 4: return b->pending.size(); case 5: return b->n_failed;
                    case 6: return b->n_relayed; case 7: return b->n_relay_failed;
                    case 8: return b->qlog[0].n_records + b->qlog[1].n_records; case 9: return b->qlog[0].n_lost + b->qlog[1].n_lost; }
    return 0;
}

}  // extern "C"
