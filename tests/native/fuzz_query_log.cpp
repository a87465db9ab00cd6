// The balancer sessions' query-log host code (bb_log_set in csrc/balancer_backend.h, used by balancer_frames.cpp,
// balancer_relay.cpp and balancer_tcp.cpp, switched on by balancer_query_log.cpp) under ASan/UBSan, with the engine stubbed out.  Every answer is its query's
// bytes, packed in reverse index order; the stand-in bb_log_batch reads every byte of every answered response and writes
// a record derived from it (reverse-packed too), and now and then reports BB_ERR_CAPACITY (with the bytes it needed, as
// the kernel leaves them) or fails outright.  The driver feeds random frame streams, hub sessions and relays with the log
// on and checks each record against the frame or answer it belongs to.  Test infrastructure only.
#include "binder_b200.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <random>
#include <vector>

static std::mt19937 g_rng(11);
static uint32_t g_max_batch = 64;

static std::vector<uint8_t> record_of(const uint8_t* r, uint32_t len) {      // the stand-in's record of one response
    std::vector<uint8_t> v(1 + len % 97);
    for (size_t k = 0; k < v.size(); k++) v[k] = (uint8_t)((len ? r[k % len] : 0) ^ k);
    return v;
}

// answers: query i -> its bytes (answered, missed or dropped at random; a relay: answered when it has an upstream), packed
// in reverse order
static int answer(const uint8_t* q, const uint32_t* q_off, const uint32_t* up_off, uint32_t n, uint8_t* out, uint32_t out_cap,
                  uint32_t* out_off, uint16_t* out_len, uint8_t* status, uint32_t* miss, uint32_t* n_miss) {
    uint32_t pos = 0, nm = 0;
    for (uint32_t j = n; j-- > 0;) {
        const uint32_t ql = q_off[j + 1] - q_off[j];
        const uint32_t roll = g_rng() % 10;
        status[j] = up_off ? (up_off[j + 1] > up_off[j] ? BB_ANSWERED : BB_DROPPED)
                           : (ql < 2 || roll < 2 ? BB_DROPPED : roll < 4 && miss ? BB_MISS_RECURSE : BB_ANSWERED);
        out_off[j] = pos; out_len[j] = 0;
        if (status[j] == BB_ANSWERED) {
            if (pos + ql > out_cap) return BB_ERR_CAPACITY;
            memcpy(out + pos, q + q_off[j], ql); out_len[j] = (uint16_t)ql; pos += ql;
        } else if (status[j] == BB_MISS_RECURSE) {
            miss[nm++] = j;
        }
    }
    out_off[n] = pos;
    if (n_miss) *n_miss = nm;
    return g_rng() % 40 == 0 ? BB_ERR_CUDA : BB_OK;
}

extern "C" {
void* bb_host_alloc(size_t n) { return malloc(n ? n : 1); }
void bb_host_free(void* p) { free(p); }
uint32_t bb_engine_max_batch(const bb_engine*) { return g_max_batch; }
uint32_t bb_engine_max_batch_bytes(const bb_engine*) { return 1u << 22; }
int bb_resolve_batch_ex(bb_engine*, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n, uint64_t, uint32_t, uint8_t* out,
                        uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status, uint32_t* miss, uint32_t* n_miss, uint32_t) {
    return answer(pkts, pkt_off, nullptr, n, out, out_cap, out_off, out_len, status, miss, n_miss);
}
int bb_resolve_batch(bb_engine* e, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n, uint64_t seed, uint32_t qidx, uint8_t* out,
                     uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status, uint32_t* miss, uint32_t* n_miss) {
    return bb_resolve_batch_ex(e, pkts, pkt_off, n, seed, qidx, out, out_cap, out_off, out_len, status, miss, n_miss, 0);
}
int bb_relay_batch(bb_engine*, const uint8_t* q, const uint32_t* q_off, const uint8_t*, const uint32_t* up_off, uint32_t n, uint32_t,
                   uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status) {
    return answer(q, q_off, up_off, n, out, out_cap, out_off, out_len, status, nullptr, nullptr);
}
int bb_log_batch(bb_engine*, const uint8_t* resp, uint32_t resp_bytes, const uint32_t* out_off, const uint16_t* out_len,
                 const uint8_t* status, uint32_t n, uint8_t* log, uint32_t log_cap, uint32_t* log_off, uint32_t* log_len,
                 uint16_t* head_len, uint32_t*) {
    if (((uintptr_t)log & 15) != 0) return BB_ERR_ARG;         // the sessions start every batch 16-byte aligned
    std::vector<std::vector<uint8_t>> recs(n);
    uint32_t total = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (status[i] != BB_ANSWERED) continue;
        if (out_off[i] + (uint64_t)out_len[i] > resp_bytes) return BB_ERR_ARG;
        recs[i] = record_of(resp + out_off[i], out_len[i]);
        total += (uint32_t)recs[i].size();
    }
    log_off[n] = total;
    const uint32_t roll = g_rng() % 25;
    if (roll == 0) return BB_ERR_CUDA;
    if (total > log_cap || roll == 1) return BB_ERR_CAPACITY;
    uint32_t pos = 0;
    for (uint32_t i = n; i-- > 0;) {
        log_off[i] = pos; log_len[i] = (uint32_t)recs[i].size(); head_len[i] = (uint16_t)(recs[i].size() < 3 ? recs[i].size() : 3);
        if (!recs[i].empty()) memcpy(log + pos, recs[i].data(), recs[i].size());
        pos += (uint32_t)recs[i].size();
    }
    return BB_OK;
}
}

static uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
static void wr32(std::vector<uint8_t>& v, uint32_t x) { for (int k = 0; k < 4; k++) v.push_back((uint8_t)(x >> (8 * k))); }

struct Sent { uint32_t ip, port, sid; std::vector<uint8_t> msg; };

// The records against the answers sent, in order: a record for each answer except those of lost batches, whose count
// is r.lost.  Every record's bytes are read (ASan sees a record outside the log buffer).
static bool check(const bb_query_log_records& r, const std::vector<Sent>& sent, bool hub, const char* what) {
    size_t j = 0;
    for (uint32_t i = 0; i < r.n; i++) {
        bool hit = false;
        for (; j < sent.size() && !hit; j++) {
            const Sent& s = sent[j];
            const std::vector<uint8_t> want = record_of(s.msg.data(), (uint32_t)s.msg.size());
            hit = r.log_len[i] == want.size() && !memcmp(r.log + r.log_off[i], want.data(), want.size()) &&
                  r.head_len[i] == (want.size() < 3 ? want.size() : 3) && r.req_id[i] == (s.msg.size() >= 2 ? (uint16_t)(s.msg[0] << 8 | s.msg[1]) : 0) &&
                  r.client_ip[i] == s.ip && r.client_port[i] == s.port && (hub ? r.session && r.session[i] == s.sid : !r.session);
        }
        if (!hit) { printf("%s: record %u matches no answer\n", what, i); return false; }
    }
    if (r.n + r.lost != sent.size()) { printf("%s: %u records + %u lost != %zu answers\n", what, r.n, r.lost, sent.size()); return false; }
    return true;
}

static std::vector<Sent> udp_frames(const uint8_t* out, size_t len) {
    std::vector<Sent> v;
    for (size_t pos = 0; pos < len;) {
        const uint32_t t = rd32(out + pos);
        if (t != BB_FRAME_OUTBOUND_UDP) { pos += 4; continue; }
        const uint32_t ln = rd32(out + pos + 12);
        v.push_back({ rd32(out + pos + 4), rd32(out + pos + 8), 0, std::vector<uint8_t>(out + pos + 16, out + pos + 16 + ln) });
        pos += 16 + ln;
    }
    return v;
}

static std::vector<uint8_t> message() {
    std::vector<uint8_t> m(g_rng() % 300);
    for (auto& c : m) c = (uint8_t)g_rng();
    return m;
}

int main(int argc, char** argv) {
    const int iters = argc > 1 ? atoi(argv[1]) : 300;
    static int engine;                                 // the sessions only hand the handle back to the stubs
    for (int it = 0; it < iters; it++) {
        g_max_batch = 1 + g_rng() % 48;
        int err = 0;
        // ---- UDP backend: feed, then relay ----
        bb_backend* b = bb_backend_create((bb_engine*)&engine, 1 + g_rng() % 64, &err);
        if (!b || bb_query_log_backend_enable(b, 1) != BB_OK) { printf("backend create failed %d\n", err); return 1; }
        std::vector<uint8_t> in;
        const uint32_t nq = g_rng() % 300;
        for (uint32_t i = 0; i < nq; i++) {
            if (g_rng() % 20 == 0) wr32(in, g_rng() % 2 ? BB_FRAME_CLIENT_HELLO : BB_FRAME_CLIENT_HEARTBEAT);
            const std::vector<uint8_t> m = message();
            wr32(in, BB_FRAME_INBOUND_UDP); wr32(in, g_rng()); wr32(in, g_rng() & 0xFFFF); wr32(in, (uint32_t)m.size());
            in.insert(in.end(), m.begin(), m.end());
        }
        const uint8_t* out = nullptr; size_t out_len = 0;
        bb_backend_misses ms;
        bb_backend_feed(b, in.data(), in.size(), 1, &out, &out_len, &ms);
        bb_query_log_records r;
        if (bb_query_log_backend(b, 0, &r) != BB_OK || !check(r, udp_frames(out, out_len), false, "feed")) return 1;
        std::vector<uint8_t> q, up; std::vector<uint32_t> qo{0}, uo{0}, ip, port;
        for (uint32_t i = 0, n = g_rng() % 200; i < n; i++) {
            const std::vector<uint8_t> m = message();
            q.insert(q.end(), m.begin(), m.end()); qo.push_back((uint32_t)q.size());
            for (uint32_t k = 0, ul = g_rng() % 3 ? 1 + g_rng() % 50 : 0; k < ul; k++) up.push_back((uint8_t)g_rng());
            uo.push_back((uint32_t)up.size()); ip.push_back(g_rng()); port.push_back(g_rng() & 0xFFFF);
        }
        const uint8_t* rout = nullptr; size_t rlen = 0;
        bb_backend_relay(b, q.data(), qo.data(), up.data(), uo.data(), ip.data(), port.data(), (uint32_t)ip.size(), &rout, &rlen);
        if (bb_query_log_backend(b, 1, &r) != BB_OK || !check(r, udp_frames(rout, rlen), false, "relay")) return 1;
        if (bb_query_log_backend(b, 0, &r) != BB_OK || !check(r, udp_frames(out, out_len), false, "feed after relay")) return 1;
        if (bb_backend_stat(b, 8) + bb_backend_stat(b, 9) != udp_frames(out, out_len).size() + udp_frames(rout, rlen).size()) {
            printf("backend stats\n"); return 1;
        }
        bb_backend_destroy(b);

        // ---- TCP hub: sessions (one not a TCP session), flush, a session closed, relay ----
        bb_tcp_hub* h = bb_tcp_hub_create((bb_engine*)&engine, 1 + g_rng() % 64, &err);
        if (!h || bb_query_log_tcp_hub_enable(h, 1) != BB_OK) { printf("hub create failed %d\n", err); return 1; }
        std::map<uint32_t, std::pair<uint32_t, uint32_t>> peer;
        std::vector<uint32_t> sids;
        for (uint32_t k = 0, ns = 1 + g_rng() % 8; k < ns; k++) {
            uint32_t sid = 0; bb_tcp_hub_open(h, &sid); sids.push_back(sid);
            std::vector<uint8_t> s;
            const bool bad = g_rng() % 6 == 0;
            wr32(s, bad ? BB_FRAME_CLIENT_HELLO : BB_FRAME_INBOUND_TCP);
            const uint32_t pip = g_rng(), pport = g_rng() & 0xFFFF;
            wr32(s, pip); wr32(s, pport); peer[sid] = { pip, pport };
            for (uint32_t i = 0, n = g_rng() % 40; i < n; i++) {
                std::vector<uint8_t> m = message();
                if (m.empty()) m.push_back(0);
                s.push_back((uint8_t)(m.size() >> 8)); s.push_back((uint8_t)m.size()); s.insert(s.end(), m.begin(), m.end());
            }
            bb_tcp_hub_feed(h, sid, s.data(), s.size());
        }
        std::map<uint32_t, size_t> seen;               // output bytes of each session before the call
        auto answers = [&]() {                         // the answers appended since `seen`, session by session
            std::map<uint32_t, std::vector<std::vector<uint8_t>>> a;
            for (uint32_t sid : sids) {
                const uint8_t* o; size_t ol;
                if (bb_tcp_hub_output(h, sid, &o, &ol, nullptr) != BB_OK) continue;
                size_t pos = seen[sid] ? seen[sid] : (ol >= 4 ? 4 : ol);
                for (; pos + 2 <= ol; pos += 2 + ((size_t)o[pos] << 8 | o[pos + 1]))
                    a[sid].push_back(std::vector<uint8_t>(o + pos + 2, o + pos + 2 + ((size_t)o[pos] << 8 | o[pos + 1])));
                seen[sid] = ol;
            }
            return a;
        };
        bb_tcp_hub_misses hm;
        answers();
        bb_tcp_hub_flush(h, 1, &hm);
        auto hub_check = [&](int which, const char* what) {
            auto a = answers();
            bb_query_log_records hr;
            if (bb_query_log_tcp_hub(h, which, &hr) != BB_OK) return false;
            // per session the records follow its answers; across sessions the stand-in's order is already checked by
            // the session ids the records carry
            size_t total = 0;
            for (auto& kv : a) {
                std::vector<Sent> sent;
                for (auto& m : kv.second) sent.push_back({ peer[kv.first].first, peer[kv.first].second, kv.first, m });
                std::vector<uint32_t> idx;
                for (uint32_t i = 0; i < hr.n; i++) if (hr.session[i] == kv.first) idx.push_back(i);
                for (size_t t = 0; t < idx.size(); t++) {
                    const uint32_t i = idx[t];
                    bool hit = false;
                    for (auto& s : sent) {
                        const std::vector<uint8_t> want = record_of(s.msg.data(), (uint32_t)s.msg.size());
                        hit |= hr.log_len[i] == want.size() && !memcmp(hr.log + hr.log_off[i], want.data(), want.size()) &&
                               hr.client_ip[i] == s.ip && hr.client_port[i] == s.port;
                    }
                    if (!hit) { printf("%s: record %u matches no answer of session %u\n", what, i, kv.first); return false; }
                }
                total += sent.size();
            }
            if (hr.n + hr.lost != total) { printf("%s: %u + %u != %zu\n", what, hr.n, hr.lost, total); return false; }
            return true;
        };
        if (!hub_check(0, "flush")) return 1;
        std::vector<uint8_t> mq(hm.pkts, hm.pkts + hm.pkt_off[hm.n]); std::vector<uint32_t> mo(hm.pkt_off, hm.pkt_off + hm.n + 1);
        std::vector<uint32_t> ms_sid(hm.session, hm.session + hm.n), muo{0};
        std::vector<uint8_t> mup;
        for (uint32_t i = 0; i < hm.n; i++) { if (g_rng() % 4) mup.push_back(1); muo.push_back((uint32_t)mup.size()); }
        if (hm.n && g_rng() % 2) {                     // a session closed between the flush and the relay
            const uint32_t gone = ms_sid[0];
            bb_tcp_hub_close(h, gone);
            sids.erase(std::find(sids.begin(), sids.end(), gone));
        }
        bb_tcp_hub_relay(h, mq.data(), mo.data(), mup.data(), muo.data(), ms_sid.data(), hm.n);
        if (!hub_check(1, "hub relay")) return 1;
        bb_query_log_tcp_hub_enable(h, 0);
        bb_query_log_records hr;
        if (bb_query_log_tcp_hub(h, 0, &hr) != BB_OK || hr.n != 0 || bb_query_log_tcp_hub(h, 2, &hr) != BB_ERR_ARG) return 1;
        bb_tcp_hub_destroy(h);
    }
    printf("OK\n");
    return 0;
}
