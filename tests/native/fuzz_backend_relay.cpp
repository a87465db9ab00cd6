// bb_backend_relay's host code (csrc/balancer_relay.cpp) under ASan/UBSan, with the engine stubbed out: the stand-in
// bb_relay_batch reads every byte of every query and upstream it is given (so an offset the session rebased wrongly is
// an out-of-bounds read), answers a relay whose upstream is non-empty with the query bytes, and fails every batch
// that holds a relay marked to fail.  Upstreams are random bytes, empty, or long.  Each call's frames are parsed back
// and checked against what the stub answered.  Test infrastructure only.
//   fuzz_backend_relay <iterations>  -> prints OK
#include "binder_b200.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

static uint32_t g_max_batch = 64;
static const uint8_t kFail = 0xEE;                     // an upstream starting with this byte fails its batch

extern "C" {
void* bb_host_alloc(size_t n) { return malloc(n ? n : 1); }
void bb_host_free(void* p) { free(p); }
uint32_t bb_engine_max_batch(const bb_engine*) { return g_max_batch; }
uint32_t bb_engine_max_batch_bytes(const bb_engine*) { return 1u << 22; }
int bb_resolve_batch(bb_engine*, const uint8_t*, const uint32_t*, uint32_t, uint64_t, uint32_t, uint8_t*, uint32_t, uint32_t*,
                     uint16_t*, uint8_t*, uint32_t*, uint32_t*) { return BB_ERR_NO_DEVICE; }
int bb_relay_batch(bb_engine*, const uint8_t* q, const uint32_t* q_off, const uint8_t* up, const uint32_t* up_off, uint32_t n,
                   uint32_t flags, uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status) {
    if (flags != 0 || q_off[0] != 0 || up_off[0] != 0) return BB_ERR_ARG;
    volatile uint32_t sum = 0;
    bool fail = false;
    uint32_t pos = 0;
    for (uint32_t i = 0; i < n; i++) {
        for (uint32_t k = up_off[i]; k < up_off[i + 1]; k++) sum += up[k];
        const uint32_t ql = q_off[i + 1] - q_off[i];
        for (uint32_t k = 0; k < ql; k++) sum += q[q_off[i] + k];
        fail |= up_off[i + 1] > up_off[i] && up[up_off[i]] == kFail;
        const bool ans = up_off[i + 1] > up_off[i];
        out_off[i] = pos; out_len[i] = ans ? (uint16_t)ql : 0; status[i] = ans ? BB_ANSWERED : BB_DROPPED;
        if (ans) {
            if (pos + ql > out_cap) return BB_ERR_CAPACITY;
            memcpy(out + pos, q + q_off[i], ql);
            pos += ql;
        }
    }
    out_off[n] = pos;
    return fail ? BB_ERR_CUDA : BB_OK;
}
}

static uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }

int main(int argc, char** argv) {
    const int iters = argc > 1 ? atoi(argv[1]) : 500;
    std::mt19937 rng(7);
    for (int it = 0; it < iters; it++) {
        g_max_batch = 1 + rng() % 48;
        static int engine;                             // the session only hands the handle back to the stubs
        int err = 0;
        bb_backend* b = bb_backend_create((bb_engine*)&engine, 1 + rng() % 64, &err);
        if (!b) { printf("create failed %d\n", err); return 1; }
        const uint32_t n = rng() % 200;
        std::vector<uint8_t> q, up; std::vector<uint32_t> qo{0}, uo{0}, ip(n), port(n);
        std::vector<int> fails(n);
        for (uint32_t i = 0; i < n; i++) {
            const uint32_t ql = rng() % 600;
            for (uint32_t k = 0; k < ql; k++) q.push_back((uint8_t)rng());
            qo.push_back((uint32_t)q.size());
            const uint32_t kind = rng() % 10, ul = kind < 3 ? 0 : kind < 9 ? rng() % 700 : 4000 + rng() % 60000;
            for (uint32_t k = 0; k < ul; k++) up.push_back((uint8_t)rng());
            if (ul && up[up.size() - ul] == kFail) up[up.size() - ul] = 0;
            if (ul && rng() % 40 == 0) { up[up.size() - ul] = kFail; fails[i] = 1; }
            uo.push_back((uint32_t)up.size());
            ip[i] = rng(); port[i] = rng() & 0xFFFF;
        }
        const uint8_t* out = nullptr; size_t out_len = 0;
        // exact-size heap copies: a read past the end of any input array is an ASan report
        uint8_t* qh = (uint8_t*)malloc(q.size() + 1); if (!q.empty()) memcpy(qh, q.data(), q.size());
        uint8_t* uh = (uint8_t*)malloc(up.size() + 1); if (!up.empty()) memcpy(uh, up.data(), up.size());
        const int rc = bb_backend_relay(b, q.empty() ? nullptr : qh, qo.data(), up.empty() ? nullptr : uh, uo.data(), ip.data(),
                                        port.data(), n, &out, &out_len);
        size_t pos = 0; uint32_t n_frames = 0;
        while (pos < out_len) {
            if (pos + 16 > out_len || rd32(out + pos) != BB_FRAME_OUTBOUND_UDP) { printf("bad frame at %zu\n", pos); return 1; }
            const uint32_t fip = rd32(out + pos + 4), fport = rd32(out + pos + 8), ln = rd32(out + pos + 12);
            if (pos + 16 + ln > out_len) { printf("frame past the end\n"); return 1; }
            bool found = false;                        // the frame is some answered relay's query, addressed to its source
            for (uint32_t i = 0; i < n && !found; i++)
                found = ip[i] == fip && port[i] == fport && qo[i + 1] - qo[i] == ln && !memcmp(out + pos + 16, qh + qo[i], ln);
            if (!found) { printf("frame matches no relay\n"); return 1; }
            pos += 16 + ln; n_frames++;
        }
        const uint64_t relayed = bb_backend_stat(b, 6), failed = bb_backend_stat(b, 7);
        bool any_fail = false;
        for (uint32_t i = 0; i < n; i++) any_fail |= fails[i];
        if (relayed != n_frames || relayed + failed > n || (any_fail != (rc == BB_ERR_CUDA)) || (!any_fail && failed) ||
            (any_fail && !failed) || (rc != BB_OK && rc != BB_ERR_CUDA)) {
            printf("counts: rc %d relayed %llu failed %llu frames %u\n", rc, (unsigned long long)relayed, (unsigned long long)failed, n_frames);
            return 1;
        }
        // argument errors: decreasing offsets, null arrays
        if (n >= 2) {
            std::vector<uint32_t> bad = qo; std::swap(bad[0], bad[1]); bad[0] = bad[1] + 1;
            if (bb_backend_relay(b, qh, bad.data(), uh, uo.data(), ip.data(), port.data(), n, &out, &out_len) != BB_ERR_ARG) return 1;
            if (bb_backend_relay(b, qh, qo.data(), uh, uo.data(), nullptr, port.data(), n, &out, &out_len) != BB_ERR_ARG) return 1;
        }
        if (bb_backend_relay(nullptr, qh, qo.data(), uh, uo.data(), ip.data(), port.data(), n, &out, &out_len) != BB_ERR_ARG) return 1;
        free(qh); free(uh);
        bb_backend_destroy(b);
    }
    printf("OK\n");
    return 0;
}
