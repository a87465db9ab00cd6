// Link-time stand-ins for the engine calls the TCP hub (binder_b200/csrc/balancer_tcp.cpp) makes, so the hub's host
// code runs without a GPU: bb_resolve_batch_ex and bb_relay_batch call back into the test (tests/test_balancer_tcp.py),
// which answers with the CPU oracles.  Test infrastructure only.
#include "binder_b200.h"
#include <cstdlib>

typedef int (*bb_stub_resolve_fn)(const uint8_t*, const uint32_t*, uint32_t, uint64_t, uint32_t, uint8_t*, uint32_t, uint32_t*,
                                  uint16_t*, uint8_t*, uint32_t*, uint32_t*, uint32_t);
typedef int (*bb_stub_relay_fn)(const uint8_t*, const uint32_t*, const uint8_t*, const uint32_t*, uint32_t, uint32_t, uint8_t*,
                                uint32_t, uint32_t*, uint16_t*, uint8_t*);
static bb_stub_resolve_fn g_resolve = nullptr;
static bb_stub_relay_fn g_relay = nullptr;
static uint32_t g_max_batch = 1u << 16, g_max_bytes = 1u << 22;

extern "C" {
void bb_stub_set(bb_stub_resolve_fn resolve, bb_stub_relay_fn relay, uint32_t max_batch, uint32_t max_bytes) {
    g_resolve = resolve; g_relay = relay; g_max_batch = max_batch; g_max_bytes = max_bytes;
}
void* bb_host_alloc(size_t n) { return malloc(n ? n : 1); }
void bb_host_free(void* p) { free(p); }
uint32_t bb_engine_max_batch(const bb_engine*) { return g_max_batch; }
uint32_t bb_engine_max_batch_bytes(const bb_engine*) { return g_max_bytes; }
int bb_resolve_batch_ex(bb_engine*, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n, uint64_t seed, uint32_t qidx_base,
                        uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status, uint32_t* miss_idx,
                        uint32_t* n_miss, uint32_t flags) {
    if (!g_resolve) return BB_ERR_NO_DEVICE;
    return g_resolve(pkts, pkt_off, n, seed, qidx_base, out, out_cap, out_off, out_len, status, miss_idx, n_miss, flags);
}
int bb_relay_batch(bb_engine*, const uint8_t* q_pkts, const uint32_t* q_off, const uint8_t* up_pkts, const uint32_t* up_off, uint32_t n,
                   uint32_t flags, uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len, uint8_t* status) {
    if (!g_relay) return BB_ERR_NO_DEVICE;
    return g_relay(q_pkts, q_off, up_pkts, up_off, n, flags, out, out_cap, out_off, out_len, status);
}
}
