// Link-time stand-in for bb_log_batch, next to tests/native/tcp_hub_stubs.cpp and backend_stubs.cpp, so the balancer
// sessions' query log (binder_b200/csrc/balancer_query_log.cpp) runs without a GPU: the call goes back into the test
// (tests/test_balancer_query_log.py), which renders the records with the restatement.  Test infrastructure only.
#include "binder_b200.h"

typedef int (*bb_stub_log_fn)(const uint8_t*, uint32_t, const uint32_t*, const uint16_t*, const uint8_t*, uint32_t, uint8_t*, uint32_t,
                              uint32_t*, uint32_t*, uint16_t*);
static bb_stub_log_fn g_log = nullptr;

extern "C" {
void bb_stub_set_log(bb_stub_log_fn log) { g_log = log; }
int bb_log_batch(bb_engine*, const uint8_t* resp, uint32_t resp_bytes, const uint32_t* out_off, const uint16_t* out_len,
                 const uint8_t* status, uint32_t n, uint8_t* log, uint32_t log_cap, uint32_t* log_off, uint32_t* log_len,
                 uint16_t* head_len, uint32_t*) {
    if (!g_log) return BB_ERR_NO_DEVICE;
    return g_log(resp, resp_bytes, out_off, out_len, status, n, log, log_cap, log_off, log_len, head_len);
}
}
