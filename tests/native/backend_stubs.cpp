// Link-time stand-in for bb_resolve_batch, so the balancer session's host code (csrc/balancer_frames.cpp,
// csrc/balancer_relay.cpp) runs on the CPU next to tests/native/tcp_hub_stubs.cpp: it forwards to that file's
// bb_resolve_batch_ex with flags 0 (the UDP path).  Test infrastructure only.
#include "binder_b200.h"

extern "C" int bb_resolve_batch(bb_engine* e, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n, uint64_t seed,
                                uint32_t qidx_base, uint8_t* out, uint32_t out_cap, uint32_t* out_off, uint16_t* out_len,
                                uint8_t* status, uint32_t* miss_idx, uint32_t* n_miss) {
    return bb_resolve_batch_ex(e, pkts, pkt_off, n, seed, qidx_base, out, out_cap, out_off, out_len, status, miss_idx, n_miss, 0);
}
