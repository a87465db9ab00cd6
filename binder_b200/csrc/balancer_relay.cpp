// bb_backend_relay: a balancer UDP session's replies to its recursion misses.  The host's upstream exchange gives each
// miss its upstream response; bb_relay_batch (flags 0: the UDP path, its 512-byte / EDNS limits) builds the replies in
// batches of the session's max_batch, and bb_frames_build wraps each answered one in an OUTBOUND_UDP frame addressed
// to the miss's source.  Kept apart from balancer_frames.cpp, which needs no relay kernel.  Host code only.
#include "balancer_backend.h"

#include <algorithm>

extern "C" {

int bb_backend_relay(bb_backend* b, const uint8_t* q_pkts, const uint32_t* q_off, const uint8_t* up_pkts, const uint32_t* up_off,
                     const uint32_t* dst_ip, const uint32_t* dst_port, uint32_t n, const uint8_t** out, size_t* out_len) {
    if (!b || !out || !out_len) return BB_ERR_ARG;
    b->r_out.clear(); b->qlog[1].clear();
    *out = b->r_out.data(); *out_len = 0;
    if (n == 0) return BB_OK;
    if (!q_off || !up_off || !dst_ip || !dst_port || (q_off[n] != q_off[0] && !q_pkts) || (up_off[n] != up_off[0] && !up_pkts))
        return BB_ERR_ARG;
    for (uint32_t i = 0; i < n; i++) if (q_off[i + 1] < q_off[i] || up_off[i + 1] < up_off[i]) return BB_ERR_ARG;
    int rc = BB_OK;
    for (uint32_t k0 = 0; k0 < n; k0 += b->max_batch) {
        const uint32_t m = std::min(b->max_batch, n - k0);
        b->r_qoff.resize(m + 1); b->r_upoff.resize(m + 1);
        for (uint32_t j = 0; j <= m; j++) { b->r_qoff[j] = q_off[k0 + j] - q_off[k0]; b->r_upoff[j] = up_off[k0 + j] - up_off[k0]; }
        const int r = bb_relay_batch(b->e, q_pkts ? q_pkts + q_off[k0] : nullptr, b->r_qoff.data(), up_pkts ? up_pkts + up_off[k0] : nullptr,
                                     b->r_upoff.data(), m, 0u, b->resp, b->resp_cap, b->resp_off, b->resp_len, b->status);
        if (r != BB_OK) {                               // the batch's relays are lost (counted); the next batch still runs
            if (rc == BB_OK) rc = r;
            b->n_relay_failed += m;
            continue;
        }
        b->qlog[1].batch(b->e, b->resp, b->resp_off, b->resp_len, b->status, m, [&](uint32_t j, uint32_t& ip, uint32_t& port, uint32_t&) {
            ip = dst_ip[k0 + j]; port = dst_port[k0 + j]; return true;
        });
        size_t need = 0;
        bb_frames_build(b->resp, b->resp_off, b->resp_len, b->status, dst_ip + k0, dst_port + k0, m, nullptr, 0, nullptr, 0, &need);
        const size_t at = b->r_out.size();
        b->r_out.resize(at + need);
        if (need) bb_frames_build(b->resp, b->resp_off, b->resp_len, b->status, dst_ip + k0, dst_port + k0, m, nullptr, 0,
                                  b->r_out.data() + at, need, &need);
        for (uint32_t j = 0; j < m; j++) b->n_relayed += b->status[j] == BB_ANSWERED;
    }
    *out = b->r_out.data(); *out_len = b->r_out.size();
    return rc;
}

}  // extern "C"
