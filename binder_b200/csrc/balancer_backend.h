// One mname-balancer UDP session around an engine: the state bb_backend_feed (balancer_frames.cpp) and
// bb_backend_relay (balancer_relay.cpp) share.  Host code only.
#pragma once
#include "../../include/binder_b200.h"

#include <vector>

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
};
