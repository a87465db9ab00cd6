// The query-log switches and record accessors of the balancer sessions (bb_backend: balancer_frames.cpp and
// balancer_relay.cpp; bb_tcp_hub: balancer_tcp.cpp; DESIGN.md section 15).  Switching the log on is what connects a
// session's record sets (bb_log_set, balancer_backend.h) to the engine's log kernel, bb_log_batch: the session sources
// call it only through that pointer, so they build and link without it.  Host code only.
#include "balancer_backend.h"

namespace {
// both record sets of a session, or neither
int set_both(bb_log_set* s, int enable) {
    int rc = s[0].set(enable, bb_log_batch);
    if (rc == BB_OK) rc = s[1].set(enable, bb_log_batch);
    if (rc != BB_OK) s[0].release();
    return rc;
}
}  // namespace

extern "C" {

int bb_query_log_backend_enable(bb_backend* b, int enable) {
    return b ? set_both(b->qlog, enable) : BB_ERR_ARG;
}

int bb_query_log_backend(const bb_backend* b, int which, bb_query_log_records* r) {
    if (!b || !r || which < 0 || which > 1) return BB_ERR_ARG;
    b->qlog[which].get(r, false);
    return BB_OK;
}

int bb_query_log_tcp_hub_enable(bb_tcp_hub* h, int enable) {
    return h ? set_both(tcp_hub_log_sets(h), enable) : BB_ERR_ARG;
}

int bb_query_log_tcp_hub(const bb_tcp_hub* h, int which, bb_query_log_records* r) {
    if (!h || !r || which < 0 || which > 1) return BB_ERR_ARG;
    tcp_hub_log_sets(const_cast<bb_tcp_hub*>(h))[which].get(r, true);
    return BB_OK;
}

}  // extern "C"
