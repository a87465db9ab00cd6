// The job count of a service answer, checked on the CPU: the device source (binder_b200/csrc/resolve_device.cuh, through
// tests/native/cuda_shim.h) sizes every query, and for each job-mode answer the count size_service() left in Res::ntask
// must equal a TaskCount walk of plan_service() over the same answer.  Built with -DBB_EMU_WALKS, it also counts the
// steps of the walks over a service's children (tests/test_service_jobs.py, tools/walk_counts.py).  Test
// infrastructure, not product.
#include "cuda_shim.h"
#include "../../binder_b200/csrc/zone_image.h"
#include "../../include/binder_b200.h"
namespace bbk { thread_local unsigned long long bb_emu_lean_count = 0, bb_emu_general_count = 0, bb_emu_walk_steps = 0; }
#include "../../binder_b200/csrc/resolve_device.cuh"

#include <vector>

thread_local uint8_t* bb_emu_smem = nullptr;
extern "C" const bb::ZoneImage* bb_zone_image(const bb_zone* z);

namespace {
using namespace bbk;
constexpr size_t OFF_IN = 16;                    // the staged tile (never 0: Res::sp == 0 means "not staged")
constexpr size_t OFF_SFX = OFF_IN + S_IN + 64;
constexpr size_t SMEM_BYTES = OFF_SFX + 256 + 64;

// The walks the kernel made over a job-mode answer's children before size_service() counted its jobs: the truncation
// walk over the answers, then — when they all fit — the one over the additionals, and a TaskCount walk of
// plan_service() whenever the count was not a build-time sum (truncated, or cut short by a malformed child).
uint32_t earlier_steps(const Res& r, const SvcView& sv, uint32_t fixed) {
    const bool srv = r.rk == RK_SVC_SRV;
    const uint32_t dol = dom_owner_len(r), dwl = dom_wire_len(r);
    uint32_t steps = 0;
    if (r.tc) {
        uint32_t total = fixed; bool full = false;
        uint64_t pm = r.perm;
        for (uint32_t t = 0; t < r.n_walk && !full; t++, pm >>= 4) {
            ++steps;
            const uint32_t inf = sv.info((uint32_t)pm & 15u), wl = (inf >> 8) & 0xFF, np = (inf >> 16) & 0xFF;
            if (inf & KID_ADDR_NULL) continue;
            const uint32_t each = srv ? 18 + wl + dwl : dol + 14, cnt = srv ? np : 1;
            uint32_t take = 0;
            while (take < cnt && total + each <= r.maxsz) { total += each; ++take; }
            if (take < cnt) full = true;
        }
        pm = r.perm;
        if (!full && srv) for (uint32_t t = 0; t < r.n_walk; t++, pm >>= 4) {
            ++steps;
            const uint32_t inf = sv.info((uint32_t)pm & 15u), wl = (inf >> 8) & 0xFF;
            if (inf & KID_ADDR_NULL) continue;
            if (total + wl + dol + 14 > r.maxsz) break;
            total += wl + dol + 14;
        }
    }
    return steps;
}
}  // namespace

// stats: [0] job-mode answers checked, [1] truncated SRV, [2] truncated A, [3] SRV runs cut inside a child (a job with a
// masked tail), [4] additionals cut (SRV, truncated, some additional kept), [5] with an OPT, [6] cut short by a malformed
// child, not truncated, [7] malformed child and truncated, [8] 16 children, [9] count mismatches, [10] first mismatching
// query (or ~0).
// steps (optional, n entries each): child-walk steps of each query now (sizing + one plan_service walk) and as the kernel
// made them before (see earlier_steps), for job-mode answers; 0 for every other query.
extern "C" int bb_emu_service_jobs(const bb_zone* zone, const char* dns_domain, const uint8_t* pkts, const uint32_t* pkt_off, uint32_t n,
                                   uint64_t seed, int tcp, unsigned long long* stats, uint32_t* steps_now, uint32_t* steps_before,
                                   uint8_t* is_srv) {
    static thread_local std::vector<uint8_t> smem(SMEM_BYTES + 1024);
    bb_emu_smem = (uint8_t*)(((uintptr_t)smem.data() + 1023) & ~(uintptr_t)1023);
    bb::EngineConst C;
    if (!bb::make_engine_const(dns_domain, false, C)) return BB_ERR_DOMAIN;
    const bb::ZoneImage* img = zone ? bb_zone_image(zone) : nullptr;
    if (!img) return BB_ERR_ARG;
    Params P; memset(&P, 0, sizeof P);
    P.pkts = pkts; P.pkt_off = pkt_off; P.n = n; P.seed = seed;
    P.table = img->slots; P.mask = img->nslots - 1; P.arena = img->arena;
    P.ready = img->ready; P.eng = &C; P.suffix_len = C.suffix_len; P.soa_len = C.soa_len; P.recursion = C.recursion; P.lean_ok = C.lean_ok;
    P.nranks = 1; P.tcp = tcp ? 1u : 0u;
    memcpy(bb_emu_smem + OFF_SFX, C.wire_tail, 256);
    for (int i = 0; i < 11; i++) stats[i] = 0;
    stats[10] = ~0ull;
    std::vector<Task> tl(TASKCAP);
    for (uint32_t q0 = 0; q0 < n; q0 += T) {
        const uint32_t nq = std::min<uint32_t>(T, n - q0);
        const uint32_t b0 = pkt_off[q0], b1 = pkt_off[q0 + nq], a0 = b0 & ~15u;
        const bool staged = b1 >= b0 && b1 - a0 <= (uint32_t)S_IN;
        if (staged) memcpy(bb_emu_smem + OFF_IN, pkts + a0, ((b1 - a0 + 15) >> 4) << 4);
        for (uint32_t t = 0; t < nq; t++) {
            const uint32_t q = q0 + t, o0 = pkt_off[q], o1 = pkt_off[q + 1];
            if (steps_now) { steps_now[q] = 0; steps_before[q] = 0; is_srv[q] = 0; }
            if (o1 < o0 || o1 - o0 > 65535u) continue;
            Res r; memset(&r, 0, sizeof r);
            r.status = ST_DROPPED; r.rk = RK_NONE;
            r.p = staged ? bb_emu_smem + OFF_IN + (o0 - a0) : pkts + o0;
            r.sp = staged ? (uint32_t)(OFF_IN + (o0 - a0)) : 0u;
            bb_emu_walk_steps = 0;
            resolve_query(P, r, o1 - o0, q, (uint32_t)OFF_SFX);
            const unsigned long long size_steps = bb_emu_walk_steps;
            if (steps_now) is_srv[q] = r.qtype == QT_SRV;
            if (!r.ntask) continue;
            const bool srv = r.rk == RK_SVC_SRV;
            TaskCount tc = { 0 };
            bb_emu_walk_steps = 0;
            plan_service(P, r, q, 0, 0, tc);
            const unsigned long long plan_steps = bb_emu_walk_steps;
            ++stats[0];
            if (r.ntask - 2 != tc.n) { if (!stats[9]++) stats[10] = q; continue; }
            TaskFill f = { tl.data() };
            if (tc.n > (uint32_t)TASKCAP) return BB_ERR_CAPACITY;
            plan_service(P, r, q, 0, 0, f);
            bool masked = false;
            for (uint32_t i = 0; i < tc.n; i++) masked |= task_exact(tl[i]);
            stats[1] += r.tc && srv; stats[2] += r.tc && !srv; stats[3] += masked; stats[4] += r.tc && srv && r.keep_add > 0;
            stats[5] += r.edns != 0; stats[6] += r.rcode == RC_SERVFAIL && !r.tc; stats[7] += r.rcode == RC_SERVFAIL && r.tc; stats[8] += r.nk == 16;
            if (steps_now) {
                SvcView sv; sv.open(P.arena, r.val);
                const uint32_t fixed = 12 + r.qn_len + 4 + (r.edns ? 11 : 0);
                const bool sums = !(sv.hflags() & (srv ? SVC_BAD_SRV : SVC_BAD_A));
                const uint32_t malformed_walk = sums ? 0u : min(r.n_walk + 1, r.nk);   // the same walk before and now
                steps_now[q] = (uint32_t)(size_steps + plan_steps);
                steps_before[q] = malformed_walk + earlier_steps(r, sv, fixed) + (uint32_t)plan_steps * ((!sums || r.tc) ? 2u : 1u);
            }
        }
    }
    return BB_OK;
}
